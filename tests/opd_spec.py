"""The numpy statement of optimistic deterministic planning (OPD, Hren & Munos 2008) that
`highwayenv_b200.planning.OpdPolicy` follows: the planner rl-agents' `DeterministicPlannerAgent` runs in the reference's
quickstart (docs/quickstart.md, `budget: 50, gamma: 0.7`), written over any way of expanding a state.

A tree per root holds `M = 1 + 5 E` nodes with `E = budget // 5` expansions; node 0 is the root (depth 0, value 0, not
terminal).  Expansion k selects, per root, the open leaf (exists, not expanded, not terminal) with the largest `upper`,
the lowest node on ties, and creates one child per available action `a` of the leaf's state at node `1 + 5 k + a`:

    depth = p.depth + 1
    value = p.value + g[p.depth] * r                   r: the reward of stepping the leaf's state with `a`
    terminal = terminated | truncated
    upper = value if terminal else value + t[depth]

with g[d] = gamma ** d and t[d] = gamma ** d / (1 - gamma) from `discount_tables`.  A root without an open leaf skips
the expansion.  The recommended action is the root child whose subtree holds the largest `value`, the lowest action
on ties.  Documented deviations from rl-agents: ties are broken by index instead of at random; rewards are not
checked to lie in [0, 1] (the bound t[d] assumes r <= 1); the tree is rebuilt at every decision (no subtree reuse).

`opd(n, budget, gamma, expand)` plans for n roots in lockstep.  `expand(k, leaves)` gets the selected node of every
root (-1: none) and returns `(available [n, 5] bool, reward [n, 5], done [n, 5] bool)` for the children it made of the
leaves' states; it stores the child of root i and action a as node `1 + 5 k + a` for the next calls.
"""
from __future__ import annotations

import numpy as np

N_ACTIONS = 5
FIELDS = ("exists", "expanded", "parent", "action", "depth", "reward", "value", "upper", "terminal")


def discount_tables(gamma: float, expansions: int):
    """(g, t) float64 [expansions + 2]: g[d] = gamma ** d, t[d] = g[d] / (1 - gamma)."""
    g = np.float64(gamma) ** np.arange(expansions + 2, dtype=np.float64)
    return g, g / (np.float64(1.0) - np.float64(gamma))


def empty_tree(n: int, expansions: int, gamma: float) -> dict:
    m = 1 + N_ACTIONS * expansions
    _, t = discount_tables(gamma, expansions)
    tree = {"exists": np.zeros((n, m), bool), "expanded": np.zeros((n, m), bool),
            "parent": np.full((n, m), -1, np.int32), "action": np.full((n, m), -1, np.int32),
            "depth": np.zeros((n, m), np.int32), "reward": np.zeros((n, m)), "value": np.zeros((n, m)),
            "upper": np.zeros((n, m)), "terminal": np.zeros((n, m), bool),
            "selected": np.full((n, expansions), -1, np.int32), "margin": np.full((n, expansions), np.inf)}
    tree["exists"][:, 0] = True
    tree["upper"][:, 0] = t[0]
    return tree


def select(tree: dict, i: int):
    """(open leaf of root i with the largest upper, the lowest node on ties; its margin over the runner-up) or (-1, inf)."""
    open_ = tree["exists"][i] & ~tree["expanded"][i] & ~tree["terminal"][i]
    nodes = np.nonzero(open_)[0]
    if nodes.size == 0:
        return -1, np.inf
    u = tree["upper"][i, nodes]
    best = int(nodes[np.argmax(u)])  # np.argmax: the first maximum, i.e. the lowest node
    rest = np.delete(u, np.argmax(u))
    return best, float(u.max() - rest.max()) if rest.size else np.inf


def record(tree: dict, k: int, i: int, p: int, available, reward, done, g, t) -> None:
    tree["expanded"][i, p] = True
    d = int(tree["depth"][i, p])
    for a in range(N_ACTIONS):
        if not available[a]:
            continue
        c = 1 + N_ACTIONS * k + a
        v = tree["value"][i, p] + g[d] * np.float64(reward[a])
        tree["exists"][i, c], tree["parent"][i, c], tree["action"][i, c] = True, p, a
        tree["depth"][i, c], tree["reward"][i, c], tree["value"][i, c] = d + 1, reward[a], v
        tree["terminal"][i, c] = bool(done[a])
        tree["upper"][i, c] = v if done[a] else v + t[d + 1]


def branch_values(tree: dict, i: int) -> np.ndarray:
    """[5]: the largest value in the subtree of each root child (-inf where the child does not exist)."""
    best = np.full(N_ACTIONS, -np.inf)
    m = tree["exists"].shape[1]
    branch = np.full(m, -1)
    for c in range(1, m):
        if not tree["exists"][i, c]:
            continue
        p = tree["parent"][i, c]
        branch[c] = tree["action"][i, c] if p == 0 else branch[p]  # parents precede their children
        best[branch[c]] = max(best[branch[c]], tree["value"][i, c])
    return best


def recommend(tree: dict, i: int):
    """(recommended action of root i, its margin over the runner-up root child)."""
    best = branch_values(tree, i)
    a = int(np.argmax(best))
    rest = np.delete(best, a)
    rest = rest[np.isfinite(rest)]
    return a, float(best[a] - rest.max()) if rest.size else np.inf


def opd(n: int, budget: int, gamma: float, expand) -> dict:
    """Plan for n roots; returns the tree fields [n, M], `selected` / `margin` [n, E] (the expanded node of every
    expansion and its upper-bound margin over the runner-up open leaf), `recommended` and `recommended_margin` [n]."""
    if not 0 <= gamma < 1:
        raise ValueError("gamma must be in [0, 1)")
    if budget < N_ACTIONS:
        raise ValueError("budget must be >= 5")
    expansions = budget // N_ACTIONS
    g, t = discount_tables(gamma, expansions)
    tree = empty_tree(n, expansions, gamma)
    for k in range(expansions):
        leaves = np.full(n, -1, np.int64)
        for i in range(n):
            leaves[i], tree["margin"][i, k] = select(tree, i)
        tree["selected"][:, k] = leaves
        available, reward, done = expand(k, leaves)
        for i in range(n):
            if leaves[i] >= 0:
                record(tree, k, i, int(leaves[i]), available[i], reward[i], done[i], g, t)
    rec = [recommend(tree, i) for i in range(n)]
    tree["recommended"] = np.array([a for a, _ in rec], np.int64)
    tree["recommended_margin"] = np.array([m for _, m in rec])
    return tree


def reference_expander(envs, copy, step, available_actions):
    """An `expand` over per-root state objects (e.g. reference envs): `copy(state)` clones a state, `step(state, a)`
    -> (reward, terminated, truncated), `available_actions(state)` -> list of actions.  The root states are envs[i]."""
    states = [{0: e} for e in envs]

    def expand(k, leaves):
        n = len(envs)
        available = np.zeros((n, N_ACTIONS), bool)
        reward, done = np.zeros((n, N_ACTIONS)), np.zeros((n, N_ACTIONS), bool)
        for i, p in enumerate(leaves):
            if p < 0:
                continue
            leaf = states[i][int(p)]
            for a in available_actions(leaf):
                child = copy(leaf)
                r, term, trunc = step(child, a)
                available[i, a], reward[i, a], done[i, a] = True, r, bool(term or trunc)
                states[i][1 + N_ACTIONS * k + a] = child
        return available, reward, done

    return expand


def replay_expander(tree: dict):
    """An `expand` that replays the children recorded in a tree (fields [n, M]): reproduces the selections and values
    of that tree from its rewards, terminal flags and available actions alone."""

    def expand(k, leaves):
        n = len(leaves)
        c = 1 + N_ACTIONS * k + np.arange(N_ACTIONS)
        available = np.zeros((n, N_ACTIONS), bool)
        reward, done = np.zeros((n, N_ACTIONS)), np.zeros((n, N_ACTIONS), bool)
        for i, p in enumerate(leaves):
            if p >= 0:
                available[i] = tree["exists"][i, c]
                reward[i], done[i] = tree["reward"][i, c], tree["terminal"][i, c]
        return available, reward, done

    return expand


def load(name: str) -> dict:
    """tests/golden/<name>.npz of oracle/gen_opd.py with the tree fields under their spec names."""
    from parity_utils import load_golden

    g = load_golden(name)
    g["tree"] = {k[4:]: g[k] for k in list(g) if k.startswith("opd_")}
    return g


FIXTURES = ["opd_highway_fast", "opd_highway", "opd_roundabout", "opd_merge"]
