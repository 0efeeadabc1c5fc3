"""The numpy statement of open-loop Monte-Carlo tree search that `highwayenv_b200.planning.MctsPolicy` follows:
rl-agents' `MCTSAgent` (`tree_search/mcts.py`) with the `random_available` prior and rollout policies, `closed_loop:
False`, written over any way of stepping a state.  rl-agents is not part of the reference, so every rule is stated here.

Budget.  `budget_split(budget, gamma)` restates rl-agents' `AbstractPlanner.allocate_budget`:
    horizon(E) = max(ceil(ln E / (2 ln(1 / gamma))), 1)
    episodes   = the largest E >= 1 with E * horizon(E) <= budget;   horizon = horizon(episodes)
gamma must lie in (0, 1); a budget with no split (budget < 1) raises ValueError.  100 at 0.7 is 20 x 5, 50 is 12 x 4.

Tree.  Per root, M = 1 + 5 * max_expansions slots; node 0 is the root.  Expanding node p takes the 5 consecutive slots
`child_base[p] + a` (a = LANE_LEFT, IDLE, LANE_RIGHT, FASTER, SLOWER) at `n_nodes`, all with `parent = p`, `action = a`;
`exists` only for the actions available in the state reached at p, whose `prior` is `1.0 / n_children[p]` (float64).
Parents precede their children in index order.  Fields per slot (FIELDS): exists, expanded (has children), parent,
action, child_base, n_children, prior, count (visits), value; an empty slot is (0, 0, -1, -1, -1, 0, 0.0, 0, 0.0) and a
bare root is an empty slot with exists = 1 and prior = 1.0.  Per root: `n_nodes` (slots in use) and `skipped`.

Episode e of root i, from a fresh copy of the root state, node = 0, depth = 0, ret = 0, done = False:
  1. descent: while depth < H, node is expanded and not done: score every existing child c of node as
         value[c] + ((T * n_children[node]) * prior[c]) / (count[c] + 1)
     (in that order of operations), take the maximum — exact ties broken by a draw among them — step with its action,
     `ret += g[depth] * r`, `done = terminated | truncated`, node = that child, depth += 1;
  2. expansion: if node is not expanded, depth < H and not done, expand node over the available actions of the
     current state — unless fewer than 5 slots are free: then `skipped[i] += 1` and node stays a leaf;
  3. rollout: if not done, for h = depth .. H - 1: a uniformly drawn available action, step, `ret += g[h] * r`, stop
     at done;
  4. backup: from node up to the root, `count += 1; value += (1.0 / count) * (ret - value)` (rl-agents' K = 1).
g[h] = gamma ** h comes from the float64 table `discount_table`.  The recommended action is the root child with the
largest count, ties by the largest value, then the lowest action (rl-agents' `selection_rule`).

Randomness.  `draw(seed, decision, root, episode, depth, purpose)` chains the SplitMix64 finaliser over the six words
(purpose 0: a descent tie-break, 1: a rollout action); of k candidates in ascending action order it picks
`((x >> 11) * k) >> 53`, i.e. floor(u * k) for u = (x >> 11) * 2**-53, computed exactly.  `decision` counts the
planner's decisions (the library keeps it on the device).

Subtree reuse (rl-agents' `step_strategy: "subtree"`), `advance(tree, actions, done)`: a root with done[i], or
without an existing child for actions[i], is cleared to a bare root; otherwise that child becomes node 0 with its
count, value and other fields kept and parent = -1, and its subtree is compacted to the front in stable index order
(the 5 slots of every kept expansion stay consecutive).

Deviations from rl-agents:
  * rl-agents seeds the copied state at every episode (`state.seed(...)`).  This statement does not: on the supported
    ids (highway, roundabout, merge, exit) `step` draws nothing from the env's stream — the reference reads
    `np_random` only while spawning at reset, in `randomize_behavior`, and in the shuffled Kinematics order, which is
    not the default — so the seed could not change any outcome.
  * `done = terminated | truncated` in the descent and in the rollout.
  * draws come from the counter-based generator above instead of the planner's `np_random`.
  * the capacity bound (and `skipped`) is new; rl-agents' tree grows without bound.

`plan(tree, ...)` plans n roots in lockstep through three callbacks: `begin_episode()` copies every root's state into
its work state, `available()` returns `[n, 5] bool` for the work states and `step(actions [n])` steps every work
state, returning `(reward [n], done [n])`.  A root whose episode has ended still gets a step (action IDLE) whose
results are ignored.  It also records, per root and episode, the backed-up `leaf`, the return `ret` and the `margin`:
the smallest gap between a chosen descent score and any other candidate's, over the episode's descent, leaving out
pairs of unvisited children (their scores are equal by construction); inf when there was no other candidate.
"""
from __future__ import annotations

import math

import numpy as np

N_ACTIONS = 5
IDLE = 1
FIELDS = ("exists", "expanded", "parent", "action", "child_base", "n_children", "prior", "count", "value")
M64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15


def horizon_of(episodes: int, gamma: float) -> int:
    return max(int(math.ceil(np.log(np.float64(episodes)) / (2 * np.log(1 / np.float64(gamma))))), 1)


def budget_split(budget: int, gamma: float):
    """(episodes, horizon) of a budget, see the module docstring."""
    if not 0.0 < gamma < 1.0:
        raise ValueError("gamma must be in (0, 1)")
    if int(budget) != budget or budget < 1:
        raise ValueError(f"budget {budget} has no split into episodes x horizon")
    e = 1
    while (e + 1) * horizon_of(e + 1, gamma) <= budget:
        e += 1
    return e, horizon_of(e, gamma)


def discount_table(gamma: float, horizon: int) -> np.ndarray:
    return np.float64(gamma) ** np.arange(horizon, dtype=np.float64)


def splitmix64(z: int) -> int:
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def draw(seed: int, decision: int, root: int, episode: int, depth: int, purpose: int) -> int:
    x = 0
    for w in (seed, decision, root, episode, depth, purpose):
        x = splitmix64((x + GOLDEN + (int(w) & M64)) & M64)
    return x


def pick(x: int, k: int) -> int:
    return ((x >> 11) * k) >> 53


def empty_tree(n: int, max_nodes: int) -> dict:
    tree = {"exists": np.zeros((n, max_nodes), bool), "expanded": np.zeros((n, max_nodes), bool),
            "parent": np.full((n, max_nodes), -1, np.int32), "action": np.full((n, max_nodes), -1, np.int32),
            "child_base": np.full((n, max_nodes), -1, np.int32), "n_children": np.zeros((n, max_nodes), np.int32),
            "prior": np.zeros((n, max_nodes)), "count": np.zeros((n, max_nodes), np.int32),
            "value": np.zeros((n, max_nodes)), "n_nodes": np.zeros(n, np.int32), "skipped": np.zeros(n, np.int32)}
    for i in range(n):
        clear(tree, i)
    return tree


def clear(tree: dict, i: int, start: int = 0) -> None:
    """Empty slots start.. of root i; start = 0 leaves a bare root."""
    for k, v in (("exists", False), ("expanded", False), ("parent", -1), ("action", -1), ("child_base", -1),
                 ("n_children", 0), ("prior", 0.0), ("count", 0), ("value", 0.0)):
        tree[k][i, start:] = v
    if start == 0:
        tree["exists"][i, 0], tree["prior"][i, 0], tree["n_nodes"][i] = True, 1.0, 1


def expand(tree: dict, i: int, p: int, available) -> bool:
    base = int(tree["n_nodes"][i])
    if base + N_ACTIONS > tree["exists"].shape[1]:
        tree["skipped"][i] += 1
        return False
    avail = np.asarray(available, bool)
    k = int(avail.sum())
    assert k >= 1, "every state has an available action (IDLE always is)"
    tree["n_nodes"][i] = base + N_ACTIONS
    tree["expanded"][i, p], tree["child_base"][i, p], tree["n_children"][i, p] = True, base, k
    for a in range(N_ACTIONS):
        c = base + a
        tree["parent"][i, c], tree["action"][i, c], tree["exists"][i, c] = p, a, avail[a]
        tree["prior"][i, c] = 1.0 / k if avail[a] else 0.0
    return True


def descend(tree: dict, i: int, p: int, temperature: float, x: int):
    """(chosen child, its action, margin) at the expanded node p of root i; x is the tie-break draw."""
    base, n = int(tree["child_base"][i, p]), int(tree["n_children"][i, p])
    cand = [a for a in range(N_ACTIONS) if tree["exists"][i, base + a]]
    score = {}
    for a in cand:
        c = base + a
        score[a] = float(tree["value"][i, c]) + ((temperature * n) * float(tree["prior"][i, c])) / (
            int(tree["count"][i, c]) + 1)
    best = max(score.values())
    ties = [a for a in cand if score[a] == best]
    a = ties[pick(x, len(ties))]
    unvisited = lambda b: tree["count"][i, base + b] == 0  # noqa: E731
    gaps = [best - score[b] for b in cand if b != a and not (unvisited(a) and unvisited(b))]
    return base + a, a, min(gaps, default=np.inf)


def rollout_action(available, x: int) -> int:
    acts = [a for a in range(N_ACTIONS) if available[a]]
    return acts[pick(x, len(acts))]


def backup(tree: dict, i: int, node: int, ret: float) -> None:
    c = node
    while c >= 0:
        tree["count"][i, c] += 1
        v = float(tree["value"][i, c])
        tree["value"][i, c] = v + (1.0 / int(tree["count"][i, c])) * (ret - v)
        c = int(tree["parent"][i, c])


def recommend(tree: dict, i: int):
    """(root child action with the largest count, ties by value then lowest action; its value margin over a root
    child of equal count, inf when the count alone decides)."""
    if not tree["expanded"][i, 0]:
        return -1, np.inf
    base = int(tree["child_base"][i, 0])
    cand = [a for a in range(N_ACTIONS) if tree["exists"][i, base + a]]
    top = max(int(tree["count"][i, base + a]) for a in cand)
    tied = [a for a in cand if tree["count"][i, base + a] == top]
    vals = {a: float(tree["value"][i, base + a]) for a in tied}
    best = max(tied, key=lambda a: vals[a])  # max(): the first maximum, the lowest action
    return best, min((vals[best] - vals[a] for a in tied if a != best), default=np.inf)


def plan(tree: dict, episodes: int, horizon: int, gamma: float, temperature: float, seed: int, decision: int,
         begin_episode, available, step) -> dict:
    """Run `episodes` episodes on every root of `tree` (updated in place); returns `leaf`, `ret`, `margin` [n, E],
    `recommended` and `recommended_margin` [n]."""
    n = tree["exists"].shape[0]
    g = discount_table(gamma, horizon)
    out = {"leaf": np.zeros((n, episodes), np.int32), "ret": np.zeros((n, episodes)),
           "margin": np.full((n, episodes), np.inf)}
    tree["skipped"][:] = 0
    for e in range(episodes):
        begin_episode()
        node, ret = np.zeros(n, np.int64), np.zeros(n)
        done, rolling = np.zeros(n, bool), np.zeros(n, bool)
        for d in range(horizon):
            avail = np.asarray(available(), bool)
            actions = np.full(n, IDLE, np.int64)
            for i in range(n):
                if done[i]:
                    continue
                if not rolling[i]:
                    if tree["expanded"][i, node[i]]:
                        node[i], actions[i], m = descend(tree, i, int(node[i]), temperature,
                                                         draw(seed, decision, i, e, d, 0))
                        out["margin"][i, e] = min(out["margin"][i, e], m)
                        continue
                    expand(tree, i, int(node[i]), avail[i])
                    rolling[i] = True
                actions[i] = rollout_action(avail[i], draw(seed, decision, i, e, d, 1))
            reward, dn = step(actions)
            for i in range(n):
                if not done[i]:
                    ret[i] = ret[i] + g[d] * float(reward[i])
                    done[i] = bool(dn[i])
        for i in range(n):
            backup(tree, i, int(node[i]), float(ret[i]))
        out["leaf"][:, e], out["ret"][:, e] = node, ret
    rec = [recommend(tree, i) for i in range(n)]
    out["recommended"] = np.array([a for a, _ in rec], np.int64)
    out["recommended_margin"] = np.array([m for _, m in rec])
    return out


def advance(tree: dict, actions, done) -> None:
    """Subtree reuse: re-root every tree at its child for actions[i] (see the module docstring)."""
    m = tree["exists"].shape[1]
    for i in range(tree["exists"].shape[0]):
        a = int(actions[i])
        c = -1
        if not done[i] and tree["expanded"][i, 0] and 0 <= a < N_ACTIONS:
            c = int(tree["child_base"][i, 0]) + a
            if not tree["exists"][i, c]:
                c = -1
        if c < 0:
            clear(tree, i)
            continue
        new = np.full(m, -1, np.int64)
        new[c], k = 0, 1
        for j in range(c + 1, m):
            p = int(tree["parent"][i, j])
            if p >= 0 and new[p] >= 0:
                new[j], k = k, k + 1
        for j in range(c, m):  # new[j] <= j: in place, ascending
            if new[j] < 0:
                continue
            for f in FIELDS:
                tree[f][i, new[j]] = tree[f][i, j]
            p, cb = int(tree["parent"][i, j]), int(tree["child_base"][i, j])
            tree["parent"][i, new[j]] = -1 if j == c else new[p]
            tree["child_base"][i, new[j]] = -1 if cb < 0 else new[cb]
        clear(tree, i, k)
        tree["n_nodes"][i] = k


# ---------------------------------------------------------------------------------------------- callbacks
def reference_callbacks(roots, copy, step, available_actions):
    """Callbacks over per-root state objects (e.g. reference envs): `copy(state)` clones a state, `step(state, a)` ->
    (reward, terminated, truncated), `available_actions(state)` -> list of actions."""
    work = []

    def begin_episode():
        work[:] = [copy(r) for r in roots]

    def available():
        out = np.zeros((len(roots), N_ACTIONS), bool)
        for i, s in enumerate(work):
            out[i, available_actions(s)] = True
        return out

    def step_all(actions):
        res = [step(s, int(a)) for s, a in zip(work, actions)]
        return np.array([r for r, _, _ in res]), np.array([bool(te or tr) for _, te, tr in res])

    return begin_episode, available, step_all


def recording(begin_episode, available, step):
    """Wrap callbacks to record what they returned: `trace` gets `available` [n, E, H, 5], `action`, `reward` and
    `done` [n, E, H] once the plan has run (see `replay_callbacks`)."""
    trace = {"available": [], "action": [], "reward": [], "done": []}

    def begin():
        for k in trace:
            trace[k].append([])
        begin_episode()

    def avail():
        a = np.asarray(available(), bool)
        trace["available"][-1].append(a)
        return a

    def st(actions):
        r, d = step(actions)
        trace["action"][-1].append(np.asarray(actions, np.int64))
        trace["reward"][-1].append(np.asarray(r, np.float64))
        trace["done"][-1].append(np.asarray(d, bool))
        return r, d

    def stacked():
        return {k: np.moveaxis(np.asarray(v), 2, 0) for k, v in trace.items()}

    return (begin, avail, st), stacked


def replay_callbacks(trace: dict):
    """Callbacks that replay a recorded trace; a step whose actions differ from the recorded ones fails."""
    pos = {"e": -1, "d": 0}

    def begin_episode():
        pos["e"], pos["d"] = pos["e"] + 1, 0

    def available():
        return trace["available"][:, pos["e"], pos["d"]]

    def step(actions):
        e, d = pos["e"], pos["d"]
        assert np.array_equal(actions, trace["action"][:, e, d]), (e, d)
        pos["d"] += 1
        return trace["reward"][:, e, d], trace["done"][:, e, d]

    return begin_episode, available, step


def load(name: str) -> dict:
    """tests/golden/<name>.npz of oracle/gen_mcts.py: `tree` (FIELDS, n_nodes, skipped), `out` (leaf, ret, margin,
    recommended, recommended_margin) and `trace` (available, action, reward, done)."""
    from parity_utils import load_golden

    g = load_golden(name)
    for part in ("tree", "out", "trace"):
        g[part] = {k[len(part) + 1:]: g[k] for k in list(g) if k.startswith(part + "_")}
    return g


FIXTURES = ["mcts_highway_fast", "mcts_highway", "mcts_roundabout", "mcts_merge"]
