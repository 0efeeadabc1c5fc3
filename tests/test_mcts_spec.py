"""CPU checks of the MCTS planner: the numpy statement of tests/mcts_spec.py (budget split, generator, descent,
expansion, backup, recommendation, subtree reuse) on hand-built trees, the committed reference fixtures replayed from
their own traces (and rerun over the live reference when it is present), and the new C-ABI entries and struct against
gcc."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from mcts_spec import (FIELDS, FIXTURES, GOLDEN, IDLE, M64, N_ACTIONS, advance, backup, budget_split, descend, draw,
                       empty_tree, expand, load, pick, plan, recommend, replay_callbacks, splitmix64)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_ENTRIES = ("hwy_mcts_advance", "hwy_mcts_backup", "hwy_mcts_recommend", "hwy_mcts_reroot")


def test_new_entries_are_exported():
    from highwayenv_b200 import _native as N

    lib = N.load()
    for sym in NEW_ENTRIES:
        assert sym in N.EXPORTS
        assert getattr(lib, sym) is not None
    assert lib.hwy_abi_version() == N.HWY_ABI_VERSION == 17


def test_tree_struct_matches_gcc():
    from highwayenv_b200 import _native as N

    names = ("temperature", "seed", "discount", "decision", "count", "prior", "walk_flags", "remap", "recommended")
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "hwyb200.h"\nint main(){printf("%zu'
           + ' %zu' * len(names) + '\\n", sizeof(HwyMctsTree)'
           + "".join(f", offsetof(HwyMctsTree, {n})" for n in names) + ');return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [C.sizeof(N.HwyMctsTree)] + [getattr(N.HwyMctsTree, n).offset for n in names]


# ------------------------------------------------------------------------------------------- budget
@pytest.mark.parametrize("budget,gamma,split", [(100, 0.7, (20, 5)), (50, 0.7, (12, 4)), (1, 0.7, (1, 1)),
                                                (2, 0.7, (2, 1)), (23, 0.5, (11, 2)), (200, 0.9, (15, 13))])
def test_budget_split(budget, gamma, split):
    from highwayenv_b200.planning import mcts_budget

    assert budget_split(budget, gamma) == split == mcts_budget(budget, gamma)
    e, h = split
    assert e * h <= budget


def test_budget_split_matches_the_library_and_is_the_largest():
    from highwayenv_b200.planning import mcts_budget
    from mcts_spec import horizon_of

    for gamma in (0.3, 0.5, 0.7, 0.9, 0.95):
        for budget in range(1, 400, 7):
            e, h = budget_split(budget, gamma)
            assert (e, h) == mcts_budget(budget, gamma)
            assert e * h <= budget < (e + 1) * horizon_of(e + 1, gamma)


@pytest.mark.parametrize("budget,gamma", [(0, 0.7), (-5, 0.7), (2.5, 0.7), (100, 0.0), (100, 1.0), (100, -0.1)])
def test_budget_rejections(budget, gamma):
    from highwayenv_b200.planning import mcts_budget

    with pytest.raises(ValueError):
        budget_split(budget, gamma)
    with pytest.raises(ValueError):
        mcts_budget(budget, gamma)


# ------------------------------------------------------------------------------------------- generator
def test_generator_words():
    assert splitmix64(GOLDEN) == 0xE220A8397B1DCDAF  # SplitMix64's first output from state 0
    assert draw(0, 0, 0, 0, 0, 0) == 0xCBD37AD29B93B094
    assert draw(12345, 1, 2, 3, 4, 1) == 0xD249A8E7EE60B191
    assert draw(12345, 1, 2, 3, 4, 0) != draw(12345, 1, 2, 3, 4, 1)
    assert draw(-1, 0, 0, 0, 0, 0) == draw(M64, 0, 0, 0, 0, 0)
    for k in range(1, 6):
        assert pick(0, k) == 0 and pick(M64, k) == k - 1
        # floor(u * k) computed exactly, where the rounded product (1 - 2**-53) * 5 would give 5
        assert pick(((1 << 53) - 1) << 11, k) == k - 1
    counts = np.bincount([pick(draw(7, 0, r, 0, 0, 1), 5) for r in range(5000)], minlength=5)
    assert counts.min() > 900


# ------------------------------------------------------------------------------------------- hand-built trees
def _root_expanded(avail=(True,) * 5, max_nodes=11):
    tree = empty_tree(1, max_nodes)
    assert expand(tree, 0, 0, avail)
    return tree


def test_expansion_layout():
    tree = _root_expanded([False, True, True, False, True])
    assert tree["n_nodes"][0] == 6 and tree["expanded"][0, 0] and tree["child_base"][0, 0] == 1
    assert tree["n_children"][0, 0] == 3
    assert np.array_equal(tree["exists"][0, 1:6], [False, True, True, False, True])
    assert np.array_equal(tree["parent"][0, 1:6], [0] * 5) and np.array_equal(tree["action"][0, 1:6], range(5))
    assert np.array_equal(tree["prior"][0, 1:6], [0.0, 1 / 3, 1 / 3, 0.0, 1 / 3])


def test_descent_ties_are_broken_by_the_draw():
    tree = _root_expanded()
    for x in (0, 1 << 62, 0xCBD37AD29B93B094, M64):
        c, a, margin = descend(tree, 0, 0, 1.0, x)
        assert a == pick(x, 5) and c == 1 + a
        assert margin == np.inf  # unvisited pairs only
    # one visited child: value 0.25 + 1 / 2 < 1 (the unvisited ones), so only the 4 unvisited ones tie
    backup(tree, 0, 1 + 2, 0.25)
    c, a, margin = descend(tree, 0, 0, 1.0, M64)
    assert a == 4 and margin == 1.0 - 0.75
    c, a, _ = descend(tree, 0, 0, 1.0, 0)
    assert a == 0
    # a visited child whose score ties with the unvisited ones: the draw picks among all five
    tree["value"][0, 3] = 0.5
    _, a, margin = descend(tree, 0, 0, 1.0, M64)
    assert a == 4 and margin == 0.0


def test_backup_is_the_running_mean():
    tree = _root_expanded()
    for ret in (1.0, 0.5, 0.3):
        backup(tree, 0, 2, ret)
    assert tree["count"][0, 2] == tree["count"][0, 0] == 3
    v = 0.0
    for k, ret in enumerate((1.0, 0.5, 0.3), 1):
        v = v + (1.0 / k) * (ret - v)
    assert tree["value"][0, 2] == tree["value"][0, 0] == v


def _scripted(n, rewards, dones, avail=None):
    """Callbacks whose step k returns rewards[k], dones[k] for every root (lists of per-step rows)."""
    calls = {"k": 0, "actions": []}

    def begin():
        pass

    def available():
        return np.ones((n, N_ACTIONS), bool) if avail is None else np.asarray(avail)

    def step(actions):
        k = calls["k"]
        calls["k"] += 1
        calls["actions"].append(np.array(actions))
        return np.full(n, rewards[k]), np.full(n, dones[k])

    return (begin, available, step), calls


def test_done_stops_the_rollout_and_later_steps_are_idle():
    tree = empty_tree(1, 11)
    cbs, calls = _scripted(1, [0.5, 9.0, 9.0], [True, False, False])
    out = plan(tree, 1, 3, 0.5, 1.0, 3, 0, *cbs)
    assert tree["expanded"][0, 0] and tree["n_nodes"][0] == 6  # expanded at depth 0, then the rollout ended
    assert out["leaf"][0, 0] == 0 and out["ret"][0, 0] == 0.5
    assert calls["actions"][0][0] == pick(draw(3, 0, 0, 0, 0, 1), 5)
    assert calls["actions"][1][0] == calls["actions"][2][0] == IDLE
    assert tree["count"][0, 0] == 1 and tree["value"][0, 0] == 0.5 and tree["count"][0, 1:].sum() == 0


def test_done_during_descent_skips_expansion_and_rollout():
    tree = _root_expanded()
    cbs, calls = _scripted(1, [1.0, 9.0, 9.0], [True, False, False])
    out = plan(tree, 1, 3, 0.5, 1.0, 0, 0, *cbs)
    leaf = out["leaf"][0, 0]
    assert leaf == 1 + calls["actions"][0][0] and not tree["expanded"][0, leaf] and tree["n_nodes"][0] == 6
    assert out["ret"][0, 0] == 1.0 and tree["count"][0, leaf] == 1


def test_descent_stops_at_the_horizon_without_expanding():
    tree = _root_expanded()
    cbs, calls = _scripted(1, [1.0], [False])
    out = plan(tree, 1, 1, 0.5, 1.0, 0, 0, *cbs)
    leaf = out["leaf"][0, 0]
    assert leaf >= 1 and not tree["expanded"][0, leaf] and tree["n_nodes"][0] == 6 and tree["skipped"][0] == 0
    assert out["ret"][0, 0] == 1.0


def test_a_full_tree_skips_the_expansion_and_rolls_out():
    tree = empty_tree(1, 6)
    cbs, calls = _scripted(1, [0.25] * 6, [False] * 6)
    out = plan(tree, 3, 2, 0.5, 1.0, 0, 0, *cbs)
    assert tree["n_nodes"][0] == 6 and tree["skipped"][0] == 2  # episodes 1 and 2 reach an unexpanded child
    assert (out["leaf"][0, 1:] >= 1).all() and not tree["expanded"][0, 1:].any()
    assert np.all(out["ret"][0] == 0.25 + 0.5 * 0.25)
    assert tree["count"][0, 0] == 3


def test_recommendation_takes_counts_then_values_then_the_lowest_action():
    tree = _root_expanded([True, True, True, False, True])
    tree["count"][0, 1:6] = [3, 5, 5, 0, 2]
    tree["value"][0, 1:6] = [9.0, 0.5, 0.7, 0.0, 9.0]
    assert recommend(tree, 0) == (2, pytest.approx(0.2))
    tree["value"][0, 3] = 0.5
    assert recommend(tree, 0) == (1, 0.0)


def _random_callbacks(n, seed, p_done=0.1):
    rng = np.random.default_rng(seed)

    def available():
        a = rng.random((n, N_ACTIONS)) < 0.7
        a[:, IDLE] = True
        a[3, 0] = False  # root 3 never has LANE_LEFT
        return a

    def step(actions):
        return rng.random(n), rng.random(n) < p_done

    return (lambda: None), available, step


def _check_compaction(before, after, i, c):
    """The subtree of old node c of root i, in old index order, equals the new tree's slots 0.. ."""
    m = before["exists"].shape[1]
    kept = [c]
    for j in range(c + 1, m):
        if before["parent"][i, j] in kept:
            kept.append(j)
    new = {j: k for k, j in enumerate(kept)}
    assert after["n_nodes"][i] == len(kept)
    for j, k in new.items():
        for f in ("exists", "expanded", "action", "n_children", "prior", "count", "value"):
            assert after[f][i, k] == before[f][i, j], (f, j, k)
        assert after["parent"][i, k] == (-1 if j == c else new[before["parent"][i, j]])
        cb = before["child_base"][i, j]
        assert after["child_base"][i, k] == (-1 if cb < 0 else new[cb])
        if after["expanded"][i, k]:  # the 5 slots stay together
            b = after["child_base"][i, k]
            assert np.array_equal(after["parent"][i, b:b + 5], [k] * 5)
            assert np.array_equal(after["action"][i, b:b + 5], range(5))
    assert not after["exists"][i, len(kept):].any() and (after["parent"][i, len(kept):] == -1).all()


def test_advance_keeps_the_subtree_compacted_and_clears_otherwise():
    n = 6
    tree = empty_tree(n, 1 + 5 * 40)
    plan(tree, 20, 4, 0.8, 1.0, 5, 0, *_random_callbacks(n, 1, p_done=0.05))
    before = {k: v.copy() for k, v in tree.items()}
    base = tree["child_base"][:, 0].copy()
    existing = [recommend(tree, i)[0] for i in range(n)]
    missing = [int(a) for a in np.nonzero(~tree["exists"][3, base[3]:base[3] + 5])[0]]
    assert missing, "root 3 needs an unavailable action"
    actions = np.array(existing[:3] + [missing[0], existing[4], 7])
    done = np.array([False, False, False, False, True, False])
    advance(tree, actions, done)
    for i in range(3):
        _check_compaction(before, tree, i, int(base[i] + actions[i]))
        assert tree["count"][i, 0] == before["count"][i, base[i] + actions[i]] > 0
    for i in (3, 4, 5):  # a missing child, done, an action out of range
        assert tree["n_nodes"][i] == 1 and tree["exists"][i].sum() == 1 and tree["count"][i, 0] == 0
        assert tree["prior"][i, 0] == 1.0 and not tree["expanded"][i, 0]
    # the re-rooted trees plan on: a later decision keeps the counts and grows the tree
    out = plan(tree, 20, 4, 0.8, 1.0, 5, 1, *_random_callbacks(n, 2, p_done=0.05))
    assert (tree["count"][:3, 0] == before["count"][np.arange(3), base[:3] + actions[:3]] + 20).all()
    assert (out["recommended"] >= 0).all()


# ------------------------------------------------------------------------------------------- fixtures
@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_trees_replay_from_their_own_traces(name):
    """The spec, fed the available actions, rewards and flags the reference produced, builds the fixture's trees
    bit for bit, taking the same actions at every step."""
    g = load(name)
    cfg = g["config"]
    n, M = g["tree"]["exists"].shape
    assert n == 32 and cfg["_budget"] == 100 and cfg["_gamma"] == 0.7 and cfg["_temperature"] == 1.0
    episodes, horizon = budget_split(cfg["_budget"], cfg["_gamma"])
    assert M == 1 + N_ACTIONS * episodes and g["trace"]["action"].shape == (n, episodes, horizon)
    tree = empty_tree(n, M)
    out = plan(tree, episodes, horizon, cfg["_gamma"], cfg["_temperature"], cfg["_seed"], 0,
               *replay_callbacks(g["trace"]))
    for k in FIELDS + ("n_nodes", "skipped"):
        assert tree[k].tobytes() == g["tree"][k].tobytes(), (name, k)
    for k in out:
        assert np.asarray(out[k]).tobytes() == np.asarray(g["out"][k]).tobytes(), (name, k)
    base = g["tree"]["child_base"][:, 0]
    assert all(np.array_equal(g["available"][i], g["tree"]["exists"][i, base[i]:base[i] + 5]) for i in range(n))
    assert (g["tree"]["skipped"] == 0).all()


@pytest.mark.parametrize("name", FIXTURES)
def test_spec_over_the_live_reference_reproduces_the_fixture(name):
    import ref_harness as rh

    if not rh.reference_available():
        pytest.skip("the reference checkout is not present")
    from gen_mcts import CASES, run

    g = load(name)
    env_id, over, seeds = CASES[name]
    env = rh.make_reference_env(env_id, over)
    env.reset(seed=seeds[0])  # record 0: the reset state of the first seed, root 0
    tree, out, _ = run([env])
    for k in FIELDS + ("n_nodes", "skipped"):
        assert tree[k][0].tobytes() == g["tree"][k][0].tobytes(), (name, k)
    for k in out:
        assert np.asarray(out[k])[0].tobytes() == np.asarray(g["out"][k])[0].tobytes(), (name, k)
