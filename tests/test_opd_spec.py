"""CPU checks of the OPD planner: the numpy statement of tests/opd_spec.py on hand-built trees and against the
committed reference fixtures (rerun over the live reference when it is present), and the new C-ABI entries and
structs against gcc."""
import copy
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from opd_spec import (FIXTURES, FIELDS, N_ACTIONS, discount_tables, empty_tree, load, opd, recommend, record,
                      reference_expander, replay_expander, select)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_ENTRIES = ("hwy_copy_env_rows", "hwy_available_actions", "hwy_opd_select", "hwy_opd_record", "hwy_opd_recommend")


def test_new_entries_are_exported():
    from highwayenv_b200 import _native as N

    lib = N.load()
    for sym in NEW_ENTRIES:
        assert sym in N.EXPORTS
        assert getattr(lib, sym) is not None
    assert lib.hwy_abi_version() == N.HWY_ABI_VERSION


def test_new_structs_match_gcc():
    from highwayenv_b200 import _native as N

    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "hwyb200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu '
           '%d\\n", sizeof(HwyRowCopy), offsetof(HwyRowCopy, row_bytes), sizeof(HwyOpdTree), '
           'offsetof(HwyOpdTree, discount), offsetof(HwyOpdTree, branch), offsetof(HwyOpdTree, upper), '
           'offsetof(HwyOpdTree, recommended), HWY_COPY_MAX_BUFS);return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [C.sizeof(N.HwyRowCopy), N.HwyRowCopy.row_bytes.offset, C.sizeof(N.HwyOpdTree),
                   N.HwyOpdTree.discount.offset, N.HwyOpdTree.branch.offset, N.HwyOpdTree.upper.offset,
                   N.HwyOpdTree.recommended.offset, N.HWY_COPY_MAX_BUFS]


def test_discount_tables_match_the_library():
    from highwayenv_b200.planning import opd_discount_tables

    for gamma, e in ((0.7, 10), (0.0, 1), (0.95, 30)):
        for a, b in zip(discount_tables(gamma, e), opd_discount_tables(gamma, e)):
            assert a.tobytes() == b.tobytes()
    g, t = discount_tables(0.5, 3)
    assert np.array_equal(g, [1, 0.5, 0.25, 0.125, 0.0625]) and np.array_equal(t, 2 * g)


def _tree(n_exp=3, gamma=0.5):
    return empty_tree(1, n_exp, gamma), discount_tables(gamma, n_exp)


def test_selection_takes_the_largest_upper_and_the_lowest_node_on_ties():
    tree, (g, t) = _tree()
    assert select(tree, 0) == (0, np.inf)  # only the root is open
    record(tree, 0, 0, 0, [True] * 5, [0.5, 1.0, 1.0, 0.2, 0.0], [False] * 5, g, t)
    assert tree["expanded"][0, 0] and np.array_equal(tree["depth"][0, 1:6], [1] * 5)
    assert np.array_equal(tree["value"][0, 1:6], [0.5, 1.0, 1.0, 0.2, 0.0])
    assert np.array_equal(tree["upper"][0, 1:6], np.array([0.5, 1.0, 1.0, 0.2, 0.0]) + t[1])
    leaf, margin = select(tree, 0)
    assert leaf == 2 and margin == 0.0  # nodes 2 and 3 tie: the lower one
    # a terminal child keeps upper = value and is never selected
    record(tree, 1, 0, 2, [True, True, False, False, True], [1.0, 0.0, 0, 0, 1.0], [True, False, False, False, False],
           g, t)
    assert tree["terminal"][0, 6] and tree["upper"][0, 6] == tree["value"][0, 6] == 1.0 + g[1] * 1.0
    assert not tree["exists"][0, 8] and not tree["exists"][0, 9]
    assert tree["value"][0, 10] == 1.0 + 0.5 * 1.0 and tree["upper"][0, 10] == 1.5 + t[2]
    leaf, margin = select(tree, 0)
    assert leaf == 3  # upper 1 + t[1] = 2.0 ties with node 10 (1.5 + t[2] = 2.0): the lower node
    assert margin == 0.0
    a, m = recommend(tree, 0)
    assert a == 1 and m == 0.5  # node 2 is action 1's child: its subtree holds 1.5 (terminal node 6); action 2's 1.0


def test_recommendation_ties_go_to_the_lowest_action_and_closed_roots_skip():
    def expand(k, leaves):
        n = len(leaves)
        return np.ones((n, 5), bool), np.ones((n, 5)), np.ones((n, 5), bool)  # every child terminal, equal rewards

    tree = opd(3, 20, 0.7, expand)
    assert np.array_equal(tree["selected"][:, 0], [0, 0, 0]) and (tree["selected"][:, 1:] == -1).all()
    assert np.array_equal(tree["recommended"], [0, 0, 0]) and (tree["recommended_margin"] == 0).all()
    assert tree["exists"][:, :6].all() and not tree["exists"][:, 6:].any()


def test_rejected_arguments():
    with pytest.raises(ValueError):
        opd(1, 50, 1.0, None)
    with pytest.raises(ValueError):
        opd(1, 4, 0.7, None)


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_trees_replay_from_their_own_rewards(name):
    """The spec, expanding with the rewards / flags / available actions the reference produced, builds the fixture's
    tree bit for bit: selections, values, bounds and the recommended action."""
    g = load(name)
    ref = g["tree"]
    n = ref["exists"].shape[0]
    assert n == 32 and g["config"]["_budget"] == 50 and g["config"]["_gamma"] == 0.7
    got = opd(n, 50, 0.7, replay_expander(ref))
    for k in FIELDS + ("selected", "margin", "recommended", "recommended_margin"):
        assert np.asarray(got[k]).tobytes() == np.asarray(ref[k]).tobytes(), (name, k)
    # the root's available actions are exactly its children
    assert np.array_equal(ref["available"], ref["exists"][:, 1:1 + N_ACTIONS])
    assert (ref["available"][:, 1]).all()


@pytest.mark.parametrize("name", FIXTURES)
def test_spec_over_the_live_reference_reproduces_the_fixture(name):
    import ref_harness as rh

    if not rh.reference_available():
        pytest.skip("the reference checkout is not present")
    from gen_opd import BUDGET, CASES, GAMMA, _step

    g = load(name)
    env_id, over, seeds = CASES[name]
    env = rh.make_reference_env(env_id, over)
    env.reset(seed=seeds[0])  # record 0: the reset state of the first seed
    expand = reference_expander([env], lambda e: copy.deepcopy(e.unwrapped), _step,
                                lambda e: e.unwrapped.get_available_actions())
    got = opd(1, BUDGET, GAMMA, expand)
    for k in FIELDS + ("selected", "margin", "recommended", "recommended_margin"):
        assert np.asarray(got[k])[0].tobytes() == np.asarray(g["tree"][k][0]).tobytes(), (name, k)
