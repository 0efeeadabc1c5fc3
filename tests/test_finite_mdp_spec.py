"""CPU checks of the finite-MDP planner: the new C-ABI entries and structs, and the numpy specification of
tests/finite_mdp_spec.py against the reference's own `to_finite_mdp()` on every fixture state."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from finite_mdp_spec import FIXTURES, load, mdp_from_grid, random_mdps, value_iteration

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_planner_entries_are_exported():
    from highwayenv_b200 import _native as N

    lib = N.load()
    for sym in ("hwy_finite_mdp", "hwy_value_iteration"):
        assert sym in N.EXPORTS
        assert getattr(lib, sym) is not None
    assert lib.hwy_abi_version() == N.HWY_ABI_VERSION == 15


def test_planner_structs_match_gcc():
    from highwayenv_b200 import _native as N

    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "hwyb200.h"\nint main(){printf("%zu %zu %zu %zu %zu\\n", '
           'sizeof(HwyFiniteMdpParams), sizeof(HwyValueIterationParams), offsetof(HwyFiniteMdpParams, collision_reward), '
           'offsetof(HwyValueIterationParams, gamma), offsetof(HwyValueIterationParams, action));return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", exe])
        sizes = [int(x) for x in subprocess.check_output([exe]).split()]
    assert sizes == [C.sizeof(N.HwyFiniteMdpParams), C.sizeof(N.HwyValueIterationParams),
                     N.HwyFiniteMdpParams.collision_reward.offset, N.HwyValueIterationParams.gamma.offset,
                     N.HwyValueIterationParams.action.offset]


@pytest.mark.parametrize("name", FIXTURES)
def test_spec_equals_the_reference_mdp_on_every_fixture_state(name):
    """The numpy statement the kernel follows, fed the reference's grid, gives the reference's MDP bit for bit."""
    g = load(name)
    cfg = g["config"]
    for k in range(g["mdp_grid"].shape[0]):
        L = int(g["mdp_n_lanes"][k])
        grid = g["mdp_grid"][k][:, :L]
        V, _, T = grid.shape
        S = V * L * T
        assert T == int(10.0 / (1 / cfg["policy_frequency"]))
        transition, reward, terminal = mdp_from_grid(grid, cfg)
        assert np.array_equal(transition, g["mdp_transition"][k, :S].astype(np.int64)), (name, k)
        assert np.array_equal(reward.view(np.uint64), g["mdp_reward"][k, :S].view(np.uint64)), (name, k)
        assert np.array_equal(terminal, g["mdp_terminal"][k, :S]), (name, k)
        # the padding rows of the fixture follow the batched layout
        s_max = g["mdp_reward"].shape[1]
        assert np.array_equal(g["mdp_transition"][k, S:], np.tile(np.arange(S, s_max)[:, None], (1, 5)))
        assert not g["mdp_reward"][k, S:].any() and g["mdp_terminal"][k, S:].all()
        assert not g["mdp_grid"][k][:, L:].any()
    assert g["mdp_grid"].shape[0] == 36


def test_fixtures_cover_the_shapes_the_issue_names():
    shapes = {name: load(name)["mdp_grid"].shape[1:] for name in FIXTURES}
    assert shapes["finite_mdp_highway"] == (3, 4, 10)
    assert shapes["finite_mdp_highway_fast_pf2"][2] == 20
    assert shapes["finite_mdp_highway_5lanes"][1] == 5
    # at least one fixture has collision cells (grid == 1) and hence terminal rows before the horizon
    assert any((load(name)["mdp_grid"] == 1).any() for name in FIXTURES)


def test_value_iteration_spec_basics():
    # a chain 0 -> 1 -> 2 (terminal) with reward 1 per step: Q converges to the steps-to-go
    transition = np.array([[1, 1], [2, 2], [2, 2]])
    reward = np.ones((3, 2))
    terminal = np.array([False, False, True])
    q, done = value_iteration(transition, reward, terminal, 1.0, 100)
    assert done == 3 and np.array_equal(q[:, 0], [3.0, 2.0, 1.0])
    q0, d0 = value_iteration(transition, reward, terminal, 1.0, 0)
    assert d0 == 0 and not q0.any()
    q1, d1 = value_iteration(transition, reward, terminal, 1.0, 2)
    assert d1 == 2 and np.array_equal(q1[:, 0], [2.0, 2.0, 1.0])
    rng = np.random.default_rng(0)
    t, r, term, ns = random_mdps(rng, 4, 50, 4)
    assert ns.min() >= 1 and ns.max() <= 50 and (t >= 0).all()
