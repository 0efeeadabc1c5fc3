"""`planning.OpdPolicy`: optimistic deterministic planning over env clones (`copy_envs` + `step`, tree kernels in
csrc/hwy_plan.cu), against the numpy statement of tests/opd_spec.py — run over the unmodified reference (fixtures
opd_*.npz, `copy.deepcopy` + `step`) and over this library's own `copy_envs` + `step` — and the network families'
`get_available_actions()` against the reference's on the fixture states."""
import numpy as np
import pytest

from obs_plugin_utils import env_state_dict, kinds
from opd_spec import FIELDS, FIXTURES, N_ACTIONS, load, opd

pytestmark = pytest.mark.gpu

MARGIN = 1e-9  # selections and recommendations closer than this are ties up to rounding: not compared
VALUE_TOL = 1e-6  # rewards accumulated over up to 10 free-running steps (positions agree to 1e-5)
TREE_EXACT = ("exists", "expanded", "parent", "action", "depth", "terminal")


def make_from_fixture(g, **kw):
    """The fixture's root states, loaded into one env each."""
    import highwayenv_b200 as hb

    env = hb.make(g["config"]["_env_id"], num_envs=g["x"].shape[0], config=dict(g["config"]["_override"]),
                  autoreset_mode="Disabled", **kw)
    env.reset(seed=0)
    sd = env_state_dict(g)
    if g["config"]["_env_id"].startswith("highway"):
        hsd = {k: sd[k] for k in ("x", "y", "heading", "speed", "target_speed", "timer", "delta", "impact_x",
                                  "impact_y", "lane", "target_lane", "crashed", "has_impact", "check_collisions",
                                  "speed_index", "time")}
        hsd["kind"] = kinds(g)
        env.load_state_dict(hsd)
    else:
        for k in ("count", "road_steps", "is_yielding"):
            sd.pop(k)
        env.load_state_dict(sd)
    env.observe()
    return env


def host_tree(policy):
    t = {k: getattr(policy.tree, k).cpu().numpy() for k in FIELDS}
    t["selected"] = policy.selected.cpu().numpy()
    t["recommended"] = policy.actions.cpu().numpy()
    return t


@pytest.mark.parametrize("name", FIXTURES)
def test_available_actions_equal_the_reference(name):
    g = load(name)
    env = make_from_fixture(g)
    got = env.get_available_actions().cpu().numpy()
    assert np.array_equal(got, g["tree"]["available"]), name
    assert np.array_equal(env._available_actions().cpu().numpy(), got)  # the kernel the planner uses


@pytest.mark.parametrize("name", FIXTURES)
def test_opd_trees_equal_the_reference(name):
    from highwayenv_b200 import planning

    g = load(name)
    ref = g["tree"]
    env = make_from_fixture(g)
    policy = planning.OpdPolicy(env, budget=g["config"]["_budget"], gamma=g["config"]["_gamma"])
    policy.act()
    got = host_tree(policy)
    n, E = ref["selected"].shape
    compared_recs, worst = 0, 0.0
    for i in range(n):
        # the trees are comparable up to the first selection whose runner-up lies within rounding of it
        close = np.nonzero(ref["margin"][i] < MARGIN)[0]
        k_star = int(close[0]) if close.size else E
        assert np.array_equal(got["selected"][i, :k_star], ref["selected"][i, :k_star]), (name, i)
        last = 1 + N_ACTIONS * k_star
        for k in TREE_EXACT:
            assert np.array_equal(got[k][i, :last], ref[k][i, :last]), (name, i, k)
        live = ref["exists"][i, :last]
        for k in ("reward", "value", "upper"):
            d = np.abs(got[k][i, :last] - ref[k][i, :last])[live]
            worst = max(worst, float(d.max(initial=0.0)))
            assert d.max(initial=0.0) <= VALUE_TOL, (name, i, k, d.max())
        if k_star == E and ref["recommended_margin"][i] >= MARGIN:
            assert got["recommended"][i] == ref["recommended"][i], (name, i)
            compared_recs += 1
    print(f"{name}: recommended action compared on {compared_recs} of {n} roots "
          f"({n - compared_recs} excluded by a margin below {MARGIN}); worst value difference {worst:.3g}")
    assert compared_recs >= n // 2


def library_expander(env, n_roots, expansions):
    """The spec's `expand` over this library: a store env with a row per node, a work env with 5 rows per root, and
    the public `copy_envs`, `get_available_actions` and `step`."""
    import highwayenv_b200 as hb
    import torch

    M = 1 + N_ACTIONS * expansions
    store = hb.make(env.ENV_ID, num_envs=n_roots * M, config=dict(env.config), autoreset_mode="Disabled")
    work = hb.make(env.ENV_ID, num_envs=n_roots * N_ACTIONS, config=dict(env.config), autoreset_mode="Disabled")
    store.copy_envs(np.arange(n_roots) * M, np.arange(n_roots), source=env)
    roots = np.arange(n_roots)

    def expand(k, leaves):
        leaf = roots * M + np.where(leaves < 0, 0, leaves)
        work.copy_envs(np.arange(n_roots * N_ACTIONS), np.repeat(leaf, N_ACTIONS), source=store)
        avail = work.get_available_actions().cpu().numpy()[::N_ACTIONS]
        _, r, te, tr, _ = work.step(torch.arange(N_ACTIONS, dtype=torch.int32, device="cuda").repeat(n_roots))
        store.copy_envs((roots[:, None] * M + 1 + N_ACTIONS * k + np.arange(N_ACTIONS)).reshape(-1),
                        np.arange(n_roots * N_ACTIONS), source=work)
        shape = (n_roots, N_ACTIONS)
        return avail, r.cpu().numpy().reshape(shape), (te | tr).cpu().numpy().reshape(shape)

    return expand


@pytest.mark.parametrize("env_id,config", [("highway-fast-v0", None), ("roundabout-v0", None),
                                           ("highway-v0", {"other_vehicles_type":
                                                           "highway_env.vehicle.behavior.LinearVehicle"})])
def test_opd_equals_the_spec_over_the_library(env_id, config):
    import highwayenv_b200 as hb
    from highwayenv_b200 import planning

    n = 64
    env = hb.make(env_id, num_envs=n, config=dict(config or {}))
    env.reset(seed=77)
    rng = np.random.default_rng(0)
    for _ in range(3):
        env.step(rng.integers(0, N_ACTIONS, size=n).astype(np.int32))
    policy = planning.OpdPolicy(env, budget=50, gamma=0.7)
    policy.act()
    got = host_tree(policy)
    want = opd(n, 50, 0.7, library_expander(env, n, 10))
    for k in FIELDS + ("selected", "recommended"):
        assert np.ascontiguousarray(got[k]).tobytes() == np.ascontiguousarray(
            want[k].astype(got[k].dtype)).tobytes(), (env_id, k)
    # a different budget and gamma, including a budget that is not a multiple of 5
    policy = planning.OpdPolicy(env, budget=23, gamma=0.5)
    policy.act()
    got = host_tree(policy)
    want = opd(n, 23, 0.5, library_expander(env, n, 4))
    for k in FIELDS + ("selected", "recommended"):
        assert np.ascontiguousarray(got[k]).tobytes() == np.ascontiguousarray(
            want[k].astype(got[k].dtype)).tobytes(), (env_id, k)


def test_second_act_does_not_sync_and_replays_in_a_cuda_graph():
    import highwayenv_b200 as hb
    import torch
    from highwayenv_b200 import planning

    env = hb.make("highway-fast-v0", num_envs=128)
    env.reset(seed=3)
    policy = planning.OpdPolicy(env)
    policy.act()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        policy.act()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        policy.act()
    for _ in range(3):
        env.step(policy.actions.clone())
        graph.replay()
        torch.cuda.synchronize()
        replayed = {k: getattr(policy.tree, k).clone() for k in FIELDS}
        replayed_actions = policy.actions.clone()
        policy.act()
        torch.cuda.synchronize()
        assert torch.equal(replayed_actions, policy.actions)
        for k in FIELDS:
            assert torch.equal(replayed[k], getattr(policy.tree, k)), k


@pytest.mark.parametrize("env_id,config,budget,gamma,error", [
    ("intersection-multi-agent-v0", None, 50, 0.7, NotImplementedError),
    ("intersection-v0", None, 50, 0.7, NotImplementedError),
    ("two-way-v0", None, 50, 0.7, NotImplementedError),
    ("highway-fast-v0", {"action": {"type": "ContinuousAction"}}, 50, 0.7, ValueError),
    ("highway-fast-v0", None, 50, 1.0, ValueError),
    ("highway-fast-v0", None, 50, -0.1, ValueError),
    ("highway-fast-v0", None, 4, 0.7, ValueError),
])
def test_rejected_configurations(env_id, config, budget, gamma, error):
    import highwayenv_b200 as hb
    from highwayenv_b200 import planning

    env = hb.make(env_id, num_envs=2, config=dict(config or {}))
    with pytest.raises(error):
        planning.OpdPolicy(env, budget=budget, gamma=gamma)
