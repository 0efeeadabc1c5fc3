"""The batched finite MDP (`env.to_finite_mdp()`, csrc/hwy_observe.cu finite_mdp_kernel), batched value iteration
(`planning.value_iteration`, csrc/hwy_plan.cu) and `planning.TtcValueIterationPolicy`.  States of reference rollouts
are injected and the MDP is compared with the reference's own `to_finite_mdp()` of that state (fixtures
finite_mdp_*.npz); the solver is compared with the numpy statement of tests/finite_mdp_spec.py, bit for bit."""
from types import SimpleNamespace

import numpy as np
import pytest

from finite_mdp_spec import FIXTURES, load, random_mdps, value_iteration_batch
from obs_plugin_utils import env_state_dict, kinds

pytestmark = pytest.mark.gpu


def make_env(g, **kw):
    import highwayenv_b200 as hb

    return hb.make(g["config"]["_env_id"], num_envs=g["x"].shape[0], config=dict(g["config"]["_override"]),
                   autoreset_mode="Disabled", **kw)


def inject(env, g, rows=None):
    sd = env_state_dict(g)
    if rows is not None:
        sd = {k: np.asarray(v)[rows] for k, v in sd.items()}
    if g["config"]["_env_id"].startswith("highway"):
        hsd = {k: sd[k] for k in ("x", "y", "heading", "speed", "target_speed", "timer", "delta", "impact_x",
                                  "impact_y", "lane", "target_lane", "crashed", "has_impact", "check_collisions",
                                  "speed_index", "time")}
        hsd["kind"] = kinds(g) if rows is None else kinds(g)[rows]
        env.load_state_dict(hsd)
    else:
        for k in ("count", "road_steps", "is_yielding"):
            sd.pop(k)
        env.load_state_dict(sd)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64) if a.dtype == np.float64 else a


def fixture_tensors(g, device="cuda"):
    import torch

    V, LM, T = g["mdp_grid"].shape[1:]
    return SimpleNamespace(
        transition=torch.from_numpy(g["mdp_transition"].astype(np.int32)).to(device),
        reward=torch.from_numpy(g["mdp_reward"]).to(device),
        terminal=torch.from_numpy(g["mdp_terminal"]).to(device),
        n_states=torch.from_numpy((V * g["mdp_n_lanes"] * T).astype(np.int32)).to(device))


@pytest.mark.parametrize("name", FIXTURES)
def test_finite_mdp_equals_the_reference(name):
    g = load(name)
    env = make_env(g)
    env.reset(seed=0)
    inject(env, g)
    mdp = env.to_finite_mdp()
    assert tuple(mdp.grid.shape[1:]) == g["mdp_grid"].shape[1:], name
    V, LM, T = g["mdp_grid"].shape[1:]
    assert np.array_equal(bits(mdp.grid.cpu().numpy()), bits(g["mdp_grid"])), name
    assert np.array_equal(mdp.n_lanes.cpu().numpy(), g["mdp_n_lanes"])
    assert np.array_equal(mdp.n_states.cpu().numpy(), V * g["mdp_n_lanes"] * T)
    assert np.array_equal(mdp.state.cpu().numpy(), g["mdp_state"])
    # the fixture is padded as the batched layout pads: rows past n_states are self-loops, reward 0, terminal
    assert np.array_equal(mdp.transition.cpu().numpy(), g["mdp_transition"]), name
    assert np.array_equal(bits(mdp.reward.cpu().numpy()), bits(g["mdp_reward"])), name
    assert np.array_equal(mdp.terminal.cpu().numpy(), g["mdp_terminal"]), name
    assert mdp.transition.dtype.itemsize == 4 and mdp.state.dtype.itemsize == 8


@pytest.mark.parametrize("name", FIXTURES)
def test_value_iteration_on_the_fixture_mdps(name):
    from highwayenv_b200 import planning

    g = load(name)
    m = fixture_tensors(g)
    n_states = m.n_states.cpu().numpy()
    for gamma in (1.0, 0.9, 0.5):
        for iterations in (0, 1, 3, 100):
            q, done = planning.value_iteration(m, gamma=gamma, iterations=iterations)
            want_q, want_done = value_iteration_batch(g["mdp_transition"], g["mdp_reward"], g["mdp_terminal"],
                                                      n_states, gamma, iterations)
            assert np.array_equal(done.cpu().numpy(), want_done), (name, gamma, iterations)
            assert np.array_equal(bits(q.cpu().numpy()), bits(want_q)), (name, gamma, iterations)


@pytest.mark.parametrize("s_max,a,n", [(300, 5, 64), (97, 3, 33), (4096, 8, 3)])
def test_value_iteration_on_random_mdps(s_max, a, n):
    """Ragged n_states, rewards on a coarse grid (ties everywhere), undiscounted cycles that never converge (the
    iteration cap) and discounted ones that do."""
    import torch

    from highwayenv_b200 import planning

    rng = np.random.default_rng(s_max + a)
    t, r, term, ns = random_mdps(rng, n, s_max, a)
    m = SimpleNamespace(transition=torch.from_numpy(t).cuda(), reward=torch.from_numpy(r).cuda(),
                        terminal=torch.from_numpy(term).cuda(), n_states=torch.from_numpy(ns).cuda())
    capped = False
    for gamma, iterations in ((1.0, 40), (0.9, 100), (0.5, 7), (0.0, 5)):
        q, done = planning.value_iteration(m, gamma=gamma, iterations=iterations)
        want_q, want_done = value_iteration_batch(t, r, term, ns, gamma, iterations)
        assert np.array_equal(done.cpu().numpy(), want_done), (gamma, iterations)
        assert np.array_equal(bits(q.cpu().numpy()), bits(want_q)), (gamma, iterations)
        capped = capped or bool((want_done == iterations).any())
    assert capped


def test_out_of_range_successor_fails_only_its_env():
    import torch

    from highwayenv_b200 import planning

    rng = np.random.default_rng(3)
    t, r, term, ns = random_mdps(rng, 6, 120, 5)
    ok_q, ok_done = value_iteration_batch(t, r, term, ns, 0.9, 50)
    t_bad = t.copy()
    t_bad[2, int(ns[2]) - 1, 4] = int(ns[2])  # one past the env's own rows
    t_bad[4, 0, 0] = -1
    ns_bad = ns.copy()
    ns_bad[5] = 121  # more states than rows
    m = SimpleNamespace(transition=torch.from_numpy(t_bad).cuda(), reward=torch.from_numpy(r).cuda(),
                        terminal=torch.from_numpy(term).cuda(), n_states=torch.from_numpy(ns_bad).cuda())
    q, done = planning.value_iteration(m, gamma=0.9, iterations=50)
    q, done = q.cpu().numpy(), done.cpu().numpy()
    for e in (2, 4, 5):
        assert done[e] == -1 and not q[e].any()
    for e in (0, 1, 3):
        assert done[e] == ok_done[e] and np.array_equal(bits(q[e]), bits(ok_q[e]))


def _rollout_env(n=256, seed=7):
    import highwayenv_b200 as hb

    env = hb.make("highway-v0", num_envs=n, config={"vehicles_count": 30})
    env.reset(seed=seed)
    rng = np.random.default_rng(seed)
    for _ in range(3):
        env.step(rng.integers(0, 5, size=n).astype(np.int32))
    return env


def _numpy_actions(mdp, gamma, iterations):
    tr, rw, te = mdp.transition.cpu().numpy(), mdp.reward.cpu().numpy(), mdp.terminal.cpu().numpy()
    q, _ = value_iteration_batch(tr, rw, te, mdp.n_states.cpu().numpy(), gamma, iterations)
    st = mdp.state.cpu().numpy()
    return np.array([np.argmax(q[e, st[e]]) for e in range(len(st))], dtype=np.int64), q


@pytest.mark.parametrize("env_id", ["highway-v0", "roundabout-v0"])
def test_policy_act_is_the_numpy_argmax(env_id):
    import highwayenv_b200 as hb
    from highwayenv_b200 import planning

    env = _rollout_env() if env_id == "highway-v0" else hb.make(env_id, num_envs=128)
    if env_id != "highway-v0":
        env.reset(seed=11)
    policy = planning.TtcValueIterationPolicy(env, gamma=0.95, iterations=60)
    act = policy.act()
    assert act.dtype.itemsize == 8 and act.device.type == "cuda" and tuple(act.shape) == (env.num_envs,)
    want, want_q = _numpy_actions(env.to_finite_mdp(), 0.95, 60)
    assert np.array_equal(act.cpu().numpy(), want)
    assert np.array_equal(bits(policy.q.cpu().numpy()), bits(want_q))
    env.step(act)


def test_second_act_does_not_sync_and_replays_in_a_cuda_graph():
    import torch

    from highwayenv_b200 import planning

    env = _rollout_env(n=512, seed=5)
    policy = planning.TtcValueIterationPolicy(env)
    policy.act()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        act = policy.act()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    want, _ = _numpy_actions(env.to_finite_mdp(), 1.0, 100)
    assert np.array_equal(act.cpu().numpy(), want)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        policy.act()
    for _ in range(2):
        env.step(policy.actions.clone())
        graph.replay()
        torch.cuda.synchronize()
        replayed, replayed_q = policy.actions.clone(), policy.q.clone()
        eager = policy.act().clone()
        assert np.array_equal(replayed.cpu().numpy(), eager.cpu().numpy())
        assert torch.equal(replayed_q, policy.q)


def test_single_env_to_finite_mdp_is_the_reference_object():
    import highwayenv_b200 as hb

    g = load("finite_mdp_roundabout")
    k = 13
    single = hb.make_single(g["config"]["_env_id"], config=dict(g["config"]["_override"]))
    single.reset(seed=0)
    inject(single.batched, g, rows=[k])
    mdp = single.unwrapped.to_finite_mdp()
    V, _, T = g["mdp_grid"].shape[1:]
    L = int(g["mdp_n_lanes"][k])
    S = V * L * T
    assert mdp.mode == "deterministic" and tuple(mdp.original_shape) == (V, L, T)
    assert mdp.state == int(g["mdp_state"][k]) and isinstance(mdp.state, int)
    assert mdp.transition.dtype == np.int64 and mdp.transition.shape == (S, 5)
    assert np.array_equal(mdp.transition, g["mdp_transition"][k, :S])
    assert np.array_equal(bits(mdp.reward), bits(g["mdp_reward"][k, :S]))
    assert mdp.terminal.dtype == bool and np.array_equal(mdp.terminal, g["mdp_terminal"][k, :S])


@pytest.mark.parametrize("env_id,config,error", [
    ("two-way-v0", None, KeyError),
    ("u-turn-v0", None, KeyError),
    ("u-turn-v1", None, KeyError),
    ("intersection-v0", None, KeyError),
    ("intersection-v2", None, KeyError),
    ("intersection-v0", {"right_lane_reward": 0.1, "lane_change_reward": 0.0}, NotImplementedError),  # 3 actions
    ("intersection-multi-agent-v0", None, NotImplementedError),
    ("intersection-v1", None, ValueError),
    ("highway-v0", {"action": {"type": "ContinuousAction"}}, ValueError),
    ("highway-v0", {"action": {"type": "DiscreteAction"}}, ValueError),
    ("highway-v0", {"policy_frequency": 7}, ValueError),  # T = 70 > 64
])
def test_rejected_configurations_raise_before_any_launch(env_id, config, error):
    import highwayenv_b200 as hb
    from highwayenv_b200 import _native as N
    from highwayenv_b200 import planning

    env = hb.make(env_id, num_envs=2, config=config)
    env.reset(seed=0)
    lib = N.load()
    before = lib.hwy_launch_count()
    with pytest.raises(error):
        env.to_finite_mdp()
    with pytest.raises(error):
        planning.TtcValueIterationPolicy(env)
    assert lib.hwy_launch_count() == before


def test_value_iteration_rejects_bad_arguments_before_any_launch():
    import torch

    from highwayenv_b200 import _native as N
    from highwayenv_b200 import planning

    rng = np.random.default_rng(1)
    t, r, term, ns = random_mdps(rng, 2, 10, 5)
    good = dict(transition=torch.from_numpy(t).cuda(), reward=torch.from_numpy(r).cuda(),
                terminal=torch.from_numpy(term).cuda(), n_states=torch.from_numpy(ns).cuda())
    lib = N.load()
    before = lib.hwy_launch_count()
    bad_inputs = [dict(good, transition=good["transition"].long()), dict(good, reward=good["reward"].float()),
                  dict(good, terminal=good["terminal"][:, :5]), dict(good, n_states=good["n_states"][:1]),
                  dict(good, reward=good["reward"].cpu()),
                  dict(good, transition=torch.zeros(1, 4097, 5, dtype=torch.int32, device="cuda"),
                       reward=torch.zeros(1, 4097, 5, dtype=torch.float64, device="cuda"),
                       terminal=torch.zeros(1, 4097, dtype=torch.bool, device="cuda"),
                       n_states=torch.zeros(1, dtype=torch.int32, device="cuda")),
                  dict(good, transition=torch.zeros(2, 10, 9, dtype=torch.int32, device="cuda"),
                       reward=torch.zeros(2, 10, 9, dtype=torch.float64, device="cuda"))]
    for kw in bad_inputs:
        with pytest.raises(ValueError):
            planning.value_iteration(SimpleNamespace(**kw))
    for gamma, iterations in ((1.5, 10), (-0.1, 10), (float("nan"), 10), (1.0, -1)):
        with pytest.raises(ValueError):
            planning.value_iteration(SimpleNamespace(**good), gamma=gamma, iterations=iterations)
    assert lib.hwy_launch_count() == before
