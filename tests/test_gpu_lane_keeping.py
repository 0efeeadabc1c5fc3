"""GPU parity of lane-keeping-v0 (hwy_lane_keeping_step / hwy_lane_keeping_reset) against the fixtures of
oracle/gen_lane_keeping.py: the device reset, free-running rollouts of 420 steps across two TimeLimit resets, the three
autoreset modes, env cloning, the host stepper's CUDA graph, the single-env facade, independence from num_envs, and the
configurations that must raise before any launch."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["lane_keeping_default", "lane_keeping_pf5", "lane_keeping_reference_state", "lane_keeping_longitudinal"]
# CUDA's atan2 / sincos against numpy's, carried through hundreds of RK4 frames without feedback: FLOAT_TOL (1e-5), the
# project's bound on positions / headings / speeds, relative above 1.  intersection-v1's free-running BicycleVehicle
# test allows 1e-4.
TOL = 1e-5
FIELDS = ("x", "y", "heading", "speed", "lateral_speed", "yaw_rate")


def load(name):
    """The fixture, plus `rng_all`: the stream words after every step (the fixture stores every 20th step's; the others
    follow from the reset's words, as tests/test_lane_keeping_spec.py checks)."""
    from test_lane_keeping_spec import stream_per_step

    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    g["config"] = {k: v for k, v in json.loads(str(g.pop("config_json"))).items() if not k.startswith("_")}
    g["rng_all"] = stream_per_step(g)[0]
    g["slot"] = {int(t): j for j, t in enumerate(g["steps"])}  # step -> index of its full-precision record
    return g


def make(config, n, mode="SameStep", **kw):
    import highwayenv_b200 as hb

    return hb.make("lane-keeping-v0", num_envs=n, config=dict(config or {}), autoreset_mode=mode, **kw)


def stacked(env, obs):
    return np.stack([obs[a].cpu().numpy() for a in env.attributes], axis=1)


def state(env):
    sd = env.state_dict()
    return np.stack([sd[k] for k in FIELDS], axis=1), sd["lane_phase"], sd["rng"].T


def close(got, want, ctx):
    err = np.abs(got - want) / np.maximum(1.0, np.abs(want))
    assert float(err.max()) <= TOL, (ctx, float(err.max()))


@pytest.mark.parametrize("name", CASES)
def test_reset_matches_reference(name):
    g = load(name)
    S = len(g["seeds"])
    env = make(g["config"], S)
    obs, info = env.reset(seed=[int(s) for s in g["seeds"]])
    st, phase, rng = state(env)
    assert np.array_equal(st, g["reset_state"]) and not phase.any()
    assert np.array_equal(rng, g["reset_rng"])  # 3 observes: 24 words with the default attributes
    o = stacked(env, obs)
    assert o.dtype == np.float64 and o.shape == g["reset_obs"].shape
    if "state" in env.attributes:
        k = env.attributes.index("state")
        assert np.array_equal(o[:, k], g["reset_obs"][:, k])
    assert float(np.abs(o - g["reset_obs"]).max()) <= 1e-12
    assert np.all(info["speed"].cpu().numpy() == 8.3) and not info["crashed"].any()


def well_conditioned(g) -> np.ndarray:
    """[S, T]: the steps of an episode before the reference's speed first comes within 1.5 m/s of 0.  Around zero speed
    the tyre model switches branches (|speed| < 1) and atan2(., speed) turns by pi when the speed changes sign, so a
    last-bit difference there is amplified without bound; the throttle fixture gets there, the others never do."""
    speed = g["speed"]
    ok = np.ones(speed.shape, dtype=bool)
    for i in range(speed.shape[0]):
        good = True
        for t in range(speed.shape[1]):
            good = good and abs(float(speed[i, t])) >= 1.5
            ok[i, t] = good
            good = good or bool(g["truncated"][i, t])  # a new episode starts from the spawn
    return ok


@pytest.mark.parametrize("name", CASES)
def test_free_running_matches_reference(name):
    """SameStep over all 420 steps: stream words, truncation and reset points exact for every env on every step; lane
    phase exact on every well-conditioned step (all of them except in the throttle fixture, >= 90 % there); observation,
    state and reward within TOL at every stored step that is well-conditioned."""
    g = load(name)
    S, T = g["actions"].shape[:2]
    ok = well_conditioned(g)
    assert ok.all() or (name == "lane_keeping_longitudinal" and ok.mean() >= 0.9)
    env = make(g["config"], S)
    env.reset(seed=[int(s) for s in g["seeds"]])
    switched = compared = 0
    for t in range(T):
        obs, rew, term, trunc, info = env.step(g["actions"][:, t])
        ctx, m, j = (name, t), ok[:, t], g["slot"].get(t)
        assert not term.any() and np.array_equal(trunc.cpu().numpy(), g["truncated"][:, t]), ctx
        st, phase, rng = state(env)
        if j is not None:
            close(rew.cpu().numpy()[m], g["reward"][m, j], ctx)
            step_obs = info["final_obs"] if t in (199, 399) else obs
            close(stacked(env, step_obs)[m], g["obs"][m, j], ctx)
            compared += int(m.sum())
        if t in (199, 399):
            r = (t + 1) // 200 - 1
            assert np.array_equal(st, g["autoreset_state"][:, r]) and not phase.any(), ctx
            assert np.array_equal(rng, g["autoreset_rng"][:, r]), ctx
            close(stacked(env, obs), g["autoreset_obs"][:, r], ctx)
        else:
            if j is not None:
                close(st[m], g["state"][m, j], ctx)
                assert np.array_equal(rng, g["rng"][:, j]), ctx
            assert np.array_equal(phase[m], g["phase"][m, t]), ctx
            assert np.array_equal(rng, g["rng_all"][:, t]), ctx
            switched += int(phase[m].sum())
    assert compared == int(ok[:, g["steps"]].sum()) and switched > 0  # the fixtures reach the lane switch


@pytest.mark.parametrize("mode", ["SameStep", "NextStep", "Disabled"])
def test_autoreset_modes_against_second_episode(mode):
    g = load("lane_keeping_default")
    S = len(g["seeds"])
    env = make(g["config"], S, mode)
    env.reset(seed=[int(s) for s in g["seeds"]])
    for t in range(200):
        obs, rew, term, trunc, info = env.step(g["actions"][:, t])
    assert trunc.cpu().numpy().all()
    last = g["slot"][199]
    if mode == "SameStep":
        close(stacked(env, info["final_obs"]), g["obs"][:, last], mode)
    else:
        close(stacked(env, obs), g["obs"][:, last], mode)
        if mode == "NextStep":  # this call resets instead of stepping: the action is ignored
            obs, rew, term, trunc, _ = env.step(np.zeros((S, 1), np.float32))
            assert not rew.cpu().numpy().any() and not trunc.cpu().numpy().any()
        else:
            obs, _ = env.reset()
    close(stacked(env, obs), g["autoreset_obs"][:, 0], mode)
    st, phase, rng = state(env)
    assert np.array_equal(rng, g["autoreset_rng"][:, 0]) and np.array_equal(st, g["autoreset_state"][:, 0])
    for t in range(200, 399):
        obs, rew, term, trunc, _ = env.step(g["actions"][:, t])
        assert not trunc.cpu().numpy().any()
        assert np.array_equal(state(env)[2], g["rng_all"][:, t]), (mode, t)
        j = g["slot"].get(t)
        if j is not None:
            close(stacked(env, obs), g["obs"][:, j], (mode, t))
            close(rew.cpu().numpy(), g["reward"][:, j], (mode, t))
            close(state(env)[0], g["state"][:, j], (mode, t))


@pytest.mark.parametrize("mode", ["SameStep", "NextStep"])
def test_copy_envs_then_steps_bit_identical(mode):
    import torch

    env = make(None, 8, mode)
    env.reset(seed=3)
    rng = np.random.default_rng(0)
    for _ in range(195):  # the 10 steps after the copy cross the TimeLimit reset
        env.step(rng.uniform(-1, 1, (8, 1)).astype(np.float32))
    env.copy_envs([4, 5, 6, 7], [0, 1, 2, 3])
    for _ in range(10):
        a = rng.uniform(-1, 1, (4, 1)).astype(np.float32)
        obs, rew, term, trunc, _ = env.step(np.concatenate([a, a]))
        o = stacked(env, obs)
        assert np.array_equal(o[:4], o[4:]) and torch.equal(rew[:4], rew[4:]) and torch.equal(trunc[:4], trunc[4:])
        st, phase, words = state(env)
        assert np.array_equal(st[:4], st[4:]) and np.array_equal(phase[:4], phase[4:])
        assert np.array_equal(words[:4, [0, 1, 4]], words[4:, [0, 1, 4]])
    copied = set(env._env_rows())
    for name, t in vars(env).items():
        if isinstance(t, torch.Tensor) and t.dim() >= 1 and t.shape[0] == 8:
            assert name in copied or name in env.ROW_EXCLUDE, name


def test_host_stepper_graph_equals_eager():
    import torch

    n = 64
    a, b = make(None, n), make(None, n)
    a.reset(seed=11)
    b.reset(seed=11)
    hs = b.host_stepper()
    rng = np.random.default_rng(1)
    for t in range(210):
        act = rng.uniform(-1.2, 1.2, (n, 1)).astype(np.float32)
        obs, rew, _, trunc, _ = a.step(act)
        hs.actions[:] = act
        h_obs, h_rew, _, h_trunc = hs.step()
        assert set(h_obs) == set(a.attributes)
        for k in a.attributes:
            assert np.array_equal(h_obs[k], obs[k].cpu().numpy()), (t, k)
        assert np.array_equal(h_rew, rew.cpu().numpy()) and np.array_equal(h_trunc, trunc.cpu().numpy())
    assert torch.equal(a._rng, b._rng)


def test_make_single_returns_numpy_dicts():
    import highwayenv_b200 as hb

    g = load("lane_keeping_default")
    env = hb.make_single("lane-keeping-v0")
    obs, info = env.reset(seed=int(g["seeds"][0]))
    assert list(obs) == ["state", "derivative", "reference_state"]
    assert all(isinstance(v, np.ndarray) and v.dtype == np.float64 and v.shape == (4, 1) for v in obs.values())
    assert info["speed"] == 8.3 and info["crashed"] is False
    assert tuple(env.action_space.shape) == (1,) and env.action_space.dtype == np.float32
    for t in range(20):
        obs, reward, terminated, truncated, info = env.step(g["actions"][0, t])
        assert isinstance(reward, float) and terminated is False and truncated is False and info == {}
    close(np.stack([obs[a] for a in obs]), g["obs"][0, 0], t)  # step 19, the first stored one
    close(np.array([reward]), g["reward"][0, :1], t)
    with pytest.raises(NotImplementedError):
        env.get_available_actions()


def test_rollout_does_not_depend_on_num_envs():
    import torch

    big_n = 1 << 20
    big, small = make(None, big_n), make(None, 1)
    big.reset(seed=0)
    i = big_n - 1
    small.reset(seed=i)
    gen = torch.Generator(device="cuda").manual_seed(5)
    for _ in range(205):
        act = torch.rand(big_n, 1, device="cuda", generator=gen) * 2 - 1
        bo, br, _, bt, _ = big.step(act)
        so, sr, _, st, _ = small.step(act[i:i + 1])
        for k in big.attributes:
            assert torch.equal(bo[k][i:i + 1], so[k])
        assert torch.equal(br[i:i + 1], sr) and torch.equal(bt[i:i + 1], st)
    assert torch.equal(big._rng[:, i:i + 1], small._rng) and torch.equal(big._state[:, i:i + 1], small._state)


def test_unsupported_inputs_raise():
    import highwayenv_b200 as hb
    from highwayenv_b200.planning import MctsPolicy, OpdPolicy, TtcValueIterationPolicy

    act = {"type": "ContinuousAction", "steering_range": [-1.0, 1.0], "longitudinal": False, "lateral": True}
    for cfg, exc in (({"action": dict(act, dynamical=False)}, NotImplementedError),
                     ({"observation": {"type": "Kinematics"}}, NotImplementedError),
                     ({"observation": {"type": "AttributesObservation", "attributes": ["state", "speed"]}},
                      ValueError)):
        with pytest.raises(exc):
            make(cfg, 4)
    with pytest.raises(NotImplementedError):
        hb.make("lane-keeping-v0", num_envs=2, render_mode="rgb_array")
    env = make(None, 4)
    env.reset(seed=0)
    for call in (env.to_finite_mdp, env.get_available_actions, env.observe, lambda: OpdPolicy(env),
                 lambda: MctsPolicy(env)):
        with pytest.raises(NotImplementedError):
            call()
    with pytest.raises(ValueError):  # planning's MDPVehicle check
        TtcValueIterationPolicy(env)
