"""GPU parity of LinearVehicle / AggressiveVehicle / DefensiveVehicle traffic on highway-v0 / highway-fast-v0
(highway_linear_step_kernel, highway_linear_reset_kernel) against the linear_* golden rollouts of the reference
(oracle/gen_linear_golden.py) and the C oracle."""
import numpy as np
import pytest

import hwy_linear_oracle as lo
from parity_utils import comparable_steps, compare_state, golden_state, load_golden, well_conditioned
import rng_craft as rc
from test_gpu_highway_parity import env_state, golden_to_sd, make_env

pytestmark = pytest.mark.gpu

CASES = ["linear_highway_fast_v20", "linear_aggressive_fast_v50", "linear_defensive_v50",
         "linear_highway_v100_continuous"]


def _sd_with_params(g, states, params, action_type):
    sd = golden_to_sd(g, states, action_type)
    sd["acceleration_parameters"] = params[..., :3]
    sd["steering_parameters"] = params[..., 3:]
    return sd


def _oracle(cfg, n, seed0):
    ob = lo.LinearOracleBatch(cfg, n, seeds=range(seed0, seed0 + n), threads=8)
    return ob.cfg, ob


def _oracle_sd(ob):
    sd = {k: ob.a[k].copy() for k in ob.a}
    sd["acceleration_parameters"] = ob.linear_params[..., :3].copy()
    sd["steering_parameters"] = ob.linear_params[..., 3:].copy()
    return sd


def _assert_rng_equal(rng_w, ob):
    assert np.array_equal(rng_w[0], ob.rng["state_hi"]) and np.array_equal(rng_w[1], ob.rng["state_lo"])
    assert np.array_equal(rng_w[2], ob.rng["inc_hi"]) and np.array_equal(rng_w[3], ob.rng["inc_lo"])
    assert np.array_equal(rng_w[4] >> np.uint64(32), ob.rng["has_uint32"].astype(np.uint64))
    hb_ = ob.rng["has_uint32"] == 1
    assert np.array_equal((rng_w[4] & np.uint64(0xFFFFFFFF))[hb_], ob.rng["uinteger"][hb_].astype(np.uint64))


@pytest.mark.parametrize("name", CASES)
def test_reset_bit_exact_vs_reference(name):
    g = load_golden(name)
    env = make_env(g["config"], len(g["seeds"]))
    obs, _ = env.reset(seed=[int(s) for s in g["seeds"]])
    sd = env.state_dict()
    for i in range(len(g["seeds"])):
        assert compare_state(golden_state(g, i, 0), env_state(sd, i), tol=0.0, ctx=f"{name}#{i}") == 0.0
    assert np.array_equal(obs.cpu().numpy(), g["obs"][:, 0])
    assert np.array_equal(sd["acceleration_parameters"], g["linear_params"][..., :3])
    assert np.array_equal(sd["steering_parameters"], g["linear_params"][..., 3:])
    assert np.array_equal(sd["rng"].T, g["rng_words"][:, 0])


@pytest.mark.parametrize("name", CASES)
def test_teacher_forced_vs_reference(name):
    g = load_golden(name)
    S, T = g["actions"].shape[:2]
    env = make_env(g["config"], S, autoreset_mode="Disabled")
    env.reset(seed=0)
    at = int(env._params.action_type)
    worst = 0.0
    for t in range(T):
        env.load_state_dict(_sd_with_params(g, [golden_state(g, i, t) for i in range(S)], g["linear_params"], at))
        obs, rew, term, trunc, info = env.step(g["actions"][:, t])
        sd = env.state_dict()
        obs, rew, term, trunc = obs.cpu().numpy(), rew.cpu().numpy(), term.cpu().numpy(), trunc.cpu().numpy()
        for i in range(S):
            ctx = f"{name} seed#{i} t={t}"
            worst = max(worst, compare_state(golden_state(g, i, t + 1), env_state(sd, i), ctx=ctx))
            assert abs(rew[i] - g["reward"][i, t]) <= 1e-9, ctx
            assert bool(term[i]) == bool(g["terminated"][i, t]), ctx
            assert bool(trunc[i]) == bool(g["truncated"][i, t]), ctx
            assert np.max(np.abs(obs[i] - g["obs"][i, t + 1])) <= 1e-6, ctx
    assert worst < 1e-9, worst


@pytest.mark.parametrize("name", CASES)
def test_free_running_vs_reference(name):
    g = load_golden(name)
    S, T = g["actions"].shape[:2]
    env = make_env(g["config"], S, autoreset_mode="Disabled")
    env.reset(seed=[int(s) for s in g["seeds"]])
    alive = np.ones(S, dtype=bool)
    compared = 0
    for t in range(T):
        obs, rew, term, trunc, _ = env.step(g["actions"][:, t])
        sd = env.state_dict()
        obs, rew, term = obs.cpu().numpy(), rew.cpu().numpy(), term.cpu().numpy()
        for i in range(S):
            st = golden_state(g, i, t + 1)
            alive[i] &= well_conditioned(st)
            if not alive[i]:
                continue
            compare_state(st, env_state(sd, i), ctx=f"{name} seed#{i} t={t}")
            assert abs(rew[i] - g["reward"][i, t]) <= 1e-9
            assert bool(term[i]) == bool(g["terminated"][i, t])
            assert np.max(np.abs(obs[i] - g["obs"][i, t + 1])) <= 1e-6
            compared += 1
    assert compared == comparable_steps(g), (compared, comparable_steps(g), S * T)


@pytest.mark.parametrize("name,n,T", [("linear_highway_fast_v20", 256, 12), ("linear_aggressive_fast_v50", 256, 12),
                                      ("linear_defensive_v50", 64, 8), ("linear_highway_v100_continuous", 32, 6)])
def test_teacher_forced_vs_oracle_many_envs(name, n, T):
    cfg = load_golden(name)["config"]
    oc, ob = _oracle(cfg, n, 5000)
    env = make_env(cfg, n, autoreset_mode="Disabled")
    env.reset(seed=5000)
    ob.reset()
    assert np.array_equal(env.state_dict()["acceleration_parameters"], ob.linear_params[..., :3])
    rng = np.random.default_rng(1)
    for t in range(T):
        env.load_state_dict(_oracle_sd(ob))
        act = (rng.integers(0, 5, size=n).astype(np.int32) if oc.action_type == 0
               else rng.uniform(-1, 1, size=(n, 2)).astype(np.float32))
        o_obs, o_rew, o_term, o_trunc = ob.step(act)
        obs, rew, term, trunc, _ = env.step(act)
        sd = env.state_dict()
        for k in ("x", "y", "heading", "speed", "timer", "target_speed"):
            assert np.max(np.abs(sd[k] - ob.a[k])) <= 1e-9, f"{name} t={t} {k}"
        for k in ("lane", "target_lane", "crashed", "has_impact"):
            assert np.array_equal(sd[k].astype(np.int32), ob.a[k].astype(np.int32)), f"{name} t={t} {k}"
        assert np.max(np.abs(rew.cpu().numpy() - o_rew)) <= 1e-9
        assert np.array_equal(term.cpu().numpy(), o_term.astype(bool))
        assert np.max(np.abs(obs.cpu().numpy() - o_obs)) <= 1e-6


@pytest.mark.parametrize("name,n", [("linear_highway_fast_v20", 128), ("linear_aggressive_fast_v50", 64),
                                    ("linear_highway_v100_continuous", 16)])
def test_fused_autoreset_equals_linear_reset(name, n):
    """Envs re-spawned by the SameStep autoreset inside the step kernel equal hwy_highway_linear_reset (the oracle's
    reset): state, parameters and generator words — on 32, 64 and 128 threads per env (V = 101 jumps past the
    PCG64 table in several hops)."""
    cfg = dict(load_golden(name)["config"])
    cfg["duration"] = 2  # frequent truncation
    oc, ob = _oracle(cfg, n, 11000)
    env = make_env(cfg, n)
    obs0, _ = env.reset(seed=11000)
    assert np.array_equal(obs0.cpu().numpy(), ob.reset())
    rng = np.random.default_rng(5)
    resets = 0
    for t in range(6):
        env.load_state_dict(_oracle_sd(ob))
        act = (rng.integers(0, 5, size=n).astype(np.int32) if oc.action_type == 0
               else rng.uniform(-1, 1, size=(n, 2)).astype(np.float32))
        o_obs, o_rew, o_term, o_trunc = ob.step(act, autoreset=True)
        obs, rew, term, trunc, info = env.step(act)
        done = (o_term | o_trunc).astype(bool)
        resets += int(done.sum())
        assert np.array_equal((term | trunc).cpu().numpy(), done)
        sd = env.state_dict()
        for k in ("x", "y", "heading", "speed", "timer", "delta", "target_speed"):
            assert np.array_equal(sd[k][done], ob.a[k][done]), (t, k)
        assert np.array_equal(sd["acceleration_parameters"][done], ob.linear_params[done, :, :3])
        assert np.array_equal(sd["steering_parameters"][done], ob.linear_params[done, :, 3:])
        assert np.array_equal(obs.cpu().numpy()[done], o_obs[done])
        _assert_rng_equal(sd["rng"], ob)
    assert resets >= n


def test_fused_autoreset_serial_fallback():
    """A Lemire rejection in the lane draw of a re-spawn sends the env to the serial draw order inside the step
    kernel: the ego's lane choice reads a buffered 32-bit 0 (crafted words, tests/rng_craft.py), which choice(3)
    rejects.  Those envs, and the ones re-spawned on the parallel path next to them, equal the linear reset."""
    name, n = "linear_highway_fast_v20", 24
    cfg = dict(load_golden(name)["config"])
    oc, ob = _oracle(cfg, n, 12000)
    env = make_env(cfg, n)
    env.reset(seed=12000)
    ob.reset()
    assert rc.lemire_rejects(0, int(oc.lanes_count))
    crafted = list(range(0, n, 2))
    for e in crafted:
        w = rc.words_of((int(ob.rng["state_hi"][e]) << 64) | int(ob.rng["state_lo"][e]),
                        (int(ob.rng["inc_hi"][e]) << 64) | int(ob.rng["inc_lo"][e]), 1, 0)
        ob.rng["has_uint32"][e], ob.rng["uinteger"][e] = 1, 0
        assert int(w[4]) == 1 << 32
    ob.a["time"][:] = float(cfg["duration"]) - 1.0 / cfg["policy_frequency"]  # every env truncates in this step
    sd = _oracle_sd(ob)
    sd["rng"] = np.stack([ob.rng["state_hi"], ob.rng["state_lo"], ob.rng["inc_hi"], ob.rng["inc_lo"],
                          (ob.rng["has_uint32"].astype(np.uint64) << np.uint64(32)) | ob.rng["uinteger"].astype(np.uint64)])
    env.load_state_dict(sd)
    act = np.ones(n, dtype=np.int32)
    o_obs, _, o_term, o_trunc = ob.step(act, autoreset=True)
    obs, _, term, trunc, _ = env.step(act)
    assert o_trunc.astype(bool).all() and trunc.cpu().numpy().all()
    sd = env.state_dict()
    for k in ("x", "y", "heading", "speed", "timer", "delta", "target_speed", "lane", "kind"):
        assert np.array_equal(sd[k], ob.a[k]), k
    assert np.array_equal(sd["acceleration_parameters"], ob.linear_params[..., :3])
    assert np.array_equal(sd["steering_parameters"], ob.linear_params[..., 3:])
    assert np.array_equal(obs.cpu().numpy(), o_obs)
    _assert_rng_equal(sd["rng"], ob)


def test_general_lanes_path_equals_congruent_path(monkeypatch):
    g = load_golden("linear_aggressive_fast_v50")
    n = 64
    a = make_env(g["config"], n, autoreset_mode="Disabled")
    b = make_env(g["config"], n, autoreset_mode="Disabled")
    a.reset(seed=77)
    b.reset(seed=77)
    rng = np.random.default_rng(9)
    for t in range(10):
        act = rng.integers(0, 5, size=n).astype(np.int32)
        oa = a.step(act)[0].cpu().numpy()
        monkeypatch.setenv("HWYB200_GENERAL_LANES", "1")
        ob_ = b.step(act)[0].cpu().numpy()
        monkeypatch.delenv("HWYB200_GENERAL_LANES")
        assert np.array_equal(oa, ob_), t
    sa, sb = a.state_dict(), b.state_dict()
    for k in sa:
        assert np.array_equal(sa[k], sb[k]), k


def test_host_stepper_graph_equals_eager_steps():
    g = load_golden("linear_highway_fast_v20")
    n = 96
    a = make_env(g["config"], n)
    b = make_env(g["config"], n)
    a.reset(seed=321)
    b.reset(seed=321)
    hs = b.host_stepper()
    rng = np.random.default_rng(4)
    for t in range(35):  # past the 30 s duration: fused re-spawns inside the graph
        act = rng.integers(0, 5, size=n).astype(np.int32)
        oa, ra, ta, ua, _ = a.step(act)
        hs.actions[:] = act
        ob_, rb, tb, ub = hs.step()
        assert np.array_equal(oa.cpu().numpy(), ob_) and np.array_equal(ra.cpu().numpy(), rb), t
        assert np.array_equal(ta.cpu().numpy(), tb) and np.array_equal(ua.cpu().numpy(), ub), t
    sa, sb = a.state_dict(), b.state_dict()
    for k in sa:
        assert np.array_equal(sa[k], sb[k]), k


def test_state_dict_round_trip_and_idm_dicts_unchanged():
    g = load_golden("linear_highway_fast_v20")
    a = make_env(g["config"], 16)
    a.reset(seed=5)
    sd = a.state_dict()
    assert sd["acceleration_parameters"].shape == (16, 21, 3) and sd["steering_parameters"].shape == (16, 21, 2)
    b = make_env(g["config"], 16)
    b.reset(seed=99)
    b.load_state_dict(sd)
    sb = b.state_dict()
    for k in sd:
        assert np.array_equal(sd[k], sb[k]), k
    cfg = dict(g["config"], other_vehicles_type="highway_env.vehicle.behavior.IDMVehicle")
    idm = make_env(cfg, 4)
    idm.reset(seed=5)
    assert "acceleration_parameters" not in idm.state_dict()


def test_road_substeps_and_single_env():
    """hwy_highway_linear_substeps against the oracle's orc_linear_highway_substeps; make_single on linear traffic."""
    import highwayenv_b200 as hb

    g = load_golden("linear_highway_fast_v20")
    cfg = dict(g["config"])
    n = 32
    env = make_env(cfg, n, autoreset_mode="Disabled")
    env.reset(seed=40)
    oc, ob = _oracle(cfg, n, 40)
    ob.reset()
    env.road_substeps(7)
    ob.substeps(7)
    sd = env.state_dict()
    for k in ("x", "y", "heading", "speed", "timer"):
        assert np.max(np.abs(sd[k] - ob.a[k])) <= 1e-9, k
    for k in ("lane", "target_lane", "crashed"):
        assert np.array_equal(sd[k].astype(np.int32), ob.a[k].astype(np.int32)), k
    single = hb.make_single("highway-fast-v0", config={k: v for k, v in cfg.items() if not k.startswith("_")})
    o, _ = single.reset(seed=3000)
    assert np.array_equal(np.asarray(o), g["obs"][0, 0])
