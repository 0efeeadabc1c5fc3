"""GPU parity of the CUDA highway path (through the C ABI) against
  (a) golden trajectories of the unmodified reference (tests/golden), and
  (b) the C oracle on many seeded envs, incl. device-side autoreset.
Bar (BASELINE.json north_star): lane / target-lane / crashed / terminated bit-exact,
positions / headings / speeds within 1e-5 abs (we observe ~1e-12)."""
import numpy as np
import pytest
import torch

import hwy_oracle as ho
from parity_utils import comparable_steps, compare_state, golden_state, load_golden, well_conditioned

pytestmark = pytest.mark.gpu

CASES = ["highway_fast_v20", "highway_fast_v50", "highway_v50", "highway_v100_continuous",
         "highway_discrete_action", "highway_fast_features", "highway_fast_features_range"]


def make_env(g_or_cfg, n, **kw):
    import highwayenv_b200 as hb

    cfg = dict(g_or_cfg)
    env_id = cfg.pop("_env_id")
    cfg.pop("_others_check_collisions", None)
    return hb.make(env_id, num_envs=n, config=cfg, **kw)


def env_state(sd, e):
    return {k: (sd[k][e] if k not in ("rng",) else None) for k in sd}


def golden_to_sd(g, states, action_type):
    """list of dump_state dicts -> load_state_dict payload"""
    n = len(states)
    V = len(states[0]["x"])
    sd = {}
    for k in ("x", "y", "heading", "speed"):
        sd[k] = np.stack([s[k] for s in states])
    sd["target_speed"] = np.stack([np.nan_to_num(s["target_speed"], nan=0.0) for s in states])
    sd["timer"] = np.stack([np.nan_to_num(s["timer"], nan=0.0) for s in states])
    sd["delta"] = np.stack([np.nan_to_num(s["delta"], nan=4.0) for s in states])
    has = np.stack([~np.isnan(s["impact"][:, 0]) for s in states])
    sd["has_impact"] = has
    sd["impact_x"] = np.stack([np.nan_to_num(s["impact"][:, 0]) for s in states])
    sd["impact_y"] = np.stack([np.nan_to_num(s["impact"][:, 1]) for s in states])
    sd["lane"] = np.stack([s["lane"] for s in states])
    sd["target_lane"] = np.stack([np.where(s["target_lane"] < 0, s["lane"], s["target_lane"]) for s in states])
    sd["crashed"] = np.stack([s["crashed"] for s in states])
    sd["check_collisions"] = np.stack([s["check_collisions"] for s in states])
    kind = np.zeros((n, V), dtype=np.int32)
    kind[:, 0] = 1 if action_type == 0 else 2
    sd["kind"] = kind
    sd["speed_index"] = np.array([s["speed_index"][0] for s in states], dtype=np.int32)
    sd["time"] = np.array([float(s["time"]) for s in states])
    return sd


@pytest.mark.parametrize("name", CASES)
def test_reset_bit_exact_vs_reference(name):
    g = load_golden(name)
    env = make_env(g["config"], len(g["seeds"]))
    obs, _ = env.reset(seed=[int(s) for s in g["seeds"]])
    sd = env.state_dict()
    for i in range(len(g["seeds"])):
        assert compare_state(golden_state(g, i, 0), env_state(sd, i), tol=0.0, ctx=f"{name}#{i}") == 0.0
    assert np.array_equal(obs.cpu().numpy(), g["obs"][:, 0])


@pytest.mark.parametrize("name", CASES)
def test_teacher_forced_vs_reference(name):
    g = load_golden(name)
    S, T = g["actions"].shape[:2]
    env = make_env(g["config"], S, autoreset_mode="Disabled")
    env.reset(seed=0)
    at = int(env._params.action_type)
    worst = 0.0
    for t in range(T):
        env.load_state_dict(golden_to_sd(g, [golden_state(g, i, t) for i in range(S)], at))
        obs, rew, term, trunc, info = env.step(g["actions"][:, t])
        sd = env.state_dict()
        obs, rew, term, trunc = obs.cpu().numpy(), rew.cpu().numpy(), term.cpu().numpy(), trunc.cpu().numpy()
        for i in range(S):
            ctx = f"{name} seed#{i} t={t}"
            st1 = golden_state(g, i, t + 1)
            worst = max(worst, compare_state(st1, env_state(sd, i), ctx=ctx))
            assert abs(rew[i] - g["reward"][i, t]) <= 1e-9, ctx
            assert bool(term[i]) == bool(g["terminated"][i, t]), ctx
            assert bool(trunc[i]) == bool(g["truncated"][i, t]), ctx
            assert np.max(np.abs(obs[i] - g["obs"][i, t + 1])) <= 1e-6, ctx
            assert abs(info["speed"][i].item() - st1["speed"][0]) <= 1e-5
            assert bool(info["crashed"][i].item()) == bool(st1["crashed"][0])
    assert worst < 1e-7, worst


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
    # every well-conditioned (seed, step) of the fixture was compared: 96-100 % of the rollout (test_host_cpu pins that)
    assert compared == comparable_steps(g), (compared, comparable_steps(g), S * T)


def _oracle_pair(name, n, seed0):
    g = load_golden(name)
    cfg = g["config"]
    oc = ho.cfg_from_dict(cfg)
    ob = ho.OracleBatch(oc, n, seeds=range(seed0, seed0 + n), threads=8)
    return g, cfg, oc, ob


@pytest.mark.parametrize("name,n,T", [("highway_fast_v50", 512, 30), ("highway_fast_v20", 256, 30),
                                      ("highway_v50", 64, 12), ("highway_v100_continuous", 32, 8),
                                      ("highway_fast_features", 128, 12), ("highway_fast_features_range", 128, 12)])
def test_teacher_forced_vs_oracle_many_envs(name, n, T):
    """Every step: inject the oracle's state, step both, compare everything."""
    g, cfg, oc, ob = _oracle_pair(name, n, 5000)
    env = make_env(cfg, n, autoreset_mode="Disabled")
    env.reset(seed=5000)
    ob.reset()
    rng = np.random.default_rng(1)
    for t in range(T):
        sd = {k: ob.a[k].copy() for k in ob.a}
        env.load_state_dict(sd)
        if oc.action_type == 0:
            act = rng.integers(0, 5, size=n).astype(np.int32)
        else:
            act = rng.uniform(-1, 1, size=(n, 2)).astype(np.float32)
        o_obs, o_rew, o_term, o_trunc = ob.step(act)
        obs, rew, term, trunc, _ = env.step(act)
        sd = env.state_dict()
        for k in ("x", "y", "heading", "speed", "timer", "target_speed"):
            d = np.max(np.abs(sd[k] - ob.a[k]))
            assert d <= 1e-7, f"{name} t={t} {k} {d}"
        for k in ("lane", "target_lane", "crashed", "has_impact"):
            assert np.array_equal(sd[k].astype(np.int32), ob.a[k].astype(np.int32)), f"{name} t={t} {k}"
        hi = ob.a["has_impact"].astype(bool)
        if hi.any():
            assert np.max(np.abs(sd["impact_x"][hi] - ob.a["impact_x"][hi])) <= 1e-7
            assert np.max(np.abs(sd["impact_y"][hi] - ob.a["impact_y"][hi])) <= 1e-7
        assert np.array_equal(sd["speed_index"], ob.a["speed_index"])
        assert np.max(np.abs(rew.cpu().numpy() - o_rew)) <= 1e-9
        assert np.array_equal(term.cpu().numpy(), o_term.astype(bool))
        assert np.array_equal(trunc.cpu().numpy(), o_trunc.astype(bool))
        assert np.max(np.abs(obs.cpu().numpy() - o_obs)) <= 1e-6


def test_autoreset_same_step_matches_oracle():
    """Device-side SameStep autoreset re-spawns from the env's own PCG64 stream, bit-exactly."""
    name, n, T = "highway_fast_v20", 128, 40
    g, cfg, oc, ob = _oracle_pair(name, n, 9000)
    env = make_env(cfg, n)  # SameStep
    obs0, _ = env.reset(seed=9000)
    assert np.array_equal(obs0.cpu().numpy(), ob.reset())
    rng = np.random.default_rng(2)
    resets = 0
    for t in range(T):
        # teacher-force to keep both sides in the same state, but keep each side's own RNG
        sd = {k: ob.a[k].copy() for k in ob.a}
        env.load_state_dict(sd)
        act = rng.integers(0, 5, size=n).astype(np.int32)
        o_obs, o_rew, o_term, o_trunc = ob.step(act, autoreset=True)
        obs, rew, term, trunc, info = env.step(act)
        done = (o_term | o_trunc).astype(bool)
        resets += int(done.sum())
        assert np.array_equal((term | trunc).cpu().numpy(), done)
        sd = env.state_dict()
        if done.any():  # freshly spawned envs are bit-identical
            for k in ("x", "y", "heading", "speed", "timer", "delta", "target_speed"):
                assert np.array_equal(sd[k][done], ob.a[k][done]), k
            assert np.array_equal(sd["lane"][done], ob.a["lane"][done])
            assert np.array_equal(obs.cpu().numpy()[done], o_obs[done])
            assert np.all(sd["time"][done] == 0)
            assert np.array_equal(info["final_obs"].cpu().numpy()[~done], obs.cpu().numpy()[~done])
        assert np.max(np.abs(obs.cpu().numpy() - o_obs)) <= 1e-6
        # the numpy PCG64 streams stay bit-identical (state, inc, buffered 32-bit half)
        rng_w = sd["rng"]
        assert np.array_equal(rng_w[0], ob.rng["state_hi"]) and np.array_equal(rng_w[1], ob.rng["state_lo"])
        assert np.array_equal(rng_w[2], ob.rng["inc_hi"]) and np.array_equal(rng_w[3], ob.rng["inc_lo"])
        assert np.array_equal(rng_w[4] >> np.uint64(32), ob.rng["has_uint32"].astype(np.uint64))
        hb_ = ob.rng["has_uint32"] == 1
        assert np.array_equal((rng_w[4] & np.uint64(0xFFFFFFFF))[hb_], ob.rng["uinteger"][hb_].astype(np.uint64))
    assert resets > n  # every env ended at least once (duration 30 < 40 steps)


@pytest.mark.parametrize("name,n", [("highway_fast_v50", 64), ("highway_v100_continuous", 16), ("highway_v50", 32)])
def test_autoreset_streams_other_configs(name, n):
    """Fused autoreset on the other thread mappings (64 / 128 threads per env, 4 lanes)."""
    g, cfg, oc, ob = _oracle_pair(name, n, 11000)
    cfg = dict(cfg)
    cfg["duration"] = 3  # force frequent truncation
    oc = ho.cfg_from_dict(cfg)
    ob = ho.OracleBatch(oc, n, seeds=range(11000, 11000 + n), threads=8)
    env = make_env(cfg, n)
    obs0, _ = env.reset(seed=11000)
    assert np.array_equal(obs0.cpu().numpy(), ob.reset())
    rng = np.random.default_rng(5)
    for t in range(8):
        env.load_state_dict({k: ob.a[k].copy() for k in ob.a})
        if oc.action_type == 0:
            act = rng.integers(0, 5, size=n).astype(np.int32)
        else:
            act = rng.uniform(-1, 1, size=(n, 2)).astype(np.float32)
        o_obs, o_rew, o_term, o_trunc = ob.step(act, autoreset=True)
        obs, rew, term, trunc, info = env.step(act)
        done = (o_term | o_trunc).astype(bool)
        sd = env.state_dict()
        for k in ("x", "y", "heading", "speed", "timer", "delta", "target_speed"):
            assert np.array_equal(sd[k][done], ob.a[k][done]), (t, k)
        assert np.array_equal(sd["lane"][done], ob.a["lane"][done])
        assert np.array_equal(obs.cpu().numpy()[done], o_obs[done])
        assert np.array_equal(sd["rng"][0], ob.rng["state_hi"]) and np.array_equal(sd["rng"][1], ob.rng["state_lo"])


def test_abi_errors_are_loud():
    import ctypes as C

    from highwayenv_b200 import _native as N

    lib = N.load()
    assert lib.hwy_highway_step(None, None, None, None, None, None, None, None, None, None, None, 0, None, None) != 0
    assert b"null" in lib.hwy_last_error()
    import highwayenv_b200 as hb

    with pytest.raises(ValueError):
        hb.make("highway-v0", num_envs=2, config={"action": {"type": "Nope"}})
    with pytest.raises(KeyError):
        hb.make("parking-v0")
    env = hb.make("highway-fast-v0", num_envs=2)
    with pytest.raises(RuntimeError):
        env.step([1, 1])  # before reset


def test_longitudinal_ties_take_the_exact_path():
    """Vehicles sharing a longitudinal coordinate (the `<=` / `>` tie rules of
    Road.neighbour_vehicles, road/road.py:539-544) route the env to the linear scans."""
    name, n = "highway_fast_v50", 64
    g, cfg, oc, ob = _oracle_pair(name, n, 7000)
    env = make_env(cfg, n, autoreset_mode="Disabled")
    env.reset(seed=7000)
    ob.reset()
    rng = np.random.default_rng(3)
    for t in range(6):
        # force ties: copy the x of vehicle k onto vehicle k+1 for a few random k per env
        for e_ in range(n):
            for k in rng.integers(1, 49, size=3):
                ob.a["x"][e_, k + 1] = ob.a["x"][e_, k]
        sd = {k: ob.a[k].copy() for k in ob.a}
        env.load_state_dict(sd)
        act = rng.integers(0, 5, size=n).astype(np.int32)
        o_obs, o_rew, o_term, o_trunc = ob.step(act)
        obs, rew, term, trunc, _ = env.step(act)
        sd = env.state_dict()
        for k in ("x", "y", "heading", "speed", "timer"):
            assert np.max(np.abs(sd[k] - ob.a[k])) <= 1e-7, (t, k)
        for k in ("lane", "target_lane", "crashed", "has_impact"):
            assert np.array_equal(sd[k].astype(np.int32), ob.a[k].astype(np.int32)), (t, k)
        assert np.array_equal(term.cpu().numpy(), o_term.astype(bool))


def test_host_stepper_graph_matches_env_step():
    """env.host_stepper(): upload + step kernel + downloads in one CUDA graph == env.step, through resets."""
    g = load_golden("highway_fast_v20")
    n = 96
    a = make_env(g["config"], n)
    b = make_env(g["config"], n)
    a.reset(seed=123)
    b.reset(seed=123)
    hs = b.host_stepper()
    rng = np.random.default_rng(4)
    for t in range(35):
        act = rng.integers(0, 5, size=n).astype(np.int32)
        oa, ra, ta, ua, _ = a.step(act)
        hs.actions[:] = act
        ob, rb, tb, ub = hs.step()
        assert np.array_equal(oa.cpu().numpy(), ob) and np.array_equal(ra.cpu().numpy(), rb), t
        assert np.array_equal(ta.cpu().numpy(), tb) and np.array_equal(ua.cpu().numpy(), ub), t
    sa, sb = a.state_dict(), b.state_dict()
    for k in sa:
        assert np.array_equal(sa[k], sb[k]), k


def test_next_step_autoreset_matches_gymnasium_semantics():
    """AutoresetMode.NEXT_STEP (gymnasium's vector default): an env that ended is RESET by the next step call
    (reset obs, reward 0, flags False) instead of being stepped.  Emulated with the oracle exactly as
    SyncVectorEnv does it, teacher-forced every step; spawns and generator streams must stay bit-identical."""
    name, n, T = "highway_fast_v20", 96, 45
    g, cfg, oc, ob = _oracle_pair(name, n, 13000)
    cfg = dict(cfg)
    cfg["duration"] = 6
    oc = ho.cfg_from_dict(cfg)
    ob = ho.OracleBatch(oc, n, seeds=range(13000, 13000 + n), threads=8)
    env = make_env(cfg, n, autoreset_mode="NextStep")
    obs0, _ = env.reset(seed=13000)
    assert np.array_equal(obs0.cpu().numpy(), ob.reset())
    rng = np.random.default_rng(8)
    pending = np.zeros(n, dtype=bool)
    n_resets = 0
    for t in range(T):
        env.load_state_dict({k: ob.a[k].copy() for k in ob.a})
        act = rng.integers(0, 5, size=n).astype(np.int32)
        snap = {k: ob.a[k].copy() for k in ob.a}
        snap_rng = ob.rng.copy()
        o_obs, o_rew, o_term, o_trunc = (x.copy() for x in ob.step(act))
        if pending.any():  # those envs are reset instead of stepped
            for k in ob.a:
                ob.a[k][pending] = snap[k][pending]
            ob.rng[pending] = snap_rng[pending]
            o_obs[pending] = ob.reset(mask=pending.astype(np.uint8))[pending]
            o_rew[pending], o_term[pending], o_trunc[pending] = 0.0, 0, 0
            n_resets += int(pending.sum())
        obs, rew, term, trunc, _ = env.step(act)
        sd = env.state_dict()
        assert np.array_equal(term.cpu().numpy(), o_term.astype(bool)) and np.array_equal(trunc.cpu().numpy(), o_trunc.astype(bool)), t
        assert np.max(np.abs(rew.cpu().numpy() - o_rew)) <= 1e-9, t
        assert np.all(rew.cpu().numpy()[pending] == 0.0)
        assert np.array_equal(obs.cpu().numpy()[pending], o_obs[pending]), t      # reset observations: bit-exact
        assert np.max(np.abs(obs.cpu().numpy() - o_obs)) <= 1e-6, t
        for k in ("x", "y", "speed", "delta", "timer"):
            assert np.array_equal(sd[k][pending], ob.a[k][pending]), (t, k)
        assert np.array_equal(sd["time"], ob.a["time"])
        assert np.array_equal(sd["rng"][0], ob.rng["state_hi"]) and np.array_equal(sd["rng"][1], ob.rng["state_lo"])
        pending = (o_term | o_trunc).astype(bool)
    assert n_resets > n
