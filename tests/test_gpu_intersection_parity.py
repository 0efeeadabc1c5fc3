"""GPU parity of intersection-v0 (RegulatedRoad, dynamic population, OccupancyGrid / 7-feature
Kinematics) through the C ABI: against golden rollouts of the unmodified reference (state, obs,
reward, flags AND the numpy generator words after every step) and against the oracle on more seeds."""
import numpy as np
import pytest

import net_oracle as no
from parity_utils import load_golden
from test_net_oracle_golden import compare_inter, inter_state

pytestmark = pytest.mark.gpu
CASES = ["intersection_kin", "intersection_grid", "intersection_v2_kin"]
V = 32


def make_env(cfg, n, **kw):
    import highwayenv_b200 as hb

    cfg = dict(cfg)
    env_id = cfg.pop("_env_id")
    cfg.pop("_others_check_collisions", None)
    return hb.make(env_id, num_envs=n, config=cfg, **kw)


def to_sd(states, rng_words=None):
    """golden schema (NaN / -1 padded beyond `count`) -> env.load_state_dict schema"""
    out = {}
    live = np.stack([np.arange(V) < int(s["count"]) for s in states])
    for k in ("x", "y", "heading", "speed", "target_speed", "timer"):
        out[k] = np.where(live, np.nan_to_num(np.stack([s[k] for s in states])), 0.0)
    out["delta"] = np.where(live, np.nan_to_num(np.stack([s["delta"] for s in states]), nan=4.0), 4.0)
    lane = np.where(live, np.stack([s["lane"] for s in states]), 0)
    tgt = np.stack([s["target_lane"] for s in states])
    out["lane"], out["target_lane"] = lane, np.where(live & (tgt >= 0), tgt, lane)
    imp = np.stack([s["impact"] for s in states])
    has = live & ~np.isnan(imp[..., 0])
    out["has_impact"] = has
    out["impact_x"], out["impact_y"] = np.where(has, imp[..., 0], 0.0), np.where(has, imp[..., 1], 0.0)
    for k in ("kind", "crashed", "is_yielding", "route_len"):
        out[k] = np.where(live, np.stack([s[k] for s in states]), 0)
    out["route"] = np.stack([s["route"] for s in states]).astype(np.int32)
    out["speed_index"] = np.array([np.ravel(s["speed_index"])[0] for s in states], dtype=np.int32)
    out["time"] = np.array([float(s["time"]) for s in states])
    out["count"] = np.array([int(s["count"]) for s in states], dtype=np.int32)
    out["road_steps"] = np.array([int(s["road_steps"]) for s in states], dtype=np.int32)
    if rng_words is not None:
        out["rng"] = np.ascontiguousarray(np.asarray(rng_words, dtype=np.uint64).T)
    return out


def oracle_view(sd):
    a = dict(sd)
    a["has_impact"] = sd["has_impact"]
    return a


@pytest.mark.parametrize("name", CASES)
def test_reset_matches_reference(name):
    """host numpy spawns + 45 warm-up substeps on the device + challenger / ego / pruning"""
    g = load_golden(name)
    S = len(g["seeds"])
    env = make_env(g["config"], S, autoreset_mode="Disabled", reset_mode="host")
    obs, _ = env.reset(seed=[int(s) for s in g["seeds"]])
    sd = env.state_dict()
    for i in range(S):
        compare_inter(inter_state(g, i, 0), oracle_view(sd), i, f"{name} reset#{i}", tol=1e-8)
        assert np.array_equal(sd["rng"][:, i], g["rng_words"][i, 0]), i
    assert np.max(np.abs(obs.cpu().numpy() - g["obs"][:, 0])) <= 1e-6


@pytest.mark.parametrize("name", CASES)
def test_teacher_forced_vs_reference(name):
    g = load_golden(name)
    S, T = g["actions"].shape[:2]
    env = make_env(g["config"], S, autoreset_mode="Disabled")
    env.reset(seed=0)
    for t in range(T):
        env.load_state_dict(to_sd([inter_state(g, i, t) for i in range(S)], g["rng_words"][:, t]))
        obs, rew, term, trunc, _ = env.step(g["actions"][:, t].astype(np.int32))
        sd = env.state_dict()
        obs, rew, term, trunc = obs.cpu().numpy(), rew.cpu().numpy(), term.cpu().numpy(), trunc.cpu().numpy()
        for i in range(S):
            ctx = f"{name} #{i} t={t}"
            compare_inter(inter_state(g, i, t + 1), oracle_view(sd), i, ctx, tol=1e-7)  # 32 seeds: crawling vehicles occur
            assert abs(rew[i] - g["reward"][i, t]) <= 1e-9, ctx
            assert bool(term[i]) == bool(g["terminated"][i, t]) and bool(trunc[i]) == bool(g["truncated"][i, t]), ctx
            assert np.max(np.abs(obs[i] - g["obs"][i, t + 1])) <= 1e-6, ctx
            assert np.array_equal(sd["rng"][:, i], g["rng_words"][i, t + 1]), ctx  # device PCG64 == numpy stream


@pytest.mark.parametrize("name,n,T", [("intersection_kin", 96, 10), ("intersection_grid", 64, 10), ("intersection_v2_kin", 96, 10)])
def test_teacher_forced_vs_oracle_many_envs(name, n, T):
    g = load_golden(name)
    ob = no.IntersectionOracle(no.graph_from_arrays(g), no.cfg_from_dict(g["config"]), n, g, g["config"])
    env = make_env(g["config"], n, autoreset_mode="Disabled", reset_mode="host")
    env.reset(seed=4200)
    for e in range(n):
        ob.reset_env(e, seed=4200 + e)
    sd = env.state_dict()
    # reset: same draws, same population; coordinates within the warm-up's accumulated rounding
    assert np.array_equal(sd["count"], ob.a["count"])
    for e in range(n):
        assert np.array_equal(sd["rng"][:, e], ob.rng_words(e)), e
    rng = np.random.default_rng(3)
    n_act = 3
    for t in range(T):
        state = {k: ob.a[k].copy() for k in ob.a}
        state["rng"] = np.stack([ob.rng_words(e) for e in range(n)], axis=1)
        env.load_state_dict(state)
        act = rng.integers(0, n_act, size=n).astype(np.int32)
        o_obs, o_rew, o_term, o_trunc = ob.step(act)
        obs, rew, term, trunc, _ = env.step(act)
        sd = env.state_dict()
        assert np.array_equal(sd["count"], ob.a["count"]), t
        live = np.arange(V)[None, :] < sd["count"][:, None]
        for k in ("x", "y", "heading", "speed", "timer", "target_speed", "delta"):
            assert np.max(np.abs(np.where(live, sd[k] - ob.a[k], 0.0))) <= 1e-7, (t, k)
        for k in ("lane", "target_lane", "crashed", "has_impact", "route_len", "kind", "is_yielding"):
            assert np.array_equal(np.where(live, sd[k], 0).astype(np.int32), np.where(live, ob.a[k], 0).astype(np.int32)), (t, k)
        assert np.array_equal(sd["speed_index"], ob.a["speed_index"])
        assert np.array_equal(sd["road_steps"], ob.a["road_steps"])
        for e in range(n):
            assert np.array_equal(sd["rng"][:, e], ob.rng_words(e)), (t, e)
        assert np.max(np.abs(rew.cpu().numpy() - o_rew)) <= 1e-9
        assert np.array_equal(term.cpu().numpy(), o_term.astype(bool))
        assert np.array_equal(trunc.cpu().numpy(), o_trunc.astype(bool))
        assert np.max(np.abs(obs.cpu().numpy().reshape(n, -1) - o_obs.reshape(n, -1))) <= 1e-6


def test_free_running_rollout_and_autoreset():
    """free-running episodes with SameStep autoreset: population stays within the slots, every
    finished env is replaced by a fresh `_make_vehicles` population, observations stay finite."""
    g = load_golden("intersection_kin")
    n = 48
    env = make_env(g["config"], n)
    env.reset(seed=11)
    rng = np.random.default_rng(1)
    resets = 0
    for t in range(30):
        obs, rew, term, trunc, info = env.step(rng.integers(0, 3, size=n).astype(np.int32))
        done = (term | trunc).cpu().numpy()
        resets += int(done.sum())
        sd = env.state_dict()
        assert np.all(sd["time"][done] == 0)
        assert np.all((sd["count"] >= 1) & (sd["count"] <= V))
        assert np.isfinite(obs.cpu().numpy()).all() and np.isfinite(rew.cpu().numpy()).all()
        if done.any():
            assert "final_obs" in info
    assert resets >= n


@pytest.mark.parametrize("name", CASES)
def test_device_reset_matches_host_reset(name):
    """The intersection reset (all of _make_vehicles in one kernel) against the numpy-exact host sequence:
    the same draws word for word, the same population, lanes and routes; coordinates within the rounding
    of CUDA-vs-numpy sin/cos carried through the 45 warm-up substeps."""
    g = load_golden(name)
    n = 192
    dev_env = make_env(g["config"], n, autoreset_mode="Disabled", reset_mode="device")
    host_env = make_env(g["config"], n, autoreset_mode="Disabled", reset_mode="host")
    o_d, _ = dev_env.reset(seed=900)
    o_h, _ = host_env.reset(seed=900)
    a, b = dev_env.state_dict(), host_env.state_dict()
    assert np.array_equal(a["rng"], b["rng"])
    assert np.array_equal(a["count"], b["count"])
    live = np.arange(V)[None, :] < a["count"][:, None]
    for k in ("lane", "target_lane", "kind", "route_len", "is_yielding", "crashed"):
        assert np.array_equal(np.where(live, a[k], 0), np.where(live, b[k], 0)), k
    assert np.array_equal(a["speed_index"], b["speed_index"]) and np.array_equal(a["road_steps"], b["road_steps"])
    for k in ("x", "y", "heading", "speed", "target_speed", "timer", "delta"):
        assert np.max(np.abs(np.where(live, a[k] - b[k], 0.0))) <= 1e-7, k
    assert np.max(np.abs(o_d.cpu().numpy() - o_h.cpu().numpy())) <= 1e-6
    # reference reset states: the device path reproduces the golden resets as well
    S = len(g["seeds"])
    env = make_env(g["config"], S, autoreset_mode="Disabled")
    obs, _ = env.reset(seed=[int(s) for s in g["seeds"]])
    sd = env.state_dict()
    for i in range(S):
        compare_inter(inter_state(g, i, 0), oracle_view(sd), i, f"{name} device reset#{i}", tol=1e-7)
        assert np.array_equal(sd["rng"][:, i], g["rng_words"][i, 0]), i
    assert np.max(np.abs(obs.cpu().numpy() - g["obs"][:, 0])) <= 1e-6


def test_device_autoreset_masks_only_finished_envs():
    g = load_golden("intersection_kin")
    n = 64
    env = make_env(g["config"], n)
    env.reset(seed=21)
    rng = np.random.default_rng(5)
    for t in range(20):
        before = env.state_dict()
        obs, rew, term, trunc, info = env.step(rng.integers(0, 3, size=n).astype(np.int32))
        done = (term | trunc).cpu().numpy()
        sd = env.state_dict()
        assert np.all(sd["time"][done] == 0) and np.all(sd["time"][~done] > 0)
        assert np.all(sd["road_steps"][done] == 45)
        # envs that go on keep their own generator stream: one step consumes at most a few draws,
        # a reset consumes dozens — and the inc half of the state never changes
        assert np.array_equal(sd["rng"][2:4], before["rng"][2:4])
        assert np.array_equal(info["final_obs"].cpu().numpy()[~done], obs.cpu().numpy()[~done])


def test_16_slot_and_32_slot_paths_agree():
    """The intersection step runs populations of <= 15 vehicles two per warp on 16 slots and the others on 32
    (work lists in spawn.scratch); without scratch every env takes the 32-slot kernel.  Same results bit for bit."""
    g = load_golden("intersection_grid")
    n = 256
    a = make_env(g["config"], n, autoreset_mode="Disabled")
    b = make_env(g["config"], n, autoreset_mode="Disabled")
    a.reset(seed=77)
    b.reset(seed=77)
    b._spawn_struct.scratch = None
    rng = np.random.default_rng(9)
    small = large = 0
    for t in range(16):  # runs past the 13 s horizon: populations keep growing, some beyond 15
        counts = a.state_dict()["count"]
        small += int((counts <= 15).sum())
        large += int((counts > 15).sum())
        act = rng.integers(0, 3, size=n).astype(np.int32)
        oa, ra, ta, ua, _ = a.step(act)
        ob, rb, tb, ub, _ = b.step(act)
        assert np.array_equal(oa.cpu().numpy(), ob.cpu().numpy()), t
        assert np.array_equal(ra.cpu().numpy(), rb.cpu().numpy()), t
        assert np.array_equal(ta.cpu().numpy(), tb.cpu().numpy()) and np.array_equal(ua.cpu().numpy(), ub.cpu().numpy())
        sa, sb = a.state_dict(), b.state_dict()
        live = np.arange(V)[None, :] < sa["count"][:, None]
        for k in sa:
            x, y = sa[k], sb[k]
            if x.ndim >= 2 and x.shape[:2] == (n, V):
                m = live.reshape(live.shape + (1,) * (x.ndim - 2))
                x, y = np.where(m, x, 0), np.where(m, y, 0)
            assert np.array_equal(x, y), (t, k)
    assert small > 0 and large > 0, (small, large)


@pytest.mark.parametrize("env_name", ["intersection_kin", "roundabout_kin"])
def test_next_step_autoreset_bookkeeping(env_name):
    """NEXT_STEP on the network envs: the call after an episode end returns the reset observation with reward 0
    and clear flags, the env restarts at time 0, and (intersection) the reset continues the env's generator from
    where the episode ended — the same stream the SameStep twin consumes."""
    g = load_golden(env_name)
    n = 64
    a = make_env(g["config"], n, autoreset_mode="NextStep")
    b = make_env(g["config"], n, autoreset_mode="SameStep")
    a.reset(seed=31)
    b.reset(seed=31)
    n_act = 3 if env_name.startswith("intersection") else 5
    rng = np.random.default_rng(6)
    pending = np.zeros(n, dtype=bool)
    first_done_checked = 0
    for t in range(30):
        act = rng.integers(0, n_act, size=n).astype(np.int32)
        obs, rew, term, trunc, _ = a.step(act)
        sd = a.state_dict()
        rew, term, trunc = rew.cpu().numpy(), term.cpu().numpy(), trunc.cpu().numpy()
        assert np.all(rew[pending] == 0) and not term[pending].any() and not trunc[pending].any()
        assert np.all(sd["time"][pending] == 0) and np.all(sd["time"][~pending] > 0)
        if t < 14:
            # until an env's first episode end both twins see identical histories; SameStep resets in the
            # ending step, NextStep one call later — from the same generator state, so the fresh populations match
            ob_, rb, tb, ub, _ = b.step(act)
            sb = b.state_dict()
            fresh = pending & (first_seen == t - 1) if t else pending
            for k in ("x", "y", "speed"):
                if fresh.any():
                    live = (np.arange(sd[k].shape[1])[None, :] < sd["count"][:, None]) if "count" in sd else np.ones_like(sd[k], bool)
                    assert np.allclose(np.where(live, sd[k], 0)[fresh], np.where(live, snap[k], 0)[fresh], rtol=0, atol=1e-9), (t, k)
            first_done_checked += int(fresh.sum())
            done_b = (tb | ub).cpu().numpy()
            snap = sb
            first_seen = np.where(done_b & (first_seen < 0), t, first_seen) if t else np.where(done_b, 0, -1)
        pending = term | trunc
    assert first_done_checked > 0


# ------------------------------------------------------------------ several controlled vehicles
def test_multi_agent_reset_and_teacher_forced_vs_reference():
    """intersection-multi-agent-v0 (two MDPVehicles, MultiAgentAction / MultiAgentObservation) against the
    reference: reset population, every step's state, stacked observations, mean reward, flags, per-agent info,
    generator words."""
    name = "intersection_multi_agent"
    g = load_golden(name)
    S, T = g["actions"].shape[:2]
    for mode in ("host", "device"):
        env = make_env(g["config"], S, autoreset_mode="Disabled", reset_mode=mode)
        obs, _ = env.reset(seed=[int(s) for s in g["seeds"]])
        sd = env.state_dict()
        for i in range(S):
            compare_inter(inter_state(g, i, 0), oracle_view(sd), i, f"{name} {mode} reset#{i}", tol=1e-7)
            assert np.array_equal(sd["rng"][:, i], g["rng_words"][i, 0]), i
        assert obs.shape == (S, 2, 15, 7)
        assert np.max(np.abs(obs.cpu().numpy() - g["obs"][:, 0])) <= 1e-6
    for t in range(T):
        st = to_sd([inter_state(g, i, t) for i in range(S)], g["rng_words"][:, t])
        st["speed_index"] = np.stack([np.asarray(g["speed_index"][i, t])[np.asarray(g["kind"][i, t]) == 1][:2]
                                      for i in range(S)])
        env.load_state_dict(st)
        obs, rew, term, trunc, info = env.step(g["actions"][:, t].astype(np.int32))
        sd = env.state_dict()
        obs, rew, term, trunc = obs.cpu().numpy(), rew.cpu().numpy(), term.cpu().numpy(), trunc.cpu().numpy()
        ar, at = info["agents_rewards"].cpu().numpy(), info["agents_terminated"].cpu().numpy()
        for i in range(S):
            ctx = f"{name} #{i} t={t}"
            compare_inter(inter_state(g, i, t + 1), oracle_view(sd), i, ctx, tol=1e-7)  # 32 seeds: crawling vehicles occur
            assert abs(rew[i] - g["reward"][i, t]) <= 1e-9, ctx
            assert bool(term[i]) == bool(g["terminated"][i, t]) and bool(trunc[i]) == bool(g["truncated"][i, t]), ctx
            assert np.max(np.abs(obs[i] - g["obs"][i, t + 1])) <= 1e-6, ctx
            assert np.max(np.abs(ar[i] - g["agents_rewards"][i, t])) <= 1e-9, ctx
            assert np.array_equal(at[i], g["agents_terminated"][i, t]), ctx
            assert np.array_equal(sd["rng"][:, i], g["rng_words"][i, t + 1]), ctx


def test_multi_agent_many_envs_vs_oracle_and_wrapper_ids():
    g = load_golden("intersection_multi_agent")
    n = 96
    ob = no.IntersectionOracle(no.graph_from_arrays(g), no.cfg_from_dict(g["config"]), n, g, g["config"])
    env = make_env(g["config"], n, autoreset_mode="Disabled", reset_mode="host")
    env.reset(seed=5100)
    for e in range(n):
        ob.reset_env(e, seed=5100 + e)
    rng = np.random.default_rng(12)
    for t in range(10):
        state = {k: ob.a[k].copy() for k in ob.a}
        state["rng"] = np.stack([ob.rng_words(e) for e in range(n)], axis=1)
        env.load_state_dict(state)
        act = rng.integers(0, 3, size=(n, 2)).astype(np.int32)
        o_obs, o_rew, o_term, o_trunc = ob.step(act)
        obs, rew, term, trunc, info = env.step(act)
        sd = env.state_dict()
        assert np.array_equal(sd["count"], ob.a["count"]), t
        live = np.arange(V)[None, :] < sd["count"][:, None]
        # controlled vehicles told to stop crawl at |v| < 1 m/s, where the reference's steering law divides by
        # not_zero(speed) and amplifies 1-ulp differences by ~1e6 per step (DESIGN.md section 4): 1e-5 is the bar
        for k in ("x", "y", "heading", "speed", "target_speed"):
            assert np.max(np.abs(np.where(live, sd[k] - ob.a[k], 0.0))) <= 1e-5, (t, k)
        for k in ("lane", "target_lane", "crashed", "kind", "is_yielding"):
            assert np.array_equal(np.where(live, sd[k], 0).astype(np.int32), np.where(live, ob.a[k], 0).astype(np.int32)), (t, k)
        assert np.array_equal(sd["speed_index"], ob.a["speed_index"])
        assert np.max(np.abs(rew.cpu().numpy() - o_rew)) <= 1e-9
        assert np.max(np.abs(info["agents_rewards"].cpu().numpy() - ob.agents_reward)) <= 1e-9
        assert np.array_equal(info["agents_terminated"].cpu().numpy(), ob.agents_terminated.astype(bool))
        assert np.array_equal(term.cpu().numpy(), o_term.astype(bool)) and np.array_equal(trunc.cpu().numpy(), o_trunc.astype(bool))
        assert np.max(np.abs(obs.cpu().numpy().reshape(n, -1) - o_obs.reshape(n, -1))) <= 1e-6
    # the wrapper ids return the per-agent entries; v2 adds the connected-lane search; SameStep autoreset on device
    import highwayenv_b200 as hb
    for env_id in ("intersection-multi-agent-v1", "intersection-multi-agent-v2"):
        w = hb.make(env_id, num_envs=32)
        o, _ = w.reset(seed=3)
        assert o.shape == (32, 2, 15, 7)
        for t in range(16):
            o, r, te, tr, info = w.step(rng.integers(0, 3, size=(32, 2)).astype(np.int32))
            assert r.shape == (32, 2) and te.shape == (32, 2) and tr.shape == (32,)
            assert np.isfinite(o.cpu().numpy()).all()
        assert bool(w.config["neighbour_vehicles_connected_lanes"]) == env_id.endswith("v2")
