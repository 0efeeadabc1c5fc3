"""Several controlled vehicles on highway-v0 / highway-fast-v0 (highway_multi_step_kernel, highway_multi_reset_kernel)
against the reference fixtures of oracle/gen_multi_agent_highway.py, and the multi-agent env surface."""
import json

import numpy as np
import pytest
import torch

import highwayenv_b200 as hb
import rng_craft as rc
from highwayenv_b200.envs.highway_env import ego_slots
from highwayenv_b200.envs.common.vector_env import pcg64_words
from parity_utils import FLOAT_TOL, golden_state, load_golden, well_conditioned

pytestmark = pytest.mark.gpu

STEP_CASES = ["multi_highway_v0_a2", "multi_highway_fast_a3", "multi_highway_fast_plain_action",
              "multi_highway_v0_continuous", "multi_highway_fast_ttc"]


def case(name):
    g = load_golden(name)
    return g, str(g["env_id"]), json.loads(str(g["config"]))


def make(env_id, cfg, n, autoreset="Disabled"):
    return hb.make(env_id, num_envs=n, config=cfg, device="cuda", autoreset_mode=autoreset)


def golden_sd(states, A, cont):
    """dump_state dicts (list order) -> load_state_dict payload, the controlled vehicles at ego_slots."""
    n, V = len(states), len(states[0]["x"])
    slots = ego_slots(V - A, A)
    sd = {k: np.stack([s[k] for s in states]) for k in ("x", "y", "heading", "speed", "lane", "crashed",
                                                       "check_collisions")}
    sd["target_speed"] = np.stack([np.nan_to_num(s["target_speed"]) for s in states])
    sd["timer"] = np.stack([np.nan_to_num(s["timer"]) for s in states])
    sd["delta"] = np.stack([np.nan_to_num(s["delta"], nan=4.0) for s in states])
    sd["has_impact"] = np.stack([~np.isnan(s["impact"][:, 0]) for s in states])
    sd["impact_x"] = np.stack([np.nan_to_num(s["impact"][:, 0]) for s in states])
    sd["impact_y"] = np.stack([np.nan_to_num(s["impact"][:, 1]) for s in states])
    sd["target_lane"] = np.stack([np.where(s["target_lane"] < 0, s["lane"], s["target_lane"]) for s in states])
    kind = np.zeros((n, V), dtype=np.int32)
    kind[:, slots] = 2 if cont else 1
    sd["kind"] = kind
    sd["speed_index"] = np.stack([s["speed_index"][slots] for s in states]).astype(np.int32)
    sd["time"] = np.array([float(s["time"]) for s in states])
    return sd


def check_state(st, sd, e, tol, ctx):
    for k in ("x", "y", "heading", "speed"):
        d = np.max(np.abs(st[k] - sd[k][e]))
        assert d <= tol, f"{ctx} {k} {d}"
    assert np.array_equal(st["lane"], sd["lane"][e]), ctx
    tl = np.where(st["target_lane"] < 0, st["lane"], st["target_lane"])
    assert np.array_equal(tl, sd["target_lane"][e]), ctx
    assert np.array_equal(st["crashed"].astype(bool), sd["crashed"][e].astype(bool)), ctx
    assert np.array_equal(~np.isnan(st["impact"][:, 0]), sd["has_impact"][e].astype(bool)), ctx
    idm = ~np.isnan(st["timer"])
    assert np.max(np.abs(st["timer"][idm] - sd["timer"][e][idm]), initial=0) <= tol, ctx
    ts = ~np.isnan(st["target_speed"])
    assert np.max(np.abs(st["target_speed"][ts] - sd["target_speed"][e][ts]), initial=0) <= tol, ctx


def env_actions(g, A, t):
    a = g["actions"][:, t]
    return a.astype(np.float32) if a.dtype.kind == "f" else a.astype(np.int64)


@pytest.mark.parametrize("name", STEP_CASES)
def test_reset_bit_exact(name):
    g, env_id, cfg = case(name)
    S, A = g["x"].shape[0], int(cfg["controlled_vehicles"])
    env = make(env_id, cfg, S)
    obs, _ = env.reset(seed=[int(s) for s in g["seeds"]])
    sd = env.state_dict()
    ref = golden_sd([golden_state(g, i, 0) for i in range(S)], A, _is_cont(env))
    for k in ("x", "y", "heading", "speed", "timer", "delta", "lane", "kind", "speed_index"):
        assert np.array_equal(np.asarray(sd[k]), ref[k]), k
    ts = ~np.isnan(g["target_speed"][:, 0])  # a plain Vehicle has none
    assert np.array_equal(sd["target_speed"][ts], g["target_speed"][:, 0][ts])
    assert np.array_equal(env.rng_words(), g["rng_words"][:, 0].T)
    assert np.array_equal(obs.cpu().numpy(), g["obs"][:, 0])


def test_resets_fixture_bit_exact():
    g = load_golden("multi_highway_resets")
    for c in range(int(g["n_configs"])):
        cfg, env_id = json.loads(str(g[f"c{c}_config"])), str(g[f"c{c}_env_id"])
        seeds = [int(s) for s in g[f"c{c}_seeds"]]
        A = int(cfg["controlled_vehicles"])
        for autoreset in ("Disabled", "SameStep"):
            env = make(env_id, cfg, len(seeds), autoreset)
            obs, _ = env.reset(seed=seeds)
            sd = env.state_dict()
            ref = golden_sd([{k: g[f"c{c}_{k}"][i] for k in ("x", "y", "heading", "speed", "target_speed", "timer",
                                                                "delta", "lane", "target_lane", "crashed", "impact",
                                                                "check_collisions", "speed_index", "time")}
                             for i in range(len(seeds))], A, False)
            for k in ("x", "y", "heading", "speed", "target_speed", "timer", "delta", "lane", "kind",
                      "check_collisions", "speed_index"):
                assert np.array_equal(np.asarray(sd[k]), ref[k]), (c, k)
            assert np.array_equal(env.rng_words(), g[f"c{c}_rng_words"].T), c
            assert np.array_equal(obs.cpu().numpy(), g[f"c{c}_obs"]), c


def _is_cont(env):
    return env.action_type.kernel_action_type == 1


@pytest.mark.parametrize("name", STEP_CASES)
def test_teacher_forced(name):
    g, env_id, cfg = case(name)
    S, T = g["actions"].shape[:2]
    A = int(cfg["controlled_vehicles"])
    env = make(env_id, cfg, S)
    env.reset(seed=0)
    for t in range(T):
        sd = golden_sd([golden_state(g, i, t) for i in range(S)], A, _is_cont(env))
        sd["rng"] = g["rng_words"][:, t].T
        env.load_state_dict(sd)
        obs, rew, term, trunc, _ = env.step(env_actions(g, A, t))
        got = env.state_dict()
        ref = golden_sd([golden_state(g, i, t + 1) for i in range(S)], A, _is_cont(env))
        for e in range(S):
            check_state(golden_state(g, e, t + 1), got, e, FLOAT_TOL, f"{name} seed {e} step {t}")
        assert np.array_equal(got["speed_index"], ref["speed_index"]), (name, t)
        assert np.max(np.abs(obs.cpu().numpy() - g["obs"][:, t + 1])) <= FLOAT_TOL, (name, t)
        assert np.max(np.abs(rew.cpu().numpy() - g["reward"][:, t])) <= FLOAT_TOL, (name, t)
        assert np.array_equal(term.cpu().numpy(), g["terminated"][:, t]), (name, t)
        assert np.array_equal(trunc.cpu().numpy(), g["truncated"][:, t]), (name, t)


@pytest.mark.parametrize("name", STEP_CASES)
def test_free_running(name):
    """Disabled autoreset from the seeded reset, over each seed's well-conditioned prefix; stream words on every step
    (a highway step draws nothing)."""
    g, env_id, cfg = case(name)
    S, T = g["actions"].shape[:2]
    A = int(cfg["controlled_vehicles"])
    env = make(env_id, cfg, S)
    env.reset(seed=[int(s) for s in g["seeds"]])
    alive = np.ones(S, dtype=bool)
    compared = 0
    for t in range(T):
        obs, rew, term, trunc, _ = env.step(env_actions(g, A, t))
        got = env.state_dict()
        assert np.array_equal(env.rng_words(), g["rng_words"][:, t + 1].T)
        for e in range(S):
            alive[e] = alive[e] and well_conditioned(golden_state(g, e, t + 1))
            if not alive[e]:
                continue
            compared += 1
            check_state(golden_state(g, e, t + 1), got, e, FLOAT_TOL, f"{name} seed {e} step {t}")
            assert abs(float(rew[e]) - g["reward"][e, t]) <= FLOAT_TOL
            assert bool(term[e]) == bool(g["terminated"][e, t])
            assert np.max(np.abs(obs[e].cpu().numpy() - g["obs"][e, t + 1])) <= FLOAT_TOL
    assert compared >= S, compared


def _end_all(env):
    env._time.fill_(float(env.config["duration"]) - 1.0 / env.config["policy_frequency"])


def _reset_configs():
    g = load_golden("multi_highway_resets")
    return [(str(g[f"c{c}_env_id"]), json.loads(str(g[f"c{c}_config"]))) for c in range(int(g["n_configs"]))]


def test_fused_respawn_matches_the_reset_fixture():
    """The SameStep respawn inside the step kernel, from the streams the fixture's seeds give, equals the reference's
    reset bit for bit: state, stream words after the spawn and observation.  Covers every configuration of the reset
    fixture, with and without initial_lane_id, A = 8 and empty near_split bins."""
    g = load_golden("multi_highway_resets")
    for c in range(int(g["n_configs"])):
        cfg, env_id = json.loads(str(g[f"c{c}_config"])), str(g[f"c{c}_env_id"])
        seeds = [int(s) for s in g[f"c{c}_seeds"]]
        A = int(cfg["controlled_vehicles"])
        env = make(env_id, cfg, len(seeds), "SameStep")
        env.reset(seed=seeds)
        words = pcg64_words([np.random.Generator(np.random.PCG64(np.random.SeedSequence(s))) for s in seeds])
        env._rng.copy_(torch.from_numpy(words.view(np.int64)).to(env.device))
        _end_all(env)
        obs, _, _, trunc, _ = env.step(np.ones((len(seeds), A), np.int64))
        assert bool(trunc.all()), c
        sd = env.state_dict()
        ref = golden_sd([{k: g[f"c{c}_{k}"][i] for k in ("x", "y", "heading", "speed", "target_speed", "timer",
                                                            "delta", "lane", "target_lane", "crashed", "impact",
                                                            "check_collisions", "speed_index", "time")}
                         for i in range(len(seeds))], A, False)
        for k in ("x", "y", "heading", "speed", "target_speed", "timer", "delta", "lane", "kind",
                  "check_collisions", "speed_index"):
            assert np.array_equal(np.asarray(sd[k]), ref[k]), (c, k)
        assert np.array_equal(env.rng_words(), g[f"c{c}_rng_words"].T), c
        assert np.array_equal(obs.cpu().numpy(), g[f"c{c}_obs"]), c


FUSED_CASES = ["multi_highway_v0_a2", "multi_highway_fast_a3", "multi_highway_v0_continuous", "reset:4", "reset:5",
               "reset:7"]


@pytest.mark.parametrize("name", FUSED_CASES)
def test_fused_autoreset_equals_standalone_reset(name):
    """SameStep respawn inside the step kernel == hwy_highway_reset of the same stream words, bit for bit, streams
    included ("reset:k": configuration k of the reset fixture; 4, 5 and 7 set initial_lane_id).  Where a lane draw can
    be rejected (3 lanes: only the word 0; numpy never rejects with 4), every third env's words are crafted so that
    output 0's low half is a rejected word (the serial fallback when the first controlled vehicle draws a lane)."""
    if name.startswith("reset:"):
        env_id, cfg = _reset_configs()[int(name[6:])]
    else:
        _, env_id, cfg = case(name)
    A = int(cfg["controlled_vehicles"])
    n = 48
    a = make(env_id, cfg, n, "SameStep")
    b = make(env_id, cfg, n, "Disabled")
    a.reset(seed=7)
    words = a.rng_words()
    L = int(a.config["lanes_count"])
    low = next((x for x in range(0, 1 << 16) if rc.lemire_rejects(x, L)), None)
    for e in range(0, n, 3) if low is not None else ():
        inc = int(words[2, e]) << 64 | int(words[3, e])
        words[:, e] = rc.words_of(rc.crafted_state(low, inc, m=0, seed=e), inc, 0, 0)
    a._rng.copy_(torch.from_numpy(words.view(np.int64)).to(a.device))
    _end_all(a)
    act = np.zeros((n, A, 2), np.float32) if _is_cont(a) else np.ones((n, A), np.int64)
    obs_a, _, _, trunc, _ = a.step(act)
    assert bool(trunc.all())
    b.reset(seed=0)
    b._rng.copy_(torch.from_numpy(words.view(np.int64)).to(b.device))
    obs_b, _ = b.reset()
    sa, sb = a.state_dict(), b.state_dict()
    for k in sa:
        if k != "time":
            assert np.array_equal(np.asarray(sa[k]), np.asarray(sb[k])), k
    assert np.array_equal(a.rng_words(), b.rng_words())
    assert np.array_equal(obs_a.cpu().numpy(), obs_b.cpu().numpy())


def test_single_agent_equivalence_and_plain_rows():
    """A = 1 under both switches equals the single-agent env; plain obs = agent 0's row of the MultiAgentObservation
    twin; MultiAgentAction(DiscreteAction) = MultiAgentAction(ContinuousAction) fed the table's rows."""
    n = 64
    one = make("highway-fast-v0", {"controlled_vehicles": 1, "action": {"type": "MultiAgentAction", "action_config": {
        "type": "DiscreteMetaAction"}}, "observation": {"type": "MultiAgentObservation", "observation_config": {
            "type": "Kinematics"}}}, n)
    ref = make("highway-fast-v0", {}, n)
    o1, _ = one.reset(seed=3)
    o2, _ = ref.reset(seed=3)
    assert tuple(o1.shape) == (n, 1, 5, 5) and torch.equal(o1[:, 0], o2)
    rng = np.random.default_rng(0)
    for _ in range(5):
        a = rng.integers(0, 5, size=n)
        r1, r2 = one.step(a[:, None]), ref.step(a)
        assert torch.equal(r1[0][:, 0], r2[0]) and torch.equal(r1[1], r2[1])
    multi = {"controlled_vehicles": 3, "action": {"type": "MultiAgentAction", "action_config": {
        "type": "DiscreteMetaAction"}}, "observation": {"type": "MultiAgentObservation", "observation_config": {
            "type": "Kinematics"}}}
    plain = dict(multi, observation={"type": "Kinematics"})
    m, p = make("highway-fast-v0", multi, n), make("highway-fast-v0", plain, n)
    om, _ = m.reset(seed=11)
    op, _ = p.reset(seed=11)
    assert torch.equal(om[:, 0], op)
    for _ in range(5):
        a = rng.integers(0, 5, size=(n, 3))
        om, op = m.step(a)[0], p.step(a)[0]
        assert torch.equal(om[:, 0], op)
    da = {"controlled_vehicles": 2, "action": {"type": "MultiAgentAction", "action_config": {"type": "DiscreteAction"}},
          "observation": {"type": "Kinematics"}}
    ca = dict(da, action={"type": "MultiAgentAction", "action_config": {"type": "ContinuousAction"}})
    d, c = make("highway-v0", da, n), make("highway-v0", ca, n)
    d.reset(seed=5)
    c.reset(seed=5)
    table = d.action_type.table
    for _ in range(4):
        k = rng.integers(0, len(table), size=(n, 2))
        od, oc = d.step(k)[0], c.step(table[k])[0]
        assert torch.equal(od, oc)


def test_env_machinery():
    cfg = {"controlled_vehicles": 2, "action": {"type": "MultiAgentAction", "action_config": {
        "type": "DiscreteMetaAction"}}, "observation": {"type": "MultiAgentObservation", "observation_config": {
            "type": "Kinematics"}}}
    n = 32
    rng = np.random.default_rng(1)
    acts = [rng.integers(0, 5, size=(n, 2)) for _ in range(6)]
    # NextStep == a Disabled twin plus an explicit masked reset of the envs that ended in the previous step
    nxt, dis = make("highway-fast-v0", cfg, n, "NextStep"), make("highway-fast-v0", cfg, n, "Disabled")
    for env in (nxt, dis):
        env.reset(seed=2)
        env._time[::2] = float(env.config["duration"]) - 1.0 / env.config["policy_frequency"]  # even envs end now
    ended = None
    for a in acts:
        on, rn, tn, un, _ = nxt.step(a)
        od, rd, td, ud, _ = dis.step(a)
        if ended is not None and ended.any():
            od, _ = dis.reset(options={"reset_mask": ended})
            keep = torch.from_numpy(~ended).to(rd.device)
            rd, td, ud = rd * keep, td & keep, ud & keep
        assert tuple(on.shape) == (n, 2, 5, 5)
        assert torch.equal(on, od) and torch.equal(rn, rd) and torch.equal(tn, td) and torch.equal(un, ud)
        sn, sdd = nxt.state_dict(), dis.state_dict()
        for k in sn:
            assert np.array_equal(np.asarray(sn[k]), np.asarray(sdd[k])), k
        ended = (td | ud).cpu().numpy()
    assert ended is not None
    env = make("highway-fast-v0", cfg, n, "SameStep")
    env.reset(seed=4)
    env.step(acts[0])
    sd = env.state_dict()
    assert sd["speed_index"].shape == (n, 2)
    twin = make("highway-fast-v0", cfg, n, "SameStep")
    twin.reset(seed=9)
    twin.load_state_dict(sd)
    clone = make("highway-fast-v0", cfg, n, "SameStep")
    clone.reset(seed=10)
    clone.copy_envs(np.arange(n), np.arange(n), source=env)
    for a in acts[1:]:
        r0, r1, r2 = env.step(a), twin.step(a), clone.step(a)
        for r in (r1, r2):
            assert torch.equal(r0[0], r[0]) and torch.equal(r0[1], r[1])
    # available actions per agent
    av = env.get_available_actions()
    assert tuple(av.shape) == (n, 2, 5) and bool(av[:, :, 1].all())
    # host stepper graph against eager steps
    e1, e2 = make("highway-fast-v0", cfg, n, "SameStep"), make("highway-fast-v0", cfg, n, "SameStep")
    e1.reset(seed=6)
    e2.reset(seed=6)
    hs = e1.host_stepper()
    for a in acts:
        hs.actions[:] = a
        out = hs.step()
        ref = e2.step(a)
        assert np.array_equal(np.asarray(out[0]), ref[0].cpu().numpy())
    # the host stepper under MultiAgentAction(DiscreteAction): one index per env and agent
    da = dict(cfg, action={"type": "MultiAgentAction", "action_config": {"type": "DiscreteAction"}})
    e1, e2 = make("highway-v0", da, n, "SameStep"), make("highway-v0", da, n, "SameStep")
    e1.reset(seed=8)
    e2.reset(seed=8)
    hs = e1.host_stepper()
    assert hs.actions.shape == (n, 2)
    for _ in range(4):
        k = rng.integers(0, len(e1.action_type.table), size=(n, 2))
        hs.actions[:] = k
        out = hs.step()
        ref = e2.step(k)
        assert np.array_equal(np.asarray(out[0]), ref[0].cpu().numpy())
        assert np.array_equal(np.asarray(out[1]), ref[1].cpu().numpy())
    # single-env wrapper against row 0 of a batched twin
    s = hb.make_single("highway-fast-v0", config=cfg, device="cuda")
    b1 = make("highway-fast-v0", cfg, 1, "Disabled")
    o, _ = s.reset(seed=0)
    ob, _ = b1.reset(seed=0)
    assert np.asarray(o).shape == (2, 5, 5) and np.array_equal(np.asarray(o), ob[0].cpu().numpy())
    for a in acts[:3]:
        o, r, *_ = s.step(a[0])
        ob, rb, *_ = b1.step(a[:1])
        assert np.array_equal(np.asarray(o), ob[0].cpu().numpy()) and r == float(rb[0])
    # road_substeps with per-agent continuous actions
    cc = dict(cfg, action={"type": "MultiAgentAction", "action_config": {"type": "ContinuousAction"}})
    env = make("highway-v0", cc, n)
    env.reset(seed=1)
    env.road_substeps(3, torch.zeros(n, 2, 2, device="cuda"))


def test_batch_independence():
    cfg = {"controlled_vehicles": 3, "action": {"type": "MultiAgentAction", "action_config": {
        "type": "DiscreteMetaAction"}}, "observation": {"type": "MultiAgentObservation", "observation_config": {
            "type": "Kinematics"}}}
    big = make("highway-fast-v0", cfg, 65536)
    big.reset(seed=0)
    rng = np.random.default_rng(3)
    acts = [rng.integers(0, 5, size=(65536, 3)) for _ in range(4)]
    ids = [0, 777, 65535]
    outs = [big.step(a)[0][ids].cpu().numpy() for a in acts]
    for k, e in enumerate(ids):
        one = make("highway-fast-v0", cfg, 1)
        one.reset(seed=[e])
        for t, a in enumerate(acts):
            o = one.step(a[e:e + 1])[0]
            assert np.array_equal(o[0].cpu().numpy(), outs[t][k]), (e, t)
