"""The rare paths of the highway spawn, end to end.  A Lemire rejection in a lane choice (p = 2^-32 per draw) sends the
fused SameStep autoreset of the step kernel to its serial fallback (thread 0 stages the spawn through HBM and rewrites
the stream words); random seeds never get there.  Crafted generator words (tests/rng_craft.py) injected through
load_state_dict put a 32-bit word 0 exactly where a chosen vehicle's lane choice reads it, and the C oracle, given the
same generator state, is the reference: states, observations and all 5 generator words bit for bit.  The same states
go through the standalone reset kernel (hwy_highway_reset, the serial choice loop) and the NextStep autoreset, and
the fused autoreset runs on the configurations the parity suite does not reset: 128 vehicles (vehicles_count = 127:
every thread of the env spawns, and the jump table is read up to its largest indices), 1, 2 and 5 lanes, and a fixed
ego lane (the ego draws no lane, which flips the parity of the requests).

Two network families draw `choice` and `normal` (the ziggurat): the roundabout reset kernel against the numpy-exact
host spawn, and the intersection's per-step _spawn_vehicle against the oracle's numpy restatement, each from crafted
words that put a Lemire rejection, a ziggurat wedge or a ziggurat tail into the draws."""
import numpy as np
import pytest

import hwy_oracle as ho
import net_oracle as no
import rng_craft as rc
from parity_utils import FLOAT_TOL, load_golden

pytestmark = pytest.mark.gpu

F64 = ("x", "y", "heading", "speed", "target_speed", "timer", "delta")
I32 = ("lane", "target_lane", "kind", "crashed", "check_collisions")
LOW0, HIGH0, OTHER_HALF = 0x5A5A5A5A << 32, 0x5A5A5A5A, 0x77777777  # a 64-bit word with its low / high half 0


def make_pair(n, seed, mode="SameStep", **over):
    """highway-fast-v0 (with `over`) on the device and in the C oracle, both reset from the same seeds"""
    import highwayenv_b200 as hb

    cfg = dict(load_golden("highway_fast_v20")["config"])
    cfg.update(over)
    oc = ho.cfg_from_dict(cfg)
    ob = ho.OracleBatch(oc, n, seeds=range(seed, seed + n), threads=8)
    env_cfg = {k: v for k, v in cfg.items() if not k.startswith("_")}
    env = hb.make(cfg["_env_id"], num_envs=n, config=env_cfg, autoreset_mode=mode)
    env.reset(seed=seed)
    ob.reset()
    return cfg, oc, ob, env


def words_of_oracle(ob):
    r = ob.rng
    return np.stack([r["state_hi"], r["state_lo"], r["inc_hi"], r["inc_lo"],
                     (r["has_uint32"].astype(np.uint64) << np.uint64(32)) | r["uinteger"].astype(np.uint64)])


def set_oracle_words(ob, w):
    ob.rng["state_hi"], ob.rng["state_lo"], ob.rng["inc_hi"], ob.rng["inc_lo"] = w[0], w[1], w[2], w[3]
    ob.rng["has_uint32"] = (w[4] >> np.uint64(32)).astype(np.uint32)
    ob.rng["uinteger"] = (w[4] & np.uint64(0xFFFFFFFF)).astype(np.uint32)


def crafted_rejections(ob, envs, V, L, ego_draws_lane=True):
    """Rewrite the generator words of the given envs so that one lane choice of the next spawn reads a 32-bit 0:
    (a) the ego's buffered half, (b) a fresh low half at vehicle k, (c) the high half vehicle k-1 opened, for
    k in {1, V // 2, V - 1}.  Returns the words [5][n] and the case of every env."""
    assert rc.lemire_rejects(0, L)  # L is not a power of two
    w = words_of_oracle(ob).copy()
    cases = [("buffered", 0)] + [(h, k) for k in (1, V // 2, V - 1) for h in ("low", "high")]
    out = {}
    for e, (half, k) in zip(envs, cases * (len(envs) // len(cases) + 1)):
        inc = (int(w[2, e]) << 64) | int(w[3, e])
        state = (int(w[0, e]) << 64) | int(w[1, e])
        if half == "buffered":
            new = rc.words_of(state, inc, 1, 0)
        else:
            has = next(h for h in (0, 1) if any(v == k and hf == half for v, _, hf in rc.spawn_requests(V, L, h, ego_draws_lane)))
            out_idx = next(o for v, o, hf in rc.spawn_requests(V, L, has, ego_draws_lane) if v == k)
            new = rc.words_of(rc.crafted_state(LOW0 if half == "low" else HIGH0, inc, m=out_idx, seed=e), inc, has,
                              OTHER_HALF)
            g = rc.generator_of(new)  # the word really is where vehicle k's choice reads it
            raw = g.bit_generator.random_raw(out_idx + 1)
            assert (int(raw[-1]) >> (0 if half == "low" else 32)) & 0xFFFFFFFF == 0
        w[:, e] = new
        out[e] = (half, k)
    return w, out


def state_of_oracle(ob):
    return {k: ob.a[k].copy() for k in ob.a}


def assert_same_envs(sd, ob, mask, what):
    for k in F64:
        assert np.array_equal(sd[k][mask].view(np.uint64), ob.a[k][mask].view(np.uint64)), (what, k)
    for k in I32:
        assert np.array_equal(sd[k][mask].astype(np.int64), ob.a[k][mask].astype(np.int64)), (what, k)
    assert np.array_equal(sd["speed_index"][mask], ob.a["speed_index"][mask]), what
    assert np.array_equal(sd["time"][mask], ob.a["time"][mask]), what


def assert_same_words(sd, ob, what):
    got, want = sd["rng"], words_of_oracle(ob)
    bad = np.nonzero((got != want).any(axis=0))[0]
    assert bad.size == 0, f"{what}: generator words differ in envs {bad[:8]} (word rows {np.nonzero((got != want).any(1))[0]})"


def _end_now(ob, envs, cfg):
    ob.a["time"][envs] = float(cfg["duration"]) - 1.0 / cfg["policy_frequency"]  # truncated by this step


@pytest.mark.parametrize("lanes", [3, 5])
def test_fused_autoreset_serial_fallback(lanes):
    """Rejecting envs, plain resets (the parallel path) and running envs in one launch."""
    n = 48
    cfg, oc, ob, env = make_pair(n, 41000, lanes_count=lanes)
    V, L = int(oc.n_vehicles), int(oc.lanes_count)
    crafted_envs = list(range(0, n, 3))            # every third env: a rejection
    plain_reset = list(range(1, n, 3))             # ends without one
    w, cases = crafted_rejections(ob, crafted_envs, V, L)
    set_oracle_words(ob, w)
    _end_now(ob, crafted_envs + plain_reset, cfg)
    sd_in = state_of_oracle(ob)
    sd_in["rng"] = w
    env.load_state_dict(sd_in)
    act = np.ones(n, dtype=np.int32)
    o_obs, _, o_term, o_trunc = ob.step(act, autoreset=True)
    obs, _, term, trunc, _ = env.step(act)
    done = (o_term | o_trunc).astype(bool)
    assert done[crafted_envs].all() and done[plain_reset].all()
    assert np.array_equal((term | trunc).cpu().numpy(), done)
    sd = env.state_dict()
    assert_same_envs(sd, ob, done, "fused autoreset")
    assert np.array_equal(obs.cpu().numpy()[done], o_obs[done])
    assert_same_words(sd, ob, "fused autoreset")
    assert len(set(cases.values())) == 7  # every case of crafted_rejections is in the batch


def test_reset_kernel_and_next_step_with_rejections():
    n = 42
    cfg, oc, ob, env = make_pair(n, 42000)
    V, L = int(oc.n_vehicles), int(oc.lanes_count)
    envs = list(range(0, n, 2))
    w, _ = crafted_rejections(ob, envs, V, L)
    # standalone reset of the masked envs (hwy_highway_reset: one thread walks the draws)
    set_oracle_words(ob, w)
    sd_in = state_of_oracle(ob)
    sd_in["rng"] = w
    env.load_state_dict(sd_in)
    mask = np.zeros(n, dtype=np.uint8)
    mask[envs] = 1
    o_obs = ob.reset(mask=mask).copy()
    obs, _ = env.reset(options={"reset_mask": mask})
    sd = env.state_dict()
    assert_same_envs(sd, ob, mask.astype(bool), "reset kernel")
    assert np.array_equal(obs.cpu().numpy()[mask.astype(bool)], o_obs[mask.astype(bool)])
    assert_same_words(sd, ob, "reset kernel")

    # NextStep: the envs that end in one step are reset by the next call
    cfg2, oc2, ob2, env2 = make_pair(n, 43000, mode="NextStep")
    w2, _ = crafted_rejections(ob2, envs, V, L)
    set_oracle_words(ob2, w2)
    _end_now(ob2, envs, cfg2)
    sd_in = state_of_oracle(ob2)
    sd_in["rng"] = w2
    env2.load_state_dict(sd_in)
    act = np.ones(n, dtype=np.int32)
    _, _, o_term, o_trunc = ob2.step(act)
    _, _, term, trunc, _ = env2.step(act)
    pending = (o_term | o_trunc).astype(bool)
    assert pending[envs].all() and np.array_equal((term | trunc).cpu().numpy(), pending)
    # stepping draws nothing on the highway, so the next call resets them from the crafted words
    o_obs2 = ob2.reset(mask=pending.astype(np.uint8)).copy()
    obs2, _, _, _, _ = env2.step(act)
    sd2 = env2.state_dict()
    assert_same_envs(sd2, ob2, pending, "NextStep reset")
    assert np.array_equal(obs2.cpu().numpy()[pending], o_obs2[pending])
    assert_same_words(sd2, ob2, "NextStep reset")


@pytest.mark.parametrize("over", [{"vehicles_count": 127}, {"lanes_count": 1}, {"lanes_count": 2},
                                  {"lanes_count": 5}, {"initial_lane_id": 1}],
                         ids=["v128", "lanes1", "lanes2", "lanes5", "ego_lane1"])
def test_fused_autoreset_other_configs(over):
    """No rejection: the parallel spawn at the largest jump indices, other lane counts, and a fixed ego lane, from
    both parities of the buffered half."""
    n = 32
    cfg, oc, ob, env = make_pair(n, 44000, **over)
    w = words_of_oracle(ob).copy()
    r = np.random.default_rng(0)
    has = r.integers(0, 2, n).astype(np.uint64)
    w[4] = (has << np.uint64(32)) | r.integers(1 << 20, 1 << 32, n).astype(np.uint64)
    set_oracle_words(ob, w)
    ends = list(range(0, n, 4)) + list(range(1, n, 4)) + list(range(2, n, 4))
    _end_now(ob, ends, cfg)
    env.load_state_dict({**state_of_oracle(ob), "rng": w})
    act = np.ones(n, dtype=np.int32)
    o_obs, _, o_term, o_trunc = ob.step(act, autoreset=True)
    obs, _, term, trunc, _ = env.step(act)
    done = (o_term | o_trunc).astype(bool)
    assert done[ends].all()
    sd = env.state_dict()
    assert_same_envs(sd, ob, done, str(over))
    assert np.array_equal(obs.cpu().numpy()[done], o_obs[done])
    assert_same_words(sd, ob, str(over))


# ------------------------------------------------------------------ network families: choice and normal
def _tail_value_ok(got, want):
    """a tail sample goes through CUDA's log1p and may differ from numpy's by an ulp (tests/test_gpu_rng_streams.py)"""
    return got == want or abs(got - want) <= np.spacing(abs(want))


def _crafted_roundabout_words(n, fixed_dest):
    """Per env one case of the roundabout spawn's draws (per traffic vehicle: normal, normal, choice(3), uniform):
    the first normal in the tail (+ / -) or the wedge, the first choice reading a buffered 0 or a fresh low half 0,
    and a tail together with a buffered 0.  Every case is checked on numpy before use."""
    cases = ["tail+", "tail-", "wedge", "buffered0", "low0", "tail+buffered0", "plain"]
    words, kinds = np.zeros((5, n), dtype=np.uint64), []
    for e in range(n):
        kind = cases[e % len(cases)]
        state, inc = rc.seeded_state(46000 + e)
        for attempt in range(64):
            has, u = (1, 0) if "buffered0" in kind else (0, 0)
            if kind.startswith("tail"):
                st = rc.crafted_state(rc.ziggurat_tail_word(kind.startswith("tail-")), inc, m=0, seed=e * 64 + attempt)
            elif kind == "wedge":
                st = rc.crafted_state(rc.ziggurat_word(1 + (e * 7 + attempt) % 255), inc, m=0, seed=e * 64 + attempt)
            elif kind == "low0":
                st = rc.crafted_state(LOW0, inc, m=2, seed=e * 64 + attempt)  # after two fast-path normals
            else:
                st = rc.step_back(state, inc, attempt)
            g = rc.make_generator(st, inc, has, u)
            x0 = g.normal()
            g.normal()
            if fixed_dest is not None:  # the first vehicle draws no destination: the first choice is vehicle 2's
                g.uniform()
                g.normal()
                g.normal()
            first32 = int(g.integers(0, 1 << 32, dtype=np.uint32))
            ok = {"tail+": x0 >= rc.ZIGGURAT_NOR_R, "tail-": x0 <= -rc.ZIGGURAT_NOR_R,
                  "wedge": abs(x0) < rc.ZIGGURAT_NOR_R,
                  "buffered0": first32 == 0, "low0": first32 == 0,
                  "tail+buffered0": x0 >= rc.ZIGGURAT_NOR_R and first32 == 0, "plain": first32 != 0}[kind]
            if kind == "wedge":  # the wedge: the first normal consumes more than its own output
                probe = rc.make_generator(st, inc)
                probe.normal()
                ok = ok and _outputs_used(st, inc, probe) >= 2
            if ok:
                break
        else:
            raise AssertionError(f"no state found for {kind}")
        words[:, e] = rc.words_of(st, inc, has, u)
        kinds.append(kind)
    return words, kinds


def _outputs_used(state, inc, g_after, limit=32):
    probe = rc.make_generator(state, inc)
    target = g_after.bit_generator.state["state"]["state"]
    for k in range(limit + 1):
        if probe.bit_generator.state["state"]["state"] == target:
            return k
        probe.bit_generator.random_raw()
    return limit + 1


def test_roundabout_reset_from_crafted_words():
    """hwy_roundabout_reset (device Pcg64::normal / choice) against the numpy-exact host spawn on the same crafted
    streams: draws, lanes, routes and all 5 generator words bit for bit; positions within the sin/cos rounding."""
    import highwayenv_b200 as hb

    g = load_golden("roundabout_ttc")
    cfg = {k: v for k, v in g["config"].items() if not k.startswith("_")}
    n = 70
    dev = hb.make(g["config"]["_env_id"], num_envs=n, config=cfg, reset_mode="device")
    host = hb.make(g["config"]["_env_id"], num_envs=n, config=cfg, reset_mode="host")
    dev.reset(seed=1)
    host.reset(seed=1)
    words, kinds = _crafted_roundabout_words(n, cfg.get("incoming_vehicle_destination"))
    for env in (dev, host):
        sd = env.state_dict()
        sd["rng"] = words
        env.load_state_dict(sd)
        assert np.array_equal(env.rng_words(), words)
    o_d, _ = dev.reset()
    o_h, _ = host.reset()
    a, b = dev.state_dict(), host.state_dict()
    wd, wh = dev.rng_words(), host.rng_words()
    bad = np.nonzero((wd != wh).any(axis=0))[0]
    assert bad.size == 0, f"generator words differ in envs {bad} ({[kinds[e] for e in bad]})"
    for k in ("lane", "target_lane", "route", "route_len", "kind", "speed_index"):
        assert np.array_equal(a[k], b[k]), k
    assert np.array_equal(a["delta"], b["delta"])
    for e in range(n):
        for v in range(a["speed"].shape[1]):
            assert _tail_value_ok(a["speed"][e, v], b["speed"][e, v]), (e, kinds[e], v)
    for k in ("x", "y", "heading", "timer"):
        assert np.max(np.abs(a[k] - b[k])) <= 1e-12, k
    assert np.max(np.abs(o_d.cpu().numpy() - o_h.cpu().numpy())) <= 1e-6
    assert len(set(kinds)) == 7  # every case is in the batch


def test_intersection_spawn_vehicle_from_crafted_words():
    """IntersectionEnv.step's _spawn_vehicle on the device (uniform, choice(range(4), 2, replace=False) = Floyd's two
    bounded draws + a masked shuffle draw, two normals) against the oracle's numpy restatement, from crafted words: a
    Lemire rejection in the first bounded draw, a tail and a wedge in the longitudinal normal."""
    import highwayenv_b200 as hb

    g = load_golden("intersection_kin")
    cfg = g["config"]
    n = 64
    ob = no.IntersectionOracle(no.graph_from_arrays(g), no.cfg_from_dict(cfg), n, g, cfg)
    env = hb.make(cfg["_env_id"], num_envs=n, config={k: v for k, v in cfg.items() if not k.startswith("_")},
                  autoreset_mode="Disabled")
    env.reset(seed=47000)
    sd = env.state_dict()
    for k in ob.a:
        if k in sd:
            ob.a[k][...] = sd[k].reshape(ob.a[k].shape)
    p = float(cfg["spawn_probability"])
    cases = ["reject", "tail+", "tail-", "wedge"]
    words = sd["rng"].copy()
    kinds = []
    for e in range(n):
        kind = cases[e % len(cases)]
        inc = (int(words[2, e]) << 64) | int(words[3, e])
        for attempt in range(256):
            s = e * 256 + attempt
            if kind == "reject":  # uniform ~ 0 (spawn), buffered 32-bit half 0: the first bounded draw rejects
                st, has, u = rc.crafted_state(0x400, inc, m=0, seed=s), 1, 0
            else:  # the normal after uniform + three 32-bit draws (outputs 1 and 2 low): output 3
                word = rc.ziggurat_tail_word(kind == "tail-") if kind.startswith("tail") else rc.ziggurat_word(1 + s % 255)
                st, has, u = rc.crafted_state(word, inc, m=3, seed=s), 0, 0
            gen = rc.make_generator(st, inc, has, u)
            if gen.uniform() > p:
                continue
            if kind == "reject":
                ok = True
            else:
                gen.choice(range(4), size=2, replace=False)
                before = rc.words_of(gen)
                x = gen.normal()
                used = _outputs_used((int(before[0]) << 64) | int(before[1]), inc, gen)
                ok = (abs(x) >= rc.ZIGGURAT_NOR_R) if kind.startswith("tail") else (used >= 2 and abs(x) < rc.ZIGGURAT_NOR_R)
            if ok:
                break
        else:
            raise AssertionError(f"no state for {kind}")
        words[:, e] = rc.words_of(st, inc, has, u)
        kinds.append(kind)
    sd["rng"] = words
    env.load_state_dict(sd)
    for e in range(n):
        ob.set_rng_words(e, words[:, e])
    act = np.ones(n, dtype=np.int32)
    ob.step(act)
    env.step(act)
    sd = env.state_dict()
    for e in range(n):
        assert np.array_equal(sd["rng"][:, e], ob.rng_words(e)), (e, kinds[e])
    assert np.array_equal(sd["count"], ob.a["count"])
    V = ob.a["count"].max()
    live = np.arange(ob.a["x"].shape[1])[None, :] < ob.a["count"][:, None]
    for k in ("lane", "target_lane", "route_len", "kind", "crashed"):
        assert np.array_equal(np.where(live, sd[k], 0).astype(np.int64), np.where(live, ob.a[k], 0).astype(np.int64)), k
    for k in ("x", "y", "heading", "speed", "target_speed", "delta"):
        assert np.max(np.abs(np.where(live, sd[k] - ob.a[k], 0.0))) <= FLOAT_TOL, k
    assert V > 0 and len(set(kinds)) == 4
