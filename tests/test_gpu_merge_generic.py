"""merge-generic-v0 / v1 on the GPU against the fixtures of the unmodified reference (oracle/gen_merge_generic.py):
device resets, teacher-forced windows and free-running SameStep rollouts (the 32-slot step with an Obstacle and the
merge reward included), get_available_actions, crafted streams, masked resets, state round trips, the host_stepper
graph, reconfiguration, make_single and 4096-env runs."""
import json
import os

import numpy as np
import pytest

from rng_craft import crafted_state, lemire_rejects, seeded_state, words_of
from test_merge_generic_spec import network_of, rederive_reset

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["mg_default", "mg_v1_default", "mg_three_lanes", "mg_one_lane_ttc", "mg_crowded_32", "mg_float_grid"]
FLOATS = ("x", "y", "heading", "speed")
TOL = 1e-6
MIN_SPEED = 1.0  # below it the steering law (not_zero(speed), controller.py:166,178) amplifies an ulp past TOL


def ill_windows(g):
    """The teacher-forced windows (seed slot, stored step index) in which the reference itself is ill conditioned: a
    vehicle that has not crashed moves slower than MIN_SPEED at the window's start or after one of its steps."""
    ms, steps = g["min_speed"], g["steps"]
    return {(k, j) for k in range(ms.shape[0]) for j in range(len(steps) - 1)
            if ms[k, int(steps[j]):int(steps[j + 1]) + 1].min() < MIN_SPEED}


def load(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    g["config"] = json.loads(str(g.pop("config_json")))
    g["slot"] = {int(t): j for j, t in enumerate(g["steps"])}
    return g


def make(g, n=None, mode="SameStep", **over):
    import highwayenv_b200 as hb

    return hb.make(g["config"]["_env_id"], num_envs=n or len(g["seeds"]),
                   config={**g["config"]["_override"], **over}, autoreset_mode=mode)


def rec_of(g, prefix, *idx):
    keys = ("x", "y", "heading", "speed", "target_speed", "timer", "delta", "lane", "target_lane", "crashed", "impact",
            "check_collisions", "speed_index", "kind", "count", "time", "obs", "rng", "available")
    return {k: g[prefix + k][idx] for k in keys}


def compare(sd, e, rec, tol, ctx, exact_ego=False):
    """Env e of state_dict sd against a fixture record: population, lanes, kinds and crash flags exact; floats within
    tol (the ego bit for bit with exact_ego).  The Obstacle (last slot) has no target speed, timer or DELTA, the ego no
    timer or DELTA, and the Obstacle no target lane.  Returns whether the floats matched."""
    c = int(rec["count"])
    assert int(sd["count"][e]) == c, ctx
    for k in ("lane", "kind"):
        assert np.array_equal(np.asarray(sd[k][e][:c]), rec[k][:c]), (ctx, k)
    assert np.array_equal(np.asarray(sd["target_lane"][e][:c - 1]), rec["target_lane"][:c - 1]), ctx
    assert np.array_equal(sd["crashed"][e][:c].astype(bool), rec["crashed"][:c].astype(bool)), ctx
    worst = 0.0
    for k in FLOATS + ("target_speed",):
        m = c - 1 if k == "target_speed" else c
        d = np.abs(np.asarray(sd[k][e][:m], dtype=np.float64) - rec[k][:m])
        worst = max(worst, float(d.max()))
        if exact_ego:
            assert d[0] == 0.0, (ctx, k)
    for k in ("timer", "delta"):  # IDM traffic only
        if c > 2:
            worst = max(worst, float(np.abs(np.asarray(sd[k][e][1:c - 1]) - rec[k][1:c - 1]).max()))
    return worst <= tol


def check_reset(g, env, obs, ids, recs):
    sd = env.state_dict()
    words = env.rng_words().T
    for e, rec in zip(ids, recs):
        assert np.array_equal(words[e], rec["rng"]), e
        assert compare(sd, e, rec, 1e-12, f"reset env {e}", exact_ego=True)
    o = obs.cpu().numpy()[ids].astype(np.float64)
    assert np.max(np.abs(o - np.stack([r["obs"] for r in recs]))) <= 1e-6
    avail = env.get_available_actions().cpu().numpy()[ids]
    assert np.array_equal(avail, np.stack([r["available"] for r in recs]))


@pytest.mark.parametrize("name", CASES)
def test_reset_matches_reference(name):
    g = load(name)
    S = len(g["seeds"])
    env = make(g)
    obs, _ = env.reset(seed=[int(s) for s in g["seeds"]])
    check_reset(g, env, obs, np.arange(S), [rec_of(g, "reset_", i) for i in range(S)])


@pytest.mark.parametrize("name", CASES)
def test_every_autoreset_from_its_stream(name):
    """Every autoreset of the fixture, one env each, from the stream words the env held before it (the steps draw
    nothing): the device reset reproduces the reference's population, lanes, kinds and stream words."""
    import torch

    g = load(name)
    before, recs = [], []
    for i in range(len(g["seeds"])):
        prev = g["reset_rng"][i]
        for j in range(g["autoreset_step"].shape[1]):
            if g["autoreset_step"][i, j] >= 0:
                before.append(prev)
                recs.append(rec_of(g, "autoreset_", i, j))
                prev = g["autoreset_rng"][i, j]
    env = make(g, len(recs))
    env.reset(seed=0)
    env._rng.copy_(torch.from_numpy(np.stack(before, axis=1).view(np.int64)).cuda())
    obs, _ = env.reset()
    check_reset(g, env, obs, np.arange(len(recs)), recs)
    if name == "mg_crowded_32":
        counts = {int(r["count"]) for r in recs}
        assert len(counts) > 1 and max(counts) < 3 + int(g["config"]["vehicles_count"])


def load_rows(env, g, rows):
    """Load the fixture's stored step records rows = [(seed slot, stored step index)] into envs 0.."""
    import torch

    V = env.V
    recs = [rec_of(g, "", k, j) for k, j in rows]
    st = {k: np.stack([r[k] for r in recs]) for k in recs[0]}
    nan0 = lambda a: np.nan_to_num(a[:, :V])  # noqa: E731
    sd = {k: nan0(st[k]) for k in ("x", "y", "heading", "speed", "target_speed", "timer")}
    sd["delta"] = np.nan_to_num(st["delta"][:, :V], nan=4.0)
    sd["impact_x"], sd["impact_y"] = nan0(st["impact"][..., 0]), nan0(st["impact"][..., 1])
    sd["has_impact"] = ~np.isnan(st["impact"][:, :V, 0])
    for k in ("lane", "kind", "crashed", "check_collisions"):
        sd[k] = st[k][:, :V]
    sd["target_lane"] = np.where(st["target_lane"][:, :V] < 0, st["lane"][:, :V], st["target_lane"][:, :V])
    sd["route"] = np.zeros((len(rows), V, 16), dtype=np.int32)
    sd["route_len"] = np.zeros((len(rows), V), dtype=np.int32)
    sd["speed_index"] = st["speed_index"][:, 0].astype(np.int32)
    sd["time"], sd["count"] = st["time"], st["count"]
    env.load_state_dict(sd, env_ids=np.arange(len(rows)))
    env._rng[:, :len(rows)] = torch.from_numpy(np.ascontiguousarray(st["rng"].T).view(np.int64)).cuda()


@pytest.mark.parametrize("name", CASES)
def test_teacher_forced_windows(name):
    """Every stored state that did not end its episode is loaded and the stored actions replayed to the next stored
    step: get_available_actions at the start; in every window the reference is well conditioned in (ill_windows),
    flags exact on every step, then the state (<= 1e-6), stream words, reward and terms (<= 1e-9) and observation
    (<= 1e-6; the grid exactly) at the next stored step."""
    import torch

    g = load(name)
    steps = g["steps"]
    rows = []
    for k in range(len(g["seeds"])):
        resets = set(int(t) for t in g["autoreset_step"][k] if t >= 0)
        rows += [(k, j) for j in range(len(steps) - 1) if int(steps[j]) not in resets]
    env = make(g, len(rows), mode="Disabled")
    env.reset(seed=0)
    load_rows(env, g, rows)
    ks, js = np.array([r[0] for r in rows]), np.array([r[1] for r in rows])
    assert np.array_equal(env.get_available_actions().cpu().numpy(), g["available"][ks, js])
    start, end = steps[js], steps[js + 1]
    ended = np.zeros(len(rows), dtype=bool)
    off = np.zeros(len(rows), dtype=bool)
    obs_tol = 0.0 if "grid" in name else 1e-6
    compared = merging = 0
    for d in range(1, int((end - start).max()) + 1):
        t = start + d
        act = g["actions"][ks, t]
        obs, rew, term, trunc, info = env.step(torch.from_numpy(np.ascontiguousarray(act)).cuda())
        term, trunc = term.cpu().numpy(), trunc.cpu().numpy()
        flags = np.stack([term, trunc, info["crashed"].cpu().numpy()], axis=-1).astype(bool)
        live = (~ended) & (~off)
        off |= live & (flags != g["flags"][ks, t]).any(-1)
        at_end = live & ~off & (t == end)
        if at_end.any():
            sd = env.state_dict()
            words = env.rng_words().T
            r = rew.cpu().numpy()
            terms = np.stack([info["rewards"][nm].cpu().numpy() for nm in env.REWARD_NAMES], axis=-1)
            o = obs.cpu().numpy().astype(np.float64)
            for i in np.nonzero(at_end)[0]:
                k, j1 = ks[i], js[i] + 1
                rec = rec_of(g, "", k, j1)
                ctx = f"window {rows[i]}"
                assert np.array_equal(words[i], rec["rng"]), ctx
                if not compare(sd, i, rec, TOL, ctx):
                    off[i] = True
                    continue
                assert abs(r[i] - g["reward"][k, j1]) <= 1e-9, ctx
                assert np.max(np.abs(terms[i] - g["terms"][k, j1])) <= 1e-9, ctx
                assert np.max(np.abs(o[i] - rec["obs"])) <= obs_tol, ctx
                compared += 1
                merging += g["terms"][k, j1, 4] != 0
        ended |= live & (term | trunc).astype(bool)
    left = {(int(ks[i]), int(js[i])) for i in np.nonzero(off)[0]}
    ill = ill_windows(g)
    assert left <= ill, sorted(left - ill)  # every window the reference is well conditioned in matches
    if name == "mg_crowded_32":
        # end_position 150: an episode lasts about 4 steps, so no window reaches the next stored step; its flags are
        # still compared on every step here, and its stored states, rewards and terms in the free-running test
        return
    assert compared >= 40
    if name == "mg_three_lanes":  # ("b","c",2) is a highway lane
        assert merging >= 10, merging


def rollout(g, env, obs_tol):
    """SameStep over the fixture's actions: env k is seed k.  Returns the (env, step) pairs that left the reference."""
    import torch

    S, T = g["actions"].shape
    res_k = np.zeros(S, dtype=int)
    alive = np.ones(S, dtype=bool)
    left = set()
    compared = merging = 0
    for t in range(T):
        alive &= g["min_speed"][:, t] >= MIN_SPEED  # the reference's well-conditioned prefix of each env
        compared += int(alive.sum())
        obs, rew, term, trunc, info = env.step(torch.from_numpy(g["actions"][:, t]).cuda())
        term, trunc = term.cpu().numpy(), trunc.cpu().numpy()
        flags = np.stack([term, trunc, info["crashed"].cpu().numpy()], axis=-1).astype(bool)
        for k in np.nonzero(alive & (flags != g["flags"][:, t]).any(-1))[0]:
            left.add((int(k), t))
            alive[k] = False
        sd = env.state_dict()
        words = env.rng_words().T
        j = g["slot"].get(t)
        for k in range(S):
            if not alive[k]:
                continue
            if term[k] or trunc[k]:
                m = res_k[k]
                assert g["autoreset_step"][k, m] == t
                rec = rec_of(g, "autoreset_", k, m)
                assert np.array_equal(words[k], rec["rng"]), (t, k)
                assert compare(sd, k, rec, 1e-12, f"reset t={t} env={k}")
                res_k[k] += 1
            elif j is not None:
                rec = rec_of(g, "", k, j)
                assert np.array_equal(words[k], rec["rng"]), (t, k)
                if not compare(sd, k, rec, TOL, f"t={t} env={k}"):
                    left.add((k, t))
                    alive[k] = False
        if j is not None:
            r = rew.cpu().numpy()
            terms = np.stack([info["rewards"][nm].cpu().numpy() for nm in env.REWARD_NAMES], axis=-1)
            assert np.max(np.abs(r - g["reward"][:, j])[alive], initial=0.0) <= 1e-9, t
            assert np.max(np.abs(terms - g["terms"][:, j])[alive], initial=0.0) <= 1e-9, t
            merging += int((alive & (g["terms"][:, j, 4] != 0)).sum())
            o = info["final_obs"].cpu().numpy().astype(np.float64)
            assert np.max(np.abs(o - g["obs"][:, j])[alive], initial=0.0) <= obs_tol, t
    return left, compared, merging


@pytest.mark.parametrize("name", CASES)
def test_free_running_matches_reference(name):
    """60 steps with SameStep autoreset over each env's well-conditioned prefix: flags exact on every step, every
    autoreset exact in population, lanes, kinds and stream words, and the stored steps' state, reward, terms and
    observation.  On 32 slots (mg_crowded_32: the Obstacle and the merge reward on the intersection family's step) and
    on a highway merging lane (mg_three_lanes) the compared rewards include non-zero merging terms."""
    g = load(name)
    env = make(g)
    env.reset(seed=[int(s) for s in g["seeds"]])
    left, compared, merging = rollout(g, env, 0.0 if "grid" in name else 1e-6)
    assert left == set(), sorted(left)
    assert compared >= 3 * len(g["seeds"])
    if name in ("mg_crowded_32", "mg_three_lanes"):
        assert merging >= 10, merging


def test_crafted_lemire_rejections_match_numpy():
    """A Lemire rejection in the first integers(3) (lanes_count 3): the device reset equals the numpy restatement
    (stream words, population, kinds and lanes exact; positions and speeds within 1e-12)."""
    import torch

    import highwayenv_b200 as hb
    from highwayenv_b200.config import default_config
    from highwayenv_b200.envs.common.vector_env import pcg64_words
    from rng_craft import generator_of

    assert lemire_rejects(0, 3)
    words = []
    for seed in range(16):
        _, inc = seeded_state(seed)
        x = int(np.random.default_rng(seed).integers(1, 1 << 32)) << 32  # low half 0: rejected for n = 3
        words.append(words_of(crafted_state(x, inc, 0, seed=seed), inc))
    cfg = default_config("merge-generic-v0")
    cfg.update(lanes_count=3, vehicles_count=5)
    net = network_of(cfg)
    env = hb.make("merge-generic-v0", num_envs=len(words), config={"lanes_count": 3, "vehicles_count": 5})
    env.reset(seed=0)
    env._rng.copy_(torch.from_numpy(np.stack(words, axis=1).view(np.int64)).cuda())
    env.reset()
    sd, got = env.state_dict(), env.rng_words().T
    for e, w in enumerate(words):
        gen = generator_of(w)
        r = rederive_reset(gen, net, cfg)
        n = len(r["x"])
        assert np.array_equal(got[e], pcg64_words([gen])[:, 0]) and sd["count"][e] == n, e
        assert np.array_equal(sd["lane"][e][:n], r["lane"]) and np.array_equal(sd["kind"][e][:n], r["kind"])
        for k in ("x", "y", "speed"):
            assert np.max(np.abs(sd[k][e][:n] - r[k])) <= 1e-12, (e, k)


@pytest.mark.parametrize("name", ["mg_default", "mg_crowded_32"])
@pytest.mark.parametrize("two_masks", [False, True])
def test_masked_reset(name, two_masks):
    """257 envs: rows the masks leave out are byte-identical; selected rows equal an unmasked reset of a copy_envs
    copy of the env."""
    import torch

    g = load(name)
    n = 257
    env, twin = make(g, n, mode="Disabled"), make(g, n, mode="Disabled")
    env.reset(seed=11)
    rng = np.random.default_rng(1)
    for _ in range(4):
        env.step(torch.from_numpy(rng.integers(0, 5, n).astype(np.int32)).cuda())
    twin.reset(seed=0)
    ids = torch.arange(n).cuda()
    twin.copy_envs(ids, ids, source=env)
    before = {k: v.clone() for k, v in env._env_rows().items()}
    ma = torch.from_numpy((rng.random(n) < 0.3).astype(np.uint8)).cuda()
    mb = torch.from_numpy((rng.random(n) < 0.3).astype(np.uint8)).cuda() if two_masks else None
    with torch.cuda.device(env.device):
        env._device_reset(ma.data_ptr(), None if mb is None else mb.data_ptr(), env._fused_out.data_ptr())
    twin.reset()
    sel = (ma.bool() | (mb.bool() if mb is not None else torch.zeros_like(ma, dtype=torch.bool))).cpu().numpy()
    after, fresh = env._env_rows(), twin._env_rows()
    for k, v in after.items():
        assert torch.equal(v[torch.from_numpy(~sel).cuda()], before[k][torch.from_numpy(~sel).cuda()]), k
        if k != "_obs":
            assert torch.equal(v[torch.from_numpy(sel).cuda()], fresh[k][torch.from_numpy(sel).cuda()]), k
    assert torch.equal(env._obs[torch.from_numpy(sel).cuda()], twin._obs[torch.from_numpy(sel).cuda()])
    assert sel.any() and (~sel).any()


@pytest.mark.parametrize("name", ["mg_three_lanes", "mg_crowded_32"])
def test_state_dict_round_trip_and_road_substeps(name):
    import torch

    g = load(name)
    a_env, b_env = make(g, 32, mode="Disabled"), make(g, 32, mode="Disabled")
    a_env.reset(seed=0)
    b_env.reset(seed=99)
    a = torch.from_numpy(np.random.default_rng(5).integers(0, 5, 32).astype(np.int32)).cuda()
    a_env.step(a)
    b_env.load_state_dict(a_env.state_dict())
    b_env._rng.copy_(a_env._rng)
    sa, sb = a_env.state_dict(), b_env.state_dict()
    assert all(np.array_equal(sa[k], sb[k]) for k in sa)
    for step in (lambda e: e.step(a), lambda e: e.road_substeps(7)):
        step(a_env)
        step(b_env)
        sa, sb = a_env.state_dict(), b_env.state_dict()
        for k in sa:
            assert np.array_equal(sa[k], sb[k]), k
        assert np.array_equal(a_env.rng_words(), b_env.rng_words())


@pytest.mark.parametrize("name", ["mg_default", "mg_crowded_32"])
def test_host_stepper_graph(name):
    import torch

    g = load(name)
    env, twin = make(g), make(g)
    for e in (env, twin):
        e.reset(seed=[int(s) for s in g["seeds"]])
    hs = env.host_stepper()
    for t in range(g["actions"].shape[1]):
        hs.actions[:] = g["actions"][:, t]
        obs, rew, term, trunc = hs.step()
        o2, r2, t2, tr2, _ = twin.step(torch.from_numpy(g["actions"][:, t]).cuda())
        assert np.array_equal(obs, o2.cpu().numpy()) and np.array_equal(rew, r2.cpu().numpy())
        assert np.array_equal(term, t2.cpu().numpy()) and np.array_equal(trunc, tr2.cpu().numpy())


@pytest.mark.parametrize("name,first", [("mg_crowded_32", {"lanes_count": 3, "vehicles_count": 3}),
                                        ("mg_default", {"lanes_count": 4, "vehicles_count": 20}),
                                        ("mg_float_grid", {"lanes_count": 1, "after_merge_length": 100})])
def test_reset_with_a_new_config(name, first):
    """An env made on one road and population and reset with options={"config": the fixture's} moves to the new
    table and slot stride and resets as the reference does; a few steps then follow the fixture."""
    import torch

    import highwayenv_b200 as hb

    g = load(name)
    S = len(g["seeds"])
    env = hb.make(g["config"]["_env_id"], num_envs=S, config={**g["config"]["_override"], **first})
    env.reset(seed=0)
    env.step(torch.zeros(S, dtype=torch.int32).cuda())
    keys = ("lanes_count", "vehicles_count", "before_merge_length", "converge_merge_length", "parallel_merge_length",
            "after_merge_length")
    back = {k: g["config"][k] for k in keys}
    obs, _ = env.reset(seed=[int(s) for s in g["seeds"]], options={"config": back})
    assert env.vp == (8 if back["vehicles_count"] <= 5 else 32) and len(env.net.lanes) == len(network_of(back).lanes)
    check_reset(g, env, obs, np.arange(S), [rec_of(g, "reset_", i) for i in range(S)])
    for t in range(5):
        _, _, term, _, _ = env.step(torch.from_numpy(g["actions"][:, t]).cuda())
        assert np.array_equal(term.cpu().numpy(), g["flags"][:, t, 0]), t


def test_copy_envs_rejected_across_roads():
    import torch

    import highwayenv_b200 as hb

    a = hb.make("merge-generic-v0", num_envs=4)
    b = hb.make("merge-generic-v0", num_envs=4, config={"after_merge_length": 120.5})
    c = hb.make("merge-generic-v0", num_envs=4, config={"vehicles_count": 12})
    for e in (a, b, c):
        e.reset(seed=0)
    ids = torch.arange(2).cuda()
    for dst, src in ((a, b), (b, a), (a, c), (c, a)):
        with pytest.raises(ValueError):
            dst.copy_envs(ids, ids, source=src)
    twin = hb.make("merge-generic-v0", num_envs=4)
    twin.reset(seed=3)
    a.copy_envs(ids, ids, source=twin)


@pytest.mark.parametrize("over", [{"lanes_count": 0}, {"lanes_count": 10}, {"after_merge_length": 80},
                                  {"vehicles_count": 30}, {"action": {"type": "ContinuousAction"}}])
def test_unsupported_configurations_raise_before_any_launch(over):
    import highwayenv_b200 as hb
    from highwayenv_b200 import _native as N

    lib = N.load()
    before = lib.hwy_launch_count()
    with pytest.raises((NotImplementedError, ValueError)):
        hb.make("merge-generic-v0", num_envs=16, config=over).reset(seed=0)
    assert lib.hwy_launch_count() == before


@pytest.mark.parametrize("env_id,over", [("merge-generic-v0", None), ("merge-generic-v1", None),
                                         ("merge-generic-v0", {"lanes_count": 4, "vehicles_count": 20})])
def test_end_to_end_4096(env_id, over):
    """4096 envs from one seed (the first 32 are the fixture's seeds 0..31 at the defaults) and 40 random steps under
    SameStep autoreset."""
    import torch

    import highwayenv_b200 as hb

    env = hb.make(env_id, num_envs=4096, config=over)
    obs, _ = env.reset(seed=0)
    if over is None:
        g = load("mg_default" if env_id.endswith("v0") else "mg_v1_default")
        check_reset(g, env, obs, np.arange(32), [rec_of(g, "reset_", i) for i in range(32)])
    rng = np.random.default_rng(0)
    done = 0
    for _ in range(40):
        obs, rew, term, trunc, info = env.step(torch.from_numpy(rng.integers(0, 5, 4096).astype(np.int32)).cuda())
        done += int((term | trunc).sum())
        assert torch.isfinite(rew).all() and torch.isfinite(obs).all()
    sd = env.state_dict()
    assert done > 0 and sd["lane"].max() < len(env.net.lanes)
    assert (sd["count"] >= 3).all() and (sd["count"] <= env.V).all()
    last = sd["count"] - 1  # the Obstacle closes every env's population
    assert (sd["kind"][np.arange(4096), last] == 3).all()


@pytest.mark.parametrize("env_id", ["merge-generic-v0", "merge-generic-v1"])
def test_make_single(env_id):
    import highwayenv_b200 as hb

    env = hb.make_single(env_id)
    obs, info = env.reset(seed=0)
    assert obs.shape == (5, 5)
    obs, rew, term, trunc, info = env.step(1)
    assert np.isfinite(rew)
