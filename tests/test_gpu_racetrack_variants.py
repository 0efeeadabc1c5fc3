"""GPU parity of racetrack-large-v0 / v1 and racetrack-oval-v0 / v1 (hwy_racetrack_reset with ego_lanes, and the
unchanged racetrack_step_kernel<8>) against the fixtures of oracle/gen_racetrack_variants.py, with the bounds of
tests/test_gpu_racetrack.py: resets, teacher-forced windows, free-running rollouts with SameStep autoreset, copy_envs
and the configurations that raise before any launch."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["racetrack_large_random", "racetrack_large_follow", "racetrack_large_traffic", "racetrack_large_v1_follow",
         "racetrack_large_speed15", "racetrack_oval_follow", "racetrack_oval_lanes2", "racetrack_oval_v1_lanes4"]
FLOATS = ("x", "y", "heading", "speed", "target_speed", "timer")
INTS = ("lane", "target_lane", "kind", "crashed")
FIELDS = FLOATS + INTS  # the fixture's row order
TOL = 1e-6  # as for racetrack-v0: CUDA's sincos and atan2 against numpy's, over the rollouts
LANE = FIELDS.index("lane")


def load(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    g["config"] = json.loads(str(g.pop("config_json")))
    g["slot"] = {int(t): j for j, t in enumerate(g["steps"])}
    g["obs_tol"] = 0.0 if g["obs"].ndim == 5 else 1e-6
    return g


def network_of(g):
    from highwayenv_b200.envs.racetrack_env import track_network

    cfg = {k: v for k, v in g["config"].items() if not k.startswith("_")}
    return track_network(g["config"]["_env_id"], cfg)


# ---------------------------------------------------------------- ill-conditioned spots, from the geometry alone
# On racetrack-v0 two lanes on one circle overlap in angle, and the last bits of atan2 / sincos decide their closest-lane
# tie.  The same kind of place is looked for here on each lane table, together with the other place where two lanes are
# equally close: a lane end that coincides with another lane's end.
def _ends(L):
    if "center" in L:
        c, r = np.asarray(L["center"], dtype=np.float64), float(L["radius"])
        return [c + r * np.array([np.cos(a), np.sin(a)]) for a in (L["start_phase"], L["end_phase"])]
    return [np.asarray(L["start"], dtype=np.float64), np.asarray(L["end"], dtype=np.float64)]


def ill_conditioned_spots(net):
    """(same_circle, coincident_ends): the pairs of table indices of lanes on the same circle whose angle ranges
    overlap, and of lanes with an end within 1e-9 m of an end of the other, from the to_config of the lane table."""
    lanes = [ld["config"] for tos in net.to_config().values() for road in tos.values() for ld in road]
    same, ends = set(), set()
    for a in range(len(lanes)):
        for b in range(a + 1, len(lanes)):
            A, B = lanes[a], lanes[b]
            if "center" in A and "center" in B and A["center"] == B["center"] and A["radius"] == B["radius"]:
                ra, rb = sorted((A["start_phase"], A["end_phase"])), sorted((B["start_phase"], B["end_phase"]))
                if min(ra[1], rb[1]) > max(ra[0], rb[0]):
                    same.add((a, b))
            if any(np.linalg.norm(p - q) <= 1e-9 for p in _ends(A) for q in _ends(B)):
                ends.add((a, b))
    return same, ends


@pytest.mark.parametrize("name", ["racetrack_large_follow", "racetrack_oval_follow", "racetrack_oval_lanes2",
                                  "racetrack_oval_v1_lanes4"])
def test_ill_conditioned_spots(name):
    """Neither new track has two lanes on one circle: every arc of a road has its own radius, and the roads' centres
    differ.  The coincident ends are the joins of consecutive roads, lane by lane, where the next lane starts exactly
    where the last one ends; the oval's ("a","b") lanes overrun ("b","c") by 1 m instead."""
    net = network_of(load(name))
    same, ends = ill_conditioned_spots(net)
    assert same == set()
    name_of = net.lane_index_of
    for a, b in ends:
        (fa, ta, ia), (fb, tb, ib) = name_of[a], name_of[b]
        assert ia == ib and (ta == fb or tb == fa), (name_of[a], name_of[b])


def crossing_windows(g, pairs):
    """[n_envs, n_stored] bool: whether the reference can move a vehicle between the two lanes of one of `pairs` in
    the window that ends at stored step j.  Before a reset inside the window the end is not stored, so a vehicle on such
    a lane at a start before it counts as crossing."""
    lanes = {x for p in pairs for x in p}
    pairs = pairs | {(b, a) for a, b in pairs}
    n = g["actions"].shape[0]
    out = np.zeros((n, len(g["steps"])), dtype=bool)

    def crosses(starts, end_state, end_count):
        for st, c in starts[:-1]:
            if any(int(x) in lanes for x in st[LANE, :c]):
                return True
        st, c = starts[-1]
        return any((int(st[LANE, v]), int(end_state[LANE, v])) in pairs for v in range(min(c, end_count)))

    for k in range(n):
        start = (g["reset_state"][k], int(g["reset_count"][k]))
        resets = {int(t): m for m, t in enumerate(g["autoreset_step"][k]) if t >= 0}
        a = -1
        for j, b in enumerate(g["steps"]):
            inner = [(g["autoreset_state"][k, resets[t]], int(g["autoreset_count"][k, resets[t]]))
                     for t in range(a + 1, int(b)) if t in resets]
            out[k, j] = crosses([start] + inner, g["state"][k, j], int(g["count"][k, j]))
            m = resets.get(int(b))
            start = (g["state"][k, j], int(g["count"][k, j])) if m is None else \
                (g["autoreset_state"][k, m], int(g["autoreset_count"][k, m]))
            a = int(b)
    return out


# The divergences from the reference in these fixtures: free-running (env, first step that differs), teacher-forced
# (env, window start index).  Each must lie in a window where the reference crosses an ill-conditioned spot.
KNOWN_FREE = {name: set() for name in CASES}
KNOWN_FORCED = {name: set() for name in CASES}


def make(g, n=None, mode="SameStep"):
    import highwayenv_b200 as hb

    return hb.make(g["config"]["_env_id"], num_envs=n or len(g["seeds"]), config=dict(g["config"]["_override"]),
                   autoreset_mode=mode)


def ours(sd, i, count):
    rows = [np.asarray(sd[k][i], dtype=np.float64) for k in FIELDS]
    return np.stack(rows)[:, :count]


def compare(st, ref, count, ctx):
    ref = ref[:, :count]
    nf = len(FLOATS)
    d = float(np.max(np.abs(st[:nf] - ref[:nf]))) if count else 0.0
    assert d <= TOL, (ctx, d)
    assert np.array_equal(st[nf:], ref[nf:]), (ctx, st[nf:], ref[nf:])
    return d


def conditioned(st, ref, count):
    ref = ref[:, :count]
    nf = len(FLOATS)
    return (not count or float(np.max(np.abs(st[:nf] - ref[:nf]))) <= TOL) and np.array_equal(st[nf:], ref[nf:])


def check_reset(g, env, obs, ids, n_ref):
    """Envs ids[k] against the fixture's first reset of seed k: stream words, populations, lanes and kinds exact, the
    ego exact and the rest within 1e-12."""
    sd = env.state_dict()
    assert np.array_equal(env.rng_words().T[ids], g["reset_rng"][:n_ref])
    assert np.array_equal(sd["count"][ids], g["reset_count"][:n_ref])
    worst = 0.0
    for k, e in enumerate(ids):
        c = int(g["reset_count"][k])
        st = ours(sd, e, c)
        assert np.array_equal(st[:, 0], g["reset_state"][k][:, 0]), k
        worst = max(worst, compare(st, g["reset_state"][k], c, f"reset#{k}"))
    assert worst <= 1e-12, worst
    o = obs.cpu().numpy()[ids].astype(np.float64)
    assert np.max(np.abs(o - g["reset_obs"][:n_ref])) <= g["obs_tol"]


@pytest.mark.parametrize("name", CASES)
def test_reset_matches_reference(name):
    g = load(name)
    env = make(g)
    obs, _ = env.reset(seed=[int(s) for s in g["seeds"]])
    check_reset(g, env, obs, np.arange(len(g["seeds"])), len(g["seeds"]))


@pytest.mark.parametrize("name,first", [("racetrack_oval_v1_lanes4", {"no_lanes": 3}),
                                        ("racetrack_oval_v1_lanes4", {"no_lanes": 2, "length": 150}),
                                        ("racetrack_large_speed15", {"speed_limit": 10.0})])
def test_reset_with_a_new_config_follows_the_new_track(name, first):
    """An env made on one track and reset with options={"config": the fixture's override} resets as the reference does
    on the new track: its lane table is rebuilt with the kernel parameters.  A few steps then follow the fixture."""
    import torch

    import highwayenv_b200 as hb

    g = load(name)
    over = dict(g["config"]["_override"])
    env = hb.make(g["config"]["_env_id"], num_envs=len(g["seeds"]), config={**over, **first})
    env.reset(seed=0)
    env.step(torch.zeros(len(g["seeds"]), env.action_size).cuda())
    back = {**over, **{k: g["config"][k] for k in first}}  # configure is a shallow update
    obs, _ = env.reset(seed=[int(s) for s in g["seeds"]], options={"config": back})
    assert len(env.net.lanes) == len(network_of(g).lanes)
    check_reset(g, env, obs, np.arange(len(g["seeds"])), len(g["seeds"]))
    for t in range(5):
        _, _, term, _, _ = env.step(torch.from_numpy(g["actions"][:, t]).cuda())
        assert np.array_equal(term.cpu().numpy(), g["flags"][:, t, 0]), t


@pytest.mark.parametrize("name", ["racetrack_large_follow", "racetrack_oval_v1_lanes4"])
def test_reset_of_4096_envs_from_one_seed(name):
    """reset(seed=0) of 4096 envs seeds env i with 0 + i: the first 32 are the fixture's seeds 0..31."""
    g = load(name)
    assert np.array_equal(g["seeds"], np.arange(32))
    env = make(g, 4096)
    obs, _ = env.reset(seed=0)
    check_reset(g, env, obs, np.arange(32), 32)


def rollout(g, env, ids=None, check_obs=True):
    """As in tests/test_gpu_racetrack.py: SameStep, env ids[k] is fixture seed k; returns the (env, step) pairs that
    left the reference."""
    import torch

    n = env.num_envs
    ids = np.arange(len(g["seeds"])) if ids is None else np.asarray(ids)
    T, size = g["actions"].shape[1:]
    extra = np.random.default_rng(7).uniform(-1, 1, size=(T, n, size)).astype(np.float32)
    res_k = np.zeros(len(ids), dtype=int)
    alive = np.ones(len(ids), dtype=bool)
    left = set()
    for t in range(T):
        a = extra[t]
        a[ids] = g["actions"][:, t]
        obs, rew, term, trunc, info = env.step(torch.from_numpy(a).cuda())
        term, trunc = term.cpu().numpy()[ids], trunc.cpu().numpy()[ids]
        crashed = info["crashed"].cpu().numpy()[ids]
        flags = np.stack([term, trunc, crashed], axis=-1).astype(bool)
        for k in np.nonzero(alive & (flags != g["flags"][:, t]).any(-1))[0]:
            left.add((int(k), t))
            alive[k] = False
        sd = env.state_dict()
        words = env.rng_words().T[ids]
        done = term | trunc
        j = g["slot"].get(t)
        for k, e in enumerate(ids):
            if not alive[k]:
                continue
            if done[k]:
                m = res_k[k]
                assert g["autoreset_step"][k, m] == t
                c = int(g["autoreset_count"][k, m])
                assert sd["count"][e] == c and np.array_equal(words[k], g["autoreset_rng"][k, m]), (t, k)
                compare(ours(sd, e, c), g["autoreset_state"][k, m], c, f"reset t={t} env={k}")
                res_k[k] += 1
            elif j is not None:
                c = int(g["count"][k, j])
                assert sd["count"][e] == c and np.array_equal(words[k], g["rng"][k, j]), (t, k)
                if not conditioned(ours(sd, e, c), g["state"][k, j], c):
                    left.add((k, t))
                    alive[k] = False
        if j is not None:
            r = rew.cpu().numpy()[ids]
            terms = np.stack([info["rewards"][nm].cpu().numpy()[ids] for nm in env.REWARD_NAMES], axis=-1)
            assert np.max(np.abs(r - g["reward"][:, j])[alive], initial=0.0) <= 1e-9, t
            assert np.max(np.abs(terms - g["terms"][:, j])[alive], initial=0.0) <= 1e-9, t
            if check_obs:
                o = info["final_obs"].cpu().numpy()[ids].astype(np.float64)
                assert np.max(np.abs(o - g["obs"][:, j])[alive], initial=0.0) <= g["obs_tol"], t
    return left


def check_left(g, left, known, name, window):
    """The envs that left the reference are exactly the known ones, each in a window where the reference crosses an
    ill-conditioned spot."""
    same, ends = ill_conditioned_spots(network_of(g))
    cross = crossing_windows(g, same | ends)
    assert left == known[name], (name, sorted(left))
    for k, t in left:
        assert cross[k, window(t)], (k, t)


@pytest.mark.parametrize("name", CASES)
def test_free_running_matches_reference(name):
    """200 steps with SameStep autoreset: flags exact on every step, every reset exact in population and stream words,
    the stored steps' state (<= 1e-6), reward (<= 1e-9), reward terms and observation."""
    g = load(name)
    env = make(g)
    env.reset(seed=[int(s) for s in g["seeds"]])
    check_left(g, rollout(g, env), KNOWN_FREE, name, lambda t: int(np.searchsorted(g["steps"], t)))


def load_reference_rows(env, g, rows):
    n = len(rows)
    V = env.V
    st = np.stack([g["state"][k, j][:, :V] for k, j in rows])
    sd = {f: st[:, i] for i, f in enumerate(FIELDS)}
    for f in ("lane", "target_lane", "kind"):
        sd[f] = sd[f].astype(np.int64)
    sd["crashed"] = sd["crashed"].astype(bool)
    imp = np.stack([g["impact"][k, j][:, :V] for k, j in rows])
    sd["impact_x"], sd["impact_y"] = imp[:, 0], imp[:, 1]
    sd["has_impact"] = np.stack([g["has_impact"][k, j][:V] for k, j in rows])
    counts = np.array([g["count"][k, j] for k, j in rows], dtype=np.int32)
    sd["check_collisions"] = np.arange(V)[None, :] < counts[:, None]
    sd["delta"] = np.full((n, V), 4.0)
    sd["speed_index"] = np.zeros(n, dtype=np.int32)
    sd["time"] = np.array([g["time"][k, j] for k, j in rows])
    sd["count"] = counts
    sd["rng"] = np.stack([g["rng"][k, j] for k, j in rows], axis=1)
    env.load_state_dict(sd, env_ids=np.arange(n))


@pytest.mark.parametrize("name", CASES)
def test_teacher_forced_windows(name):
    """Every stored state that did not end its episode is loaded and the stored actions replayed to the next stored
    step: flags exact on every step up to the first episode end, then state, stream words, reward, terms and
    observation at the next stored step."""
    import torch

    g = load(name)
    steps = g["steps"]
    rows = []
    for k in range(len(g["seeds"])):
        resets = set(int(t) for t in g["autoreset_step"][k] if t >= 0)
        rows += [(k, j) for j in range(len(steps) - 1) if int(steps[j]) not in resets]
    env = make(g, len(rows), mode="Disabled")
    env.reset(seed=0)
    load_reference_rows(env, g, rows)
    ks, js = np.array([r[0] for r in rows]), np.array([r[1] for r in rows])
    start, end = steps[js], steps[js + 1]
    ended = np.zeros(len(rows), dtype=bool)
    off = np.zeros(len(rows), dtype=bool)
    for d in range(1, int((end - start).max()) + 1):
        t = start + d
        act = g["actions"][ks, np.minimum(t, g["actions"].shape[1] - 1)]
        obs, rew, term, trunc, info = env.step(torch.from_numpy(np.ascontiguousarray(act)).cuda())
        term, trunc = term.cpu().numpy(), trunc.cpu().numpy()
        flags = np.stack([term, trunc, info["crashed"].cpu().numpy()], axis=-1).astype(bool)
        live = (~ended) & (~off) & (t <= end)
        off |= live & (flags != g["flags"][ks, np.minimum(t, g["flags"].shape[1] - 1)]).any(-1)
        at_end = live & ~off & (t == end)
        if at_end.any():
            sd = env.state_dict()
            words = env.rng_words().T
            r = rew.cpu().numpy()
            terms = np.stack([info["rewards"][nm].cpu().numpy() for nm in env.REWARD_NAMES], axis=-1)
            o = obs.cpu().numpy().astype(np.float64)
            for i in np.nonzero(at_end)[0]:
                k, j1 = ks[i], js[i] + 1
                c = int(g["count"][k, j1])
                ctx = f"window {rows[i]}"
                assert sd["count"][i] == c and np.array_equal(words[i], g["rng"][k, j1]), ctx
                if not conditioned(ours(sd, i, c), g["state"][k, j1], c):
                    off[i] = True
                    continue
                assert abs(r[i] - g["reward"][k, j1]) <= 1e-9, ctx
                assert np.max(np.abs(terms[i] - g["terms"][k, j1])) <= 1e-9, ctx
                assert np.max(np.abs(o[i] - g["obs"][k, j1])) <= g["obs_tol"], ctx
        ended |= live & (term | trunc).astype(bool)
    left = {(int(ks[i]), int(js[i])) for i in np.nonzero(off)[0]}
    check_left(g, left, KNOWN_FORCED, name, lambda j: j + 1)


@pytest.mark.parametrize("name", ["racetrack_large_traffic", "racetrack_oval_v1_lanes4"])
def test_copy_envs_rows_stay_identical(name):
    import torch

    g = load(name)
    env = make(g, 64)
    env.reset(seed=list(range(64)))
    rng = np.random.default_rng(3)
    size = env.action_size
    act = lambda: torch.from_numpy(rng.uniform(-1, 1, size=(64, size)).astype(np.float32)).cuda()  # noqa: E731
    for _ in range(5):
        env.step(act())
    src, dst = np.arange(32), np.arange(32, 64)
    env.copy_envs(torch.from_numpy(dst).cuda(), torch.from_numpy(src).cuda())
    for _ in range(30):
        a = act()
        a[32:] = a[:32]
        obs, rew, term, trunc, _ = env.step(a)
        sd = env.state_dict()
        for k, v in sd.items():
            if np.ndim(v) and np.shape(v)[0] == 64:
                assert np.array_equal(v[dst], v[src]), k
        assert np.array_equal(env.rng_words()[:, dst], env.rng_words()[:, src])
        for t in (obs, rew, term, trunc):
            assert torch.equal(t[32:], t[:32])


def test_copy_envs_rejected_across_tracks():
    """copy_envs between different tracks raises before any launch: another class (racetrack-v0, the large track,
    the oval), an oval of another no_lanes or length, or a large track of another speed_limit."""
    import torch

    import highwayenv_b200 as hb
    from highwayenv_b200 import _native as N

    envs = {"v0": hb.make("racetrack-v0", num_envs=4), "large": hb.make("racetrack-large-v0", num_envs=4),
            "oval": hb.make("racetrack-oval-v0", num_envs=4),
            "oval4": hb.make("racetrack-oval-v0", num_envs=4, config={"no_lanes": 4}),
            "oval150": hb.make("racetrack-oval-v0", num_envs=4, config={"length": 150}),
            "large15": hb.make("racetrack-large-v0", num_envs=4, config={"speed_limit": 15})}
    for e in envs.values():
        e.reset(seed=0)
    ids = torch.arange(2).cuda()
    lib = N.load()
    before = lib.hwy_launch_count()
    for dst, src, exc in [("large", "v0", TypeError), ("v0", "large", TypeError), ("oval", "large", TypeError),
                          ("oval", "oval4", ValueError), ("oval4", "oval", ValueError), ("oval", "oval150", ValueError),
                          ("large", "large15", ValueError)]:
        with pytest.raises(exc):
            envs[dst].copy_envs(ids, ids, source=envs[src])
    assert lib.hwy_launch_count() == before
    envs["oval"].copy_envs(ids + 2, ids)  # within one track
    twin = hb.make("racetrack-oval-v0", num_envs=4)
    twin.reset(seed=7)
    envs["oval"].copy_envs(ids, ids, source=twin)


@pytest.mark.parametrize("env_id,over", [
    ("racetrack-oval-v0", {"no_lanes": 0}), ("racetrack-oval-v0", {"length": 0}), ("racetrack-oval-v1", {"no_lanes": 5}),
    ("racetrack-oval-v0", {"no_lanes": 1}), ("racetrack-oval-v0", {"block_lane": True}),
    ("racetrack-oval-v1", {"force_decision": True}), ("racetrack-large-v0", {"other_vehicles": 8}),
    ("racetrack-large-v1", {"action": {"type": "DiscreteMetaAction"}}),
])
def test_unsupported_configurations_raise_before_any_launch(env_id, over):
    import highwayenv_b200 as hb
    from highwayenv_b200 import _native as N

    lib = N.load()
    before = lib.hwy_launch_count()
    with pytest.raises((NotImplementedError, ValueError)):
        hb.make(env_id, num_envs=16, config=over).reset(seed=0)
    assert lib.hwy_launch_count() == before


@pytest.mark.parametrize("env_id,over", [("racetrack-large-v0", None), ("racetrack-oval-v1", {"no_lanes": 4})])
def test_end_to_end_4096(env_id, over):
    """hb.make of 4096 envs, reset(seed=0) and 50 steps of random steering: the ego starts on one of its ego_lanes lanes
    of ("a","b"), and the autoresets keep every env on the track's lane table."""
    import torch

    import highwayenv_b200 as hb

    env = hb.make(env_id, num_envs=4096, config=over)
    obs, _ = env.reset(seed=0)
    net = env.net
    lanes = env.state_dict()["lane"][:, 0]
    k = 4 if over else 2
    assert set(np.unique(lanes)) == {net.index[("a", "b", i)] for i in range(k)}
    rng = np.random.default_rng(0)
    for _ in range(50):
        obs, rew, term, trunc, info = env.step(torch.from_numpy(rng.uniform(-1, 1, (4096, 1)).astype(np.float32)).cuda())
    assert torch.isfinite(rew).all() and ((rew >= 0) & (rew <= 1)).all()
    assert (term.cpu().numpy().sum() > 0) and env.state_dict()["lane"].max() < len(net.lanes)


def test_state_dict_round_trip_and_road_substeps():
    import torch

    g = load("racetrack_oval_v1_lanes4")
    a_env, b_env = make(g, 32, mode="Disabled"), make(g, 32, mode="Disabled")
    a_env.reset(seed=0)
    b_env.reset(seed=99)
    rng = np.random.default_rng(5)
    a = torch.from_numpy(rng.uniform(-1, 1, size=(32, 1)).astype(np.float32)).cuda()
    a_env.step(a)
    b_env.load_state_dict(a_env.state_dict())
    b_env._rng.copy_(a_env._rng)
    frames = a_env.config["simulation_frequency"] // a_env.config["policy_frequency"]
    a_env.road_substeps(frames)
    b_env.step(a)
    sa, sb = a_env.state_dict(), b_env.state_dict()
    for k in ("x", "y", "heading", "speed", "target_speed", "timer", "lane", "target_lane", "crashed", "count"):
        assert np.array_equal(sa[k], sb[k]), k


@pytest.mark.parametrize("name", ["racetrack_large_follow", "racetrack_oval_follow"])
def test_host_stepper_graph(name):
    import torch

    g = load(name)
    env, twin = make(g, 32), make(g, 32)
    for e in (env, twin):
        e.reset(seed=[int(s) for s in g["seeds"]])
    hs = env.host_stepper()
    for t in range(40):
        hs.actions[:] = g["actions"][:, t]
        obs, rew, term, trunc = hs.step()
        o2, r2, t2, tr2, _ = twin.step(torch.from_numpy(g["actions"][:, t]).cuda())
        assert np.array_equal(obs, o2.cpu().numpy()) and np.array_equal(rew, r2.cpu().numpy())
        assert np.array_equal(term, t2.cpu().numpy()) and np.array_equal(trunc, tr2.cpu().numpy())
        assert np.array_equal(term, g["flags"][:, t, 0])


@pytest.mark.parametrize("env_id", ["racetrack-large-v0", "racetrack-large-v1", "racetrack-oval-v0",
                                    "racetrack-oval-v1"])
def test_make_single(env_id):
    import highwayenv_b200 as hb

    env = hb.make_single(env_id)
    obs, info = env.reset(seed=0)
    assert obs.shape == (2, 12, 12) and env.action_space.shape == (1,)
    obs, rew, term, trunc, info = env.step(np.array([0.1], dtype=np.float32))
    assert set(info["rewards"]) == {"lane_centering_reward", "action_reward", "collision_reward", "on_road_reward"}
