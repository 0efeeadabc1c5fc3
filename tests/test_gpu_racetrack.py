"""GPU parity of racetrack-v0 / racetrack-v1 (hwy_racetrack_reset / hwy_racetrack_step) against the fixtures of
oracle/gen_racetrack.py: the device reset, free-running rollouts with SameStep autoreset (terminations, truncations,
rewards, stream words, the OccupancyGrid), many envs, NextStep, env cloning, state_dict, road_substeps and the host
stepper's CUDA graph."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["racetrack_random", "racetrack_follow", "racetrack_traffic", "racetrack_v1_follow", "racetrack_kinematics"]
FLOATS = ("x", "y", "heading", "speed", "target_speed", "timer")
INTS = ("lane", "target_lane", "kind", "crashed")
FIELDS = FLOATS + INTS  # the fixture's row order
TOL = 1e-6  # positions / headings / speeds / timers: CUDA's sincos and atan2 against numpy's, over the rollouts


def load(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    g["config"] = json.loads(str(g.pop("config_json")))
    g["slot"] = {int(t): j for j, t in enumerate(g["steps"])}
    g["obs_tol"] = 0.0 if g["obs"].ndim == 5 else 1e-6  # the grid is exact; Kinematics rows are float32 of fp64
    return g


# ---------------------------------------------------------------- the one ill-conditioned place of the track
# Lane 1 of ("g","h") ends at 165 deg and lane 1 of ("h","i") starts at 170 deg on the same circle (center (18.1,
# -18.1), radius 30).  Between the two angles both lanes contain the vehicle, and get_closest_lane_index compares two
# mathematically equal distances (same |lateral|, same heading term): the last bits of atan2 / sincos decide which lane
# wins, and so on which substep the vehicle's lane index moves on, which can shift an IDM vehicle's lane-change timer
# by whole substeps.  Every other pair of lanes differs in center or radius.  Which windows of the reference pass a
# vehicle through that place is decided from the reference's states alone (crossing_windows); a divergence is allowed
# only where it is listed below and falls in such a window.
def _gh1():
    from highwayenv_b200.envs.racetrack_env import make_racetrack_network

    return make_racetrack_network().index[("g", "h", 1)]


def _on_gh1(st, count):
    return st[6, :count] == _gh1()


def window_crosses(starts, end_state, end_count):
    """Whether the reference can have moved a vehicle off ("g","h",1) within a window.  `starts`: the (state, count)
    the window starts from and each reset inside it, in order; `end_state` follows the last of them.  Before a reset
    inside the window the end is not stored, so a vehicle on ("g","h",1) at such a start counts as crossing."""
    for st, c in starts[:-1]:
        if _on_gh1(st, c).any():
            return True
    st, c = starts[-1]
    n = min(c, end_count)
    return bool((_on_gh1(st, n) & (end_state[6, :n] != _gh1())).any())


def crossing_windows(g):
    """[n_envs, n_stored] bool: whether the reference can pass a vehicle through the overlap in the window that ends
    at stored step j (it starts after the previous stored step, or at the first reset)."""
    n, T = g["actions"].shape[:2]
    out = np.zeros((n, len(g["steps"])), dtype=bool)
    for k in range(n):
        start = (g["reset_state"][k], int(g["reset_count"][k]))
        resets = {int(t): m for m, t in enumerate(g["autoreset_step"][k]) if t >= 0}
        a = -1
        for j, b in enumerate(g["steps"]):
            inner = [(g["autoreset_state"][k, resets[t]], int(g["autoreset_count"][k, resets[t]]))
                     for t in range(a + 1, int(b)) if t in resets]
            out[k, j] = window_crosses([start] + inner, g["state"][k, j], int(g["count"][k, j]))
            m = resets.get(int(b))
            start = (g["state"][k, j], int(g["count"][k, j])) if m is None else \
                (g["autoreset_state"][k, m], int(g["autoreset_count"][k, m]))
            a = int(b)
    return out


def window_of(g, t):
    """Index of the stored window (a, b] that contains step t."""
    return int(np.searchsorted(g["steps"], t))


# The divergences the lane overlap causes in these fixtures, each in a window where the reference passes a vehicle
# through it: free-running (env, first stored step that differs), teacher-forced (env, window start index).
KNOWN_FREE = {"racetrack_random": set(), "racetrack_follow": set(), "racetrack_traffic": {(6, 129)},
              "racetrack_v1_follow": set(), "racetrack_kinematics": {(5, 119), (6, 159)}}
KNOWN_FORCED = {"racetrack_random": set(), "racetrack_follow": set(), "racetrack_traffic": set(),
                "racetrack_v1_follow": set(), "racetrack_kinematics": {(5, 10), (6, 14)}}


def make(g, n=None, mode="SameStep"):
    import highwayenv_b200 as hb

    return hb.make(g["config"]["_env_id"], num_envs=n or len(g["seeds"]), config=dict(g["config"]["_override"]),
                   autoreset_mode=mode)


def ours(sd, i, count):
    """Env i's state in the fixture's row order, the first `count` slots."""
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
    """True while the env follows the reference: floats within TOL, lanes, target lanes, kinds and crashes equal."""
    ref = ref[:, :count]
    nf = len(FLOATS)
    return (not count or float(np.max(np.abs(st[:nf] - ref[:nf]))) <= TOL) and np.array_equal(st[nf:], ref[nf:])


@pytest.mark.parametrize("name", CASES)
def test_reset_matches_reference(name):
    g = load(name)
    env = make(g)
    obs, _ = env.reset(seed=[int(s) for s in g["seeds"]])
    sd = env.state_dict()
    assert np.array_equal(env.rng_words().T, g["reset_rng"])
    assert np.array_equal(sd["count"], g["reset_count"])
    worst = 0.0
    for i in range(len(g["seeds"])):
        c = int(g["reset_count"][i])
        st = ours(sd, i, c)
        # the ego is placed on a straight lane (exact); the others through CUDA's sincos on the arcs
        assert np.array_equal(st[:, 0], g["reset_state"][i][:, 0]), i
        worst = max(worst, compare(st, g["reset_state"][i], c, f"reset#{i}"))
    assert worst <= 1e-12, worst
    assert np.max(np.abs(obs.cpu().numpy().astype(np.float64) - g["reset_obs"])) <= g["obs_tol"]


def rollout(g, env, ids=None, check_obs=True):
    """Steps `env` (SameStep) with the fixture's actions; env ids[k] is fixture seed k.  Every env is checked on every
    step (flags), at every reset (population, stream words, state) and at the stored steps (state, stream words,
    reward, reward terms, observation).  An env that leaves the reference (flags, or its state by more than TOL or in
    a discrete field) is recorded as (env, step) and followed no further.  Returns the recorded set."""
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
            terms = np.stack([info["rewards"][name].cpu().numpy()[ids] for name in env.REWARD_NAMES], axis=-1)
            assert np.max(np.abs(r - g["reward"][:, j])[alive], initial=0.0) <= 1e-9, t
            assert np.max(np.abs(terms - g["terms"][:, j])[alive], initial=0.0) <= 1e-9, t
            if check_obs:  # the observation of the step (final_obs where SameStep reset the env)
                o = info["final_obs"].cpu().numpy()[ids].astype(np.float64)
                assert np.max(np.abs(o - g["obs"][:, j])[alive], initial=0.0) <= g["obs_tol"], t
    return left


def check_left(g, left, known, name):
    """The envs that left the reference are exactly the known ones, and each left in a window where the reference
    passes a vehicle through the lane overlap."""
    cross = crossing_windows(g)
    assert left == known[name], (name, sorted(left))
    for k, t in left:
        assert cross[k, window_of(g, t)], (k, t)


@pytest.mark.parametrize("name", CASES)
def test_free_running_matches_reference(name):
    """200 steps with SameStep autoreset: terminations, truncations and crashes exact on every step, every reset exact
    in population and stream words, the stored steps' state (<= 1e-6), reward (<= 1e-9), reward terms and
    observation.  The only envs allowed to leave the reference are the listed ones at the lane overlap."""
    g = load(name)
    env = make(g)
    env.reset(seed=[int(s) for s in g["seeds"]])
    check_left(g, rollout(g, env), KNOWN_FREE, name)


def load_reference_rows(env, g, rows):
    """Load the fixture's stored states (k, j) into the env rows 0.. in order: state, pending impacts, clock, count and
    stream words."""
    n = len(rows)
    V = env.V
    st = np.stack([g["state"][k, j][:, :V] for k, j in rows])  # [n, fields, V]
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
    """Every stored state (that did not end its episode) is loaded and the stored actions replayed up to the next
    stored step: flags exact on every step up to the first episode end, and at the next stored step the state
    (<= 1e-6), stream words, reward (<= 1e-9), reward terms and observation.  The only windows allowed to leave the
    reference are the listed ones at the lane overlap."""
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
    assert left == KNOWN_FORCED[name], (name, sorted(left))
    cross = crossing_windows(g)
    for k, j in left:
        assert cross[k, j + 1], (k, j)


def test_many_envs_independent_of_num_envs():
    """racetrack_traffic's 32 seeds inside a batch of 65 536 envs (the other envs act at random)."""
    g = load("racetrack_traffic")
    n = 65536
    env = make(g, n)
    ids = np.arange(0, n, n // 32)[:32]
    seeds = np.arange(n) + 10_000
    seeds[ids] = g["seeds"]
    env.reset(seed=[int(s) for s in seeds])
    check_left(g, rollout(g, env, ids, check_obs=False), KNOWN_FREE, "racetrack_traffic")


@pytest.mark.parametrize("n", [32, 65536])
def test_next_step_autoreset(n):
    """NextStep, with the fixture's 32 seeds alone or spread over a batch of 65 536 envs (the others act at random):
    the call after an episode ends returns the reset observation with reward 0 and both flags False, and the flags of
    every other call are the reference's."""
    import torch

    g = load("racetrack_random")
    env = make(g, n, mode="NextStep")
    ids = np.arange(0, n, n // 32)[:32]
    seeds = np.arange(n) + 10_000
    seeds[ids] = g["seeds"]
    env.reset(seed=[int(s) for s in seeds])
    T = g["actions"].shape[1]
    extra = np.random.default_rng(9).uniform(-1, 1, size=(n, 1)).astype(np.float32)
    pending = np.zeros(len(ids), dtype=bool)
    res_k = np.zeros(len(ids), dtype=int)
    lag = np.zeros(len(ids), dtype=int)  # steps this env is behind the fixture
    checked = 0
    for t in range(T):
        # env k plays the fixture's action of its own episode step (NextStep spends one call on each reset)
        a = extra.copy()
        a[ids] = np.stack([g["actions"][k, min(t - lag[k], T - 1)] for k in range(len(ids))])
        obs, rew, term, trunc, _ = env.step(torch.from_numpy(a).cuda())
        rew, term, trunc = rew.cpu().numpy()[ids], term.cpu().numpy()[ids], trunc.cpu().numpy()[ids]
        o = obs.cpu().numpy()[ids].astype(np.float64)
        for k in np.nonzero(pending)[0]:
            m = res_k[k]
            assert rew[k] == 0.0 and not term[k] and not trunc[k]
            assert np.array_equal(o[k], g["autoreset_obs"][k, m]), (t, k)
            res_k[k] += 1
            lag[k] += 1
            checked += 1
        for k in np.nonzero(~pending)[0]:
            tf = t - lag[k]
            if tf < T:
                assert bool(term[k]) == g["flags"][k, tf, 0], (t, k)
        pending = (term | trunc).astype(bool)
    assert checked >= 100


def test_copy_envs_rows_stay_identical():
    import torch

    g = load("racetrack_traffic")
    env = make(g, 64)
    env.reset(seed=list(range(64)))
    rng = np.random.default_rng(3)
    act = lambda: torch.from_numpy(rng.uniform(-1, 1, size=(64, 2)).astype(np.float32)).cuda()  # noqa: E731
    for _ in range(5):
        env.step(act())
    copied = set(env._env_rows())
    for name, t in vars(env).items():  # every per-env tensor is copied or declared as not part of the state
        if isinstance(t, torch.Tensor) and t.dim() >= 1 and t.shape[0] == 64:
            assert name in copied or name in env.ROW_EXCLUDE, name
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


def test_state_dict_round_trip_and_road_substeps():
    """load_state_dict reproduces a batch; road_substeps replays the ego's persisting action, so a step followed by
    `frames` substeps equals two steps with the same action."""
    import torch

    g = load("racetrack_traffic")
    a_env, b_env = make(g, 32, mode="Disabled"), make(g, 32, mode="Disabled")
    a_env.reset(seed=0)
    b_env.reset(seed=99)
    rng = np.random.default_rng(5)
    a = torch.from_numpy(rng.uniform(-1, 1, size=(32, 2)).astype(np.float32)).cuda()
    a_env.step(a)
    b_env.load_state_dict(a_env.state_dict())
    b_env._rng.copy_(a_env._rng)
    frames = a_env.config["simulation_frequency"] // a_env.config["policy_frequency"]
    a_env.road_substeps(frames)
    b_env.step(a)
    sa, sb = a_env.state_dict(), b_env.state_dict()
    for k in ("x", "y", "heading", "speed", "target_speed", "timer", "lane", "target_lane", "crashed", "count"):
        assert np.array_equal(sa[k], sb[k]), k


def test_host_stepper_graph():
    import torch

    g = load("racetrack_follow")
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


def test_make_single():
    import highwayenv_b200 as hb

    env = hb.make_single("racetrack-v0")
    obs, info = env.reset(seed=0)
    assert obs.shape == (2, 12, 12) and env.action_space.shape == (1,)
    obs, rew, term, trunc, info = env.step(np.array([0.1], dtype=np.float32))
    assert set(info["rewards"]) == {"lane_centering_reward", "action_reward", "collision_reward", "on_road_reward"}
