"""The highway step kernel at the edges of its discrete decisions, against the unmodified reference (fixtures
highway_edges_*.npz, oracle/gen_highway_edges.py): front-neighbour ties (each candidate front vehicle leaves the
follower with another speed) and lane membership at lat = +-3 and s = -5, the lane-change timer, speed and reachability
gates, both side lanes passing MOBIL, the abort of an ongoing change in list order, touching and nearly touching
rectangles (also a moving, uncrashed one) with the impact's direction, and the Kinematics rows at the perception
distance, the -10 m gate and |d| ties.

Every state is loaded with load_state_dict and
  * advanced by road_substeps(1): lane, target_lane, crashed and has_impact equal the reference's, the continuous
    fields within 1e-7 (what the parity tests hold the kernel to after a whole step);
  * observed by observe() under every Kinematics configuration of the fixture: the reference's float32 bytes;
  * (frozen states: every vehicle crashed at speed 0) stepped once: the fused epilogue's observation is the same
    bytes and the state is unchanged;
on every instantiation the dispatcher can pick for its vehicle count: the congruent-lane and the general-geometry
kernels (HWYB200_GENERAL_LANES=1), dense and TPE-thread env segments (HWYB200_EPB).

MOBIL's jerk and new_following_pred_a and the abort's d* are reached through idm_pow / sqrt chains that are faithful
to a few ulp, not correctly rounded like numpy's pow.  The cases bisected onto those thresholds (adjacent doubles of
the bisected position) sit inside WINDOW_ABS of the quantity, where the kernel may take either answer: their vehicles
are excluded from the comparison (run with -s to see in-window disagreements).  The same thresholds are also
bracketed 1e-8 m and 1e-6 m past the edge on both sides (jerk_out, pred_a_out, abort_dstar_out), outside the window:
there the decision must be the reference's on every instantiation."""
import json

import numpy as np
import pytest

from parity_utils import load_golden

pytestmark = pytest.mark.gpu

FILES = ["highway_edges_v0_v20", "highway_edges_fast_v50", "highway_edges_v0_v100", "highway_edges_fast_v5"]
# (dense envs per block, TPE-thread envs per block) for each vehicle count: dense segments run when epb * TPE exceeds
# half of the 512-thread block limit (hwy_highway.cu launch_step)
EPB = {21: (12, 8), 51: (5, 4), 101: (3, 2), 6: (12, 8)}
VARIANTS = ["auto", "general", "dense", "tpe"]
CONT = ("x", "y", "heading", "speed", "timer", "target_speed")
CONT_TOL = 1e-7
# idm_pow and the device sqrt / division chain are within 4 ulp of numpy's results (test_gpu_device_math.py); the
# compared quantities are sums of a few such terms of magnitude <= 20 (m/s^2, m), so 2^-40 bounds their difference
WINDOW_ABS = 2.0 ** -40


def fixture(name):
    g = load_golden(name)
    g["obs_cfgs"] = json.loads(str(g["obs_cfgs_json"]))
    return g


def state_dict(g, prefix=""):
    """the fixture's dump_state arrays [S, V] as a load_state_dict payload (the controlled vehicle is an MDPVehicle)"""
    p = lambda k: np.asarray(g[prefix + k])  # noqa: E731
    S, V = p("x").shape
    sd = {k: p(k).copy() for k in ("x", "y", "heading", "speed")}
    sd["target_speed"] = np.nan_to_num(p("target_speed"), nan=0.0)
    sd["timer"] = np.nan_to_num(p("timer"), nan=0.0)
    sd["delta"] = np.nan_to_num(p("delta"), nan=4.0)
    imp = p("impact")
    sd["has_impact"] = ~np.isnan(imp[..., 0])
    sd["impact_x"], sd["impact_y"] = np.nan_to_num(imp[..., 0]), np.nan_to_num(imp[..., 1])
    sd["lane"] = p("lane").astype(np.int32)
    sd["target_lane"] = np.where(p("target_lane") < 0, p("lane"), p("target_lane")).astype(np.int32)
    sd["crashed"] = p("crashed").astype(bool)
    sd["check_collisions"] = p("check_collisions").astype(bool)
    kind = np.zeros((S, V), dtype=np.int32)
    kind[:, 0] = 1
    sd["kind"] = kind
    sd["speed_index"] = p("speed_index")[:, 0].astype(np.int32)
    sd["time"] = np.asarray(g[prefix + "time"], dtype=np.float64).reshape(S)
    return sd


def windowed_slots(g):
    """[S, V] bool: the vehicles of threshold cases whose reference quantity is inside the faithful window"""
    S, V = np.asarray(g["x"]).shape
    out = np.zeros((S, V), dtype=bool)
    for c in np.nonzero(g["case_window"])[0]:
        if abs(float(g["case_q"][c]) - float(g["case_t"][c])) <= WINDOW_ABS * max(1.0, abs(float(g["case_t"][c]))):
            slots = g["case_slots"][c]
            out[g["case_state"][c], slots[slots >= 0]] = True
    return out


def make(g, obs_cfg=None, variant="auto", monkeypatch=None):
    import highwayenv_b200 as hb

    cfg = dict(g["config"])
    env_id = cfg.pop("_env_id")
    if obs_cfg is not None:
        cfg["observation"] = dict(obs_cfg)
    V = int(cfg["vehicles_count"]) + 1
    if variant == "general":
        monkeypatch.setenv("HWYB200_GENERAL_LANES", "1")
    elif variant in ("dense", "tpe"):
        monkeypatch.setenv("HWYB200_EPB", str(EPB[V][variant == "tpe"]))
    S = np.asarray(g["x"]).shape[0]
    env = hb.make(env_id, num_envs=S, config=cfg, autoreset_mode="Disabled")
    env.reset(seed=0)
    env.load_state_dict(state_dict(g))
    return env


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", FILES)
def test_one_substep_matches_reference(name, variant, monkeypatch):
    g = fixture(name)
    env = make(g, variant=variant, monkeypatch=monkeypatch)
    env.road_substeps(1)
    got = env.state_dict()
    want = state_dict(g, "after_")
    skip = windowed_slots(g)
    kinds = np.asarray(g["case_kind"])
    for k in ("lane", "target_lane", "crashed", "has_impact"):
        a, b = np.asarray(got[k]).astype(np.int32), np.asarray(want[k]).astype(np.int32)
        bad = (a != b) & ~skip
        if bad.any():
            s, v = np.argwhere(bad)[0]
            cases = [str(g["case_label"][c]) for c in np.nonzero(g["case_state"] == s)[0] if v in g["case_slots"][c]]
            raise AssertionError(f"{name} {variant} {k}: state {s} slot {v} got {a[s, v]} want {b[s, v]} {cases}")
        if (a != b).any():
            print(f"\n{name} {variant}: {k} differs on {int((a != b).sum())} in-window vehicles")
    for k in CONT:
        d = np.abs(np.asarray(got[k]) - want[k])
        d[skip] = 0.0
        assert np.max(d) <= CONT_TOL, (name, variant, k, float(np.max(d)), np.argwhere(d > CONT_TOL)[:3])
    hi = want["has_impact"] & ~skip
    for k in ("impact_x", "impact_y"):
        d = np.abs(np.asarray(got[k])[hi] - want[k][hi])
        assert d.size == 0 or np.max(d) <= CONT_TOL, (name, variant, k, float(np.max(d)))
    assert set(np.unique(kinds)) <= {"neighbours", "lane_change", "collisions", "kinematics"}


@pytest.mark.parametrize("name", FILES)
def test_observe_bit_exact(name):
    """highway_observe_kernel: every Kinematics configuration, the reference's float32 bytes"""
    g = fixture(name)
    for k, cfg in enumerate(g["obs_cfgs"]):
        env = make(g, cfg)
        got = env.observe().cpu().numpy()
        want = np.asarray(g[f"obs_{k}"])
        assert got.shape == want.shape and got.dtype == want.dtype, (name, k, got.shape, want.shape)
        bad = np.nonzero(np.any((got.view(np.int32) != want.view(np.int32)).reshape(len(want), -1), axis=1))[0]
        assert not len(bad), (name, k, cfg, bad[:5], got[bad[0]], want[bad[0]])


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", FILES)
def test_frozen_step_epilogue_bit_exact(name, variant, monkeypatch):
    """the step kernel's fused Kinematics epilogue on the frozen states (every vehicle crashed at speed 0): the
    observation of the crafted state, and the state unchanged"""
    g = fixture(name)
    frozen = np.asarray(g["frozen"])
    assert frozen.any()
    for k, cfg in enumerate(g["obs_cfgs"]):
        env = make(g, cfg, variant, monkeypatch)
        before = env.state_dict()
        obs, *_ = env.step(np.ones(env.num_envs, dtype=np.int32))  # IDLE
        got = obs.cpu().numpy()[frozen]
        want = np.asarray(g[f"obs_{k}"])[frozen]
        bad = np.nonzero(np.any((got.view(np.int32) != want.view(np.int32)).reshape(len(want), -1), axis=1))[0]
        assert not len(bad), (name, variant, k, cfg, bad[:5])
        after = env.state_dict()
        for key in ("x", "y", "heading", "speed", "lane", "target_lane", "crashed", "has_impact"):
            assert np.array_equal(np.asarray(after[key])[frozen], np.asarray(before[key])[frozen]), (name, k, key)


def test_fixture_coverage():
    """each step-kernel width (V <= 32, 33-64, 65-128) and both collision regimes (every vehicle checks: the
    rank-pruned sweep; only the controlled vehicle: the single-checker sweep) have every kind"""
    seen = {}
    for name in FILES:
        g = fixture(name)
        V = np.asarray(g["x"]).shape[1]
        seen[(V, g["config"]["_env_id"])] = set(np.unique(g["case_kind"]).tolist())
    full = {"neighbours", "lane_change", "collisions", "kinematics"}
    assert seen[(21, "highway-v0")] == full and seen[(51, "highway-fast-v0")] == full
    assert seen[(101, "highway-v0")] == full and seen[(6, "highway-fast-v0")] == {"kinematics"}


@pytest.mark.parametrize("name", FILES[:3])
def test_threshold_cases_outside_the_window_are_compared(name):
    """each MOBIL / d* threshold has cases outside the window on both sides, which the substep test compares"""
    g = fixture(name)
    w = windowed_slots(g)
    for label in ("jerk_out", "pred_a_out", "abort_dstar_out"):
        cs = [c for c in range(len(g["case_label"])) if str(g["case_label"][c]) == label]
        assert len(cs) == 4, (name, label)
        sides = {np.sign(float(g["case_q"][c]) - float(g["case_t"][c])) for c in cs}
        assert sides == {-1.0, 1.0}, (name, label)
        for c in cs:
            s, q = int(g["case_state"][c]), int(g["case_slots"][c][0])
            assert not w[s, q], (name, label, c)
