"""The highway step-kernel edge fixtures (tests/golden/highway_edges_*.npz, oracle/gen_highway_edges.py) on the CPU:
every case sits where it claims (exact ties with ==, ulp distances in exact rational arithmetic), the alternative
answer of each case is a different outcome, the frozen states stay frozen, and the C oracle, which referees much of
the GPU suite, agrees with the reference on every case: one orc_highway_substeps with the discrete outputs exactly
equal, and orc_highway_observe bit for bit."""
import json
from fractions import Fraction

import numpy as np
import pytest

from parity_utils import load_golden

FILES = ["highway_edges_v0_v20", "highway_edges_fast_v50", "highway_edges_v0_v100", "highway_edges_fast_v5"]
CONT_TOL = 1e-9
WINDOW_ABS = 2.0 ** -40  # the GPU test's faithful window around the MOBIL / d* thresholds (test_gpu_highway_edges.py)
DIAG = float(np.sqrt(5.0 ** 2 + 2.0 ** 2))


def fixture(name):
    g = load_golden(name)
    g["obs_cfgs"] = json.loads(str(g["obs_cfgs_json"]))
    return g


def cases(g, label):
    return [c for c in range(len(g["case_label"])) if str(g["case_label"][c]) == label]


def slot(g, c, j):
    return int(g["case_slots"][c][j])


def nudged(t: float, k: int) -> float:
    x = t
    for _ in range(abs(k)):
        x = float(np.nextafter(x, np.inf if k > 0 else -np.inf))
    return x


@pytest.mark.parametrize("name", FILES)
def test_cases_sit_on_their_edges(name):
    g = fixture(name)
    x, y = np.asarray(g["x"]), np.asarray(g["y"])
    seen = set()
    for c in range(len(g["case_label"])):
        label, s = str(g["case_label"][c]), int(g["case_state"][c])
        q, t, k = float(g["case_q"][c]), float(g["case_t"][c]), int(g["case_ulp"][c])
        seen.add(label)
        if label.startswith("lat"):  # lat = y - 4 * lane exactly (lane direction (1, 0))
            f, a = slot(g, c, 0), slot(g, c, 1)
            lat = Fraction(y[s, a]) - Fraction(y[s, f])
            assert Fraction(q) == lat and q == nudged(t, k), (name, c, q, t, k)
        elif label == "s-5":
            a = slot(g, c, 0)
            assert q == x[s, a] == nudged(-5.0, k), (name, c)
        elif label == "norm200":
            e, a = slot(g, c, 0), slot(g, c, 2)
            assert y[s, a] == y[s, e] and Fraction(x[s, a]) - Fraction(x[s, e]) == Fraction(q)
            assert q == nudged(200.0, k)
        elif label == "d-10":
            e, a = slot(g, c, 0), slot(g, c, 2)
            assert Fraction(x[s, a]) - Fraction(x[s, e]) == Fraction(q) and q == nudged(-10.0, k)
        elif label in ("dx5", "dy2"):
            a, b = slot(g, c, 0), slot(g, c, 1)
            axis = x if label == "dx5" else y
            diff = Fraction(axis[s, b]) - Fraction(axis[s, a])
            assert (diff > Fraction(t)) == (k > 0) and (diff == Fraction(t)) == (k == 0), (name, c)
        elif label in ("timer", "speed"):
            assert (q > t) == (k > 0) and abs(k) <= 1, (name, c)
        elif label in ("jerk", "pred_a", "abort_dstar"):
            # bracketed: the two sides of a threshold are adjacent doubles of the bisected position (about 1e-13 m
            # apart, and these quantities change by less than 1e3 per m), so the quantity sits within 1e-9 of it
            assert abs(Fraction(q) - Fraction(t)) <= Fraction(1, 10**9), (name, c, q, t)
        elif label in ("jerk_out", "pred_a_out", "abort_dstar_out"):
            # 1e-8 or 1e-6 m past the edge: outside the window, on the side the case is on
            assert WINDOW_ABS * max(1.0, abs(t)) < abs(q - t) < 1e-3, (name, c, q, t)
        elif label == "abort_d":
            assert (q, t) in ((0.0, 0.0), (8.0, 0.0)) and k == (0 if q == 0 else 10**9), (name, c, q, k)  # 10**9: "far above"
        elif label in ("sep_x", "sep_y"):
            a, b = slot(g, c, 0), slot(g, c, 1)
            gap = float(Fraction(x[s, b] - x[s, a]) - 5) if label == "sep_x" else float(
                Fraction(y[s, b]) - Fraction(y[s, a]) - 2)
            assert 0.9e-7 < gap < 1.1e-5, (name, c, gap)
        elif label in ("displacement", "touch_moving"):
            # q: the standing vehicle's x from the mover's post-move x; t: the same at the last (will_)intersecting x
            assert (q > t) == (k > 0) and (q == t) == (k == 0), (name, c, q, t, k)
        elif label == "rotated":
            a, b = slot(g, c, 0), slot(g, c, 1)
            dist = float(np.hypot(x[s, b] - x[s, a], y[s, b] - y[s, a]))
            assert abs(dist - q) < 1e-11 and abs(float(g["heading"][s, a])) <= 0.78, (name, c)
        elif label == "pruned_bound":
            e, b = slot(g, c, 0), slot(g, c, 1)
            # after the controlled vehicle's move the centres are more than a diagonal apart, but within the sweep's
            # bound diag + max(speed) * dt, which a third vehicle sets
            gap = float(g["after_x"][s, b] - g["after_x"][s, e])
            assert DIAG < gap < DIAG + float(np.max(g["speed"][s])) / g["config"]["simulation_frequency"], (name, c)
            assert np.max(g["speed"][s]) > g["speed"][s, e]
    assert {"side_by_side+2.5", "same_s", "equal_float_keys", "lat+3", "lat-3", "s-5", "timer", "speed",
            "reachable_s0", "both_sides", "jerk", "pred_a", "abort_d", "abort_dstar", "abort_order",
            "abort_by_ego"} <= seen or name.endswith("v5"), sorted(seen)
    # both sides of every bracketed threshold
    for label in ("jerk", "pred_a"):
        sides = {np.sign(float(g["case_q"][c]) - float(g["case_t"][c])) for c in cases(g, label)}
        assert len(sides) == 2 or name.endswith("v5"), (name, label, sides)


@pytest.mark.parametrize("name", FILES)
def test_alternatives_are_distinguishable(name):
    """the outcome each edge decides differs between its two sides"""
    g = fixture(name)
    tl, lane = np.asarray(g["after_target_lane"]), np.asarray(g["after_lane"])
    imp = ~np.isnan(np.asarray(g["after_impact"])[..., 0])
    if name.endswith("v5"):
        return
    for label in ("timer", "speed", "reachable_s0", "jerk", "pred_a"):
        changed = set()
        for c in cases(g, label):
            q_slot = slot(g, c, 0)
            s = int(g["case_state"][c])
            changed.add(bool(tl[s, q_slot] != np.asarray(g["target_lane"])[s, q_slot]))
        assert changed == {True, False}, (name, label)
    for label in ("dx5", "dy2"):
        hits = {bool(imp[int(g["case_state"][c]), slot(g, c, 1)]) for c in cases(g, label)}
        assert hits == {True, False}, (name, label)
    # list order: Q (lane 2 -> 1) aborts only when O, whose MOBIL sets its target this act(), comes before it
    seen = set()
    for c in cases(g, "abort_order"):
        s = int(g["case_state"][c])
        sl = [int(v) for v in g["case_slots"][c] if v >= 0]
        q = [v for v in sl if g["lane"][s, v] == 2 and g["target_lane"][s, v] == 1][0]
        o = [v for v in sl if g["lane"][s, v] == 0 and g["after_target_lane"][s, v] == 1][0]
        aborted = bool(tl[s, q] == 2)
        assert aborted == (o < q), (name, c)
        seen.add(aborted)
    assert seen == {True, False}, name
    # the follower's speed after the substep is the one behind the reference's front vehicle, and differs from the
    # one behind the other candidate
    speeds = np.asarray(g["after_speed"])
    n_fronts = 0
    for c in range(len(g["case_label"])):
        f, front, want, alt = g["case_fronts"][c]
        if f < 0:
            continue
        s = int(g["case_state"][c])
        assert speeds[s, int(f)] == want != alt, (name, c, str(g["case_label"][c]), speeds[s, int(f)], want, alt)
        n_fronts += 1
    assert n_fronts >= 20, n_fronts
    for label in ("jerk_out", "pred_a_out"):
        changed = {bool(tl[int(g["case_state"][c]), slot(g, c, 0)] != g["target_lane"][int(g["case_state"][c]),
                                                                                         slot(g, c, 0)])
                   for c in cases(g, label)}
        assert changed == {True, False}, (name, label)
    aborts = {bool(tl[int(g["case_state"][c]), slot(g, c, 0)] == lane[int(g["case_state"][c]), slot(g, c, 0)])
              for c in cases(g, "abort_dstar_out")}
    assert aborts == {True, False}, name
    crashed = np.asarray(g["after_crashed"])
    for c in cases(g, "touch_moving") + cases(g, "displacement"):
        s, e, k = int(g["case_state"][c]), slot(g, c, 0), int(g["case_ulp"][c])
        assert not g["crashed"][s, e], (name, c)
        if str(g["case_label"][c]) == "touch_moving":  # touching intersects (interval distance 0 is not > 0)
            assert crashed[s, e] == (k <= 0) and imp[s, e], (name, c)
        else:
            assert imp[s, e] == (k <= 0) and not crashed[s, e], (name, c)
    for c in cases(g, "pruned_bound"):
        assert imp[int(g["case_state"][c]), slot(g, c, 0)], (name, c)


@pytest.mark.parametrize("name", FILES[:3])
def test_collision_corners_are_separately_rounded(name):
    """the reference's polygon() corners of every collision case are (c * l + (-s) * w) + x and (s * l + c * w) + y with
    each product rounded on its own (numpy's 2 x 2 @ 2 x 4 product, no fused multiply-add), as the oracle's polygon()
    and the device's make_polygon compute them"""
    g = fixture(name)
    coll = [c for c in range(len(g["case_kind"])) if str(g["case_kind"][c]) == "collisions"]
    corners = np.asarray(g["collision_corners"])
    assert len(coll) == len(corners)
    local = [(-2.5, -1.0), (-2.5, 1.0), (2.5, 1.0), (2.5, -1.0)]
    rotated = 0
    for i, c in enumerate(coll):
        s = int(g["case_state"][c])
        for j in range(2):
            v = slot(g, c, j)
            h, px, py = (float(g[k][s, v]) for k in ("heading", "x", "y"))
            co, si = float(np.cos(h)), float(np.sin(h))
            want = np.array([[(co * a + (-si) * b) + px, (si * a + co * b) + py] for a, b in local])
            assert np.array_equal(corners[i, j], want), (name, c, j)
            rotated += h != 0.0
    assert rotated >= 12, rotated

@pytest.mark.parametrize("name", FILES)
def test_frozen_states_stay_frozen(name):
    g = fixture(name)
    fz = np.asarray(g["frozen"])
    assert fz.any()
    for k in ("x", "y", "heading", "speed", "lane", "crashed"):
        assert np.array_equal(np.asarray(g[k])[fz], np.asarray(g["after_" + k])[fz]), k
    assert np.all(np.asarray(g["crashed"])[fz]) and np.all(np.asarray(g["speed"])[fz] == 0)
    assert np.all(np.isnan(np.asarray(g["after_impact"])[fz]))


def oracle(g, obs_cfg=None):
    import hwy_oracle as ho

    cfg = dict(g["config"])
    if obs_cfg is not None:
        cfg["observation"] = dict(obs_cfg)
    S, V = np.asarray(g["x"]).shape
    ob = ho.OracleBatch(ho.cfg_from_dict(cfg), S)
    for e in range(S):
        ob.load_state(e, {k: np.asarray(g[k])[e] for k in ("x", "y", "heading", "speed", "target_speed", "timer",
                                                           "delta", "lane", "target_lane", "crashed", "impact",
                                                           "check_collisions", "speed_index", "time")})
    return ob


@pytest.mark.parametrize("name", FILES)
def test_oracle_substep_equals_reference(name):
    g = fixture(name)
    ob = oracle(g)
    S = ob.n
    for e in range(S):
        ob.substeps(e, 1)
    a = ob.a
    want_tl = np.where(np.asarray(g["after_target_lane"]) < 0, g["after_lane"], g["after_target_lane"])
    for k, want in (("lane", g["after_lane"]), ("target_lane", want_tl), ("crashed", g["after_crashed"]),
                    ("has_impact", ~np.isnan(np.asarray(g["after_impact"])[..., 0]))):
        bad = np.argwhere(a[k].astype(np.int32) != np.asarray(want).astype(np.int32))
        assert not len(bad), (name, k, bad[:5], [str(g["case_label"][c]) for c in range(len(g["case_label"]))
                                                 if g["case_state"][c] == bad[0][0]])
    for k in ("x", "y", "heading", "speed", "timer"):
        d = np.abs(a[k] - np.nan_to_num(np.asarray(g["after_" + k])))
        assert np.max(d) <= CONT_TOL, (name, k, float(np.max(d)))
    hi = a["has_impact"].astype(bool)
    imp = np.asarray(g["after_impact"])
    assert np.max(np.abs(a["impact_x"][hi] - imp[..., 0][hi]), initial=0.0) <= CONT_TOL
    assert np.max(np.abs(a["impact_y"][hi] - imp[..., 1][hi]), initial=0.0) <= CONT_TOL


@pytest.mark.parametrize("name", FILES)
def test_oracle_observe_equals_reference(name):
    g = fixture(name)
    for k, cfg in enumerate(g["obs_cfgs"]):
        ob = oracle(g, cfg)
        want = np.asarray(g[f"obs_{k}"])
        for e in range(ob.n):
            got = ob.observe(e)
            assert np.array_equal(got.view(np.int32), want[e].view(np.int32)), (name, k, cfg, e, got, want[e])


def test_fixtures_are_small():
    import os

    from parity_utils import GOLDEN

    sizes = [os.path.getsize(os.path.join(GOLDEN, n + ".npz")) for n in FILES]
    assert sum(sizes) < 400e3, sizes
