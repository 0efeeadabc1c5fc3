"""Generate the highway step-kernel edge fixtures tests/golden/highway_edges_*.npz from the UNMODIFIED reference (build
container only).

    python oracle/gen_highway_edges.py

The step kernel reaches discrete answers (which vehicle is in front, whether a lane change fires or is aborted,
whether a pair collides and which way the impact acts, which vehicle fills which Kinematics row) through comparisons
that random rollouts never bring to their edge.  Here each state is a reference reset whose vehicles are moved to
crafted poses on the reference's own objects (position, heading, speed, lane_index / lane, target_lane_index, timer,
target_speed, crashed), and the reference records

  * `ref_harness.dump_state` of the crafted state (keys without prefix),
  * its Kinematics observation under every configuration of OBS_CFGS (`obs_<k>`),
  * the state after exactly one `road.act(); road.step(1 / simulation_frequency)` (`after_<key>`), which is what
    `env.road_substeps(1)` implements.

Each state holds one or more cases, separated along the road (groups 400 m apart; the vehicles a state does not use
are parked 6 km down the road).  Kinds:

  neighbours   ties and membership edges of Road.neighbour_vehicles (road/road.py:483-547): two members side by side at
               one s, a member at the querier's own s, equal float32 keys of different doubles, lat = +-3 and s = -5
               within a few ulp; every candidate front vehicle has another speed, so the follower's speed tells them
               apart
  lane_change  the timer (LANE_CHANGE_DELAY < timer), |speed| < 1, is_reachable_from (0 <= s), both side lanes passing
               MOBIL (the right one wins), MOBIL's jerk, new_following_pred_a and the abort's d* bisected onto
               their thresholds (adjacent doubles) and bracketed 1e-8 m and 1e-6 m past them, the abort of an
               ongoing change at d = 0, in list order (an earlier vehicle's target set in the
               same act() is seen, a later one's is not), and the controlled vehicle causing an abort
  collisions   aligned rectangles touching (dx = 5, dy = 2) and a few ulp apart, separations of 1e-7 .. 1e-5 m,
               coincident and mirrored centres, a vehicle with several will_intersect partners below and above its
               slot, gaps that only the controlled vehicle's displacement closes, the moving (uncrashed) controlled
               vehicle touching a standing one, rotated pairs within +-0.78 rad
  kinematics   frozen states (every vehicle crashed at speed 0, no two rectangles touching, so Vehicle.step leaves the
               world unchanged bit for bit): norm = PERCEPTION_DISTANCE and -10 m within a few ulp, |d| ties (ahead /
               behind, side by side, three-way), a tie group across the vehicles_count - 1 cutoff, fewer candidates
               than rows, ranges landing on +-1

Every threshold case records the reference's value of the compared quantity (`case_q`), the threshold (`case_t`),
their distance in ulp of the threshold (`case_ulp`) and whether the kernel reaches it through an idm_pow / sqrt chain
(`case_window`).  The file also records numpy's version.
"""
from __future__ import annotations

import copy
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ref_harness as rh  # noqa: E402
from gen_obs_edges import nudge  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

# name -> (env id, config override, reset seed, kinds)
ALL_KINDS = ("neighbours", "lane_change", "collisions", "kinematics")
FILES = {
    "highway_edges_v0_v20": ("highway-v0", {"vehicles_count": 20}, 3100, ALL_KINDS),
    "highway_edges_fast_v50": ("highway-fast-v0", {"vehicles_count": 50}, 3110, ALL_KINDS),
    "highway_edges_v0_v100": ("highway-v0", {"vehicles_count": 100}, 3120, ALL_KINDS),
    "highway_edges_fast_v5": ("highway-fast-v0", {"vehicles_count": 5}, 3130, ("kinematics",)),
}
OBS_CFGS = [
    {"type": "Kinematics"},
    {"type": "Kinematics", "see_behind": True},
    {"type": "Kinematics", "absolute": True},
    {"type": "Kinematics", "normalize": False},
    {"type": "Kinematics", "clip": False, "vehicles_count": 7},
    {"type": "Kinematics", "features": ["presence", "x", "y", "heading", "cos_h", "sin_h", "long_off", "lat_off",
                                        "ang_off"]},
    {"type": "Kinematics", "features": ["presence", "x", "y", "vx", "vy"],
     "features_range": {"x": [-30, 30], "y": [-8, 8], "vx": [-20, 20], "vy": [-20, 20]}},
    {"type": "Kinematics", "vehicles_count": 16, "see_behind": True},
]
GROUP_SPACING = 400.0
MAX_GROUPS = 12  # per state: the last group ends well before the parked vehicles
PARK_X = 6000.0
KIN_EGO = (3000.0, 4.0)
# metres past a bisected MOBIL / d* edge: outside the window in which the device's idm_pow / sqrt chain may take either
# side (the compared quantities move by more than 1e-3 per metre there)
OFFSETS = (-1e-6, -1e-8, 1e-8, 1e-6)


class Case:
    """One crafted situation: vehicle specs by role, the roles in ascending slot order, and what it pins."""

    def __init__(self, kind, label, specs, order=None, anchored=False, q=np.nan, t=np.nan, ulp=0, window=False,
                 check=None, fronts=None):
        self.kind, self.label, self.specs = kind, label, specs
        # fronts = (follower, candidates): the follower's front vehicle is one of the candidates, and its speed after
        # the substep tells which (recorded with the speed the other candidate would have given)
        self.fronts = fronts
        self.order = order or list(specs)
        self.anchored = anchored  # absolute x (s = -5, x = 0): one such case per state, at group origin 0
        self.q, self.t, self.ulp, self.window = q, t, ulp, window
        self.check = check  # check(env, roles) -> None, asserts on the crafted reference state


def spec(x, y, speed, heading=0.0, target_lane=None, timer=0.0, target_speed=None, crashed=False, nudge=None):
    """nudge = (axis, k): the placed (absolute) coordinate moved by k ulp"""
    return dict(x=float(x), y=float(y), speed=float(speed), heading=float(heading), target_lane=target_lane,
                timer=float(timer), target_speed=target_speed, crashed=crashed, nudge=nudge)


FAR = 10**9  # case_ulp of a quantity more than a billion doubles from its threshold: only the side is meant


def ulps(q: float, t: float) -> int:
    """signed distance of q from t in doubles (exactly, from the integer pattern when both share a sign), clamped to
    +-FAR"""
    if q == t:
        return 0
    a, b = (int(v) for v in np.array([q, t], dtype=np.float64).view(np.int64))
    n = (a - b if q >= 0 else b - a) if (q >= 0) == (t >= 0) else FAR
    return int(np.sign(q - t)) * min(abs(n), FAR)


def lane_of(env, x, y, heading):
    return env.road.network.get_closest_lane_index(np.array([x, y], dtype=np.float64), heading)


def place(env, v, s, x0):
    v.position = np.array([s["x"] + x0, s["y"]], dtype=np.float64)
    if s.get("nudge"):
        axis, k = s["nudge"]
        v.position[axis] = nudge(float(v.position[axis]), k)
    v.heading = s["heading"]
    v.speed = s["speed"]
    v.lane_index = lane_of(env, v.position[0], v.position[1], v.heading)
    v.lane = env.road.network.get_lane(v.lane_index)
    if hasattr(v, "target_lane_index"):
        tl = s["target_lane"]
        v.target_lane_index = v.lane_index if tl is None else ("0", "1", int(tl))
    if hasattr(v, "target_speed"):
        v.target_speed = s["speed"] if s["target_speed"] is None else float(s["target_speed"])
    if hasattr(v, "timer"):
        v.timer = s["timer"]
    v.crashed = bool(s["crashed"])
    v.impact = None


def park(env, v, k, frozen):
    lanes = int(env.config["lanes_count"])
    place(env, v, spec(PARK_X + 30.0 * k, 4.0 * (k % lanes), 0.0 if frozen else 25.0, crashed=frozen), 0.0)


# ------------------------------------------------------------------ reference helpers
def accel(env, me, ego, front):
    return float(me.acceleration(ego_vehicle=ego, front_vehicle=front))


def neighbours(env, v, lane=None):
    return env.road.neighbour_vehicles(v, lane)


def clipped_accel(v, front):
    """IDMVehicle.act's acceleration of v (not changing lanes) behind `front`, clipped to +-ACC_MAX (behavior.py:133-134)"""
    return float(np.clip(v.acceleration(ego_vehicle=v, front_vehicle=front), -v.ACC_MAX, v.ACC_MAX))


def distinct_fronts(f, cands):
    """the follower's clipped acceleration, and so its speed after the substep, differs with each candidate as its
    front vehicle"""
    def check(env, r):
        a = [clipped_accel(r[f], r[c]) for c in cands]
        assert len(set(a)) == len(a), (f, cands, a)
    return check


# ------------------------------------------------------------------ neighbours
def neighbour_cases(lanes):
    out = []
    # two members of lane 1 at one s: A on the centre line, B 2.5 m to the side (lane 2 or 0), not touching
    for side in (+2.5, -2.5):
        for order in (["F", "A", "B", "C"], ["F", "B", "A", "C"], ["B", "A", "F", "C"]):
            # 70 m ahead: the follower brakes by about 1 to 2 m/s^2, below ACC_MAX, differently behind 22 and 26 m/s
            specs = {"F": spec(0, 4, 24), "A": spec(70, 4, 22), "B": spec(70, 4 + side, 26), "C": spec(130, 4, 27)}

            def check(env, r):
                front, _ = neighbours(env, r["F"])
                later = max((r["A"], r["B"]), key=lambda v: env.road.vehicles.index(v))
                assert front is later
                distinct_fronts("F", ["A", "B"])(env, r)
            out.append(Case("neighbours", f"side_by_side{side:+}", specs, order, check=check, fronts=("F", ["A", "B"])))
    # a member at exactly the querier's own s (it counts as front), 2.5 m to the side
    for order in (["F", "A", "C"], ["A", "F", "C"]):
        specs = {"F": spec(0, 4, 22), "A": spec(0, 6.5, 15), "C": spec(40, 4, 26)}

        def check(env, r):
            assert neighbours(env, r["F"])[0] is r["A"]
            distinct_fronts("F", ["A", "C"])(env, r)
        out.append(Case("neighbours", "same_s", specs, order, check=check, fronts=("F", ["A", "C"])))
    # equal float keys of different doubles: A and B round to one float32, the smaller double is in front
    for order in (["F", "A", "B"], ["F", "B", "A"]):
        specs = {"F": spec(0, 4, 24), "A": spec(70, 4, 22), "B": spec(70, 6.5, 26)}

        def check(env, r):
            r["B"].position[0] = float(np.nextafter(r["A"].position[0], np.inf))
            assert np.float32(r["B"].position[0]) == np.float32(r["A"].position[0])
            assert neighbours(env, r["F"])[0] is r["A"]
            distinct_fronts("F", ["A", "B"])(env, r)
        out.append(Case("neighbours", "equal_float_keys", specs, order, check=check, fronts=("F", ["A", "B"])))
    # lat = +-3 (|lat| <= width / 2 + 1) within a few ulp: A is a member of two lanes or of one
    for k in (-4, -2, -1, 0, 1, 2, 4):
        for sign, fl in ((+1, 1), (-1, 2)):
            y = nudge(4.0 * fl + 3.0 * sign, k * sign)
            specs = {"F": spec(0, 4.0 * fl, 24), "A": spec(20, y, 16), "C": spec(60, 4.0 * fl, 28)}

            def check(env, r, k=k, sign=sign):
                lat = r["F"].lane.local_coordinates(r["A"].position)[1]
                assert abs(lat) == 3.0 or (abs(lat) > 3.0) == (k > 0), (lat, k)
                assert neighbours(env, r["F"])[0] is (r["A"] if k <= 0 else r["C"])
                distinct_fronts("F", ["A", "C"])(env, r)
                return float(lat)
            out.append(Case("neighbours", f"lat{3 * sign:+d}", specs, ["F", "A", "C"], t=3.0 * sign, check=check,
                            fronts=("F", ["A", "C"])))
    # s = -5 (on_lane's -VEHICLE_LENGTH <= s) within a few ulp, at the start of the road
    for k in (-2, -1, 0, 1, 2):
        specs = {"F": spec(-30, 4, 20), "A": spec(nudge(-5.0, k), 4, 13), "C": spec(30, 4, 27)}

        def check(env, r, k=k):
            assert neighbours(env, r["F"])[0] is (r["A"] if k >= 0 else r["C"])
            distinct_fronts("F", ["A", "C"])(env, r)
            return float(r["F"].lane.local_coordinates(r["A"].position)[0])
        out.append(Case("neighbours", "s-5", specs, ["A", "F", "C"], anchored=True, t=-5.0, check=check,
                        fronts=("F", ["A", "C"])))
    return out


# ------------------------------------------------------------------ lane changes
def lane_change_cases(env0, lanes):
    out = []
    # a slow leader ahead of Q in lane 1, both side lanes free: MOBIL passes for both
    def blocked(q_over=None, lead_gap=25.0, lead_speed=15.0):
        s = {"Q": spec(0, 4, 25, target_speed=30, timer=2.0), "L": spec(lead_gap, 4, lead_speed)}
        if q_over:
            s["Q"].update(q_over)
        return s

    for t in (1.0, float(np.nextafter(1.0, 2.0))):
        out.append(Case("lane_change", "timer", blocked({"timer": t}), q=t, t=1.0, ulp=ulps(t, 1.0)))
    for sp in (1.0, float(np.nextafter(1.0, 0.0)), -1.0, float(np.nextafter(-1.0, 0.0))):
        s = blocked({"speed": sp}, lead_gap=12.0, lead_speed=0.0)

        def check(env, r):
            assert r["Q"].mobil(("0", "1", 2)) and r["Q"].mobil(("0", "1", 0))
        out.append(Case("lane_change", "speed", s, q=abs(sp), t=1.0, ulp=ulps(abs(sp), 1.0), check=check))
    for x in (0.0, float(np.nextafter(0.0, -1.0))):
        s = {"Q": spec(x, 4, 25, target_speed=30, timer=2.0), "L": spec(25, 4, 15)}
        out.append(Case("lane_change", "reachable_s0", s, anchored=True, q=x, t=0.0, ulp=-1 if x < 0 else 0))

    def both(env, r):
        assert r["Q"].mobil(("0", "1", 0)) and r["Q"].mobil(("0", "1", 2))
    out.append(Case("lane_change", "both_sides", blocked(), check=both))

    # MOBIL thresholds by bisection on the reference's own functions
    out += bisect_cases(env0)

    # abort of an ongoing change: Q (lane 0 -> 1) and O (lane 2 -> 1) at lane distance d
    env = env0
    for d in (0.0, 8.0):
        s = {"Q": spec(0, 0.8, 22, target_lane=1), "O": spec(d, 7.2, 20, target_lane=1)}
        out.append(Case("lane_change", "abort_d", s, ["Q", "O"], q=d, t=0.0, ulp=ulps(d, 0.0)))
        out.append(Case("lane_change", "abort_d", s, ["O", "Q"], q=d, t=0.0, ulp=ulps(d, 0.0)))
    # outside the faithful window: d* - 1e-6 / - 1e-8 (abort) and d* + 1e-8 / + 1e-6 (no abort), in metres
    for off in OFFSETS:
        out.append(Case("lane_change", "abort_dstar_out", {"Q": spec(0, 0.8, 22, target_lane=1),
                                                          "O": spec(0, 7.2, 20, target_lane=1)},
                        ["Q", "O"], window=True, check=("dstar", 0, off)))
    # d around d* = desired_gap(Q, O): O ahead of Q
    for k in (-2, -1, 0, 1, 2):
        out.append(Case("lane_change", "abort_dstar", {"Q": spec(0, 0.8, 22, target_lane=1),
                                                      "O": spec(0, 7.2, 20, target_lane=1)},
                        ["Q", "O"], window=True, ulp=k, check=("dstar", k, 0.0)))
    # list order: O (lane 0) has a slow leader and a free lane 1, its MOBIL sets target 1 in this act(); Q (lane 2 ->
    # 1) sees it when O is the earlier slot
    for order in (["O", "Q", "L"], ["Q", "O", "L"], ["L", "Q", "O"]):
        s = {"O": spec(12, 0, 24, target_speed=30, timer=2.0), "L": spec(32, 0, 12),
             "Q": spec(0, 7.2, 22, target_lane=1)}

        def check(env, r):
            assert r["O"].mobil(("0", "1", 1)) and r["O"].target_lane_index[2] == 0
            d = r["Q"].lane_distance_to(r["O"])
            assert 0 < d < r["Q"].desired_gap(r["Q"], r["O"])
        out.append(Case("lane_change", "abort_order", s, order, check=check))
    # the controlled vehicle (lane 0 -> 1) causes the abort of Q (lane 2 -> 1)
    out.append(Case("lane_change", "abort_by_ego", {"E": spec(10, 0.8, 25, target_lane=1),
                                                   "Q": spec(0, 7.2, 22, target_lane=1)}, ["E", "Q"]))
    return out


def bisect_double(f, lo, hi):
    """adjacent doubles (a, b) with f(a) != f(b), f monotone between lo and hi"""
    fa = f(lo)
    assert f(hi) != fa
    assert 0 <= lo < hi
    a, b = (int(x) for x in np.array([lo, hi]).view(np.int64))
    while b - a > 1:
        m = (a + b) // 2
        if f(float(np.int64(m).view(np.float64))) == fa:
            a = m
        else:
            b = m
    return float(np.int64(a).view(np.float64)), float(np.int64(b).view(np.float64))


def bisect_cases(env0):
    """jerk around LANE_CHANGE_MIN_ACC_GAIN (on the leader's gap) and new_following_pred_a around
    -LANE_CHANGE_MAX_BRAKING_IMPOSED (on the new follower's gap); the gap is solved on a scratch copy of the state"""
    out = []
    # jerk: Q in lane 0 (one side lane), leader L in lane 0 at gap g, lane 1 free
    for side, off in ((0, 0.0), (1, 0.0)) + tuple((int(o > 0), o) for o in OFFSETS):
        out.append(Case("lane_change", "jerk" if off == 0 else "jerk_out",
                        {"Q": spec(0, 0, 25, target_speed=30, timer=2.0), "L": spec(30, 0, 22)}, window=True,
                        check=("jerk", side, off)))
    # new_following_pred_a: Q in lane 0 behind a very slow leader, N in lane 1 behind Q at gap g, faster than Q
    for side, off in ((0, 0.0), (1, 0.0)) + tuple((int(o > 0), o) for o in OFFSETS):
        out.append(Case("lane_change", "pred_a" if off == 0 else "pred_a_out",
                        {"Q": spec(0, 0, 20, target_speed=30, timer=2.0), "L": spec(20, 0, 5), "N": spec(-20, 4, 28)},
                        window=True, check=("pred_a", side, off)))
    return out


def solve(env, case, r):
    """move the bisected vehicle of a threshold case onto its edge (off != 0: that many metres past it, on the side of
    the edge's double k); sets case.q / t / ulp"""
    what, k, off = case.check
    Q = r["Q"]
    if what == "dstar":
        O = r["O"]

        def d_minus(x):
            O.position[0] = x
            return Q.lane_distance_to(O) < Q.desired_gap(Q, O)
        d_star = Q.desired_gap(Q, O)
        a, b = bisect_double(d_minus, Q.position[0] + d_star - 1, Q.position[0] + d_star + 1)
        x = nudge(b, k) if off == 0 else (a if off < 0 else b) + off  # b: the first x with d >= d*
        O.position[0] = x
        case.q, case.t = float(Q.lane_distance_to(O)), float(Q.desired_gap(Q, O))
        case.ulp = ulps(case.q, case.t)
        return
    if what == "jerk":
        L = r["L"]

        def jerk(x):
            L.position[0] = x
            new_pre, _ = env.road.neighbour_vehicles(Q, ("0", "1", 1))
            old_pre, _ = env.road.neighbour_vehicles(Q)
            return Q.acceleration(Q, new_pre) - Q.acceleration(Q, old_pre)
        a, b = bisect_double(lambda x: jerk(x) < Q.LANE_CHANGE_MIN_ACC_GAIN, Q.position[0] + 6, Q.position[0] + 400)
        x = (b if k else a) + off  # a: the largest gap with jerk >= 0.2 (change), b: the next double (no change)
        case.q, case.t = float(jerk(x)), float(Q.LANE_CHANGE_MIN_ACC_GAIN)
        case.ulp = ulps(case.q, case.t)
        assert bool(Q.mobil(("0", "1", 1))) == (not k)
        return
    if what == "pred_a":
        N = r["N"]

        def pred(x):
            N.position[0] = x
            return Q.acceleration(N, Q)
        lim = -Q.LANE_CHANGE_MAX_BRAKING_IMPOSED
        a, b = bisect_double(lambda x: pred(x) < lim, Q.position[0] - 200, Q.position[0] - 6)
        x = (b if k else a) + off  # a: the smallest gap with pred_a >= -2 (change), b: the next double (refused)
        case.q, case.t = float(pred(x)), float(lim)
        case.ulp = ulps(case.q, case.t)
        assert bool(Q.mobil(("0", "1", 1))) == (not k)
        return
    raise ValueError(what)


# ------------------------------------------------------------------ collisions
def collision_cases(fast):
    """static pairs are crashed at speed 0 (they do not move, and only the impact tells will_intersect apart); in
    highway-fast-v0 only the controlled vehicle checks collisions, so every pair there involves it"""
    out = []
    E = "E"
    st = dict(speed=0.0, crashed=True)
    pairs = []
    for k in (-1, 0, 1, 2, 4):
        pairs.append(("dx5", spec(0, 4, **st), spec(5.0, 4, nudge=(0, k), **st), 5.0, k))
        pairs.append(("dy2", spec(0, 4, **st), spec(0.5, 6.0, nudge=(1, k), **st), 2.0, k))
    for gap in (1e-7, 1e-5):
        pairs.append(("sep_x", spec(0, 4, **st), spec(5.0 + gap, 4, **st), gap, 0))
    for gap, k in ((1e-7, 0), (1e-6, -2), (1e-6, 0), (1e-6, 2), (1e-5, 0)):
        pairs.append(("sep_y", spec(0, 4, **st), spec(1.0, 6.0 + gap, nudge=(1, k), **st), gap, k))
    pairs.append(("coincident", spec(0, 4, **st), spec(0, 4, **st), 0.0, 0))
    pairs.append(("coincident_rot", spec(0, 4, heading=0.3, **st), spec(0, 4, heading=-0.2, **st), 0.0, 0))
    pairs.append(("mirror", spec(0, 4, **st), spec(3.0, 5.0, **st), 0.0, 0))
    pairs.append(("mirror", spec(3.0, 5.0, **st), spec(0, 4, **st), 0.0, 0))
    for label, a, b, q, k in pairs:
        roles = {E if fast else "A": a, "B": b}
        out.append(Case("collisions", label, roles, list(roles), t=q, ulp=k, check=("static",)))
    # rotated pairs within +-0.78 rad: B moved along a direction onto the touching edge, then a few ulp either side
    for h_a, h_b, ang in ((0.5, -0.3, 0.2), (0.78, 0.1, 1.3), (-0.6, 0.6, -0.7)):
        for k in (-2, 0, 2):
            roles = {E if fast else "A": spec(0, 4, heading=h_a, **st), "B": spec(0, 4, heading=h_b, **st)}
            c = Case("collisions", "rotated", roles, list(roles), ulp=k, check=("rotated", ang, k))
            out.append(c)
    # several will_intersect partners below and above the middle slot (impact = the largest partner's)
    roles = {"P1": spec(-4.5, 4.4, **st), E if fast else "M": spec(0, 4, **st), "P2": spec(4.0, 3.5, **st),
             "P3": spec(0.5, 5.9, **st)}
    for order in (["P1", "M", "P2", "P3"], ["P2", "P3", "M", "P1"], ["P3", "M", "P1", "P2"]):
        o = [E if (x == "M" and fast) else x for x in order]
        out.append(Case("collisions", "multi_partner", dict(roles), o))
    # a gap the controlled vehicle's displacement closes (speed_control holds its speed: target_speed = speed)
    for k in (-2, 0, 2):
        roles = {"E": spec(0, 4, 15.0, target_speed=15.0), "B": spec(10, 4, **st)}
        out.append(Case("collisions", "displacement", roles, ["E", "B"], ulp=k, check=("displacement", k)))
    # the moving, uncrashed controlled vehicle touching a standing one after its move (touching intersects: crashed)
    # and one double further apart (only will_intersect: the impact)
    for k in (-1, 0, 1):
        roles = {"E": spec(0, 4, 15.0, target_speed=15.0), "B": spec(8, 4, **st)}
        out.append(Case("collisions", "touch_moving", roles, ["E", "B"], ulp=k, check=("touch_moving", k)))
    if not fast:
        # the rank-pruned sweep: a centre gap of 7 m (above diag = 5.39) closed by the controlled vehicle's
        # displacement; the fastest vehicle of the env is a third one
        roles = {"E": spec(0, 8, 40.0, target_speed=40.0), "B": spec(7.0 + 40.0 / 15, 8, **st),
                 "T": spec(200, 0, 42.0, target_speed=42.0)}
        out.append(Case("collisions", "pruned_bound", roles, ["E", "B", "T"]))
        roles = {"E": spec(0, 8, 25.0, target_speed=25.0), "B": spec(6.2 + 25.0 / 15, 8, **st),
                 "T": spec(200, 0, 40.0, target_speed=40.0)}
        out.append(Case("collisions", "pruned_bound", roles, ["E", "B", "T"]))
    return out


def solve_collision(env, case, r, dt):
    from highway_env import utils

    what = case.check[0]
    if what == "rotated":
        _, ang, k = case.check
        A = [v for n, v in r.items() if n != "B"][0]
        B = r["B"]
        c0 = A.position.copy()
        u = np.array([np.cos(ang), np.sin(ang)])

        def sep(t):
            B.position = c0 + t * u
            return not utils.are_polygons_intersecting(A.polygon(), B.polygon(), np.zeros(2), np.zeros(2))[0]
        a, b = bisect_double(sep, 0.0, 12.0)
        B.position = c0 + b * u
        B.position[0] = nudge(float(B.position[0]), k)
        case.q = float(b)
        return
    if what in ("displacement", "touch_moving"):
        # post-move positions: E moves by fl(speed * dt) (heading 0, no steering, no acceleration); B stands still
        _, k = case.check
        E, B = r["E"], r["B"]
        step = float(E.speed * dt)
        xe = float(E.position[0] + step)

        def will(xb):
            x_now = E.position[0]
            E.position[0] = xe  # the post-move polygon
            pa = E.polygon()
            E.position[0] = x_now
            B.position[0] = xb
            return utils.are_polygons_intersecting(pa, B.polygon(), E.velocity * dt, np.zeros(2))[
                1 if what == "displacement" else 0]
        lo, hi = (xe + 5.0, xe + 5.0 + 2 * step) if what == "displacement" else (xe + 4.0, xe + 6.0)
        a, b = bisect_double(lambda x: not will(x), lo, hi)  # a: the last x that (will) intersect, b: the next
        B.position[0] = nudge(a, k)
        case.q = float(B.position[0] - xe)
        case.t = float(a - xe)
        case.ulp = k
        return
    raise ValueError(what)


# ------------------------------------------------------------------ kinematics (frozen)
def kinematics_cases(env0, lanes):
    out = []
    fr = dict(speed=0.0, crashed=True)
    ex, ey = KIN_EGO
    # norm = 200 (PERCEPTION_DISTANCE, strict) within a few ulp: straight ahead (exact) and in a side lane
    for k in (-4, -2, -1, 0, 1, 2, 4):
        specs = {"E": spec(0, 0, **fr), "A": spec(nudge(ex + 200.0, k) - ex, 0, **fr),
                 "B": spec(0, 4.0, **fr), "C": spec(20, -4.0, **fr)}
        out.append(Case("kinematics", "norm200", specs, ["E", "C", "A", "B"], q=200.0, t=200.0, ulp=k,
                        check=("norm", k)))
    # d = -10 (-2 * LENGTH < d, strict) within a few ulp
    for k in (-2, -1, 0, 1, 2):
        specs = {"E": spec(0, 0, **fr), "A": spec(nudge(ex - 10.0, k) - ex, 0, **fr), "B": spec(30, 4.0, **fr)}
        out.append(Case("kinematics", "d-10", specs, ["E", "B", "A"], t=-10.0,
                        check=lambda env, r: float(r["E"].lane_distance_to(r["A"]))))
    # |d| ties: ahead / behind / side by side, three-way
    up = 4.0 if lanes > 2 else 0.0
    specs = {"E": spec(0, 0, **fr), "A": spec(15, 0, **fr), "B": spec(-15, 0, **fr), "C": spec(15, -4, **fr),
             "D": spec(-6, up, heading=0.4, **fr), "G": spec(6, -4, heading=-0.3, **fr), "H": spec(6, 0, **fr)}
    for order in (["E", "A", "B", "C", "D", "G", "H"], ["E", "H", "C", "B", "G", "A", "D"]):
        out.append(Case("kinematics", "ties", specs, order))
    # a tie group across the cutoff (vehicles_count - 1 = 4 rows): two nearer, then four at |d| = 30
    specs = {"E": spec(0, 0, **fr), "N1": spec(10, 0, **fr), "N2": spec(20, -4, **fr), "T1": spec(30, 0, **fr),
             "T2": spec(30, -4, **fr), "T3": spec(30, up, heading=0.2, **fr), "T4": spec(-30, 0, **fr)}
    for order in (["E", "T3", "T1", "N2", "T4", "T2", "N1"], ["E", "T2", "T4", "T3", "N1", "T1", "N2"]):
        out.append(Case("kinematics", "cutoff_ties", specs, order))
    # fewer candidates than rows, ranges exactly on +-1 (x [-30, 30], y [-8, 8]) and a lateral offset
    specs = {"E": spec(0, 0, **fr), "A": spec(30, 0, **fr), "B": spec(-30, 0.7, heading=0.5, **fr)}
    out.append(Case("kinematics", "few_and_ranges", specs, ["E", "B", "A"]))
    specs = {"E": spec(0, 0, **fr), "A": spec(12, -4, **fr), "B": spec(25, up, heading=-0.6, **fr)}
    out.append(Case("kinematics", "few_and_ranges", specs, ["E", "A", "B"]))
    return out


# ------------------------------------------------------------------ generation
def build_states(env_id, over, seed, kinds):
    """[(env, [Case]), ...]: each state a fresh reference reset with its cases crafted in"""
    env0 = rh.make_reference_env(env_id, over)
    env0.reset(seed=seed)
    lanes = int(env0.config["lanes_count"])
    fast = env_id == "highway-fast-v0"
    V = len(env0.road.vehicles)
    cases = []
    for kind in kinds:
        if kind == "neighbours":
            cases += neighbour_cases(lanes)
        elif kind == "lane_change":
            cases += lane_change_cases(env0, lanes)
        elif kind == "collisions":
            cases += collision_cases(fast)
        elif kind == "kinematics":
            cases += kinematics_cases(env0, lanes)
    states = []
    cur = None
    for c in cases:
        n = len(c.specs)
        uses_ego = any(r == "E" for r in c.specs)
        if n - (1 if uses_ego else 0) > V - 1:  # (the small file: the cases with more vehicles than it has)
            continue
        solo = c.kind == "kinematics" or uses_ego
        if (cur is None or solo or cur["solo"] or cur["free"] < n + (0 if uses_ego else 0)
                or cur["kind"] != c.kind or (c.anchored and cur["anchored"]) or len(cur["cases"]) >= MAX_GROUPS):
            cur = {"cases": [], "free": V - 1, "solo": solo, "kind": c.kind, "anchored": False}
            states.append(cur)
        assert n - (1 if uses_ego else 0) <= cur["free"], (c.label, n, V)
        cur["cases"].append(c)
        cur["free"] -= n - (1 if uses_ego else 0)
        cur["anchored"] |= c.anchored
    out = []
    dt = 1.0 / env0.config["simulation_frequency"]
    for s in states:
        env = rh.make_reference_env(env_id, over)
        env.reset(seed=seed)
        vs = list(env.road.vehicles)
        frozen = s["kind"] == "kinematics"
        free = list(range(1, V))
        roles_all = []
        g = 0
        for c in s["cases"]:
            if c.kind == "kinematics":
                x0 = KIN_EGO[0]
            elif c.anchored:
                x0 = 0.0
            else:
                g += 1
                x0 = 100.0 + GROUP_SPACING * g
            r = {}
            for role in c.order:
                v = vs[0] if role == "E" else vs[free.pop(0)]
                sp = dict(c.specs[role])
                if c.kind == "kinematics":
                    sp["y"] = KIN_EGO[1] + sp["y"]
                place(env, v, sp, x0)
                r[role] = v
            roles_all.append((c, r))
        if not any(r for c, r in roles_all if "E" in r):
            park(env, vs[0], 0, frozen)
        for k, slot in enumerate(free):
            park(env, vs[slot], k + 1, frozen)
        # MOBIL's jerk reads the vehicles ahead in the side lane, which the other solved cases may move: it goes last
        for c, r in sorted(roles_all, key=lambda cr: isinstance(cr[0].check, tuple) and cr[0].check[0] == "jerk"):
            if isinstance(c.check, tuple):
                if c.check[0] in ("dstar", "jerk", "pred_a"):
                    solve(env, c, r)
                elif c.check[0] == "static":
                    A, B = (r[role] for role in c.order[:2])
                    c.q = float(B.position[0] - A.position[0]) if c.label in ("dx5", "sep_x") else (
                        float(B.position[1] - A.position[1]) if c.label in ("dy2", "sep_y") else np.nan)
                elif c.check[0] in ("rotated", "displacement", "touch_moving"):
                    solve_collision(env, c, r, dt)
                elif c.check[0] == "norm":
                    A, E = r["A"], r["E"]
                    # side-lane vehicle B at norm 200 within the same k: x from the reference's own norm
                    k = c.check[1]
                    B = r["B"]
                    a, b = bisect_double(lambda x: np.linalg.norm(np.array([x, B.position[1]]) - E.position) < 200.0,
                                         E.position[0] + 150.0, E.position[0] + 201.0)
                    B.position[0] = nudge(b, k)  # b: the first x with norm >= 200
                    c.q = float(np.linalg.norm(A.position - E.position))
                    c.ulp = ulps(c.q, c.t)
            elif c.check is not None:
                q = c.check(env, r)
                if q is not None:
                    c.q, c.ulp = q, ulps(q, c.t)
            for v in r.values():  # lane_index of a moved vehicle, target lane kept
                v.lane_index = lane_of(env, v.position[0], v.position[1], v.heading)
                v.lane = env.road.network.get_lane(v.lane_index)
        out.append((env, roles_all, frozen))
    return out, dt


def run_substep(env, dt):
    env.road.act()
    env.road.step(dt)


def generate(name, env_id, over, seed, kinds):
    from highway_env.envs.common.observation import observation_factory

    states, dt = build_states(env_id, over, seed, kinds)
    before, after, obs = [], [], [[] for _ in OBS_CFGS]
    rows = {k: [] for k in ("case_state", "case_kind", "case_label", "case_q", "case_t", "case_ulp", "case_window",
                            "case_slots", "case_fronts")}
    corners = []
    for si, (env, roles_all, frozen) in enumerate(states):
        d0 = rh.dump_state(env)
        before.append(d0)
        vs = list(env.road.vehicles)
        for c, r in roles_all:
            slots = np.full(8, -1, dtype=np.int32)
            for j, role in enumerate(c.order):
                slots[j] = vs.index(r[role])
            rows["case_state"].append(si)
            rows["case_kind"].append(c.kind)
            rows["case_label"].append(c.label)
            rows["case_q"].append(float(c.q))
            rows["case_t"].append(float(c.t))
            rows["case_ulp"].append(int(c.ulp))
            rows["case_window"].append(bool(c.window))
            rows["case_slots"].append(slots)
            # (follower slot, its front's slot, the follower's speed after the substep behind that front and behind
            # the other candidate): IDMVehicle.act's clipped acceleration, then Vehicle.step's speed += a * dt
            fr = np.array([-1, -1, np.nan, np.nan])
            if c.fronts:
                f = r[c.fronts[0]]
                front = env.road.neighbour_vehicles(f)[0]
                cands = [r[x] for x in c.fronts[1]]
                assert front in cands and f.target_lane_index == f.lane_index and f.timer <= f.LANE_CHANGE_DELAY
                alt = [v for v in cands if v is not front][0]
                fr = np.array([vs.index(f), vs.index(front), f.speed + clipped_accel(f, front) * dt,
                               f.speed + clipped_accel(f, alt) * dt])
                assert fr[2] != fr[3], (c.label, fr)
            rows["case_fronts"].append(fr)
            if c.kind == "collisions":
                corners.append(np.stack([np.asarray(r[role].polygon()[:4]) for role in c.order[:2]]))
        for k, cfg in enumerate(OBS_CFGS):
            obs[k].append(np.asarray(observation_factory(env, dict(cfg)).observe(), dtype=np.float32).copy())
        if frozen:
            twin = copy.deepcopy(env)
            twin.step(1)  # IDLE: a whole policy step of the frozen world
            d1 = rh.dump_state(twin)
            for key in ("x", "y", "heading", "speed", "lane", "target_lane", "crashed"):
                assert np.array_equal(d0[key], d1[key]), (name, si, key)
            assert np.all(np.isnan(d1["impact"])), (name, si)
            o1 = np.asarray(observation_factory(twin, dict(OBS_CFGS[0])).observe(), dtype=np.float32)
            assert np.array_equal(o1, obs[0][-1]), (name, si)
        run_substep(env, dt)
        after.append(rh.dump_state(env))
    out = {k: np.stack([s[k] for s in before]) for k in before[0]}
    out.update({"after_" + k: np.stack([s[k] for s in after]) for k in after[0]})
    for k in range(len(OBS_CFGS)):
        out[f"obs_{k}"] = np.stack(obs[k])
    out["case_state"] = np.array(rows["case_state"], dtype=np.int32)
    out["case_kind"] = np.array(rows["case_kind"])
    out["case_label"] = np.array(rows["case_label"])
    out["case_q"] = np.array(rows["case_q"], dtype=np.float64)
    out["case_t"] = np.array(rows["case_t"], dtype=np.float64)
    out["case_ulp"] = np.array(rows["case_ulp"], dtype=np.int64)
    out["case_window"] = np.array(rows["case_window"], dtype=np.bool_)
    out["case_slots"] = np.stack(rows["case_slots"])
    out["case_fronts"] = np.stack(rows["case_fronts"]).astype(np.float64)
    out["frozen"] = np.array([f for _, _, f in states], dtype=np.bool_)
    if corners:
        out["collision_corners"] = np.stack(corners)
    env = rh.make_reference_env(env_id, over)
    env.reset(seed=seed)
    cfg = dict(env.config)
    cfg["_env_id"] = env_id
    out["config_json"] = np.array(json.dumps(cfg))
    out["obs_cfgs_json"] = np.array(json.dumps(OBS_CFGS))
    out["numpy_version"] = np.array(np.__version__)
    path = os.path.join(OUT, name + ".npz")
    with open(path, "wb") as f:  # np.savez_compressed stamps the zip members with the time: write them fixed
        _savez_fixed(f, out)
    print(f"{name}: {len(before)} states, {len(rows['case_state'])} cases -> {path} ({os.path.getsize(path)/1e3:.0f} kB)")


def _savez_fixed(f, arrays):
    """np.savez_compressed with a fixed member timestamp, so that regenerating gives byte-identical files"""
    import io
    import zipfile

    with zipfile.ZipFile(f, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k, a in arrays.items():
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(a), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


if __name__ == "__main__":
    if not rh.reference_available():
        raise SystemExit("reference not mounted; golden fixtures can only be generated in the build container")
    rh._ensure_imports()
    only = sys.argv[1:]
    for name, case in FILES.items():
        if not only or name in only:
            generate(name, *case)
