"""Generate the lane edge fixtures tests/golden/lane_edges_<family>.npz from the UNMODIFIED reference (build container
only).

    python oracle/gen_lane_edges.py [family ...]

The network kernels skip most lanes of the closest-lane search and of the neighbour search with lower bounds that
need no sqrt, atan2 or sin (hwy_lanes.cuh closest_lane_prunable, lane_maybe_on).  Rollouts almost never put a vehicle
within a few ulp of the edges those bounds and the lane functions decide on.  Here every lane of each table the product
ships gets crafted points on both sides of each such edge.  An edge is a real quantity q(x, y) of the lane and a
threshold T; its crossing is found by bisection on the float grid of one coordinate (`axis`), 60-digit mpmath deciding
the side: `base` is the last float before q - T changes sign, and the stored points are base moved by k = 0, +-1, +-2,
+-4 ulp along the axis, each with its side sign(q - T) (0: exactly on the edge).

  straight / sine   straight lateral at +-width/2 (the boundary with the adjacent lane) and +-(width/2 + 1) (on_lane's
                    margin, lane_maybe_on's gate); longitudinal at -LENGTH, 0, length, length + LENGTH (the end point is
                    the junction with the successors; lateral 0 or a random offset)
  sine              |straight lateral| - |amplitude| = gate, and pulsation * s + phase at pi/2 + k pi (|sin| = 1)
  circular          r = radius +- width/2, radius +- gate, the squared-slack boundaries r^2 = (radius +- gate)^2 (1 +- 1e-12),
                    r halfway to every concentric arc (ties between two arcs); the radial lines through both end points
                    (cross product 0 and +-1e-6); distance gate + LENGTH + 1e-6 to the nearer end point outside the
                    sector; phi - start_phase = +-pi (the ray opposite the start, where the phase wrap switches); the
                    centre itself (kind `centre`, no bisection)
  heading           most edges' first point gets the heading heading_at(s) +- pi moved by k ulp (the wrap of the
                    angle term); the others a heading near the lane's

Stored per point: x, y, heading, the crafted lane, kind, threshold, axis, k, side, base; the reference's
local_coordinates, position(s, lat), heading_at(s) and distance_with_heading on the crafted lane, on_lane(margin=1) of
every lane (bit mask), get_closest_lane_index, and the two smallest distance_with_heading values over the table (the
faithful window of a closest-lane tie).  Neighbour scenes: 8- and 32-vehicle scenes of crafted points around one lane
(drawn with replacement: exact position ties), each vehicle's lane from the reference's Vehicle constructor, and
Road.neighbour_vehicles(v) of every vehicle with neighbour_vehicles_connected_lanes False and True.  The file also
records numpy's version and how many of the stored arctan2 arguments numpy and math.atan2 round differently.
"""
from __future__ import annotations

import math
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import ref_harness as rh  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
NUDGES = (-4, -2, -1, 0, 1, 2, 4)
LENGTH = 5.0  # AbstractLane.VEHICLE_LENGTH
KINDS = ("lat", "lon", "sine_gate", "sine_peak", "radius", "cross_s", "cross_e", "end_reach", "wrap", "centre")
SCENES = {8: 24, 32: 8}
FAMILIES = ("roundabout", "intersection", "racetrack", "merge", "u_turn", "two_way", "exit", "lane_keeping")
ENV_IDS = {"roundabout": "roundabout-v0", "intersection": "intersection-v0", "merge": "merge-v0",
           "u_turn": "u-turn-v0", "two_way": "two-way-v0", "exit": "exit-v0"}
DPS = 60


def make_env(family):
    rh._ensure_imports()
    if family == "racetrack":
        from highway_env.envs.racetrack_env import RacetrackEnv

        env = RacetrackEnv()
    elif family == "lane_keeping":
        from highway_env.envs.lane_keeping_env import LaneKeepingEnv

        env = LaneKeepingEnv()
    else:
        env = rh.make_reference_env(ENV_IDS[family])
    env.reset(seed=0)
    return env


def nudge(x: float, k: int) -> float:
    for _ in range(abs(k)):
        x = float(np.nextafter(x, np.inf if k > 0 else -np.inf))
    return x


def lane_params(lane):
    """the lane's attributes as exact mpmath numbers"""
    import mpmath
    from highway_env.road.lane import CircularLane, SineLane

    m = mpmath.mpf
    if isinstance(lane, CircularLane):
        return dict(type=2, cx=m(float(lane.center[0])), cy=m(float(lane.center[1])), radius=m(float(lane.radius)),
                    sp=m(float(lane.start_phase)), direction=m(float(lane.direction)))
    p = dict(type=1 if isinstance(lane, SineLane) else 0, sx=m(float(lane.start[0])), sy=m(float(lane.start[1])),
             dx=m(float(lane.direction[0])), dy=m(float(lane.direction[1])), lx=m(float(lane.direction_lateral[0])),
             ly=m(float(lane.direction_lateral[1])))
    if isinstance(lane, SineLane):
        p.update(amp=m(float(lane.amplitude)), w=m(float(lane.pulsation)), ph=m(float(lane.phase)))
    return p


def quantity(kind, P, ends, x, y):
    """q(x, y) of an edge kind, exact in 60-digit mpmath (x, y, the lane's attributes and `ends` are doubles)"""
    import mpmath

    x, y = mpmath.mpf(float(x)), mpmath.mpf(float(y))
    if P["type"] == 2:
        wx, wy = x - P["cx"], y - P["cy"]
        if kind == "radius":
            return mpmath.sqrt(wx * wx + wy * wy)
        (sx, sy), (ex, ey) = ends
        if kind == "cross_s":
            return P["direction"] * ((sx - P["cx"]) * wy - (sy - P["cy"]) * wx)
        if kind == "cross_e":
            return P["direction"] * (wx * (ey - P["cy"]) - wy * (ex - P["cx"]))
        if kind == "end_reach":
            return min(mpmath.sqrt((x - sx) ** 2 + (y - sy) ** 2), mpmath.sqrt((x - ex) ** 2 + (y - ey) ** 2))
        if kind == "wrap":  # cross product with the ray at start_phase + pi
            return -mpmath.cos(P["sp"]) * wy + mpmath.sin(P["sp"]) * wx
        raise ValueError(kind)
    ddx, ddy = x - P["sx"], y - P["sy"]
    lon, lat = ddx * P["dx"] + ddy * P["dy"], ddx * P["lx"] + ddy * P["ly"]
    if kind == "lat":
        return lat
    if kind == "lon":
        return lon
    if kind == "sine_gate":
        return abs(lat) - abs(P["amp"])
    if kind == "sine_peak":
        return P["w"] * lon + P["ph"]
    raise ValueError(kind)


def threshold_value(T):
    import mpmath

    if isinstance(T, tuple):  # ("pi", a, b): a * pi / 2 + b;  ("sqrt", a, b): a * sqrt(b)
        if T[0] == "pi":
            return T[1] * mpmath.pi / 2 + T[2]
        return mpmath.mpf(T[1]) * mpmath.sqrt(mpmath.mpf(T[2]))
    return mpmath.mpf(T)


def side(kind, P, ends, T, x, y) -> int:
    import mpmath

    with mpmath.workdps(DPS):
        d = quantity(kind, P, ends, x, y) - threshold_value(T)
        return 0 if d == 0 else (1 if d > 0 else -1)


def crossing(kind, P, ends, T, p0, axis):
    """the last float b of coordinate `axis` (the other coordinate fixed) before q - T changes sign, searching around
    p0; None when no change of sign is found nearby"""
    p = [float(p0[0]), float(p0[1])]

    def s_at(v):
        q = list(p)
        q[axis] = v
        return side(kind, P, ends, T, q[0], q[1])

    c = p[axis]
    for rel in (1e-12, 1e-9, 1e-6, 1e-3):
        delta = rel * max(1.0, abs(c))
        lo, hi = c - delta, c + delta
        slo, shi = s_at(lo), s_at(hi)
        if slo != shi and slo != 0 and shi != 0:
            break
    else:
        return None
    while float(np.nextafter(lo, hi)) != hi:
        mid = lo + (hi - lo) / 2
        if mid in (lo, hi):
            break
        sm = s_at(mid)
        if sm == slo:
            lo = mid
        else:
            hi = mid
    return lo


def lane_edges(lane, lanes, rng):
    """(kind, threshold, point near the edge, axis) of every crafted edge of one lane"""
    from highway_env.road.lane import CircularLane, SineLane

    w = float(lane.width)
    gate = w / 2 + 1.0
    out = []

    def axis_of(gx, gy):
        return 0 if abs(gx) >= abs(gy) else 1

    if isinstance(lane, CircularLane):
        c, R = np.array(lane.center, dtype=np.float64), float(lane.radius)
        mid_phase = (lane.start_phase + lane.end_phase) / 2
        radii = [R + w / 2, R - w / 2, R + gate, R - gate, ("sqrt", R + gate, 1 + 1e-12)]
        if R - gate > 0:
            radii.append(("sqrt", R - gate, 1 - 1e-12))
        for other in lanes:
            if other is not lane and isinstance(other, CircularLane) and np.array_equal(other.center, lane.center):
                radii.append((R + float(other.radius)) / 2)
        for T in radii:
            r = float(threshold_value(T)) if isinstance(T, tuple) else T
            if r <= 0:
                continue
            ph = mid_phase + float(rng.uniform(-0.3, 0.3))
            p = c + r * np.array([math.cos(ph), math.sin(ph)])
            out.append(("radius", T, p, axis_of(math.cos(ph), math.sin(ph))))
        for kind, ph in (("cross_s", lane.start_phase), ("cross_e", lane.end_phase)):
            for T in (0.0, 1e-6, -1e-6):
                r = R + float(rng.uniform(-gate, gate))
                p = c + r * np.array([math.cos(ph), math.sin(ph)])
                out.append((kind, T, p, axis_of(-math.sin(ph), math.cos(ph))))
        reach = gate + LENGTH + 1e-6
        for end_phase, sgn in ((lane.start_phase, -1), (lane.end_phase, 1)):
            e = c + R * np.array([math.cos(end_phase), math.sin(end_phase)])
            tang = lane.direction * sgn * np.array([-math.sin(end_phase), math.cos(end_phase)])
            p = e + reach * tang  # beyond the end, outside the sector
            out.append(("end_reach", reach, p, axis_of(*tang)))
        ph = lane.start_phase + math.pi
        p = c + R * np.array([math.cos(ph), math.sin(ph)])
        out.append(("wrap", 0.0, p, axis_of(-math.sin(ph), math.cos(ph))))
        return out
    L = float(lane.length)
    d, lat_dir = np.array(lane.direction), np.array(lane.direction_lateral)
    start = np.array(lane.start, dtype=np.float64)
    for T in (w / 2, -w / 2, gate, -gate):
        s = float(rng.uniform(0, L))
        out.append(("lat", T, start + s * d + T * lat_dir, axis_of(*lat_dir)))
    for T in (-LENGTH, 0.0, L, L + LENGTH):
        lat = 0.0 if rng.random() < 0.5 else float(rng.uniform(-w / 2, w / 2))
        out.append(("lon", T, start + T * d + lat * lat_dir, axis_of(*d)))
    if isinstance(lane, SineLane):
        A = abs(float(lane.amplitude))
        for T in (gate, ):
            for sgn in (1, -1):
                s = float(rng.uniform(0, L))
                out.append(("sine_gate", T, start + s * d + sgn * (A + T) * lat_dir, axis_of(*lat_dir)))
        om, ph = float(lane.pulsation), float(lane.phase)
        for k in range(0, 8):  # pi/2 + k pi within the lane
            s = ((2 * k + 1) * math.pi / 2 - ph) / om
            if 0 <= s <= L:
                lat = float(rng.uniform(-gate, gate))
                out.append(("sine_peak", ("pi", 2 * k + 1, 0.0), start + s * d + lat * lat_dir, axis_of(*d)))
    return out


def generate(family):
    rh._ensure_imports()
    from highway_env.road.lane import CircularLane
    from highway_env.road.road import Road
    from highway_env.vehicle.kinematics import Vehicle

    env = make_env(family)
    net = env.road.network
    lanes = [lane for _, lane in rh.lane_list(env)]
    idx = {li: k for k, (li, _) in enumerate(rh.lane_list(env))}
    rng = np.random.default_rng(sum(map(ord, family)))
    rec = {k: [] for k in ("x", "y", "h", "lane", "kind", "threshold", "axis", "k", "side", "base", "heading_kind")}
    ends_of = {}
    for li, lane in enumerate(lanes):
        ends = None
        if isinstance(lane, CircularLane):
            ends = (tuple(float(v) for v in lane.position(0, 0)), tuple(float(v) for v in lane.position(lane.length, 0)))
        ends_of[li] = ends
        P = lane_params(lane)
        for kind, T, p0, axis in lane_edges(lane, lanes, rng):
            b = crossing(kind, P, ends, T, p0, axis)
            if b is None:
                raise RuntimeError(f"{family} lane {li}: no crossing for {kind} {T}")
            for j, k in enumerate(NUDGES):
                q = [float(p0[0]), float(p0[1])]
                q[axis] = nudge(b, k)
                s_ref = float(lane.local_coordinates(np.array(q))[0])
                hk = 0
                if j == 0 and rng.random() < 0.7:  # heading_at(s) +- pi, moved by a few ulp
                    hk = int(rng.choice([-1, 1]))
                    h = nudge(float(lane.heading_at(s_ref)) + hk * math.pi, int(rng.choice(NUDGES)))
                else:
                    h = float(lane.heading_at(s_ref)) + float(rng.normal(0, 0.2))
                for key, v in (("x", q[0]), ("y", q[1]), ("h", h), ("lane", li), ("kind", KINDS.index(kind)),
                               ("threshold", float(threshold_value(T))), ("axis", axis), ("k", k),
                               ("side", side(kind, P, ends, T, q[0], q[1])), ("base", b), ("heading_kind", hk)):
                    rec[key].append(v)
        if isinstance(lane, CircularLane):  # the centre
            for k in NUDGES:
                q = [nudge(float(lane.center[0]), k), float(lane.center[1])]
                for key, v in (("x", q[0]), ("y", q[1]), ("h", float(rng.uniform(-np.pi, np.pi))), ("lane", li),
                               ("kind", KINDS.index("centre")), ("threshold", 0.0), ("axis", 0), ("k", k),
                               ("side", 1 if k else 0), ("base", float(lane.center[0])), ("heading_kind", 0)):
                    rec[key].append(v)
    out = {k: np.array(v) for k, v in rec.items()}
    for k in ("lane", "kind", "axis", "k", "side", "heading_kind"):
        out[k] = out[k].astype(np.int32)
    n = len(out["x"])
    s_own, lat_own, d_own, px, py, hd = (np.zeros(n) for _ in range(6))
    on_mask = np.zeros(n, dtype=np.int64)
    closest, d1, d2 = np.zeros(n, dtype=np.int32), np.zeros(n), np.zeros(n)
    atan_args = []
    for i in range(n):
        pos = np.array([out["x"][i], out["y"][i]])
        h = float(out["h"][i])
        lane = lanes[out["lane"][i]]
        s, lat = lane.local_coordinates(pos)
        s_own[i], lat_own[i] = s, lat
        d_own[i] = lane.distance_with_heading(pos, h)
        px[i], py[i] = lane.position(s, lat)
        hd[i] = lane.heading_at(s)
        ds = []
        for l2, L2 in enumerate(lanes):
            s2, lat2 = L2.local_coordinates(pos)
            if L2.on_lane(pos, s2, lat2, margin=1):
                on_mask[i] |= 1 << l2
            ds.append(L2.distance_with_heading(pos, h))
            if isinstance(L2, CircularLane):
                atan_args.append((pos[1] - L2.center[1], pos[0] - L2.center[0]))
        closest[i] = idx[net.get_closest_lane_index(pos, h)]
        srt = sorted(ds)
        d1[i], d2[i] = srt[0], srt[1] if len(srt) > 1 else np.inf
    out.update(s=s_own, lat=lat_own, d=d_own, px=px, py=py, heading_at=hd, on_mask=on_mask, closest=closest,
               d1=d1, d2=d2)
    # neighbour scenes
    succ = {}
    for l1, (li, _) in enumerate(rh.lane_list(env)):
        succ[l1] = [l2 for l2, (lj, _) in enumerate(rh.lane_list(env))
                    if lj[0] == li[1] or lj[1] == li[0] or lj[:2] == li[:2]]
    for V, count in SCENES.items():
        sx, sy, sh, slane, sfront = (np.zeros((count, V)) for _ in range(5))
        fronts, rears = np.full((2, count, V), -1, dtype=np.int32), np.full((2, count, V), -1, dtype=np.int32)
        for sc in range(count):
            L0 = int(rng.integers(len(lanes)))
            pool = np.nonzero(np.isin(out["lane"], succ[L0]))[0]
            pick = rng.choice(pool, size=V, replace=True)
            for conn in (0, 1):
                road = Road(network=net, vehicles=[], np_random=np.random.RandomState(0),
                            neighbour_vehicles_connected_lanes=bool(conn))
                vs = [Vehicle(road, np.array([out["x"][p], out["y"][p]]), float(out["h"][p]), 10.0) for p in pick]
                road.vehicles = vs
                for j, v in enumerate(vs):
                    f, r = road.neighbour_vehicles(v)
                    fronts[conn, sc, j] = -1 if f is None else vs.index(f)
                    rears[conn, sc, j] = -1 if r is None else vs.index(r)
                    if conn == 0:
                        sx[sc, j], sy[sc, j], sh[sc, j] = v.position[0], v.position[1], v.heading
                        slane[sc, j] = idx[v.lane_index]
        out[f"scene{V}_x"], out[f"scene{V}_y"], out[f"scene{V}_h"] = sx, sy, sh
        out[f"scene{V}_lane"] = slane.astype(np.int32)
        out[f"scene{V}_front"], out[f"scene{V}_rear"] = fronts, rears
    out.update(rh.dump_network(env))
    out["numpy_version"] = np.array(np.__version__)
    out["arctan2_libm_disagree"] = np.int64(sum(float(np.arctan2(y, x)) != math.atan2(y, x) for y, x in atan_args))
    out["arctan2_args"] = np.int64(len(atan_args))
    path = os.path.join(OUT, f"lane_edges_{family}.npz")
    np.savez_compressed(path, **out)
    print(f"lane_edges_{family}: {len(lanes)} lanes, {n} points, arctan2 numpy != libm on "
          f"{int(out['arctan2_libm_disagree'])} of {len(atan_args)} -> {path} ({os.path.getsize(path) / 1e3:.0f} kB)")


if __name__ == "__main__":
    if not rh.reference_available():
        raise SystemExit("reference not mounted; golden fixtures can only be generated in the build container")
    import mpmath

    mpmath.mp.dps = DPS
    for fam in sys.argv[1:] or FAMILIES:
        generate(fam)
