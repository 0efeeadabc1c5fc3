"""The lane edge fixtures (tests/golden/lane_edges_*.npz, oracle/gen_lane_edges.py) on the CPU: the crafted points
really sit within their stated number of ulp of their edges (60-digit mpmath), the host lane table's geometry
(NetworkTable, used by the roundabout and intersection host resets) equals the reference bit for bit, and the C
oracle's lane functions and closest-lane search equal it except where numpy's and the C library's arctan2 / sin may
round differently (a faithful window of a few ulp)."""
import math

import numpy as np
import pytest

FAMILIES = ("roundabout", "intersection", "racetrack", "merge", "u_turn", "two_way", "exit", "lane_keeping")
KINDS = ("lat", "lon", "sine_gate", "sine_peak", "radius", "cross_s", "cross_e", "end_reach", "wrap", "centre")
LENGTH = 5.0


def load(family):
    from parity_utils import load_golden

    return load_golden(f"lane_edges_{family}")


def table(d):
    """a NetworkTable whose lanes are the fixture's (the reference's attributes, bit for bit)"""
    from highwayenv_b200 import _native as N
    from highwayenv_b200.road.network import NetworkTable

    net = NetworkTable()
    n = len(d["net_type"])
    net.lanes = [{k: (int(d["net_" + k][l]) if k in N.NET_LANE_INT_FIELDS else float(d["net_" + k][l]))
                  for k in N.NET_LANE_INT_FIELDS + N.NET_LANE_F64_FIELDS if "net_" + k in d} for l in range(n)]
    return net


def quantity(kind, L, ends, x, y):
    import mpmath

    m = lambda v: mpmath.mpf(float(v))  # noqa: E731
    x, y = m(x), m(y)
    if L["type"] == 2:
        wx, wy = x - m(L["cx"]), y - m(L["cy"])
        (sx, sy), (ex, ey) = ((m(a), m(b)) for a, b in ends)
        return {"radius": lambda: mpmath.sqrt(wx * wx + wy * wy),
                "cross_s": lambda: m(L["direction"]) * ((sx - m(L["cx"])) * wy - (sy - m(L["cy"])) * wx),
                "cross_e": lambda: m(L["direction"]) * (wx * (ey - m(L["cy"])) - wy * (ex - m(L["cx"]))),
                "end_reach": lambda: min(mpmath.sqrt((x - sx) ** 2 + (y - sy) ** 2),
                                         mpmath.sqrt((x - ex) ** 2 + (y - ey) ** 2)),
                "wrap": lambda: -mpmath.cos(m(L["start_phase"])) * wy + mpmath.sin(m(L["start_phase"])) * wx}[kind]()
    ddx, ddy = x - m(L["sx"]), y - m(L["sy"])
    lon, lat = ddx * m(L["dx"]) + ddy * m(L["dy"]), ddx * m(L["lx"]) + ddy * m(L["ly"])
    return {"lat": lat, "lon": lon, "sine_gate": abs(lat) - abs(m(L["amplitude"])),
            "sine_peak": m(L["pulsation"]) * lon + m(L["phase"])}[kind]


def threshold(kind, L, t):
    """the exact threshold of a stored (double) one: pi / 2 multiples and the squared-slack radii are irrational"""
    import mpmath

    if kind == "sine_peak":
        return round(float(t) / (math.pi / 2)) * mpmath.pi / 2
    if kind == "radius":
        gate = L["width"] / 2 + 1.0
        for a, b in ((L["radius"] + gate, 1 + 1e-12), (L["radius"] - gate, 1 - 1e-12)):
            exact = mpmath.mpf(a) * mpmath.sqrt(mpmath.mpf(b))
            if float(exact) == float(t) and float(t) not in (a, ):
                return exact
    return mpmath.mpf(float(t))


def arc_ends(net, l):
    L = net.lanes[l]
    if L["type"] != 2:
        return None
    return tuple((float(a[0]), float(b[0])) for a, b in (net.position(l, [0.0], [0.0]),
                                                          net.position(l, [L["length"]], [0.0])))


def sign(v):
    return 0 if v == 0 else (1 if v > 0 else -1)


@pytest.mark.parametrize("family", FAMILIES)
def test_fixture_points_sit_on_their_edges(family):
    """every stored point is base moved by k ulp along its axis, the edge lies between base and the next float (60-digit
    mpmath), and the point is on the side its label says"""
    import mpmath

    d = load(family)
    net = table(d)
    ends = {l: arc_ends(net, l) for l in range(len(net.lanes))}
    checked_bases = {}
    counts = dict.fromkeys(KINDS, 0)
    with mpmath.workdps(60):
        for i in range(len(d["x"])):
            kind, l, axis, k = KINDS[int(d["kind"][i])], int(d["lane"][i]), int(d["axis"][i]), int(d["k"][i])
            p = [float(d["x"][i]), float(d["y"][i])]
            b = float(d["base"][i])
            moved = b
            for _ in range(abs(k)):
                moved = float(np.nextafter(moved, np.inf if k > 0 else -np.inf))
            assert p[axis] == moved, (family, i)
            if kind == "centre":
                assert b == net.lanes[l]["cx"] and p[1] == net.lanes[l]["cy"]
                continue
            L = net.lanes[l]
            T = threshold(kind, L, d["threshold"][i])
            side = sign(quantity(kind, L, ends[l], p[0], p[1]) - T)
            assert side == int(d["side"][i]), (family, i, kind)
            key = (l, kind, float(d["threshold"][i]), b, p[1 - axis])
            if key not in checked_bases:
                q0, q1 = list(p), list(p)
                q0[axis], q1[axis] = b, float(np.nextafter(b, np.inf))
                s0 = sign(quantity(kind, L, ends[l], *q0) - T)
                s1 = sign(quantity(kind, L, ends[l], *q1) - T)
                assert s0 != s1 or s0 == 0, (family, i, kind)
                checked_bases[key] = True
                counts[kind] += 1
    print(family, "edges per kind", {k: v for k, v in counts.items() if v})
    assert counts["lat"] and counts["lon"]


def scales(d):
    """the magnitudes the rounding of a lane's s and lateral scale with: on an arc (|start_phase| + pi) * radius and the
    radius (atan2's and sqrt's operands); on a sine lane the length and the amplitude"""
    arc = d["net_type"] == 2
    s_scale = np.where(arc, (np.abs(d["net_start_phase"]) + np.pi) * d["net_radius"], d["net_length"])
    lat_scale = np.where(arc, d["net_radius"], np.abs(d["net_amplitude"]) + d["net_width"])
    return s_scale, lat_scale


def window(d):
    """closest-lane faithful window: the reference's two smallest distance_with_heading within a bound of the
    rounding of their circular / sine terms (s = phi * radius and the angle: a few thousand ulp of radius * pi), and the
    points where an arc's phase wraps"""
    r_max = float(np.max(np.abs(d["net_radius"]))) if len(d["net_radius"]) else 0.0
    tol = 2.0 ** -40 * (1.0 + np.abs(d["d1"]) + 4 * r_max)
    return ((d["d2"] - d["d1"]) <= tol) | wrap_window(d)


def wrap_window(d):
    """points on the ray opposite an arc's start (phi - start_phase within 1e-9 of +-pi): an arctan2 an ulp apart puts
    s at either end of the wrap, +-pi * radius, and so changes that arc's distance by 2 pi radius"""
    near = np.zeros(len(d["x"]), dtype=bool)
    for l in np.nonzero(d["net_type"] == 2)[0]:
        phi = np.arctan2(d["y"] - d["net_cy"][l], d["x"] - d["net_cx"][l])
        w = ((phi - d["net_start_phase"][l]) + np.pi) % (2 * np.pi) - np.pi
        near |= np.abs(np.abs(w) - np.pi) <= 1e-9
    return near


@pytest.mark.parametrize("family", FAMILIES)
def test_host_table_geometry_equals_reference(family):
    """NetworkTable.local_coordinates / position / heading_at on the crafted lane and closest_lane over the table,
    bit for bit (numpy on both sides; local_coordinates rounds its dot products and norm as np.dot does)"""
    d = load(family)
    net = table(d)
    lanes = d["lane"]
    for l in np.unique(lanes):
        sel = lanes == l
        s, lat = net.local_coordinates(int(l), d["x"][sel], d["y"][sel])
        assert np.array_equal(s, d["s"][sel]) and np.array_equal(lat, d["lat"][sel]), (family, int(l))
        px, py = net.position(int(l), d["s"][sel], d["lat"][sel])
        assert np.array_equal(px, d["px"][sel]) and np.array_equal(py, d["py"][sel]), (family, int(l))
        assert np.array_equal(net.heading_at(int(l), d["s"][sel]), d["heading_at"][sel]), (family, int(l))
    got = net.closest_lane(d["x"], d["y"], d["h"])
    assert np.array_equal(got, d["closest"]), (family, np.nonzero(got != d["closest"])[0][:10])


@pytest.mark.parametrize("family", FAMILIES)
def test_c_oracle_lanes_equal_reference(family):
    """the C oracle's lane functions (libm's atan2 / sin / atan) and net_closest_lane: bit for bit on straight lanes,
    within 4 ulp of the reference elsewhere, and the same closest lane outside the faithful window"""
    import ctypes as C

    import net_oracle as no

    d = load(family)
    g = no.graph_from_arrays(d)
    lib = no.lib()
    s_, lat_ = C.c_double(), C.c_double()
    worst = 0.0
    s_scale, lat_scale = scales(d)
    flips = 0
    for i in range(len(d["x"])):
        l = int(d["lane"][i])
        L = g.lanes[l]
        lib.net_lane_local(C.byref(L), float(d["x"][i]), float(d["y"][i]), C.byref(s_), C.byref(lat_))
        if int(d["net_type"][l]) == 0:
            assert (s_.value, lat_.value) == (d["s"][i], d["lat"][i]), (family, i)
        else:
            for got, want, scale in ((s_.value, d["s"][i], s_scale[l]), (lat_.value, d["lat"][i], lat_scale[l])):
                if KINDS[int(d["kind"][i])] == "wrap" and got == -want:  # phi - start_phase = +-pi: either end
                    flips += 1
                    continue
                err = abs(got - want) / np.spacing(max(scale, abs(want)))
                worst = max(worst, err)
                assert err <= 4, (family, i, got, want)
    in_window = window(d)
    diff = 0
    for i in range(len(d["x"])):
        got = lib.net_closest_lane(C.byref(g), float(d["x"][i]), float(d["y"][i]), float(d["h"][i]))
        if got != d["closest"][i]:
            diff += 1
            assert in_window[i], (family, i, got, int(d["closest"][i]))
    print(family, f"oracle worst {worst:.1f} ulp, {flips} phase-wrap flips at +-pi; closest-lane differences {diff}, all in the "
          f"{int(in_window.sum())} window points; arctan2 numpy != libm on {int(d['arctan2_libm_disagree'])} of "
          f"{int(d['arctan2_args'])} (numpy {d['numpy_version']})")


def test_fixtures_cover_the_tables():
    """one file per lane table the product ships, with the lane kinds the issue names, under 2 MB in all"""
    import os

    from parity_utils import GOLDEN

    total = 0
    for family in FAMILIES:
        d = load(family)
        total += os.path.getsize(os.path.join(GOLDEN, f"lane_edges_{family}.npz"))
        kinds = {KINDS[k] for k in np.unique(d["kind"])}
        types = set(np.unique(d["net_type"]).tolist())
        assert {"lat", "lon"} <= kinds
        if 1 in types:
            assert {"sine_gate", "sine_peak"} <= kinds, family
        if 2 in types:
            assert {"radius", "cross_s", "cross_e", "end_reach", "wrap", "centre"} <= kinds, family
        assert set(np.unique(d["lane"]).tolist()) == set(range(len(d["net_type"]))), family
        assert d["scene8_front"].shape[0] == 2 and d["scene32_front"].shape[0] == 2
    n_lanes = {f: len(load(f)["net_type"]) for f in ("roundabout", "intersection", "racetrack")}
    assert n_lanes == {"roundabout": 32, "intersection": 20, "racetrack": 18}
    assert total < 2.2e6, total
