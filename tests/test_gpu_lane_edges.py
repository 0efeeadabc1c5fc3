"""The network kernels' lane geometry, closest-lane pruning and neighbour pre-test at their edges, on the crafted points
of tests/golden/lane_edges_*.npz (oracle/gen_lane_edges.py), through the library's test entries
hwy_debug_network_lanes / hwy_debug_network_closest_lanes / hwy_debug_network_neighbours:

  geometry     lane_local / lane_position / lane_heading_at / lane_distance_with_heading bit for bit on straight lanes,
               within a stated ulp bound of 60-digit mpmath on sine and circular lanes (run with -s for the maxima)
  soundness    lane_maybe_on false => lane_local + lane_on(margin=1) false; closest_lane_prunable(L, p, bd) true =>
               the device's |lat| + max(s - length, 0) + max(-s, 0) > bd, bd driven through that bound, its
               neighbouring doubles, +-2^-20 relative and 0, with a fresh circle cache and with one carried over the
               table as closest_lane_group scans it.  No exceptions: this holds whatever atan2 / sin round to.
  closest lane closest_lane_group on 257 envs per table and thread mapping (vp 8 and 32) with right, adjacent and far
               starting lanes equals the first minimum of the device's own distance_with_heading over all lanes, bit
               for bit, with the candidate list overflowing into the in-place path; and the fixture's
               get_closest_lane_index outside the faithful window of its two smallest distances
  neighbours   the neighbour search on the fixture scenes equals an unfiltered restatement of neighbour_vehicles on the
               device's own lane_local, and the fixture outside faithful windows

Reads only the fixtures."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from test_lane_edges_spec import FAMILIES, KINDS, load, scales, window

pytestmark = pytest.mark.gpu

ULP_BOUND = 8  # ulp of the lane's scale (test_lane_edges_spec.scales) on sine and circular lanes
K_CAND = {8: 40, 32: 48}  # closest_lane_group's shared candidate list (hwy_network.cu kCand)


def N():
    from highwayenv_b200 import _native

    return _native


def graph_struct(d):
    n = N()
    g = n.HwyNetGraph()
    g.n_lanes, g.n_nodes = len(d["net_type"]), len(d["net_succ_count"])
    for k in range(g.n_lanes):
        for f in n.NET_LANE_INT_FIELDS:
            if "net_" + f in d:
                setattr(g.lanes[k], f, int(d["net_" + f][k]))
        for f in n.NET_LANE_F64_FIELDS:
            setattr(g.lanes[k], f, float(d["net_" + f][k]))
    for node in range(g.n_nodes):
        g.succ_count[node] = int(d["net_succ_count"][node])
        for j in range(n.HWY_NET_MAX_SUCC):
            g.succ[node][j] = int(d["net_succ"][node][j])
    return g


def lanes_op(g, op, rows):
    """hwy_debug_network_lanes on rows [n][<= HWY_LANES_IN]"""
    n = N()
    code, width = n.LANE_OPS[op]
    a = np.zeros((len(rows), n.HWY_LANES_IN))
    a[:, :rows.shape[1]] = rows
    d_in = torch.from_numpy(a).cuda()
    d_out = torch.full((len(rows), width), -7.0, dtype=torch.float64, device="cuda")
    n.check(n.load().hwy_debug_network_lanes(C.byref(g), code, d_in.data_ptr(), d_out.data_ptr(), len(rows), None))
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()
    return out[:, 0] if width == 1 else out


def all_pairs(d):
    """(point, lane) rows over every point and every lane of the table"""
    n_l = len(d["net_type"])
    P = len(d["x"])
    lane = np.tile(np.arange(n_l), P)
    pt = np.repeat(np.arange(P), n_l)
    return pt, lane


def lower_bound(d, lane, s, lat):
    """the device's |lat| + max(s - length, 0) + max(-s, 0), summed in the kernels' order"""
    length = d["net_length"][lane]
    return (np.abs(lat) + np.maximum(s - length, 0.0)) + np.maximum(0.0 - s, 0.0)


# ------------------------------------------------------------------ geometry
def exact_local(L, x, y):
    import mpmath

    m = lambda v: mpmath.mpf(float(v))  # noqa: E731
    x, y = m(x), m(y)
    if int(L["type"]) == 2:
        wx, wy = x - m(L["cx"]), y - m(L["cy"])
        sp = m(L["start_phase"])
        dphi = mpmath.atan2(wy, wx) - sp
        dphi = dphi - 2 * mpmath.pi * mpmath.floor((dphi + mpmath.pi) / (2 * mpmath.pi))
        return m(L["direction"]) * dphi * m(L["radius"]), m(L["direction"]) * (m(L["radius"]) - mpmath.sqrt(wx * wx + wy * wy))
    ddx, ddy = x - m(L["sx"]), y - m(L["sy"])
    lon, lat = ddx * m(L["dx"]) + ddy * m(L["dy"]), ddx * m(L["lx"]) + ddy * m(L["ly"])
    if int(L["type"]) == 1:
        lat = lat - m(L["amplitude"]) * mpmath.sin(m(L["pulsation"]) * lon + m(L["phase"]))
    return lon, lat


def exact_heading(L, s):
    import mpmath

    m = lambda v: mpmath.mpf(float(v))  # noqa: E731
    if int(L["type"]) == 2:
        return m(L["direction"]) * m(s) / m(L["radius"]) + m(L["start_phase"]) + mpmath.pi / 2 * m(L["direction"])
    return m(L["heading"]) + mpmath.atan(m(L["amplitude"]) * m(L["pulsation"]) *
                                         mpmath.cos(m(L["pulsation"]) * m(s) + m(L["phase"])))


def exact_position(L, s, lat):
    import mpmath

    m = lambda v: mpmath.mpf(float(v))  # noqa: E731
    if int(L["type"]) == 2:
        phi = m(L["direction"]) * m(s) / m(L["radius"]) + m(L["start_phase"])
        rr = m(L["radius"]) - m(lat) * m(L["direction"])
        return m(L["cx"]) + rr * mpmath.cos(phi), m(L["cy"]) + rr * mpmath.sin(phi)
    lat = m(lat) + m(L["amplitude"]) * mpmath.sin(m(L["pulsation"]) * m(s) + m(L["phase"]))
    return m(L["sx"]) + m(s) * m(L["dx"]) + lat * m(L["lx"]), m(L["sy"]) + m(s) * m(L["dy"]) + lat * m(L["ly"])


@pytest.mark.parametrize("family", FAMILIES)
def test_lane_geometry(family):
    import mpmath

    d = load(family)
    g = graph_struct(d)
    lane = d["lane"].astype(np.float64)
    loc = lanes_op(g, "local", np.stack([lane, d["x"], d["y"]], 1))
    pos = lanes_op(g, "position", np.stack([lane, d["s"], d["lat"]], 1))
    hd = lanes_op(g, "heading_at", np.stack([lane, d["s"]], 1))
    dwh = lanes_op(g, "distance_with_heading", np.stack([lane, d["x"], d["y"], d["h"]], 1))
    assert np.array_equal(dwh[:, 1:], loc), family  # distance_with_heading's own local coordinates
    types = d["net_type"][d["lane"]]
    st = types == 0
    assert np.array_equal(loc[st, 0], d["s"][st]) and np.array_equal(loc[st, 1], d["lat"][st]), family
    assert np.array_equal(pos[st, 0], d["px"][st]) and np.array_equal(pos[st, 1], d["py"][st]), family
    assert np.array_equal(hd[st], d["heading_at"][st]) and np.array_equal(dwh[st, 0], d["d"][st]), family
    # no transcendental function on the path: the straight part of a sine lane's lateral is not separable, but its
    # longitudinal is, and the arc's heading_at is arithmetic only
    sine = types == 1
    assert np.array_equal(loc[sine, 0], d["s"][sine]), family
    s_scale, lat_scale = scales(d)
    worst = {"s": 0.0, "lat": 0.0, "x": 0.0, "y": 0.0, "heading": 0.0}
    flips = 0
    names = {k: d["net_" + k] for k in ("type", "cx", "cy", "radius", "start_phase", "direction", "sx", "sy", "dx",
                                        "dy", "lx", "ly", "amplitude", "pulsation", "phase", "heading")}
    m = mpmath.mpf
    with mpmath.workdps(60):
        for i in np.nonzero(~st)[0]:
            l = int(d["lane"][i])
            L = {k: v[l] for k, v in names.items()}
            es, elat = exact_local(L, d["x"][i], d["y"][i])
            err = abs(loc[i, 0] - es)
            if types[i] == 2 and abs(abs(es) - mpmath.pi * m(L["radius"])) <= 1e-9 * m(L["radius"]):
                # phi - start_phase = +-pi: an atan2 an ulp apart gives the other end of the wrap, s -+ 2 pi radius
                alt = abs(loc[i, 0] - (es - mpmath.sign(es) * 2 * mpmath.pi * m(L["radius"])))
                flips += alt < err
                err = min(err, alt)
            worst["s"] = max(worst["s"], float(err) / np.spacing(max(s_scale[l], abs(loc[i, 0]))))
            worst["lat"] = max(worst["lat"], float(abs(loc[i, 1] - elat)) / np.spacing(max(lat_scale[l], abs(loc[i, 1]))))
            ex, ey = exact_position(L, d["s"][i], d["lat"][i])
            xy_scale = max(abs(float(ex)), abs(float(ey)), lat_scale[l] + abs(float(L["cx"])) + abs(float(L["cy"])))
            worst["x"] = max(worst["x"], float(abs(pos[i, 0] - ex)) / np.spacing(xy_scale))
            worst["y"] = max(worst["y"], float(abs(pos[i, 1] - ey)) / np.spacing(xy_scale))
            eh = exact_heading(L, d["s"][i])
            worst["heading"] = max(worst["heading"], float(abs(hd[i] - eh)) / np.spacing(max(abs(float(eh)), 1.0)))
    print(family, "worst ulp on sine / circular lanes", {k: round(v, 2) for k, v in worst.items()},
          f"phase-wrap flips {flips}")
    assert max(worst.values()) <= ULP_BOUND, (family, worst)


# ------------------------------------------------------------------ soundness of the two pre-tests
@pytest.mark.parametrize("family", FAMILIES)
def test_maybe_on_is_sound(family):
    d = load(family)
    g = graph_struct(d)
    pt, lane = all_pairs(d)
    rows = np.stack([lane.astype(np.float64), d["x"][pt], d["y"][pt]], 1)
    on = lanes_op(g, "on", rows)
    maybe = lanes_op(g, "maybe_on", rows)
    bad = np.nonzero((maybe == 0) & (on == 1))[0]
    assert len(bad) == 0, (family, [(int(pt[b]), int(lane[b])) for b in bad[:10]])
    # and on_lane(margin=1) itself against the reference's, on straight lanes (exact there)
    ref_on = (d["on_mask"][pt] >> lane) & 1
    straight = d["net_type"][lane] == 0
    assert np.array_equal(on[straight], ref_on[straight].astype(np.float64)), family
    print(family, f"{len(rows)} (point, lane) pairs: on {int(on.sum())}, maybe_on {int(maybe.sum())}")


@pytest.mark.parametrize("family", FAMILIES)
def test_closest_lane_pruning_is_sound(family):
    d = load(family)
    g = graph_struct(d)
    pt, lane = all_pairs(d)
    loc = lanes_op(g, "local", np.stack([lane.astype(np.float64), d["x"][pt], d["y"][pt]], 1))
    lb = lower_bound(d, lane, loc[:, 0], loc[:, 1])
    bds = [lb, np.nextafter(lb, -np.inf), np.nextafter(lb, np.inf), lb * (1 - 2.0 ** -20), lb * (1 + 2.0 ** -20),
           np.zeros_like(lb)]
    pruned_total = 0
    for bd in bds:
        pr = lanes_op(g, "prunable", np.stack([lane.astype(np.float64), d["x"][pt], d["y"][pt], bd], 1))
        bad = np.nonzero((pr == 1) & ~(lb > bd))[0]
        assert len(bad) == 0, (family, [(int(pt[b]), int(lane[b]), float(lb[b]), float(bd[b])) for b in bad[:5]])
        pruned_total += int(pr.sum())
    # the carried circle cache, as closest_lane_group scans the table: hint = the crafted lane, bd through the bound of
    # another lane of the table and the hint's own distance_with_heading
    n_l = len(d["net_type"])
    lbm = lb.reshape(-1, n_l)
    P = len(d["x"])
    rng = np.random.default_rng(7)
    other = rng.integers(n_l, size=P)
    own = lanes_op(g, "distance_with_heading", np.stack([d["lane"].astype(np.float64), d["x"], d["y"], d["h"]], 1))[:, 0]
    base = lbm[np.arange(P), other]
    for bd in (base, np.nextafter(base, -np.inf), np.nextafter(base, np.inf), own, base * (1 + 2.0 ** -20)):
        scan = lanes_op(g, "prunable_scan", np.stack([d["lane"].astype(np.float64), d["x"], d["y"], bd], 1))[:, :n_l]
        bad = np.nonzero((scan == 1) & ~(lbm > bd[:, None]))
        assert len(bad[0]) == 0, (family, list(zip(bad[0][:5].tolist(), bad[1][:5].tolist())))
        assert not scan[np.arange(P), d["lane"]].any()
    print(family, f"pruning sound on {len(lb) * len(bds)} (point, lane, bd) triples, {pruned_total} pruned")


# ------------------------------------------------------------------ closest_lane_group
def net_state(n_envs, vp, x, y, h, lanes, count):
    n = N()
    dev = "cuda"
    z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=dev)  # noqa: E731
    t = {k: z(n_envs, vp, 2, dtype=torch.float64) for k in ("pos", "hs", "tt", "imp")}
    t["pos"][:, :, 0], t["pos"][:, :, 1] = torch.from_numpy(x).to(dev), torch.from_numpy(y).to(dev)
    t["hs"][:, :, 0], t["hs"][:, :, 1] = torch.from_numpy(h).to(dev), 10.0
    m = (lanes.astype(np.int64) << n.META_LANE_SHIFT) | (lanes.astype(np.int64) << n.META_TARGET_SHIFT) | n.META_PRESENT
    t["meta"] = torch.from_numpy(m.astype(np.int32)).to(dev)
    t["delta"] = z(n_envs, vp, dtype=torch.float64)
    t["route"], t["route_len"] = z(n_envs, vp, n.HWY_NET_MAX_ROUTE, dtype=torch.int32), z(n_envs, vp, dtype=torch.int32)
    t["speed_index"], t["time"] = z(n_envs, dtype=torch.int32), z(n_envs, dtype=torch.float64)
    t["count"] = torch.from_numpy(np.asarray(count, dtype=np.int32)).to(dev)
    t["road_steps"] = z(n_envs, dtype=torch.int32)
    st = n.HwyNetState()
    st.n_envs, st.vp = n_envs, vp
    for k in ("pos", "hs", "tt", "imp", "delta", "meta", "route", "route_len", "speed_index", "time", "count",
              "road_steps"):
        setattr(st, k, t[k].data_ptr())
    p = n.HwyNetParams()
    p.n_vehicles, p.simulation_frequency, p.policy_frequency, p.n_target_speeds = vp, 15, 1, 3
    p.obs_vehicles_count, p.obs_features = 5, 5
    return p, st, t


def device_graph(g):
    return torch.from_numpy(np.frombuffer(bytes(g), dtype=np.uint8).copy()).cuda()


@pytest.mark.parametrize("vp", [8, 32])
@pytest.mark.parametrize("family", FAMILIES)
def test_closest_lane_group(family, vp):
    n = N()
    d = load(family)
    g = graph_struct(d)
    n_l, P = len(d["net_type"]), len(d["x"])
    n_envs = 257  # a partial last block on both mappings
    rng = np.random.default_rng(vp * 1000 + len(family))
    pick = rng.integers(P, size=(n_envs, vp))
    x, y, h = d["x"][pick], d["y"][pick], d["h"][pick]
    flat = pick.reshape(-1)
    # every lane's distance_with_heading on the device: the exact argmin (first minimum) and the hints
    pt = np.repeat(flat, n_l)
    lane = np.tile(np.arange(n_l), len(flat))
    dwh = lanes_op(g, "distance_with_heading", np.stack([lane.astype(np.float64), d["x"][pt], d["y"][pt], d["h"][pt]],
                                                        1)).reshape(len(flat), n_l, 3)
    best = np.argmin(dwh[:, :, 0], axis=1)
    # starting lanes: right, adjacent (next in the table, the same road or the successor's), far (largest distance)
    mode = rng.integers(3, size=len(flat))
    hint = np.where(mode == 0, best, np.where(mode == 1, (best + 1) % n_l, np.argmax(dwh[:, :, 0], axis=1)))
    count = np.full(n_envs, vp)
    count[::5] = rng.integers(1, vp + 1, size=len(count[::5]))  # some envs with fewer vehicles
    p, st, t = net_state(n_envs, vp, x, y, h, hint.reshape(n_envs, vp), count)
    out_lane = torch.full((n_envs, vp), -9, dtype=torch.int32, device="cuda")
    out_s, out_lat = (torch.zeros(n_envs, vp, dtype=torch.float64, device="cuda") for _ in range(2))
    dg = device_graph(g)
    n.check(n.load().hwy_debug_network_closest_lanes(C.byref(p), dg.data_ptr(), C.byref(st), out_lane.data_ptr(),
                                                     out_s.data_ptr(), out_lat.data_ptr(), None))
    torch.cuda.synchronize()
    got, gs, glat = (a.cpu().numpy().reshape(-1) for a in (out_lane, out_s, out_lat))
    present = (np.arange(vp)[None, :] < count[:, None]).reshape(-1)
    assert (got[~present] == -1).all()
    k = np.nonzero(present)[0]
    assert np.array_equal(got[k], best[k]), (family, vp, np.nonzero(got[k] != best[k])[0][:10])
    assert np.array_equal(gs[k], dwh[k, best[k], 1]) and np.array_equal(glat[k], dwh[k, best[k], 2]), (family, vp)
    # the candidate list: (vehicle, lane) pairs that survive the pruning, per env, as the group scans them
    bd = dwh[np.arange(len(flat)), hint, 0]
    scan = lanes_op(g, "prunable_scan", np.stack([hint.astype(np.float64), d["x"][flat], d["y"][flat], bd], 1))[:, :n_l]
    survivors = (n_l - 1 - scan.sum(axis=1)) * present
    per_env = survivors.reshape(n_envs, vp).sum(axis=1)
    overflow = int((per_env > K_CAND[vp]).sum())
    # the reference's own closest lane, outside the faithful window of its two smallest distances
    in_window = window(d)[flat]
    diff = np.nonzero((got != d["closest"][flat]) & present)[0]
    assert in_window[diff].all(), (family, vp, diff[~in_window[diff]][:10])
    print(family, f"vp {vp}: {len(k)} vehicles, envs past the {K_CAND[vp]}-slot candidate list {overflow} of {n_envs} "
          f"(max {int(per_env.max())} candidates); differences from the reference {len(diff)}, all among "
          f"{int((in_window & present).sum())} in the faithful window")
    if (n_l - 1) * vp >= 2 * K_CAND[vp]:  # tables with room for twice the list
        assert overflow > 0, (family, vp, int(per_env.max()))


# ------------------------------------------------------------------ neighbours
def restated_neighbours(d, loc, lanes_v, V, connected):
    """Road.neighbour_vehicles(v) of every vehicle (road/road.py:483-547) on the device's lane_local of every vehicle
    on every lane, loc [V][n_lanes][2], in the reference's list order with its tie rules"""
    n_l = len(d["net_type"])
    from_node, to_node, lane_id = d["net_from_node"], d["net_to_node"], d["net_lane_id"]
    road_first, road_count = d["net_road_first"], d["net_road_count"]
    width, length = d["net_width"], d["net_length"]
    front, rear = np.full(V, -1), np.full(V, -1)
    for veh in range(V):
        L = int(lanes_v[veh])
        s = loc[veh, L, 0]
        search = [(L, 0.0)]
        if connected:
            for k in range(int(d["net_succ_count"][to_node[L]])):
                f = int(d["net_succ"][to_node[L], k])
                search.append((f + (lane_id[L] if lane_id[L] < road_count[f] else 0), length[L]))
            for l0 in range(n_l):
                if lane_id[l0] == 0 and to_node[l0] == from_node[L]:
                    pl = l0 + (lane_id[L] if lane_id[L] < road_count[l0] else 0)
                    search.append((pl, -length[pl]))
        s_front = s_rear = None
        for v in range(V):
            if v == veh:
                continue
            for sl, off in search:
                s_v, lat_v = loc[v, sl]
                if not (abs(lat_v) <= width[sl] / 2 + 1 and -5.0 <= s_v < length[sl] + 5.0):
                    continue
                s_v = s_v + off
                if s <= s_v and (s_front is None or s_v <= s_front):
                    s_front, front[veh] = s_v, v
                if s_v < s and (s_rear is None or s_v > s_rear):
                    s_rear, rear[veh] = s_v, v
                break
    return front, rear


def scene_window(d, loc, V):
    """a scene whose neighbours a few ulp of atan2 / sin could change: some vehicle's lane_local on a sine or circular
    lane within a few thousand ulp of on_lane's edges, or two vehicles' s on such a lane that close together"""
    s_scale, lat_scale = scales(d)
    curved = d["net_type"] != 0
    tol_s, tol_lat = 2.0 ** -40 * (1 + s_scale), 2.0 ** -40 * (1 + lat_scale)
    s, lat = loc[..., 0], loc[..., 1]
    edge = ((np.abs(np.abs(lat) - (d["net_width"] / 2 + 1)) <= tol_lat) | (np.abs(s + 5) <= tol_s) |
            (np.abs(s - d["net_length"] - 5) <= tol_s) | (np.abs(s - d["net_length"]) <= tol_s) | (np.abs(s) <= tol_s))
    if (edge & curved).any():
        return True
    for l in np.nonzero(curved)[0]:
        ss = np.sort(s[:, l])
        if (np.diff(ss) <= tol_s[l]).any() and (np.diff(ss) > 0).any():
            return True
    return False


@pytest.mark.parametrize("vp", [8, 32])
@pytest.mark.parametrize("family", FAMILIES)
def test_neighbours(family, vp):
    n = N()
    d = load(family)
    g = graph_struct(d)
    dg = device_graph(g)
    n_l = len(d["net_type"])
    mismatch, windows, scenes = 0, 0, 0
    for V in (8, 32):
        if V > vp:
            continue
        xs, ys, hs, ls = (d[f"scene{V}_{k}"] for k in ("x", "y", "h", "lane"))
        S = len(xs)
        pad = lambda a, fill: np.concatenate([a, np.full((S, vp - V), fill, dtype=a.dtype)], 1)  # noqa: E731
        x, y, h, lanes = pad(xs, 0.0), pad(ys, 0.0), pad(hs, 0.0), pad(ls, 0)
        loc = lanes_op(g, "local", np.stack([np.tile(np.arange(n_l), S * V).astype(np.float64),
                                             np.repeat(xs.reshape(-1), n_l), np.repeat(ys.reshape(-1), n_l)], 1))
        loc = loc.reshape(S, V, n_l, 2)
        for conn in (0, 1):
            p, st, t = net_state(S, vp, x, y, h, lanes, np.full(S, V))
            p.n_vehicles = V
            p.connected_lanes = conn
            front, rear = (torch.full((S, vp), -9, dtype=torch.int32, device="cuda") for _ in range(2))
            n.check(n.load().hwy_debug_network_neighbours(C.byref(p), dg.data_ptr(), C.byref(st), None,
                                                          front.data_ptr(), rear.data_ptr(), None))
            torch.cuda.synchronize()
            f, r = front.cpu().numpy()[:, :V], rear.cpu().numpy()[:, :V]
            for sc in range(S):
                rf, rr = restated_neighbours(d, loc[sc], ls[sc], V, conn)
                assert np.array_equal(f[sc], rf) and np.array_equal(r[sc], rr), (family, vp, V, conn, sc)
                scenes += 1
                win = scene_window(d, loc[sc], V)
                windows += win
                ok = np.array_equal(f[sc], d[f"scene{V}_front"][conn, sc]) and np.array_equal(
                    r[sc], d[f"scene{V}_rear"][conn, sc])
                if not ok:
                    mismatch += 1
                    assert win, (family, vp, V, conn, sc)
    print(family, f"vp {vp}: {scenes} scene searches equal the restatement; {mismatch} differ from the reference, "
          f"all among {windows} in a faithful window")
