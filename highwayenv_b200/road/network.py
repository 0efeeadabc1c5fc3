"""Road network tables for the device kernels.

Host-side counterpart of the reference's ``RoadNetwork`` (highway_env/road/road.py:21-389) and
lane classes (highway_env/road/lane.py:159-384).  The reference keeps ``graph[from][to] -> list
of lane objects`` keyed by node NAMES and walks it with Python dict iteration; the kernels need
integer tables.  ``NetworkTable`` records lanes in insertion order, numbers nodes, and emits
the lanes in *graph enumeration order* (from-node first-insertion order, then to-node insertion
order, then lane id — the order ``get_closest_lane_index`` scans, road.py:65-71) together with
per-node successor lists (``graph[node].keys()`` order, used by ``next_lane``, road.py:119-128).

Lane parameters are computed with the same numpy expressions as the lane constructors
(``StraightLane.__init__`` lane.py:183-194, ``CircularLane.__init__`` :314-336) so that the
tables are bit-identical to the reference's attributes (checked against a dump of the
reference's network in tests/test_host_cpu.py).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from .. import _native as N

LaneIndex = Tuple[str, str, int]


def _two_sum(a, b):
    """s + e == a + b exactly (Knuth)"""
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _two_prod(a, b):
    """h + l == a * b exactly (Dekker, Veltkamp splitting)"""
    def split(x):
        c = 134217729.0 * x  # 2^27 + 1
        hi = c - (c - x)
        return hi, x - hi

    h = a * b
    ah, al = split(a)
    bh, bl = split(b)
    return h, ((ah * bh - h) + ah * bl + al * bh) + al * bl


def dot2(a0, a1, b0, b1):
    """np.dot([a0, a1], [b0, b1]) element-wise: numpy's 2-vector dot is one fma, fma(a1, b1, a0 * b0) (pinned by
    tests/test_rng_craft.py).  The exact value h + l + p is summed with error-free transformations; the few elements
    whose rounding the fast sum cannot settle (within 2^-40 of a rounding boundary, or a power-of-two result) are
    rounded by math.fsum."""
    a0, a1, b0, b1 = (np.asarray(v, dtype=np.float64) for v in (a0, a1, b0, b1))
    p = a0 * b0
    h, l = _two_prod(a1, b1)
    s, e = _two_sum(h, p)
    t, f = _two_sum(e, l)
    r, g = _two_sum(s, t)
    z = g + f  # the exact value is r + g + f
    with np.errstate(invalid="ignore", over="ignore"):
        hard = ~(np.abs(z) < np.spacing(np.abs(r)) * (0.5 - 2.0 ** -40)) | (np.abs(np.frexp(r)[0]) == 0.5)
    hard &= np.isfinite(h) & np.isfinite(p)
    if hard.any():
        r = np.array(r, dtype=np.float64, copy=True)
        hb, lb, pb = np.broadcast_arrays(h, l, p)
        for k in zip(*np.nonzero(hard)):
            r[k] = math.fsum((float(hb[k]), float(lb[k]), float(pb[k])))
    return r


class NetworkTable:
    def __init__(self) -> None:
        self._graph: Dict[str, Dict[str, List[dict]]] = {}

    # ------------------------------------------------------------------ construction
    def _add(self, _from: str, _to: str, lane: dict) -> None:
        self._graph.setdefault(_from, {}).setdefault(_to, []).append(lane)

    def add_straight(self, _from: str, _to: str, start, end, width: float = 4.0, forbidden: bool = False,
                     speed_limit: float = 20.0, priority: int = 0, sine: Optional[Tuple[float, float, float]] = None) -> None:
        """StraightLane (lane.py:159-213) or, with sine=(amplitude, pulsation, phase), SineLane (:236-289)."""
        start, end = np.array(start, dtype=np.float64), np.array(end, dtype=np.float64)
        heading = np.arctan2(end[1] - start[1], end[0] - start[0])
        length = np.linalg.norm(end - start)
        direction = (end - start) / length
        lane = dict(type=N.LANE_SINE if sine else N.LANE_STRAIGHT, width=width, speed_limit=speed_limit,
                    length=float(length), sx=start[0], sy=start[1], ex=end[0], ey=end[1], dx=direction[0],
                    dy=direction[1], lx=-direction[1], ly=direction[0], heading=float(heading),
                    forbidden=int(forbidden), priority=int(priority))
        if sine:
            lane.update(amplitude=float(sine[0]), pulsation=float(sine[1]), phase=float(sine[2]))
        self._add(_from, _to, lane)

    def add_circular(self, _from: str, _to: str, center, radius: float, start_phase: float, end_phase: float,
                     clockwise: bool = True, width: float = 4.0, forbidden: bool = False,
                     speed_limit: float = 20.0, priority: int = 0) -> None:
        """CircularLane (lane.py:311-358)."""
        direction = 1 if clockwise else -1
        lane = dict(type=N.LANE_CIRCULAR, width=width, speed_limit=speed_limit,
                    length=float(radius * (end_phase - start_phase) * direction), cx=float(center[0]),
                    cy=float(center[1]), radius=float(radius), start_phase=float(start_phase),
                    end_phase=float(end_phase), direction=float(direction), forbidden=int(forbidden),
                    priority=int(priority))
        self._add(_from, _to, lane)

    # ------------------------------------------------------------------ (de)serialisation
    _CLASS_PATHS = {N.LANE_STRAIGHT: "highway_env.road.lane.StraightLane", N.LANE_SINE: "highway_env.road.lane.SineLane",
                    N.LANE_CIRCULAR: "highway_env.road.lane.CircularLane"}

    def to_config(self) -> dict:
        """RoadNetwork.to_config (road/road.py:379-389) with AbstractLane.to_config of each lane class
        (road/lane.py:221-233, 296-309, 369-384): {from: {to: [{"class_path", "config"}, ...]}} in insertion order.
        `line_types` (a rendering attribute) is emitted only when the lane was given one."""
        out: dict = {}
        for f, tos in self._graph.items():
            out[f] = {}
            for t, lanes in tos.items():
                out[f][t] = []
                for L in lanes:
                    if L["type"] == N.LANE_CIRCULAR:
                        cfg = {"center": [L["cx"], L["cy"]], "radius": L["radius"], "start_phase": L["start_phase"],
                               "end_phase": L["end_phase"], "clockwise": L["direction"] > 0}
                    else:
                        cfg = {"start": [L["sx"], L["sy"]], "end": [L["ex"], L["ey"]]}
                    cfg.update(width=L["width"], forbidden=bool(L["forbidden"]), speed_limit=L["speed_limit"],
                               priority=L["priority"])
                    if L.get("line_types") is not None:
                        cfg["line_types"] = L["line_types"]
                    if L["type"] == N.LANE_SINE:
                        cfg.update(amplitude=L["amplitude"], pulsation=L["pulsation"], phase=L["phase"])
                    out[f][t].append({"class_path": self._CLASS_PATHS[L["type"]], "config": cfg})
        return out

    @classmethod
    def from_config(cls, config: dict) -> "NetworkTable":
        """RoadNetwork.from_config (road/road.py:370-377): rebuilds the table from the reference's (or our) dict
        through the same constructors, so the lane parameters come out bit-identical."""
        net = cls()
        for f, tos in config.items():
            for t, lanes in tos.items():
                for ld in lanes:
                    name, c = ld["class_path"].rsplit(".", 1)[-1], dict(ld["config"])
                    common = dict(width=float(c.get("width", 4.0)), forbidden=bool(c.get("forbidden", False)),
                                  speed_limit=float(c.get("speed_limit", 20.0)), priority=int(c.get("priority", 0)))
                    if name == "CircularLane":
                        net.add_circular(f, t, c["center"], c["radius"], c["start_phase"], c["end_phase"],
                                         clockwise=bool(c.get("clockwise", True)), **common)
                    elif name in ("StraightLane", "SineLane"):
                        sine = (c["amplitude"], c["pulsation"], c["phase"]) if name == "SineLane" else None
                        net.add_straight(f, t, c["start"], c["end"], sine=sine, **common)
                    else:
                        raise NotImplementedError(f"lane class {ld['class_path']!r} (PolyLane) is not on the accelerated path")
                    if c.get("line_types") is not None:
                        net._graph[f][t][-1]["line_types"] = list(c["line_types"])
        net.finalize()
        return net

    # ------------------------------------------------------------------ tables
    def finalize(self) -> None:
        self.node_id: Dict[str, int] = {}
        for f in self._graph:
            self.node_id.setdefault(f, len(self.node_id))
        for f in self._graph:
            for t in self._graph[f]:
                self.node_id.setdefault(t, len(self.node_id))
        self.lanes: List[dict] = []
        self.index: Dict[LaneIndex, int] = {}
        for f, tos in self._graph.items():
            for t, lanes in tos.items():
                first = len(self.lanes)
                for lid, lane in enumerate(lanes):
                    lane = dict(lane, from_node=self.node_id[f], to_node=self.node_id[t], lane_id=lid,
                                road_first=first, road_count=len(lanes),
                                # intersection_env.py:354-373 tests node NAMES: ("il" in from) and ("o" in to)
                                exit_lane=int("il" in f and "o" in t))
                    self.index[(f, t, lid)] = len(self.lanes)
                    self.lanes.append(lane)
        if len(self.lanes) > N.HWY_NET_MAX_LANES or len(self.node_id) > N.HWY_NET_MAX_NODES:
            raise ValueError("road network too large for the device tables")
        self.lane_index_of = {v: k for k, v in self.index.items()}
        self.arrays = {}
        for k in N.NET_LANE_INT_FIELDS:
            self.arrays[k] = np.array([int(l.get(k, 0)) for l in self.lanes], dtype=np.int32)
        for k in N.NET_LANE_F64_FIELDS:
            self.arrays[k] = np.array([float(l.get(k, 0.0)) for l in self.lanes], dtype=np.float64)
        n_nodes = len(self.node_id)
        self.succ = np.full((n_nodes, N.HWY_NET_MAX_SUCC), -1, dtype=np.int32)
        self.succ_count = np.zeros(n_nodes, dtype=np.int32)
        for f, tos in self._graph.items():
            if len(tos) > N.HWY_NET_MAX_SUCC:
                raise ValueError("too many roads leave one node")
            for t in tos:
                self.succ[self.node_id[f], self.succ_count[self.node_id[f]]] = self.index[(f, t, 0)]
                self.succ_count[self.node_id[f]] += 1

    def to_struct(self) -> N.HwyNetGraph:
        g = N.HwyNetGraph()
        g.n_lanes, g.n_nodes = len(self.lanes), len(self.node_id)
        for k, lane in enumerate(self.lanes):
            for f in N.NET_LANE_INT_FIELDS:
                setattr(g.lanes[k], f, int(self.arrays[f][k]))
            for f in N.NET_LANE_F64_FIELDS:
                setattr(g.lanes[k], f, float(self.arrays[f][k]))
        for node in range(g.n_nodes):
            g.succ_count[node] = int(self.succ_count[node])
            for j in range(N.HWY_NET_MAX_SUCC):
                g.succ[node][j] = int(self.succ[node][j])
        return g

    def export_arrays(self) -> dict:
        """Same keys as the reference dump used by the tests (`net_*`)."""
        out = {"net_" + k: v for k, v in self.arrays.items()}
        out["net_succ"], out["net_succ_count"] = self.succ, self.succ_count
        out["net_node_names"] = np.array(list(self.node_id.keys()))
        return out

    # ------------------------------------------------------------------ routing (host only)
    def shortest_path(self, start: str, goal: str) -> List[str]:
        """RoadNetwork.shortest_path / bfs_paths (road.py:159-188): BFS with SORTED successors."""
        queue = [(start, [start])]
        while queue:
            node, path = queue.pop(0)
            if node not in self._graph:
                continue
            for nxt in sorted(k for k in self._graph[node] if k not in path):
                if nxt == goal:
                    return path + [nxt]
                if nxt in self._graph:
                    queue.append((nxt, path + [nxt]))
        return []

    def plan_route(self, lane_index: LaneIndex, destination: str) -> List[Tuple[str, str, Optional[int]]]:
        """ControlledVehicle.plan_route_to (vehicle/controller.py:71-87)."""
        path = self.shortest_path(lane_index[1], destination)
        if path:
            return [lane_index] + [(path[i], path[i + 1], None) for i in range(len(path) - 1)]
        return [lane_index]

    def encode_route(self, route: Sequence[Tuple[str, str, Optional[int]]]) -> Tuple[np.ndarray, int]:
        if len(route) > N.HWY_NET_MAX_ROUTE:
            raise ValueError("route longer than HWY_NET_MAX_ROUTE")
        enc = np.zeros(N.HWY_NET_MAX_ROUTE, dtype=np.int32)
        for k, (f, t, lid) in enumerate(route):
            enc[k] = self.node_id[f] | (self.node_id[t] << 8) | (((-1 if lid is None else int(lid)) + 1) << 16)
        return enc, len(route)

    def route_table(self, destinations: Sequence[str]) -> Tuple[np.ndarray, np.ndarray]:
        """The encoded plan_route(lane, destination) of every lane and destination: [lanes, D, MAX_ROUTE], [lanes, D]."""
        table = np.zeros((len(self.lanes), len(destinations), N.HWY_NET_MAX_ROUTE), dtype=np.int32)
        lens = np.zeros((len(self.lanes), len(destinations)), dtype=np.int32)
        for l in range(len(self.lanes)):
            for d, dest in enumerate(destinations):
                table[l, d], lens[l, d] = self.encode_route(self.plan_route(self.lane_index_of[l], dest))
        return table, lens

    # ------------------------------------------------------------------ vectorised lane geometry (host reset)
    def position(self, lane: int, s, lat):
        """lane.position(s, lat) for arrays s, lat (lane.py:192-197,268-273,338-342)."""
        L = self.lanes[lane]
        s, lat = np.asarray(s, dtype=np.float64), np.asarray(lat, dtype=np.float64)
        if L["type"] == N.LANE_CIRCULAR:
            phi = L["direction"] * s / L["radius"] + L["start_phase"]
            rr = L["radius"] - lat * L["direction"]
            return L["cx"] + rr * np.cos(phi), L["cy"] + rr * np.sin(phi)
        if L["type"] == N.LANE_SINE:
            lat = lat + L["amplitude"] * np.sin(L["pulsation"] * s + L["phase"])
        return (L["sx"] + s * L["dx"]) + lat * L["lx"], (L["sy"] + s * L["dy"]) + lat * L["ly"]

    def heading_at(self, lane: int, s):
        L = self.lanes[lane]
        s = np.asarray(s, dtype=np.float64)
        if L["type"] == N.LANE_CIRCULAR:
            phi = L["direction"] * s / L["radius"] + L["start_phase"]
            return phi + np.pi / 2 * L["direction"]
        if L["type"] == N.LANE_SINE:
            return L["heading"] + np.arctan(L["amplitude"] * L["pulsation"] * np.cos(L["pulsation"] * s + L["phase"]))
        return np.full_like(s, L["heading"])

    def local_coordinates(self, lane: int, x, y):
        L = self.lanes[lane]
        x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
        if L["type"] == N.LANE_CIRCULAR:
            dx, dy = x - L["cx"], y - L["cy"]
            phi = np.arctan2(dy, dx)
            phi = L["start_phase"] + (((phi - L["start_phase"]) + np.pi) % (2 * np.pi) - np.pi)
            r = np.sqrt(dot2(dx, dy, dx, dy))  # np.linalg.norm
            return L["direction"] * (phi - L["start_phase"]) * L["radius"], L["direction"] * (L["radius"] - r)
        dx, dy = x - L["sx"], y - L["sy"]
        lon = dot2(dx, dy, L["dx"], L["dy"])
        lat = dot2(dx, dy, L["lx"], L["ly"])
        if L["type"] == N.LANE_SINE:
            lat = lat - L["amplitude"] * np.sin(L["pulsation"] * lon + L["phase"])
        return lon, lat

    def closest_lane(self, x, y, heading):
        """get_closest_lane_index (road.py:55-71) for arrays of poses: first minimum wins."""
        x, y, heading = (np.asarray(a, dtype=np.float64) for a in (x, y, heading))
        best = np.zeros(x.shape, dtype=np.int32)
        best_d = np.full(x.shape, np.inf)
        for k, L in enumerate(self.lanes):
            s, r = self.local_coordinates(k, x, y)
            angle = np.abs(((heading - self.heading_at(k, s)) + np.pi) % (2 * np.pi) - np.pi)
            d = np.abs(r) + np.maximum(s - L["length"], 0) + np.maximum(0 - s, 0) + 1.0 * angle
            better = d < best_d
            best = np.where(better, k, best)
            best_d = np.where(better, d, best_d)
        return best
