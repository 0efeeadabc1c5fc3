"""ctypes binding of oracle/net_oracle.c (general road network: roundabout-v0) plus the numpy
restatement of RoundaboutEnv._make_vehicles.  TEST INFRASTRUCTURE ONLY (see hwy_oracle.py)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import warnings

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libnet_oracle.so")

NET_MAX_LANES, NET_MAX_NODES, NET_MAX_SUCC, NET_MAX_ROUTE, NET_MAX_TARGET_SPEEDS = 64, 64, 6, 16, 8
OBS_KINEMATICS, OBS_OCCUPANCY, OBS_TTC = 0, 1, 2
KIND_IDM, KIND_MDP, KIND_VEHICLE = 0, 1, 2

_LANE_I = ("type", "from_node", "to_node", "lane_id", "road_first", "road_count", "forbidden", "priority",
           "exit_lane", "_pad")
_LANE_F = ("width", "speed_limit", "length", "sx", "sy", "ex", "ey", "dx", "dy", "lx", "ly", "heading",
           "amplitude", "pulsation", "phase", "cx", "cy", "radius", "start_phase", "end_phase", "direction")


class NetLane(C.Structure):
    _fields_ = [(k, C.c_int32) for k in _LANE_I] + [(k, C.c_double) for k in _LANE_F]


class NetGraph(C.Structure):
    _fields_ = [
        ("n_lanes", C.c_int32), ("n_nodes", C.c_int32),
        ("lanes", NetLane * NET_MAX_LANES),
        ("succ_count", C.c_int32 * NET_MAX_NODES),
        ("succ", (C.c_int32 * NET_MAX_SUCC) * NET_MAX_NODES),
    ]


class NetCfg(C.Structure):
    _fields_ = (
        [(k, C.c_int32) for k in (
            "n_vehicles", "simulation_frequency", "policy_frequency", "n_target_speeds", "obs_type",
            "obs_vehicles_count", "obs_see_behind", "obs_absolute", "obs_normalize", "obs_clip",
            "ttc_horizon", "normalize_reward")]
        + [("duration", C.c_double), ("target_speeds", C.c_double * NET_MAX_TARGET_SPEEDS)]
        + [(k, C.c_double) for k in (
            "obs_x_lo", "obs_x_hi", "obs_y_lo", "obs_y_hi", "obs_vx_lo", "obs_vx_hi", "obs_vy_lo", "obs_vy_hi",
            "collision_reward", "high_speed_reward", "lane_change_reward",
            "acc_max", "comfort_acc_max", "comfort_acc_min", "distance_wanted", "time_wanted",
            "politeness", "lane_change_min_acc_gain", "lane_change_max_braking_imposed", "lane_change_delay",
            "perception_distance")]
        + [(k, C.c_int32) for k in ("regulated", "action_mode", "reward_type", "obs_features", "offroad_terminal",
                                    "connected_lanes")]
        + [(k, C.c_double) for k in ("arrived_reward", "reward_speed_lo", "reward_speed_hi", "right_lane_reward",
                                     "merging_speed_reward")]
        + [("merge_lane", C.c_int32), ("_pad3", C.c_int32), ("left_lane_reward", C.c_double),
           ("ego_pursuit_tau", C.c_double), ("goal_reward", C.c_double), ("exit_lane_a", C.c_int32),
           ("exit_lane_b", C.c_int32),
           ("action_type", C.c_int32), ("act_clip", C.c_int32), ("dynamical", C.c_int32), ("obs_n_feat", C.c_int32),
           ("acc_lo", C.c_double), ("acc_hi", C.c_double), ("steer_lo", C.c_double), ("steer_hi", C.c_double),
           ("obs_feat", C.c_int32 * 16), ("obs_feat_ranged", C.c_int32 * 16),
           ("obs_feat_lo", C.c_double * 16), ("obs_feat_hi", C.c_double * 16),
           ("obs_exit_lane", C.c_int32), ("_pad4", C.c_int32)]
    )


_SF = ("x", "y", "heading", "speed", "target_speed", "timer", "delta", "impact_x", "impact_y")
_SI = ("lane", "target_lane", "kind", "crashed", "has_impact", "check_collisions")


NET_MAX_FEATURES = 16
FEATURE_CODES = {"presence": 0, "x": 1, "y": 2, "vx": 3, "vy": 4, "heading": 5, "cos_h": 6, "sin_h": 7, "cos_d": 8,
                 "sin_d": 9, "long_off": 10, "lat_off": 11, "ang_off": 12, "on_road": 13}
FEAT_UNKNOWN = 14


class NetGridCfg(C.Structure):
    _fields_ = [("n_features", C.c_int32), ("features", C.c_int32 * NET_MAX_FEATURES),
                ("ranged", C.c_int32 * NET_MAX_FEATURES),
                ("range_lo", C.c_double * NET_MAX_FEATURES), ("range_hi", C.c_double * NET_MAX_FEATURES),
                ("x_ranged", C.c_int32), ("y_ranged", C.c_int32),
                ("x_lo", C.c_double), ("x_hi", C.c_double), ("y_lo", C.c_double), ("y_hi", C.c_double),
                ("grid_lo", C.c_double * 2), ("grid_step", C.c_double * 2), ("shape", C.c_int32 * 2),
                ("align_to_vehicle_axes", C.c_int32), ("clip", C.c_int32), ("as_image", C.c_int32),
                ("observe_intentions", C.c_int32)]


def grid_cfg(features=None, grid_size=None, grid_step=None, features_range=None, absolute=False,
             align_to_vehicle_axes=False, clip=True, as_image=False, **_):
    """OccupancyGridObservation.__init__ (envs/common/observation.py:286-333) -> NetGridCfg"""
    gc = NetGridCfg()
    features = list(features) if features is not None else ["presence", "vx", "vy", "on_road"]
    size = np.array(grid_size if grid_size is not None else [[-5.5 * 5, 5.5 * 5], [-5.5 * 5, 5.5 * 5]], dtype=np.float64)
    step = np.array(grid_step if grid_step is not None else [5, 5], dtype=np.float64)
    shape = np.asarray(np.floor((size[:, 1] - size[:, 0]) / step), dtype=np.intp)
    fr = features_range or {"vx": [-80.0, 80.0], "vy": [-80.0, 80.0]}
    gc.n_features = len(features)
    for k, f in enumerate(features):
        gc.features[k] = FEATURE_CODES.get(f, FEAT_UNKNOWN)
        if f in fr and f != "on_road":
            gc.ranged[k], gc.range_lo[k], gc.range_hi[k] = 1, float(fr[f][0]), float(fr[f][1])
    if "x" in fr:
        gc.x_ranged, gc.x_lo, gc.x_hi = 1, float(fr["x"][0]), float(fr["x"][1])
    if "y" in fr:
        gc.y_ranged, gc.y_lo, gc.y_hi = 1, float(fr["y"][0]), float(fr["y"][1])
    gc.grid_lo[0], gc.grid_lo[1] = float(size[0, 0]), float(size[1, 0])
    gc.grid_step[0], gc.grid_step[1] = float(step[0]), float(step[1])
    gc.shape[0], gc.shape[1] = int(shape[0]), int(shape[1])
    gc.align_to_vehicle_axes, gc.clip, gc.as_image = int(bool(align_to_vehicle_axes)), int(bool(clip)), int(bool(as_image))
    gc.observe_intentions = 1
    return gc


class NetState(C.Structure):
    _fields_ = ([(k, C.c_void_p) for k in _SF] + [(k, C.c_void_p) for k in _SI]
                + [("route", C.c_void_p), ("route_len", C.c_void_p), ("speed_index", C.c_void_p),
                   ("time", C.c_void_p), ("count", C.c_void_p), ("is_yielding", C.c_void_p),
                   ("road_steps", C.c_void_p), ("no_lane_change", C.c_void_p), ("lat_speed", C.c_void_p),
                   ("yaw_rate", C.c_void_p)])


def _stale() -> bool:
    src = [os.path.join(_HERE, f) for f in ("net_oracle.c", "net_oracle.h")]
    return not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < max(map(os.path.getmtime, src))


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "net_oracle.c")
    if force or _stale():
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=gnu11",
                               "-o", _LIB_PATH, src, "-lm"])
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):  # build() made it; a read-only tree must not be written to
            build()
        elif _stale():
            warnings.warn(f"{_LIB_PATH} is older than its sources: run build() to use the edited oracle")
        _lib = C.CDLL(_LIB_PATH)
        _lib.net_step.restype = None
        _lib.net_step.argtypes = [C.POINTER(NetGraph), C.POINTER(NetCfg), C.POINTER(NetState), C.c_int,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.net_step_continuous.restype = None
        _lib.net_step_continuous.argtypes = [C.POINTER(NetGraph), C.POINTER(NetCfg), C.POINTER(NetState), C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.net_observe.restype = None
        _lib.net_observe.argtypes = [C.POINTER(NetGraph), C.POINTER(NetCfg), C.POINTER(NetState), C.c_void_p]
        _lib.net_step_agents.restype = None
        _lib.net_step_agents.argtypes = [C.POINTER(NetGraph), C.POINTER(NetCfg), C.POINTER(NetState), C.c_void_p,
                                         C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p]
        _lib.net_observe_agents.restype = None
        _lib.net_observe_agents.argtypes = [C.POINTER(NetGraph), C.POINTER(NetCfg), C.POINTER(NetState), C.c_int,
                                            C.c_void_p]
        _lib.net_neighbours.restype = None
        _lib.net_neighbours.argtypes = [C.POINTER(NetGraph), C.POINTER(NetCfg), C.POINTER(NetState), C.c_int, C.c_int,
                                        C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        _lib.net_rotated_rectangles_intersect.restype = C.c_int
        _lib.net_rotated_rectangles_intersect.argtypes = [C.c_double] * 10
        _lib.net_substeps.restype = None
        _lib.net_substeps.argtypes = [C.POINTER(NetGraph), C.POINTER(NetCfg), C.POINTER(NetState), C.c_int]
        _lib.net_has_arrived.restype = C.c_int
        _lib.net_has_arrived.argtypes = [C.POINTER(NetGraph), C.POINTER(NetState), C.c_int]
        _lib.net_obs_size.restype = C.c_int
        _lib.net_obs_size.argtypes = [C.POINTER(NetCfg)]
        _lib.net_closest_lane.restype = C.c_int
        _lib.net_closest_lane.argtypes = [C.POINTER(NetGraph), C.c_double, C.c_double, C.c_double]
        _lib.net_observe_grid.restype = None
        _lib.net_observe_grid.argtypes = [C.POINTER(NetGraph), C.POINTER(NetState), C.c_int, C.c_int,
                                          C.POINTER(NetGridCfg), C.c_void_p]
        _lib.net_observe_ttc_from.restype = None
        _lib.net_observe_ttc_from.argtypes = [C.POINTER(NetGraph), C.POINTER(NetCfg), C.POINTER(NetState), C.c_int,
                                              C.c_int, C.c_int, C.c_void_p]
        _lib.net_observe_lidar.restype = None
        _lib.net_observe_lidar.argtypes = [C.POINTER(NetState), C.c_int, C.c_int, C.c_int, C.c_double, C.c_int,
                                           C.c_void_p]
        for name in ("net_lane_local", "net_lane_position"):
            getattr(_lib, name).restype = None
            getattr(_lib, name).argtypes = [C.POINTER(NetLane), C.c_double, C.c_double,
                                            C.POINTER(C.c_double), C.POINTER(C.c_double)]
        _lib.net_lane_heading_at.restype = C.c_double
        _lib.net_lane_heading_at.argtypes = [C.POINTER(NetLane), C.c_double]
    return _lib


def graph_from_arrays(d: dict) -> NetGraph:
    """d: the `net_*` arrays of a golden fixture (ref_harness.dump_network) or of the product's
    lane table export."""
    g = NetGraph()
    n = len(d["net_type"])
    g.n_lanes, g.n_nodes = n, len(d["net_succ_count"])
    for k in range(n):
        for f in _LANE_I:
            setattr(g.lanes[k], f, int(d["net_" + f][k]) if "net_" + f in d else 0)
        for f in _LANE_F:
            setattr(g.lanes[k], f, float(d["net_" + f][k]))
    for node in range(g.n_nodes):
        g.succ_count[node] = int(d["net_succ_count"][node])
        for j in range(NET_MAX_SUCC):
            g.succ[node][j] = int(d["net_succ"][node][j]) if j < d["net_succ"].shape[1] else -1
    return g


def cfg_from_dict(config: dict, n_vehicles: int = 5) -> NetCfg:
    """roundabout-v0 / intersection-v0 config dict (envs/roundabout_env.py:13-42,
    envs/intersection_env.py:17-60 over abstract.py:102-125)."""
    c = NetCfg()
    intersection = "spawn_probability" in config
    obs, act = config["observation"], config["action"]
    if obs["type"] == "MultiAgentObservation":  # observation.py:588-604: one observation per controlled vehicle
        obs = obs["observation_config"]
    if act["type"] == "MultiAgentAction":  # action.py:301-333
        act = act["action_config"]
    c.n_vehicles = n_vehicles
    c.simulation_frequency = int(config["simulation_frequency"])
    c.policy_frequency = int(config["policy_frequency"])
    ts = act.get("target_speeds")
    ts = list(np.linspace(20, 30, 3)) if ts is None else [float(t) for t in ts]
    c.n_target_speeds = len(ts)
    for i, t in enumerate(ts):
        c.target_speeds[i] = t
    c.obs_features = 5
    if act["type"] in ("ContinuousAction", "DiscreteAction"):  # action.py:73-196
        c.action_type, c.act_clip = 1, int(bool(act.get("clip", True)))
        c.dynamical = int(bool(act.get("dynamical", False)))
        ar, sr = act.get("acceleration_range") or (-5, 5.0), act.get("steering_range") or (-np.pi / 4, np.pi / 4)
        c.acc_lo, c.acc_hi, c.steer_lo, c.steer_hi = float(ar[0]), float(ar[1]), float(sr[0]), float(sr[1])
    if obs["type"] == "OccupancyGrid":
        c.obs_type = OBS_OCCUPANCY
        c.obs_vehicles_count = 5
    elif obs["type"] == "TimeToCollision":
        c.obs_type = OBS_TTC
        c.ttc_horizon = int(obs.get("horizon", 10))
        c.obs_vehicles_count = 5
    else:
        assert obs["type"] in ("Kinematics", "ExitObservation")
        c.obs_type = OBS_KINEMATICS
        c.obs_vehicles_count = int(obs.get("vehicles_count", 5))
        c.obs_see_behind = int(bool(obs.get("see_behind", False)))
        c.obs_absolute = int(bool(obs.get("absolute", False)))
        c.obs_normalize = int(bool(obs.get("normalize", True)))
        c.obs_clip = int(bool(obs.get("clip", True)))
        feats = obs.get("features") or ["presence", "x", "y", "vx", "vy"]
        generic = not (feats[:5] == ["presence", "x", "y", "vx", "vy"] and feats[5:] in ([], ["cos_h", "sin_h"]))
        c.obs_features = len(feats)
        fr = obs.get("features_range")
        if generic:  # any Vehicle.to_dict column list, per-column ranges
            assert fr is not None, "generic Kinematics columns: give features_range"
            c.obs_n_feat = len(feats)
            for k, f in enumerate(feats):
                c.obs_feat[k] = FEATURE_CODES[f]
                if f in fr:
                    c.obs_feat_ranged[k], c.obs_feat_lo[k], c.obs_feat_hi[k] = 1, float(fr[f][0]), float(fr[f][1])
        if fr is None:  # observation.py:214-226, computed once at the first observe: ego on ("a","b",1), 2 side lanes
            assert "_default_side_lanes" in config, "no features_range: the fixture records the side-lane count"
            w = 4.0 * int(config["_default_side_lanes"])
            fr = {"x": [-200.0, 200.0], "y": [-w, w], "vx": [-80.0, 80.0], "vy": [-80.0, 80.0]}
        (c.obs_x_lo, c.obs_x_hi), (c.obs_y_lo, c.obs_y_hi) = map(lambda r: map(float, r), (fr["x"], fr["y"]))
        (c.obs_vx_lo, c.obs_vx_hi), (c.obs_vy_lo, c.obs_vy_hi) = map(lambda r: map(float, r), (fr["vx"], fr["vy"]))
    c.normalize_reward = int(bool(config.get("normalize_reward", False)))  # merge-v0 has no such key
    c.duration = float(config.get("duration", float("inf")))  # AbstractEnv has no duration; merge never truncates
    c.collision_reward = float(config["collision_reward"])
    c.high_speed_reward = float(config["high_speed_reward"])
    c.lane_change_reward = float(config.get("lane_change_reward", 0))
    c.acc_max, c.comfort_acc_max, c.comfort_acc_min = 6.0, 3.0, -5.0
    c.distance_wanted, c.time_wanted = 10.0, 1.5
    if intersection:  # intersection_env.py:262-265 overrides + RegulatedRoad
        c.distance_wanted, c.comfort_acc_max, c.comfort_acc_min = 7.0, 6.0, -3.0
        c.regulated, c.reward_type = 1, 1
        c.action_mode = 1 if (act.get("longitudinal", True) and not act.get("lateral", True)) else 0
        c.arrived_reward = float(config["arrived_reward"])
        c.reward_speed_lo, c.reward_speed_hi = (float(v) for v in config["reward_speed_range"])
        c.offroad_terminal = int(bool(config["offroad_terminal"]))
    if "merging_speed_reward" in config:  # merge-v0 (envs/merge_env.py:24-37)
        c.reward_type = 2
        c.right_lane_reward = float(config["right_lane_reward"])
        c.merging_speed_reward = float(config["merging_speed_reward"])
        c.reward_speed_lo, c.reward_speed_hi = (float(v) for v in config["reward_speed_range"])
        c.merge_lane = int(config["_merge_lane"])
    if "left_lane_reward" in config:  # two-way-v0 (envs/two_way_env.py:17-33) / u-turn-v0 (envs/u_turn_env.py:14-33)
        c.reward_type = 3
        c.left_lane_reward = float(config["left_lane_reward"])
        if "reward_speed_range" in config:  # u-turn
            c.reward_type = 4
            c.reward_speed_lo, c.reward_speed_hi = (float(v) for v in config["reward_speed_range"])
            # u_turn_env.py:196 sets ego.PURSUIT_TAU, but steering_control reads self.TAU_PURSUIT
            # (controller.py:28,159): the assignment is inert in the reference, so the default tau applies
            c.ego_pursuit_tau = 0.0
    c.obs_exit_lane = -1
    if "goal_reward" in config:  # exit-v0 (envs/exit_env.py:18-44)
        c.reward_type = 5
        c.goal_reward = float(config["goal_reward"])
        c.right_lane_reward = float(config["right_lane_reward"])
        c.reward_speed_lo, c.reward_speed_hi = (float(v) for v in config["reward_speed_range"])
        c.exit_lane_a, c.exit_lane_b = int(config["_exit_lane_a"]), int(config["_exit_lane_b"])
        if obs["type"] == "ExitObservation":
            c.obs_exit_lane = int(config["_obs_exit_lane"])
    c.connected_lanes = int(bool(config.get("neighbour_vehicles_connected_lanes", False)))
    c.politeness, c.lane_change_min_acc_gain = 0.0, 0.2
    c.lane_change_max_braking_imposed, c.lane_change_delay = 2.0, 1.0
    c.perception_distance = 200.0
    return c


class NetOracleBatch:
    """n roundabout envs stepped one by one through the C oracle."""

    def __init__(self, graph: NetGraph, cfg: NetCfg, n_envs: int):
        self.g, self.cfg, self.n, self.V = graph, cfg, int(n_envs), int(cfg.n_vehicles)
        n, V = self.n, self.V
        self.a = {k: np.zeros((n, V), dtype=np.float64) for k in _SF}
        self.a.update({k: np.zeros((n, V), dtype=np.int32) for k in _SI})
        self.a["route"] = np.zeros((n, V, NET_MAX_ROUTE), dtype=np.int32)
        self.a["route_len"] = np.zeros((n, V), dtype=np.int32)
        self.a["speed_index"] = np.zeros(n, dtype=np.int32)
        self.a["time"] = np.zeros(n, dtype=np.float64)
        self.a["count"] = np.full(n, V, dtype=np.int32)
        self.a["is_yielding"] = np.zeros((n, V), dtype=np.int32)
        self.a["road_steps"] = np.zeros(n, dtype=np.int32)
        self.a["no_lane_change"] = np.zeros((n, V), dtype=np.int32)
        self.a["lat_speed"] = np.zeros((n, V), dtype=np.float64)
        self.a["yaw_rate"] = np.zeros((n, V), dtype=np.float64)
        self.obs_size = lib().net_obs_size(C.byref(cfg))
        self.obs = np.zeros((n, self.obs_size), dtype=np.float32)
        self.reward = np.zeros(n, dtype=np.float64)
        self.terminated = np.zeros(n, dtype=np.int32)
        self.truncated = np.zeros(n, dtype=np.int32)

    def _state(self, e: int) -> NetState:
        st = NetState()
        for k in list(_SF) + list(_SI) + ["route", "route_len", "is_yielding"]:
            setattr(st, k, self.a[k][e].ctypes.data)
        st.speed_index = self.a["speed_index"][e:e + 1].ctypes.data
        st.time = self.a["time"][e:e + 1].ctypes.data
        st.count = self.a["count"][e:e + 1].ctypes.data
        st.road_steps = self.a["road_steps"][e:e + 1].ctypes.data
        st.no_lane_change = self.a["no_lane_change"][e].ctypes.data
        st.lat_speed, st.yaw_rate = self.a["lat_speed"][e].ctypes.data, self.a["yaw_rate"][e].ctypes.data
        return st

    def observe(self):
        for e in range(self.n):
            st = self._state(e)
            lib().net_observe(C.byref(self.g), C.byref(self.cfg), C.byref(st), self.obs[e].ctypes.data)
        return self.obs

    # ---- observation plugins on any road family (net_oracle.h "observation plugins")
    def _ego(self, e: int) -> int:
        cnt = int(self.a["count"][e])
        k = np.nonzero(np.isin(self.a["kind"][e, :cnt], (KIND_MDP, 2)))[0]
        return int(k[0]) if len(k) else 0

    def observe_grid(self, gc: "NetGridCfg", egos=None):
        out = np.zeros((self.n, gc.n_features, gc.shape[0], gc.shape[1]), dtype=np.float32)
        for e in range(self.n):
            st = self._state(e)
            lib().net_observe_grid(C.byref(self.g), C.byref(st), int(self.a["count"][e]),
                                   self._ego(e) if egos is None else int(egos[e]), C.byref(gc), out[e].ctypes.data)
        return out

    def observe_ttc(self, egos=None):
        n_t = int(self.cfg.ttc_horizon * self.cfg.policy_frequency)
        out = np.zeros((self.n, 3, 3, n_t), dtype=np.float32)
        for e in range(self.n):
            st = self._state(e)
            si = int(np.ravel(self.a["speed_index"][e])[0])
            lib().net_observe_ttc_from(C.byref(self.g), C.byref(self.cfg), C.byref(st), int(self.a["count"][e]),
                                       self._ego(e) if egos is None else int(egos[e]), si, out[e].ctypes.data)
        return out

    def observe_lidar(self, cells=16, maximum_range=60.0, normalize=True, egos=None):
        out = np.zeros((self.n, cells, 2), dtype=np.float32)
        for e in range(self.n):
            st = self._state(e)
            lib().net_observe_lidar(C.byref(st), int(self.a["count"][e]), self._ego(e) if egos is None else int(egos[e]),
                                    int(cells), float(maximum_range), int(bool(normalize)), out[e].ctypes.data)
        return out

    def step(self, actions):
        if self.cfg.action_type == 1:  # ContinuousAction: float32 [n, 2]
            acts = np.ascontiguousarray(actions, dtype=np.float32).reshape(self.n, 2)
        for e in range(self.n):
            st = self._state(e)
            if self.cfg.action_type == 1:
                lib().net_step_continuous(C.byref(self.g), C.byref(self.cfg), C.byref(st), acts[e].ctypes.data,
                                          self.obs[e].ctypes.data, self.reward[e:e + 1].ctypes.data,
                                          self.terminated[e:e + 1].ctypes.data, self.truncated[e:e + 1].ctypes.data)
                continue
            lib().net_step(C.byref(self.g), C.byref(self.cfg), C.byref(st), int(actions[e]),
                           self.obs[e].ctypes.data, self.reward[e:e + 1].ctypes.data,
                           self.terminated[e:e + 1].ctypes.data, self.truncated[e:e + 1].ctypes.data)
        return self.obs, self.reward, self.terminated, self.truncated

    def load_state(self, e: int, st: dict):
        for k in ("x", "y", "heading", "speed"):
            self.a[k][e] = st[k]
        self.a["target_speed"][e] = np.nan_to_num(st["target_speed"])
        self.a["timer"][e] = np.nan_to_num(st["timer"])
        self.a["delta"][e] = np.nan_to_num(st["delta"], nan=4.0)
        self.a["lane"][e] = st["lane"]
        self.a["target_lane"][e] = np.where(np.asarray(st["target_lane"]) < 0, st["lane"], st["target_lane"])
        self.a["crashed"][e] = st["crashed"]
        has = ~np.isnan(st["impact"][:, 0])
        self.a["has_impact"][e] = has
        self.a["impact_x"][e] = np.where(has, st["impact"][:, 0], 0.0)
        self.a["impact_y"][e] = np.where(has, st["impact"][:, 1], 0.0)
        self.a["check_collisions"][e] = st["check_collisions"]
        if "kind" in st:
            self.a["kind"][e] = st["kind"]
            self.a["count"][e] = int(st["count"])
            self.a["is_yielding"][e] = st["is_yielding"]
            self.a["road_steps"][e] = int(st["road_steps"])
        else:
            kind = np.full(self.V, KIND_IDM, dtype=np.int32)
            kind[0] = KIND_MDP
            self.a["kind"][e] = kind
        self.a["no_lane_change"][e] = st["no_lane_change"] if "no_lane_change" in st else 0
        self.a["lat_speed"][e] = np.nan_to_num(st["lat_speed"]) if "lat_speed" in st else 0.0
        self.a["yaw_rate"][e] = np.nan_to_num(st["yaw_rate"]) if "yaw_rate" in st else 0.0
        self.a["route"][e], self.a["route_len"][e] = st["route"], st["route_len"]
        if self.a["speed_index"].ndim == 2:  # one entry per controlled vehicle, in list order
            si = np.asarray(st["speed_index"])[np.asarray(st["kind"]) == KIND_MDP]
            self.a["speed_index"][e, :len(si)] = si
        else:
            self.a["speed_index"][e] = st["speed_index"][0]
        self.a["time"][e] = float(st["time"])


class IntersectionOracle(NetOracleBatch):
    """intersection-v0: the C oracle for act/step/observe/reward plus the numpy restatement of the
    dynamic population (envs/intersection_env.py:136-140,245-366): per-step _clear_vehicles /
    _spawn_vehicle and the _make_vehicles warm-up, drawing from each env's numpy Generator."""

    VMAX = 32

    def __init__(self, graph: NetGraph, cfg: NetCfg, n_envs: int, net_arrays: dict, config: dict):
        cfg.n_vehicles = self.VMAX
        super().__init__(graph, cfg, n_envs)
        self.config = config
        self.net = net_arrays
        names = [str(x) for x in net_arrays["net_node_names"]]
        self.node = {nm: i for i, nm in enumerate(names)}
        self.names = names
        self.lane_of = {}
        for k in range(len(net_arrays["net_type"])):
            self.lane_of[(names[net_arrays["net_from_node"][k]], names[net_arrays["net_to_node"][k]],
                          int(net_arrays["net_lane_id"][k]))] = k
        self.succ = {nm: [] for nm in names}
        for k in range(len(net_arrays["net_type"])):
            f, t = names[net_arrays["net_from_node"][k]], names[net_arrays["net_to_node"][k]]
            if t not in self.succ[f]:
                self.succ[f].append(t)
        self.rng = [np.random.Generator(np.random.PCG64(0)) for _ in range(n_envs)]
        self.a["count"][:] = 0
        # several controlled vehicles: MultiAgentAction / MultiAgentObservation (intersection-multi-agent-v0)
        self.A = int(config.get("controlled_vehicles", 1))
        if self.A > 1:
            self.a["speed_index"] = np.zeros((n_envs, self.A), dtype=np.int32)
            self.obs = np.zeros((n_envs, self.A * self.obs_size), dtype=np.float32)
            self.agents_reward = np.zeros((n_envs, self.A), dtype=np.float64)
            self.agents_terminated = np.zeros((n_envs, self.A), dtype=np.int32)

    # ---- helpers
    def set_rng_words(self, e, w):
        st = self.rng[e].bit_generator.state
        st["state"]["state"] = (int(w[0]) << 64) | int(w[1])
        st["state"]["inc"] = (int(w[2]) << 64) | int(w[3])
        st["has_uint32"], st["uinteger"] = int(w[4]) >> 32, int(w[4]) & 0xFFFFFFFF
        self.rng[e].bit_generator.state = st

    def rng_words(self, e):
        st = self.rng[e].bit_generator.state
        m = (1 << 64) - 1
        return np.array([st["state"]["state"] >> 64, st["state"]["state"] & m, st["state"]["inc"] >> 64,
                         st["state"]["inc"] & m, (int(st["has_uint32"]) << 32) | int(st["uinteger"])], dtype=np.uint64)

    def _lane_pos(self, lane, s):
        x, y = C.c_double(), C.c_double()
        lib().net_lane_position(C.byref(self.g.lanes[lane]), float(s), 0.0, C.byref(x), C.byref(y))
        return x.value, y.value

    def _shortest_path(self, start, goal):
        queue = [(start, [start])]
        while queue:
            node, path = queue.pop(0)
            for nxt in sorted(k for k in self.succ.get(node, []) if k not in path):
                if nxt == goal:
                    return path + [nxt]
                if self.succ.get(nxt):
                    queue.append((nxt, path + [nxt]))
        return []

    def _route(self, lane, destination):
        f, t, lid = self.names[self.g.lanes[lane].from_node], self.names[self.g.lanes[lane].to_node], self.g.lanes[lane].lane_id
        path = self._shortest_path(t, destination)
        route = [(f, t, lid)] + [(path[i], path[i + 1], None) for i in range(len(path) - 1)]
        enc = np.zeros(NET_MAX_ROUTE, dtype=np.int32)
        for k, (a, b, l) in enumerate(route):
            enc[k] = self.node[a] | (self.node[b] << 8) | (((-1 if l is None else l) + 1) << 16)
        return enc, len(route)

    def _append(self, e, x, y, heading, speed, kind, route, delta, target_speed=None, timer=None):
        n = int(self.a["count"][e])
        lane = lib().net_closest_lane(C.byref(self.g), x, y, heading)
        a = self.a
        a["x"][e, n], a["y"][e, n], a["heading"][e, n], a["speed"][e, n] = x, y, heading, speed
        a["target_speed"][e, n] = speed if target_speed is None else target_speed
        a["timer"][e, n] = ((x + y) * np.pi) % 1.0 if timer is None else timer
        a["delta"][e, n] = delta
        a["impact_x"][e, n] = a["impact_y"][e, n] = 0.0
        a["lane"][e, n] = a["target_lane"][e, n] = lane
        a["kind"][e, n], a["crashed"][e, n], a["has_impact"][e, n] = kind, 0, 0
        a["check_collisions"][e, n], a["is_yielding"][e, n] = 1, 0
        a["route"][e, n], a["route_len"][e, n] = self._route(lane, route)
        a["count"][e] = n + 1
        return n

    # ---- envs/intersection_env.py:325-352
    def _spawn_vehicle(self, e, longitudinal=0.0, position_deviation=1.0, speed_deviation=1.0,
                       spawn_probability=0.6, go_straight=False):
        g = self.rng[e]
        if g.uniform() > spawn_probability:
            return
        route = g.choice(range(4), size=2, replace=False)
        route[1] = (route[0] + 2) % 4 if go_straight else route[1]
        lane = self.lane_of[("o" + str(route[0]), "ir" + str(route[0]), 0)]
        lon = longitudinal + 5.0 + g.normal() * position_deviation
        speed = 8.0 + g.normal() * speed_deviation
        x, y = self._lane_pos(lane, lon)
        heading = lib().net_lane_heading_at(C.byref(self.g.lanes[lane]), float(lon))
        n = int(self.a["count"][e])
        for v in range(n):
            if np.linalg.norm(np.array([self.a["x"][e, v] - x, self.a["y"][e, v] - y])) < 15:
                return
        if n >= self.VMAX:
            raise RuntimeError("vehicle capacity exceeded")
        delta = None
        idx = self._append(e, x, y, heading, speed, KIND_IDM, "o" + str(route[1]), 4.0)
        self.a["delta"][e, idx] = g.uniform(low=3.5, high=4.5)

    # ---- envs/intersection_env.py:354-366
    def _clear_vehicles(self, e):
        n = int(self.a["count"][e])
        keep = []
        for v in range(n):
            L = self.g.lanes[int(self.a["lane"][e, v])]
            s_, lat_ = C.c_double(), C.c_double()
            lib().net_lane_local(C.byref(L), float(self.a["x"][e, v]), float(self.a["y"][e, v]), C.byref(s_), C.byref(lat_))
            leaving = bool(L.exit_lane) and s_.value >= L.length - 4 * 5.0
            if self.a["kind"][e, v] in (KIND_MDP, KIND_VEHICLE) or not leaving:
                keep.append(v)
        if len(keep) != n:
            for k in self.a:
                if k in ("speed_index", "time", "count", "road_steps"):
                    continue
                self.a[k][e, :len(keep)] = self.a[k][e, keep]
            self.a["count"][e] = len(keep)

    # ---- envs/intersection_env.py:245-323
    def reset_env(self, e, seed=None):
        if seed is not None:
            self.rng[e] = np.random.Generator(np.random.PCG64(np.random.SeedSequence(int(seed))))
        g = self.rng[e]
        self.a["count"][e] = 0
        self.a["road_steps"][e] = 0
        self.a["time"][e] = 0.0
        n_vehicles = int(self.config["initial_vehicle_count"])
        for t in range(n_vehicles - 1):
            self._spawn_vehicle(e, np.linspace(0, 80, n_vehicles)[t])
        st = self._state(e)
        lib().net_substeps(C.byref(self.g), C.byref(self.cfg), C.byref(st), 3 * int(self.config["simulation_frequency"]))
        self._spawn_vehicle(e, 60, spawn_probability=1.0, go_straight=True, position_deviation=0.1, speed_deviation=0.0)
        for ego_id in range(self.A):  # :291-315, one controlled vehicle per access road
            ego_lane = self.lane_of[("o%d" % (ego_id % 4), "ir%d" % (ego_id % 4), 0)]
            destination = self.config["destination"] or "o" + str(g.integers(1, 4))
            x, y = self._lane_pos(ego_lane, 60.0 + 5.0 * g.normal(1.0))
            heading = lib().net_lane_heading_at(C.byref(self.g.lanes[ego_lane]), 60.0)
            speed_limit = self.g.lanes[ego_lane].speed_limit
            ts = [self.cfg.target_speeds[i] for i in range(self.cfg.n_target_speeds)]
            si = int(np.clip(np.round((speed_limit - ts[0]) / (ts[-1] - ts[0]) * (len(ts) - 1)), 0, len(ts) - 1))
            if self.cfg.action_type == 1:  # vehicle_class = Vehicle / BicycleVehicle: plan_route_to raises
                idx = self._append(e, x, y, heading, speed_limit, KIND_VEHICLE, destination, 4.0, target_speed=0.0, timer=0.0)
                self.a["route_len"][e, idx] = 0  # AttributeError -> no route, no speed index (:309-315)
                self.a["lat_speed"][e, idx] = self.a["yaw_rate"][e, idx] = 0.0
                si = -1
            else:
                self._append(e, x, y, heading, speed_limit, KIND_MDP, destination, 4.0, target_speed=ts[si], timer=0.0)
            if self.A > 1:
                self.a["speed_index"][e, ego_id] = si
            else:
                self.a["speed_index"][e] = si
            # prevent early collisions: drop the TRAFFIC within 20 m of this controlled vehicle (:317-323)
            n = int(self.a["count"][e])
            keep = [v for v in range(n) if self.a["kind"][e, v] in (KIND_MDP, KIND_VEHICLE) or not (
                np.linalg.norm(np.array([self.a["x"][e, v] - x, self.a["y"][e, v] - y])) < 20)]
            for k in self.a:
                if k in ("speed_index", "time", "count", "road_steps"):
                    continue
                self.a[k][e, :len(keep)] = self.a[k][e, keep]
            self.a["count"][e] = len(keep)

    def observe(self):
        if self.A == 1:
            return super().observe()
        for e in range(self.n):
            st = self._state(e)
            lib().net_observe_agents(C.byref(self.g), C.byref(self.cfg), C.byref(st), self.A, self.obs[e].ctypes.data)
        return self.obs

    def _step_agents(self, actions):
        acts = np.ascontiguousarray(actions, dtype=np.int32).reshape(self.n, self.A)
        for e in range(self.n):
            st = self._state(e)
            lib().net_step_agents(C.byref(self.g), C.byref(self.cfg), C.byref(st), acts[e].ctypes.data, self.A,
                                  self.obs[e].ctypes.data, self.reward[e:e + 1].ctypes.data,
                                  self.terminated[e:e + 1].ctypes.data, self.truncated[e:e + 1].ctypes.data,
                                  self.agents_reward[e].ctypes.data, self.agents_terminated[e].ctypes.data)
        return self.obs, self.reward, self.terminated, self.truncated

    def step(self, actions):
        out = super().step(actions) if self.A == 1 else self._step_agents(actions)
        p = float(self.config["spawn_probability"])
        for e in range(self.n):
            self._clear_vehicles(e)
            self._spawn_vehicle(e, spawn_probability=p)
        return out


class ExitOracle(NetOracleBatch):
    """exit-v0 (envs/exit_env.py): the C oracle for act / step / observe / reward plus the numpy restatement of
    ExitEnv._create_vehicles (:107-145) on each env's numpy Generator.  `lanes` maps (from, to, id) to table indices;
    lanes 0..lanes_count-1 are ("0", "1", id)."""

    def __init__(self, graph: NetGraph, cfg: NetCfg, n_envs: int, config: dict, node_names):
        cfg.n_vehicles = int(config["vehicles_count"]) + 1
        super().__init__(graph, cfg, n_envs)
        self.config = config
        names = [str(x) for x in node_names]
        self.node = {nm: i for i, nm in enumerate(names)}
        self.rng = [np.random.Generator(np.random.PCG64(0)) for _ in range(n_envs)]
        self.a["no_lane_change"][:, 1:] = 1  # vehicle.enable_lane_change = False (:143)
        self.a["check_collisions"][...] = 1
        self.a["kind"][:, 0] = KIND_MDP

    def _route_to_3(self, lane_idx: int):
        L = self.g.lanes[lane_idx]
        enc = np.zeros(NET_MAX_ROUTE, dtype=np.int32)
        enc[0] = L.from_node | (L.to_node << 8) | ((L.lane_id + 1) << 16)
        enc[1] = self.node["1"] | (self.node["2"] << 8)  # ("1", "2", None)
        enc[2] = self.node["2"] | (self.node["3"] << 8)  # ("2", "3", None)
        return enc, 3

    def reset_env(self, e: int, seed=None):
        if seed is not None:
            self.rng[e] = np.random.Generator(np.random.PCG64(np.random.SeedSequence(int(seed))))
        g, cfg, a = self.rng[e], self.config, self.a
        n_lanes = int(cfg["lanes_count"])
        xs = []

        def create_random(lane_id, speed, spacing):  # Vehicle.create_random (vehicle/kinematics.py:50-104), lane given
            L = self.g.lanes[lane_id]  # ("0", "1", lane_id)
            default_spacing = 12 + 1.0 * speed
            offset = spacing * default_spacing * np.exp(-5 / 40 * n_lanes)
            x0 = np.max(xs) if xs else 3 * offset
            x0 += offset * g.uniform(0.9, 1.1)
            px, py = C.c_double(), C.c_double()
            lib().net_lane_position(C.byref(L), float(x0), 0.0, C.byref(px), C.byref(py))
            return px.value, py.value, L.heading

        ts = [self.cfg.target_speeds[i] for i in range(self.cfg.n_target_speeds)]
        for v in range(self.V):
            if v == 0:
                x, y, h = create_random(0, 25.0, float(cfg["ego_spacing"]))
                speed = 25.0
            else:
                lanes = np.arange(n_lanes)
                lane_id = int(g.choice(lanes, size=1, p=lanes / lanes.sum()).astype(int)[0])
                speed = float(self.g.lanes[lane_id].speed_limit)
                x, y, h = create_random(lane_id, speed, 1 / float(cfg["vehicles_density"]))
            L0 = self.g.lanes[0]
            s0, lat0 = C.c_double(), C.c_double()
            lib().net_lane_local(C.byref(L0), x, y, C.byref(s0), C.byref(lat0))
            xs.append(s0.value)
            lane = lib().net_closest_lane(C.byref(self.g), x, y, h)
            a["x"][e, v], a["y"][e, v], a["heading"][e, v], a["speed"][e, v] = x, y, h, speed
            a["lane"][e, v] = a["target_lane"][e, v] = lane
            a["crashed"][e, v] = a["has_impact"][e, v] = 0
            a["impact_x"][e, v] = a["impact_y"][e, v] = 0.0
            a["delta"][e, v] = 4.0
            if v == 0:  # MDPVehicle.__init__ (controller.py:283-293): speed index of its speed, target speed from it
                si = int(np.clip(np.round((speed - ts[0]) / (ts[-1] - ts[0]) * (len(ts) - 1)), 0, len(ts) - 1))
                a["speed_index"][e] = si
                a["target_speed"][e, v], a["timer"][e, v] = ts[si], 0.0
                a["route_len"][e, v] = 0
            else:
                a["target_speed"][e, v] = speed
                a["timer"][e, v] = ((x + y) * np.pi) % 1.0  # IDMVehicle.__init__ (behavior.py:64)
                a["route"][e, v], a["route_len"][e, v] = self._route_to_3(lane)
        a["time"][e] = 0.0

    def rng_words(self, e):
        st = self.rng[e].bit_generator.state
        m = (1 << 64) - 1
        return np.array([st["state"]["state"] >> 64, st["state"]["state"] & m, st["state"]["inc"] >> 64,
                         st["state"]["inc"] & m, (int(st["has_uint32"]) << 32) | int(st["uinteger"])], dtype=np.uint64)
