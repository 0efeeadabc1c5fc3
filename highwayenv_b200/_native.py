"""ctypes binding of the C ABI declared in include/hwyb200.h.

The shared library ``csrc/libhwyb200.so`` is built in-tree by ``highwayenv_b200.build``
(nvcc, sm_90a).  There is NO CPU fallback: if the library is missing, or no CUDA device is
visible when a kernel entry point is called, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("HWYB200_LIB") or os.path.join(_HERE, "csrc", "libhwyb200.so")

HWY_ABI_VERSION = 13  # bump with every change of a struct or signature: a stale libhwyb200.so then fails to load
HWY_MAX_LANES = 8
HWY_MAX_TARGET_SPEEDS = 8
HWY_MAX_VEHICLES = 128
HWY_MAX_OBS_VEHICLES = 16
HWY_REWARD_TERMS = 5

KIND_IDM, KIND_MDP, KIND_VEHICLE = 0, 1, 2
META_LANE_SHIFT, META_TARGET_SHIFT = 0, 8
META_CRASHED, META_HAS_IMPACT, META_CHECK_COLLISIONS = 1 << 16, 1 << 17, 1 << 18
META_KIND_SHIFT, META_PRESENT = 19, 1 << 21
AUTORESET_DISABLED, AUTORESET_SAME_STEP = 0, 1


class HwyStraightLane(C.Structure):
    _fields_ = [(n, C.c_double) for n in (
        "start_x", "start_y", "dir_x", "dir_y", "lat_x", "lat_y", "heading", "length", "width",
        "speed_limit")]


HWY_MAX_OBS_FEATURES = 16
FEATURE_CODES = {"presence": 0, "x": 1, "y": 2, "vx": 3, "vy": 4, "heading": 5, "cos_h": 6, "sin_h": 7,
                 "cos_d": 8, "sin_d": 9, "long_off": 10, "lat_off": 11, "ang_off": 12}


class HwyHighwayParams(C.Structure):
    _fields_ = (
        [(n, C.c_int32) for n in (
            "lanes_count", "n_vehicles", "simulation_frequency", "policy_frequency", "action_type",
            "others_check_collisions", "normalize_reward", "offroad_terminal", "obs_vehicles_count",
            "obs_see_behind", "obs_absolute", "obs_normalize", "obs_clip", "n_target_speeds",
            "initial_lane_id", "act_clip")]
        + [("duration", C.c_double), ("target_speeds", C.c_double * HWY_MAX_TARGET_SPEEDS)]
        + [(n, C.c_double) for n in (
            "collision_reward", "right_lane_reward", "high_speed_reward", "reward_speed_lo",
            "reward_speed_hi", "acc_lo", "acc_hi", "steer_lo", "steer_hi", "ego_spacing",
            "vehicles_density", "ego_speed", "spawn_exp", "acc_max", "comfort_acc_max",
            "comfort_acc_min", "distance_wanted", "time_wanted", "politeness",
            "lane_change_min_acc_gain", "lane_change_max_braking_imposed", "lane_change_delay",
            "delta_lo", "delta_hi", "perception_distance")]
        + [("lanes", HwyStraightLane * HWY_MAX_LANES)]
        + [("obs_n_features", C.c_int32), ("_pad_obs", C.c_int32),
           ("obs_feature", C.c_int32 * HWY_MAX_OBS_FEATURES), ("obs_feature_ranged", C.c_int32 * HWY_MAX_OBS_FEATURES),
           ("obs_feature_lo", C.c_double * HWY_MAX_OBS_FEATURES), ("obs_feature_hi", C.c_double * HWY_MAX_OBS_FEATURES)]
    )


class HwyHighwayState(C.Structure):
    _fields_ = [
        ("n_envs", C.c_int32), ("vp", C.c_int32),
        ("pos", C.c_void_p), ("hs", C.c_void_p), ("tt", C.c_void_p), ("imp", C.c_void_p),
        ("delta", C.c_void_p), ("meta", C.c_void_p), ("speed_index", C.c_void_p),
        ("time", C.c_void_p), ("rng", C.c_void_p), ("reward_terms", C.c_void_p),
    ]



# ---- general road networks (roundabout-v0)
HWY_NET_MAX_LANES, HWY_NET_MAX_NODES, HWY_NET_MAX_SUCC, HWY_NET_MAX_ROUTE, HWY_NET_GROUP = 32, 64, 6, 16, 8
HWY_NET_GROUP_LARGE = 32
LANE_STRAIGHT, LANE_SINE, LANE_CIRCULAR = 0, 1, 2
OBS_KINEMATICS, OBS_OCCUPANCY, OBS_TTC = 0, 1, 2
META_YIELDING = 1 << 22

NET_LANE_INT_FIELDS = ("type", "from_node", "to_node", "lane_id", "road_first", "road_count", "forbidden",
                       "priority", "exit_lane", "_pad")
NET_LANE_F64_FIELDS = ("width", "speed_limit", "length", "sx", "sy", "ex", "ey", "dx", "dy", "lx", "ly",
                       "heading", "amplitude", "pulsation", "phase", "cx", "cy", "radius", "start_phase",
                       "end_phase", "direction")


class HwyNetLane(C.Structure):
    _fields_ = [(n, C.c_int32) for n in NET_LANE_INT_FIELDS] + [(n, C.c_double) for n in NET_LANE_F64_FIELDS]


class HwyNetGraph(C.Structure):
    _fields_ = [
        ("n_lanes", C.c_int32), ("n_nodes", C.c_int32),
        ("lanes", HwyNetLane * HWY_NET_MAX_LANES),
        ("succ_count", C.c_int32 * HWY_NET_MAX_NODES),
        ("succ", (C.c_int32 * HWY_NET_MAX_SUCC) * HWY_NET_MAX_NODES),
    ]


class HwyNetParams(C.Structure):
    _fields_ = (
        [(n, C.c_int32) for n in (
            "n_vehicles", "simulation_frequency", "policy_frequency", "n_target_speeds", "obs_type",
            "obs_vehicles_count", "obs_see_behind", "obs_absolute", "obs_normalize", "obs_clip",
            "ttc_horizon", "normalize_reward")]
        + [("duration", C.c_double), ("target_speeds", C.c_double * HWY_MAX_TARGET_SPEEDS)]
        + [(n, C.c_double) for n in (
            "obs_x_lo", "obs_x_hi", "obs_y_lo", "obs_y_hi", "obs_vx_lo", "obs_vx_hi", "obs_vy_lo",
            "obs_vy_hi", "collision_reward", "high_speed_reward", "lane_change_reward", "acc_max",
            "comfort_acc_max", "comfort_acc_min", "distance_wanted", "time_wanted", "politeness",
            "lane_change_min_acc_gain", "lane_change_max_braking_imposed", "lane_change_delay",
            "perception_distance")]
        + [(n, C.c_int32) for n in ("regulated", "action_mode", "reward_type", "obs_features", "offroad_terminal",
                                    "dynamic_population", "connected_lanes", "n_agents")]
        + [(n, C.c_double) for n in ("arrived_reward", "reward_speed_lo", "reward_speed_hi", "right_lane_reward",
                                     "merging_speed_reward")]
        + [("merge_lane", C.c_int32), ("_pad_merge", C.c_int32), ("left_lane_reward", C.c_double),
           ("goal_reward", C.c_double), ("exit_lane_a", C.c_int32), ("exit_lane_b", C.c_int32),
           ("obs_exit_lane", C.c_int32), ("_pad_exit", C.c_int32),
           ("action_type", C.c_int32), ("act_clip", C.c_int32), ("dynamical", C.c_int32), ("obs_n_feat", C.c_int32),
           ("acc_lo", C.c_double), ("acc_hi", C.c_double), ("steer_lo", C.c_double), ("steer_hi", C.c_double),
           ("obs_feat", C.c_int32 * HWY_MAX_OBS_FEATURES), ("obs_feat_ranged", C.c_int32 * HWY_MAX_OBS_FEATURES),
           ("obs_feat_lo", C.c_double * HWY_MAX_OBS_FEATURES), ("obs_feat_hi", C.c_double * HWY_MAX_OBS_FEATURES)]
    )


class HwyNetState(C.Structure):
    _fields_ = [
        ("n_envs", C.c_int32), ("vp", C.c_int32),
        ("pos", C.c_void_p), ("hs", C.c_void_p), ("tt", C.c_void_p), ("imp", C.c_void_p),
        ("delta", C.c_void_p), ("meta", C.c_void_p), ("route", C.c_void_p), ("route_len", C.c_void_p),
        ("speed_index", C.c_void_p), ("time", C.c_void_p), ("count", C.c_void_p), ("road_steps", C.c_void_p),
        ("rng", C.c_void_p), ("reward_terms", C.c_void_p), ("overflow", C.c_void_p),
    ]


class HwyIntersectionSpawn(C.Structure):
    _fields_ = [("spawn_lane", C.c_int32 * 4), ("spawn_probability", C.c_double),
                ("route_table", C.c_void_p), ("route_len", C.c_void_p),
                ("ego_lane", C.c_int32), ("ego_destination", C.c_int32), ("initial_vehicle_count", C.c_int32),
                ("_pad", C.c_int32), ("scratch", C.c_void_p)]


class HwyMergeSpawn(C.Structure):
    _fields_ = [("lane_ab", C.c_int32 * 2), ("lane_jk", C.c_int32), ("ego_speed_index", C.c_int32),
                ("obstacle_x", C.c_double), ("obstacle_y", C.c_double)]


KIND_OBSTACLE = 3
META_NO_LANE_CHANGE = 1 << 23


class HwyUTurnSpawn(C.Structure):
    _fields_ = [("lane", C.c_int32 * 8), ("longitudinal", C.c_double * 8), ("speed", C.c_double * 8),
                ("ego_speed_index", C.c_int32), ("_pad", C.c_int32), ("route_table", C.c_void_p), ("route_len", C.c_void_p)]


class HwyTwoWaySpawn(C.Structure):
    _fields_ = [("lane_ab1", C.c_int32), ("lane_ba0", C.c_int32), ("ego_speed_index", C.c_int32), ("_pad", C.c_int32)]


class HwyExitSpawn(C.Structure):
    _fields_ = [("lanes_count", C.c_int32), ("n_vehicles", C.c_int32), ("ego_speed_index", C.c_int32), ("_pad", C.c_int32),
                ("ego_speed", C.c_double), ("ego_spacing", C.c_double), ("vehicles_density", C.c_double),
                ("spawn_exp", C.c_double), ("cdf", C.c_double * HWY_MAX_LANES),
                ("route_12", C.c_int32), ("route_23", C.c_int32)]


class HwyRoundaboutSpawn(C.Structure):
    _fields_ = [
        ("ego_lane", C.c_int32), ("spawn_lane", C.c_int32 * 4), ("fixed_destination", C.c_int32),
        ("ego_speed_index", C.c_int32), ("_pad", C.c_int32),
        ("base_longitudinal", C.c_double * 4),
        ("ego_longitudinal", C.c_double), ("ego_heading_longitudinal", C.c_double), ("ego_speed", C.c_double),
        ("position_deviation", C.c_double), ("speed_deviation", C.c_double), ("traffic_speed", C.c_double),
        ("delta_lo", C.c_double), ("delta_hi", C.c_double),
        ("route_table", C.c_void_p), ("route_len", C.c_void_p),
    ]


FEAT_ON_ROAD, FEAT_UNKNOWN = 13, 14
HWY_NET_MAX_ROUTE = 16


class HwyObsView(C.Structure):
    """Read-only view of a state of either family for the observation plugins (include/hwyb200.h)."""
    _fields_ = [("n_envs", C.c_int32), ("vp", C.c_int32), ("n_vehicles", C.c_int32), ("n_agents", C.c_int32),
                ("pos", C.c_void_p), ("hs", C.c_void_p), ("meta", C.c_void_p), ("count", C.c_void_p),
                ("route", C.c_void_p), ("route_len", C.c_void_p), ("speed_index", C.c_void_p)]


class HwyGridParams(C.Structure):
    _fields_ = [("n_features", C.c_int32), ("features", C.c_int32 * HWY_MAX_OBS_FEATURES),
                ("ranged", C.c_int32 * HWY_MAX_OBS_FEATURES),
                ("range_lo", C.c_double * HWY_MAX_OBS_FEATURES), ("range_hi", C.c_double * HWY_MAX_OBS_FEATURES),
                ("x_ranged", C.c_int32), ("y_ranged", C.c_int32),
                ("x_lo", C.c_double), ("x_hi", C.c_double), ("y_lo", C.c_double), ("y_hi", C.c_double),
                ("grid_lo", C.c_double * 2), ("grid_step", C.c_double * 2), ("shape", C.c_int32 * 2),
                ("align_to_vehicle_axes", C.c_int32), ("clip", C.c_int32), ("as_image", C.c_int32),
                ("observe_intentions", C.c_int32)]


class HwyTtcParams(C.Structure):
    _fields_ = [("horizon", C.c_int32), ("policy_frequency", C.c_int32), ("n_target_speeds", C.c_int32),
                ("_pad", C.c_int32), ("target_speeds", C.c_double * HWY_MAX_TARGET_SPEEDS)]


class HwyLidarParams(C.Structure):
    _fields_ = [("cells", C.c_int32), ("normalize", C.c_int32), ("maximum_range", C.c_double)]


EXPORTS = (
    "hwy_observe_grid", "hwy_observe_ttc", "hwy_observe_lidar", "hwy_exit_reset",
    "hwy_abi_version", "hwy_last_error", "hwy_highway_slot_stride", "hwy_highway_reset",
    "hwy_highway_observe", "hwy_highway_step", "hwy_highway_autoreset", "hwy_highway_substeps", "hwy_launch_count",
    "hwy_network_obs_size", "hwy_network_step", "hwy_network_observe", "hwy_roundabout_reset",
    "hwy_intersection_step", "hwy_network_substeps", "hwy_intersection_reset", "hwy_intersection_step_agents",
    "hwy_debug_network_neighbours", "hwy_debug_rotated_rectangles_intersect", "hwy_merge_reset",
    "hwy_two_way_reset", "hwy_u_turn_reset",
)

_lib = None


def load():
    """Load libhwyb200.so (raises RuntimeError when it has not been built)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m highwayenv_b200.build` "
            "(nvcc, sm_90a). highwayenv_b200 has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    lib.hwy_abi_version.restype = C.c_int
    lib.hwy_last_error.restype = C.c_char_p
    lib.hwy_launch_count.restype = C.c_uint64
    lib.hwy_highway_slot_stride.restype = C.c_int
    lib.hwy_highway_slot_stride.argtypes = [C.c_int]
    P, S = C.POINTER(HwyHighwayParams), C.POINTER(HwyHighwayState)
    lib.hwy_highway_reset.restype = C.c_int
    lib.hwy_highway_reset.argtypes = [P, S, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hwy_highway_observe.restype = C.c_int
    lib.hwy_highway_observe.argtypes = [P, S, C.c_void_p, C.c_void_p]
    lib.hwy_highway_step.restype = C.c_int
    lib.hwy_highway_step.argtypes = [P, S, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                     C.c_void_p, C.c_void_p]
    lib.hwy_highway_substeps.restype = C.c_int
    lib.hwy_highway_substeps.argtypes = [P, S, C.c_int, C.c_void_p, C.c_void_p]
    lib.hwy_highway_autoreset.restype = C.c_int
    lib.hwy_highway_autoreset.argtypes = [P, S, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    NP, NG, NS = C.POINTER(HwyNetParams), C.c_void_p, C.POINTER(HwyNetState)
    lib.hwy_network_obs_size.restype = C.c_int
    lib.hwy_network_obs_size.argtypes = [NP]
    lib.hwy_network_step.restype = C.c_int
    lib.hwy_network_step.argtypes = [NP, NG, NS, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hwy_network_observe.restype = C.c_int
    lib.hwy_network_observe.argtypes = [NP, NG, NS, C.c_void_p, C.c_void_p]
    lib.hwy_intersection_step.restype = C.c_int
    lib.hwy_intersection_step.argtypes = [NP, NG, C.POINTER(HwyIntersectionSpawn), NS, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hwy_intersection_step_agents.restype = C.c_int
    lib.hwy_intersection_step_agents.argtypes = [NP, NG, C.POINTER(HwyIntersectionSpawn), NS] + [C.c_void_p] * 10
    lib.hwy_debug_network_neighbours.restype = C.c_int
    lib.hwy_debug_network_neighbours.argtypes = [NP, NG, NS, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hwy_debug_rotated_rectangles_intersect.restype = C.c_int
    lib.hwy_debug_rotated_rectangles_intersect.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.hwy_u_turn_reset.restype = C.c_int
    lib.hwy_u_turn_reset.argtypes = [NP, NG, C.POINTER(HwyUTurnSpawn), NS, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p]
    lib.hwy_two_way_reset.restype = C.c_int
    lib.hwy_two_way_reset.argtypes = [NP, NG, C.POINTER(HwyTwoWaySpawn), NS, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p]
    lib.hwy_exit_reset.restype = C.c_int
    lib.hwy_exit_reset.argtypes = [NP, NG, C.POINTER(HwyExitSpawn), NS, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p]
    lib.hwy_merge_reset.restype = C.c_int
    lib.hwy_merge_reset.argtypes = [NP, NG, C.POINTER(HwyMergeSpawn), NS, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p]
    lib.hwy_intersection_reset.restype = C.c_int
    lib.hwy_intersection_reset.argtypes = [NP, NG, C.POINTER(HwyIntersectionSpawn), NS, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hwy_network_substeps.restype = C.c_int
    lib.hwy_network_substeps.argtypes = [NP, NG, NS, C.c_void_p, C.c_int, C.c_void_p]
    lib.hwy_roundabout_reset.restype = C.c_int
    lib.hwy_roundabout_reset.argtypes = [NP, NG, C.POINTER(HwyRoundaboutSpawn), NS, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p, C.c_void_p]
    OV = C.POINTER(HwyObsView)
    lib.hwy_observe_grid.restype = C.c_int
    lib.hwy_observe_grid.argtypes = [NG, OV, C.POINTER(HwyGridParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hwy_observe_ttc.restype = C.c_int
    lib.hwy_observe_ttc.argtypes = [NG, OV, C.POINTER(HwyTtcParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hwy_observe_lidar.restype = C.c_int
    lib.hwy_observe_lidar.argtypes = [OV, C.POINTER(HwyLidarParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    if lib.hwy_abi_version() != HWY_ABI_VERSION:
        raise RuntimeError("libhwyb200.so ABI version mismatch; rebuild")
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        raise RuntimeError("hwyb200: " + load().hwy_last_error().decode())
