"""ctypes binding of the C ABI declared in include/hwyb200.h.

The shared library ``csrc/libhwyb200.so`` is built in-tree by ``highwayenv_b200.build``
(nvcc, sm_90a).  There is NO CPU fallback: if the library is missing, or no CUDA device is
visible when a kernel entry point is called, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("HWYB200_LIB") or os.path.join(_HERE, "csrc", "libhwyb200.so")

HWY_ABI_VERSION = 17 # bump with every change of a struct or signature: a stale libhwyb200.so then fails to load
HWY_MAX_LANES = 8
HWY_MAX_TARGET_SPEEDS = 8
HWY_MAX_VEHICLES = 128
HWY_MAX_OBS_VEHICLES = 16
HWY_REWARD_TERMS = 5

KIND_IDM, KIND_MDP, KIND_VEHICLE = 0, 1, 2
META_LANE_SHIFT, META_TARGET_SHIFT = 0, 8
META_CRASHED, META_HAS_IMPACT, META_CHECK_COLLISIONS = 1 << 16, 1 << 17, 1 << 18
META_KIND_SHIFT, META_PRESENT = 19, 1 << 21
META_ORDER_SHIFT = 24  # highway: 7 bits, the stored road order (include/hwyb200.h); a checked hint, not state
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
        + [("obs_n_features", C.c_int32), ("n_agents", C.c_int16), ("multi_action", C.c_uint8),
           ("multi_obs", C.c_uint8),
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


HWY_LINEAR_PARAMS = 5


class HwyLinearTraffic(C.Structure):
    """LinearVehicle traffic of the highway family (include/hwyb200.h)."""
    _fields_ = [("params", C.c_void_p), ("acc_lo", C.c_double * 3), ("acc_span", C.c_double * 3),
                ("steer_lo", C.c_double * 2), ("steer_span", C.c_double * 2)]


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
        + [("merge_lane", C.c_int32), ("merge_end_lane", C.c_int32), ("left_lane_reward", C.c_double),
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
                ("obstacle_x", C.c_double), ("obstacle_y", C.c_double),
                ("lanes_count", C.c_int32), ("vehicles_count", C.c_int32), ("max_position", C.c_double)]


KIND_OBSTACLE = 3
META_NO_LANE_CHANGE = 1 << 23

META_FLAG_BITS = {"crashed": META_CRASHED, "has_impact": META_HAS_IMPACT, "check_collisions": META_CHECK_COLLISIONS,
                  "is_yielding": META_YIELDING, "no_lane_change": META_NO_LANE_CHANGE}


def unpack_meta(meta, flags) -> dict:
    """Per-vehicle meta words -> lane, target_lane, kind and the bool arrays of the named META_FLAG_BITS."""
    meta = np.asarray(meta)
    out = {"lane": (meta >> META_LANE_SHIFT) & 0xFF, "target_lane": (meta >> META_TARGET_SHIFT) & 0xFF,
           "kind": (meta >> META_KIND_SHIFT) & 3}
    for name in flags:
        out[name] = (meta & META_FLAG_BITS[name]) != 0
    return out


def pack_meta(fields: dict, flags) -> np.ndarray:
    """Inverse of unpack_meta for the named flags (every one of them must be in `fields`); sets META_PRESENT."""
    meta = ((np.asarray(fields["lane"], dtype=np.int64) << META_LANE_SHIFT)
            | (np.asarray(fields["target_lane"], dtype=np.int64) << META_TARGET_SHIFT)
            | (np.asarray(fields["kind"], dtype=np.int64) << META_KIND_SHIFT) | META_PRESENT)
    for name in flags:
        meta = meta | np.where(np.asarray(fields[name], dtype=bool), META_FLAG_BITS[name], 0)
    return meta.astype(np.int32)


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


class HwyRoundaboutGenericSpawn(C.Structure):
    _fields_ = [("ego_lane", C.c_int32), ("spawn_road", C.c_int32 * 7), ("vehicles_count", C.c_int32),
                ("fixed_destination", C.c_int32), ("ego_speed_index", C.c_int32), ("route_width", C.c_int32),
                ("route_table", C.c_void_p), ("route_len", C.c_void_p)]


class HwyRacetrackParams(C.Structure):
    _fields_ = [("other_vehicles", C.c_int32), ("terminate_off_road", C.c_int32), ("lane_ab", C.c_int32),
                ("lane_bc", C.c_int32), ("n_from_nodes", C.c_int32), ("ego_lanes", C.c_int32),
                ("lane_centering_cost", C.c_double), ("lane_centering_reward", C.c_double),
                ("action_reward", C.c_double), ("collision_reward", C.c_double), ("on_road_reward", C.c_double)]


# HwyNetScenario.kind: the union member the network reset / step / substeps entry points read
(HWY_SCENARIO_NONE, HWY_SCENARIO_ROUNDABOUT, HWY_SCENARIO_ROUNDABOUT_GENERIC, HWY_SCENARIO_MERGE, HWY_SCENARIO_TWO_WAY,
 HWY_SCENARIO_U_TURN, HWY_SCENARIO_EXIT, HWY_SCENARIO_INTERSECTION, HWY_SCENARIO_RACETRACK) = range(9)


class HwyNetScenarioUnion(C.Union):
    _fields_ = [("roundabout", HwyRoundaboutSpawn), ("roundabout_generic", HwyRoundaboutGenericSpawn),
                ("merge", HwyMergeSpawn), ("two_way", HwyTwoWaySpawn), ("u_turn", HwyUTurnSpawn), ("exit", HwyExitSpawn),
                ("intersection", HwyIntersectionSpawn), ("racetrack", HwyRacetrackParams)]


class HwyNetScenario(C.Structure):
    _fields_ = [("kind", C.c_int32), ("_pad", C.c_int32), ("u", HwyNetScenarioUnion)]


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


class HwyFiniteMdpParams(C.Structure):
    _fields_ = [("policy_frequency", C.c_int32), ("n_target_speeds", C.c_int32), ("l_max", C.c_int32),
                ("n_t", C.c_int32), ("horizon", C.c_double), ("target_speeds", C.c_double * HWY_MAX_TARGET_SPEEDS),
                ("collision_reward", C.c_double), ("right_lane_reward", C.c_double), ("high_speed_reward", C.c_double),
                ("lane_change_reward", C.c_double)]


HWY_VI_MAX_STATES, HWY_VI_MAX_ACTIONS = 4096, 8


class HwyValueIterationParams(C.Structure):
    _fields_ = [("n_envs", C.c_int32), ("s_max", C.c_int32), ("n_actions", C.c_int32), ("iterations", C.c_int32),
                ("gamma", C.c_double), ("state", C.c_void_p), ("action", C.c_void_p)]


HWY_COPY_MAX_BUFS = 32


class HwyRowCopy(C.Structure):
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("row_bytes", C.c_int64)]


class HwyOpdTree(C.Structure):
    _fields_ = ([("n_roots", C.c_int32), ("max_nodes", C.c_int32), ("expansions", C.c_int32), ("n_actions", C.c_int32)]
                + [(n, C.c_void_p) for n in ("discount", "bound", "exists", "expanded", "terminal", "parent", "action",
                                             "depth", "branch", "reward", "value", "upper", "selected", "leaf_row",
                                             "recommended")])


class HwyMctsTree(C.Structure):
    _fields_ = ([("n_roots", C.c_int32), ("max_nodes", C.c_int32), ("episodes", C.c_int32), ("horizon", C.c_int32),
                 ("temperature", C.c_double), ("seed", C.c_uint64)]
                + [(n, C.c_void_p) for n in ("discount", "decision", "exists", "expanded", "parent", "action",
                                             "child_base", "n_children", "count", "prior", "value", "n_nodes",
                                             "skipped", "walk_node", "walk_return", "walk_flags", "leaf", "returns",
                                             "remap", "actions", "recommended")])


class HwyLidarParams(C.Structure):
    _fields_ = [("cells", C.c_int32), ("normalize", C.c_int32), ("maximum_range", C.c_double)]


# ---- lane-keeping-v0
HWY_LK_MAX_ATTR = 3
LK_ATTRIBUTES = {"state": 0, "derivative": 1, "reference_state": 2}  # HwyLaneKeepingParams.attr codes


class HwyLaneKeepingParams(C.Structure):
    _fields_ = ([("frames", C.c_int32), ("n_attr", C.c_int32), ("attr", C.c_int32 * HWY_LK_MAX_ATTR)]
                + [(n, C.c_int32) for n in ("longitudinal", "lateral", "act_clip", "max_episode_steps", "autoreset")]
                + [(n, C.c_double) for n in ("dt", "state_noise", "derivative_noise", "acc_lo", "acc_hi", "steer_lo",
                                             "steer_hi", "x0", "y0", "heading0", "speed0")]
                + [("lanes", HwyNetLane * 2)])


class HwyLaneKeepingState(C.Structure):
    _fields_ = [("n_envs", C.c_int32), ("_pad", C.c_int32), ("state", C.c_void_p), ("lane_phase", C.c_void_p),
                ("elapsed", C.c_void_p), ("rng", C.c_void_p)]


EXPORTS = (
    "hwy_observe_grid", "hwy_observe_ttc", "hwy_observe_lidar",
    "hwy_abi_version", "hwy_last_error", "hwy_highway_slot_stride", "hwy_highway_reset",
    "hwy_highway_observe", "hwy_highway_step", "hwy_highway_substeps", "hwy_launch_count",
    "hwy_network_obs_size", "hwy_network_reset", "hwy_network_step", "hwy_network_substeps", "hwy_network_observe",
    "hwy_debug_network_neighbours", "hwy_debug_rotated_rectangles_intersect",
    "hwy_debug_math", "hwy_debug_pcg64", "hwy_finite_mdp",
    "hwy_value_iteration", "hwy_copy_env_rows", "hwy_available_actions", "hwy_opd_select", "hwy_opd_record",
    "hwy_opd_recommend", "hwy_mcts_advance", "hwy_mcts_backup", "hwy_mcts_recommend", "hwy_mcts_reroot",
    "hwy_lane_keeping_reset", "hwy_lane_keeping_step",
    "hwy_debug_network_lanes", "hwy_debug_network_closest_lanes",
)

# hwy_debug_math ops and their operand / result counts per input (include/hwyb200.h)
MATH_OPS = {"sincos": (0, 1, 2), "idm_pow": (1, 2, 1), "exp_dlog": (2, 2, 1), "py_mod_pos": (3, 2, 1),
            "wrap_to_pi": (4, 1, 1), "not_zero": (5, 1, 1), "div_finite": (6, 2, 1), "dot2": (7, 4, 1),
            "norm2": (8, 2, 1), "beta_of_controlled": (9, 1, 2), "beta_of_angle": (10, 1, 2),
            "speed_to_index": (11, 2 + HWY_MAX_TARGET_SPEEDS, 1)}
# hwy_debug_network_lanes ops and their result counts per input (HWY_LANES_IN operands each; include/hwyb200.h)
HWY_LANES_IN = 5
LANE_OPS = {"local": (0, 2), "position": (1, 2), "heading_at": (2, 1), "distance_with_heading": (3, 3), "on": (4, 1),
            "maybe_on": (5, 1), "prunable": (6, 1), "prunable_scan": (7, HWY_NET_MAX_LANES)}
# hwy_debug_pcg64 draw kinds
PCG_OPS = {"next64": 0, "next32": 1, "next_double": 2, "uniform": 3, "normal": 4, "choice": 5, "pcg_at": 6}

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
    # the highway reset / step / substeps take the LinearVehicle traffic T (None: IDMVehicle traffic)
    P, S, T = C.POINTER(HwyHighwayParams), C.POINTER(HwyHighwayState), C.POINTER(HwyLinearTraffic)
    lib.hwy_highway_reset.restype = C.c_int
    lib.hwy_highway_reset.argtypes = [P, S, T, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hwy_highway_observe.restype = C.c_int
    lib.hwy_highway_observe.argtypes = [P, S, C.c_void_p, C.c_void_p]
    lib.hwy_highway_step.restype = C.c_int
    lib.hwy_highway_step.argtypes = [P, S, T, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                     C.c_void_p, C.c_void_p]
    lib.hwy_highway_substeps.restype = C.c_int
    lib.hwy_highway_substeps.argtypes = [P, S, T, C.c_int, C.c_void_p, C.c_void_p]
    # the network reset / step / substeps take the scenario SC (None: kind NONE, except for the reset)
    NP, NG, NS, SC = C.POINTER(HwyNetParams), C.c_void_p, C.POINTER(HwyNetState), C.POINTER(HwyNetScenario)
    lib.hwy_network_obs_size.restype = C.c_int
    lib.hwy_network_obs_size.argtypes = [NP]
    lib.hwy_network_reset.restype = C.c_int
    lib.hwy_network_reset.argtypes = [NP, NG, SC, NS] + [C.c_void_p] * 5
    lib.hwy_network_step.restype = C.c_int
    lib.hwy_network_step.argtypes = [NP, NG, SC, NS] + [C.c_void_p] * 10
    lib.hwy_network_substeps.restype = C.c_int
    lib.hwy_network_substeps.argtypes = [NP, NG, SC, NS, C.c_void_p, C.c_int, C.c_void_p]
    lib.hwy_network_observe.restype = C.c_int
    lib.hwy_network_observe.argtypes = [NP, NG, NS, C.c_void_p, C.c_void_p]
    lib.hwy_debug_network_neighbours.restype = C.c_int
    lib.hwy_debug_network_neighbours.argtypes = [NP, NG, NS, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hwy_debug_network_closest_lanes.restype = C.c_int
    lib.hwy_debug_network_closest_lanes.argtypes = [NP, NG, NS, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hwy_debug_network_lanes.restype = C.c_int
    lib.hwy_debug_network_lanes.argtypes = [C.POINTER(HwyNetGraph), C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    lib.hwy_debug_rotated_rectangles_intersect.restype = C.c_int
    lib.hwy_debug_rotated_rectangles_intersect.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    lib.hwy_debug_math.restype = C.c_int
    lib.hwy_debug_math.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    lib.hwy_debug_pcg64.restype = C.c_int
    lib.hwy_debug_pcg64.argtypes = [C.c_int, C.c_int, C.c_double, C.c_double, C.c_int, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_int, C.c_void_p]
    OV = C.POINTER(HwyObsView)
    lib.hwy_observe_grid.restype = C.c_int
    lib.hwy_observe_grid.argtypes = [NG, OV, C.POINTER(HwyGridParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hwy_observe_ttc.restype = C.c_int
    lib.hwy_observe_ttc.argtypes = [NG, OV, C.POINTER(HwyTtcParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hwy_observe_lidar.restype = C.c_int
    lib.hwy_observe_lidar.argtypes = [OV, C.POINTER(HwyLidarParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.hwy_finite_mdp.restype = C.c_int
    lib.hwy_finite_mdp.argtypes = [NG, OV, C.POINTER(HwyFiniteMdpParams)] + [C.c_void_p] * 8
    lib.hwy_value_iteration.restype = C.c_int
    lib.hwy_value_iteration.argtypes = [C.POINTER(HwyValueIterationParams)] + [C.c_void_p] * 7
    lib.hwy_copy_env_rows.restype = C.c_int
    lib.hwy_copy_env_rows.argtypes = [C.POINTER(HwyRowCopy), C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    lib.hwy_available_actions.restype = C.c_int
    lib.hwy_available_actions.argtypes = [NG, OV, C.c_int, C.c_void_p, C.c_void_p]
    OT = C.POINTER(HwyOpdTree)
    lib.hwy_opd_select.restype = C.c_int
    lib.hwy_opd_select.argtypes = [OT, C.c_int, C.c_void_p]
    lib.hwy_opd_record.restype = C.c_int
    lib.hwy_opd_record.argtypes = [OT, C.c_int] + [C.c_void_p] * 5
    lib.hwy_opd_recommend.restype = C.c_int
    lib.hwy_opd_recommend.argtypes = [OT, C.c_void_p]
    MT = C.POINTER(HwyMctsTree)
    lib.hwy_mcts_advance.restype = C.c_int
    lib.hwy_mcts_advance.argtypes = [MT, C.c_int, C.c_int] + [C.c_void_p] * 5
    lib.hwy_mcts_backup.restype = C.c_int
    lib.hwy_mcts_backup.argtypes = [MT, C.c_int, C.c_void_p, C.c_void_p]
    lib.hwy_mcts_recommend.restype = C.c_int
    lib.hwy_mcts_recommend.argtypes = [MT, C.c_void_p]
    lib.hwy_mcts_reroot.restype = C.c_int
    lib.hwy_mcts_reroot.argtypes = [MT, C.c_void_p, C.c_void_p, C.c_void_p]
    LP, LS = C.POINTER(HwyLaneKeepingParams), C.POINTER(HwyLaneKeepingState)
    lib.hwy_lane_keeping_reset.restype = C.c_int
    lib.hwy_lane_keeping_reset.argtypes = [LP, LS] + [C.c_void_p] * 4
    lib.hwy_lane_keeping_step.restype = C.c_int
    lib.hwy_lane_keeping_step.argtypes = [LP, LS] + [C.c_void_p] * 7
    if lib.hwy_abi_version() != HWY_ABI_VERSION:
        raise RuntimeError("libhwyb200.so ABI version mismatch; rebuild")
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc != 0:
        raise RuntimeError("hwyb200: " + load().hwy_last_error().decode())
