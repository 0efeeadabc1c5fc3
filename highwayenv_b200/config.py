"""Environment configuration dictionaries (same keys and defaults as the reference).

Restates, per registered id, the class-chain ``default_config()`` of the reference:
``AbstractEnv.default_config`` (highway_env/envs/common/abstract.py:102-125) <-
``HighwayEnv`` (envs/highway_env.py:25-53) <- ``HighwayEnvFast`` (:162-175), and the
validation rule of ``utils.update_config`` (highway_env/utils.py:440-478): a nested mapping
override must redefine every key of the mapping it replaces.  ``configure`` itself is a
shallow ``dict.update`` (abstract.py:127-129).
"""
from __future__ import annotations

import copy
from typing import Any, Mapping


def abstract_default_config() -> dict:
    return {
        "observation": {"type": "Kinematics"},
        "action": {"type": "DiscreteMetaAction"},
        "simulation_frequency": 15,
        "policy_frequency": 1,
        "other_vehicles_type": "highway_env.vehicle.behavior.IDMVehicle",
        "screen_width": 600,
        "screen_height": 150,
        "centering_position": [0.3, 0.5],
        "scaling": 5.5,
        "show_trajectories": False,
        "render_agent": True,
        "offscreen_rendering": None,
        "manual_control": False,
        "real_time_rendering": False,
        "neighbour_vehicles_connected_lanes": False,
    }


def update_config_check(config: Mapping[str, Any], delta: Mapping[str, Any], path: str = "config") -> None:
    for key, val in config.items():
        if key not in delta or not isinstance(val, Mapping):
            continue
        sub = f"{path}.{key}"
        new_val = delta[key]
        assert isinstance(new_val, Mapping), f"{sub} must be a mapping, got {type(new_val).__name__}"
        if key in ("action", "observation"):
            nested = new_val.get(key + "_config")
            if isinstance(nested, Mapping):
                new_val = {**new_val, **nested}
        missing_keys = val.keys() - new_val.keys()
        assert not missing_keys, f"{sub} invalid: {missing_keys=}"
        update_config_check(val, new_val, sub)


def update_config(config: dict, delta: Mapping[str, Any]) -> dict:
    update_config_check(config, delta)
    config.update(delta)
    return config


def highway_default_config() -> dict:
    config = abstract_default_config()
    update_config(config, {
        "observation": {"type": "Kinematics"},
        "action": {"type": "DiscreteMetaAction"},
        "lanes_count": 4,
        "vehicles_count": 50,
        "controlled_vehicles": 1,
        "initial_lane_id": None,
        "duration": 40,
        "ego_spacing": 2,
        "vehicles_density": 1,
        "collision_reward": -1,
        "right_lane_reward": 0.1,
        "high_speed_reward": 0.4,
        "lane_change_reward": 0,
        "reward_speed_range": [20, 30],
        "normalize_reward": True,
        "offroad_terminal": False,
    })
    return config


def highway_fast_default_config() -> dict:
    cfg = highway_default_config()
    update_config(cfg, {
        "simulation_frequency": 5,
        "lanes_count": 3,
        "vehicles_count": 20,
        "duration": 30,
        "ego_spacing": 1.5,
    })
    return cfg


# backend keys the reference ignores
BACKEND_DEFAULTS = {"num_envs": 1, "device": "cuda"}

DEFAULTS = {
    "highway-v0": highway_default_config,
    "highway-fast-v0": highway_fast_default_config,
}


def default_config(env_id: str) -> dict:
    return copy.deepcopy(DEFAULTS[env_id]())


def roundabout_default_config() -> dict:
    """RoundaboutEnv.default_config (highway_env/envs/roundabout_env.py:13-42)."""
    config = abstract_default_config()
    update_config(config, {
        "observation": {
            "type": "Kinematics",
            "absolute": True,
            "features_range": {"x": [-100, 100], "y": [-100, 100], "vx": [-15, 15], "vy": [-15, 15]},
        },
        "action": {"type": "DiscreteMetaAction", "target_speeds": [0, 8, 16]},
        "incoming_vehicle_destination": None,
        "collision_reward": -1,
        "high_speed_reward": 0.2,
        "right_lane_reward": 0,
        "lane_change_reward": -0.05,
        "screen_width": 600,
        "screen_height": 600,
        "centering_position": [0.5, 0.6],
        "duration": 11,
        "normalize_reward": True,
    })
    return config


DEFAULTS["roundabout-v0"] = roundabout_default_config


def intersection_default_config() -> dict:
    """IntersectionEnv.default_config (highway_env/envs/intersection_env.py:17-60)."""
    config = abstract_default_config()
    update_config(config, {
        "observation": {
            "type": "Kinematics",
            "vehicles_count": 15,
            "features": ["presence", "x", "y", "vx", "vy", "cos_h", "sin_h"],
            "features_range": {"x": [-100, 100], "y": [-100, 100], "vx": [-20, 20], "vy": [-20, 20]},
            "absolute": True,
            "flatten": False,
            "observe_intentions": False,
        },
        "action": {"type": "DiscreteMetaAction", "longitudinal": True, "lateral": False,
                   "target_speeds": [0, 4.5, 9]},
        "duration": 13,
        "destination": "o1",
        "controlled_vehicles": 1,
        "initial_vehicle_count": 10,
        "spawn_probability": 0.6,
        "screen_width": 600,
        "screen_height": 600,
        "centering_position": [0.5, 0.6],
        "scaling": 5.5 * 1.3,
        "collision_reward": -5,
        "high_speed_reward": 1,
        "arrived_reward": 1,
        "reward_speed_range": [7.0, 9.0],
        "normalize_reward": False,
        "offroad_terminal": False,
    })
    return config


DEFAULTS["intersection-v0"] = intersection_default_config


def _connected(base):
    """ConnectedLaneNeighboursMixin.default_config (envs/common/abstract.py:26-37)."""
    def make() -> dict:
        config = base()
        update_config(config, {"neighbour_vehicles_connected_lanes": True})
        return config
    return make


def roundabout_generic_default_config() -> dict:
    """RoundaboutGenericEnv.default_config (highway_env/envs/roundabout_env.py:407-419)."""
    config = roundabout_default_config()
    update_config(config, {"roundabout_radius": 20, "roundabout_lanes": 2, "vehicles_count": 5, "duration": 17})
    return config


DEFAULTS["roundabout-v1"] = _connected(roundabout_default_config)
DEFAULTS["roundabout-generic-v0"] = roundabout_generic_default_config
DEFAULTS["roundabout-generic-v1"] = _connected(roundabout_generic_default_config)
DEFAULTS["intersection-v2"] = _connected(intersection_default_config)


def multi_agent_intersection_default_config() -> dict:
    """MultiAgentIntersectionEnv.default_config (envs/intersection_env.py:376-420)."""
    config = intersection_default_config()
    update_config(config, {
        "action": {
            "type": "MultiAgentAction",
            "action_config": {"type": "DiscreteMetaAction", "lateral": False, "longitudinal": True,
                              "target_speeds": [0, 4.5, 9]},
        },
        "observation": {
            "type": "MultiAgentObservation",
            "observation_config": {
                "type": "Kinematics",
                "vehicles_count": 15,
                "features": ["presence", "x", "y", "vx", "vy", "cos_h", "sin_h"],
                "features_range": {"x": [-100, 100], "y": [-100, 100], "vx": [-20, 20], "vy": [-20, 20]},
                "absolute": True,
                "flatten": False,
                "observe_intentions": False,
            },
        },
        "controlled_vehicles": 2,
    })
    return config


DEFAULTS["intersection-multi-agent-v0"] = multi_agent_intersection_default_config
DEFAULTS["intersection-multi-agent-v1"] = multi_agent_intersection_default_config
DEFAULTS["intersection-multi-agent-v2"] = _connected(multi_agent_intersection_default_config)


def merge_default_config() -> dict:
    """MergeEnv.default_config (highway_env/envs/merge_env.py:24-37) over AbstractEnv's."""
    config = abstract_default_config()
    update_config(config, {
        "collision_reward": -1,
        "right_lane_reward": 0.1,
        "high_speed_reward": 0.2,
        "reward_speed_range": [20, 30],
        "merging_speed_reward": -0.5,
        "lane_change_reward": -0.05,
    })
    return config


DEFAULTS["merge-v0"] = merge_default_config
DEFAULTS["merge-v1"] = _connected(merge_default_config)


def merge_generic_default_config() -> dict:
    """MergeGenericEnv.default_config (highway_env/envs/merge_env.py:217-236)."""
    config = merge_default_config()
    update_config(config, {"lanes_count": 2, "vehicles_count": 3, "before_merge_length": 150,
                           "converge_merge_length": 80, "parallel_merge_length": 80, "after_merge_length": 150})
    return config


DEFAULTS["merge-generic-v0"] = merge_generic_default_config
DEFAULTS["merge-generic-v1"] = _connected(merge_generic_default_config)


def two_way_default_config() -> dict:
    """TwoWayEnv.default_config (highway_env/envs/two_way_env.py:17-33) over AbstractEnv's."""
    config = abstract_default_config()
    update_config(config, {
        "observation": {"type": "TimeToCollision", "horizon": 5},
        "action": {"type": "DiscreteMetaAction"},
        "collision_reward": 0,
        "left_lane_constraint": 1,
        "left_lane_reward": 0.2,
        "high_speed_reward": 0.8,
    })
    return config


DEFAULTS["two-way-v0"] = two_way_default_config


def u_turn_default_config() -> dict:
    """UTurnEnv.default_config (highway_env/envs/u_turn_env.py:14-33) over AbstractEnv's."""
    config = abstract_default_config()
    update_config(config, {
        "observation": {"type": "TimeToCollision", "horizon": 16},
        "action": {"type": "DiscreteMetaAction", "target_speeds": [8, 16, 24]},
        "screen_width": 789,
        "screen_height": 289,
        "duration": 10,
        "collision_reward": -1.0,
        "left_lane_reward": 0.1,
        "high_speed_reward": 0.4,
        "reward_speed_range": [8, 24],
        "normalize_reward": True,
        "offroad_terminal": False,
    })
    return config


DEFAULTS["u-turn-v0"] = u_turn_default_config
DEFAULTS["u-turn-v1"] = _connected(u_turn_default_config)


def exit_default_config() -> dict:
    """ExitEnv.default_config (highway_env/envs/exit_env.py:18-44) over HighwayEnv's."""
    config = highway_default_config()
    update_config(config, {
        "observation": {
            "type": "ExitObservation",
            "vehicles_count": 15,
            "features": ["presence", "x", "y", "vx", "vy", "cos_h", "sin_h"],
            "clip": False,
        },
        "action": {"type": "DiscreteMetaAction", "target_speeds": [18, 24, 30]},
        "lanes_count": 6,
        "collision_reward": 0,
        "high_speed_reward": 0.1,
        "right_lane_reward": 0,
        "normalize_reward": True,
        "goal_reward": 1,
        "vehicles_count": 20,
        "vehicles_density": 1.5,
        "controlled_vehicles": 1,
        "duration": 18,
        "simulation_frequency": 5,
        "scaling": 5,
    })
    return config


DEFAULTS["exit-v0"] = exit_default_config
DEFAULTS["exit-v1"] = _connected(exit_default_config)


def continuous_intersection_default_config() -> dict:
    """ContinuousIntersectionEnv.default_config (highway_env/envs/intersection_env.py:432-473)."""
    import numpy as np

    config = intersection_default_config()
    update_config(config, {
        "observation": {
            "type": "Kinematics",
            "vehicles_count": 5,
            "features": ["presence", "x", "y", "vx", "vy", "long_off", "lat_off", "ang_off"],
            "features_range": {"x": [-100, 100], "y": [-100, 100], "vx": [-20, 20], "vy": [-20, 20]},
            "absolute": True,
            "flatten": False,
            "observe_intentions": False,
        },
        "action": {
            "type": "ContinuousAction",
            "steering_range": [-np.pi / 3, np.pi / 3],
            "longitudinal": True,
            "lateral": True,
            "dynamical": True,
            "target_speeds": [0, 4.5, 9],
        },
    })
    return config


DEFAULTS["intersection-v1"] = continuous_intersection_default_config


def lane_keeping_default_config() -> dict:
    """LaneKeepingEnv.default_config (highway_env/envs/lane_keeping_env.py:25-52) over AbstractEnv's."""
    import numpy as np

    config = abstract_default_config()
    update_config(config, {
        "observation": {
            "type": "AttributesObservation",
            "attributes": ["state", "derivative", "reference_state"],
        },
        "action": {
            "type": "ContinuousAction",
            "steering_range": [-np.pi / 3, np.pi / 3],
            "longitudinal": False,
            "lateral": True,
            "dynamical": True,
        },
        "simulation_frequency": 10,
        "policy_frequency": 10,
        "state_noise": 0.05,
        "derivative_noise": 0.05,
        "screen_width": 600,
        "screen_height": 250,
        "scaling": 7,
        "centering_position": [0.4, 0.5],
    })
    return config


DEFAULTS["lane-keeping-v0"] = lane_keeping_default_config


def racetrack_default_config() -> dict:
    """RacetrackEnv.default_config (highway_env/envs/racetrack_env.py:28-64) over AbstractEnv's."""
    config = abstract_default_config()
    update_config(config, {
        "observation": {
            "type": "OccupancyGrid",
            "features": ["presence", "on_road"],
            "grid_size": [[-18, 18], [-18, 18]],
            "grid_step": [3, 3],
            "as_image": False,
            "align_to_vehicle_axes": True,
        },
        "action": {
            "type": "ContinuousAction",
            "longitudinal": False,
            "lateral": True,
            "target_speeds": [0, 5, 10],
        },
        "simulation_frequency": 15,
        "policy_frequency": 5,
        "duration": 300,
        "collision_reward": -1,
        "lane_centering_cost": 4,
        "lane_centering_reward": 1,
        "action_reward": -0.3,
        "controlled_vehicles": 1,
        "other_vehicles": 1,
        "screen_width": 600,
        "screen_height": 600,
        "centering_position": [0.5, 0.5],
        "speed_limit": 10.0,
        "terminate_off_road": True,
    })
    return config


DEFAULTS["racetrack-v0"] = racetrack_default_config
DEFAULTS["racetrack-v1"] = _connected(racetrack_default_config)
# RacetrackEnvLarge keeps RacetrackEnv.default_config
DEFAULTS["racetrack-large-v0"] = racetrack_default_config
DEFAULTS["racetrack-large-v1"] = _connected(racetrack_default_config)


def racetrack_oval_default_config() -> dict:
    """RacetrackEnvOval.default_config (highway_env/envs/racetrack_env.py:894-934): RacetrackEnv's and the oval's keys."""
    config = racetrack_default_config()
    update_config(config, {"length": 100, "no_lanes": 3, "block_lane": False, "force_decision": False})
    return config


DEFAULTS["racetrack-oval-v0"] = racetrack_oval_default_config
DEFAULTS["racetrack-oval-v1"] = _connected(racetrack_oval_default_config)
