"""Batched exit-v0 / exit-v1 on the H100 backend.

Host-side mirror of the reference's ``ExitEnv`` (highway_env/envs/exit_env.py:15-210): a highway in three sections
("0"->"1" with `lanes_count` lanes, "1"->"2" with one more — the exit lane —, "2"->"3") and a circular exit ramp
("2"->"exit"); the controlled MDPVehicle and `vehicles_count` IDM vehicles routed to "3" with lane changes disabled;
``ExitObservation`` (a Kinematics table whose ego row carries the longitudinal coordinate on the exit lane,
envs/common/observation.py:624-675); reward with a goal term for targeting the exit lane (:147-198).

21 vehicles need the 32-slot network kernels (the intersection family's `network_step_kernel<32>` without rules or
population changes); the device reset draws from the env's numpy stream (weighted `choice(p=...)` + `uniform`).
"""
from __future__ import annotations

import numpy as np

from .. import _native as N
from ..road.network import NetworkTable
from .common.action import speed_to_index
from .common.observation import OBSERVATION_TYPES, KinematicObservation
from .roundabout_env import BatchedRoundaboutEnv


class ExitObservation(KinematicObservation):
    """ExitObservation (reference observation.py:624-675): KinematicObservation whose ego row has
    x = exit_lane.local_coordinates(ego.position)[0] for the exit lane ("1", "2", -1).  Only defined on the exit envs
    (the reference hard-codes that lane index)."""


OBSERVATION_TYPES["ExitObservation"] = ExitObservation


def make_exit_network(lanes_count: int = 6, road_length: float = 1000, exit_position: float = 400,
                      exit_length: float = 100) -> NetworkTable:
    """ExitEnv._create_road (exit_env.py:56-105): RoadNetwork.straight_road_network x 3 (road/road.py:291-321), lane
    speed limits 26 - 3.4 * id, and the forbidden circular exit lane."""
    net = NetworkTable()
    for (f, t), n_l, start, length in ((("0", "1"), lanes_count, 0.0, exit_position),
                                       (("1", "2"), lanes_count + 1, exit_position, exit_length),
                                       (("2", "3"), lanes_count, exit_position + exit_length,
                                        road_length - exit_position - exit_length)):
        for lane in range(n_l):
            rotation = np.array([[np.cos(0.0), np.sin(0.0)], [-np.sin(0.0), np.cos(0.0)]])
            origin = rotation @ np.array([start, lane * 4.0])
            end = rotation @ np.array([start + length, lane * 4.0])
            net.add_straight(f, t, origin, end, speed_limit=26 - 3.4 * lane)
    exit_pos = np.array([exit_position + exit_length, lanes_count * 4.0])
    radius = 150
    net.add_circular("2", "exit", exit_pos + np.array([0, radius]), radius, 3 * np.pi / 2, 2 * np.pi, forbidden=True)
    net.finalize()
    return net


class BatchedExitEnv(BatchedRoundaboutEnv):
    ENV_ID = "exit-v0"
    SLOTS = N.HWY_NET_GROUP_LARGE
    N_VEHICLES = 21
    REWARD_NAMES = ("collision_reward", "goal_reward", "high_speed_reward", "right_lane_reward")  # _rewards :164-176

    def __init__(self, config=None, **kw):
        cfg = self.default_config()
        if config:
            cfg.update(config)
        self.N_VEHICLES = int(cfg["vehicles_count"]) + 1
        if not 1 <= self.N_VEHICLES <= N.HWY_NET_GROUP_LARGE:
            raise ValueError(f"vehicles_count must be <= {N.HWY_NET_GROUP_LARGE - 1}")
        if int(cfg.get("controlled_vehicles", 1)) != 1:
            raise NotImplementedError("controlled_vehicles != 1 on exit-v0")
        self.EGO_SIDE_LANES = int(cfg["lanes_count"])  # the controlled vehicle spawns on ("0", "1", 0)
        super().__init__(config=config, **kw)

    def _make_network(self) -> NetworkTable:
        n_l = int(self.config["lanes_count"])
        if not 2 <= n_l <= N.HWY_MAX_LANES - 1:
            raise ValueError("lanes_count out of range")
        return make_exit_network(n_l)

    def define_spaces(self) -> None:
        if self.reset_mode != "device":
            raise NotImplementedError("exit envs reset on the device")
        cfg = self.config
        if cfg.get("other_vehicles_type") != "highway_env.vehicle.behavior.IDMVehicle":
            raise NotImplementedError("only IDMVehicle traffic is on the accelerated path")
        cfg.setdefault("lane_change_reward", 0.0)
        super().define_spaces()
        p = self._params
        p.reward_type = 5
        p.goal_reward = float(cfg["goal_reward"])
        p.right_lane_reward = float(cfg["right_lane_reward"])
        p.reward_speed_lo, p.reward_speed_hi = (float(v) for v in cfg["reward_speed_range"])
        n_l = int(cfg["lanes_count"])
        p.exit_lane_a, p.exit_lane_b = self.net.index[("1", "2", n_l)], self.net.index[("2", "exit", 0)]
        p.obs_exit_lane = self.net.index[("1", "2", n_l)] if isinstance(self.observation_type, ExitObservation) else 0

    def _build_spawn_tables(self) -> None:
        cfg, net = self.config, self.net
        n_l = int(cfg["lanes_count"])
        s = N.HwyExitSpawn()
        s.lanes_count, s.n_vehicles = n_l, self.N_VEHICLES
        ts = self.action_type.target_speeds
        s.ego_speed_index = speed_to_index(ts, 25.0)
        s.ego_speed, s.ego_spacing = 25.0, float(cfg["ego_spacing"])
        s.vehicles_density = float(cfg["vehicles_density"])
        s.spawn_exp = float(np.exp(-5 / 40 * n_l))
        lanes = np.arange(n_l)
        p = lanes / lanes.sum()
        cdf = p.cumsum()  # Generator.choice(a, size, p): cdf = p.cumsum(); cdf /= cdf[-1]; searchsorted(random(), "right")
        cdf /= cdf[-1]
        for k in range(n_l):
            s.cdf[k] = float(cdf[k])
        s.route_12 = int(net.encode_route([("1", "2", None)])[0][0])
        s.route_23 = int(net.encode_route([("2", "3", None)])[0][0])
        self._scenario = N.HwyNetScenario(kind=N.HWY_SCENARIO_EXIT, u=N.HwyNetScenarioUnion(exit=s))

    def _step_result(self, info):
        info["is_success"] = self._reward_terms[:, 1] > 0  # ExitEnv.step (:51-54): info["is_success"]
        return super()._step_result(info)


class BatchedConnectedLaneExitEnv(BatchedExitEnv):
    """`exit-v1`: ConnectedLaneNeighboursMixin (envs/common/abstract.py:26-37)."""

    ENV_ID = "exit-v1"
