"""Batched u-turn-v0 on the H100 backend.

Host-side mirror of the reference's ``UTurnEnv`` (highway_env/envs/u_turn_env.py): two lanes a->b, a
counter-clockwise circular U-turn b->c (two CircularLanes), two lanes c->d back; the controlled MDPVehicle and six
IDM vehicles placed on fixed lanes with normal-jittered positions / speeds, all routed to "d"; TimeToCollision with
a 16 s horizon; reward (:36-72) = collision, current lane id, clipped speed, normalised, times on_road; terminated
on a crash, truncated at ``duration`` = 10 s.  Same 8-slot kernels as roundabout-v0.
"""
from __future__ import annotations

import numpy as np

from .. import _native as N
from ..road.network import NetworkTable
from .common.action import speed_to_index
from .roundabout_env import BatchedRoundaboutEnv


def make_u_turn_network(length: float = 128) -> NetworkTable:
    """UTurnEnv._make_road (u_turn_env.py:84-177)."""
    net = NetworkTable()
    w = 4.0  # StraightLane.DEFAULT_WIDTH
    net.add_straight("c", "d", [length, w], [0, w])
    net.add_straight("c", "d", [length, 0], [0, 0])
    center = [length, w + 20]
    radius, alpha = 20, 0
    for r in (radius, radius + w):
        net.add_circular("b", "c", center, r, np.deg2rad(90 - alpha), np.deg2rad(-90 + alpha), clockwise=False)
    offset = 2 * radius
    net.add_straight("a", "b", [0, (2 * w + offset) - w], [length, (2 * w + offset) - w])
    net.add_straight("a", "b", [0, 2 * w + offset], [length, 2 * w + offset])
    net.finalize()
    return net


class BatchedUTurnEnv(BatchedRoundaboutEnv):
    ENV_ID = "u-turn-v0"
    N_VEHICLES = 7
    EGO_SIDE_LANES = 2  # ("a", "b", 0 / 1)
    REWARD_NAMES = ("collision_reward", "left_lane_reward", "high_speed_reward", "on_road_reward")  # _rewards :61-72
    # _make_vehicles (:203-275): (lane, longitudinal, speed) of the six IDM vehicles
    TRAFFIC = [(("a", "b", 0), 25.0, 13.5), (("a", "b", 1), 56.0, 14.5), (("b", "c", 1), 0.5, 4.5),
               (("b", "c", 0), 17.5, 5.5), (("c", "d", 0), 1.0, 3.5), (("c", "d", 1), 30.0, 5.5)]

    def _make_network(self) -> NetworkTable:
        return make_u_turn_network()

    def define_spaces(self) -> None:
        if self.reset_mode != "device":
            raise NotImplementedError("u-turn-v0 resets on the device")
        cfg = self.config
        cfg.setdefault("lane_change_reward", 0.0)
        super().define_spaces()
        p = self._params
        p.reward_type = 4
        p.left_lane_reward = float(cfg["left_lane_reward"])
        p.reward_speed_lo, p.reward_speed_hi = (float(v) for v in cfg["reward_speed_range"])

    def _build_spawn_tables(self) -> None:
        net = self.net
        self._route_tables(["d"])
        s = N.HwyUTurnSpawn()
        s.lane[0] = net.index[("a", "b", 0)]
        for k, (li, lon, speed) in enumerate(self.TRAFFIC, start=1):
            s.lane[k], s.longitudinal[k], s.speed[k] = net.index[li], lon, speed
        ts = self.action_type.target_speeds
        s.ego_speed_index = speed_to_index(ts, 16.0)
        s.route_table, s.route_len = self._route_table.data_ptr(), self._route_table_len.data_ptr()
        self._scenario = N.HwyNetScenario(kind=N.HWY_SCENARIO_U_TURN, u=N.HwyNetScenarioUnion(u_turn=s))


class BatchedConnectedLaneUTurnEnv(BatchedUTurnEnv):
    """`u-turn-v1`: ConnectedLaneNeighboursMixin (envs/common/abstract.py:26-37)."""

    ENV_ID = "u-turn-v1"
