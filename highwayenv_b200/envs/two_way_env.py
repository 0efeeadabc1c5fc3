"""Batched two-way-v0 on the H100 backend.

Host-side mirror of the reference's ``TwoWayEnv`` (highway_env/envs/two_way_env.py): a two-lane road a->b whose left
lane is shared with oncoming traffic on ("b", "a", 0); the controlled MDPVehicle, three IDM vehicles ahead and two
oncoming ones, all created with ``enable_lane_change=False`` (a per-vehicle flag in the state's meta word);
TimeToCollision observation with a 5 s horizon; reward = 0.8 * speed_index / 2 + 0.2 * (how far left the TARGET lane
is) (:35-55); terminated on a crash, never truncated (:57-62).  Same 8-slot kernels as roundabout-v0.
"""
from __future__ import annotations

from .. import _native as N
from ..road.network import NetworkTable
from .common.action import speed_to_index
from .roundabout_env import BatchedRoundaboutEnv


def make_two_way_network(length: float = 800) -> NetworkTable:
    """TwoWayEnv._make_road (two_way_env.py:68-111)."""
    net = NetworkTable()
    net.add_straight("a", "b", [0, 0], [length, 0])
    net.add_straight("a", "b", [0, 4.0], [length, 4.0])
    net.add_straight("b", "a", [length, 0], [0, 0])
    net.finalize()
    return net


class BatchedTwoWayEnv(BatchedRoundaboutEnv):
    ENV_ID = "two-way-v0"
    N_VEHICLES = 6
    EGO_SIDE_LANES = 2  # ("a", "b", 0 / 1)
    REWARD_NAMES = ("high_speed_reward", "left_lane_reward")  # _rewards :50-59

    def _make_network(self) -> NetworkTable:
        return make_two_way_network()

    def define_spaces(self) -> None:
        if self.reset_mode != "device":
            raise NotImplementedError("two-way-v0 resets on the device")
        cfg = self.config
        for key, default in (("normalize_reward", False), ("duration", float("inf")), ("lane_change_reward", 0.0)):
            cfg.setdefault(key, default)  # AbstractEnv has none of these; TwoWayEnv never truncates
        super().define_spaces()
        p = self._params
        p.reward_type = 3
        p.left_lane_reward = float(cfg["left_lane_reward"])
        p.duration = float("inf")

    def _build_spawn_tables(self) -> None:
        s = N.HwyTwoWaySpawn()
        s.lane_ab1, s.lane_ba0 = self.net.index[("a", "b", 1)], self.net.index[("b", "a", 0)]
        ts = self.action_type.target_speeds
        s.ego_speed_index = speed_to_index(ts, 30.0)
        self._scenario = N.HwyNetScenario(kind=N.HWY_SCENARIO_TWO_WAY, u=N.HwyNetScenarioUnion(two_way=s))
