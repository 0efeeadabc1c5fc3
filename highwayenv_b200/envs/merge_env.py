"""Batched merge-v0 / merge-v1 on the H100 backend.

Host-side mirror of the reference's ``MergeEnv`` (highway_env/envs/merge_env.py): a two-lane highway a->b->c->d
with an access ramp j->k (straight) ->b (sine) ->c (third, forbidden lane) that ends on an ``Obstacle``; the
controlled MDPVehicle, three IDM vehicles, and one merging IDM vehicle on the ramp.  Same kernels as roundabout-v0
(8 vehicle slots per env): the Obstacle occupies the slot after the five vehicles (kind 3: it never acts or moves,
is seen by the neighbour search, IDM and the Kinematics observation, and takes no impact of its own).  Reward
(:39-78) adds an altruistic penalty for slow vehicles on the merging lane; the episode ends on a crash or past
x = 370 and is never truncated (:80-84).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .. import _native as N
from ..road.network import NetworkTable
from ..spaces import Box
from .roundabout_env import BatchedRoundaboutEnv


def make_merge_network() -> NetworkTable:
    """MergeEnv._make_road (merge_env.py:90-148)."""
    net = NetworkTable()
    ends = [150, 80, 80, 150]  # before, converging, merge, after
    y = [0, 4.0]
    for i in range(2):
        net.add_straight("a", "b", [0, y[i]], [sum(ends[:2]), y[i]])
        net.add_straight("b", "c", [sum(ends[:2]), y[i]], [sum(ends[:3]), y[i]])
        net.add_straight("c", "d", [sum(ends[:3]), y[i]], [sum(ends), y[i]])
    amplitude = 3.25
    jk_start, jk_end = np.array([0, 6.5 + 4 + 4]), np.array([ends[0], 6.5 + 4 + 4])
    net.add_straight("j", "k", jk_start, jk_end, forbidden=True)
    jk = NetworkTable()
    jk.add_straight("j", "k", jk_start, jk_end)
    jk.finalize()
    kb_start = np.array(jk.position(0, float(ends[0]), -amplitude), dtype=np.float64)
    kb_end = np.array(jk.position(0, float(sum(ends[:2])), -amplitude), dtype=np.float64)
    net.add_straight("k", "b", kb_start, kb_end, forbidden=True,
                     sine=(amplitude, 2 * np.pi / (2 * ends[1]), np.pi / 2))
    kb = NetworkTable()
    kb.add_straight("k", "b", kb_start, kb_end, sine=(amplitude, 2 * np.pi / (2 * ends[1]), np.pi / 2))
    kb.finalize()
    bc_start = np.array(kb.position(0, float(ends[1]), 0.0), dtype=np.float64)
    net.add_straight("b", "c", bc_start, bc_start + [ends[2], 0], forbidden=True)
    net.finalize()
    return net


class BatchedMergeEnv(BatchedRoundaboutEnv):
    ENV_ID = "merge-v0"
    N_VEHICLES = 6  # five vehicles + the Obstacle
    EGO_SIDE_LANES = 2  # the controlled vehicle spawns on ("a", "b", 1): normalize_obs' default y-range (observation.py:214-226)
    REWARD_NAMES = ("collision_reward", "right_lane_reward", "high_speed_reward", "lane_change_reward", "merging_speed_reward")  # _rewards :62-77

    def _make_network(self) -> NetworkTable:
        return make_merge_network()

    def define_spaces(self) -> None:
        if self.reset_mode != "device":
            raise NotImplementedError("merge envs reset on the device (hwy_merge_reset)")
        cfg = self.config
        cfg.setdefault("normalize_reward", False)
        cfg.setdefault("duration", float("inf"))  # AbstractEnv has no duration; MergeEnv never truncates
        super().define_spaces()
        p = self._params
        p.reward_type = 2
        p.right_lane_reward = float(cfg["right_lane_reward"])
        p.merging_speed_reward = float(cfg["merging_speed_reward"])
        p.reward_speed_lo, p.reward_speed_hi = (float(v) for v in cfg["reward_speed_range"])
        p.merge_lane = self.net.index[("b", "c", 2)]
        p.duration = float("inf")

    def _build_spawn_tables(self) -> None:
        net = self.net
        s = N.HwyMergeSpawn()
        s.lane_ab[0], s.lane_ab[1] = net.index[("a", "b", 0)], net.index[("a", "b", 1)]
        s.lane_jk = net.index[("j", "k", 0)]
        ts = self.action_type.target_speeds
        s.ego_speed_index = int(np.clip(np.round((30.0 - ts[0]) / (ts[-1] - ts[0]) * (ts.size - 1)), 0, ts.size - 1))
        ox, oy = net.position(net.index[("b", "c", 2)], 80.0, 0.0)
        s.obstacle_x, s.obstacle_y = float(ox), float(oy)
        self._spawn_struct = s

    def _device_reset(self, mask_a, mask_b, obs_ptr) -> None:
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_merge_reset(
                C.byref(self._params), self._graph_dev.data_ptr(), C.byref(self._spawn_struct), C.byref(self._state),
                self._rng.data_ptr(), mask_a, mask_b, obs_ptr, self._stream()))


class BatchedConnectedLaneMergeEnv(BatchedMergeEnv):
    """`merge-v1`: ConnectedLaneNeighboursMixin (envs/common/abstract.py:26-37)."""

    ENV_ID = "merge-v1"
