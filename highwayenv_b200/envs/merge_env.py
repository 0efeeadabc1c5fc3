"""Batched merge-v0 / merge-v1 on the H100 backend.

Host-side mirror of the reference's ``MergeEnv`` (highway_env/envs/merge_env.py): a two-lane highway a->b->c->d
with an access ramp j->k (straight) ->b (sine) ->c (third, forbidden lane) that ends on an ``Obstacle``; the
controlled MDPVehicle, three IDM vehicles, and one merging IDM vehicle on the ramp.  Same kernels as roundabout-v0
(8 vehicle slots per env): the Obstacle occupies the slot after the five vehicles (kind 3: it never acts or moves,
is seen by the neighbour search, IDM and the Kinematics observation, and takes no impact of its own).  Reward
(:39-78) adds an altruistic penalty for slow vehicles on the merging lane; the episode ends on a crash or past
x = 370 and is never truncated (:80-84).

merge-generic-v0 / v1 (``MergeGenericEnv``, :193-379) run the same task on a road built from the config, with a
rejection-sampled traffic population, and reset on the device only; see ``BatchedMergeGenericEnv``.
"""
from __future__ import annotations

import numbers

import numpy as np

from .. import _native as N
from ..road.network import NetworkTable
from ..spaces import Box
from .common.action import speed_to_index
from .common.config_road import ConfigRoadMixin
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
            raise NotImplementedError("merge envs reset on the device")
        cfg = self.config
        cfg.setdefault("normalize_reward", False)
        cfg.setdefault("duration", float("inf"))  # AbstractEnv has no duration; MergeEnv never truncates
        super().define_spaces()
        p = self._params
        p.reward_type = 2
        p.right_lane_reward = float(cfg["right_lane_reward"])
        p.merging_speed_reward = float(cfg["merging_speed_reward"])
        p.reward_speed_lo, p.reward_speed_hi = (float(v) for v in cfg["reward_speed_range"])
        p.merge_lane = self.net.index.get(("b", "c", 2), -1)  # a one-lane generic merge has no such lane
        p.duration = float("inf")

    def _build_spawn_tables(self) -> None:
        net = self.net
        s = N.HwyMergeSpawn()
        s.lane_ab[0], s.lane_ab[1] = net.index[("a", "b", 0)], net.index[("a", "b", 1)]
        s.lane_jk = net.index[("j", "k", 0)]
        ts = self.action_type.target_speeds
        s.ego_speed_index = speed_to_index(ts, 30.0)
        ox, oy = net.position(net.index[("b", "c", 2)], 80.0, 0.0)
        s.obstacle_x, s.obstacle_y = float(ox), float(oy)
        self._scenario = N.HwyNetScenario(kind=N.HWY_SCENARIO_MERGE, u=N.HwyNetScenarioUnion(merge=s))


class BatchedConnectedLaneMergeEnv(BatchedMergeEnv):
    """`merge-v1`: ConnectedLaneNeighboursMixin (envs/common/abstract.py:26-37)."""

    ENV_ID = "merge-v1"


GENERIC_MAX_LANES = 9  # 3 lanes_count + 3 lanes: 10 would need 33 of the 32-lane table


def make_merge_generic_network(lanes: int = 2, pre: float = 150, conv: float = 80, par: float = 80,
                               after: float = 150) -> NetworkTable:
    """MergeGenericEnv._make_road (merge_env.py:238-318) with the reference's float64 expressions: three
    straight_road_network roads of `lanes` lanes at speed limit 30 (road/road.py:292-321), a->b over [0, pre + conv],
    b->c over [pre + conv, + par], c->d over [pre + conv + par, + after]; then the forbidden ramp at speed limit 30: j->k
    straight at y = 4 lanes + 6.5, k->b a sine lane, and lane `lanes` of b->c.  Table order a->b, b->c (lanes + 1 lanes),
    c->d, j->k, k->b: 3 lanes + 3 lanes."""
    if not 1 <= lanes <= GENERIC_MAX_LANES:
        raise ValueError(f"lanes must be in 1..{GENERIC_MAX_LANES}")
    net = NetworkTable()
    n, s, cl = 0, 1, 3  # LineType NONE, STRIPED, CONTINUOUS_LINE (road/lane.py:150-156)

    def lane(f, t, start, end, line_types, **kw):
        net.add_straight(f, t, start, end, speed_limit=30, **kw)
        net._graph[f][t][-1]["line_types"] = list(line_types)

    def straight_road(f, t, start, length):  # RoadNetwork.straight_road_network, angle 0
        for k in range(lanes):
            lane(f, t, [start, k * 4], [start + length, k * 4], (cl if k == 0 else s, cl if k == lanes - 1 else n))

    straight_road("a", "b", 0, pre + conv)
    straight_road("b", "c", pre + conv, par)
    straight_road("c", "d", pre + conv + par, after)
    amplitude = 3.25
    y_parallel = lanes * 4  # StraightLane.DEFAULT_WIDTH
    y_approach = y_parallel + 2 * amplitude
    lane("j", "k", [0, y_approach], [pre, y_approach], (cl, cl), forbidden=True)
    lane("k", "b", [pre, y_parallel + amplitude], [pre + conv, y_parallel + amplitude], (cl, cl), forbidden=True,
         sine=(amplitude, 2 * np.pi / (2 * conv), np.pi / 2))
    lane("b", "c", [pre + conv, y_parallel], [pre + conv + par, y_parallel], (s, cl), forbidden=True)
    net.finalize()
    return net


_GENERIC_NETS: dict = {}
MERGE_LENGTH_KEYS = ("before_merge_length", "converge_merge_length", "parallel_merge_length", "after_merge_length")


def merge_generic_network(lanes, pre, conv, par, after) -> NetworkTable:
    """The lane table of config["lanes_count"] and the four section lengths, cached per key."""
    key = (int(lanes), pre, conv, par, after)
    if key not in _GENERIC_NETS:
        _GENERIC_NETS[key] = make_merge_generic_network(*key)
    return _GENERIC_NETS[key]


def check_merge_generic(cfg: dict, env_id: str) -> None:
    """The generic merge's own keys: raises for what the reference cannot build or the kernels cannot hold."""
    lanes, count = cfg["lanes_count"], cfg["vehicles_count"]
    if isinstance(lanes, bool) or not isinstance(lanes, numbers.Integral):
        raise ValueError("lanes_count must be an integer (the reference raises TypeError in range(lanes_count))")
    if lanes < 1:
        raise ValueError("lanes_count must be >= 1 (the reference raises KeyError on the ego's lane)")
    if lanes > GENERIC_MAX_LANES:
        raise NotImplementedError(f"lanes_count > {GENERIC_MAX_LANES} on {env_id}: {3 * lanes + 3} lanes exceed the "
                                  f"{N.HWY_NET_MAX_LANES}-lane table")
    pre, conv, par, after = (cfg[k] for k in MERGE_LENGTH_KEYS)
    for v in (pre, conv, par, after):
        if isinstance(v, bool) or not isinstance(v, numbers.Real):
            raise ValueError("the merge section lengths must be numbers")
    if not all(v > 0 for v in (pre, conv, par)):
        raise ValueError("All road segments must have positive length")
    if not after >= 90:
        raise ValueError("The after merge road segment must have length >= 90")
    if isinstance(count, bool) or not isinstance(count, numbers.Integral):
        raise ValueError("vehicles_count must be an integer")
    if count > N.HWY_NET_GROUP_LARGE - 3:
        raise NotImplementedError(f"vehicles_count > {N.HWY_NET_GROUP_LARGE - 3} on {env_id}: the ego, its traffic, "
                                  f"the merging vehicle and the Obstacle fill at most {N.HWY_NET_GROUP_LARGE} slots")


class BatchedMergeGenericEnv(ConfigRoadMixin, BatchedMergeEnv):
    """`merge-generic-v0`: MergeGenericEnv (merge_env.py:193-375), MergeEnv's reward and dynamics on a road of
    config["lanes_count"] lanes (1..9) and four configurable section lengths, with config["vehicles_count"] traffic
    vehicles placed by rejection sampling (HWY_SCENARIO_MERGE with lanes_count > 0).  A vehicle whose 10 tries fail is
    skipped, so the population, and with it the Obstacle's slot (count - 1), varies per env.  The ego, up to 5 traffic
    vehicles, the merging vehicle and the Obstacle run on 8 slots; 6 to 29 traffic vehicles on 32 slots (the
    intersection family's step without rules or spawns).  Terminated past end_position = the road's length - 90.
    The lane table follows the config: reset(options={"config": ...}) rebuilds it and re-allocates."""

    ENV_ID = "merge-generic-v0"
    ROAD_KEYS = ("lanes_count",) + MERGE_LENGTH_KEYS

    def define_spaces(self) -> None:
        if self.reset_mode != "device":
            raise NotImplementedError(f"{self.ENV_ID} resets on the device")
        cfg = self.config
        check_merge_generic(cfg, self.ENV_ID)
        lanes = int(cfg["lanes_count"])
        self.EGO_SIDE_LANES = lanes  # the ego's road a->b has `lanes` side lanes: Kinematics y in +-4 lanes
        # the ego, the traffic, the merging vehicle and the Obstacle
        self._use_road(merge_generic_network(lanes, *(cfg[k] for k in MERGE_LENGTH_KEYS)),
                       1 + max(int(cfg["vehicles_count"]), 0) + 2)
        super().define_spaces()
        # end_position = pre + conv + par + after - 90 (:249): the c->d lanes end at x = (pre + conv + par) + after
        self._params.merge_end_lane = self.net.index[("c", "d", 0)]

    def _build_spawn_tables(self) -> None:
        net, cfg = self.net, self.config
        lanes = int(cfg["lanes_count"])
        s = N.HwyMergeSpawn()
        s.lane_ab[0], s.lane_ab[1] = net.index[("a", "b", 0)], net.index[("a", "b", min(1, lanes - 1))]
        s.lane_jk = net.index[("j", "k", 0)]
        s.ego_speed_index = speed_to_index(self.action_type.target_speeds, 30.0)
        ox, oy = net.position(net.index[("b", "c", lanes)], cfg["parallel_merge_length"], 0.0)  # lbc.position(par, 0)
        s.obstacle_x, s.obstacle_y = float(ox), float(oy)
        s.lanes_count, s.vehicles_count = lanes, int(cfg["vehicles_count"])
        s.max_position = cfg["before_merge_length"] + cfg["converge_merge_length"] + cfg["parallel_merge_length"]
        self._scenario = N.HwyNetScenario(kind=N.HWY_SCENARIO_MERGE, u=N.HwyNetScenarioUnion(merge=s))


class BatchedConnectedLaneMergeGenericEnv(BatchedMergeGenericEnv):
    """`merge-generic-v1`: ConnectedLaneNeighboursMixin over the generic merge."""

    ENV_ID = "merge-generic-v1"
