"""Batched racetrack-v0 / racetrack-v1, racetrack-large-v0 / v1 and racetrack-oval-v0 / v1 on the H100 backend.

Host-side mirror of the reference's ``RacetrackEnv`` (highway_env/envs/racetrack_env.py:15-425): a closed two-lane
track of 9 roads (straight and circular, width 5, speed limit 10), one controlled plain ``Vehicle`` steered through
``ContinuousAction`` (lateral, optionally longitudinal), an ``IDMVehicle`` ahead of it on ("b", "c") and up to
``other_vehicles - 1`` more on random lanes, each dropped when it spawns within 20 m of one already placed.  The
default observation is a 12 x 12 OccupancyGrid (presence, on_road) aligned with the vehicle, observed by the standalone
grid kernel; Kinematics is written by the step kernel itself.

Stepping runs in ``hwy_network_step`` with HWY_SCENARIO_RACETRACK (include/hwyb200.h) on the 8-slot network state:
the network kernels' substep with a plain ego, then the racetrack reward (:66-83), termination (crash, or off road with
``terminate_off_road``) and truncation at ``duration``.  Resets run in ``hwy_network_reset`` from each env's numpy
stream, in the reference's draw order (:374-425).  The plain Vehicle's action dict persists between steps
(kinematics.py:119-128): the state keeps it in the ego's (target_speed, timer) pair as (acceleration, steering), which
``road_substeps`` replays.

The large track (``RacetrackEnvLarge``, 9 roads x 3 lanes) and the oval (``RacetrackEnvOval``, 8 roads x ``no_lanes``)
run on the same kernels with their own lane tables; only the ego's lane draw differs (``HwyRacetrackParams.ego_lanes``).
"""
from __future__ import annotations

import numpy as np
import torch

from .. import _native as N
from ..road.network import NetworkTable
from ..spaces import Box, batch_space
from .common.action import ContinuousAction
from .common.observation import KinematicObservation, OccupancyGridObservation, select_network_observation
from .common.vector_env import BatchedNetworkEnv

# LineType (road/lane.py:12-20): NONE 0, STRIPED 1, CONTINUOUS 2
_N, _S, _C = 0, 1, 2


def make_racetrack_network() -> NetworkTable:
    """RacetrackEnv._make_road (racetrack_env.py:94-358), lanes in the reference's insertion order.  Some arcs end at
    different angles on their two lanes (136 / 137 deg, 170 / 165 deg, 56 / 58 deg, 240-270 / 238-268 deg); they are
    copied as they are."""
    net = NetworkTable()
    d = np.deg2rad

    def straight(f, t, start, end, lt):
        net.add_straight(f, t, start, end, width=5, speed_limit=10.0)
        net._graph[f][t][-1]["line_types"] = list(lt)

    def arc(f, t, center, radius, a0, a1, clockwise, lt):
        net.add_circular(f, t, center, radius, d(a0), d(a1), clockwise=clockwise, width=5, speed_limit=10.0)
        net._graph[f][t][-1]["line_types"] = list(lt)

    straight("a", "b", [42, 0], [100, 0], (_C, _S))
    straight("a", "b", [42, 5], [100, 5], (_S, _C))
    arc("b", "c", [100, -20], 20, 90, -1, False, (_C, _N))
    arc("b", "c", [100, -20], 20 + 5, 90, -1, False, (_S, _C))
    straight("c", "d", [120, -20], [120, -30], (_C, _N))
    straight("c", "d", [125, -20], [125, -30], (_S, _C))
    arc("d", "e", [105, -30], 15, 0, -181, False, (_C, _N))
    arc("d", "e", [105, -30], 15 + 5, 0, -181, False, (_S, _C))
    arc("e", "f", [70, -30], 15 + 5, 0, 136, True, (_C, _S))
    arc("e", "f", [70, -30], 15, 0, 137, True, (_N, _C))
    straight("f", "g", [55.7, -15.7], [35.7, -35.7], (_C, _N))
    straight("f", "g", [59.3934, -19.2], [39.3934, -39.2], (_S, _C))
    arc("g", "h", [18.1, -18.1], 25, 315, 170, False, (_C, _N))
    arc("g", "h", [18.1, -18.1], 25 + 5, 315, 165, False, (_S, _C))
    arc("h", "i", [18.1, -18.1], 25, 170, 56, False, (_C, _N))
    arc("h", "i", [18.1, -18.1], 25 + 5, 170, 58, False, (_S, _C))
    arc("i", "a", [43.2, 23.4], 18.5 + 5, 240, 270, True, (_C, _S))
    arc("i", "a", [43.2, 23.4], 18.5, 238, 268, True, (_N, _C))
    net.finalize()
    return net


def make_racetrack_large_network(speed_limit: float = 10.0) -> NetworkTable:
    """RacetrackEnvLarge._make_road (racetrack_env.py:439-875): 9 roads x 3 lanes, width 5, every lane at
    config["speed_limit"], lanes in the reference's insertion order.  The end points of the slants and the arc centres
    are computed with the reference's float64 expressions, in its order.  Some arcs end at different angles on their
    lanes (136 / 137 / 137 deg, 202 / 205 / 205 deg, 210-88 / 210-90 / 212-88 deg); they are copied as they are."""
    net = NetworkTable()
    d = np.deg2rad
    w, w2 = 5, 10

    def straight(f, t, start, end, lt):
        net.add_straight(f, t, start, end, width=w, speed_limit=speed_limit)
        net._graph[f][t][-1]["line_types"] = list(lt)

    def arc(f, t, center, radius, a0, a1, lt, clockwise=False):
        net.add_circular(f, t, center, radius, d(a0), d(a1), clockwise=clockwise, width=w, speed_limit=speed_limit)
        net._graph[f][t][-1]["line_types"] = list(lt)

    straight("a", "b", [42, 0], [200, 0], (_C, _S))
    straight("a", "b", [42, w], [200, w], (_S, _S))
    straight("a", "b", [42, w2], [200, w2], (_N, _C))
    arc("b", "c", [200, -20], 20, 90, -1, (_C, _N))
    arc("b", "c", [200, -20], 20 + w, 90, -1, (_S, _S))
    arc("b", "c", [200, -20], 20 + w2, 90, -1, (_N, _C))
    straight("c", "d", [220, -20], [220, -60 + -1.0], (_C, _N))
    straight("c", "d", [220 + w, -20], [220 + w, -60 + -1.0], (_S, _S))
    straight("c", "d", [220 + w2, -20], [220 + w2, -60 + -1.0], (_N, _C))
    arc("d", "e", [205, -60], 15, 0, -181, (_C, _N))
    arc("d", "e", [205, -60], 15 + w, 0, -181, (_S, _S))
    arc("d", "e", [205, -60], 15 + w2, 0, -181, (_N, _C))
    arc("e", "f", [170, -60], 15 + 5, 0, 136, (_C, _N), clockwise=True)
    arc("e", "f", [170, -60], 15, 0, 137, (_S, _S), clockwise=True)
    arc("e", "f", [170, -60], 15 - w, 0, 137, (_N, _C), clockwise=True)
    extend = np.array([-30, -30])
    start6, end6 = np.array([155.7, -45.7]), np.array([135.7, -65.7]) + extend
    start6_2, end6_2 = np.array([159.3934, -49.2]), np.array([139.3934, -69.2]) + extend
    start6_3 = np.array([start6[0] + 2 * (start6_2[0] - start6[0]), start6[1] + 2 * (start6_2[1] - start6[1])])
    end6_3 = np.array([end6[0] + 2 * (end6_2[0] - end6[0]), end6[1] + 2 * (end6_2[1] - end6[1])])
    straight("f", "g", start6, end6, (_C, _N))
    straight("f", "g", start6_2, end6_2, (_S, _S))
    straight("f", "g", start6_3, end6_3, (_N, _C))
    center7, r7, theta7, theta7_end = np.array([118.1, -48.1]) + extend, 25, 317, 205
    arc("g", "h", center7, r7, theta7, theta7_end - 3, (_C, _N))
    arc("g", "h", center7, r7 + 5, theta7, theta7_end, (_S, _S))
    arc("g", "h", center7, r7 + w2, theta7, theta7_end, (_N, _C))
    r9, rad = 15, d(30)
    starts8 = [np.array([center7[0] + r * np.cos(d(theta7_end)), center7[1] + r * np.sin(d(theta7_end))])
               for r in (r7, r7 + w, r7 + w2)]
    ends8 = [np.array([42 - r * np.cos(rad), -r9 - r * np.sin(rad)]) for r in (r9, r9 + w, r9 + w2)]
    straight("h", "i", starts8[0], ends8[0], (_C, _N))
    straight("h", "i", starts8[1], ends8[1], (_S, _S))
    straight("h", "i", starts8[2], ends8[2], (_N, _C))
    center9 = np.array([42, -r9])
    arc("i", "a", center9, r9, 210, 88, (_C, _N))
    arc("i", "a", center9, r9 + w, 210, 90, (_S, _S))
    arc("i", "a", center9, r9 + w2, 212, 88, (_N, _C))
    net.finalize()
    return net


OVAL_MAX_LANES = 4  # 8 roads x 4 lanes fill the 32-lane table


def make_racetrack_oval_network(length: float = 100, no_lanes: int = 3) -> NetworkTable:
    """RacetrackEnvOval._make_road (racetrack_env.py:936-1337) for a given `length` of the horizontal straights and
    `no_lanes` lanes per road: 8 roads, width 5, speed limit 10, lanes in the reference's insertion order (the inner
    lane, the middle lanes outwards, the outer lane).  The roadblock obstacles are not part of the network."""
    if not 2 <= no_lanes <= OVAL_MAX_LANES:
        raise ValueError(f"no_lanes must be in 2..{OVAL_MAX_LANES}")
    net = NetworkTable()
    d = np.deg2rad
    n = no_lanes

    def lane_types(inner, middle):
        return [inner] + [middle] * (n - 2) + [(_S, _C)]  # the inner lane, the middle lanes, the outer lane

    def straights(f, t, ends, lts):
        for (start, end), lt in zip(ends, lts):
            net.add_straight(f, t, start, end, width=5, speed_limit=10.0)
            net._graph[f][t][-1]["line_types"] = list(lt)

    def arcs(f, t, center, radius, a0, a1, lts):
        for i, lt in enumerate(lts):
            net.add_circular(f, t, center, radius + i * 5, d(a0), d(a1), clockwise=False, width=5, speed_limit=10.0)
            net._graph[f][t][-1]["line_types"] = list(lt)

    turn, side = lane_types((_C, _N), (_S, _N)), range(n)
    straights("a", "b", [([0, i * 5], [length + 1, i * 5]) for i in side], lane_types((_C, _S), (_S, _N)))
    arcs("b", "c", [length, -20], 20, 90, 0, turn)
    straights("c", "d", [([length + 20 + i * 5, -20], [length + 20 + i * 5, -50]) for i in side], turn)
    arcs("d", "e", [length + 5, -50], 15, 0, -90, turn)
    straights("e", "f", [([length + 5, -(65 + i * 5)], [-5, -(65 + i * 5)]) for i in side], turn)
    arcs("f", "g", [-5, -50], 15, -90, -180, turn)
    straights("g", "h", [([-20 - i * 5, -50], [-20 - i * 5, -20]) for i in side], turn)
    arcs("h", "a", [0, -20], 20, 180, 90, lane_types((_C, _N), (_S, _C)))  # its middle lanes: (STRIPED, CONTINUOUS)
    net.finalize()
    return net


_HOST_NETS: dict = {}


def track_network(env_id: str, cfg: dict) -> NetworkTable:
    """The lane table of `env_id` under `cfg` (cached per track): racetrack-v0 / v1, the large track at
    config["speed_limit"], or the oval of config["length"] and config["no_lanes"] (already checked)."""
    base = env_id.rsplit("-", 1)[0]
    if base == "racetrack-large":
        key = (base, float(cfg["speed_limit"]))
    elif base == "racetrack-oval":
        key = (base, cfg["length"], int(cfg["no_lanes"]))
    else:
        key = ("racetrack",)
    if key not in _HOST_NETS:
        if key[0] == "racetrack-large":
            _HOST_NETS[key] = make_racetrack_large_network(key[1])
        elif key[0] == "racetrack-oval":
            _HOST_NETS[key] = make_racetrack_oval_network(key[1], key[2])
        else:
            _HOST_NETS[key] = make_racetrack_network()
    return _HOST_NETS[key]


def _check_oval(cfg: dict, env_id: str) -> None:
    """The oval's own keys (RacetrackEnvOval.default_config, :894-934) that the accelerated path does not run."""
    length, no_lanes = cfg["length"], cfg["no_lanes"]
    if no_lanes == 0 or length == 0:
        raise NotImplementedError(f"random length / no_lanes (0) on {env_id}: the reference draws them from an "
                                  "unseeded np.random.default_rng(), which no seed reproduces")
    if isinstance(no_lanes, bool) or int(no_lanes) != no_lanes or no_lanes < 0:
        raise ValueError("no_lanes must be a non-negative integer")
    if no_lanes > OVAL_MAX_LANES:
        raise NotImplementedError(f"no_lanes > {OVAL_MAX_LANES} on {env_id}: 8 roads x {no_lanes} lanes exceed the "
                                  f"{N.HWY_NET_MAX_LANES}-lane table")
    if no_lanes == 1:
        raise ValueError("no_lanes 1: the reference builds the inner and the outer lane on the same line")
    if isinstance(length, bool) or not np.isfinite(float(length)) or length < 0:
        raise ValueError("length must be a positive number")
    for key in ("block_lane", "force_decision"):
        if cfg.get(key, False):
            raise NotImplementedError(f"{key}=True on {env_id}: its Obstacles do not fit the 8-slot state")


def racetrack_params(cfg: dict, env_id: str = "racetrack-v0") -> dict:
    """The kernel parameters of a racetrack config (HwyNetParams, HwyRacetrackParams) and its action / observation
    plugins; raises for what the accelerated path does not run, before anything touches the device.  `env_id` picks
    the track: racetrack-v0 / v1, racetrack-large-v0 / v1 or racetrack-oval-v0 / v1."""
    oval = env_id.startswith("racetrack-oval")
    if oval:
        _check_oval(cfg, env_id)
    act, obs = cfg["action"], cfg["observation"]
    if act["type"] != "ContinuousAction":
        raise NotImplementedError(f"action type {act['type']!r} on {env_id} (ContinuousAction only)")
    if int(cfg["controlled_vehicles"]) != 1:
        raise NotImplementedError(f"controlled_vehicles > 1 on {env_id}")
    if obs["type"] not in ("OccupancyGrid", "Kinematics"):
        raise NotImplementedError(f"observation type {obs['type']!r} on {env_id} (OccupancyGrid, Kinematics)")
    other = int(cfg["other_vehicles"])
    if other > N.HWY_NET_GROUP - 1:
        raise NotImplementedError(f"other_vehicles > {N.HWY_NET_GROUP - 1}: 8 slots hold the ego, the front "
                                  "vehicle and at most 6 more")
    if other < 0:
        raise ValueError("other_vehicles must be >= 0")
    longi, lat = bool(act.get("longitudinal", True)), bool(act.get("lateral", True))
    if not (longi or lat):
        raise ValueError("Either longitudinal and/or lateral control must be enabled")
    if act.get("dynamical", False):
        raise NotImplementedError(f"dynamical=True (BicycleVehicle) on {env_id}")
    # ContinuousAction checks the remaining keywords; it stands for the two-axis form the kernel reads
    at = ContinuousAction(**dict(act, longitudinal=True, lateral=True))
    action_size = 2 if longi and lat else 1
    V = other + 1 if other > 0 else 1  # ego, front vehicle, integers(other_vehicles) < other_vehicles more
    p = N.HwyNetParams()
    p.n_vehicles = V
    p.simulation_frequency, p.policy_frequency = int(cfg["simulation_frequency"]), int(cfg["policy_frequency"])
    ts = np.array(act.get("target_speeds") or [0, 5, 10], dtype=np.float64)[:3]
    p.n_target_speeds = int(ts.size)
    for k, t in enumerate(ts):
        p.target_speeds[k] = float(t)
    # the kernel reads (throttle, steering) pairs; a missing axis is staged as 0 and maps to exactly 0 through the
    # range (0, 0): 0 + ((0 - -1) * 0) / 2 = +0.0 in float32
    p.action_type, p.act_clip, p.dynamical = 1, int(at.clip), 0
    p.acc_lo, p.acc_hi = (float(at.acceleration_range[0]), float(at.acceleration_range[1])) if longi else (0.0, 0.0)
    p.steer_lo, p.steer_hi = (float(at.steering_range[0]), float(at.steering_range[1])) if lat else (0.0, 0.0)
    net = track_network(env_id, cfg)
    # Kinematics' default y range spans all_side_lanes of the ego's spawn road ("a","b"): 2 lanes on racetrack-v0,
    # 3 on the large track, no_lanes on the oval
    ab_lanes = net.lanes[net.index[("a", "b", 0)]]["road_count"]
    plugin, fused = select_network_observation(None, p, obs, ts, ab_lanes, fuse_ttc=False, fuse_grid=False,
                                               feature_columns=True)
    assert isinstance(plugin, (KinematicObservation, OccupancyGridObservation))
    p.duration = float(cfg["duration"])
    p.collision_reward = float(cfg["collision_reward"])
    # IDMVehicle class constants (vehicle/behavior.py:21-46)
    p.acc_max, p.comfort_acc_max, p.comfort_acc_min = 6.0, 3.0, -5.0
    p.distance_wanted, p.time_wanted = 10.0, 1.5
    p.politeness, p.lane_change_min_acc_gain = 0.0, 0.2
    p.lane_change_max_braking_imposed, p.lane_change_delay = 2.0, 1.0
    p.perception_distance = 200.0
    p.connected_lanes = int(bool(cfg.get("neighbour_vehicles_connected_lanes", False)))
    rp = N.HwyRacetrackParams()
    rp.other_vehicles = other
    rp.terminate_off_road = int(bool(cfg["terminate_off_road"]))
    rp.lane_ab, rp.lane_bc = net.index[("a", "b", 0)], net.index[("b", "c", 0)]
    rp.n_from_nodes = len(net._graph)
    # the ego's lane draw: integers(2) in RacetrackEnv._make_vehicles (also the large track's), integers(no_lanes) in
    # the oval's; the front vehicle takes the same lane id on ("b","c")
    rp.ego_lanes = int(cfg["no_lanes"]) if oval else 2
    # the reset cannot read the device table; the lane ids it draws must exist on both roads
    if rp.ego_lanes > min(net.lanes[rp.lane_ab]["road_count"], net.lanes[rp.lane_bc]["road_count"]):
        raise ValueError(f"ego_lanes {rp.ego_lanes} exceeds the lanes of ('a','b') or ('b','c') on {env_id}")
    rp.lane_centering_cost = float(cfg["lane_centering_cost"])
    rp.lane_centering_reward = float(cfg["lane_centering_reward"])
    rp.action_reward = float(cfg["action_reward"])
    rp.collision_reward = float(cfg["collision_reward"])
    rp.on_road_reward = float(cfg.get("on_road_reward", 0))
    return dict(params=p, race=rp, action_type=at, observation_type=plugin, fused=fused, lateral=lat,
                action_size=action_size, V=V, net=net)


class BatchedRacetrackEnv(BatchedNetworkEnv):
    ENV_ID = "racetrack-v0"
    # _rewards (:72-83), in the reference's order
    REWARD_NAMES = ("lane_centering_reward", "action_reward", "collision_reward", "on_road_reward")
    META_FLAGS = ("crashed", "has_impact", "check_collisions")
    ROW_EXCLUDE = BatchedNetworkEnv.ROW_EXCLUDE | {"_pair_buf"}  # staging, rewritten by every step

    def _make_network(self) -> NetworkTable:
        return self._track

    @property
    def _race(self) -> N.HwyRacetrackParams:
        """The scenario's racetrack parameters, a view into `_scenario`: writes reach the kernels."""
        return self._scenario.u.racetrack

    # ------------------------------------------------------------------ configuration
    def define_spaces(self) -> None:
        if self.reset_mode != "device":
            raise NotImplementedError(f"{self.ENV_ID} resets on the device")
        spec = racetrack_params(self.config, self.ENV_ID)
        # the lane table follows the config (the oval's length / no_lanes, the large track's speed_limit): after
        # reset(options={"config": ...}) picks another track, `net` rebuilds the table and its device copy
        if self._net is not spec["net"]:
            self._net = None
        self._track = spec["net"]
        self._params = spec["params"]
        self._scenario = N.HwyNetScenario(kind=N.HWY_SCENARIO_RACETRACK,
                                          u=N.HwyNetScenarioUnion(racetrack=spec["race"]))
        self.action_type, self.observation_type = spec["action_type"], spec["observation_type"]
        self.lateral, self.action_size, self.V = spec["lateral"], spec["action_size"], spec["V"]
        self._plugin_standalone = not spec["fused"]
        self.single_observation_space = self.observation_type.space()
        self.single_action_space = Box(-1.0, 1.0, shape=(self.action_size,), dtype=np.float32)
        self.observation_space = batch_space(self.single_observation_space, self.num_envs)
        self.action_space = batch_space(self.single_action_space, self.num_envs)
        self.obs_shape = tuple(self.single_observation_space.shape)

    def _allocate(self) -> None:
        n = self.num_envs
        self.net  # the lane table on the device (_graph_dev)
        st = self._allocate_network_state(N.HWY_NET_GROUP)
        self._count = torch.zeros(n, dtype=torch.int32, device=self.device)
        st.count = self._count.data_ptr()
        # the actions as passed [N, action_size]; with one control axis, the (throttle, steering) pairs the kernel reads
        self._action_buf = torch.zeros(n, self.action_size, dtype=torch.float32, device=self.device)
        self._pair_buf = None if self.action_size == 2 else torch.zeros(n, 2, dtype=torch.float32, device=self.device)

    # ------------------------------------------------------------------ actions
    def _stage_actions(self, actions) -> torch.Tensor:
        act = super()._stage_actions(actions)
        if self._pair_buf is not None:  # one control axis: the other stays 0
            self._pair_buf[:, 1 if self.lateral else 0].copy_(act[:, 0])
        return act

    def to_finite_mdp(self):
        raise NotImplementedError(f"to_finite_mdp on {self.ENV_ID}: the finite MDP needs DiscreteMetaAction")

    def get_available_actions(self):
        raise NotImplementedError(f"get_available_actions on {self.ENV_ID}: ContinuousAction has no discrete actions")

    def copy_envs(self, dst_ids, src_ids, source=None) -> None:
        """BatchedVectorEnv.copy_envs; two envs of one class may still run different tracks (the oval's length /
        no_lanes, the large track's speed_limit), and a state only means something on its own lane table."""
        if source is not None and type(source) is type(self) and source._track is not self._track:
            raise ValueError(f"copy_envs between {self.ENV_ID} envs on different tracks (length, no_lanes or "
                             "speed_limit)")
        super().copy_envs(dst_ids, src_ids, source)

    # ------------------------------------------------------------------ state import / export
    def _env_rows(self) -> dict:
        rows = super()._env_rows()
        rows["_count"] = self._count
        return rows

    def state_dict(self) -> dict:
        """The per-vehicle fields [N, V]; `count` vehicles of each env are on the road.  The ego's target_speed /
        timer hold its persisting (acceleration, steering) action."""
        sd = super().state_dict()
        del sd["rng"]  # per-env fields only; the streams are rng_words()
        sd["count"] = self._count.cpu().numpy()
        return sd

    def load_state_dict(self, sd: dict, env_ids=None) -> None:
        super().load_state_dict(sd, env_ids)
        idx = slice(None) if env_ids is None else torch.from_numpy(np.asarray(env_ids, dtype=np.int64)).to(self.device)
        self._count[idx] = torch.from_numpy(np.asarray(sd["count"], dtype=np.int32).reshape(-1)).to(self.device)
        self._route_len[idx] = 0


class BatchedConnectedLaneRacetrackEnv(BatchedRacetrackEnv):
    """`racetrack-v1`: ConnectedLaneNeighboursMixin (envs/common/abstract.py:26-37)."""

    ENV_ID = "racetrack-v1"


class BatchedRacetrackLargeEnv(BatchedRacetrackEnv):
    """`racetrack-large-v0`: RacetrackEnvLarge (racetrack_env.py:432-875), the three-lane track of 27 lanes with
    RacetrackEnv's config, rules and _make_vehicles (the ego on ("a","b",integers(2)))."""

    ENV_ID = "racetrack-large-v0"


class BatchedConnectedLaneRacetrackLargeEnv(BatchedRacetrackLargeEnv):
    """`racetrack-large-v1`: ConnectedLaneNeighboursMixin over the large track."""

    ENV_ID = "racetrack-large-v1"


class BatchedRacetrackOvalEnv(BatchedRacetrackEnv):
    """`racetrack-oval-v0`: RacetrackEnvOval (racetrack_env.py:882-1392), an oval of 8 roads x config["no_lanes"] lanes
    (2..4) with horizontal straights of config["length"]; the ego on ("a","b",integers(no_lanes)).  Random length /
    no_lanes (0) and the block_lane / force_decision obstacles raise."""

    ENV_ID = "racetrack-oval-v0"



class BatchedConnectedLaneRacetrackOvalEnv(BatchedRacetrackOvalEnv):
    """`racetrack-oval-v1`: ConnectedLaneNeighboursMixin over the oval."""

    ENV_ID = "racetrack-oval-v1"
