"""Batched roundabout-v0 on the H100 backend.

Host-side mirror of the reference's ``RoundaboutEnv`` (highway_env/envs/roundabout_env.py:12-391):
same config dictionary, road geometry and spawn procedure; stepping runs in
``hwy_network_step`` (include/hwyb200.h) for ``num_envs`` independent roundabouts.

Every env owns the numpy ``Generator(PCG64)`` stream a reference env seeded with
``seed + env_index_offset + i`` would own; ``_make_vehicles`` draws from it in the reference's
order (normal, normal, choice, uniform per traffic vehicle).  Two reset modes:

* ``reset_mode="device"`` (default): ``hwy_roundabout_reset`` re-spawns on the GPU from the stream
  (PCG64 + numpy's ziggurat normal restated on the device).  Draws, lanes and routes are identical
  to the reference; spawn coordinates go through CUDA's sin/cos instead of numpy's and may differ
  in the last ulp (~1e-15 m).  SameStep autoreset stays on the device.
* ``reset_mode="host"``: the spawn is rebuilt with numpy (bit-identical to the reference) and
  uploaded; autoreset round-trips through the host.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .. import _native as N
from ..road.network import NetworkTable
from ..spaces import Discrete, batch_space
from .common.action import DiscreteMetaAction, speed_to_index
from .common.observation import select_network_observation
from .common.vector_env import BatchedNetworkEnv


def make_roundabout_network() -> NetworkTable:
    """RoundaboutEnv._make_road (roundabout_env.py:77-315): two rings of 8 circular arcs
    (radii 20 / 24 m), and per branch a straight access road, a sine entry and a sine exit."""
    net = NetworkTable()
    center, radius, alpha = [0, 0], 20, 24
    radii = [radius, radius + 4]
    # (from, to, start angle [deg], end angle [deg]) in the reference's insertion order
    arcs = [
        ("se", "ex", 90 - alpha, alpha), ("ex", "ee", alpha, -alpha), ("ee", "nx", -alpha, -90 + alpha),
        ("nx", "ne", -90 + alpha, -90 - alpha), ("ne", "wx", -90 - alpha, -180 + alpha),
        ("wx", "we", -180 + alpha, -180 - alpha), ("we", "sx", 180 - alpha, 90 + alpha),
        ("sx", "se", 90 + alpha, 90 - alpha),
    ]
    for lane in (0, 1):
        for f, t, a0, a1 in arcs:
            net.add_circular(f, t, center, radii[lane], np.deg2rad(a0), np.deg2rad(a1), clockwise=False)
    access, dev, a = 170, 85, 5
    delta_st = 0.2 * dev
    delta_en = dev - delta_st
    w = 2 * np.pi / dev
    ph_in, ph_out = -np.pi / 2, -np.pi / 2 + w * delta_en
    # south
    net.add_straight("ser", "ses", [2, access], [2, dev / 2])
    net.add_straight("ses", "se", [2 + a, dev / 2], [2 + a, dev / 2 - delta_st], sine=(a, w, ph_in))
    net.add_straight("sx", "sxs", [-2 - a, -dev / 2 + delta_en], [-2 - a, dev / 2], sine=(a, w, ph_out))
    net.add_straight("sxs", "sxr", [-2, dev / 2], [-2, access])
    # east
    net.add_straight("eer", "ees", [access, -2], [dev / 2, -2])
    net.add_straight("ees", "ee", [dev / 2, -2 - a], [dev / 2 - delta_st, -2 - a], sine=(a, w, ph_in))
    net.add_straight("ex", "exs", [-dev / 2 + delta_en, 2 + a], [dev / 2, 2 + a], sine=(a, w, ph_out))
    net.add_straight("exs", "exr", [dev / 2, 2], [access, 2])
    # north
    net.add_straight("ner", "nes", [-2, -access], [-2, -dev / 2])
    net.add_straight("nes", "ne", [-2 - a, -dev / 2], [-2 - a, -dev / 2 + delta_st], sine=(a, w, ph_in))
    net.add_straight("nx", "nxs", [2 + a, dev / 2 - delta_en], [2 + a, -dev / 2], sine=(a, w, ph_out))
    net.add_straight("nxs", "nxr", [2, -dev / 2], [2, -access])
    # west
    net.add_straight("wer", "wes", [-access, 2], [-dev / 2, 2])
    net.add_straight("wes", "we", [-dev / 2, 2 + a], [-dev / 2 + delta_st, 2 + a], sine=(a, w, ph_in))
    net.add_straight("wx", "wxs", [dev / 2 - delta_en, -2 - a], [-dev / 2, -2 - a], sine=(a, w, ph_out))
    net.add_straight("wxs", "wxr", [-dev / 2, -2], [-access, -2])
    net.finalize()
    return net


class RoundaboutSpawner:
    """RoundaboutEnv._make_vehicles (roundabout_env.py:317-391) with numpy, for a list of per-env
    generators (CPU only; testable without a GPU)."""

    N_VEHICLES = 5
    DESTINATIONS = ["exr", "sxr", "nxr"]  # roundabout_env.py:345

    def __init__(self, net: NetworkTable, config: dict, target_speeds: np.ndarray) -> None:
        self.net, self.config, self.target_speeds = net, config, np.asarray(target_speeds, dtype=np.float64)
        # plan_route_to of every (closest lane at spawn, destination) pair; "nxs" is the controlled vehicle's
        self.routes, self.route_lens = net.route_table(self.DESTINATIONS + ["nxs"])

    def spawn(self, rngs) -> dict:
        net, m, V = self.net, len(rngs), self.N_VEHICLES
        position_deviation = speed_deviation = 2.0
        fixed_dest = self.config["incoming_vehicle_destination"]
        # per-env draws, in the reference's order: for each of the 4 traffic vehicles
        # normal (longitudinal), normal (speed), choice(destinations), uniform (DELTA)
        lon = np.zeros((m, 4))
        spd = np.zeros((m, 4))
        dest = np.zeros((m, 4), dtype=np.int64)
        delta = np.zeros((m, 4))
        base_lon = [5.0, 20.0 * float(1), 20.0 * float(-1), 50.0]
        for k, g in enumerate(rngs):
            for j in range(4):
                lon[k, j] = base_lon[j] + g.normal() * position_deviation
                spd[k, j] = 16.0 + g.normal() * speed_deviation if j else 16 + g.normal() * speed_deviation
                if j == 0 and fixed_dest is not None:
                    dest[k, j] = int(fixed_dest)
                else:
                    dest[k, j] = self.DESTINATIONS.index(str(g.choice(self.DESTINATIONS)))
                delta[k, j] = g.uniform(low=3.5, high=4.5)  # randomize_behavior, behavior.py:66-69
        spawn_lane = [net.index[("we", "sx", 1)], net.index[("we", "sx", 0)], net.index[("we", "sx", 0)],
                      net.index[("eer", "ees", 0)]]
        x, y, h, v = (np.zeros((m, V)) for _ in range(4))
        ego_lane = net.index[("ser", "ses", 0)]
        ex, ey = net.position(ego_lane, 125.0, 0.0)
        x[:, 0], y[:, 0], h[:, 0], v[:, 0] = ex, ey, net.heading_at(ego_lane, 140.0), 8.0
        for j in range(4):
            px, py = net.position(spawn_lane[j], lon[:, j], 0.0)  # make_on_lane, objects.py:68-90
            x[:, j + 1], y[:, j + 1] = px, py
            h[:, j + 1] = net.heading_at(spawn_lane[j], lon[:, j])
            v[:, j + 1] = spd[:, j]
        lane = np.stack([net.closest_lane(x[:, c], y[:, c], h[:, c]) for c in range(V)], axis=1)
        route = np.zeros((m, V, N.HWY_NET_MAX_ROUTE), dtype=np.int32)
        route_len = np.zeros((m, V), dtype=np.int32)
        for k in range(m):
            route[k, 0], route_len[k, 0] = self.routes[lane[k, 0], 3], self.route_lens[lane[k, 0], 3]
            for j in range(4):
                route[k, j + 1] = self.routes[lane[k, j + 1], dest[k, j]]
                route_len[k, j + 1] = self.route_lens[lane[k, j + 1], dest[k, j]]
        ts = self.target_speeds
        si = speed_to_index(ts, 8.0)
        target_speed = v.copy()
        target_speed[:, 0] = ts[si]
        timer = ((x + y) * np.pi) % 1.0  # IDMVehicle.__init__, behavior.py:64
        timer[:, 0] = 0.0
        dl = np.full((m, V), 4.0)
        dl[:, 1:] = delta
        kind = np.zeros((m, V), dtype=np.int64)
        kind[:, 0] = N.KIND_MDP
        return dict(x=x, y=y, heading=h, speed=v, target_speed=target_speed, timer=timer, delta=dl, lane=lane,
                    target_lane=lane.copy(), kind=kind, route=route, route_len=route_len,
                    speed_index=np.full(m, si, dtype=np.int32))



class BatchedRoundaboutEnv(BatchedNetworkEnv):
    ENV_ID = "roundabout-v0"
    N_VEHICLES = 5
    EGO_SIDE_LANES = 1  # lanes of the road the controlled vehicle spawns on (default Kinematics y-range)
    REWARD_NAMES = ("collision_reward", "high_speed_reward", "lane_change_reward", "on_road_reward")  # _rewards :58-65
    META_FLAGS = ("crashed", "no_lane_change", "has_impact", "check_collisions")
    RESET_ENTRY = "hwy_roundabout_reset"  # the scenario's reset kernel (same arguments for every roundabout-family env)

    def _make_network(self) -> NetworkTable:
        return make_roundabout_network()

    # ------------------------------------------------------------------ configuration
    def define_spaces(self) -> None:
        cfg = self.config
        act = cfg["action"]
        if act["type"] != "DiscreteMetaAction":
            if act["type"] in ("ContinuousAction", "DiscreteAction", "MultiAgentAction"):
                raise NotImplementedError(f"action type {act['type']!r} on roundabout-v0")
            raise ValueError("Unknown action type")
        self.action_type = DiscreteMetaAction(**act)
        if self.action_type.target_speeds.size > 3:
            raise NotImplementedError("more than 3 target speeds on the network kernels")
        p = N.HwyNetParams()
        p.n_vehicles = self.N_VEHICLES
        p.simulation_frequency = int(cfg["simulation_frequency"])
        p.policy_frequency = int(cfg["policy_frequency"])
        p.n_target_speeds = int(self.action_type.target_speeds.size)
        for k, t in enumerate(self.action_type.target_speeds):
            p.target_speeds[k] = float(t)
        self.observation_type, fused = select_network_observation(
            self, p, cfg["observation"], self.action_type.target_speeds, self.EGO_SIDE_LANES)
        self._plugin_standalone = not fused
        self.single_observation_space = self.observation_type.space()
        p.normalize_reward = int(bool(cfg["normalize_reward"]))
        p.duration = float(cfg["duration"])
        p.collision_reward = float(cfg["collision_reward"])
        p.high_speed_reward = float(cfg["high_speed_reward"])
        p.lane_change_reward = float(cfg["lane_change_reward"])
        p.acc_max, p.comfort_acc_max, p.comfort_acc_min = 6.0, 3.0, -5.0  # behavior.py:21-46
        p.distance_wanted, p.time_wanted = 10.0, 1.5
        p.politeness, p.lane_change_min_acc_gain = 0.0, 0.2
        p.lane_change_max_braking_imposed, p.lane_change_delay = 2.0, 1.0
        p.perception_distance = 200.0
        p.connected_lanes = int(bool(cfg.get("neighbour_vehicles_connected_lanes", False)))
        self._params = p
        self.single_action_space = Discrete(5)
        self.observation_space = batch_space(self.single_observation_space, self.num_envs)
        self.action_space = batch_space(self.single_action_space, self.num_envs)
        self.obs_shape = tuple(self.single_observation_space.shape)

    def _allocate(self) -> None:
        n, vp = self.num_envs, self.SLOTS
        self.V = self.N_VEHICLES
        st = self._allocate_network_state(vp)
        self._action_buf = torch.zeros(n, dtype=torch.int32, device=self.device)
        if vp == N.HWY_NET_GROUP_LARGE:  # the 32-slot kernels read the population and RegulatedRoad.steps from the state
            self._count = torch.full((n,), self.N_VEHICLES, dtype=torch.int32, device=self.device)
            self._road_steps = torch.zeros(n, dtype=torch.int32, device=self.device)
            st.count, st.road_steps = self._count.data_ptr(), self._road_steps.data_ptr()
        self._build_spawn_tables()

    def _build_spawn_tables(self) -> None:
        """Host-planned routes for every (closest lane at spawn, destination) pair + spawn constants."""
        net = self.net
        sp = self.spawner = RoundaboutSpawner(net, self.config, self.action_type.target_speeds)
        self._route_table = torch.from_numpy(sp.routes).to(self.device)
        self._route_table_len = torch.from_numpy(sp.route_lens).to(self.device)
        s = N.HwyRoundaboutSpawn()
        s.ego_lane = net.index[("ser", "ses", 0)]
        for j, li in enumerate([("we", "sx", 1), ("we", "sx", 0), ("we", "sx", 0), ("eer", "ees", 0)]):
            s.spawn_lane[j] = net.index[li]
        fd = self.config["incoming_vehicle_destination"]
        s.fixed_destination = -1 if fd is None else int(fd)
        s.ego_speed_index = speed_to_index(self.action_type.target_speeds, 8.0)
        for j, b in enumerate([5.0, 20.0, -20.0, 50.0]):
            s.base_longitudinal[j] = b
        s.ego_longitudinal, s.ego_heading_longitudinal, s.ego_speed = 125.0, 140.0, 8.0
        s.position_deviation, s.speed_deviation, s.traffic_speed = 2.0, 2.0, 16.0
        s.delta_lo, s.delta_hi = 3.5, 4.5
        s.route_table, s.route_len = self._route_table.data_ptr(), self._route_table_len.data_ptr()
        self._spawn_struct = s

    # ------------------------------------------------------------------ family kernels
    def _device_reset(self, mask_a, mask_b, obs_ptr) -> None:
        with torch.cuda.device(self.device):
            N.check(getattr(self._lib, self.RESET_ENTRY)(
                C.byref(self._params), self._graph_dev.data_ptr(), C.byref(self._spawn_struct),
                C.byref(self._state), self._rng.data_ptr(), mask_a, mask_b, obs_ptr, self._stream()))

    def _step_kernels(self, act) -> None:
        with torch.cuda.device(self.device):
            if self.SLOTS == N.HWY_NET_GROUP:
                N.check(self._lib.hwy_network_step(
                    C.byref(self._params), self._graph_dev.data_ptr(), C.byref(self._state), act.data_ptr(),
                    self._fused_out.data_ptr(), self._reward.data_ptr(), self._terminated.data_ptr(),
                    self._truncated.data_ptr(), self._info_speed.data_ptr(), self._info_crashed.data_ptr(),
                    self._stream()))
            else:  # 32 slots: the intersection family's kernel without rules / population changes
                N.check(self._lib.hwy_intersection_step(
                    C.byref(self._params), self._graph_dev.data_ptr(), None, C.byref(self._state), act.data_ptr(),
                    self._fused_out.data_ptr(), self._reward.data_ptr(), self._terminated.data_ptr(),
                    self._truncated.data_ptr(), self._info_speed.data_ptr(), self._info_crashed.data_ptr(),
                    self._stream()))

    def get_available_actions(self) -> torch.Tensor:
        """DiscreteMetaAction.get_available_actions (envs/common/action.py:262-298, AbstractEnv.get_available_actions
        abstract.py:357-358) for every env at once, on the device: a bool mask [N, 5] over (LANE_LEFT, IDLE,
        LANE_RIGHT, FASTER, SLOWER).  A lane change is available when the side lane exists on the ego's road and
        `is_reachable_from` the ego's position (road/lane.py:104-118, circular and sine lanes included); FASTER /
        SLOWER unless the speed index sits at the end of `target_speeds`."""
        return self._available_actions()

    # ------------------------------------------------------------------ host-exact reset
    def _reset_envs(self, env_ids: np.ndarray) -> None:
        sp = self.spawner.spawn([self._rngs[e] for e in env_ids])
        dev, V = self.device, self.N_VEHICLES
        idx = torch.from_numpy(np.asarray(env_ids, dtype=np.int64)).to(dev)
        f = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
        self._pos[idx, :V] = f(np.stack([sp["x"], sp["y"]], axis=-1))
        self._hs[idx, :V] = f(np.stack([sp["heading"], sp["speed"]], axis=-1))
        self._tt[idx, :V] = f(np.stack([sp["target_speed"], sp["timer"]], axis=-1))
        self._imp[idx, :V] = 0.0
        self._delta[idx, :V] = f(sp["delta"])
        self._meta[idx, :V] = f(N.pack_meta(sp, ()) | N.META_CHECK_COLLISIONS)
        self._route[idx, :V] = f(sp["route"])
        self._route_len[idx, :V] = f(sp["route_len"])
        self._speed_index[idx] = f(sp["speed_index"])
        self._time[idx] = 0.0

    # ------------------------------------------------------------------ state import / export
    def state_dict(self) -> dict:
        sd = super().state_dict()
        del sd["rng"]  # per-env fields only; the streams are rng_words()
        sd["route"], sd["route_len"] = self._route[:, :self.V].cpu().numpy(), self._route_len[:, :self.V].cpu().numpy()
        return sd

    def load_state_dict(self, sd: dict, env_ids=None) -> None:
        super().load_state_dict(sd if "no_lane_change" in sd else {**sd, "no_lane_change": False}, env_ids)
        idx = slice(None) if env_ids is None else torch.from_numpy(np.asarray(env_ids, dtype=np.int64)).to(self.device)
        self._route[idx, :self.V] = torch.from_numpy(np.ascontiguousarray(sd["route"], dtype=np.int32)).to(self.device)
        self._route_len[idx, :self.V] = torch.from_numpy(
            np.ascontiguousarray(sd["route_len"], dtype=np.int32)).to(self.device)


class BatchedConnectedLaneRoundaboutEnv(BatchedRoundaboutEnv):
    """`roundabout-v1`: ConnectedLaneNeighboursMixin (envs/common/abstract.py:26-37) — `neighbour_vehicles` also
    searches the lane segments connected to the queried lane (road/road.py:509-529)."""

    ENV_ID = "roundabout-v1"
