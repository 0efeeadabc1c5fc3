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
from typing import Any, Optional

import numpy as np
import torch

from .. import _native as N
from ..config import default_config
from ..road.network import NetworkTable
from ..spaces import Box, Discrete, batch_space
from .common.action import DiscreteMetaAction
from .common.observation import (KinematicObservation, LidarObservation, ObservationHost, OccupancyGridObservation,
                                 TimeToCollisionObservation, observation_factory)


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
        self._route_cache = {}

    def _route_of(self, lane_idx: int, destination: str):
        key = (lane_idx, destination)
        if key not in self._route_cache:
            li = self.net.lane_index_of[lane_idx]
            self._route_cache[key] = self.net.encode_route(self.net.plan_route(li, destination))
        return self._route_cache[key]

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
            route[k, 0], route_len[k, 0] = self._route_of(int(lane[k, 0]), "nxs")
            for j in range(4):
                route[k, j + 1], route_len[k, j + 1] = self._route_of(int(lane[k, j + 1]), self.DESTINATIONS[dest[k, j]])
        ts = self.target_speeds
        si = int(np.clip(np.round((8.0 - ts[0]) / (ts[-1] - ts[0]) * (ts.size - 1)), 0, ts.size - 1))
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



class BatchedRoundaboutEnv(ObservationHost):
    ENV_ID = "roundabout-v0"
    N_VEHICLES = 5
    EGO_SIDE_LANES = 1  # lanes of the road the controlled vehicle spawns on (default Kinematics y-range)
    SLOTS = N.HWY_NET_GROUP  # vehicle slots per env: 8 (one warp serves four envs) or 32 (HWY_NET_GROUP_LARGE)
    REWARD_NAMES = ("collision_reward", "high_speed_reward", "lane_change_reward", "on_road_reward")  # _rewards :58-65
    _kernel_events = None  # bench.py hook: list of (start, end) CUDA events around the step kernels
    metadata = {"render_modes": [], "autoreset_mode": "SameStep"}

    @classmethod
    def default_config(cls) -> dict:
        return default_config(cls.ENV_ID)

    def __init__(self, config: Optional[dict] = None, render_mode: Optional[str] = None, num_envs: int = 1,
                 device: Any = None, autoreset_mode: str = "SameStep", env_index_offset: int = 0,
                 reset_mode: str = "device") -> None:
        if render_mode is not None:
            raise NotImplementedError("rendering is out of scope of the accelerated path")
        if not torch.cuda.is_available():
            raise RuntimeError("highwayenv_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        if autoreset_mode not in ("SameStep", "NextStep", "Disabled"):
            raise ValueError(autoreset_mode)
        if autoreset_mode == "NextStep" and reset_mode != "device":
            raise NotImplementedError("NextStep autoreset uses the device reset")
        self._lib = N.load()
        self.render_mode = None
        self.num_envs = int(num_envs)
        self.device = torch.device(device if device is not None else "cuda")
        if reset_mode not in ("device", "host"):
            raise ValueError("reset_mode must be 'device' or 'host'")
        self.reset_mode = reset_mode
        self.autoreset_mode = autoreset_mode
        self.env_index_offset = int(env_index_offset)
        self.config = self.default_config()
        if config:
            self.config.update(config)
        self.net = self._make_network()
        self._graph_dev = torch.from_numpy(
            np.frombuffer(bytes(self.net.to_struct()), dtype=np.uint8).copy()).to(self.device)
        self._rngs = None
        self.define_spaces()
        self._allocate()

    def _make_network(self) -> NetworkTable:
        return make_roundabout_network()

    # ------------------------------------------------------------------ configuration
    def configure(self, config: Optional[dict]) -> None:
        if config:
            self.config.update(config)

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
        obs = cfg["observation"]
        p = N.HwyNetParams()
        p.n_vehicles = self.N_VEHICLES
        p.simulation_frequency = int(cfg["simulation_frequency"])
        p.policy_frequency = int(cfg["policy_frequency"])
        p.n_target_speeds = int(self.action_type.target_speeds.size)
        for k, t in enumerate(self.action_type.target_speeds):
            p.target_speeds[k] = float(t)
        self._configure_observation(p, obs)
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
        self.spawner = RoundaboutSpawner(self.net, self.config, self.action_type.target_speeds) if self.ENV_ID.startswith("roundabout") else None
        self.observation_space = batch_space(self.single_observation_space, self.num_envs)
        self.action_space = batch_space(self.single_action_space, self.num_envs)
        self.obs_shape = tuple(self.single_observation_space.shape)

    # ------------------------------------------------------------------ observation plugin (one registry, any env)
    FUSED_TTC_MAX_T, FUSED_TTC_MAX_SPEEDS = 16, 3  # EnvStage's shared TimeToCollision grid (hwy_network.cu)

    def _configure_observation(self, p, obs: dict) -> None:
        """Select the plugin with the reference's factory rule; decide whether the step kernel writes it itself
        (fused: Kinematics with 5 / 7 columns, the default OccupancyGrid, TimeToCollision up to 16 time cells) or a
        standalone kernel runs after the step (envs/common/observation.py)."""
        plugin = observation_factory(self, obs)
        self.observation_type = plugin
        fused = False
        if isinstance(plugin, TimeToCollisionObservation):
            plugin.bind(p.policy_frequency, self.action_type.target_speeds)
            n_t = plugin.horizon * p.policy_frequency
            if n_t <= self.FUSED_TTC_MAX_T and p.n_target_speeds <= self.FUSED_TTC_MAX_SPEEDS:
                p.obs_type, p.ttc_horizon, p.obs_vehicles_count, fused = N.OBS_TTC, plugin.horizon, 5, True
        elif isinstance(plugin, OccupancyGridObservation):
            if plugin.is_default:
                p.obs_type, p.obs_vehicles_count, fused = N.OBS_OCCUPANCY, 5, True
        elif isinstance(plugin, KinematicObservation):
            feats = plugin.features
            if feats[:5] != ["presence", "x", "y", "vx", "vy"] or feats[5:] not in ([], ["cos_h", "sin_h"]):
                raise NotImplementedError(f"Kinematics features {feats} on the network kernels "
                                          "(presence, x, y, vx, vy [, cos_h, sin_h])")
            if obs.get("observe_intentions"):
                raise NotImplementedError("Kinematics observe_intentions on the network kernels")
            fr = plugin.features_range
            if fr is None:  # normalize_obs (observation.py:214-226), computed at the first observation of an episode:
                w = 4.0 * self.EGO_SIDE_LANES  # all_side_lanes of the controlled vehicle's spawn road
                fr = {"x": [-5.0 * 40.0, 5.0 * 40.0], "y": [-w, w], "vx": [-2 * 40.0, 2 * 40.0], "vy": [-2 * 40.0, 2 * 40.0]}
            p.obs_type, p.obs_features = N.OBS_KINEMATICS, len(feats)
            p.obs_vehicles_count = plugin.vehicles_count
            p.obs_see_behind, p.obs_absolute = int(plugin.see_behind), int(plugin.absolute)
            p.obs_normalize, p.obs_clip = int(plugin.normalize), int(plugin.clip)
            (p.obs_x_lo, p.obs_x_hi), (p.obs_y_lo, p.obs_y_hi) = (map(float, fr["x"]), map(float, fr["y"]))
            (p.obs_vx_lo, p.obs_vx_hi), (p.obs_vy_lo, p.obs_vy_hi) = (map(float, fr["vx"]), map(float, fr["vy"]))
            fused = True
        self._plugin_standalone = not fused
        if not fused:  # the step kernel writes one Kinematics row into a scratch buffer; the plugin observes after it
            p.obs_type, p.obs_features, p.obs_vehicles_count = N.OBS_KINEMATICS, 5, 1
            p.obs_x_lo = p.obs_y_lo = p.obs_vx_lo = p.obs_vy_lo = -1.0
            p.obs_x_hi = p.obs_y_hi = p.obs_vx_hi = p.obs_vy_hi = 1.0
        self.single_observation_space = plugin.space()

    def _obs_view(self):
        if getattr(self, "_plugin_view", None) is None:
            v = N.HwyObsView()
            v.n_envs, v.vp, v.n_vehicles = self.num_envs, self.vp, self.N_VEHICLES
            v.n_agents = int(getattr(self._params, "n_agents", 0))
            v.pos, v.hs, v.meta = self._pos.data_ptr(), self._hs.data_ptr(), self._meta.data_ptr()
            cnt = getattr(self, "_count", None)
            v.count = None if cnt is None else cnt.data_ptr()
            v.route, v.route_len = self._route.data_ptr(), self._route_len.data_ptr()
            v.speed_index = self._speed_index.data_ptr()
            self._plugin_view = v
        return self._plugin_view, self._graph_dev.data_ptr()

    def _out_obs(self) -> torch.Tensor:
        if getattr(self.observation_type, "as_image", False):
            return self._obs.to(torch.uint8)
        return self._obs

    def _allocate(self) -> None:
        n, dev, vp = self.num_envs, self.device, self.SLOTS
        z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=dev)  # noqa: E731
        self.V, self.vp = self.N_VEHICLES, vp
        self._pos, self._hs, self._tt, self._imp = (z(n, vp, 2, dtype=torch.float64) for _ in range(4))
        self._delta = z(n, vp, dtype=torch.float64)
        self._meta = z(n, vp, dtype=torch.int32)
        self._route = z(n, vp, N.HWY_NET_MAX_ROUTE, dtype=torch.int32)
        self._route_len = z(n, vp, dtype=torch.int32)
        self._speed_index = z(n, dtype=torch.int32)
        self._time = z(n, dtype=torch.float64)
        self._obs = z(n, *self.obs_shape, dtype=torch.float32)
        self._final_obs = z(n, *self.obs_shape, dtype=torch.float32)
        # what the step / reset / observe kernels write: the observation itself, or a scratch row when a standalone
        # plugin observes after them
        self._fused_out = z(n, 5, dtype=torch.float32) if self._plugin_standalone else self._obs
        self._plugin_view = None
        self._reward = z(n, dtype=torch.float64)
        self._terminated = z(n, dtype=torch.uint8)
        self._truncated = z(n, dtype=torch.uint8)
        self._info_speed = z(n, dtype=torch.float64)
        self._info_crashed = z(n, dtype=torch.uint8)
        self._reward_terms = z(n, N.HWY_REWARD_TERMS, dtype=torch.float64)
        self._action_buf = z(n, dtype=torch.int32)
        # numpy PCG64 words (device reset mode).  A re-allocation (reset(options={"config": ...})) must keep the
        # env's stream: the reference's np_random survives a reset without a seed (abstract.py:219-249)
        old_rng = getattr(self, "_rng", None)
        self._rng = z(5, n, dtype=torch.int64)
        if old_rng is not None and old_rng.shape == self._rng.shape:
            self._rng.copy_(old_rng)
        self._build_spawn_tables()
        st = N.HwyNetState()
        st.n_envs, st.vp = n, vp
        st.pos, st.hs, st.tt, st.imp = (t.data_ptr() for t in (self._pos, self._hs, self._tt, self._imp))
        st.delta, st.meta = self._delta.data_ptr(), self._meta.data_ptr()
        st.route, st.route_len = self._route.data_ptr(), self._route_len.data_ptr()
        st.speed_index, st.time = self._speed_index.data_ptr(), self._time.data_ptr()
        st.reward_terms = self._reward_terms.data_ptr()
        if vp == N.HWY_NET_GROUP_LARGE:  # the 32-slot kernels read the population and RegulatedRoad.steps from the state
            self._count = torch.full((n,), self.N_VEHICLES, dtype=torch.int32, device=dev)
            self._road_steps = z(n, dtype=torch.int32)
            st.count, st.road_steps = self._count.data_ptr(), self._road_steps.data_ptr()
        self._state = st

    def _build_spawn_tables(self) -> None:
        """Host-planned routes for every (closest lane at spawn, destination) pair + spawn constants."""
        net, sp = self.net, self.spawner
        n_l = len(net.lanes)
        table = np.zeros((n_l, 4, N.HWY_NET_MAX_ROUTE), dtype=np.int32)
        lens = np.zeros((n_l, 4), dtype=np.int32)
        for l in range(n_l):
            for d, dest in enumerate(sp.DESTINATIONS + ["nxs"]):
                table[l, d], lens[l, d] = sp._route_of(l, dest)
        self._route_table = torch.from_numpy(table).to(self.device)
        self._route_table_len = torch.from_numpy(lens).to(self.device)
        s = N.HwyRoundaboutSpawn()
        s.ego_lane = net.index[("ser", "ses", 0)]
        for j, li in enumerate([("we", "sx", 1), ("we", "sx", 0), ("we", "sx", 0), ("eer", "ees", 0)]):
            s.spawn_lane[j] = net.index[li]
        fd = self.config["incoming_vehicle_destination"]
        s.fixed_destination = -1 if fd is None else int(fd)
        ts = self.action_type.target_speeds
        s.ego_speed_index = int(np.clip(np.round((8.0 - ts[0]) / (ts[-1] - ts[0]) * (ts.size - 1)), 0, ts.size - 1))
        for j, b in enumerate([5.0, 20.0, -20.0, 50.0]):
            s.base_longitudinal[j] = b
        s.ego_longitudinal, s.ego_heading_longitudinal, s.ego_speed = 125.0, 140.0, 8.0
        s.position_deviation, s.speed_deviation, s.traffic_speed = 2.0, 2.0, 16.0
        s.delta_lo, s.delta_hi = 3.5, 4.5
        s.route_table, s.route_len = self._route_table.data_ptr(), self._route_table_len.data_ptr()
        self._spawn_struct = s

    def _device_reset(self, mask_a, mask_b, obs_ptr) -> None:
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_roundabout_reset(
                C.byref(self._params), self._graph_dev.data_ptr(), C.byref(self._spawn_struct),
                C.byref(self._state), self._rng.data_ptr(), mask_a, mask_b, obs_ptr, self._stream()))

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    # ------------------------------------------------------------------ host-exact reset
    def _spawn(self, env_ids: np.ndarray) -> dict:
        return self.spawner.spawn([self._rngs[e] for e in env_ids])

    def _upload(self, env_ids: np.ndarray, sp: dict) -> None:
        dev, V = self.device, self.N_VEHICLES
        idx = torch.from_numpy(np.asarray(env_ids, dtype=np.int64)).to(dev)
        f = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
        self._pos[idx, :V] = f(np.stack([sp["x"], sp["y"]], axis=-1))
        self._hs[idx, :V] = f(np.stack([sp["heading"], sp["speed"]], axis=-1))
        self._tt[idx, :V] = f(np.stack([sp["target_speed"], sp["timer"]], axis=-1))
        self._imp[idx, :V] = 0.0
        self._delta[idx, :V] = f(sp["delta"])
        meta = ((sp["lane"].astype(np.int64) << N.META_LANE_SHIFT) | (sp["target_lane"].astype(np.int64) << N.META_TARGET_SHIFT)
                | (sp["kind"] << N.META_KIND_SHIFT) | N.META_CHECK_COLLISIONS | N.META_PRESENT).astype(np.int32)
        self._meta[idx, :V] = f(meta)
        self._route[idx, :V] = f(sp["route"])
        self._route_len[idx, :V] = f(sp["route_len"])
        self._speed_index[idx] = f(sp["speed_index"])
        self._time[idx] = 0.0

    def _seed_streams(self, seed) -> None:
        n = self.num_envs
        if seed is None:
            ss = np.random.SeedSequence()
            seeds = [int(s.generate_state(1)[0]) for s in ss.spawn(n)]
        elif isinstance(seed, (int, np.integer)):
            seeds = [int(seed) + self.env_index_offset + i for i in range(n)]
        else:
            seeds = [int(s) for s in seed]
        self._rngs = [np.random.Generator(np.random.PCG64(np.random.SeedSequence(s))) for s in seeds]
        self.np_random_seed = seeds
        if self.reset_mode == "device":
            words = np.zeros((5, n), dtype=np.uint64)
            m64 = (1 << 64) - 1
            for i, g in enumerate(self._rngs):
                st = g.bit_generator.state
                sv, inc = st["state"]["state"], st["state"]["inc"]
                words[:, i] = (sv >> 64, sv & m64, inc >> 64, inc & m64, (int(st["has_uint32"]) << 32) | int(st["uinteger"]))
            self._rng.copy_(torch.from_numpy(words.view(np.int64)).to(self.device))

    # ------------------------------------------------------------------ gym API
    def reset(self, *, seed=None, options: Optional[dict] = None):
        if options and "config" in options:
            self.configure(options["config"])
            self.define_spaces()
            self._allocate()
        if seed is not None or self._rngs is None:
            self._seed_streams(seed)
        mask = None
        if options and options.get("reset_mask") is not None:
            mask = np.asarray(options["reset_mask"]).astype(bool)
        if self.reset_mode == "device":
            mt = None
            if mask is not None:
                mt = torch.from_numpy(mask.astype(np.uint8)).to(self.device)
                self._mask_keepalive = mt
            self._device_reset(None if mt is None else mt.data_ptr(), None, None)
        else:
            ids = np.arange(self.num_envs) if mask is None else np.nonzero(mask)[0]
            if len(ids):
                self._upload(ids, self._spawn(ids))
        self._autoreset_envs = None
        self.observe()
        return self._out_obs(), {"speed": self._hs[:, 0, 1], "crashed": (self._meta[:, 0] & N.META_CRASHED) != 0}

    def observe(self) -> torch.Tensor:
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_network_observe(C.byref(self._params), self._graph_dev.data_ptr(),
                                                  C.byref(self._state), self._fused_out.data_ptr(), self._stream()))
        if self._plugin_standalone:
            self._observe_plugin(self._obs)
        return self._out_obs()

    def step(self, actions):
        if self._rngs is None:
            raise RuntimeError("call reset() before step()")
        buf = self._action_buf
        if isinstance(actions, torch.Tensor) and actions.device == buf.device and actions.dtype == buf.dtype \
                and actions.shape == buf.shape and actions.is_contiguous():
            act = actions
        elif isinstance(actions, torch.Tensor):  # dtype / device conversion without a host round trip
            buf.copy_(actions.reshape(buf.shape), non_blocking=True)
            act = buf
        else:
            buf.copy_(torch.from_numpy(np.ascontiguousarray(np.asarray(actions).reshape(tuple(buf.shape))))
                      .to(buf.dtype), non_blocking=True)
            act = buf
        kev = self._kernel_events
        if kev is not None:  # bench.py: CUDA events around the step kernel(s) alone
            kev.append((torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)))
            kev[-1][0].record(torch.cuda.current_stream(self.device))
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
        if kev is not None:
            kev[-1][1].record(torch.cuda.current_stream(self.device))
        info = {"speed": self._info_speed, "crashed": self._info_crashed.view(torch.bool), "action": act,
                "rewards": {name: self._reward_terms[:, k] for k, name in enumerate(self.REWARD_NAMES)}}
        plugin = self._plugin_standalone
        if plugin:
            self._observe_plugin(self._obs)
        if self.autoreset_mode == "SameStep" and self.reset_mode == "device":
            self._final_obs.copy_(self._obs)
            info["final_obs"] = self._final_obs
            self._device_reset(self._terminated.data_ptr(), self._truncated.data_ptr(), self._fused_out.data_ptr())
            if plugin:
                self._observe_plugin(self._obs, self._terminated, self._truncated)
        elif self.autoreset_mode == "NextStep":  # see BatchedHighwayEnv._next_step_autoreset
            prev = getattr(self, "_autoreset_envs", None)
            if prev is not None:
                self._device_reset(prev.data_ptr(), None, self._fused_out.data_ptr())
                if plugin:
                    self._observe_plugin(self._obs, prev)
                keep = prev == 0
                self._reward.mul_(keep)
                self._terminated.mul_(keep)
                self._truncated.mul_(keep)
            self._autoreset_envs = (self._terminated | self._truncated).contiguous()
        elif self.autoreset_mode == "SameStep":
            done = (self._terminated | self._truncated).cpu().numpy().astype(bool)
            if done.any():
                self._final_obs.copy_(self._obs)
                info["final_obs"] = self._final_obs
                ids = np.nonzero(done)[0]
                self._upload(ids, self._spawn(ids))
                self.observe()
        return (self._out_obs(), self._reward, self._terminated.view(torch.bool), self._truncated.view(torch.bool), info)

    def road_substeps(self, n_substeps: int) -> None:
        """The reference's operator seam (`AbstractEnv._simulate` without `action_type.act`, abstract.py:304-307):
        `n_substeps` x (`Road.act()`; `Road.step(1 / simulation_frequency)`, with the RegulatedRoad rules where the
        scenario has them) on the device state of every env and nothing else — no observation, reward, clock,
        population change or autoreset; the controlled vehicle acts like `ControlledVehicle.act(None)`."""
        if self._rngs is None:
            raise RuntimeError("call reset() before road_substeps()")
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_network_substeps(C.byref(self._params), self._graph_dev.data_ptr(),
                                                   C.byref(self._state), None, int(n_substeps), self._stream()))

    def host_stepper(self):
        """Host-buffer stepping through one CUDA graph (envs/common/host_stepper.py)."""
        from .common.host_stepper import HostStepper

        return HostStepper(self)

    def close(self) -> None:
        pass

    @property
    def unwrapped(self):
        return self

    # ------------------------------------------------------------------ state import / export
    def state_dict(self) -> dict:
        V = self.V
        pos, hs, tt, imp = (t[:, :V].cpu().numpy() for t in (self._pos, self._hs, self._tt, self._imp))
        meta = self._meta[:, :V].cpu().numpy()
        return {
            "x": pos[..., 0].copy(), "y": pos[..., 1].copy(), "heading": hs[..., 0].copy(),
            "speed": hs[..., 1].copy(), "target_speed": tt[..., 0].copy(), "timer": tt[..., 1].copy(),
            "delta": self._delta[:, :V].cpu().numpy(), "impact_x": imp[..., 0].copy(), "impact_y": imp[..., 1].copy(),
            "lane": (meta >> N.META_LANE_SHIFT) & 0xFF, "target_lane": (meta >> N.META_TARGET_SHIFT) & 0xFF,
            "kind": (meta >> N.META_KIND_SHIFT) & 3, "crashed": (meta & N.META_CRASHED) != 0,
            "no_lane_change": (meta & N.META_NO_LANE_CHANGE) != 0,
            "has_impact": (meta & N.META_HAS_IMPACT) != 0, "check_collisions": (meta & N.META_CHECK_COLLISIONS) != 0,
            "route": self._route[:, :V].cpu().numpy(), "route_len": self._route_len[:, :V].cpu().numpy(),
            "speed_index": self._speed_index.cpu().numpy(), "time": self._time.cpu().numpy(),
        }

    def load_state_dict(self, sd: dict) -> None:
        n, V, dev = self.num_envs, self.V, self.device
        f = lambda k: torch.from_numpy(np.ascontiguousarray(sd[k], dtype=np.float64)).to(dev)  # noqa: E731
        self._pos[:, :V, 0], self._pos[:, :V, 1] = f("x"), f("y")
        self._hs[:, :V, 0], self._hs[:, :V, 1] = f("heading"), f("speed")
        self._tt[:, :V, 0], self._tt[:, :V, 1] = f("target_speed"), f("timer")
        self._imp[:, :V, 0], self._imp[:, :V, 1] = f("impact_x"), f("impact_y")
        self._delta[:, :V] = f("delta")
        meta = ((np.asarray(sd["lane"], dtype=np.int64) << N.META_LANE_SHIFT)
                | (np.asarray(sd["target_lane"], dtype=np.int64) << N.META_TARGET_SHIFT)
                | (np.asarray(sd["kind"], dtype=np.int64) << N.META_KIND_SHIFT)
                | np.where(np.asarray(sd["crashed"], dtype=bool), N.META_CRASHED, 0)
                | np.where(np.asarray(sd["has_impact"], dtype=bool), N.META_HAS_IMPACT, 0)
                | np.where(np.asarray(sd["check_collisions"], dtype=bool), N.META_CHECK_COLLISIONS, 0)
                | (np.where(np.asarray(sd["no_lane_change"], dtype=bool), N.META_NO_LANE_CHANGE, 0)
                   if "no_lane_change" in sd else 0)
                | N.META_PRESENT).astype(np.int32)
        self._meta[:, :V] = torch.from_numpy(meta.reshape(n, V)).to(dev)
        self._route[:, :V] = torch.from_numpy(np.ascontiguousarray(sd["route"], dtype=np.int32)).to(dev)
        self._route_len[:, :V] = torch.from_numpy(np.ascontiguousarray(sd["route_len"], dtype=np.int32)).to(dev)
        self._speed_index.copy_(torch.from_numpy(np.asarray(sd["speed_index"], dtype=np.int32).reshape(n)))
        self._time.copy_(torch.from_numpy(np.asarray(sd["time"], dtype=np.float64).reshape(n)))
        if self._rngs is None:
            self._seed_streams(0)
        if "rng" in sd:  # the env streams: [5][n] words, the layout of state_dict()["rng"]
            w = np.ascontiguousarray(sd["rng"], dtype=np.uint64).reshape(5, n)
            self._rng.copy_(torch.from_numpy(w.view(np.int64)).to(dev))
            for e, g in enumerate(self._rngs):
                g.bit_generator.state = {
                    "bit_generator": "PCG64", "state": {"state": (int(w[0, e]) << 64) | int(w[1, e]),
                                                        "inc": (int(w[2, e]) << 64) | int(w[3, e])},
                    "has_uint32": int(w[4, e]) >> 32, "uinteger": int(w[4, e]) & 0xFFFFFFFF}

    def rng_words(self) -> np.ndarray:
        """The env streams as [5][n] words (state hi, lo, inc hi, lo, has_uint32 << 32 | uinteger): the device words
        of reset_mode="device", the numpy generators' of the host-exact reset."""
        if self.reset_mode == "device":
            return self._rng.cpu().numpy().view(np.uint64).copy()
        m = (1 << 64) - 1
        w = np.zeros((5, self.num_envs), dtype=np.uint64)
        for e, g in enumerate(self._rngs):
            st = g.bit_generator.state
            s, inc = st["state"]["state"], st["state"]["inc"]
            w[:, e] = (s >> 64, s & m, inc >> 64, inc & m, (int(st["has_uint32"]) << 32) | int(st["uinteger"]))
        return w


class BatchedConnectedLaneRoundaboutEnv(BatchedRoundaboutEnv):
    """`roundabout-v1`: ConnectedLaneNeighboursMixin (envs/common/abstract.py:26-37) — `neighbour_vehicles` also
    searches the lane segments connected to the queried lane (road/road.py:509-529)."""

    ENV_ID = "roundabout-v1"
