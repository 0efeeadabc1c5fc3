"""Batched intersection-v0 on the H100 backend.

Host-side mirror of the reference's ``IntersectionEnv`` (highway_env/envs/intersection_env.py):
4-way crossing with 20 lanes and priorities, ``RegulatedRoad`` yielding rules, a population that
changes every step (``_clear_vehicles`` / ``_spawn_vehicle``), Kinematics (7 features) or
OccupancyGrid observation, 3 longitudinal meta-actions.

Stepping — including the RegulatedRoad rules and the per-step clear/spawn with the env's numpy
stream — runs in ``hwy_intersection_step``.  ``reset`` has two implementations of
``_make_vehicles`` (:245-323):

* ``reset_mode="device"`` (default): ``hwy_intersection_reset`` — draws, warm-up simulation,
  challenger, controlled vehicle and pruning in one kernel over the envs that finished; this is
  what the SameStep autoreset uses, so a step never leaves the GPU.
* ``reset_mode="host"``: the same sequence with numpy generators on the host (bit-identical to
  the reference's draws and lane arithmetic) and only the 3 s warm-up on the device
  (``hwy_network_substeps``); used by the parity tests against the reference's reset states.

Both consume the env's PCG64 stream identically (checked word for word in the tests).
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
from .common.action import ContinuousAction, DiscreteAction
from .common.observation import (KinematicObservation, ObservationHost, OccupancyGridObservation,
                                 observation_factory)

VMAX = N.HWY_NET_GROUP_LARGE


def make_intersection_network() -> NetworkTable:
    """IntersectionEnv._make_road (intersection_env.py:142-243): per corner an incoming road, right
    turn, left turn, straight crossing and exit; priorities 3/1 (horizontal/vertical), left turns -1."""
    net = NetworkTable()
    lane_width = 4
    right_turn_radius = lane_width + 5
    left_turn_radius = right_turn_radius + lane_width
    outer_distance = right_turn_radius + lane_width / 2
    access_length = 50 + 50
    for corner in range(4):
        angle = np.radians(90 * corner)
        priority = 3 if corner % 2 else 1
        rot = np.array([[np.cos(angle), -np.sin(angle)], [np.sin(angle), np.cos(angle)]])
        o, ir = "o" + str(corner), "ir" + str(corner)
        net.add_straight(o, ir, rot @ np.array([lane_width / 2, access_length + outer_distance]),
                         rot @ np.array([lane_width / 2, outer_distance]), priority=priority, speed_limit=10.0)
        net.add_circular(ir, "il" + str((corner - 1) % 4), rot @ np.array([outer_distance, outer_distance]),
                         right_turn_radius, angle + np.radians(180), angle + np.radians(270), clockwise=True,
                         priority=priority, speed_limit=10.0)
        net.add_circular(ir, "il" + str((corner + 1) % 4),
                         rot @ np.array([-left_turn_radius + lane_width / 2, left_turn_radius - lane_width / 2]),
                         left_turn_radius, angle + np.radians(0), angle + np.radians(-90), clockwise=False,
                         priority=priority - 1, speed_limit=10.0)
        net.add_straight(ir, "il" + str((corner + 2) % 4), rot @ np.array([lane_width / 2, outer_distance]),
                         rot @ np.array([lane_width / 2, -outer_distance]), priority=priority, speed_limit=10.0)
        ex_start = rot @ np.flip([lane_width / 2, access_length + outer_distance], axis=0)
        ex_end = rot @ np.flip([lane_width / 2, outer_distance], axis=0)
        net.add_straight("il" + str((corner - 1) % 4), "o" + str((corner - 1) % 4), ex_end, ex_start,
                         priority=priority, speed_limit=10.0)
    net.finalize()
    return net


_F64 = ("x", "y", "heading", "speed", "target_speed", "timer", "delta", "impact_x", "impact_y")


class BatchedIntersectionEnv(ObservationHost):
    ENV_ID = "intersection-v0"
    MULTI_AGENT_WRAPPER = False
    REWARD_NAMES = ("collision_reward", "high_speed_reward", "arrived_reward", "on_road_reward")  # _agent_rewards :95-105
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
        if reset_mode not in ("device", "host"):
            raise ValueError(reset_mode)
        self.reset_mode = reset_mode
        self._lib = N.load()
        self.render_mode = None
        self.num_envs = int(num_envs)
        self.device = torch.device(device if device is not None else "cuda")
        self.autoreset_mode = autoreset_mode
        self.env_index_offset = int(env_index_offset)
        self.config = self.default_config()
        if config:
            self.config.update(config)
        self.net = make_intersection_network()
        self._graph_dev = torch.from_numpy(np.frombuffer(bytes(self.net.to_struct()), dtype=np.uint8).copy()).to(self.device)
        self._rngs = None
        self._route_cache = {}
        self.define_spaces()
        self._allocate()

    def configure(self, config: Optional[dict]) -> None:
        if config:
            self.config.update(config)

    # ------------------------------------------------------------------ spaces / parameters
    def define_spaces(self) -> None:
        cfg = self.config
        act, obs = cfg["action"], cfg["observation"]
        # MultiAgentAction / MultiAgentObservation (action.py:301-333, observation.py:588-604): the same plugin per
        # controlled vehicle; tuples of the reference become a leading agent axis here
        self.n_agents = int(cfg.get("controlled_vehicles", 1))
        multi = act["type"] == "MultiAgentAction" or obs["type"] == "MultiAgentObservation"
        if multi:
            if act["type"] != "MultiAgentAction" or obs["type"] != "MultiAgentObservation":
                raise NotImplementedError("MultiAgentAction and MultiAgentObservation go together here")
            act, obs = act["action_config"], obs["observation_config"]
        elif self.n_agents != 1:
            raise NotImplementedError("controlled_vehicles > 1 needs MultiAgentAction / MultiAgentObservation")
        if not 1 <= self.n_agents <= 4:
            raise ValueError("controlled_vehicles must be in 1..4")
        self.multi_agent = multi
        # ContinuousAction / DiscreteAction (envs/common/action.py:73-196; the reference's intersection-v1): the controlled
        # vehicle is a plain Vehicle, or with dynamical=True a BicycleVehicle (vehicle/dynamics.py)
        self.action_type = None
        longi, lat = act.get("longitudinal", True), act.get("lateral", True)
        if act["type"] in ("ContinuousAction", "DiscreteAction"):
            if multi:
                raise NotImplementedError("MultiAgentAction over ContinuousAction")
            self.action_type = (DiscreteAction if act["type"] == "DiscreteAction" else ContinuousAction)(**act)
        elif act["type"] != "DiscreteMetaAction":
            if act["type"] == "MultiAgentAction":
                raise NotImplementedError("nested MultiAgentAction")
            raise ValueError("Unknown action type")
        elif not longi:
            raise NotImplementedError("lateral-only meta-actions")
        ts = act.get("target_speeds")
        self.target_speeds = np.linspace(20, 30, 3) if ts is None else np.array(ts, dtype=np.float64)
        if self.target_speeds.size > 3:
            raise NotImplementedError("more than 3 target speeds on the network kernels")
        p = N.HwyNetParams()
        p.n_vehicles = VMAX
        p.simulation_frequency, p.policy_frequency = int(cfg["simulation_frequency"]), int(cfg["policy_frequency"])
        p.n_target_speeds = int(self.target_speeds.size)
        for k, t in enumerate(self.target_speeds):
            p.target_speeds[k] = float(t)
        p.action_mode = 1 if not lat else 0
        self.single_action_space = Discrete(3 if not lat else 5)
        if self.action_type is not None:
            if self.reset_mode != "device":
                raise NotImplementedError("ContinuousAction / DiscreteAction envs reset on the device")
            at = self.action_type
            p.action_type, p.act_clip, p.dynamical = 1, int(at.clip), int(at.dynamical)
            p.acc_lo, p.acc_hi = float(at.acceleration_range[0]), float(at.acceleration_range[1])
            p.steer_lo, p.steer_hi = float(at.steering_range[0]), float(at.steering_range[1])
            self.single_action_space = at.space()
        p.obs_features = 5
        # ---- observation plugin: the reference's factory rule (one registry, envs/common/observation.py); the step
        # kernel writes Kinematics (5 / 7 columns) and the default OccupancyGrid itself, any other plugin observes
        # with its standalone kernel after the step
        plugin = observation_factory(self, obs)
        self.observation_type = plugin
        fused = False
        if isinstance(plugin, OccupancyGridObservation) and plugin.is_default and not multi:
            p.obs_type, p.obs_vehicles_count, fused = N.OBS_OCCUPANCY, 5, True
        elif isinstance(plugin, KinematicObservation):
            feats = plugin.features
            if obs.get("observe_intentions"):
                raise NotImplementedError("Kinematics observe_intentions")
            fr = plugin.features_range
            if feats[:5] != ["presence", "x", "y", "vx", "vy"] or feats[5:] not in ([], ["cos_h", "sin_h"]):
                # any Vehicle.to_dict column list (vehicle/kinematics.py:237-261) with per-column ranges
                rng = fr if fr is not None else {"x": [-200.0, 200.0], "y": [-4.0, 4.0], "vx": [-80.0, 80.0], "vy": [-80.0, 80.0]}
                p.obs_n_feat = len(feats)
                for k, f in enumerate(feats):
                    p.obs_feat[k] = N.FEATURE_CODES[f]
                    if f in rng:
                        p.obs_feat_ranged[k], p.obs_feat_lo[k], p.obs_feat_hi[k] = 1, float(rng[f][0]), float(rng[f][1])
            if fr is None:  # normalize_obs (observation.py:214-226): the controlled vehicle spawns on a one-lane road
                fr = {"x": [-5.0 * 40.0, 5.0 * 40.0], "y": [-4.0, 4.0], "vx": [-2 * 40.0, 2 * 40.0], "vy": [-2 * 40.0, 2 * 40.0]}
            p.obs_type, p.obs_features = N.OBS_KINEMATICS, len(feats)
            p.obs_vehicles_count = plugin.vehicles_count
            p.obs_see_behind, p.obs_absolute = int(plugin.see_behind), int(plugin.absolute)
            p.obs_normalize, p.obs_clip = int(plugin.normalize), int(plugin.clip)
            (p.obs_x_lo, p.obs_x_hi), (p.obs_y_lo, p.obs_y_hi) = (map(float, fr["x"]), map(float, fr["y"]))
            (p.obs_vx_lo, p.obs_vx_hi), (p.obs_vy_lo, p.obs_vy_hi) = (map(float, fr["vx"]), map(float, fr["vy"]))
            fused = True
        if hasattr(plugin, "bind"):  # TimeToCollision
            plugin.bind(p.policy_frequency, self.target_speeds)
        self._plugin_standalone = not fused
        if not fused:  # scratch row for the kernels' own epilogue
            p.obs_type, p.obs_features, p.obs_vehicles_count = N.OBS_KINEMATICS, 5, 1
            p.obs_x_lo = p.obs_y_lo = p.obs_vx_lo = p.obs_vy_lo = -1.0
            p.obs_x_hi = p.obs_y_hi = p.obs_vx_hi = p.obs_vy_hi = 1.0
        self.single_observation_space = plugin.space()
        p.normalize_reward = int(bool(cfg["normalize_reward"]))
        p.duration = float(cfg["duration"])
        p.collision_reward, p.high_speed_reward = float(cfg["collision_reward"]), float(cfg["high_speed_reward"])
        p.arrived_reward = float(cfg["arrived_reward"])
        p.reward_speed_lo, p.reward_speed_hi = (float(v) for v in cfg["reward_speed_range"])
        p.offroad_terminal = int(bool(cfg["offroad_terminal"]))
        # IDMVehicle constants as overridden by _make_vehicles (intersection_env.py:262-265)
        p.acc_max, p.comfort_acc_max, p.comfort_acc_min = 6.0, 6.0, -3.0
        p.distance_wanted, p.time_wanted = 7.0, 1.5
        p.politeness, p.lane_change_min_acc_gain = 0.0, 0.2
        p.lane_change_max_braking_imposed, p.lane_change_delay = 2.0, 1.0
        p.perception_distance = 200.0
        p.regulated, p.reward_type, p.dynamic_population = 1, 1, 1
        p.connected_lanes = int(bool(cfg.get("neighbour_vehicles_connected_lanes", False)))
        self._params = p
        self.observation_space = batch_space(self.single_observation_space, self.num_envs)
        self.action_space = batch_space(self.single_action_space, self.num_envs)
        p.n_agents = self.n_agents if multi else 0
        self._params = p
        if multi:  # Tuple spaces of the reference -> one leading agent axis
            per = self.single_observation_space
            self.single_observation_space = Box(low=-np.inf, high=np.inf, shape=(self.n_agents,) + tuple(per.shape),
                                                dtype=np.float32)
            self.agent_action_space = self.single_action_space
            self.single_action_space = Box(low=0, high=self.agent_action_space.n - 1, shape=(self.n_agents,),
                                           dtype=np.int64)
            self.observation_space = batch_space(self.single_observation_space, self.num_envs)
            self.action_space = batch_space(self.single_action_space, self.num_envs)
        self.obs_shape = tuple(self.single_observation_space.shape)

    def _allocate(self) -> None:
        n, dev, vp = self.num_envs, self.device, VMAX
        z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=dev)  # noqa: E731
        self.vp = vp
        self._pos, self._hs, self._tt, self._imp = (z(n, vp, 2, dtype=torch.float64) for _ in range(4))
        self._delta = z(n, vp, dtype=torch.float64)
        self._meta = z(n, vp, dtype=torch.int32)
        self._route = z(n, vp, N.HWY_NET_MAX_ROUTE, dtype=torch.int32)
        self._route_len = z(n, vp, dtype=torch.int32)
        A = self.n_agents
        self._speed_index = z(n * A, dtype=torch.int32)
        self._agents_reward = z(n, A, dtype=torch.float64)
        self._agents_terminated = z(n, A, dtype=torch.uint8)
        self._time = z(n, dtype=torch.float64)
        self._count = z(n, dtype=torch.int32)
        self._road_steps = z(n, dtype=torch.int32)
        self._reward_terms = z(n, N.HWY_REWARD_TERMS, dtype=torch.float64)
        self._overflow = z(n, dtype=torch.int32)  # spawns dropped because all 32 slots were taken (loud, see step())
        old_rng = getattr(self, "_rng", None)  # keep the env's numpy stream across a re-allocation
        self._rng = z(5, n, dtype=torch.int64)
        if old_rng is not None and old_rng.shape == self._rng.shape:
            self._rng.copy_(old_rng)
        self._obs = z(n, *self.obs_shape, dtype=torch.float32)
        self._final_obs = z(n, *self.obs_shape, dtype=torch.float32)
        self._fused_out = z(n, A, 5, dtype=torch.float32) if self._plugin_standalone else self._obs
        self._plugin_view = None
        self._reward = z(n, dtype=torch.float64)
        self._terminated, self._truncated = z(n, dtype=torch.uint8), z(n, dtype=torch.uint8)
        self._info_speed, self._info_crashed = z(n, dtype=torch.float64), z(n, dtype=torch.uint8)
        if self.action_type is not None:  # ContinuousAction: float32 (throttle, steering); DiscreteAction gathers into it
            self._action_buf = z(n, 2, dtype=torch.float32)
        else:
            self._action_buf = z(n, A, dtype=torch.int32) if self.multi_agent else z(n, dtype=torch.int32)
        st = N.HwyNetState()
        st.n_envs, st.vp = n, vp
        st.pos, st.hs, st.tt, st.imp = (t.data_ptr() for t in (self._pos, self._hs, self._tt, self._imp))
        st.delta, st.meta = self._delta.data_ptr(), self._meta.data_ptr()
        st.route, st.route_len = self._route.data_ptr(), self._route_len.data_ptr()
        st.speed_index, st.time = self._speed_index.data_ptr(), self._time.data_ptr()
        st.count, st.road_steps, st.rng = self._count.data_ptr(), self._road_steps.data_ptr(), self._rng.data_ptr()
        st.overflow = self._overflow.data_ptr()
        st.reward_terms = self._reward_terms.data_ptr()
        self._state = st
        # plan_route_to(lane, "o"+k) for every lane (vehicle/controller.py:71-87)
        n_l = len(self.net.lanes)
        table = np.zeros((n_l, 4, N.HWY_NET_MAX_ROUTE), dtype=np.int32)
        lens = np.zeros((n_l, 4), dtype=np.int32)
        for l in range(n_l):
            for k in range(4):
                table[l, k], lens[l, k] = self._route_of(l, "o" + str(k))
        self._route_table = torch.from_numpy(table).to(dev)
        self._route_table_len = torch.from_numpy(lens).to(dev)
        sp = N.HwyIntersectionSpawn()
        for k in range(4):
            sp.spawn_lane[k] = self.net.index[("o" + str(k), "ir" + str(k), 0)]
        sp.spawn_probability = float(self.config["spawn_probability"])
        sp.route_table, sp.route_len = self._route_table.data_ptr(), self._route_table_len.data_ptr()
        sp.ego_lane = self.net.index[("o0", "ir0", 0)]
        dest = self.config["destination"]
        if dest is not None and (not isinstance(dest, str) or dest not in ("o0", "o1", "o2", "o3")):
            raise ValueError(f"destination {dest!r}")
        sp.ego_destination = -1 if dest is None else int(dest[1:])
        sp.initial_vehicle_count = int(self.config["initial_vehicle_count"])
        self._scratch = z(2 * (n + 1), dtype=torch.int32)
        sp.scratch = self._scratch.data_ptr()
        self._spawn_struct = sp

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _route_of(self, lane_idx: int, destination: str):
        key = (lane_idx, destination)
        if key not in self._route_cache:
            self._route_cache[key] = self.net.encode_route(
                self.net.plan_route(self.net.lane_index_of[lane_idx], destination))
        return self._route_cache[key]

    # ------------------------------------------------------------------ state import / export
    def state_dict(self) -> dict:
        pos, hs, tt, imp = (t.cpu().numpy() for t in (self._pos, self._hs, self._tt, self._imp))
        meta = self._meta.cpu().numpy()
        return {
            "x": pos[..., 0].copy(), "y": pos[..., 1].copy(), "heading": hs[..., 0].copy(), "speed": hs[..., 1].copy(),
            "target_speed": tt[..., 0].copy(), "timer": tt[..., 1].copy(), "delta": self._delta.cpu().numpy(),
            "impact_x": imp[..., 0].copy(), "impact_y": imp[..., 1].copy(),
            "lane": (meta >> N.META_LANE_SHIFT) & 0xFF, "target_lane": (meta >> N.META_TARGET_SHIFT) & 0xFF,
            "kind": (meta >> N.META_KIND_SHIFT) & 3, "crashed": (meta & N.META_CRASHED) != 0,
            "has_impact": (meta & N.META_HAS_IMPACT) != 0, "check_collisions": (meta & N.META_CHECK_COLLISIONS) != 0,
            "is_yielding": (meta & N.META_YIELDING) != 0,
            # BicycleVehicle.lateral_speed / yaw_rate (vehicle/dynamics.py:52-53) live in the tt pair of a plain Vehicle
            "lat_speed": np.where(((meta >> N.META_KIND_SHIFT) & 3) == N.KIND_VEHICLE, tt[..., 0], 0.0),
            "yaw_rate": np.where(((meta >> N.META_KIND_SHIFT) & 3) == N.KIND_VEHICLE, tt[..., 1], 0.0),
            "route": self._route.cpu().numpy(), "route_len": self._route_len.cpu().numpy(),
            "speed_index": (self._speed_index.cpu().numpy().reshape(self.num_envs, self.n_agents)
                            if self.multi_agent else self._speed_index.cpu().numpy()),
            "time": self._time.cpu().numpy(),
            "count": self._count.cpu().numpy(), "road_steps": self._road_steps.cpu().numpy(),
            "rng": self._rng.cpu().numpy().view(np.uint64),
        }

    def load_state_dict(self, sd: dict, env_ids=None) -> None:
        dev = self.device
        idx = slice(None) if env_ids is None else torch.from_numpy(np.asarray(env_ids, dtype=np.int64)).to(dev)
        f = lambda a, dt=np.float64: torch.from_numpy(np.ascontiguousarray(np.nan_to_num(np.asarray(a, dtype=dt)))).to(dev)  # noqa: E731
        self._pos[idx] = f(np.stack([sd["x"], sd["y"]], axis=-1))
        self._hs[idx] = f(np.stack([sd["heading"], sd["speed"]], axis=-1))
        ts, tm = np.asarray(sd["target_speed"], dtype=np.float64), np.asarray(sd["timer"], dtype=np.float64)
        if "lat_speed" in sd:  # plain Vehicle slots carry (lateral_speed, yaw_rate) instead of (target_speed, timer)
            plain = np.asarray(sd["kind"]) == N.KIND_VEHICLE
            ts, tm = np.where(plain, np.nan_to_num(sd["lat_speed"]), ts), np.where(plain, np.nan_to_num(sd["yaw_rate"]), tm)
        self._tt[idx] = f(np.stack([ts, tm], axis=-1))
        self._imp[idx] = f(np.stack([sd["impact_x"], sd["impact_y"]], axis=-1))
        self._delta[idx] = f(sd["delta"])
        meta = ((np.asarray(sd["lane"], dtype=np.int64) << N.META_LANE_SHIFT)
                | (np.asarray(sd["target_lane"], dtype=np.int64) << N.META_TARGET_SHIFT)
                | (np.asarray(sd["kind"], dtype=np.int64) << N.META_KIND_SHIFT)
                | np.where(np.asarray(sd["crashed"], dtype=bool), N.META_CRASHED, 0)
                | np.where(np.asarray(sd["has_impact"], dtype=bool), N.META_HAS_IMPACT, 0)
                | np.where(np.asarray(sd["is_yielding"], dtype=bool), N.META_YIELDING, 0)
                | N.META_CHECK_COLLISIONS | N.META_PRESENT).astype(np.int32)
        self._meta[idx] = torch.from_numpy(meta).to(dev)
        self._route[idx] = torch.from_numpy(np.ascontiguousarray(sd["route"], dtype=np.int32)).to(dev)
        self._route_len[idx] = torch.from_numpy(np.ascontiguousarray(sd["route_len"], dtype=np.int32)).to(dev)
        si = torch.from_numpy(np.ascontiguousarray(np.asarray(sd["speed_index"], dtype=np.int32)).reshape(-1, self.n_agents)).to(dev)
        self._speed_index.view(self.num_envs, self.n_agents)[idx] = si
        self._time[idx] = torch.from_numpy(np.asarray(sd["time"], dtype=np.float64).reshape(-1)).to(dev)
        self._count[idx] = torch.from_numpy(np.asarray(sd["count"], dtype=np.int32).reshape(-1)).to(dev)
        self._road_steps[idx] = torch.from_numpy(np.asarray(sd["road_steps"], dtype=np.int32).reshape(-1)).to(dev)
        if "rng" in sd:
            w = torch.from_numpy(np.ascontiguousarray(sd["rng"]).view(np.int64)).to(dev)
            if env_ids is None:
                self._rng.copy_(w)
            else:
                self._rng[:, idx] = w
        if self._rngs is None:
            self._rngs = [None] * self.num_envs

    # ------------------------------------------------------------------ reset (_make_vehicles, host + device warm-up)
    def _empty_rows(self, m: int) -> dict:
        sd = {k: np.zeros((m, VMAX)) for k in _F64}
        sd["delta"][:] = 4.0
        for k in ("lane", "target_lane", "kind", "crashed", "has_impact", "is_yielding", "route_len"):
            sd[k] = np.zeros((m, VMAX), dtype=np.int64)
        sd["route"] = np.zeros((m, VMAX, N.HWY_NET_MAX_ROUTE), dtype=np.int32)
        sd["speed_index"] = np.zeros((m, self.n_agents), dtype=np.int32)
        sd["time"] = np.zeros(m)
        sd["count"] = np.zeros(m, dtype=np.int32)
        sd["road_steps"] = np.zeros(m, dtype=np.int32)
        return sd

    def _append(self, sd: dict, k: int, x, y, h, speed, kind, destination, delta, target_speed=None, timer=None) -> int:
        n = int(sd["count"][k])
        lane = int(self.net.closest_lane(np.array([x]), np.array([y]), np.array([h]))[0])
        sd["x"][k, n], sd["y"][k, n], sd["heading"][k, n], sd["speed"][k, n] = x, y, h, speed
        sd["target_speed"][k, n] = speed if target_speed is None else target_speed
        sd["timer"][k, n] = ((x + y) * np.pi) % 1.0 if timer is None else timer
        sd["delta"][k, n] = delta
        sd["impact_x"][k, n] = sd["impact_y"][k, n] = 0.0
        sd["lane"][k, n] = sd["target_lane"][k, n] = lane
        sd["kind"][k, n] = kind
        sd["crashed"][k, n] = sd["has_impact"][k, n] = sd["is_yielding"][k, n] = 0
        sd["route"][k, n], sd["route_len"][k, n] = self._route_of(lane, destination)
        sd["count"][k] = n + 1
        return n

    def _spawn_vehicle(self, sd, k, g, longitudinal=0.0, position_deviation=1.0, speed_deviation=1.0,
                       spawn_probability=0.6, go_straight=False) -> None:
        """IntersectionEnv._spawn_vehicle (intersection_env.py:325-352)."""
        if g.uniform() > spawn_probability:
            return
        route = g.choice(range(4), size=2, replace=False)
        route[1] = (route[0] + 2) % 4 if go_straight else route[1]
        lane = self.net.index[("o" + str(route[0]), "ir" + str(route[0]), 0)]
        lon = longitudinal + 5.0 + g.normal() * position_deviation
        speed = 8.0 + g.normal() * speed_deviation
        px, py = self.net.position(lane, lon, 0.0)
        x, y, h = float(px), float(py), float(self.net.heading_at(lane, lon))
        n = int(sd["count"][k])
        for v in range(n):
            if np.linalg.norm(np.array([sd["x"][k, v] - x, sd["y"][k, v] - y])) < 15:
                return
        if n >= VMAX:
            return
        self._append(sd, k, x, y, h, speed, N.KIND_IDM, "o" + str(route[1]), g.uniform(low=3.5, high=4.5))

    def _reset_envs(self, ids: np.ndarray) -> None:
        cfg, m = self.config, len(ids)
        sd = self._empty_rows(m)
        n_vehicles = int(cfg["initial_vehicle_count"])
        lon0 = np.linspace(0, 80, n_vehicles)
        for k, e in enumerate(ids):
            for t in range(n_vehicles - 1):
                self._spawn_vehicle(sd, k, self._rngs[e], lon0[t])
        self.load_state_dict(sd, ids)
        mask = torch.zeros(self.num_envs, dtype=torch.uint8, device=self.device)
        mask[torch.from_numpy(np.asarray(ids, dtype=np.int64)).to(self.device)] = 1
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_network_substeps(C.byref(self._params), self._graph_dev.data_ptr(),
                                                   C.byref(self._state), mask.data_ptr(),
                                                   3 * int(cfg["simulation_frequency"]), self._stream()))
        full = self.state_dict()
        sd = {k: (v[ids].copy() if k != "rng" else None) for k, v in full.items()}
        sd.pop("rng")
        ts = self.target_speeds
        sd["speed_index"] = np.asarray(sd["speed_index"]).reshape(m, self.n_agents)
        for k, e in enumerate(ids):
            g = self._rngs[e]
            self._spawn_vehicle(sd, k, g, 60, spawn_probability=1.0, go_straight=True, position_deviation=0.1,
                                speed_deviation=0.0)
            for agent in range(self.n_agents):  # :291-323, one controlled vehicle per access road
                ego_lane = self.net.index[("o%d" % (agent % 4), "ir%d" % (agent % 4), 0)]
                destination = cfg["destination"] or "o" + str(g.integers(1, 4))
                px, py = self.net.position(ego_lane, 60.0 + 5.0 * g.normal(1.0), 0.0)
                x, y, h = float(px), float(py), float(self.net.heading_at(ego_lane, 60.0))
                speed_limit = self.net.lanes[ego_lane]["speed_limit"]
                si = int(np.clip(np.round((speed_limit - ts[0]) / (ts[-1] - ts[0]) * (ts.size - 1)), 0, ts.size - 1))
                self._append(sd, k, x, y, h, speed_limit, N.KIND_MDP, destination, 4.0, target_speed=ts[si], timer=0.0)
                sd["speed_index"][k, agent] = si
                n = int(sd["count"][k])
                keep = [v for v in range(n) if sd["kind"][k, v] == N.KIND_MDP or not (
                    np.linalg.norm(np.array([sd["x"][k, v] - x, sd["y"][k, v] - y])) < 20)]
                for name, arr in sd.items():
                    if name in ("speed_index", "time", "count", "road_steps"):
                        continue
                    arr[k, :len(keep)] = arr[k, keep]
                sd["count"][k] = len(keep)
            sd["time"][k] = 0.0
        words = np.zeros((5, m), dtype=np.uint64)
        m64 = (1 << 64) - 1
        for k, e in enumerate(ids):
            st = self._rngs[e].bit_generator.state
            sv, inc = st["state"]["state"], st["state"]["inc"]
            words[:, k] = (sv >> 64, sv & m64, inc >> 64, inc & m64, (int(st["has_uint32"]) << 32) | int(st["uinteger"]))
        sd["rng"] = words
        self.load_state_dict(sd, ids)

    def _device_reset(self, mask_a, mask_b, obs_ptr, final_obs_ptr) -> None:
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_intersection_reset(
                C.byref(self._params), self._graph_dev.data_ptr(), C.byref(self._spawn_struct), C.byref(self._state),
                mask_a, mask_b, obs_ptr, final_obs_ptr, self._stream()))

    def _sync_host_rngs(self, ids) -> None:
        """The device advanced the streams (per-step spawns): mirror them into the host generators."""
        words = self._rng.cpu().numpy().view(np.uint64)
        for e in ids:
            g = self._rngs[e]
            st = g.bit_generator.state
            st["state"]["state"] = (int(words[0, e]) << 64) | int(words[1, e])
            st["state"]["inc"] = (int(words[2, e]) << 64) | int(words[3, e])
            st["has_uint32"], st["uinteger"] = int(words[4, e]) >> 32, int(words[4, e]) & 0xFFFFFFFF
            g.bit_generator.state = st

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
        fresh = seed is not None or self._rngs is None or any(g is None for g in self._rngs)
        if fresh:
            self._seed_streams(seed)
        mask = None
        if options and options.get("reset_mask") is not None:
            mask = np.asarray(options["reset_mask"]).astype(bool)
        if self.reset_mode == "device":
            mt = None if mask is None else torch.from_numpy(mask.astype(np.uint8)).to(self.device)
            self._device_reset(None if mt is None else mt.data_ptr(), None, None, None)
        else:
            ids = np.arange(self.num_envs) if mask is None else np.nonzero(mask)[0]
            if not fresh:
                self._sync_host_rngs(ids)
            if len(ids):
                self._reset_envs(ids)
        self._autoreset_envs = None
        self.observe()
        return self._out_obs(), {"speed": self._info_speed, "crashed": self._info_crashed.view(torch.bool)}

    def observe(self) -> torch.Tensor:
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_network_observe(C.byref(self._params), self._graph_dev.data_ptr(),
                                                  C.byref(self._state), self._fused_out.data_ptr(), self._stream()))
        if self._plugin_standalone:
            self._observe_plugin(self._obs)
        return self._out_obs()

    def _out_obs(self) -> torch.Tensor:
        if getattr(self.observation_type, "as_image", False):
            return self._obs.to(torch.uint8)
        return self._obs

    def _obs_view(self):
        if self._plugin_view is None:
            v = N.HwyObsView()
            v.n_envs, v.vp, v.n_vehicles, v.n_agents = self.num_envs, self.vp, VMAX, (self.n_agents if self.multi_agent else 0)
            v.pos, v.hs, v.meta = self._pos.data_ptr(), self._hs.data_ptr(), self._meta.data_ptr()
            v.count = self._count.data_ptr()
            v.route, v.route_len = self._route.data_ptr(), self._route_len.data_ptr()
            v.speed_index = self._speed_index.data_ptr()
            self._plugin_view = v
        return self._plugin_view, self._graph_dev.data_ptr()

    def step(self, actions):
        if self._rngs is None:
            raise RuntimeError("call reset() before step()")
        buf = self._action_buf
        table = getattr(self.action_type, "table", None)
        if table is not None:  # DiscreteAction (action.py:165-196): index -> (throttle, steering), then ContinuousAction
            if getattr(self, "_action_table", None) is None or self._action_table.device != buf.device:
                self._action_table = torch.from_numpy(table).to(buf.device)
            idx = actions if isinstance(actions, torch.Tensor) else torch.from_numpy(np.asarray(actions))
            torch.index_select(self._action_table, 0, idx.to(device=buf.device, dtype=torch.long).reshape(-1), out=buf)
            act = buf
        elif isinstance(actions, torch.Tensor) and actions.device == buf.device and actions.dtype == buf.dtype \
                and actions.shape == buf.shape and actions.is_contiguous():
            act = actions
        elif isinstance(actions, torch.Tensor):  # dtype / device conversion without a host round trip
            buf.copy_(actions.reshape(buf.shape), non_blocking=True)
            act = buf
        else:
            a = np.asarray(actions)
            buf.copy_(torch.from_numpy(np.ascontiguousarray(a.reshape(tuple(buf.shape)))).to(buf.dtype), non_blocking=True)
            act = buf
        prev = getattr(self, "_autoreset_envs", None) if self.autoreset_mode == "NextStep" else None
        rng_before = self._rng.clone() if prev is not None else None  # a step draws from the env's generator
        kev = self._kernel_events
        if kev is not None:  # bench.py: CUDA events around the step kernel(s) alone
            kev.append((torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)))
            kev[-1][0].record(torch.cuda.current_stream(self.device))
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_intersection_step_agents(
                C.byref(self._params), self._graph_dev.data_ptr(), C.byref(self._spawn_struct), C.byref(self._state),
                act.data_ptr(), self._fused_out.data_ptr(), self._reward.data_ptr(), self._terminated.data_ptr(),
                self._truncated.data_ptr(), self._info_speed.data_ptr(), self._info_crashed.data_ptr(),
                self._agents_reward.data_ptr() if self.multi_agent else None,
                self._agents_terminated.data_ptr() if self.multi_agent else None, self._stream()))
        if kev is not None:
            kev[-1][1].record(torch.cuda.current_stream(self.device))
        # "spawn_overflow" [N] int32: how many accepted spawns found all 32 vehicle slots of the env taken since the env
        # was constructed.  The reference's vehicle list is unbounded; a non-zero entry means that env no longer
        # follows the reference (reachable only with `duration` >> 13 s or a high spawn_probability).
        info = {"speed": self._info_speed, "crashed": self._info_crashed.view(torch.bool), "action": act,
                "spawn_overflow": self._overflow,
                "rewards": {name: self._reward_terms[:, k] for k, name in enumerate(self.REWARD_NAMES)}}
        if self.multi_agent:  # IntersectionEnv._info (:124-132)
            info["agents_rewards"] = self._agents_reward
            info["agents_terminated"] = self._agents_terminated.view(torch.bool)
        plugin = self._plugin_standalone
        if plugin:
            self._observe_plugin(self._obs)
        if self.autoreset_mode == "SameStep" and self.reset_mode == "device":
            info["final_obs"] = self._final_obs
            if plugin:
                self._final_obs.copy_(self._obs)
                self._device_reset(self._terminated.data_ptr(), self._truncated.data_ptr(), self._fused_out.data_ptr(), None)
                self._observe_plugin(self._obs, self._terminated, self._truncated)
            else:
                self._device_reset(self._terminated.data_ptr(), self._truncated.data_ptr(), self._obs.data_ptr(),
                                   self._final_obs.data_ptr())
        elif self.autoreset_mode == "NextStep":
            # gymnasium NEXT_STEP: envs that ended in the previous step are reset by this call instead of stepped;
            # their generator is rewound to where the episode ended, then _make_vehicles runs on the device
            if prev is not None:
                self._rng.copy_(torch.where(prev.bool().unsqueeze(0), rng_before, self._rng))
                self._device_reset(prev.data_ptr(), None, self._fused_out.data_ptr(), None)
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
                self._sync_host_rngs(ids)
                self._reset_envs(ids)
                self.observe()
        if self.multi_agent and self.MULTI_AGENT_WRAPPER:
            # MultiAgentWrapper.step (envs/common/abstract.py:468-477): per-agent rewards and terminal flags
            return (self._out_obs(), self._agents_reward, self._agents_terminated.view(torch.bool),
                    self._truncated.view(torch.bool), info)
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


class BatchedContinuousIntersectionEnv(BatchedIntersectionEnv):
    """`intersection-v1` (ContinuousIntersectionEnv, envs/intersection_env.py:431-473): ContinuousAction with the
    dynamical BicycleVehicle (vehicle/dynamics.py:33-160: RK4 over a 6-state tyre model), steering range +-pi/3, and an
    8-column absolute Kinematics observation (presence, x, y, vx, vy, long_off, lat_off, ang_off).  Under RegulatedRoad
    such an ego is not a ControlledVehicle: `is_conflict_possible` forward-simulates a copy of it
    (Vehicle.predict_trajectory_constant_speed, vehicle/kinematics.py:179-198) — restated in the rules kernel."""

    ENV_ID = "intersection-v1"


class BatchedConnectedLaneIntersectionEnv(BatchedIntersectionEnv):
    """`intersection-v2`: ConnectedLaneNeighboursMixin (envs/common/abstract.py:26-37) — `neighbour_vehicles` also
    searches the lane segments connected to the queried lane (road/road.py:509-529)."""

    ENV_ID = "intersection-v2"


class BatchedMultiAgentIntersectionEnv(BatchedIntersectionEnv):
    """`intersection-multi-agent-v0` (MultiAgentIntersectionEnv, envs/intersection_env.py:376-420): two controlled
    vehicles, tuple actions / observations as a leading agent axis, mean reward, any-crashed / all-arrived
    termination, `info["agents_rewards"]`, `info["agents_terminated"]`."""

    ENV_ID = "intersection-multi-agent-v0"


class BatchedMultiAgentWrappedIntersectionEnv(BatchedMultiAgentIntersectionEnv):
    """`intersection-multi-agent-v1`: the same behind MultiAgentWrapper (abstract.py:468-477) — `step` returns the
    per-agent rewards and terminal flags [N, agents] in place of the scalar ones."""

    ENV_ID = "intersection-multi-agent-v1"
    MULTI_AGENT_WRAPPER = True


class BatchedConnectedLaneMultiAgentIntersectionEnv(BatchedMultiAgentWrappedIntersectionEnv):
    """`intersection-multi-agent-v2`: + ConnectedLaneNeighboursMixin."""

    ENV_ID = "intersection-multi-agent-v2"
