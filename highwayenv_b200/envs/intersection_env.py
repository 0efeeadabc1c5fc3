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

import numpy as np
import torch

from .. import _native as N
from ..road.network import NetworkTable
from ..spaces import Box, Discrete, batch_space
from .common.action import ContinuousAction, DiscreteAction, speed_to_index
from .common.observation import select_network_observation
from .common.vector_env import BatchedNetworkEnv

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


class BatchedIntersectionEnv(BatchedNetworkEnv):
    ENV_ID = "intersection-v0"
    SLOTS = VMAX
    V = VMAX
    MULTI_AGENT_WRAPPER = False
    REWARD_NAMES = ("collision_reward", "high_speed_reward", "arrived_reward", "on_road_reward")  # _agent_rewards :95-105
    META_FLAGS = ("crashed", "has_impact", "check_collisions", "is_yielding")
    NEXT_STEP_REWINDS_RNG = True  # the step spawns vehicles from the env's stream (_spawn_vehicle)

    def _make_network(self) -> NetworkTable:
        return make_intersection_network()

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
        self.observation_type, fused = select_network_observation(
            self, p, obs, self.target_speeds, 1, fuse_ttc=False, fuse_grid=not multi, feature_columns=True)
        self._plugin_standalone = not fused
        self.single_observation_space = self.observation_type.space()
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
        p.n_agents = self.n_agents if multi else 0
        self._params = p
        self.observation_space = batch_space(self.single_observation_space, self.num_envs)
        self.action_space = batch_space(self.single_action_space, self.num_envs)
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
        n, dev, A = self.num_envs, self.device, self.n_agents
        z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=dev)  # noqa: E731
        st = self._allocate_network_state(VMAX)
        self._agents_reward = z(n, A, dtype=torch.float64)
        self._agents_terminated = z(n, A, dtype=torch.uint8)
        self._count = z(n, dtype=torch.int32)
        self._road_steps = z(n, dtype=torch.int32)
        self._overflow = z(n, dtype=torch.int32)  # spawns dropped because all 32 slots were taken (loud, see step())
        if self.action_type is not None:  # ContinuousAction: float32 (throttle, steering); DiscreteAction gathers into it
            self._action_buf = z(n, 2, dtype=torch.float32)
        else:
            self._action_buf = z(n, A, dtype=torch.int32) if self.multi_agent else z(n, dtype=torch.int32)
        st.count, st.road_steps, st.rng = self._count.data_ptr(), self._road_steps.data_ptr(), self._rng.data_ptr()
        st.overflow = self._overflow.data_ptr()
        self._routes, self._route_lens = self._route_tables(["o0", "o1", "o2", "o3"])
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

    # ------------------------------------------------------------------ state import / export
    def state_dict(self) -> dict:
        sd = super().state_dict()
        plain = sd["kind"] == N.KIND_VEHICLE
        # BicycleVehicle.lateral_speed / yaw_rate (vehicle/dynamics.py:52-53) live in the tt pair of a plain Vehicle
        sd["lat_speed"] = np.where(plain, sd["target_speed"], 0.0)
        sd["yaw_rate"] = np.where(plain, sd["timer"], 0.0)
        sd["route"], sd["route_len"] = self._route.cpu().numpy(), self._route_len.cpu().numpy()
        if self.multi_agent:
            sd["speed_index"] = sd["speed_index"].reshape(self.num_envs, self.n_agents)
        sd["count"], sd["road_steps"] = self._count.cpu().numpy(), self._road_steps.cpu().numpy()
        return sd

    def load_state_dict(self, sd: dict, env_ids=None) -> None:
        dev = self.device
        sd = {**sd, **{k: np.nan_to_num(np.asarray(sd[k], dtype=np.float64)) for k in _F64}, "check_collisions": True}
        if "lat_speed" in sd:  # plain Vehicle slots carry (lateral_speed, yaw_rate) instead of (target_speed, timer)
            plain = np.asarray(sd["kind"]) == N.KIND_VEHICLE
            sd["target_speed"] = np.where(plain, np.nan_to_num(sd["lat_speed"]), sd["target_speed"])
            sd["timer"] = np.where(plain, np.nan_to_num(sd["yaw_rate"]), sd["timer"])
        super().load_state_dict(sd, env_ids)
        idx = slice(None) if env_ids is None else torch.from_numpy(np.asarray(env_ids, dtype=np.int64)).to(dev)
        self._route[idx] = torch.from_numpy(np.ascontiguousarray(sd["route"], dtype=np.int32)).to(dev)
        self._route_len[idx] = torch.from_numpy(np.ascontiguousarray(sd["route_len"], dtype=np.int32)).to(dev)
        self._count[idx] = torch.from_numpy(np.asarray(sd["count"], dtype=np.int32).reshape(-1)).to(dev)
        self._road_steps[idx] = torch.from_numpy(np.asarray(sd["road_steps"], dtype=np.int32).reshape(-1)).to(dev)

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
        d = int(destination[1:])
        sd["route"][k, n], sd["route_len"][k, n] = self._routes[lane, d], self._route_lens[lane, d]
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
                si = speed_to_index(ts, speed_limit)
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
        self.load_state_dict(sd, ids)

    # ------------------------------------------------------------------ family kernels
    def _device_reset(self, mask_a, mask_b, obs_ptr, final_obs_ptr=None) -> None:
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_intersection_reset(
                C.byref(self._params), self._graph_dev.data_ptr(), C.byref(self._spawn_struct), C.byref(self._state),
                mask_a, mask_b, obs_ptr, final_obs_ptr, self._stream()))

    def _reset_info(self) -> dict:
        return {"speed": self._info_speed, "crashed": self._info_crashed.view(torch.bool)}

    def _step_kernels(self, act) -> None:
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_intersection_step_agents(
                C.byref(self._params), self._graph_dev.data_ptr(), C.byref(self._spawn_struct), C.byref(self._state),
                act.data_ptr(), self._fused_out.data_ptr(), self._reward.data_ptr(), self._terminated.data_ptr(),
                self._truncated.data_ptr(), self._info_speed.data_ptr(), self._info_crashed.data_ptr(),
                self._agents_reward.data_ptr() if self.multi_agent else None,
                self._agents_terminated.data_ptr() if self.multi_agent else None, self._stream()))

    def _step_info(self, act) -> dict:
        info = super()._step_info(act)
        # "spawn_overflow" [N] int32: how many accepted spawns found all 32 vehicle slots of the env taken since the env
        # was constructed.  The reference's vehicle list is unbounded; a non-zero entry means that env no longer
        # follows the reference (reachable only with `duration` >> 13 s or a high spawn_probability).
        info["spawn_overflow"] = self._overflow
        if self.multi_agent:  # IntersectionEnv._info (:124-132)
            info["agents_rewards"] = self._agents_reward
            info["agents_terminated"] = self._agents_terminated.view(torch.bool)
        return info

    def _same_step_autoreset(self, info) -> None:
        if self.reset_mode != "device" or self._plugin_standalone:
            return super()._same_step_autoreset(info)
        info["final_obs"] = self._final_obs  # the reset kernel writes the final observation of the finished envs
        self._device_reset(self._terminated.data_ptr(), self._truncated.data_ptr(), self._obs.data_ptr(),
                           self._final_obs.data_ptr())

    def _step_result(self, info):
        if self.multi_agent and self.MULTI_AGENT_WRAPPER:
            # MultiAgentWrapper.step (envs/common/abstract.py:468-477): per-agent rewards and terminal flags
            return (self._out_obs(), self._agents_reward, self._agents_terminated.view(torch.bool),
                    self._truncated.view(torch.bool), info)
        return super()._step_result(info)


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
