"""Batched highway-v0 / highway-fast-v0 on the H100 backend.

Host-side mirror of the reference's ``HighwayEnv`` / ``HighwayEnvFast``
(highway_env/envs/highway_env.py:16-182) over ``AbstractEnv``
(highway_env/envs/common/abstract.py:40-465): same ``config`` dictionary, same
``reset(seed=, options=)`` / ``step(action)`` contract, same observation/action plugin
selection — but one instance owns ``num_envs`` independent roads that live in HBM and are
stepped in lock-step by ``hwy_highway_step`` (include/hwyb200.h).  The batched surface is
gymnasium's ``VectorEnv`` shape (``num_envs``, ``single_observation_space``,
``single_action_space``, batched 5-tuples, autoreset modes), as exercised by the reference's
tests/envs/test_gym.py:138-177.

Env ``i`` owns the numpy ``Generator(PCG64)`` stream a reference env seeded with
``seed + env_index_offset + i`` would own; every ``_reset`` (including device-side
autoresets) consumes it in the reference's draw order, so spawns are bit-identical.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .. import _native as N
from ..spaces import Box, batch_space
from .common.action import action_factory
from .common.observation import KinematicObservation, observation_factory
from .common.vector_env import BatchedVectorEnv
from ..road.network import NetworkTable

IDM_VEHICLE = "highway_env.vehicle.behavior.IDMVehicle"
# LinearVehicle and its subclasses (vehicle/behavior.py:350-583) -> LANE_CHANGE_MIN_ACC_GAIN.  On the highway the three
# are one model: randomize_behavior overwrites the subclasses' ACCELERATION_PARAMETERS with draws from the
# ACCELERATION_RANGE they inherit from LinearVehicle.
LINEAR_VEHICLE_TYPES = {
    "highway_env.vehicle.behavior.LinearVehicle": 0.2,
    "highway_env.vehicle.behavior.AggressiveVehicle": 1.0,
    "highway_env.vehicle.behavior.DefensiveVehicle": 1.0,
}


def linear_ranges():
    """LinearVehicle.ACCELERATION_RANGE / STEERING_RANGE (behavior.py:353-371) as (lo, hi - lo) per parameter, with
    the reference's numpy arithmetic (KP_HEADING = 1 / TAU_HEADING, KP_LATERAL = 1 / TAU_LATERAL, controller.py:24-33)."""
    kp_heading, kp_lateral = 1 / 0.2, 1 / 0.6
    acc = np.array([0.3, 0.3, 2.0])
    steer = np.array([kp_heading, kp_heading * kp_lateral])
    acc_range = np.array([0.5 * acc, 1.5 * acc])
    steer_range = np.array([steer - np.array([0.07, 1.5]), steer + np.array([0.07, 1.5])])
    return acc_range[0], acc_range[1] - acc_range[0], steer_range[0], steer_range[1] - steer_range[0]


class BatchedHighwayEnv(BatchedVectorEnv):
    """``num_envs`` independent highway roads stepped by the sm_90a kernels."""

    ENV_ID = "highway-v0"
    OTHERS_CHECK_COLLISIONS = True

    PERCEPTION_DISTANCE = 5.0 * 40.0  # abstract.py:56
    REWARD_NAMES = ("collision_reward", "right_lane_reward", "high_speed_reward", "on_road_reward")  # _rewards :118-137
    _allocated_for = None
    n_agents = 1
    multi_agent = False

    # ------------------------------------------------------------------ configuration
    def define_spaces(self) -> None:
        """Plugin selection by ``config[...]["type"]`` (abstract.py:154-161).

        ``config["controlled_vehicles"]`` = A > 1 spawns A controlled vehicles (highway_env.py:72-98).
        MultiAgentAction / MultiAgentObservation (action.py:301-333, observation.py:588-604) wrap one plugin per
        controlled vehicle; their tuples become a leading agent axis here: actions [N, A] (DiscreteMetaAction,
        DiscreteAction) or [N, A, 2] (ContinuousAction), observations [N, A, ...].  The two switches are independent:
        a plain action type drives the first controlled vehicle only, a plain observation observes from it only."""
        cfg = self.config
        act_cfg, obs_cfg = cfg["action"], cfg["observation"]
        self.n_agents = int(cfg.get("controlled_vehicles", 1))
        if not 1 <= self.n_agents <= 8:
            raise ValueError("controlled_vehicles must be in 1..8")
        self.multi_action = act_cfg["type"] == "MultiAgentAction"
        self.multi_obs = obs_cfg["type"] == "MultiAgentObservation"
        if self.multi_action:
            act_cfg = act_cfg["action_config"]
        if self.multi_obs:
            obs_cfg = obs_cfg["observation_config"]
        self.multi_agent = self.multi_action or self.multi_obs
        self.observation_type = observation_factory(self, obs_cfg)
        self.action_type = action_factory(self, act_cfg)
        # the step kernel's own epilogue is Kinematics; any other plugin runs its standalone kernel after the step
        # (envs/common/observation.py) while the kernel writes default Kinematics rows into a scratch buffer
        self._plugin_standalone = self.observation_type.standalone
        self._fused_obs = KinematicObservation() if self._plugin_standalone else self.observation_type
        if hasattr(self.observation_type, "bind"):  # TimeToCollision: the observer's target speeds
            if not hasattr(self.action_type, "target_speeds"):
                raise ValueError("TimeToCollision needs an MDPVehicle observer (DiscreteMetaAction): "
                                 "compute_ttc_grid reads vehicle.target_speeds (finite_mdp.py:104-163)")
            self.observation_type.bind(self.config["policy_frequency"], self.action_type.target_speeds)
        self.single_observation_space = self.observation_type.space()
        self.single_action_space = self.action_type.space()
        A = self.n_agents
        if self.multi_obs:
            per = self.single_observation_space
            self.agent_observation_space = per
            self.single_observation_space = Box(low=per.low.min() if per.low.size else -np.inf,
                                                high=per.high.max() if per.high.size else np.inf,
                                                shape=(A,) + tuple(per.shape), dtype=per.dtype)
        if self.multi_action:
            per = self.single_action_space
            self.agent_action_space = per
            if hasattr(per, "n"):  # DiscreteMetaAction / DiscreteAction index per agent
                self.single_action_space = Box(low=0, high=per.n - 1, shape=(A,), dtype=np.int64)
            else:
                self.single_action_space = Box(-1.0, 1.0, shape=(A, 2), dtype=np.float32)
        self.observation_space = batch_space(self.single_observation_space, self.num_envs)
        self.action_space = batch_space(self.single_action_space, self.num_envs)
        self._params = self._build_params()

    def _build_params(self) -> N.HwyHighwayParams:
        cfg = self.config
        A = self.n_agents
        ovt = cfg.get("other_vehicles_type")
        if ovt != IDM_VEHICLE and ovt not in LINEAR_VEHICLE_TYPES:
            raise NotImplementedError("only IDMVehicle and LinearVehicle / AggressiveVehicle / DefensiveVehicle traffic "
                                      "is on the accelerated path")
        self._linear = ovt in LINEAR_VEHICLE_TYPES
        if self._linear and A > 1:
            raise NotImplementedError("LinearVehicle traffic with several controlled vehicles")
        if cfg.get("neighbour_vehicles_connected_lanes"):
            raise NotImplementedError("connected-lane neighbour search (v1/v2 ids) is not implemented")
        if cfg.get("manual_control"):
            raise NotImplementedError("manual_control")
        p = N.HwyHighwayParams()
        lanes = int(cfg["lanes_count"])
        if not 1 <= lanes <= N.HWY_MAX_LANES:
            raise ValueError(f"lanes_count must be in 1..{N.HWY_MAX_LANES}")
        p.lanes_count = lanes
        p.n_vehicles = int(cfg["vehicles_count"]) + A
        if p.n_vehicles > N.HWY_MAX_VEHICLES:
            raise ValueError(f"vehicles_count + controlled_vehicles must be <= {N.HWY_MAX_VEHICLES}")
        # one controlled vehicle (A = 1) runs the single-agent kernels whatever the switches: same layout and draws
        p.n_agents = A if A > 1 else 0
        p.multi_action = int(self.multi_action and A > 1)
        p.multi_obs = int(self.multi_obs and A > 1 and not self._plugin_standalone)
        p.simulation_frequency = int(cfg["simulation_frequency"])
        p.policy_frequency = int(cfg["policy_frequency"])
        p.others_check_collisions = int(self.OTHERS_CHECK_COLLISIONS)
        p.normalize_reward = int(bool(cfg["normalize_reward"]))
        p.offroad_terminal = int(bool(cfg["offroad_terminal"]))
        ili = cfg.get("initial_lane_id")
        p.initial_lane_id = -1 if ili is None else int(ili)
        p.duration = float(cfg["duration"])
        p.collision_reward = float(cfg["collision_reward"])
        p.right_lane_reward = float(cfg["right_lane_reward"])
        p.high_speed_reward = float(cfg["high_speed_reward"])
        p.reward_speed_lo, p.reward_speed_hi = (float(v) for v in cfg["reward_speed_range"])
        p.ego_spacing = float(cfg["ego_spacing"])
        p.vehicles_density = float(cfg["vehicles_density"])
        p.ego_speed = 25.0  # highway_env.py:83
        p.spawn_exp = float(np.exp(-5 / 40 * lanes))  # kinematics.py:95
        # IDMVehicle class constants, behavior.py:21-46
        p.acc_max, p.comfort_acc_max, p.comfort_acc_min = 6.0, 3.0, -5.0
        p.distance_wanted, p.time_wanted = 5.0 + 5.0, 1.5
        p.politeness, p.lane_change_min_acc_gain = 0.0, 0.2
        p.lane_change_max_braking_imposed, p.lane_change_delay = 2.0, 1.0
        p.delta_lo, p.delta_hi = 3.5, 4.5
        if self._linear:  # LinearVehicle.TIME_WANTED (behavior.py:373) and the class's LANE_CHANGE_MIN_ACC_GAIN
            p.time_wanted = 2.5
            p.lane_change_min_acc_gain = LINEAR_VEHICLE_TYPES[ovt]
        p.perception_distance = self.PERCEPTION_DISTANCE
        self._fused_obs.fill_params(p)
        self.action_type.fill_params(p)
        # RoadNetwork.straight_road_network(lanes, speed_limit=30) (road/road.py:291-321) with
        # StraightLane.__init__ arithmetic (road/lane.py:183-194)
        width, length, speed_limit, angle, start = 4.0, 10000.0, 30.0, 0.0, 0.0
        rotation = np.array([[np.cos(angle), np.sin(angle)], [-np.sin(angle), np.cos(angle)]])
        for l in range(lanes):
            origin = rotation @ np.array([start, l * width])
            end = rotation @ np.array([start + length, l * width])
            L = p.lanes[l]
            L.start_x, L.start_y = float(origin[0]), float(origin[1])
            L.heading = float(np.arctan2(end[1] - origin[1], end[0] - origin[0]))
            L.length = float(np.linalg.norm(end - origin))
            direction = (end - origin) / L.length
            L.dir_x, L.dir_y = float(direction[0]), float(direction[1])
            L.lat_x, L.lat_y = float(-direction[1]), float(direction[0])
            L.width, L.speed_limit = width, speed_limit
        return p

    # ------------------------------------------------------------------ device buffers
    def _allocate(self) -> None:
        n, dev = self.num_envs, self.device
        V = int(self._params.n_vehicles)
        vp = int(self._lib.hwy_highway_slot_stride(V))
        K = int(self._params.obs_vehicles_count)
        F = int(self._params.obs_n_features) or 5
        plugin_shape = tuple(self.observation_type.space().shape) if self._plugin_standalone else None  # per agent
        A = self.n_agents
        key = (n, vp, K, F, int(self._params.action_type), plugin_shape, self._linear, A, self.multi_action,
               self.multi_obs)
        if self._allocated_for == key:
            return
        z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=dev)  # noqa: E731
        self.V, self.vp, self.K = V, vp, K
        self._pos = z(n, vp, 2, dtype=torch.float64)
        self._hs = z(n, vp, 2, dtype=torch.float64)
        self._tt = z(n, vp, 2, dtype=torch.float64)
        self._imp = z(n, vp, 2, dtype=torch.float64)
        self._delta = z(n, vp, dtype=torch.float64)
        self._meta = z(n, vp, dtype=torch.int32)
        self._speed_index = z(n, A, dtype=torch.int32) if A > 1 or self.multi_agent else z(n, dtype=torch.int32)
        self._time = z(n, dtype=torch.float64)
        # what the step / reset kernels write (under MultiAgentObservation one Kinematics block per agent)
        KA = (A,) if self.multi_obs else ()
        self._fused_out = z(n, *KA, K, F, dtype=torch.float32) if plugin_shape is None else z(n, K, F, dtype=torch.float32)
        if plugin_shape is None:
            self._obs = self._fused_out
            self._final_obs = z(n, *KA, K, F, dtype=torch.float32)
        else:
            self._obs = z(n, *KA, *plugin_shape, dtype=torch.float32)
            self._final_obs = z(n, *KA, *plugin_shape, dtype=torch.float32)
        # TimeToCollision observing the first of several controlled vehicles reads its speed index from here
        self._speed_index0 = z(n, dtype=torch.int32) if A > 1 and not self.multi_obs else None
        self._plugin_view = None
        self._reward = z(n, dtype=torch.float64)
        self._terminated = z(n, dtype=torch.uint8)
        self._truncated = z(n, dtype=torch.uint8)
        self._info_speed = z(n, dtype=torch.float64)
        self._info_crashed = z(n, dtype=torch.uint8)
        self._reward_terms = z(n, N.HWY_REWARD_TERMS, dtype=torch.float64)
        AA = (A,) if self.multi_action else ()
        if self._params.action_type == 0:
            self._action_buf = z(n, *AA, dtype=torch.int32)
        else:
            self._action_buf = z(n, *AA, 2, dtype=torch.float32)
        st = N.HwyHighwayState()
        st.n_envs, st.vp = n, vp
        st.pos, st.hs, st.tt, st.imp = (t.data_ptr() for t in (self._pos, self._hs, self._tt, self._imp))
        st.delta, st.meta = self._delta.data_ptr(), self._meta.data_ptr()
        st.speed_index, st.time, st.rng = (
            self._speed_index.data_ptr(), self._time.data_ptr(), self._rng.data_ptr())
        st.reward_terms = self._reward_terms.data_ptr()
        self._state = st
        self._traffic = None
        if self._linear:  # per-vehicle ACCELERATION_PARAMETERS (3) + STEERING_PARAMETERS (2), see HwyLinearTraffic
            self._linear_params = z(n, vp, N.HWY_LINEAR_PARAMS, dtype=torch.float64)
            t = N.HwyLinearTraffic()
            t.params = self._linear_params.data_ptr()
            acc_lo, acc_span, steer_lo, steer_span = linear_ranges()
            t.acc_lo[:], t.acc_span[:] = [float(x) for x in acc_lo], [float(x) for x in acc_span]
            t.steer_lo[:], t.steer_span[:] = [float(x) for x in steer_lo], [float(x) for x in steer_span]
            self._traffic = t
        # the traffic argument of the reset / step / substeps entry points (None: IDMVehicle traffic)
        self._traffic_arg = None if self._traffic is None else C.byref(self._traffic)
        self._allocated_for = key

    # ------------------------------------------------------------------ family kernels
    def _reset(self, mask) -> None:
        self._device_reset(None if mask is None else mask.data_ptr(), None, self._fused_out.data_ptr())
        if self._plugin_standalone:
            self._observe_plugin(self._obs, mask)

    def _device_reset(self, mask_a, mask_b, obs_ptr) -> None:
        """Re-spawn the envs set in mask_a or mask_b (every env without masks) from their streams."""
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_highway_reset(C.byref(self._params), C.byref(self._state), self._traffic_arg,
                                                mask_a, mask_b, obs_ptr, self._stream()))

    def _step_kernels(self, act) -> None:
        ai = act.data_ptr() if self._params.action_type == 0 else None
        af = act.data_ptr() if self._params.action_type == 1 else None
        # the step kernel re-spawns finished envs itself unless a standalone plugin must observe the final state first
        fused_reset = self.autoreset_mode == "SameStep" and not self._plugin_standalone
        args = (ai, af, self._fused_out.data_ptr(), self._reward.data_ptr(), self._terminated.data_ptr(),
                self._truncated.data_ptr(), self._info_speed.data_ptr(), self._info_crashed.data_ptr(),
                N.AUTORESET_SAME_STEP if fused_reset else N.AUTORESET_DISABLED,
                self._final_obs.data_ptr() if fused_reset else None, self._stream())
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_highway_step(C.byref(self._params), C.byref(self._state), self._traffic_arg, *args))

    def _same_step_autoreset(self, info) -> None:
        if self._plugin_standalone:
            super()._same_step_autoreset(info)
        else:
            info["final_obs"] = self._out_final_obs()

    def _observe_kernel(self) -> None:
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_highway_observe(C.byref(self._params), C.byref(self._state),
                                                  self._fused_out.data_ptr(), self._stream()))

    def _obs_view(self):
        """The state as a HwyObsView + the lane table of RoadNetwork.straight_road_network
        (road/road.py:291-321) as a device HwyNetGraph."""
        if self._plugin_view is None:
            net = NetworkTable()
            for l in range(int(self._params.lanes_count)):
                L = self._params.lanes[l]
                net.add_straight("0", "1", [L.start_x, L.start_y],
                                 [L.start_x + L.length * L.dir_x, L.start_y + L.length * L.dir_y], width=L.width,
                                 speed_limit=L.speed_limit)
            net.finalize()
            self._plugin_graph = torch.from_numpy(
                np.frombuffer(bytes(net.to_struct()), dtype=np.uint8).copy()).to(self.device)
            v = N.HwyObsView()
            multi_obs = self.multi_obs and self.n_agents > 1
            v.n_envs, v.vp, v.n_vehicles, v.n_agents = self.num_envs, self.vp, self.V, self.n_agents if multi_obs else 0
            v.pos, v.hs, v.meta = self._pos.data_ptr(), self._hs.data_ptr(), self._meta.data_ptr()
            si = self._speed_index if self._speed_index0 is None else self._speed_index0
            v.speed_index = si.data_ptr()
            self._plugin_view = v
        return self._plugin_view, self._plugin_graph.data_ptr()

    def _observe_plugin(self, out, mask_a=None, mask_b=None) -> None:
        if self._speed_index0 is not None:  # the first controlled vehicle's column of [N, A]
            self._speed_index0.copy_(self._speed_index[:, 0])
        super()._observe_plugin(out, mask_a, mask_b)

    def ego_slots(self) -> list:
        """The slot of each controlled vehicle in the spawn layout of _create_vehicles (highway_env.py:72-98): bin k
        of near_split(vehicles_count, controlled_vehicles) is controlled vehicle k followed by its traffic."""
        return ego_slots(int(self._params.n_vehicles) - self.n_agents, self.n_agents)

    def get_available_actions(self) -> torch.Tensor:
        """DiscreteMetaAction.get_available_actions (envs/common/action.py:262-299, AbstractEnv.get_available_actions
        abstract.py:357-358) for every env at once: a bool mask [N, 5] over (LANE_LEFT, IDLE, LANE_RIGHT, FASTER,
        SLOWER).  A lane change is available when the side lane exists and `is_reachable_from` the ego's position
        (road/lane.py:104-118); FASTER / SLOWER unless the speed index sits at the end of `target_speeds`."""
        if self._params.action_type != 0:
            raise AttributeError("available actions are defined for DiscreteMetaAction only")
        lanes = [self._params.lanes[k] for k in range(int(self._params.lanes_count))]
        table = torch.tensor([[L.start_x, L.start_y, L.dir_x, L.dir_y, L.lat_x, L.lat_y, L.length, L.width] for L in lanes],
                             dtype=torch.float64, device=self._pos.device)
        si = self._speed_index.view(self.num_envs, -1).long()
        masks = []
        for a, slot in enumerate(self.ego_slots() if self.multi_action else [0]):
            lane = ((self._meta[:, slot] >> N.META_LANE_SHIFT) & 0xFF).long()
            masks.append(available_actions_mask(self._pos[:, slot, 0], self._pos[:, slot, 1], lane, si[:, a], table,
                                                int(self._params.n_target_speeds)))
        return torch.stack(masks, dim=1) if self.multi_action else masks[0]

    def road_substeps(self, n_substeps: int, action=None) -> None:
        """The reference's operator seam (`AbstractEnv._simulate` without `action_type.act`, abstract.py:304-307):
        `n_substeps` x (`Road.act()`; `Road.step(1 / simulation_frequency)`) on the device state and nothing else — no
        observation, reward, clock or autoreset.  The controlled vehicle acts like `ControlledVehicle.act(None)`; with
        ContinuousAction, `action` ([N, 2] in [-1, 1]; [N, A, 2] under MultiAgentAction) is the action dict the plain
        Vehicle keeps (default zeros)."""
        if not self._seeded:
            raise RuntimeError("call reset() before road_substeps()")
        af = None
        if action is not None:
            if self._params.action_type != 1:
                raise ValueError("action is only meaningful for a ContinuousAction ego")
            if getattr(self.action_type, "table", None) is not None:
                raise ValueError("pass the continuous (throttle, steering) pair, not a DiscreteAction index")
            af = self._stage_actions(action).data_ptr()
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_highway_substeps(C.byref(self._params), C.byref(self._state), self._traffic_arg,
                                                   int(n_substeps), af, self._stream()))

    def _env_rows(self) -> dict:
        rows = super()._env_rows()
        if self._traffic is not None:
            rows["_linear_params"] = self._linear_params
        return rows

    # ------------------------------------------------------------------ state import / export
    def state_dict(self) -> dict:
        """The base fields; with LinearVehicle traffic also every vehicle's ``acceleration_parameters`` [N, V, 3] and
        ``steering_parameters`` [N, V, 2] (zero for the controlled vehicle)."""
        sd = super().state_dict()
        if self._traffic is not None:
            lp = self._linear_params[:, :self.V].cpu().numpy()
            sd["acceleration_parameters"] = lp[..., :3].copy()
            sd["steering_parameters"] = lp[..., 3:].copy()
        return sd

    def load_state_dict(self, sd: dict, env_ids=None) -> None:
        """The base fields; with several controlled vehicles every env may hold at most `controlled_vehicles` slots of
        an MDPVehicle / Vehicle kind (their speed indices are [N, A])."""
        if self.n_agents > 1:
            kind = np.asarray(sd["kind"])
            n_ctrl = ((kind == N.KIND_MDP) | (kind == N.KIND_VEHICLE)).reshape(-1, kind.shape[-1]).sum(axis=1)
            if (n_ctrl > self.n_agents).any():
                raise ValueError(f"a state with more than controlled_vehicles = {self.n_agents} controlled vehicles "
                                 "in an env")
        super().load_state_dict(sd, env_ids)
        if self._traffic is not None and "acceleration_parameters" in sd:
            idx = slice(None) if env_ids is None else torch.from_numpy(np.asarray(env_ids, dtype=np.int64)).to(self.device)
            lp = np.concatenate([np.asarray(sd["acceleration_parameters"], dtype=np.float64),
                                 np.asarray(sd["steering_parameters"], dtype=np.float64)], axis=-1)
            self._linear_params[idx, :self.V] = torch.from_numpy(np.ascontiguousarray(lp)).to(self.device)


class BatchedHighwayEnvFast(BatchedHighwayEnv):
    """highway-fast-v0: 5 Hz simulation, 3 lanes, 20 vehicles, 30 s, and only the controlled
    vehicle checks collisions (reference envs/highway_env.py:154-182)."""

    ENV_ID = "highway-fast-v0"
    OTHERS_CHECK_COLLISIONS = False


def ego_slots(vehicles_count: int, controlled_vehicles: int) -> list:
    """Slots of the controlled vehicles: near_split(vehicles_count, num_bins=controlled_vehicles) (utils.py:355) gives
    the quotient, + 1 for the first `remainder` bins, and each bin is one controlled vehicle then its traffic."""
    q, r = divmod(int(vehicles_count), int(controlled_vehicles))
    return [k * (q + 1) + min(k, r) for k in range(int(controlled_vehicles))]


def available_actions_mask(x, y, lane, speed_index, lane_table, n_speeds: int, vehicle_length: float = 5.0):
    """Pure tensor form of DiscreteMetaAction.get_available_actions on a straight multi-lane road (any device).

    lane_table: [L, 8] = (start_x, start_y, dir_x, dir_y, lat_x, lat_y, length, width) per lane; returns bool [N, 5]
    in label order LANE_LEFT, IDLE, LANE_RIGHT, FASTER, SLOWER (action.py:204)."""
    n_lanes = lane_table.shape[0]
    out = torch.zeros((x.shape[0], 5), dtype=torch.bool, device=x.device)
    out[:, 1] = True  # IDLE
    for col, step in ((0, -1), (2, +1)):  # side_lanes: id - 1, id + 1 on the same road (road/road.py:200-211)
        side = lane + step
        exists = (side >= 0) & (side < n_lanes)
        t = lane_table[side.clamp(0, n_lanes - 1)]
        dx, dy = x - t[:, 0], y - t[:, 1]
        lon = dx * t[:, 2] + dy * t[:, 3]
        lat = dx * t[:, 4] + dy * t[:, 5]
        out[:, col] = exists & (lat.abs() <= 2 * t[:, 7]) & (lon >= 0) & (lon < t[:, 6] + vehicle_length)
    out[:, 3] = speed_index < n_speeds - 1
    out[:, 4] = speed_index > 0
    return out


from .common.host_stepper import HostStepper  # noqa: E402,F401  (re-export: the stepper serves every env family)
