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
from typing import Any, Optional, Sequence

import numpy as np
import torch

from .. import _native as N
from ..config import default_config
from ..spaces import batch_space
from .common.action import action_factory
from .common.observation import KinematicObservation, ObservationHost, observation_factory
from ..road.network import NetworkTable


def _pcg64_words(seeds: Sequence[int]) -> np.ndarray:
    """gymnasium seeding (np_random): Generator(PCG64(SeedSequence(seed))) -> [5, n] uint64."""
    out = np.zeros((5, len(seeds)), dtype=np.uint64)
    mask = (1 << 64) - 1
    for i, sd in enumerate(seeds):
        st = np.random.PCG64(np.random.SeedSequence(int(sd))).state
        s, inc = st["state"]["state"], st["state"]["inc"]
        out[0, i], out[1, i] = s >> 64, s & mask
        out[2, i], out[3, i] = inc >> 64, inc & mask
        out[4, i] = (int(st["has_uint32"]) << 32) | int(st["uinteger"])
    return out


class BatchedHighwayEnv(ObservationHost):
    """``num_envs`` independent highway roads stepped by the sm_90a kernels."""

    ENV_ID = "highway-v0"
    OTHERS_CHECK_COLLISIONS = True
    metadata = {"render_modes": [], "autoreset_mode": "SameStep"}

    PERCEPTION_DISTANCE = 5.0 * 40.0  # abstract.py:56
    REWARD_NAMES = ("collision_reward", "right_lane_reward", "high_speed_reward", "on_road_reward")  # _rewards :118-137
    _kernel_events = None  # bench.py hook: list of (start, end) CUDA events around the step kernels

    @classmethod
    def default_config(cls) -> dict:
        return default_config(cls.ENV_ID)

    def __init__(self, config: Optional[dict] = None, render_mode: Optional[str] = None,
                 num_envs: int = 1, device: Any = None, autoreset_mode: str = "SameStep",
                 env_index_offset: int = 0) -> None:
        if render_mode is not None:
            raise NotImplementedError("rendering is out of scope of the accelerated path (render_mode=None)")
        if not torch.cuda.is_available():
            raise RuntimeError("highwayenv_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self._lib = N.load()
        self.render_mode = None
        self.num_envs = int(num_envs)
        if self.num_envs < 1:
            raise ValueError("num_envs must be >= 1")
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.type != "cuda":
            raise RuntimeError("highwayenv_b200 only runs on CUDA devices")
        if autoreset_mode not in ("SameStep", "NextStep", "Disabled"):
            raise ValueError(f"autoreset_mode {autoreset_mode!r} (SameStep, NextStep, Disabled)")
        self.autoreset_mode = autoreset_mode
        self.env_index_offset = int(env_index_offset)
        self.config = self.default_config()
        self.configure(config)
        self._seeded = False
        self._allocated_for = None
        self.define_spaces()
        self._allocate()

    # ------------------------------------------------------------------ configuration
    def configure(self, config: Optional[dict]) -> None:
        """Shallow update, as the reference (abstract.py:127-129)."""
        if config:
            self.config.update(config)

    def define_spaces(self) -> None:
        """Plugin selection by ``config[...]["type"]`` (abstract.py:154-161)."""
        self.observation_type = observation_factory(self, self.config["observation"])
        self.action_type = action_factory(self, self.config["action"])
        # the step kernel's own epilogue is Kinematics; any other plugin runs its standalone kernel after the step
        # (envs/common/observation.py) while the kernel writes default Kinematics rows into a scratch buffer
        self._fused_obs = KinematicObservation() if self.observation_type.standalone else self.observation_type
        if hasattr(self.observation_type, "bind"):  # TimeToCollision: the observer's target speeds
            if not hasattr(self.action_type, "target_speeds"):
                raise ValueError("TimeToCollision needs an MDPVehicle observer (DiscreteMetaAction): "
                                 "compute_ttc_grid reads vehicle.target_speeds (finite_mdp.py:104-163)")
            self.observation_type.bind(self.config["policy_frequency"], self.action_type.target_speeds)
        self.single_observation_space = self.observation_type.space()
        self.single_action_space = self.action_type.space()
        self.observation_space = batch_space(self.single_observation_space, self.num_envs)
        self.action_space = batch_space(self.single_action_space, self.num_envs)
        self._params = self._build_params()

    def _build_params(self) -> N.HwyHighwayParams:
        cfg = self.config
        if cfg.get("controlled_vehicles", 1) != 1:
            raise NotImplementedError("controlled_vehicles != 1 (multi-agent) is not on the accelerated path")
        if cfg.get("other_vehicles_type") != "highway_env.vehicle.behavior.IDMVehicle":
            raise NotImplementedError("only IDMVehicle traffic is on the accelerated path")
        if cfg.get("neighbour_vehicles_connected_lanes"):
            raise NotImplementedError("connected-lane neighbour search (v1/v2 ids) is not implemented")
        if cfg.get("manual_control"):
            raise NotImplementedError("manual_control")
        p = N.HwyHighwayParams()
        lanes = int(cfg["lanes_count"])
        if not 1 <= lanes <= N.HWY_MAX_LANES:
            raise ValueError(f"lanes_count must be in 1..{N.HWY_MAX_LANES}")
        p.lanes_count = lanes
        p.n_vehicles = int(cfg["vehicles_count"]) + 1
        if p.n_vehicles > N.HWY_MAX_VEHICLES:
            raise ValueError(f"vehicles_count must be <= {N.HWY_MAX_VEHICLES - 1}")
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
        plugin_shape = tuple(self.single_observation_space.shape) if self.observation_type.standalone else None
        key = (n, vp, K, F, int(self._params.action_type), plugin_shape)
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
        self._speed_index = z(n, dtype=torch.int32)
        self._time = z(n, dtype=torch.float64)
        self._rng = z(5, n, dtype=torch.int64)  # uint64 words, bit-cast
        self._fused_out = z(n, K, F, dtype=torch.float32)  # what the step / reset kernels write
        if plugin_shape is None:
            self._obs = self._fused_out
            self._final_obs = z(n, K, F, dtype=torch.float32)
        else:
            self._obs = z(n, *plugin_shape, dtype=torch.float32)
            self._final_obs = z(n, *plugin_shape, dtype=torch.float32)
        self._plugin_view = None
        self._reward = z(n, dtype=torch.float64)
        self._terminated = z(n, dtype=torch.uint8)
        self._truncated = z(n, dtype=torch.uint8)
        self._info_speed = z(n, dtype=torch.float64)
        self._info_crashed = z(n, dtype=torch.uint8)
        self._reward_terms = z(n, N.HWY_REWARD_TERMS, dtype=torch.float64)
        if self._params.action_type == 0:
            self._action_buf = z(n, dtype=torch.int32)
        else:
            self._action_buf = z(n, 2, dtype=torch.float32)
        st = N.HwyHighwayState()
        st.n_envs, st.vp = n, vp
        st.pos, st.hs, st.tt, st.imp = (t.data_ptr() for t in (self._pos, self._hs, self._tt, self._imp))
        st.delta, st.meta = self._delta.data_ptr(), self._meta.data_ptr()
        st.speed_index, st.time, st.rng = (
            self._speed_index.data_ptr(), self._time.data_ptr(), self._rng.data_ptr())
        st.reward_terms = self._reward_terms.data_ptr()
        self._state = st
        self._allocated_for = key
        self._seeded = False

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    # ------------------------------------------------------------------ gym API
    def _seed_streams(self, seed) -> None:
        if seed is None:
            ss = np.random.SeedSequence()
            seeds = [int(s.generate_state(1)[0]) for s in ss.spawn(self.num_envs)]
        elif isinstance(seed, (int, np.integer)):
            seeds = [int(seed) + self.env_index_offset + i for i in range(self.num_envs)]
        else:
            seeds = [int(s) for s in seed]
            if len(seeds) != self.num_envs:
                raise ValueError("seed sequence must have num_envs entries")
        words = _pcg64_words(seeds)
        self._rng.copy_(torch.from_numpy(words.view(np.int64)).to(self.device))
        self.np_random_seed = seeds
        self._seeded = True

    def reset(self, *, seed=None, options: Optional[dict] = None):
        """Reset every env (or ``options["reset_mask"]``); returns (obs [N,K,5] f32, info)."""
        if options and "config" in options:
            self.configure(options["config"])
            self.define_spaces()
            self._allocate()
        if seed is not None or not self._seeded:
            self._seed_streams(seed)
        mask_ptr = None
        if options and options.get("reset_mask") is not None:
            mask = torch.as_tensor(options["reset_mask"]).to(device=self.device, dtype=torch.uint8).contiguous()
            if mask.shape != (self.num_envs,):
                raise ValueError("reset_mask must have shape (num_envs,)")
            self._mask_keepalive = mask
            mask_ptr = mask.data_ptr()
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_highway_reset(C.byref(self._params), C.byref(self._state), mask_ptr,
                                                self._fused_out.data_ptr(), self._stream()))
        if self.observation_type.standalone:
            self._observe_plugin(self._obs, None if mask_ptr is None else self._mask_keepalive)
        self._autoreset_envs = None
        info = {"speed": self._hs[:, 0, 1], "crashed": (self._meta[:, 0] & N.META_CRASHED) != 0}
        return self._out_obs(), info

    def _stage_actions(self, actions) -> torch.Tensor:
        buf = self._action_buf
        table = getattr(self.action_type, "table", None)
        if table is not None:  # DiscreteAction (action.py:165-196): index -> (throttle, steering), then ContinuousAction
            if getattr(self, "_action_table", None) is None or self._action_table.device != buf.device:
                self._action_table = torch.from_numpy(table).to(buf.device)
            idx = actions if isinstance(actions, torch.Tensor) else torch.from_numpy(np.asarray(actions))
            idx = idx.to(device=buf.device, dtype=torch.long).reshape(-1)
            if idx.numel() != buf.shape[0]:
                raise ValueError("one action per env")
            # (the check reads the device: not under CUDA-graph capture — HostStepper checks its host array instead)
            if not torch.cuda.is_current_stream_capturing() and bool(((idx < 0) | (idx >= table.shape[0])).any()):
                raise IndexError("list index out of range")  # all_actions[action] in the reference
            torch.index_select(self._action_table, 0, idx, out=buf)
            return buf
        if isinstance(actions, torch.Tensor):
            if actions.device == buf.device and actions.dtype == buf.dtype and actions.is_contiguous() \
                    and actions.shape == buf.shape:
                return actions
            buf.copy_(actions.reshape(buf.shape), non_blocking=True)
            return buf
        a = np.asarray(actions)
        buf.copy_(torch.from_numpy(np.ascontiguousarray(a.reshape(tuple(buf.shape)))).to(buf.dtype),
                  non_blocking=True)
        return buf

    def step(self, actions):
        """One policy step of all envs.

        ``actions``: [N] integers (DiscreteMetaAction) or [N, 2] float32 (ContinuousAction);
        device tensors are used in place.  Returns device tensors
        ``(obs [N,K,F] f32, reward [N] f64, terminated [N] bool, truncated [N] bool, info)``;
        the buffers are reused by the next call.
        """
        if not self._seeded:
            raise RuntimeError("call reset() before step()")
        act = self._stage_actions(actions)
        ai = act.data_ptr() if self._params.action_type == 0 else None
        af = act.data_ptr() if self._params.action_type == 1 else None
        same_step = self.autoreset_mode == "SameStep"
        plugin = self.observation_type.standalone
        fused_reset = same_step and not plugin  # a standalone plugin must observe the final state before the reset
        kev = self._kernel_events
        if kev is not None:  # bench.py: CUDA events around the step kernel(s) alone
            kev.append((torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)))
            kev[-1][0].record(torch.cuda.current_stream(self.device))
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_highway_step(
                C.byref(self._params), C.byref(self._state), ai, af, self._fused_out.data_ptr(),
                self._reward.data_ptr(), self._terminated.data_ptr(), self._truncated.data_ptr(),
                self._info_speed.data_ptr(), self._info_crashed.data_ptr(),
                N.AUTORESET_SAME_STEP if fused_reset else N.AUTORESET_DISABLED,
                self._final_obs.data_ptr() if fused_reset else None, self._stream()))
        if kev is not None:
            kev[-1][1].record(torch.cuda.current_stream(self.device))
        # AbstractEnv._info (abstract.py:200-217): speed, crashed, action and the un-weighted reward terms of _rewards
        info = {"speed": self._info_speed, "crashed": self._info_crashed.view(torch.bool), "action": act,
                "rewards": {name: self._reward_terms[:, k] for k, name in enumerate(self.REWARD_NAMES)}}
        if plugin:
            self._observe_plugin(self._obs)
            if same_step:  # observe, keep as final_obs, re-spawn the finished envs, observe those again
                self._final_obs.copy_(self._obs)
                with torch.cuda.device(self.device):
                    N.check(self._lib.hwy_highway_autoreset(
                        C.byref(self._params), C.byref(self._state), self._terminated.data_ptr(),
                        self._truncated.data_ptr(), self._fused_out.data_ptr(), self._stream()))
                self._observe_plugin(self._obs, self._terminated, self._truncated)
        if same_step:
            info["final_obs"] = self._final_obs
        elif self.autoreset_mode == "NextStep":
            self._next_step_autoreset()
        return (self._out_obs(), self._reward, self._terminated.view(torch.bool),
                self._truncated.view(torch.bool), info)

    def _out_obs(self) -> torch.Tensor:
        if getattr(self.observation_type, "as_image", False):  # OccupancyGrid(as_image=True): uint8 (observation.py:336-338)
            return self._obs.to(torch.uint8)
        return self._obs

    def _obs_view(self):
        """ObservationHost: the state as a HwyObsView + the lane table of RoadNetwork.straight_road_network
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
            v.n_envs, v.vp, v.n_vehicles, v.n_agents = self.num_envs, self.vp, self.V, 0
            v.pos, v.hs, v.meta = self._pos.data_ptr(), self._hs.data_ptr(), self._meta.data_ptr()
            v.speed_index = self._speed_index.data_ptr()
            self._plugin_view = v
        return self._plugin_view, self._plugin_graph.data_ptr()

    def _next_step_autoreset(self) -> None:
        """gymnasium AutoresetMode.NEXT_STEP (the vector default): an env that ended in the previous step is
        reset by this call instead of stepped — reset observation, reward 0, both flags False.  The step
        kernel has already advanced those envs; their state is simply replaced by the masked device reset
        (stepping draws nothing from the env's generator on this road family)."""
        prev = getattr(self, "_autoreset_envs", None)
        if prev is not None:
            with torch.cuda.device(self.device):
                N.check(self._lib.hwy_highway_reset(C.byref(self._params), C.byref(self._state), prev.data_ptr(),
                                                    self._fused_out.data_ptr(), self._stream()))
            if self.observation_type.standalone:
                self._observe_plugin(self._obs, prev)
            keep = prev == 0
            self._reward.mul_(keep)
            self._terminated.mul_(keep)
            self._truncated.mul_(keep)
        self._autoreset_envs = (self._terminated | self._truncated).contiguous()

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
        lane = ((self._meta[:, 0] >> N.META_LANE_SHIFT) & 0xFF).long()
        return available_actions_mask(self._pos[:, 0, 0], self._pos[:, 0, 1], lane, self._speed_index.long(), table,
                                      int(self._params.n_target_speeds))

    def road_substeps(self, n_substeps: int, action=None) -> None:
        """The reference's operator seam (`AbstractEnv._simulate` without `action_type.act`, abstract.py:304-307):
        `n_substeps` x (`Road.act()`; `Road.step(1 / simulation_frequency)`) on the device state and nothing else — no
        observation, reward, clock or autoreset.  The controlled vehicle acts like `ControlledVehicle.act(None)`; with
        ContinuousAction, `action` ([N, 2] in [-1, 1]) is the action dict the plain Vehicle keeps (default zeros)."""
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
            N.check(self._lib.hwy_highway_substeps(C.byref(self._params), C.byref(self._state), int(n_substeps), af,
                                                   self._stream()))

    def host_stepper(self) -> "HostStepper":
        """Host-buffer stepping through one CUDA graph (see HostStepper)."""
        return HostStepper(self)

    def observe(self) -> torch.Tensor:
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_highway_observe(C.byref(self._params), C.byref(self._state),
                                                  self._fused_out.data_ptr(), self._stream()))
        if self.observation_type.standalone:
            self._observe_plugin(self._obs)
        return self._out_obs()

    def close(self) -> None:
        pass

    @property
    def unwrapped(self):
        return self

    # ------------------------------------------------------------------ state import / export
    STATE_FIELDS = ("x", "y", "heading", "speed", "target_speed", "timer", "delta", "impact_x",
                    "impact_y", "lane", "target_lane", "kind", "crashed", "has_impact",
                    "check_collisions", "speed_index", "time")

    def state_dict(self) -> dict:
        """Per-field numpy arrays [N, V] (the reference's per-vehicle attributes)."""
        V = self.V
        pos, hs, tt, imp = (t[:, :V].cpu().numpy() for t in (self._pos, self._hs, self._tt, self._imp))
        meta = self._meta[:, :V].cpu().numpy()
        return {
            "x": pos[..., 0].copy(), "y": pos[..., 1].copy(),
            "heading": hs[..., 0].copy(), "speed": hs[..., 1].copy(),
            "target_speed": tt[..., 0].copy(), "timer": tt[..., 1].copy(),
            "delta": self._delta[:, :V].cpu().numpy(),
            "impact_x": imp[..., 0].copy(), "impact_y": imp[..., 1].copy(),
            "lane": (meta >> N.META_LANE_SHIFT) & 0xFF,
            "target_lane": (meta >> N.META_TARGET_SHIFT) & 0xFF,
            "kind": (meta >> N.META_KIND_SHIFT) & 3,
            "crashed": (meta & N.META_CRASHED) != 0,
            "has_impact": (meta & N.META_HAS_IMPACT) != 0,
            "check_collisions": (meta & N.META_CHECK_COLLISIONS) != 0,
            "speed_index": self._speed_index.cpu().numpy(),
            "time": self._time.cpu().numpy(),
            "rng": self._rng.cpu().numpy().view(np.uint64),
        }

    def load_state_dict(self, sd: dict) -> None:
        """Inverse of :meth:`state_dict` (how oracle / reference states are injected)."""
        n, V, dev = self.num_envs, self.V, self.device
        f = lambda k: torch.from_numpy(np.ascontiguousarray(sd[k], dtype=np.float64)).to(dev)  # noqa: E731
        self._pos[:, :V, 0], self._pos[:, :V, 1] = f("x"), f("y")
        self._hs[:, :V, 0], self._hs[:, :V, 1] = f("heading"), f("speed")
        self._tt[:, :V, 0], self._tt[:, :V, 1] = f("target_speed"), f("timer")
        self._imp[:, :V, 0], self._imp[:, :V, 1] = f("impact_x"), f("impact_y")
        self._delta[:, :V] = f("delta")
        meta = (
            (np.asarray(sd["lane"], dtype=np.int64) << N.META_LANE_SHIFT)
            | (np.asarray(sd["target_lane"], dtype=np.int64) << N.META_TARGET_SHIFT)
            | (np.asarray(sd["kind"], dtype=np.int64) << N.META_KIND_SHIFT)
            | np.where(np.asarray(sd["crashed"], dtype=bool), N.META_CRASHED, 0)
            | np.where(np.asarray(sd["has_impact"], dtype=bool), N.META_HAS_IMPACT, 0)
            | np.where(np.asarray(sd["check_collisions"], dtype=bool), N.META_CHECK_COLLISIONS, 0)
            | N.META_PRESENT
        ).astype(np.int32)
        self._meta[:, :V] = torch.from_numpy(meta.reshape(n, V)).to(dev)
        self._speed_index.copy_(torch.from_numpy(np.asarray(sd["speed_index"], dtype=np.int32).reshape(n)))
        self._time.copy_(torch.from_numpy(np.asarray(sd["time"], dtype=np.float64).reshape(n)))
        if "rng" in sd:
            self._rng.copy_(torch.from_numpy(np.ascontiguousarray(sd["rng"]).view(np.int64)))
        self._seeded = True


class BatchedHighwayEnvFast(BatchedHighwayEnv):
    """highway-fast-v0: 5 Hz simulation, 3 lanes, 20 vehicles, 30 s, and only the controlled
    vehicle checks collisions (reference envs/highway_env.py:154-182)."""

    ENV_ID = "highway-fast-v0"
    OTHERS_CHECK_COLLISIONS = False


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
