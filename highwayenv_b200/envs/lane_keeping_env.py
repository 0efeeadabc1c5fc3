"""Batched lane-keeping-v0 on the H100 backend.

Host-side mirror of the reference's ``LaneKeepingEnv`` (highway_env/envs/lane_keeping_env.py): one dynamical
``BicycleVehicle`` per env steers along a SineLane with no traffic, a ContinuousAction on the steering (and optionally
the throttle), and a noisy ``AttributesObservation`` — a Dict of float64 (4, 1) arrays drawn from the env's numpy stream.
The registration's ``TimeLimit(max_episode_steps=200)`` is the only end of an episode: ``terminated`` is always False.

Step and reset run in ``hwy_lane_keeping_step`` / ``hwy_lane_keeping_reset`` (csrc/hwy_lane_keeping.cu), one thread per
env; with SameStep autoreset the step kernel also writes the final observation and resets the truncated envs.
Observations are a dict of [N, 4, 1] float64 views of one [N, n_attr, 4, 1] buffer, in the configured attribute order.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from .. import _native as N
from ..road.network import NetworkTable
from ..spaces import Box, Dict, batch_space
from .common.vector_env import BatchedVectorEnv

MAX_EPISODE_STEPS = 200  # highway_env/__init__.py:89-92
STATE_FIELDS = ("x", "y", "heading", "speed", "lateral_speed", "yaw_rate")  # BicycleVehicle.state (dynamics.py:57-68)


def make_lane_keeping_network() -> NetworkTable:
    """LaneKeepingEnv._make_road (lane_keeping_env.py:88-127): the sine lane a -> b and the straight lane c -> d the
    episode starts on.  The reference's third lane d -> a is never the env's lane and nothing on this road reads the
    vehicle's own closest lane, so it is left out."""
    net = NetworkTable()
    net.add_straight("a", "b", [0, 0], [500, 0], width=10, sine=(5, 2 * np.pi / 100, 0))
    net.add_straight("c", "d", [50, 50], [115, 15], width=10)
    net.finalize()
    return net


def lane_keeping_params(cfg: dict, autoreset_mode: str = "SameStep") -> N.HwyLaneKeepingParams:
    """The kernel parameters of a lane-keeping-v0 configuration.  Every unsupported input raises here, before any
    launch: other observation or action types, unknown attributes, dynamical=False (the reference's observation reads
    BicycleVehicle.derivative, so a kinematic Vehicle fails there with AttributeError), speed_range, manual_control."""
    obs, act = cfg["observation"], cfg["action"]
    if obs["type"] != "AttributesObservation":
        raise NotImplementedError(f"observation type {obs['type']!r} on lane-keeping-v0 (AttributesObservation)")
    attributes = list(obs["attributes"])
    unknown = [a for a in attributes if a not in N.LK_ATTRIBUTES]
    if unknown:
        raise ValueError(f"unknown attributes {unknown} (state, derivative, reference_state)")
    if not attributes or len(set(attributes)) != len(attributes):
        raise ValueError("attributes must be a non-empty list without repeats")
    if act["type"] != "ContinuousAction":
        raise NotImplementedError(f"action type {act['type']!r} on lane-keeping-v0 (ContinuousAction)")
    if not act.get("dynamical", False):
        raise NotImplementedError("lane-keeping-v0 needs the dynamical BicycleVehicle (dynamical=True)")
    if act.get("speed_range") is not None:
        raise NotImplementedError("speed_range (per-vehicle MIN/MAX_SPEED override) is not supported")
    longi, lat = bool(act.get("longitudinal", True)), bool(act.get("lateral", True))
    if not (longi or lat):
        raise ValueError("Either longitudinal and/or lateral control must be enabled")  # action.py:120-123
    sf, pf = int(cfg["simulation_frequency"]), int(cfg["policy_frequency"])
    if sf < 1 or pf < 1 or sf // pf < 1:
        raise ValueError("simulation_frequency and policy_frequency must be >= 1, policy_frequency <= "
                         "simulation_frequency")
    if cfg.get("manual_control"):
        raise NotImplementedError("manual_control")
    acc_range = tuple(act.get("acceleration_range") or (-5, 5.0))  # ContinuousAction.ACCELERATION_RANGE
    steer_range = tuple(act.get("steering_range") or (-np.pi / 4, np.pi / 4))
    net = make_lane_keeping_network()
    lane_cd, lane_ab = net.index[("c", "d", 0)], net.index[("a", "b", 0)]
    graph = net.to_struct()
    p = N.HwyLaneKeepingParams()
    p.frames = sf // pf
    p.dt = 1 / sf
    p.n_attr = len(attributes)
    for k, a in enumerate(attributes):
        p.attr[k] = N.LK_ATTRIBUTES[a]
    p.longitudinal, p.lateral, p.act_clip = int(longi), int(lat), int(bool(act.get("clip", True)))
    p.acc_lo, p.acc_hi = float(acc_range[0]), float(acc_range[1])
    p.steer_lo, p.steer_hi = float(steer_range[0]), float(steer_range[1])
    p.state_noise, p.derivative_noise = float(cfg["state_noise"]), float(cfg["derivative_noise"])
    p.max_episode_steps = MAX_EPISODE_STEPS
    p.autoreset = N.AUTORESET_SAME_STEP if autoreset_mode == "SameStep" else N.AUTORESET_DISABLED
    # _make_vehicles (:129-138): lane_cd.position(50, -4), heading lane_cd.heading_at(0), speed 8.3
    x0, y0 = net.position(lane_cd, 50.0, -4.0)
    p.x0, p.y0 = float(x0), float(y0)
    p.heading0, p.speed0 = float(net.heading_at(lane_cd, 0.0)), 8.3
    p.lanes[0], p.lanes[1] = graph.lanes[lane_cd], graph.lanes[lane_ab]
    return p


class BatchedLaneKeepingEnv(BatchedVectorEnv):
    ENV_ID = "lane-keeping-v0"
    REWARD_NAMES = ()
    V = 1
    NEXT_STEP_REWINDS_RNG = True  # every step draws the observation noise, also in envs NextStep then resets
    ROW_EXCLUDE = BatchedVectorEnv.ROW_EXCLUDE | {"_crashed"}

    # ------------------------------------------------------------------ spaces / parameters
    def define_spaces(self) -> None:
        p = lane_keeping_params(self.config, self.autoreset_mode)
        self._params = p
        self.attributes = tuple(self.config["observation"]["attributes"])
        self.action_type = None
        self.single_observation_space = Dict(
            {a: Box(-np.inf, np.inf, shape=(4, 1), dtype=np.float64) for a in self.attributes})
        self.single_action_space = Box(-1.0, 1.0, shape=(p.longitudinal + p.lateral,), dtype=np.float32)
        self.observation_space = batch_space(self.single_observation_space, self.num_envs)
        self.action_space = batch_space(self.single_action_space, self.num_envs)

    def _allocate(self) -> None:
        n, dev = self.num_envs, self.device
        z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=dev)  # noqa: E731
        self._state = z(6, n, dtype=torch.float64)
        self._lane_phase, self._elapsed = z(n, dtype=torch.int32), z(n, dtype=torch.int32)
        self._obs = z(n, len(self.attributes), 4, 1, dtype=torch.float64)
        self._final_obs = torch.zeros_like(self._obs)
        self._fused_out = self._obs
        self._reward = z(n, dtype=torch.float64)
        self._terminated, self._truncated = z(n, dtype=torch.uint8), z(n, dtype=torch.uint8)
        self._action_buf = z(n, self.single_action_space.shape[0], dtype=torch.float32)
        self._crashed = z(n, dtype=torch.bool)  # the vehicle is alone on the road: it never crashes
        self._plugin_standalone = False
        s = N.HwyLaneKeepingState()
        s.n_envs = n
        s.state, s.lane_phase, s.elapsed = self._state.data_ptr(), self._lane_phase.data_ptr(), self._elapsed.data_ptr()
        s.rng = self._rng.data_ptr()
        self._lk_state = s

    # ------------------------------------------------------------------ family kernels
    def _device_reset(self, mask_a, mask_b, obs_ptr) -> None:
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_lane_keeping_reset(C.byref(self._params), C.byref(self._lk_state), mask_a, mask_b,
                                                     obs_ptr, self._stream()))

    def _reset(self, mask) -> None:
        self._device_reset(None if mask is None else mask.data_ptr(), None, self._obs.data_ptr())

    def _step_kernels(self, act) -> None:
        with torch.cuda.device(self.device):
            N.check(self._lib.hwy_lane_keeping_step(
                C.byref(self._params), C.byref(self._lk_state), act.data_ptr(), self._obs.data_ptr(),
                self._final_obs.data_ptr(), self._reward.data_ptr(), self._terminated.data_ptr(),
                self._truncated.data_ptr(), self._stream()))

    def _reset_info(self) -> dict:
        return {"speed": self._state[3], "crashed": self._crashed}

    def _step_info(self, act) -> dict:
        return {}  # LaneKeepingEnv.step returns info = {}

    def _same_step_autoreset(self, info) -> None:
        # the step kernel has written the final observation of the truncated envs and reset them
        info["final_obs"] = self._out_final_obs()

    def _as_dict(self, t: torch.Tensor) -> dict:
        return {a: t[:, k] for k, a in enumerate(self.attributes)}

    def _out_obs(self) -> dict:
        return self._as_dict(self._obs)

    def _out_final_obs(self) -> dict:
        """Rows of the envs truncated by this step; the other rows hold an earlier final observation."""
        return self._as_dict(self._final_obs)

    # ------------------------------------------------------------------ what this env does not have
    def observe(self):
        raise NotImplementedError("lane-keeping-v0 draws its observation noise from the env's stream: the observation "
                                  "comes from reset() and step() only")

    def to_finite_mdp(self):
        raise NotImplementedError("to_finite_mdp needs an MDPVehicle ego on a road with traffic; lane-keeping-v0 has "
                                  "a BicycleVehicle alone")

    def get_available_actions(self):
        raise NotImplementedError("get_available_actions is a DiscreteMetaAction method; lane-keeping-v0 uses "
                                  "ContinuousAction")

    # ------------------------------------------------------------------ cloning / state import / export
    def _env_rows(self) -> dict:
        rows = {"_state": self._state.t(), "_lane_phase": self._lane_phase, "_elapsed": self._elapsed,
                "_rng": self._rng.t(), "_obs": self._obs}
        if self._autoreset_envs is not None:
            rows["_autoreset_envs"] = self._autoreset_envs
        return rows

    def state_dict(self) -> dict:
        """BicycleVehicle.state as [N] float64 arrays, the lane phase (0: on c -> d with the sine lane queued, 1: on
        the sine lane), the steps since the last reset and the stream words [5, N]."""
        st = self._state.cpu().numpy()
        sd = {k: st[j].copy() for j, k in enumerate(STATE_FIELDS)}
        sd["lane_phase"] = self._lane_phase.cpu().numpy()
        sd["elapsed_steps"] = self._elapsed.cpu().numpy()
        sd["rng"] = self._rng.cpu().numpy().view(np.uint64)
        return sd

    def load_state_dict(self, sd: dict, env_ids=None) -> None:
        """Inverse of :meth:`state_dict` for every env or the rows `env_ids`.  An env never seeded is first seeded as
        reset(seed=0) would; `sd["rng"]` then replaces the words."""
        dev = self.device
        idx = slice(None) if env_ids is None else torch.from_numpy(np.asarray(env_ids, dtype=np.int64)).to(dev)
        st = np.stack([np.asarray(sd[k], dtype=np.float64).reshape(-1) for k in STATE_FIELDS])
        self._state[:, idx] = torch.from_numpy(st).to(dev)
        self._lane_phase[idx] = torch.from_numpy(np.asarray(sd["lane_phase"], dtype=np.int32).reshape(-1)).to(dev)
        self._elapsed[idx] = torch.from_numpy(np.asarray(sd["elapsed_steps"], dtype=np.int32).reshape(-1)).to(dev)
        if not self._seeded:
            self._seed_streams(0)
        if "rng" in sd:
            w = np.ascontiguousarray(sd["rng"], dtype=np.uint64).reshape(5, -1)
            self._rng[:, idx] = torch.from_numpy(w.view(np.int64)).to(dev)
