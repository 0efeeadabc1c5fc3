"""Observation plugins of the batched backend: ONE registry for every env family.

Mirror of the reference's ``observation_factory`` (highway_env/envs/common/observation.py:772-794), which builds any
``ObservationType`` on any env.  Here a plugin is a host-side descriptor (constructor arguments, ``space()``) plus a
device observer:

* every env family has a *fused* observation written by its step kernel (Kinematics on the straight-highway
  family; Kinematics / default OccupancyGrid / TimeToCollision on the general-network family) — the fast path the
  BASELINE configs use;
* every other (env, observation) pair steps with the family's cheapest fused observation into a scratch buffer and
  then runs the plugin's *standalone* kernel (``hwy_observe_grid`` / ``hwy_observe_ttc`` / ``hwy_observe_lidar``,
  include/hwyb200.h) on the device state — any plugin on any env, as in the reference.

The env side of the contract is ``BatchedVectorEnv._obs_view`` (envs/common/vector_env.py).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from ... import _native as N
from ...spaces import Box


class ObservationType:
    """Host-side descriptor of one observation plugin."""

    standalone = False  # True: observed by its own kernel after the step (BatchedVectorEnv._observe_plugin)

    def space(self):
        raise NotImplementedError

    def fill_params(self, p) -> None:  # fused plugins of the highway family
        raise NotImplementedError

    def observe(self, env, out: torch.Tensor, mask_a=None, mask_b=None) -> None:  # standalone plugins
        raise NotImplementedError


class KinematicObservation(ObservationType):
    """Kinematics of the ego and its nearest vehicles (reference observation.py:155-276):
    row 0 is the ego, the others the closest vehicles by |longitudinal distance on the ego's lane|
    within PERCEPTION_DISTANCE; columns are any of `Vehicle.to_dict`'s keys (vehicle/kinematics.py:237-261):
    presence, x, y, vx, vy, heading, cos_h, sin_h, cos_d, sin_d, long_off, lat_off, ang_off, with an
    optional `features_range` (every listed feature present in the table is mapped to [-1, 1])."""

    FEATURES = ["presence", "x", "y", "vx", "vy"]

    def __init__(self, features=None, vehicles_count: int = 5, features_range=None,
                 absolute: bool = False, order: str = "sorted", normalize: bool = True,
                 clip: bool = True, see_behind: bool = False, observe_intentions: bool = False,
                 include_obstacles: bool = True, **kwargs):
        self.features = list(features) if features else list(self.FEATURES)
        unknown = [f for f in self.features if f not in N.FEATURE_CODES]
        if unknown:
            raise KeyError(f"{unknown} not in index")  # what `df[self.features]` raises in the reference
        if len(self.features) > N.HWY_MAX_OBS_FEATURES:
            raise ValueError(f"at most {N.HWY_MAX_OBS_FEATURES} features")
        self.features_range = None if features_range is None else {k: [float(v[0]), float(v[1])]
                                                                   for k, v in features_range.items()}
        if order != "sorted":
            raise NotImplementedError("order='shuffled' draws from env.np_random on the host")
        if not 1 <= int(vehicles_count) <= N.HWY_MAX_OBS_VEHICLES:
            raise ValueError(f"vehicles_count must be in 1..{N.HWY_MAX_OBS_VEHICLES}")
        self.vehicles_count = int(vehicles_count)
        self.absolute, self.normalize, self.clip = bool(absolute), bool(normalize), bool(clip)
        self.see_behind = bool(see_behind)

    def space(self):
        return Box(low=-np.inf, high=np.inf, shape=(self.vehicles_count, len(self.features)),
                   dtype=np.float32)

    def fill_params(self, p):
        p.obs_vehicles_count = self.vehicles_count
        p.obs_see_behind = int(self.see_behind)
        p.obs_absolute = int(self.absolute)
        p.obs_normalize = int(self.normalize)
        p.obs_clip = int(self.clip)
        if self.features == self.FEATURES and self.features_range is None:
            p.obs_n_features = 0  # default columns and ranges: the specialised epilogue
            return
        ranges = self.features_range
        if ranges is None:  # normalize_obs (observation.py:214-226): side lanes of the straight road = lanes_count
            ranges = {"x": [-5.0 * 40.0, 5.0 * 40.0], "y": [-4.0 * p.lanes_count, 4.0 * p.lanes_count],
                      "vx": [-2 * 40.0, 2 * 40.0], "vy": [-2 * 40.0, 2 * 40.0]}
        p.obs_n_features = len(self.features)
        for c, f in enumerate(self.features):
            p.obs_feature[c] = N.FEATURE_CODES[f]
            p.obs_feature_ranged[c] = int(f in ranges)
            if f in ranges:
                p.obs_feature_lo[c], p.obs_feature_hi[c] = ranges[f]


class _Standalone(ObservationType):
    standalone = True

    @staticmethod
    def _ptr(t):
        return None if t is None else t.data_ptr()


class OccupancyGridObservation(_Standalone):
    """OccupancyGridObservation (reference observation.py:279-499): a grid of cells around the observer with one
    layer per feature (any `Vehicle.to_dict` key, or `on_road`), `grid_size` / `grid_step`, optional
    `features_range`, `align_to_vehicle_axes`, `clip`, `as_image`.  `absolute=True` raises NotImplementedError in the
    reference too (:362-363)."""

    FEATURES = ["presence", "vx", "vy", "on_road"]
    GRID_SIZE = [[-5.5 * 5, 5.5 * 5], [-5.5 * 5, 5.5 * 5]]
    GRID_STEP = [5, 5]

    def __init__(self, features=None, grid_size=None, grid_step=None, features_range=None, absolute: bool = False,
                 align_to_vehicle_axes: bool = False, clip: bool = True, as_image: bool = False, **kwargs):
        self.features = list(features) if features is not None else list(self.FEATURES)
        if len(self.features) > N.HWY_MAX_OBS_FEATURES:
            raise ValueError(f"at most {N.HWY_MAX_OBS_FEATURES} grid features")
        self.grid_size = np.array(grid_size if grid_size is not None else self.GRID_SIZE, dtype=np.float64)
        self.grid_step = np.array(grid_step if grid_step is not None else self.GRID_STEP, dtype=np.float64)
        self.grid_shape = tuple(int(v) for v in np.asarray(
            np.floor((self.grid_size[:, 1] - self.grid_size[:, 0]) / self.grid_step), dtype=np.intp))
        self.features_range = features_range
        if absolute:
            raise NotImplementedError()  # as the reference's observe() (:362-363)
        self.align_to_vehicle_axes, self.clip, self.as_image = bool(align_to_vehicle_axes), bool(clip), bool(as_image)

    @property
    def is_default(self) -> bool:
        """The configuration the network step kernels write themselves (BASELINE config 3)."""
        return (self.features == self.FEATURES and self.grid_shape == (11, 11) and not self.features_range
                and np.array_equal(self.grid_size, np.array(self.GRID_SIZE)) and np.array_equal(self.grid_step, [5, 5])
                and not self.align_to_vehicle_axes and self.clip and not self.as_image)

    def space(self):
        shape = (len(self.features),) + self.grid_shape
        if self.as_image:
            return Box(low=0, high=255, shape=shape, dtype=np.uint8)
        return Box(low=-np.inf, high=np.inf, shape=shape, dtype=np.float32)

    def params(self) -> N.HwyGridParams:
        p = N.HwyGridParams()
        fr = self.features_range or {"vx": [-2 * 40.0, 2 * 40.0], "vy": [-2 * 40.0, 2 * 40.0]}  # normalize (:340-352)
        p.n_features = len(self.features)
        for k, f in enumerate(self.features):
            p.features[k] = N.FEAT_ON_ROAD if f == "on_road" else N.FEATURE_CODES.get(f, N.FEAT_UNKNOWN)
            if f in fr and f != "on_road":
                p.ranged[k], p.range_lo[k], p.range_hi[k] = 1, float(fr[f][0]), float(fr[f][1])
        if "x" in fr:
            p.x_ranged, p.x_lo, p.x_hi = 1, float(fr["x"][0]), float(fr["x"][1])
        if "y" in fr:
            p.y_ranged, p.y_lo, p.y_hi = 1, float(fr["y"][0]), float(fr["y"][1])
        p.grid_lo[0], p.grid_lo[1] = float(self.grid_size[0, 0]), float(self.grid_size[1, 0])
        p.grid_step[0], p.grid_step[1] = float(self.grid_step[0]), float(self.grid_step[1])
        p.shape[0], p.shape[1] = self.grid_shape
        p.align_to_vehicle_axes, p.clip, p.as_image = int(self.align_to_vehicle_axes), int(self.clip), int(self.as_image)
        p.observe_intentions = 1
        return p

    def observe(self, env, out, mask_a=None, mask_b=None):
        view, graph = env._obs_view()
        with torch.cuda.device(env.device):
            N.check(env._lib.hwy_observe_grid(graph, C.byref(view), C.byref(self.params()), self._ptr(mask_a),
                                              self._ptr(mask_b), out.data_ptr(), env._stream()))


class TimeToCollisionObservation(_Standalone):
    """TimeToCollisionObservation (reference observation.py:115-152): [3 speeds, 3 lanes, horizon * policy_frequency]
    around the observer's speed index and lane; needs an MDPVehicle observer (DiscreteMetaAction)."""

    def __init__(self, horizon: int = 10, **kwargs):
        self.horizon = int(horizon)
        self.policy_frequency = 1
        self.target_speeds = np.linspace(20, 30, 3)

    def bind(self, policy_frequency: int, target_speeds) -> None:
        self.policy_frequency = int(policy_frequency)
        self.target_speeds = np.asarray(target_speeds, dtype=np.float64)

    def space(self, policy_frequency: int = None):
        pf = self.policy_frequency if policy_frequency is None else int(policy_frequency)
        return Box(low=0, high=1, shape=(3, 3, int(self.horizon * pf)), dtype=np.float32)

    def observe(self, env, out, mask_a=None, mask_b=None):
        p = N.HwyTtcParams()
        p.horizon, p.policy_frequency, p.n_target_speeds = self.horizon, self.policy_frequency, int(self.target_speeds.size)
        for k, t in enumerate(self.target_speeds):
            p.target_speeds[k] = float(t)
        view, graph = env._obs_view()
        with torch.cuda.device(env.device):
            N.check(env._lib.hwy_observe_ttc(graph, C.byref(view), C.byref(p), self._ptr(mask_a), self._ptr(mask_b),
                                             out.data_ptr(), env._stream()))


class LidarObservation(_Standalone):
    """LidarObservation (reference observation.py:678-769): per angular cell the distance to the closest vehicle /
    road object within `maximum_range` and its radial relative speed, [cells, 2]."""

    def __init__(self, cells: int = 16, maximum_range: float = 60, normalize: bool = True, **kwargs):
        self.cells, self.maximum_range, self.normalize = int(cells), float(maximum_range), bool(normalize)

    def space(self):
        high = 1 if self.normalize else self.maximum_range
        return Box(low=-high, high=high, shape=(self.cells, 2), dtype=np.float32)

    def observe(self, env, out, mask_a=None, mask_b=None):
        p = N.HwyLidarParams()
        p.cells, p.normalize, p.maximum_range = self.cells, int(self.normalize), self.maximum_range
        view, _ = env._obs_view()
        with torch.cuda.device(env.device):
            N.check(env._lib.hwy_observe_lidar(C.byref(view), C.byref(p), self._ptr(mask_a), self._ptr(mask_b),
                                               out.data_ptr(), env._stream()))


OBSERVATION_TYPES = {
    "Kinematics": KinematicObservation,
    "OccupancyGrid": OccupancyGridObservation,
    "TimeToCollision": TimeToCollisionObservation,
    "LidarObservation": LidarObservation,
}
_KNOWN_UNSUPPORTED = ("KinematicsGoal", "GrayscaleObservation", "AttributesObservation", "TupleObservation")


def observation_factory(env, config: dict) -> ObservationType:
    """Same selection rule and error as the reference factory (observation.py:772-794).  MultiAgentObservation is
    resolved by the env (it wraps one of these per controlled vehicle, observation.py:588-604); ExitObservation is
    registered by envs/exit_env.py."""
    kind = config["type"]
    if kind in OBSERVATION_TYPES:
        return OBSERVATION_TYPES[kind](**config)
    if kind in _KNOWN_UNSUPPORTED:
        raise NotImplementedError(f"observation type {kind!r} is not on the accelerated path "
                                  "(needs the renderer, goal envs or tuple spaces)")
    raise ValueError("Unknown observation type")


FUSED_TTC_MAX_T, FUSED_TTC_MAX_SPEEDS = 16, 3  # EnvStage's shared TimeToCollision grid (hwy_network.cu)


def select_network_observation(env, p: N.HwyNetParams, config: dict, target_speeds, ego_side_lanes: int,
                               fuse_ttc: bool = True, fuse_grid: bool = True, feature_columns: bool = False):
    """Select the plugin with the reference's factory rule for a network-kernel env and decide whether the step
    kernel writes it itself (fused: Kinematics with 5 / 7 columns, or any columns with `feature_columns`; the default
    OccupancyGrid with `fuse_grid`; TimeToCollision up to 16 time cells with `fuse_ttc`) or a standalone kernel runs
    after the step.  Fills the observation fields of `p`; returns (plugin, fused)."""
    plugin = observation_factory(env, config)
    fused = False
    if isinstance(plugin, TimeToCollisionObservation):
        plugin.bind(p.policy_frequency, target_speeds)
        n_t = plugin.horizon * p.policy_frequency
        if fuse_ttc and n_t <= FUSED_TTC_MAX_T and p.n_target_speeds <= FUSED_TTC_MAX_SPEEDS:
            p.obs_type, p.ttc_horizon, p.obs_vehicles_count, fused = N.OBS_TTC, plugin.horizon, 5, True
    elif isinstance(plugin, OccupancyGridObservation):
        if fuse_grid and plugin.is_default:
            p.obs_type, p.obs_vehicles_count, fused = N.OBS_OCCUPANCY, 5, True
    elif isinstance(plugin, KinematicObservation):
        feats = plugin.features
        if config.get("observe_intentions"):
            raise NotImplementedError("Kinematics observe_intentions on the network kernels")
        # normalize_obs (observation.py:214-226), computed at the first observation of an episode: the y-range spans
        # all_side_lanes of the controlled vehicle's spawn road
        w = 4.0 * ego_side_lanes
        fr = plugin.features_range
        if fr is None:
            fr = {"x": [-5.0 * 40.0, 5.0 * 40.0], "y": [-w, w], "vx": [-2 * 40.0, 2 * 40.0], "vy": [-2 * 40.0, 2 * 40.0]}
        if feats[:5] != ["presence", "x", "y", "vx", "vy"] or feats[5:] not in ([], ["cos_h", "sin_h"]):
            if not feature_columns:
                raise NotImplementedError(f"Kinematics features {feats} on the network kernels "
                                          "(presence, x, y, vx, vy [, cos_h, sin_h])")
            # any Vehicle.to_dict column list (vehicle/kinematics.py:237-261) with per-column ranges
            p.obs_n_feat = len(feats)
            for k, f in enumerate(feats):
                p.obs_feat[k] = N.FEATURE_CODES[f]
                if f in fr:
                    p.obs_feat_ranged[k], p.obs_feat_lo[k], p.obs_feat_hi[k] = 1, float(fr[f][0]), float(fr[f][1])
        p.obs_type, p.obs_features = N.OBS_KINEMATICS, len(feats)
        p.obs_vehicles_count = plugin.vehicles_count
        p.obs_see_behind, p.obs_absolute = int(plugin.see_behind), int(plugin.absolute)
        p.obs_normalize, p.obs_clip = int(plugin.normalize), int(plugin.clip)
        (p.obs_x_lo, p.obs_x_hi), (p.obs_y_lo, p.obs_y_hi) = (map(float, fr["x"]), map(float, fr["y"]))
        (p.obs_vx_lo, p.obs_vx_hi), (p.obs_vy_lo, p.obs_vy_hi) = (map(float, fr["vx"]), map(float, fr["vy"]))
        fused = True
    if not fused:  # the kernels write one Kinematics row into a scratch buffer; the plugin observes after them
        p.obs_type, p.obs_features, p.obs_vehicles_count = N.OBS_KINEMATICS, 5, 1
        p.obs_x_lo = p.obs_y_lo = p.obs_vx_lo = p.obs_vy_lo = -1.0
        p.obs_x_hi = p.obs_y_hi = p.obs_vx_hi = p.obs_vy_hi = 1.0
    return plugin, fused
