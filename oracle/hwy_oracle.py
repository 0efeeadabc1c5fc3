"""ctypes binding of the CPU oracle (oracle/hwy_oracle.c).  TEST INFRASTRUCTURE ONLY.

Only tests/, ``__graft_entry__.smoke()`` and bench.py's cpu_baseline / ``--impl reference``
legs may import this module; the product (``highwayenv_b200``) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import warnings

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libhwy_oracle.so")

ORC_MAX_TARGET_SPEEDS = 8
KIND_IDM, KIND_MDP, KIND_VEHICLE = 0, 1, 2


class OrcHighwayCfg(C.Structure):
    _fields_ = [
        ("lanes_count", C.c_int32),
        ("n_vehicles", C.c_int32),
        ("simulation_frequency", C.c_int32),
        ("policy_frequency", C.c_int32),
        ("action_type", C.c_int32),
        ("others_check_collisions", C.c_int32),
        ("normalize_reward", C.c_int32),
        ("offroad_terminal", C.c_int32),
        ("obs_vehicles_count", C.c_int32),
        ("obs_see_behind", C.c_int32),
        ("obs_absolute", C.c_int32),
        ("obs_normalize", C.c_int32),
        ("obs_clip", C.c_int32),
        ("n_target_speeds", C.c_int32),
        ("initial_lane_id", C.c_int32),
        ("act_clip", C.c_int32),
        ("duration", C.c_double),
        ("lane_length", C.c_double),
        ("lane_width", C.c_double),
        ("speed_limit", C.c_double),
        ("target_speeds", C.c_double * ORC_MAX_TARGET_SPEEDS),
        ("collision_reward", C.c_double),
        ("right_lane_reward", C.c_double),
        ("high_speed_reward", C.c_double),
        ("reward_speed_lo", C.c_double),
        ("reward_speed_hi", C.c_double),
        ("acc_lo", C.c_double),
        ("acc_hi", C.c_double),
        ("steer_lo", C.c_double),
        ("steer_hi", C.c_double),
        ("ego_spacing", C.c_double),
        ("vehicles_density", C.c_double),
        ("ego_speed", C.c_double),
        ("spawn_exp", C.c_double),
        ("acc_max", C.c_double),
        ("comfort_acc_max", C.c_double),
        ("comfort_acc_min", C.c_double),
        ("distance_wanted", C.c_double),
        ("time_wanted", C.c_double),
        ("politeness", C.c_double),
        ("lane_change_min_acc_gain", C.c_double),
        ("lane_change_max_braking_imposed", C.c_double),
        ("lane_change_delay", C.c_double),
        ("delta_lo", C.c_double),
        ("delta_hi", C.c_double),
        ("perception_distance", C.c_double),
        ("obs_n_features", C.c_int32), ("_pad_obs", C.c_int32),
        ("obs_feature", C.c_int32 * 16), ("obs_feature_ranged", C.c_int32 * 16),
        ("obs_feature_lo", C.c_double * 16), ("obs_feature_hi", C.c_double * 16),
    ]


class OrcPcg64(C.Structure):
    _fields_ = [
        ("state_hi", C.c_uint64),
        ("state_lo", C.c_uint64),
        ("inc_hi", C.c_uint64),
        ("inc_lo", C.c_uint64),
        ("has_uint32", C.c_uint32),
        ("uinteger", C.c_uint32),
    ]


PCG_DTYPE = np.dtype(
    [
        ("state_hi", "<u8"),
        ("state_lo", "<u8"),
        ("inc_hi", "<u8"),
        ("inc_lo", "<u8"),
        ("has_uint32", "<u4"),
        ("uinteger", "<u4"),
    ]
)

_F64 = ("x", "y", "heading", "speed", "target_speed", "timer", "delta", "impact_x", "impact_y")
_I32 = ("lane", "target_lane", "kind", "crashed", "has_impact", "check_collisions")


class OrcHighwayState(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in _F64] + [(k, C.c_void_p) for k in _I32] + [
        ("speed_index", C.c_void_p), ("time", C.c_void_p)]


class OrcBatch(C.Structure):
    _fields_ = (
        [("n_envs", C.c_int32)]
        + [(k, C.c_void_p) for k in _F64]
        + [(k, C.c_void_p) for k in _I32]
        + [("speed_index", C.c_void_p), ("time", C.c_void_p), ("rng", C.c_void_p)]
    )


def _stale() -> bool:
    src = [os.path.join(_HERE, f) for f in ("hwy_oracle.c", "hwy_oracle.h")]
    return not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < max(map(os.path.getmtime, src))


def build(force: bool = False) -> str:
    """Compile the oracle with gcc (seconds).  Building the checker is not using it."""
    src = os.path.join(_HERE, "hwy_oracle.c")
    if force or _stale():
        subprocess.check_call(
            [
                "gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=gnu11",
                "-o", _LIB_PATH, src, "-lm", "-lpthread",
            ]
        )
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):  # build() made it; a read-only tree must not be written to
            build()
        elif _stale():
            warnings.warn(f"{_LIB_PATH} is older than its sources: run build() to use the edited oracle")
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_wrap_to_pi.restype = C.c_double
        _lib.orc_wrap_to_pi.argtypes = [C.c_double]
        _lib.orc_not_zero.restype = C.c_double
        _lib.orc_not_zero.argtypes = [C.c_double]
        _lib.orc_rotated_rectangles_intersect.restype = C.c_int
        _lib.orc_rotated_rectangles_intersect.argtypes = [C.c_double] * 10
        _lib.orc_rng_uniform.restype = C.c_double
        _lib.orc_rng_uniform.argtypes = [C.POINTER(OrcPcg64), C.c_double, C.c_double]
        _lib.orc_rng_choice.restype = C.c_int64
        _lib.orc_rng_choice.argtypes = [C.POINTER(OrcPcg64), C.c_int64]
        _lib.orc_polygons_intersecting.restype = None
        _lib.orc_highway_reset_batch.restype = None
        _lib.orc_highway_reset_batch.argtypes = [
            C.POINTER(OrcHighwayCfg), C.POINTER(OrcBatch), C.c_void_p, C.c_void_p, C.c_int,
        ]
        _lib.orc_highway_substeps.restype = None
        _lib.orc_highway_substeps.argtypes = [C.POINTER(OrcHighwayCfg), C.POINTER(OrcHighwayState), C.c_int]
        _lib.orc_highway_observe.restype = None
        _lib.orc_highway_observe.argtypes = [C.POINTER(OrcHighwayCfg), C.POINTER(OrcHighwayState), C.c_void_p]
        _lib.orc_highway_step_batch.restype = None
        _lib.orc_highway_step_batch.argtypes = [
            C.POINTER(OrcHighwayCfg), C.POINTER(OrcBatch), C.c_void_p, C.c_void_p, C.c_void_p,
            C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
        ]
    return _lib


def pcg_state_from_seed(seed: int) -> tuple:
    """gymnasium seeding: Generator(PCG64(SeedSequence(seed))) — state as 6 ints."""
    st = np.random.PCG64(np.random.SeedSequence(int(seed))).state
    s, inc = st["state"]["state"], st["state"]["inc"]
    m = (1 << 64) - 1
    return (s >> 64, s & m, inc >> 64, inc & m, int(st["has_uint32"]), int(st["uinteger"]))


def pcg_states(seeds) -> np.ndarray:
    out = np.zeros(len(seeds), dtype=PCG_DTYPE)
    for i, sd in enumerate(seeds):
        out[i] = pcg_state_from_seed(sd)
    return out


def cfg_from_dict(config: dict) -> OrcHighwayCfg:
    """Build the oracle config from a FULL reference-style config dict (defaults merged:
    highway_env/envs/highway_env.py:25-53,162-175 over abstract.py:102-125)."""
    c = OrcHighwayCfg()
    obs = config["observation"]
    act = config["action"]
    assert obs["type"] == "Kinematics", obs
    c.lanes_count = int(config["lanes_count"])
    c.n_vehicles = int(config["vehicles_count"]) + 1
    c.simulation_frequency = int(config["simulation_frequency"])
    c.policy_frequency = int(config["policy_frequency"])
    c.action_type = {"DiscreteMetaAction": 0, "ContinuousAction": 1, "DiscreteAction": 1}[act["type"]]
    c.others_check_collisions = int(config.get("_others_check_collisions", 1))
    c.normalize_reward = int(bool(config["normalize_reward"]))
    c.offroad_terminal = int(bool(config["offroad_terminal"]))
    c.obs_vehicles_count = int(obs.get("vehicles_count", 5))
    c.obs_see_behind = int(bool(obs.get("see_behind", False)))
    c.obs_absolute = int(bool(obs.get("absolute", False)))
    c.obs_normalize = int(bool(obs.get("normalize", True)))
    c.obs_clip = int(bool(obs.get("clip", True)))
    feats, fr = obs.get("features"), obs.get("features_range")
    if (feats and list(feats) != ["presence", "x", "y", "vx", "vy"]) or fr is not None:
        feats = list(feats) if feats else ["presence", "x", "y", "vx", "vy"]
        codes = ["presence", "x", "y", "vx", "vy", "heading", "cos_h", "sin_h", "cos_d", "sin_d", "long_off",
                 "lat_off", "ang_off"]
        if fr is None:  # observation.py:214-226
            lanes = int(config["lanes_count"])
            fr = {"x": [-200.0, 200.0], "y": [-4.0 * lanes, 4.0 * lanes], "vx": [-80.0, 80.0], "vy": [-80.0, 80.0]}
        c.obs_n_features = len(feats)
        for k, f in enumerate(feats):
            c.obs_feature[k] = codes.index(f)
            c.obs_feature_ranged[k] = int(f in fr)
            if f in fr:
                c.obs_feature_lo[k], c.obs_feature_hi[k] = float(fr[f][0]), float(fr[f][1])
    ts = act.get("target_speeds")
    ts = list(np.linspace(20, 30, 3)) if ts is None else [float(t) for t in ts]
    c.n_target_speeds = len(ts)
    for i, t in enumerate(ts):
        c.target_speeds[i] = t
    ili = config.get("initial_lane_id")
    c.initial_lane_id = -1 if ili is None else int(ili)
    c.act_clip = int(bool(act.get("clip", True)))
    c.duration = float(config["duration"])
    c.lane_length = 10000.0
    c.lane_width = 4.0
    c.speed_limit = 30.0
    c.collision_reward = float(config["collision_reward"])
    c.right_lane_reward = float(config["right_lane_reward"])
    c.high_speed_reward = float(config["high_speed_reward"])
    c.reward_speed_lo = float(config["reward_speed_range"][0])
    c.reward_speed_hi = float(config["reward_speed_range"][1])
    ar = act.get("acceleration_range") or (-5, 5.0)
    sr = act.get("steering_range") or (-np.pi / 4, np.pi / 4)
    c.acc_lo, c.acc_hi = float(ar[0]), float(ar[1])
    c.steer_lo, c.steer_hi = float(sr[0]), float(sr[1])
    c.ego_spacing = float(config["ego_spacing"])
    c.vehicles_density = float(config["vehicles_density"])
    c.ego_speed = 25.0
    c.spawn_exp = float(np.exp(-5 / 40 * c.lanes_count))
    c.acc_max, c.comfort_acc_max, c.comfort_acc_min = 6.0, 3.0, -5.0
    c.distance_wanted, c.time_wanted = 5.0 + 5.0, 1.5
    c.politeness, c.lane_change_min_acc_gain = 0.0, 0.2
    c.lane_change_max_braking_imposed, c.lane_change_delay = 2.0, 1.0
    c.delta_lo, c.delta_hi = 3.5, 4.5
    c.perception_distance = 5.0 * 40.0
    return c


def discrete_action_table(actions_per_axis: int = 3) -> np.ndarray:
    """DiscreteAction.act (action.py:188-196): all_actions = product of linspace(low, high, k) per axis"""
    import itertools

    low, high = np.full(2, -1.0, dtype=np.float32), np.full(2, 1.0, dtype=np.float32)
    axes = np.linspace(low, high, actions_per_axis).T
    return np.array(list(itertools.product(*axes)), dtype=np.float32)


class OracleBatch:
    """n_envs highway envs stepped by the C oracle (SoA numpy buffers [n_envs, V])."""

    def __init__(self, cfg: OrcHighwayCfg, n_envs: int, seeds=None, threads: int = 1):
        self.cfg = cfg
        self.n = int(n_envs)
        self.V = int(cfg.n_vehicles)
        self.K = int(cfg.obs_vehicles_count)
        self.threads = threads
        self.a = {k: np.zeros((self.n, self.V), dtype=np.float64) for k in _F64}
        self.a.update({k: np.zeros((self.n, self.V), dtype=np.int32) for k in _I32})
        self.a["speed_index"] = np.zeros(self.n, dtype=np.int32)
        self.a["time"] = np.zeros(self.n, dtype=np.float64)
        self.rng = pcg_states(seeds if seeds is not None else range(self.n))
        self._b = OrcBatch()
        self._b.n_envs = self.n
        for k in list(_F64) + list(_I32) + ["speed_index", "time"]:
            setattr(self._b, k, self.a[k].ctypes.data)
        self._b.rng = self.rng.ctypes.data
        self.obs = np.zeros((self.n, self.K, int(cfg.obs_n_features) or 5), dtype=np.float32)
        self.reward = np.zeros(self.n, dtype=np.float64)
        self.terminated = np.zeros(self.n, dtype=np.uint8)
        self.truncated = np.zeros(self.n, dtype=np.uint8)

    def reset(self, mask=None):
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        lib().orc_highway_reset_batch(
            C.byref(self.cfg), C.byref(self._b), None if m is None else m.ctypes.data,
            self.obs.ctypes.data, self.threads,
        )
        return self.obs

    def step(self, actions, autoreset: bool = False):
        ai = af = None
        if self.cfg.action_type == 0:
            ai = np.ascontiguousarray(actions, dtype=np.int32)
        else:
            af = np.ascontiguousarray(actions, dtype=np.float32).reshape(self.n, 2)
        lib().orc_highway_step_batch(
            C.byref(self.cfg), C.byref(self._b),
            None if ai is None else ai.ctypes.data, None if af is None else af.ctypes.data,
            self.obs.ctypes.data, self.reward.ctypes.data, self.terminated.ctypes.data,
            self.truncated.ctypes.data, int(autoreset), self.threads,
        )
        return self.obs, self.reward, self.terminated, self.truncated

    def env_state(self, e: int) -> OrcHighwayState:
        """env slot e as the single-env OrcHighwayState of orc_highway_substeps / orc_highway_observe (views of the
        batch arrays)"""
        st = OrcHighwayState()
        for k in list(_F64) + list(_I32):
            setattr(st, k, self.a[k][e].ctypes.data)
        st.speed_index = self.a["speed_index"][e:].ctypes.data
        st.time = self.a["time"][e:].ctypes.data
        return st

    def substeps(self, e: int, n: int) -> None:
        """n x (Road.act(); Road.step(dt)) on env slot e"""
        lib().orc_highway_substeps(C.byref(self.cfg), C.byref(self.env_state(e)), int(n))

    def observe(self, e: int) -> np.ndarray:
        out = np.zeros(self.obs.shape[1:], dtype=np.float32)
        lib().orc_highway_observe(C.byref(self.cfg), C.byref(self.env_state(e)), out.ctypes.data)
        return out

    def load_state(self, e: int, st: dict):
        """Inject a state dumped by ref_harness.dump_state into env slot e."""
        for k in ("x", "y", "heading", "speed"):
            self.a[k][e] = st[k]
        self.a["target_speed"][e] = np.nan_to_num(st["target_speed"], nan=0.0)
        self.a["timer"][e] = np.nan_to_num(st["timer"], nan=0.0)
        self.a["delta"][e] = np.nan_to_num(st["delta"], nan=4.0)
        self.a["lane"][e] = st["lane"]
        self.a["target_lane"][e] = np.where(st["target_lane"] < 0, st["lane"], st["target_lane"])
        self.a["crashed"][e] = st["crashed"]
        has = ~np.isnan(st["impact"][:, 0])
        self.a["has_impact"][e] = has
        self.a["impact_x"][e] = np.where(has, st["impact"][:, 0], 0.0)
        self.a["impact_y"][e] = np.where(has, st["impact"][:, 1], 0.0)
        self.a["check_collisions"][e] = st["check_collisions"]
        kind = np.full(self.V, KIND_IDM, dtype=np.int32)
        kind[0] = KIND_MDP if self.cfg.action_type == 0 else KIND_VEHICLE
        self.a["kind"][e] = kind
        self.a["speed_index"][e] = st["speed_index"][0]
        self.a["time"][e] = float(st["time"])
