"""ctypes binding of the linear-traffic CPU oracle (oracle/hwy_linear_oracle.c).  TEST INFRASTRUCTURE ONLY.

LinearVehicle / AggressiveVehicle / DefensiveVehicle traffic (vehicle/behavior.py:350-583) on highway-v0 /
highway-fast-v0.  Only tests/ may import this module; the product (``highwayenv_b200``) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import warnings

import numpy as np

import hwy_oracle as ho

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libhwy_linear_oracle.so")

B = "highway_env.vehicle.behavior."
# LinearVehicle and its subclasses -> LANE_CHANGE_MIN_ACC_GAIN (behavior.py:43, 537, 552)
LINEAR_TYPES = {B + "LinearVehicle": 0.2, B + "AggressiveVehicle": 1.0, B + "DefensiveVehicle": 1.0}


class OrcLinearTraffic(C.Structure):
    _fields_ = [("acc_lo", C.c_double * 3), ("acc_span", C.c_double * 3), ("steer_lo", C.c_double * 2),
                ("steer_span", C.c_double * 2)]


def linear_ranges():
    """LinearVehicle.ACCELERATION_RANGE / STEERING_RANGE (behavior.py:353-371) as (lo, hi - lo) pairs, numpy arithmetic;
    Aggressive / Defensive inherit both ranges."""
    kp_heading, kp_lateral = 1 / 0.2, 1 / 0.6  # controller.py:24-33
    acc = np.array([0.3, 0.3, 2.0])
    steer = np.array([kp_heading, kp_heading * kp_lateral])
    acc_range = np.array([0.5 * acc, 1.5 * acc])
    steer_range = np.array([steer - np.array([0.07, 1.5]), steer + np.array([0.07, 1.5])])
    return acc_range[0], acc_range[1] - acc_range[0], steer_range[0], steer_range[1] - steer_range[0]


def traffic() -> OrcLinearTraffic:
    t = OrcLinearTraffic()
    acc_lo, acc_span, steer_lo, steer_span = linear_ranges()
    t.acc_lo[:], t.acc_span[:] = list(acc_lo), list(acc_span)
    t.steer_lo[:], t.steer_span[:] = list(steer_lo), list(steer_span)
    return t


def cfg_from_dict(config: dict) -> ho.OrcHighwayCfg:
    """hwy_oracle.cfg_from_dict with the traffic class's TIME_WANTED (2.5, behavior.py:373) and
    LANE_CHANGE_MIN_ACC_GAIN."""
    ovt = config["other_vehicles_type"]
    if ovt not in LINEAR_TYPES:
        raise ValueError(f"not a linear traffic class: {ovt}")
    c = ho.cfg_from_dict(config)
    c.time_wanted = 2.5
    c.lane_change_min_acc_gain = LINEAR_TYPES[ovt]
    return c


def _stale() -> bool:
    src = [os.path.join(_HERE, f) for f in ("hwy_linear_oracle.c", "hwy_linear_oracle.h", "hwy_oracle.c",
                                            "hwy_oracle.h")]
    return not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < max(map(os.path.getmtime, src))


def build(force: bool = False) -> str:
    """Compile the oracle with gcc (seconds): hwy_oracle.c is #included by hwy_linear_oracle.c."""
    if force or _stale():
        subprocess.check_call(["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-std=gnu11", "-o", _LIB_PATH,
                               os.path.join(_HERE, "hwy_linear_oracle.c"), "-lm", "-lpthread"])
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
        P, T, Bt = C.POINTER(ho.OrcHighwayCfg), C.POINTER(OrcLinearTraffic), C.POINTER(ho.OrcBatch)
        _lib.orc_linear_acceleration.restype = C.c_double
        _lib.orc_linear_acceleration.argtypes = [C.POINTER(C.c_double), C.c_double, C.c_double, C.c_int, C.c_double,
                                                 C.c_double, C.c_double, C.c_double]
        _lib.orc_linear_steering.restype = C.c_double
        _lib.orc_linear_steering.argtypes = [C.POINTER(C.c_double)] + [C.c_double] * 4
        _lib.orc_linear_highway_reset_batch.restype = None
        _lib.orc_linear_highway_reset_batch.argtypes = [P, T, Bt, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        _lib.orc_linear_highway_step_batch.restype = None
        _lib.orc_linear_highway_step_batch.argtypes = [P, T, Bt, C.c_void_p] + [C.c_void_p] * 6 + [C.c_int, C.c_int]
        _lib.orc_linear_highway_substeps_batch.restype = None
        _lib.orc_linear_highway_substeps_batch.argtypes = [P, Bt, C.c_void_p, C.c_int, C.c_int]
    return _lib


class LinearOracleBatch(ho.OracleBatch):
    """hwy_oracle.OracleBatch with linear traffic: ``linear_params`` [n_envs, V, 5] holds every vehicle's
    ACCELERATION_PARAMETERS (3) and STEERING_PARAMETERS (2)."""

    def __init__(self, config: dict, n_envs: int, seeds=None, threads: int = 1):
        super().__init__(cfg_from_dict(config), n_envs, seeds=seeds, threads=threads)
        self.traffic = traffic()
        self.linear_params = np.zeros((self.n, self.V, 5), dtype=np.float64)

    def reset(self, mask=None):
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        lib().orc_linear_highway_reset_batch(C.byref(self.cfg), C.byref(self.traffic), C.byref(self._b),
                                             self.linear_params.ctypes.data, None if m is None else m.ctypes.data,
                                             self.obs.ctypes.data, self.threads)
        return self.obs

    def step(self, actions, autoreset: bool = False):
        ai = af = None
        if self.cfg.action_type == 0:
            ai = np.ascontiguousarray(actions, dtype=np.int32)
        else:
            af = np.ascontiguousarray(actions, dtype=np.float32).reshape(self.n, 2)
        lib().orc_linear_highway_step_batch(
            C.byref(self.cfg), C.byref(self.traffic), C.byref(self._b), self.linear_params.ctypes.data,
            None if ai is None else ai.ctypes.data, None if af is None else af.ctypes.data, self.obs.ctypes.data,
            self.reward.ctypes.data, self.terminated.ctypes.data, self.truncated.ctypes.data, int(autoreset),
            self.threads)
        return self.obs, self.reward, self.terminated, self.truncated

    def substeps(self, n_substeps: int):
        """Road.act() + Road.step(dt), n_substeps times, on every env (the controlled vehicle acts with None)."""
        lib().orc_linear_highway_substeps_batch(C.byref(self.cfg), C.byref(self._b), self.linear_params.ctypes.data,
                                                int(n_substeps), self.threads)
