"""Action plugins of the batched backend (host-side descriptors).

Mirror of the reference's string-keyed ``action_factory``
(highway_env/envs/common/action.py:336-346): the same ``config["action"]["type"]`` names and
keyword arguments select an ``ActionType`` whose job here is only to describe the action
space and to fill the kernel parameters — the arithmetic of ``ActionType.act`` runs on the
device in the first substep of ``hwy_highway_step``.
"""
from __future__ import annotations

import itertools

import numpy as np

from ... import _native as N
from ...spaces import Box, Discrete


class ActionType:
    """What the ego-vehicle of every env executes (one action per env per step)."""

    kernel_action_type: int  # HwyHighwayParams.action_type
    ego_kind: int            # vehicle class of the controlled vehicle (action.py vehicle_class)

    def space(self):
        raise NotImplementedError

    def fill_params(self, p: N.HwyHighwayParams) -> None:
        raise NotImplementedError


class DiscreteMetaAction(ActionType):
    """Lane-change / cruise-control meta-actions (reference action.py:199-298).

    Labels (action.py:204): 0 LANE_LEFT, 1 IDLE, 2 LANE_RIGHT, 3 FASTER, 4 SLOWER; the ego is
    an ``MDPVehicle`` tracking one of ``target_speeds`` (controller.py:256-344).
    """

    ACTIONS_ALL = {0: "LANE_LEFT", 1: "IDLE", 2: "LANE_RIGHT", 3: "FASTER", 4: "SLOWER"}
    kernel_action_type = 0
    ego_kind = N.KIND_MDP

    def __init__(self, longitudinal: bool = True, lateral: bool = True, target_speeds=None, **kwargs):
        if not (longitudinal and lateral):
            # ACTIONS_LONGI / ACTIONS_LAT variants (action.py:206-210) are used by intersection-v0
            raise NotImplementedError(
                "DiscreteMetaAction with longitudinal/lateral disabled is not on the highway path"
            )
        self.target_speeds = (
            np.linspace(20, 30, 3) if target_speeds is None else np.array(target_speeds, dtype=np.float64)
        )
        if not 1 <= self.target_speeds.size <= N.HWY_MAX_TARGET_SPEEDS:
            raise ValueError(f"target_speeds must have 1..{N.HWY_MAX_TARGET_SPEEDS} entries")
        self.actions = self.ACTIONS_ALL
        self.actions_indexes = {v: k for k, v in self.actions.items()}

    def space(self):
        return Discrete(len(self.actions))

    def fill_params(self, p):
        p.action_type = 0
        p.n_target_speeds = int(self.target_speeds.size)
        for k, t in enumerate(self.target_speeds):
            p.target_speeds[k] = float(t)
        p.act_clip = 1
        p.acc_lo, p.acc_hi = -5.0, 5.0
        p.steer_lo, p.steer_hi = -np.pi / 4, np.pi / 4


class ContinuousAction(ActionType):
    """[throttle, steering] in [-1, 1]^2 mapped to acceleration / steering ranges
    (reference action.py:73-162); the ego is a plain kinematic ``Vehicle``."""

    ACCELERATION_RANGE = (-5, 5.0)
    STEERING_RANGE = (-np.pi / 4, np.pi / 4)
    kernel_action_type = 1
    ego_kind = N.KIND_VEHICLE

    def __init__(self, acceleration_range=None, steering_range=None, speed_range=None,
                 longitudinal: bool = True, lateral: bool = True, dynamical: bool = False,
                 clip: bool = True, **kwargs):
        if not (longitudinal and lateral):
            raise NotImplementedError("ContinuousAction needs both longitudinal and lateral control here")
        # dynamical=True selects BicycleVehicle (vehicle/dynamics.py:33-160): on the network kernels only
        self.dynamical = bool(dynamical)
        if speed_range is not None:
            raise NotImplementedError("speed_range (per-vehicle MIN/MAX_SPEED override) is not supported")
        self.acceleration_range = tuple(acceleration_range) if acceleration_range else self.ACCELERATION_RANGE
        self.steering_range = tuple(steering_range) if steering_range else self.STEERING_RANGE
        self.clip = bool(clip)

    def space(self):
        return Box(-1.0, 1.0, shape=(2,), dtype=np.float32)

    def fill_params(self, p):
        if self.dynamical:
            raise NotImplementedError("dynamical=True (BicycleVehicle) is implemented on the intersection family only")
        p.action_type = 1
        p.n_target_speeds = 3
        for k, t in enumerate(np.linspace(20, 30, 3)):
            p.target_speeds[k] = float(t)
        p.act_clip = int(self.clip)
        p.acc_lo, p.acc_hi = float(self.acceleration_range[0]), float(self.acceleration_range[1])
        p.steer_lo, p.steer_hi = float(self.steering_range[0]), float(self.steering_range[1])


class DiscreteAction(ContinuousAction):
    """A uniform quantisation of ContinuousAction (reference action.py:165-196): action k selects
    `itertools.product(*np.linspace(low, high, actions_per_axis).T)[k]`, which then goes through
    ContinuousAction.act.  The float32 table is built with the reference's expressions; the
    lookup is a device gather in front of the continuous-action kernel path."""

    def __init__(self, actions_per_axis: int = 3, **kwargs):
        super().__init__(**kwargs)
        self.actions_per_axis = int(actions_per_axis)
        if self.actions_per_axis < 1:
            raise ValueError("actions_per_axis must be >= 1")
        cont = super().space()
        axes = np.linspace(cont.low, cont.high, self.actions_per_axis).T
        self.table = np.array(list(itertools.product(*axes)), dtype=np.float32)

    def space(self):
        return Discrete(self.actions_per_axis ** 2)


def speed_to_index(target_speeds, speed) -> int:
    """MDPVehicle.speed_to_index (vehicle/controller.py): the index of the target speed closest to `speed`."""
    ts = np.asarray(target_speeds, dtype=np.float64)
    return int(np.clip(np.round((speed - ts[0]) / (ts[-1] - ts[0]) * (ts.size - 1)), 0, ts.size - 1))


ACTION_TYPES = {
    "DiscreteMetaAction": DiscreteMetaAction,
    "ContinuousAction": ContinuousAction,
    "DiscreteAction": DiscreteAction,
}


def action_factory(env, config: dict) -> ActionType:
    """Same selection rule and error as the reference factory (action.py:336-346)."""
    kind = config["type"]
    if kind in ACTION_TYPES:
        return ACTION_TYPES[kind](**config)
    if kind in ("MultiAgentAction",):
        raise NotImplementedError(f"action type {kind!r} is not on the accelerated path yet")
    raise ValueError("Unknown action type")
