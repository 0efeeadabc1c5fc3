"""CPU checks of LinearVehicle / AggressiveVehicle / DefensiveVehicle traffic on the highway family: the restated
controllers against the reference's own methods, the C oracle (oracle/hwy_linear_oracle.c) against the linear_* golden rollouts (oracle/
gen_linear_golden.py), the new ABI structs, and the traffic types that stay unsupported."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import hwy_linear_oracle as lo
from parity_utils import compare_state, golden_state, load_golden

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ["linear_highway_fast_v20", "linear_aggressive_fast_v50", "linear_defensive_v50",
         "linear_highway_v100_continuous"]
B = "highway_env.vehicle.behavior."


def _reference():
    import ref_harness as rh

    if not rh.reference_available():
        pytest.skip("the reference is not mounted")
    return rh


def test_ranges_equal_the_reference_class_attributes():
    rh = _reference()
    env = rh.make_reference_env("highway-fast-v0", {"other_vehicles_type": B + "LinearVehicle"})
    env.reset(seed=0)
    lin = type(env.road.vehicles[1])
    acc_lo, acc_span, steer_lo, steer_span = lo.linear_ranges()
    assert np.array_equal(acc_lo, lin.ACCELERATION_RANGE[0])
    assert np.array_equal(acc_span, lin.ACCELERATION_RANGE[1] - lin.ACCELERATION_RANGE[0])
    assert np.array_equal(steer_lo, lin.STEERING_RANGE[0])
    assert np.array_equal(steer_span, lin.STEERING_RANGE[1] - lin.STEERING_RANGE[0])
    from highwayenv_b200.envs import highway_env as he

    for a, b in zip(he.linear_ranges(), lo.linear_ranges()):
        assert np.array_equal(a, b)
    assert he.LINEAR_VEHICLE_TYPES == lo.LINEAR_TYPES


def test_controllers_equal_the_reference_bit_for_bit():
    """orc_linear_acceleration / orc_linear_steering (what the kernel restates, with the same fma chains) against
    LinearVehicle.acceleration / steering_control on random states."""
    rh = _reference()
    env = rh.make_reference_env("highway-v0", {"other_vehicles_type": B + "LinearVehicle", "lanes_count": 4})
    env.reset(seed=1)
    lib = lo.lib()
    rng = np.random.default_rng(7)
    caller, ego, front = env.road.vehicles[1], env.road.vehicles[2], env.road.vehicles[3]
    lanes = env.road.network.graph["0"]["1"]
    n = 4000
    for k in range(n):
        caller.ACCELERATION_PARAMETERS = lo.linear_ranges()[0] + rng.uniform(size=3) * lo.linear_ranges()[1]
        caller.STEERING_PARAMETERS = lo.linear_ranges()[2] + rng.uniform(size=2) * lo.linear_ranges()[3]
        for v in (caller, ego, front):
            lane = int(rng.integers(0, 4))
            v.position = np.array([rng.uniform(0, 500), 4.0 * lane + rng.normal(0, 1.5)])
            v.heading = float(rng.normal(0, 0.3))
            v.speed = float(rng.choice([rng.uniform(-2, 40), rng.uniform(-0.02, 0.02), 0.0]))
            v.target_speed = float(rng.uniform(15, 35))
            v.lane_index = ("0", "1", lane)
            v.lane = lanes[lane]
        with_front = k % 3 != 0
        want = caller.acceleration(ego_vehicle=ego, front_vehicle=front if with_front else None)
        d = ego.lane_distance_to(front) if with_front else 0.0
        a = (C.c_double * 3)(*caller.ACCELERATION_PARAMETERS)
        got = lib.orc_linear_acceleration(a, ego.target_speed, ego.speed, int(with_front), front.speed, d,
                                          caller.DISTANCE_WANTED, caller.TIME_WANTED)
        assert np.float64(got).view(np.uint64) == np.float64(want).view(np.uint64), (k, got, want)
        tl = int(rng.integers(0, 4))
        want = caller.steering_control(("0", "1", tl))
        s, lat = lanes[tl].local_coordinates(caller.position)
        p = (C.c_double * 2)(*caller.STEERING_PARAMETERS)
        got = lib.orc_linear_steering(p, lanes[tl].heading, caller.heading, lat, caller.speed)
        assert np.float64(got).view(np.uint64) == np.float64(want).view(np.uint64), (k, got, want)


def _got(ob, e):
    g = {k: ob.a[k][e] for k in ob.a if k not in ("speed_index", "time")}
    g["speed_index"] = ob.a["speed_index"][e]
    return g


@pytest.mark.parametrize("name", CASES)
def test_oracle_reset_matches_reference(name):
    g = load_golden(name)
    ob = lo.LinearOracleBatch(g["config"], len(g["seeds"]), seeds=g["seeds"])
    obs = ob.reset()
    for i in range(len(g["seeds"])):
        assert compare_state(golden_state(g, i, 0), _got(ob, i), tol=0.0, ctx=f"{name}#{i}") == 0.0
        assert np.array_equal(obs[i], g["obs"][i, 0])
    assert np.array_equal(ob.linear_params, g["linear_params"])
    w = g["rng_words"][:, 0]
    assert np.array_equal(ob.rng["state_hi"], w[:, 0]) and np.array_equal(ob.rng["state_lo"], w[:, 1])
    assert np.array_equal(ob.rng["has_uint32"].astype(np.uint64), w[:, 4] >> np.uint64(32))


@pytest.mark.parametrize("name", CASES)
def test_oracle_teacher_forced_steps(name):
    g = load_golden(name)
    S, T = g["actions"].shape[:2]
    ob = lo.LinearOracleBatch(g["config"], S, seeds=g["seeds"])
    ob.linear_params[:] = g["linear_params"]
    worst = 0.0
    for t in range(T):
        for i in range(S):
            ob.load_state(i, golden_state(g, i, t))
        obs, rew, term, trunc = ob.step(g["actions"][:, t])
        for i in range(S):
            ctx = f"{name} seed#{i} t={t}"
            worst = max(worst, compare_state(golden_state(g, i, t + 1), _got(ob, i), ctx=ctx))
            assert abs(rew[i] - g["reward"][i, t]) <= 1e-9, ctx
            assert bool(term[i]) == bool(g["terminated"][i, t]), ctx
            assert np.max(np.abs(obs[i] - g["obs"][i, t + 1])) <= 1e-6, ctx
    assert worst < 1e-9, worst


def test_fixtures_exercise_lane_changes_and_each_class():
    for name in CASES:
        g = load_golden(name)
        assert len(g["seeds"]) == 32
        assert (g["target_lane"][:, 1:, 1:] != g["lane"][:, 1:, 1:]).any(), name  # MOBIL fired somewhere
        assert not g["linear_params"][:, 0].any() and g["linear_params"][:, 1:].all(), name
    kinds = {load_golden(n)["config"]["other_vehicles_type"].rsplit(".", 1)[1] for n in CASES}
    assert kinds == {"LinearVehicle", "AggressiveVehicle", "DefensiveVehicle"}


def test_linear_entries_and_struct():
    from highwayenv_b200 import _native as N

    lib = N.load()
    # LinearVehicle traffic is the `t` argument of the unified entries, not a second set of entry points
    hdr = open(os.path.join(ROOT, "include", "hwyb200.h")).read()
    for sym in ("hwy_highway_linear_reset", "hwy_highway_linear_step", "hwy_highway_linear_autoreset",
                "hwy_highway_linear_substeps", "hwy_highway_autoreset"):
        assert sym not in N.EXPORTS and sym not in hdr, sym
    # a traffic struct without its parameter buffer is refused before any device call
    p, s, t = N.HwyHighwayParams(), N.HwyHighwayState(), N.HwyLinearTraffic()
    P, S, T = C.byref(p), C.byref(s), C.byref(t)
    for rc in (lib.hwy_highway_reset(P, S, T, None, None, None, None),
               lib.hwy_highway_step(P, S, T, None, None, None, None, None, None, None, None, 0, None, None),
               lib.hwy_highway_substeps(P, S, T, 1, None, None)):
        assert rc != 0 and b"null linear traffic parameters" in lib.hwy_last_error()
    assert lib.hwy_abi_version() == N.HWY_ABI_VERSION == 17
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "hwyb200.h"\nint main(){printf("%zu %zu %zu %zu %zu %d\\n", '
           'sizeof(HwyLinearTraffic), offsetof(HwyLinearTraffic, acc_span), offsetof(HwyLinearTraffic, steer_lo), '
           'offsetof(HwyLinearTraffic, steer_span), offsetof(HwyLinearTraffic, acc_lo), HWY_LINEAR_PARAMS);return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    T = N.HwyLinearTraffic
    assert got == [C.sizeof(T), T.acc_span.offset, T.steer_lo.offset, T.steer_span.offset, T.acc_lo.offset,
                   N.HWY_LINEAR_PARAMS]


@pytest.mark.parametrize("ovt", [B + "IntervalVehicle", "highway_env.vehicle.kinematics.Vehicle", B + "Nope"])
def test_other_traffic_types_still_raise(ovt):
    """Only IDMVehicle and the linear classes are on the accelerated path: the highway family (both env ids) and
    the network family that reads the key (exit-v0) raise before touching a device."""
    from highwayenv_b200.envs.exit_env import BatchedExitEnv
    from highwayenv_b200.envs.highway_env import BatchedHighwayEnv, BatchedHighwayEnvFast

    for cls in (BatchedHighwayEnv, BatchedHighwayEnvFast):
        env = object.__new__(cls)
        env.config = dict(cls.default_config(), other_vehicles_type=ovt)
        with pytest.raises(NotImplementedError):
            env._build_params()
    env = object.__new__(BatchedExitEnv)
    env.reset_mode = "device"
    for t in (ovt, B + "LinearVehicle", B + "AggressiveVehicle", B + "DefensiveVehicle"):  # exit keeps IDM only
        env.config = dict(BatchedExitEnv.default_config(), other_vehicles_type=t)
        with pytest.raises(NotImplementedError, match="IDMVehicle"):
            env.define_spaces()
