"""Multi-agent highway-v0 / highway-fast-v0 without a GPU: the spawn layout, the rejections before any launch, the
spaces of the four MultiAgentAction / MultiAgentObservation combinations, the parameter struct against gcc, and (when
the reference checkout is present) the fixtures re-run live."""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from highwayenv_b200 import _native as N
from highwayenv_b200.config import default_config
from highwayenv_b200.envs.highway_env import BatchedHighwayEnv, BatchedHighwayEnvFast, ego_slots

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_harness as rh  # noqa: E402


def near_split(x, num_bins):
    """utils.near_split(x, num_bins=...) (utils.py:355): quotient + 1 for the first `remainder` bins."""
    q, r = divmod(x, num_bins)
    return [q + 1] * r + [q] * (num_bins - r)


def spec_env(cls=BatchedHighwayEnv, num_envs=2, **cfg):
    """define_spaces() of an env without its constructor's device checks (what raises before any launch)."""
    env = cls.__new__(cls)
    env.num_envs = num_envs
    env.config = default_config(cls.ENV_ID)
    env.config.update(cfg)
    env.define_spaces()
    return env


def multi(A, action="DiscreteMetaAction", observation="Kinematics", multi_action=True, multi_obs=True, **extra):
    act = {"type": action}
    obs = {"type": observation}
    return dict(controlled_vehicles=A,
                action={"type": "MultiAgentAction", "action_config": act} if multi_action else act,
                observation={"type": "MultiAgentObservation", "observation_config": obs} if multi_obs else obs,
                **extra)


@pytest.mark.parametrize("count,A", [(50, 2), (20, 3), (3, 5), (0, 4), (119, 8), (7, 7), (10, 1)])
def test_slot_layout_matches_near_split(count, A):
    bins = near_split(count, A)
    want, s = [], 0
    for b in bins:
        want.append(s)
        s += 1 + b
    assert ego_slots(count, A) == want
    assert s == count + A


def test_slot_layout_against_the_reference():
    if not rh.reference_available():
        pytest.skip("reference checkout not present")
    rh._ensure_imports()
    from highway_env.utils import near_split as ref_near_split

    for count in range(0, 60):
        for A in range(1, 9):
            assert near_split(count, A) == list(ref_near_split(count, num_bins=A)), (count, A)


def test_rejections_before_any_launch():
    with pytest.raises(ValueError):
        spec_env(**multi(9))
    with pytest.raises(ValueError):
        spec_env(**multi(0))
    with pytest.raises(NotImplementedError):
        spec_env(other_vehicles_type="highway_env.vehicle.behavior.LinearVehicle", **multi(2))
    with pytest.raises(ValueError):
        spec_env(vehicles_count=121, **multi(8))
    spec_env(vehicles_count=120, **multi(8))
    from highwayenv_b200 import planning

    env = spec_env(**multi(2))
    with pytest.raises(NotImplementedError):
        planning.mdp_params(env)
    for name in ("OPD", "MCTS"):
        with pytest.raises(NotImplementedError):
            planning._check_tree_search_env(env, name)


@pytest.mark.parametrize("ma,mo", [(True, True), (True, False), (False, True), (False, False)])
def test_space_shapes(ma, mo):
    A = 3
    env = spec_env(BatchedHighwayEnvFast, num_envs=4, **multi(A, multi_action=ma, multi_obs=mo))
    assert env.n_agents == A and env.multi_agent == (ma or mo)
    assert env.single_observation_space.shape == ((A,) if mo else ()) + (5, 5)
    assert env.observation_space.shape == (4,) + env.single_observation_space.shape
    assert env.single_action_space.shape == ((A,) if ma else ())
    p = env._params
    assert (p.n_agents, p.multi_action, p.multi_obs, p.n_vehicles) == (A, int(ma), int(mo), 20 + A)
    cont = spec_env(num_envs=4, **multi(A, action="ContinuousAction", multi_action=ma, multi_obs=mo))
    assert cont.single_action_space.shape == ((A, 2) if ma else (2,))
    ttc = spec_env(num_envs=4, **multi(A, observation="TimeToCollision", multi_action=ma, multi_obs=mo))
    assert ttc.single_observation_space.shape == ((A,) if mo else ()) + (3, 3, 10)
    assert ttc._params.multi_obs == 0  # a standalone plugin observes per agent, not the step kernel


def test_one_agent_runs_the_single_agent_kernels():
    env = spec_env(**multi(1))
    assert (env._params.n_agents, env._params.multi_action, env._params.multi_obs) == (0, 0, 0)
    assert env.single_observation_space.shape == (1, 5, 5) and env.single_action_space.shape == (1,)


def test_new_struct_fields_against_gcc():
    fields = ("obs_n_features", "n_agents", "multi_action", "multi_obs", "obs_feature")
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "hwyb200.h"\nint main(){printf("%zu %zu ' + \
          ' '.join(["%zu"] * len(fields)) + '\\n", sizeof(HwyHighwayParams), sizeof(((HwyHighwayParams*)0)->n_agents), ' + \
          ', '.join(f"offsetof(HwyHighwayParams, {f})" for f in fields) + ');return 0;}\n'
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    want = [C.sizeof(N.HwyHighwayParams), C.sizeof(C.c_int16)] + [getattr(N.HwyHighwayParams, f).offset for f in fields]
    assert got == want


def test_abi_refuses_bad_agent_counts_before_the_device():
    lib = N.load()
    p, s = N.HwyHighwayParams(), N.HwyHighwayState()
    p.lanes_count, p.n_vehicles, p.obs_vehicles_count, p.n_target_speeds = 3, 5, 5, 3
    p.simulation_frequency = p.policy_frequency = 1
    for A, msg in ((9, b"n_agents"), (-1, b"n_agents"), (6, b"n_agents exceeds")):
        p.n_agents = A
        assert lib.hwy_highway_observe(C.byref(p), C.byref(s), None, None) != 0
        assert msg in lib.hwy_last_error(), lib.hwy_last_error()


FIXTURES = ["multi_highway_v0_a2", "multi_highway_fast_a3", "multi_highway_fast_plain_action",
            "multi_highway_v0_continuous", "multi_highway_fast_ttc"]


@pytest.mark.parametrize("name", FIXTURES + ["multi_highway_resets"])
def test_fixture_reruns_live(name):
    """Seed 0 of each fixture (configuration 0 of the resets) re-run on the unmodified reference, step by step."""
    if not rh.reference_available():
        pytest.skip("reference checkout not present")
    import gen_multi_agent_highway as gm

    g = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    if name == "multi_highway_resets":
        cfg, env_id = json.loads(str(g["c0_config"])), str(g["c0_env_id"])
        out = rh.rollout(env_id, cfg, int(g["c0_seeds"][0]), [])
        for k in ("x", "y", "speed", "lane", "obs", "rng_words"):
            assert np.array_equal(np.asarray(out[k])[0], g[f"c0_{k}"][0]), k
        return
    env_id, cfg, A, kind, _, T = gm.CASES[name]
    out = rh.rollout(env_id, cfg, 0, gm.actions_for(kind, A, 0, T))
    for k in ("x", "y", "heading", "speed", "lane", "target_lane", "crashed", "obs", "rng_words"):
        assert np.array_equal(np.asarray(out[k]), g[k][0]), k
    for k in ("reward", "terminated", "truncated"):
        assert np.array_equal(out[k], g[k][0]), k


def test_load_state_dict_refuses_surplus_controlled_vehicles():
    """speed_index holds [N, A]: a state with more controlled kinds than controlled_vehicles in an env is refused
    before anything reaches the device."""
    env = spec_env(**multi(2))
    kind = np.zeros((2, 22), dtype=np.int32)
    kind[:, [0, 11]] = N.KIND_MDP
    kind[1, 5] = N.KIND_VEHICLE
    with pytest.raises(ValueError):
        env.load_state_dict({"kind": kind})
