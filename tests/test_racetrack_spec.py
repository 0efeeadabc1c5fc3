"""racetrack-v0 / racetrack-v1 without a GPU: the lane table and default config against the reference's, the reset draws
of the fixtures (oracle/gen_racetrack.py) re-derived with numpy, the float32 action arithmetic the kernel restates, the
C structs against gcc, the configurations that raise before any launch, and one seed rerun against the live reference
when it is present."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = ["racetrack_random", "racetrack_follow", "racetrack_traffic", "racetrack_v1_follow", "racetrack_kinematics"]


def load(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    g["config"] = json.loads(str(g.pop("config_json")))
    return g


def config_of(g):
    return {k: v for k, v in g["config"].items() if not k.startswith("_")}


def test_network_matches_reference_to_config():
    from highwayenv_b200.envs.racetrack_env import make_racetrack_network
    from highwayenv_b200.road.network import NetworkTable

    with open(os.path.join(GOLDEN, "pinned_to_config_racetrack_v0.json")) as f:
        ref = json.load(f)
    net = make_racetrack_network()
    ours = json.loads(json.dumps(net.to_config()))
    # lane order, geometry, line types and speed limits, insertion order included
    assert list(ours) == list(ref)
    for f in ref:
        assert list(ours[f]) == list(ref[f])
        for t in ref[f]:
            assert ours[f][t] == ref[f][t], (f, t)
    assert len(net.lanes) == 18 and all(L["speed_limit"] == 10.0 and L["width"] == 5 for L in net.lanes)
    back = NetworkTable.from_config(ref)
    for k, v in net.arrays.items():
        assert np.array_equal(back.arrays[k], v), k


@pytest.mark.parametrize("env_id,name", [("racetrack-v0", "racetrack_random"), ("racetrack-v1", "racetrack_v1_follow")])
def test_default_config_matches_reference(env_id, name):
    from highwayenv_b200.config import default_config

    ref = config_of(load(name))
    ours = json.loads(json.dumps(default_config(env_id)))
    # AbstractEnv reads offscreen_rendering from the environment of the process that made the fixture
    ref.pop("offscreen_rendering"), ours.pop("offscreen_rendering")
    assert ours == ref


def rederive_reset(gen, net, other):
    """_make_vehicles (racetrack_env.py:374-425) with numpy on `gen`: (count, x, y) of the placed vehicles."""
    ego_id = gen.integers(2)
    lon = gen.uniform(20, 50)
    xs, ys = [], []
    x, y = net.position(net.index[("a", "b", int(ego_id))], lon, 0.0)
    xs.append(float(x)), ys.append(float(y))
    if other > 0:
        lane = net.index[("b", "c", int(ego_id))]
        lon = gen.uniform(low=0.0, high=net.lanes[net.index[("b", "c", 0)]]["length"])
        gen.uniform(high=3.0)
        x, y = net.position(lane, lon, 0.0)
        xs.append(float(x)), ys.append(float(y))
        froms = list(net._graph)
        for _ in range(gen.integers(other)):
            f = gen.choice(froms)
            t = gen.choice(list(net._graph[f]))
            lid = gen.integers(len(net._graph[f][t]))
            lane = net.index[(str(f), str(t), int(lid))]
            lon = gen.uniform(low=0.0, high=net.lanes[lane]["length"])
            gen.uniform(high=3.0)
            x, y = net.position(lane, lon, 0.0)
            if all(np.linalg.norm(np.array([x, y]) - np.array([a, b])) >= 20 for a, b in zip(xs, ys)):
                xs.append(float(x)), ys.append(float(y))
    return len(xs), np.array(xs), np.array(ys)


@pytest.mark.parametrize("name", CASES)
def test_reset_draws_match_stream_words(name):
    """Every reset of the fixture, re-derived from the words before it: the steps draw nothing, so the words before an
    autoreset are those of the previous reset."""
    from highwayenv_b200.envs.common.vector_env import pcg64_words, set_pcg64_words
    from highwayenv_b200.envs.racetrack_env import make_racetrack_network

    g = load(name)
    net = make_racetrack_network()
    other = int(config_of(g)["other_vehicles"])
    n_resets = 0
    for i, seed in enumerate(g["seeds"]):
        gen = np.random.Generator(np.random.PCG64(np.random.SeedSequence(int(seed))))
        records = [(g["reset_rng"][i], g["reset_count"][i], g["reset_state"][i])]
        records += [(g["autoreset_rng"][i, j], g["autoreset_count"][i, j], g["autoreset_state"][i, j])
                    for j in range(g["autoreset_step"].shape[1]) if g["autoreset_step"][i, j] >= 0]
        for words, count, st in records:
            n, xs, ys = rederive_reset(gen, net, other)
            assert np.array_equal(pcg64_words([gen])[:, 0], words)
            assert n == count
            assert np.allclose(st[0, :n], xs, rtol=0, atol=1e-12) and np.allclose(st[1, :n], ys, rtol=0, atol=1e-12)
            n_resets += 1
            set_pcg64_words([gen], words[:, None])
    assert n_resets > len(g["seeds"])


def test_staged_throttle_is_exact_zero():
    """A lateral-only action is staged as (0, steering) with the acceleration range (0, 0): the kernel's float32 lmap
    (action.py:136-160, utils.lmap) then yields +0.0, the reference's "acceleration": 0."""
    f = np.float32
    for lo_hi in [(0.0, 0.0)]:
        acc = f(lo_hi[0]) + (f(0.0) - f(-1.0)) * f(lo_hi[1] - lo_hi[0]) / f(2.0)
        assert acc == 0.0 and not np.signbit(acc) and acc.dtype == np.float32


@pytest.mark.parametrize("name", CASES)
def test_action_norm_and_reward_terms(name):
    """np.linalg.norm of the float32 action equals the kernel's sqrt(a0 * a0 + a1 * a1) in float32 (a missing axis
    staged as 0), and the reward's rounding (racetrack_env.py:66-70): on a StraightLane, whose local_coordinates returns
    python floats, NEP 50 keeps the partial sums with the float32 action term in float32 through the collision term; on
    a CircularLane (np.float64 coordinates) they are float64.  Then the int64 on_road term, lmap and * on_road."""
    from highwayenv_b200 import _native as N
    from highwayenv_b200.envs.racetrack_env import make_racetrack_network

    g = load(name)
    cfg = config_of(g)
    steps = g["steps"]
    acts = g["actions"][:, steps]
    pair = np.zeros(acts.shape[:2] + (2,), dtype=np.float32)
    pair[..., 2 - acts.shape[-1]:] = acts
    norm = np.sqrt(pair[..., 0] * pair[..., 0] + pair[..., 1] * pair[..., 1], dtype=np.float32)
    assert np.array_equal(norm.astype(np.float64), g["terms"][..., 1])
    lc, _, col, on_road = (g["terms"][..., k] for k in range(4))
    types = make_racetrack_network().arrays["type"]
    straight = types[g["state"][:, :, 6, 0].astype(int)] == N.LANE_STRAIGHT  # the ego's lane after the step
    f = np.float32
    term = f(cfg["action_reward"]) * norm
    s32 = ((f(cfg["lane_centering_reward"] * lc) + term) + f(cfg["collision_reward"] * col)).astype(np.float64)
    s64 = (cfg["lane_centering_reward"] * lc + term.astype(np.float64)) + cfg["collision_reward"] * col
    rew = np.where(straight, s32, s64) + 0.0 * on_road
    rew = 0.0 + (rew - cfg["collision_reward"]) * (1.0 - 0.0) / (1.0 - cfg["collision_reward"])
    assert np.array_equal(rew * on_road, g["reward"])
    assert straight.any() and (~straight).any()


def test_struct_layout_matches_gcc():
    import ctypes as C

    from highwayenv_b200 import _native as N

    names = [f for f, _ in N.HwyRacetrackParams._fields_]
    src = ('#include <stddef.h>\n#include <stdio.h>\n#include "hwyb200.h"\nint main(){'
           + 'printf("%zu\\n", sizeof(HwyRacetrackParams));'
           + "".join(f'printf("%zu\\n", offsetof(HwyRacetrackParams, {f}));' for f in names) + "return 0;}\n")
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    want = [C.sizeof(N.HwyRacetrackParams)] + [getattr(N.HwyRacetrackParams, f).offset for f in names]
    assert got == want
    hdr = open(os.path.join(ROOT, "include", "hwyb200.h")).read()
    assert "#define HWY_ABI_VERSION 17" in hdr and N.HWY_ABI_VERSION == 17
    # the racetrack runs on the network entry points with its scenario, not on entry points of its own
    for sym in ("hwy_network_reset", "hwy_network_step", "hwy_network_substeps"):
        assert sym in N.EXPORTS and sym + "(" in hdr
    for sym in ("hwy_racetrack_reset", "hwy_racetrack_step"):
        assert sym not in N.EXPORTS and sym not in hdr, sym


def _cfg(**over):
    from highwayenv_b200.config import default_config

    cfg = default_config("racetrack-v0")
    for k, v in over.items():
        # a new observation type starts from that type's defaults, as in the reference's config dict
        keep = k == "action" or (k == "observation" and "type" not in v)
        cfg[k] = {**cfg[k], **v} if keep else v
    return cfg


def test_supported_configuration_parameters():
    from highwayenv_b200 import _native as N
    from highwayenv_b200.envs.racetrack_env import racetrack_params

    sp = racetrack_params(_cfg())
    p, rp = sp["params"], sp["race"]
    assert (sp["action_size"], sp["V"], sp["fused"]) == (1, 2, False)
    assert sp["observation_type"].space().shape == (2, 12, 12)
    assert (p.acc_lo, p.acc_hi, p.steer_lo, p.steer_hi) == (0.0, 0.0, -np.pi / 4, np.pi / 4)
    assert (p.action_type, p.dynamical, p.act_clip, p.n_vehicles) == (1, 0, 1, 2)
    assert (rp.lane_ab, rp.lane_bc, rp.n_from_nodes, rp.other_vehicles, rp.terminate_off_road) == (0, 2, 9, 1, 1)
    sp = racetrack_params(_cfg(other_vehicles=6, action={"longitudinal": True}, observation={"type": "Kinematics"}))
    assert (sp["action_size"], sp["V"], sp["fused"]) == (2, 7, True)
    assert (sp["params"].acc_lo, sp["params"].acc_hi, sp["params"].obs_type) == (-5.0, 5.0, N.OBS_KINEMATICS)
    sp = racetrack_params(_cfg(action={"longitudinal": True, "lateral": False}))
    assert (sp["action_size"], sp["params"].steer_lo, sp["params"].steer_hi) == (1, 0.0, 0.0)


@pytest.mark.parametrize("over,exc", [
    ({"action": {"dynamical": True}}, NotImplementedError),
    ({"action": {"type": "DiscreteMetaAction"}}, NotImplementedError),
    ({"action": {"type": "DiscreteAction"}}, NotImplementedError),
    ({"action": {"lateral": False, "longitudinal": False}}, ValueError),
    ({"controlled_vehicles": 2}, NotImplementedError),
    ({"observation": {"type": "TimeToCollision"}}, NotImplementedError),
    ({"observation": {"type": "LidarObservation"}}, NotImplementedError),
    ({"other_vehicles": 8}, NotImplementedError),
])
def test_unsupported_configuration_raises(over, exc):
    from highwayenv_b200.envs.racetrack_env import racetrack_params

    with pytest.raises(exc):
        racetrack_params(_cfg(**over))


def test_planners_and_discrete_queries_raise():
    """to_finite_mdp, get_available_actions, OpdPolicy and MctsPolicy refuse racetrack before any launch."""
    from highwayenv_b200 import planning
    from highwayenv_b200.envs.racetrack_env import BatchedRacetrackEnv

    env = BatchedRacetrackEnv.__new__(BatchedRacetrackEnv)
    env.n_agents, env.multi_agent = 1, False
    with pytest.raises(NotImplementedError):
        env.to_finite_mdp()
    with pytest.raises(NotImplementedError):
        env.get_available_actions()
    assert "racetrack-v0" not in planning.OPD_ENV_IDS and "racetrack-v1" not in planning.MCTS_ENV_IDS
    for policy in (planning.OpdPolicy, planning.MctsPolicy):
        with pytest.raises(NotImplementedError):
            policy(env)


def test_registered():
    import highwayenv_b200 as hb

    assert hb.REGISTRY["racetrack-v0"].endswith(":BatchedRacetrackEnv")
    assert hb.REGISTRY["racetrack-v1"].endswith(":BatchedConnectedLaneRacetrackEnv")


def test_one_seed_rerun_against_reference():
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import gen_racetrack as gr

    if not gr.rh.reference_available():
        pytest.skip("the reference checkout is not present")
    g = load("racetrack_follow")
    env_id, over, policy = gr.CASES["racetrack_follow"]
    _, actions, first, flags, per_step, resets = gr.run_seed(env_id, over, policy, int(g["seeds"][3]))
    assert np.array_equal(actions, g["actions"][3]) and np.array_equal(flags, g["flags"][3])
    assert np.array_equal(first["state"], g["reset_state"][3]) and np.array_equal(first["rng"], g["reset_rng"][3])
    for j, t in enumerate(g["steps"]):
        assert np.array_equal(per_step[t]["state"], g["state"][3, j]) and per_step[t]["reward"] == g["reward"][3, j]
