"""racetrack-large-v0 / v1 and racetrack-oval-v0 / v1 without a GPU: both lane tables against the reference's pinned
to_config, the default configs, every reset of the fixtures (oracle/gen_racetrack_variants.py) re-derived with numpy,
the reward rounding, the HwyRacetrackParams layout and the configurations that raise before any launch."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = ["racetrack_large_random", "racetrack_large_follow", "racetrack_large_traffic", "racetrack_large_v1_follow",
         "racetrack_large_speed15", "racetrack_oval_follow", "racetrack_oval_lanes2", "racetrack_oval_v1_lanes4"]


def load(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    g["config"] = json.loads(str(g.pop("config_json")))
    return g


def config_of(g):
    return {k: v for k, v in g["config"].items() if not k.startswith("_")}


def network_of(g):
    from highwayenv_b200.envs.racetrack_env import track_network

    return track_network(g["config"]["_env_id"], config_of(g))


@pytest.mark.parametrize("fname,builder,n_lanes", [
    ("pinned_to_config_racetrack_large_v0.json", ("large", ()), 27),
    ("pinned_to_config_racetrack_oval_v0.json", ("oval", (100, 3)), 24),
    ("pinned_to_config_racetrack_oval_v0_lanes2.json", ("oval", (100, 2)), 16),
    ("pinned_to_config_racetrack_oval_v0_lanes4.json", ("oval", (100, 4)), 32),
])
def test_network_matches_reference_to_config(fname, builder, n_lanes):
    """Lane order, geometry, line types and speed limits, insertion order included."""
    from highwayenv_b200 import _native as N
    from highwayenv_b200.envs.racetrack_env import make_racetrack_large_network, make_racetrack_oval_network
    from highwayenv_b200.road.network import NetworkTable

    with open(os.path.join(GOLDEN, fname)) as f:
        ref = json.load(f)
    kind, args = builder
    net = make_racetrack_large_network(*args) if kind == "large" else make_racetrack_oval_network(*args)
    ours = json.loads(json.dumps(net.to_config()))
    assert list(ours) == list(ref)
    for f in ref:
        assert list(ours[f]) == list(ref[f])
        for t in ref[f]:
            assert ours[f][t] == ref[f][t], (f, t)
    assert len(net.lanes) == n_lanes <= N.HWY_NET_MAX_LANES
    assert all(L["speed_limit"] == 10.0 and L["width"] == 5 for L in net.lanes)
    back = NetworkTable.from_config(ref)
    for k, v in net.arrays.items():
        assert np.array_equal(back.arrays[k], v), k


@pytest.mark.parametrize("length,no_lanes", [(150, 2), (100.5, 3), (7, 4)])
def test_oval_network_for_other_lengths(length, no_lanes):
    """The oval's geometry scales with length: the straights of ("a","b") run from x = 0 to length + 1 and every lane of
    one road shares its centre, 5 m apart."""
    from highwayenv_b200.envs.racetrack_env import make_racetrack_oval_network

    net = make_racetrack_oval_network(length, no_lanes)
    assert len(net.lanes) == 8 * no_lanes and list(net._graph) == list("abcdefgh")
    for i in range(no_lanes):
        L = net.lanes[net.index[("a", "b", i)]]
        assert (L["sx"], L["sy"], L["ex"], L["ey"]) == (0, 5 * i, length + 1, 5 * i)
        arc = net.lanes[net.index[("b", "c", i)]]
        assert (arc["cx"], arc["cy"], arc["radius"]) == (length, -20, 20 + 5 * i)


@pytest.mark.parametrize("env_id,name", [("racetrack-large-v0", "racetrack_large_random"),
                                         ("racetrack-large-v1", "racetrack_large_v1_follow"),
                                         ("racetrack-oval-v0", "racetrack_oval_follow")])
def test_default_config_matches_reference(env_id, name):
    from highwayenv_b200.config import default_config

    ref = config_of(load(name))
    ours = json.loads(json.dumps(default_config(env_id)))
    ref.pop("offscreen_rendering"), ours.pop("offscreen_rendering")
    assert ours == ref


def rederive_reset(gen, net, other, ego_lanes):
    """_make_vehicles (racetrack_env.py:374-425, the oval's :1340-1392) with numpy on `gen`: (count, x, y) of the
    placed vehicles."""
    ego_id = gen.integers(ego_lanes)
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
    """Every reset of the fixture, re-derived from the words before it (the steps draw nothing): integers(2) for the
    ego's lane on the large track, integers(no_lanes) on the oval."""
    from highwayenv_b200.envs.common.vector_env import pcg64_words, set_pcg64_words
    from highwayenv_b200.envs.racetrack_env import racetrack_params

    g = load(name)
    cfg = config_of(g)
    net = network_of(g)
    ego_lanes = racetrack_params(cfg, g["config"]["_env_id"])["race"].ego_lanes
    assert ego_lanes == (cfg["no_lanes"] if "oval" in name else 2)
    other = int(cfg["other_vehicles"])
    n_resets, ego_lane_ids = 0, set()
    for i, seed in enumerate(g["seeds"]):
        gen = np.random.Generator(np.random.PCG64(np.random.SeedSequence(int(seed))))
        records = [(g["reset_rng"][i], g["reset_count"][i], g["reset_state"][i])]
        records += [(g["autoreset_rng"][i, j], g["autoreset_count"][i, j], g["autoreset_state"][i, j])
                    for j in range(g["autoreset_step"].shape[1]) if g["autoreset_step"][i, j] >= 0]
        for words, count, st in records:
            n, xs, ys = rederive_reset(gen, net, other, ego_lanes)
            assert np.array_equal(pcg64_words([gen])[:, 0], words)
            assert n == count
            assert np.allclose(st[0, :n], xs, rtol=0, atol=1e-12) and np.allclose(st[1, :n], ys, rtol=0, atol=1e-12)
            ego_lane_ids.add(net.lanes[int(st[6, 0])]["lane_id"])
            # make_on_lane(speed=None): the lane's speed limit, config["speed_limit"] on the large track, 10 on the oval
            assert st[3, 0] == net.lanes[int(st[6, 0])]["speed_limit"] == (cfg["speed_limit"] if "large" in name else 10)
            n_resets += 1
            set_pcg64_words([gen], words[:, None])
    assert n_resets > len(g["seeds"])
    assert ego_lane_ids == set(range(ego_lanes))  # every lane the draw can give was drawn


@pytest.mark.parametrize("name", CASES)
def test_action_norm_and_reward_terms(name):
    """The reward's rounding on the stored terms (racetrack_env.py:66-83), as for racetrack-v0: float32 partial sums
    on a StraightLane, float64 on a CircularLane, then the on_road term, lmap and * on_road."""
    from highwayenv_b200 import _native as N

    g = load(name)
    cfg = config_of(g)
    acts = g["actions"][:, g["steps"]]
    pair = np.zeros(acts.shape[:2] + (2,), dtype=np.float32)
    pair[..., 2 - acts.shape[-1]:] = acts
    norm = np.sqrt(pair[..., 0] * pair[..., 0] + pair[..., 1] * pair[..., 1], dtype=np.float32)
    assert np.array_equal(norm.astype(np.float64), g["terms"][..., 1])
    lc, _, col, on_road = (g["terms"][..., k] for k in range(4))
    types = network_of(g).arrays["type"]
    straight = types[g["state"][:, :, 6, 0].astype(int)] == N.LANE_STRAIGHT
    f = np.float32
    term = f(cfg["action_reward"]) * norm
    s32 = ((f(cfg["lane_centering_reward"] * lc) + term) + f(cfg["collision_reward"] * col)).astype(np.float64)
    s64 = (cfg["lane_centering_reward"] * lc + term.astype(np.float64)) + cfg["collision_reward"] * col
    rew = np.where(straight, s32, s64) + 0.0 * on_road
    rew = 0.0 + (rew - cfg["collision_reward"]) * (1.0 - 0.0) / (1.0 - cfg["collision_reward"])
    assert np.array_equal(rew * on_road, g["reward"])
    # random steering leaves the large track's 158 m first straight before any stored step reaches an arc
    assert straight.any() and ((~straight).any() or name == "racetrack_large_random")


def test_struct_layout_matches_gcc():
    """ego_lanes takes the place of the former padding word: the size and every other offset are unchanged."""
    from highwayenv_b200 import _native as N

    T = N.HwyRacetrackParams
    names = [f for f, _ in T._fields_]
    assert "_pad" not in names and T.ego_lanes.offset == 20 and C.sizeof(T) == 64
    assert [getattr(T, f).offset for f in names] == [0, 4, 8, 12, 16, 20, 24, 32, 40, 48, 56]
    src = ('#include <stddef.h>\n#include <stdio.h>\n#include "hwyb200.h"\nint main(){'
           + 'printf("%zu\\n", sizeof(HwyRacetrackParams));'
           + "".join(f'printf("%zu\\n", offsetof(HwyRacetrackParams, {f}));' for f in names) + "return 0;}\n")
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [C.sizeof(T)] + [getattr(T, f).offset for f in names]


def _cfg(env_id, **over):
    from highwayenv_b200.config import default_config

    cfg = default_config(env_id)
    for k, v in over.items():
        keep = k == "action" or (k == "observation" and "type" not in v)
        cfg[k] = {**cfg[k], **v} if (keep and isinstance(v, dict)) else v
    return cfg


@pytest.mark.parametrize("env_id", ["racetrack-large-v0", "racetrack-large-v1", "racetrack-oval-v0",
                                    "racetrack-oval-v1"])
def test_supported_configuration_parameters(env_id):
    from highwayenv_b200.envs.racetrack_env import racetrack_params

    sp = racetrack_params(_cfg(env_id), env_id)
    p, rp = sp["params"], sp["race"]
    assert (sp["action_size"], sp["V"], sp["fused"]) == (1, 2, False)
    assert sp["observation_type"].space().shape == (2, 12, 12)
    oval = "oval" in env_id
    assert (rp.lane_ab, rp.lane_bc, rp.n_from_nodes, rp.ego_lanes) == ((0, 3, 8, 3) if oval else (0, 3, 9, 2))
    assert p.connected_lanes == int(env_id.endswith("v1"))
    # Kinematics' default y range: +-4 m per lane of ("a","b") (normalize_obs, observation.py:214-226)
    sp = racetrack_params(_cfg(env_id, observation={"type": "Kinematics"}), env_id)
    assert (sp["params"].obs_y_lo, sp["params"].obs_y_hi) == (-12.0, 12.0)  # 3 lanes on both tracks by default
    if oval:
        for n in (2, 4):
            rp = racetrack_params(_cfg(env_id, no_lanes=n, length=150), env_id)["race"]
            assert (rp.lane_ab, rp.lane_bc, rp.n_from_nodes, rp.ego_lanes) == (0, n, 8, n)
            p = racetrack_params(_cfg(env_id, no_lanes=n, observation={"type": "Kinematics"}), env_id)["params"]
            assert (p.obs_y_lo, p.obs_y_hi) == (-4.0 * n, 4.0 * n)


@pytest.mark.parametrize("env_id", ["racetrack-large-v0", "racetrack-oval-v0"])
@pytest.mark.parametrize("over,exc", [
    ({"action": {"dynamical": True}}, NotImplementedError),
    ({"action": {"type": "DiscreteMetaAction"}}, NotImplementedError),
    ({"action": {"type": "DiscreteAction"}}, NotImplementedError),
    ({"action": {"lateral": False, "longitudinal": False}}, ValueError),
    ({"controlled_vehicles": 2}, NotImplementedError),
    ({"observation": {"type": "TimeToCollision"}}, NotImplementedError),
    ({"observation": {"type": "LidarObservation"}}, NotImplementedError),
    ({"other_vehicles": 8}, NotImplementedError),
    ({"other_vehicles": -1}, ValueError),
])
def test_racetrack_rejections_hold_on_the_new_tracks(env_id, over, exc):
    """Everything racetrack-v0 rejects is rejected on the large track and the oval, with the same exception type."""
    from highwayenv_b200.envs.racetrack_env import racetrack_params

    with pytest.raises(exc):
        racetrack_params(_cfg("racetrack-v0", **over), "racetrack-v0")
    with pytest.raises(exc):
        racetrack_params(_cfg(env_id, **over), env_id)


@pytest.mark.parametrize("env_id", ["racetrack-oval-v0", "racetrack-oval-v1"])
@pytest.mark.parametrize("over,exc", [
    ({"no_lanes": 0}, NotImplementedError),  # random no_lanes from an unseeded generator
    ({"length": 0}, NotImplementedError),  # random length from an unseeded generator
    ({"no_lanes": 5}, NotImplementedError),  # 40 lanes: more than the 32-lane table
    ({"no_lanes": 7}, NotImplementedError),
    ({"no_lanes": 1}, ValueError),  # two coincident lanes per road
    ({"no_lanes": 2.5}, ValueError),
    ({"length": -10}, ValueError),
    ({"block_lane": True}, NotImplementedError),
    ({"force_decision": True}, NotImplementedError),
])
def test_oval_rejections(env_id, over, exc):
    from highwayenv_b200.envs.racetrack_env import racetrack_params

    with pytest.raises(exc):
        racetrack_params(_cfg(env_id, **over), env_id)


def test_planners_and_discrete_queries_raise():
    from highwayenv_b200 import planning
    from highwayenv_b200.envs.racetrack_env import BatchedRacetrackLargeEnv, BatchedRacetrackOvalEnv

    for cls in (BatchedRacetrackLargeEnv, BatchedRacetrackOvalEnv):
        env = cls.__new__(cls)
        env.n_agents, env.multi_agent = 1, False
        with pytest.raises(NotImplementedError):
            env.to_finite_mdp()
        with pytest.raises(NotImplementedError):
            env.get_available_actions()
        assert cls.ENV_ID not in planning.OPD_ENV_IDS and cls.ENV_ID not in planning.MCTS_ENV_IDS
        for policy in (planning.OpdPolicy, planning.MctsPolicy):
            with pytest.raises(NotImplementedError):
                policy(env)


def test_registered():
    import highwayenv_b200 as hb
    from highwayenv_b200.config import default_config

    for env_id, cls in [("racetrack-large-v0", "BatchedRacetrackLargeEnv"),
                        ("racetrack-large-v1", "BatchedConnectedLaneRacetrackLargeEnv"),
                        ("racetrack-oval-v0", "BatchedRacetrackOvalEnv"),
                        ("racetrack-oval-v1", "BatchedConnectedLaneRacetrackOvalEnv")]:
        assert hb.REGISTRY[env_id].endswith(":" + cls)
        assert default_config(env_id)["neighbour_vehicles_connected_lanes"] is env_id.endswith("v1")
    oval = default_config("racetrack-oval-v0")
    assert (oval["length"], oval["no_lanes"], oval["block_lane"], oval["force_decision"]) == (100, 3, False, False)


@pytest.mark.parametrize("env_id,first,then,lanes", [
    ("racetrack-oval-v1", {}, {"no_lanes": 4}, 32), ("racetrack-oval-v0", {"no_lanes": 4}, {"length": 150}, 32),
    ("racetrack-large-v0", {}, {"speed_limit": 15}, 27), ("racetrack-v0", {}, {"speed_limit": 15}, 18),
])
def test_reconfigure_rebuilds_the_lane_table(env_id, first, then, lanes):
    """reset(options={"config": ...}) runs configure, define_spaces and _allocate: when the new config picks another
    track, the env's lane table and its device copy follow it, so the kernel parameters and the table agree."""
    import torch

    import highwayenv_b200 as hb
    from highwayenv_b200.config import default_config
    from highwayenv_b200.envs.racetrack_env import track_network

    mod, cls = hb.REGISTRY[env_id].split(":")
    cls = getattr(__import__(mod, fromlist=[cls]), cls)
    env = cls.__new__(cls)  # the host half of __init__: no device needed
    env.num_envs, env.device, env.reset_mode = 2, torch.device("cpu"), "device"
    env.config = default_config(env_id)
    env.configure(first)
    env.define_spaces()
    old, old_dev = env.net, env._graph_dev
    env.configure(then)
    env.define_spaces()
    net = env.net
    assert net is track_network(env_id, env.config) and len(net.lanes) == lanes
    changed = env_id != "racetrack-v0"  # racetrack-v0's table does not depend on the config
    assert (net is not old) == changed and (env._graph_dev is not old_dev) == changed
    assert bytes(env._graph_dev.numpy()) == bytes(net.to_struct())
    assert env._race.lane_bc == net.index[("b", "c", 0)] and env._race.n_from_nodes == len(net._graph)
    assert env._race.ego_lanes <= net.lanes[net.index[("a", "b", 0)]]["road_count"]
    if "speed_limit" in then and env_id != "racetrack-v0":
        assert all(L["speed_limit"] == 15.0 for L in net.lanes)
