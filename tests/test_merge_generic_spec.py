"""merge-generic-v0 / v1 without a GPU: the lane tables against the reference's pinned to_config, the default configs,
every reset of the fixtures (oracle/gen_merge_generic.py) re-derived with numpy from the stream words before it, the
termination threshold, the extended HwyMergeSpawn and HwyNetParams.merge_end_lane layouts, registration and the
configurations that raise before any launch."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = ["mg_default", "mg_v1_default", "mg_three_lanes", "mg_one_lane_ttc", "mg_crowded_32", "mg_float_grid"]
LENGTHS = ("before_merge_length", "converge_merge_length", "parallel_merge_length", "after_merge_length")


def load(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    g["config"] = json.loads(str(g.pop("config_json")))
    return g


def config_of(g):
    return {k: v for k, v in g["config"].items() if not k.startswith("_")}


def network_of(cfg):
    from highwayenv_b200.envs.merge_env import merge_generic_network

    return merge_generic_network(cfg["lanes_count"], *(cfg[k] for k in LENGTHS))


def records(g, i):
    """(stream words, record) of seed i's seeded reset and of each autoreset, in order."""
    out = [(g["reset_rng"][i], {k[6:]: g[k][i] for k in g if k.startswith("reset_")})]
    for j in range(g["autoreset_step"].shape[1]):
        if g["autoreset_step"][i, j] >= 0:
            out.append((g["autoreset_rng"][i, j], {k[10:]: g[k][i, j] for k in g if k.startswith("autoreset_")
                                                   and k != "autoreset_step"}))
    return out


PINNED = [(2, 150, 80, 80, 150), (1, 150, 80, 80, 150), (3, 97.5, 62.25, 80.5, 120.5), (9, 150, 80, 80, 150)]


@pytest.mark.parametrize("lanes,pre,conv,par,after", PINNED)
def test_network_matches_reference_to_config(lanes, pre, conv, par, after):
    """Lane order, geometry, line types and speed limits, insertion order included, bit for bit."""
    from highwayenv_b200 import _native as N
    from highwayenv_b200.envs.merge_env import make_merge_generic_network, merge_generic_network
    from highwayenv_b200.road.network import NetworkTable

    with open(os.path.join(GOLDEN, f"pinned_to_config_merge_generic_l{lanes}_{pre}_{conv}_{par}_{after}.json")) as f:
        ref = json.load(f)
    net = make_merge_generic_network(lanes, pre, conv, par, after)
    ours = json.loads(json.dumps(net.to_config()))
    assert list(ours) == list(ref)
    for f in ref:
        assert list(ours[f]) == list(ref[f])
        for t in ref[f]:
            assert ours[f][t] == ref[f][t], (f, t)
    assert len(net.lanes) == 3 * lanes + 3 <= N.HWY_NET_MAX_LANES
    back = NetworkTable.from_config(ref)
    for k, v in net.arrays.items():
        assert np.array_equal(back.arrays[k], v), k
    assert all(L["speed_limit"] == 30 for L in net.lanes)  # merge-v0's lanes keep the default 20
    assert merge_generic_network(lanes, pre, conv, par, after) is merge_generic_network(lanes, pre, conv, par, after)


@pytest.mark.parametrize("env_id,name", [("merge-generic-v0", "mg_default"), ("merge-generic-v1", "mg_v1_default")])
def test_default_config_matches_reference(env_id, name):
    from highwayenv_b200.config import default_config

    ref = config_of(load(name))
    ours = json.loads(json.dumps(default_config(env_id)))
    ref.pop("offscreen_rendering"), ours.pop("offscreen_rendering")
    assert ours == ref
    assert [ours[k] for k in ("lanes_count", "vehicles_count") + LENGTHS] == [2, 3, 150, 80, 80, 150]


def rederive_reset(gen, net, cfg):
    """MergeGenericEnv._make_vehicles (merge_env.py:320-368) and the Obstacle with numpy on `gen`: per placed object
    (x, y, speed, target speed, kind, closest lane at heading 0), the Obstacle last."""
    lanes = int(cfg["lanes_count"])
    pre, conv, par = (cfg[k] for k in LENGTHS[:3])
    ab = [net.index[("a", "b", k)] for k in range(lanes)]
    x, y = net.position(ab[lanes - 1], 30.0, 0.0)
    placed = [(float(x), float(y), 30.0, np.nan, 1)]
    spawned = {k: [] for k in range(lanes)}
    spawned[lanes - 1].append(30.0)
    for _ in range(int(cfg["vehicles_count"])):
        for _ in range(10):
            k = int(gen.integers(lanes))
            lon = gen.uniform(0, pre + conv + par)
            if all(abs(lon - p) > 15.0 for p in spawned[k]):
                x, y = net.position(ab[k], lon, 0.0)
                speed = 30.0 + gen.uniform(-2.0, 2.0)
                placed.append((float(x), float(y), speed, speed, 0))
                spawned[k].append(lon)
                break
    x, y = net.position(net.index[("j", "k", 0)], 60.0, 0.0)
    placed.append((float(x), float(y), 20.0, 30.0, 0))
    x, y = net.position(net.index[("b", "c", lanes)], par, 0.0)
    placed.append((float(x), float(y), 0.0, np.nan, 3))
    xs, ys = (np.array([v[k] for v in placed]) for k in range(2))
    return dict(x=xs, y=ys, speed=np.array([v[2] for v in placed]), target_speed=np.array([v[3] for v in placed]),
                kind=np.array([v[4] for v in placed]), lane=net.closest_lane(xs, ys, np.zeros_like(xs)))


@pytest.mark.parametrize("name", CASES)
def test_reset_draws_match_stream_words(name):
    """Every reset of the fixture re-derived from the words before it (the steps draw nothing): stream words,
    population, kinds, positions, speeds and lanes all exact; headings 0."""
    from highwayenv_b200.envs.common.vector_env import pcg64_words, set_pcg64_words

    g = load(name)
    cfg = config_of(g)
    net = network_of(cfg)
    full = 3 + int(cfg["vehicles_count"])
    n_resets, counts = 0, []
    for i, seed in enumerate(g["seeds"]):
        gen = np.random.Generator(np.random.PCG64(np.random.SeedSequence(int(seed))))
        for words, rec in records(g, i):
            r = rederive_reset(gen, net, cfg)
            assert np.array_equal(pcg64_words([gen])[:, 0], words)
            n = len(r["x"])
            assert n == int(rec["count"]), (name, i)
            for k in ("x", "y", "speed", "kind"):
                assert np.array_equal(rec[k][:n], r[k]), (name, i, k)
            assert np.array_equal(rec["target_speed"][1:n - 1], r["target_speed"][1:n - 1])
            assert np.array_equal(rec["heading"][:n], np.zeros(n))
            assert np.array_equal(rec["lane"][:n], r["lane"])
            assert np.array_equal(rec["delta"][1:n - 1], np.full(n - 2, 4.0))  # no randomize_behavior
            counts.append(n)
            n_resets += 1
            set_pcg64_words([gen], words[:, None])
    assert n_resets > len(g["seeds"])
    if name == "mg_crowded_32":  # the population varies: every reset skipped a vehicle, some more than others
        assert max(counts) < full and min(counts) < max(counts)
    else:
        assert min(counts) == full


@pytest.mark.parametrize("name", CASES)
def test_end_position_is_the_lane_end_minus_90(name):
    """end_position = pre + conv + par + after - 90 equals, bit for bit, the stored end x of the ("c","d") lanes
    (start + length, the sum the reference forms) - 90, which is what the step compares the ego's x with."""
    g = load(name)
    net = network_of(config_of(g))
    ends = {float(net.lanes[net.index[("c", "d", k)]]["ex"]) for k in range(int(g["config"]["lanes_count"]))}
    assert len(ends) == 1
    assert np.array_equal(ends.pop() - 90.0, g["reset_end_position"][0])
    assert len(set(g["reset_end_position"].tolist())) == 1


def test_float_lengths_give_a_non_integer_end_position():
    g = load("mg_float_grid")
    assert float(g["reset_end_position"][0]) == 97.5 + 62.25 + 80.5 + 120.5 - 90 == 270.75


def _gcc_offsets(struct, fields):
    src = ('#include <stddef.h>\n#include <stdio.h>\n#include "hwyb200.h"\nint main(){'
           + f'printf("%zu\\n", sizeof({struct}));'
           + "".join(f'printf("%zu\\n", offsetof({struct}, {f}));' for f in fields) + "return 0;}\n")
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", exe])
        return [int(x) for x in subprocess.check_output([exe]).split()]


def test_struct_layout_matches_gcc():
    from highwayenv_b200 import _native as N

    T = N.HwyMergeSpawn
    names = [f for f, _ in T._fields_]
    assert C.sizeof(T) == 48 and (T.lanes_count.offset, T.vehicles_count.offset, T.max_position.offset) == (32, 36, 40)
    assert _gcc_offsets("HwyMergeSpawn", names) == [C.sizeof(T)] + [getattr(T, f).offset for f in names]
    P = N.HwyNetParams
    assert C.sizeof(P) == 832 and P.merge_end_lane.offset == 364
    assert _gcc_offsets("HwyNetParams", ["merge_lane", "merge_end_lane", "left_lane_reward"]) == \
        [832, P.merge_lane.offset, 364, P.left_lane_reward.offset]
    S = N.HwyNetScenario
    assert C.sizeof(S) == 192 and S.u.offset == 8
    assert _gcc_offsets("HwyNetScenario", ["kind", "u"]) == [192, 0, 8]


def _host_env(env_id, over=None, reset_mode="device"):
    """The host half of __init__ (configure + define_spaces): no device needed."""
    import torch

    import highwayenv_b200 as hb
    from highwayenv_b200.config import default_config

    mod, cls = hb.REGISTRY[env_id].split(":")
    cls = getattr(__import__(mod, fromlist=[cls]), cls)
    env = cls.__new__(cls)
    env.num_envs, env.device, env.reset_mode = 2, torch.device("cpu"), reset_mode
    env.config = default_config(env_id)
    env.configure(over)
    env.define_spaces()
    env._build_spawn_tables()  # the scenario (no device buffers on these families)
    return env


@pytest.mark.parametrize("env_id", ["merge-generic-v0", "merge-generic-v1"])
@pytest.mark.parametrize("over,exc", [
    ({"lanes_count": 0}, ValueError),
    ({"lanes_count": -1}, ValueError),
    ({"lanes_count": 2.0}, ValueError),
    ({"lanes_count": True}, ValueError),
    ({"lanes_count": 10}, NotImplementedError),
    ({"before_merge_length": 0}, ValueError),
    ({"converge_merge_length": -5}, ValueError),
    ({"parallel_merge_length": 0.0}, ValueError),
    ({"after_merge_length": 89.99}, ValueError),
    ({"vehicles_count": 30}, NotImplementedError),
    ({"vehicles_count": 50}, NotImplementedError),
    ({"vehicles_count": 2.5}, ValueError),
    ({"action": {"type": "ContinuousAction"}}, NotImplementedError),
    ({"action": {"type": "DiscreteAction"}}, NotImplementedError),
    ({"action": {"type": "Nothing"}}, ValueError),
])
def test_rejections(env_id, over, exc):
    """Raised by define_spaces, which __init__ and reset(options={"config": ...}) run before any allocation or
    launch."""
    with pytest.raises(exc):
        _host_env(env_id, over)


def test_rejections_quote_the_reference():
    with pytest.raises(ValueError, match="All road segments must have positive length"):
        _host_env("merge-generic-v0", {"converge_merge_length": 0})
    with pytest.raises(ValueError, match="The after merge road segment must have length >= 90"):
        _host_env("merge-generic-v0", {"after_merge_length": 60})


def test_host_reset_mode_raises():
    with pytest.raises(NotImplementedError):
        _host_env("merge-generic-v0", reset_mode="host")


@pytest.mark.parametrize("over,slots,V,lanes,merge_lane", [
    ({}, 8, 6, 9, 4), ({"vehicles_count": 5}, 8, 8, 9, 4), ({"vehicles_count": 6}, 32, 9, 9, 4),
    ({"vehicles_count": 29, "lanes_count": 1}, 32, 32, 6, -1), ({"vehicles_count": -3}, 8, 3, 9, 4),
    ({"lanes_count": 3, "vehicles_count": 0}, 8, 3, 12, 5), ({"lanes_count": 9}, 8, 6, 30, 11),
])
def test_slots_and_parameters(over, slots, V, lanes, merge_lane):
    env = _host_env("merge-generic-v0", over)
    L = env.config["lanes_count"]
    assert (env.SLOTS, env.N_VEHICLES, env._params.n_vehicles, len(env.net.lanes)) == (slots, V, V, lanes)
    p = env._params
    assert p.reward_type == 2 and p.connected_lanes == 0 and p.merge_lane == merge_lane
    assert p.merge_end_lane == env.net.index[("c", "d", 0)] == 2 * L + 1
    assert (p.obs_y_lo, p.obs_y_hi) == (-4.0 * L, 4.0 * L)  # all_side_lanes of ("a","b",L-1)
    sp = env._scenario.u.merge
    assert (env._scenario.kind, sp.lanes_count, sp.vehicles_count) == (3, L, env.config["vehicles_count"])
    assert (sp.lane_ab[0], sp.lane_jk, sp.max_position) == (0, 3 * L + 1, 310.0)
    assert (sp.obstacle_x, sp.obstacle_y) == (310.0, 4.0 * L)
    assert _host_env("merge-generic-v1", over)._params.connected_lanes == 1


def test_merge_v0_keeps_its_threshold_and_spawn():
    """merge-v0 leaves merge_end_lane 0 (x > 370) and lanes_count 0 (its fixed placement)."""
    env = _host_env("merge-v0")
    assert env._params.merge_end_lane == 0 and env._scenario.u.merge.lanes_count == 0
    assert env._params.merge_lane == env.net.index[("b", "c", 2)]


def test_reconfigure_rebuilds_the_lane_table():
    """A new lanes_count or length rebuilds the table and its device copy; the same key keeps both."""
    from highwayenv_b200.envs.merge_env import merge_generic_network

    env = _host_env("merge-generic-v0")
    old, old_dev = env.net, env._graph_dev
    env.configure({"vehicles_count": 12})
    env.define_spaces()
    assert env.net is old and env._graph_dev is old_dev and env.SLOTS == 32
    env.configure({"lanes_count": 3, "after_merge_length": 120.5})
    env.define_spaces()
    assert env.net is merge_generic_network(3, 150, 80, 80, 120.5) and env.net is not old
    assert env._graph_dev is not old_dev and bytes(env._graph_dev.numpy()) == bytes(env.net.to_struct())
    assert len(env.net.lanes) == 12 and env._params.obs_y_hi == 12.0


def test_planners_raise():
    from highwayenv_b200 import planning
    from highwayenv_b200.envs.merge_env import BatchedMergeGenericEnv

    env = BatchedMergeGenericEnv.__new__(BatchedMergeGenericEnv)
    env.n_agents, env.multi_agent = 1, False
    with pytest.raises(NotImplementedError):
        env.to_finite_mdp()
    for env_id in ("merge-generic-v0", "merge-generic-v1"):
        assert env_id not in planning.OPD_ENV_IDS and env_id not in planning.MCTS_ENV_IDS
    for policy in (planning.OpdPolicy, planning.MctsPolicy):
        with pytest.raises(NotImplementedError):
            policy(env)


def test_registered():
    import highwayenv_b200 as hb
    from highwayenv_b200 import _native as N
    from highwayenv_b200.config import default_config

    for env_id, cls in [("merge-generic-v0", "BatchedMergeGenericEnv"),
                        ("merge-generic-v1", "BatchedConnectedLaneMergeGenericEnv")]:
        assert hb.REGISTRY[env_id].endswith(":" + cls)
        assert default_config(env_id)["neighbour_vehicles_connected_lanes"] is env_id.endswith("v1")
    assert N.HWY_ABI_VERSION == 17
    assert N.HWY_SCENARIO_RACETRACK == 8  # no new scenario kind: merge-generic is HWY_SCENARIO_MERGE
