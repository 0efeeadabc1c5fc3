"""roundabout-generic-v0 / v1 without a GPU: the lane tables against the reference's pinned to_config, the default
configs, every reset of the fixtures (oracle/gen_roundabout_generic.py) re-derived with numpy from the stream words
before it, the HwyRoundaboutGenericSpawn layout, registration and the configurations that raise before any launch."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = ["rg_default", "rg_v1_default", "rg_r5_crowded", "rg_one_lane_r40_grid", "rg_32_slots", "rg_dest_ttc"]


def load(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    g["config"] = json.loads(str(g.pop("config_json")))
    return g


def config_of(g):
    return {k: v for k, v in g["config"].items() if not k.startswith("_")}


def network_of(cfg):
    from highwayenv_b200.envs.roundabout_env import roundabout_generic_network

    return roundabout_generic_network(cfg["roundabout_radius"], cfg["roundabout_lanes"])


def records(g, i):
    """(stream words, record) of seed i's seeded reset and of each autoreset, in order."""
    out = [(g["reset_rng"][i], {k[6:]: g[k][i] for k in g if k.startswith("reset_")})]
    for j in range(g["autoreset_step"].shape[1]):
        if g["autoreset_step"][i, j] >= 0:
            out.append((g["autoreset_rng"][i, j], {k[10:]: g[k][i, j] for k in g if k.startswith("autoreset_")
                                                   and k != "autoreset_step"}))
    return out


@pytest.mark.parametrize("radius,lanes,n_lanes", [(20, 2, 32), (20, 1, 24), (5, 2, 32), (60, 1, 24)])
def test_network_matches_reference_to_config(radius, lanes, n_lanes):
    """Lane order, geometry, line types and speed limits, insertion order included, bit for bit."""
    from highwayenv_b200 import _native as N
    from highwayenv_b200.envs.roundabout_env import make_roundabout_generic_network, roundabout_generic_network
    from highwayenv_b200.road.network import NetworkTable

    with open(os.path.join(GOLDEN, f"pinned_to_config_roundabout_generic_r{radius}_l{lanes}.json")) as f:
        ref = json.load(f)
    net = make_roundabout_generic_network(radius, lanes)
    ours = json.loads(json.dumps(net.to_config()))
    assert list(ours) == list(ref)
    for f in ref:
        assert list(ours[f]) == list(ref[f])
        for t in ref[f]:
            assert ours[f][t] == ref[f][t], (f, t)
    assert len(net.lanes) == n_lanes == 8 * lanes + 16 <= N.HWY_NET_MAX_LANES
    back = NetworkTable.from_config(ref)
    for k, v in net.arrays.items():
        assert np.array_equal(back.arrays[k], v), k
    assert roundabout_generic_network(float(radius), lanes) is roundabout_generic_network(radius, lanes)


def test_no_ill_conditioned_lane_pairs():
    """No two lanes share a circle with overlapping angles, and no two straight lanes overlap on one line: the
    consecutive arcs of a ring only meet end to start and the rings lie 4 m apart."""
    for radius, lanes in [(20, 2), (20, 1), (5, 2), (40, 1), (30, 2), (60, 1)]:
        net = network_of({"roundabout_radius": radius, "roundabout_lanes": lanes})
        arcs = [L for L in net.lanes if L["type"] == 2]
        for a in range(len(arcs)):
            for b in range(a + 1, len(arcs)):
                A, B = arcs[a], arcs[b]
                if (A["cx"], A["cy"], A["radius"]) != (B["cx"], B["cy"], B["radius"]):
                    continue
                lo_a, hi_a = sorted((A["start_phase"], A["end_phase"]))
                lo_b, hi_b = sorted((B["start_phase"], B["end_phase"]))
                for turn in (-2 * np.pi, 0.0, 2 * np.pi):  # the phases of one circle are equal modulo 2 pi
                    assert min(hi_a, hi_b + turn) - max(lo_a, lo_b + turn) <= 1e-12, (radius, lanes, a, b)
        straight = [L for L in net.lanes if L["type"] == 0]
        for a in range(len(straight)):
            for b in range(a + 1, len(straight)):
                A, B = straight[a], straight[b]
                collinear = abs(A["dx"] * B["dy"] - A["dy"] * B["dx"]) < 1e-12 and \
                    abs((B["sx"] - A["sx"]) * A["dy"] - (B["sy"] - A["sy"]) * A["dx"]) < 1e-9
                if collinear:  # e.g. ("ser","ses") and ("nxs","nxr") on x = 2, on either side of the ring
                    sa = sorted(((A["sx"] - A["sx"]) * A["dx"] + (A["sy"] - A["sy"]) * A["dy"], A["length"]))
                    pb = [(B[p + "x"] - A["sx"]) * A["dx"] + (B[p + "y"] - A["sy"]) * A["dy"] for p in "se"]
                    assert min(sa[1], max(pb)) - max(sa[0], min(pb)) < 0, (radius, lanes, a, b)


@pytest.mark.parametrize("env_id,name", [("roundabout-generic-v0", "rg_default"),
                                         ("roundabout-generic-v1", "rg_v1_default")])
def test_default_config_matches_reference(env_id, name):
    from highwayenv_b200.config import default_config

    ref = config_of(load(name))
    ours = json.loads(json.dumps(default_config(env_id)))
    ref.pop("offscreen_rendering"), ours.pop("offscreen_rendering")
    assert ours == ref
    assert (ours["roundabout_radius"], ours["roundabout_lanes"], ours["vehicles_count"], ours["duration"]) == \
        (20, 2, 5, 17)


SPAWN_ROADS = [("we", "sx"), ("sx", "se"), ("ee", "nx"), ("nx", "ne"), ("eer", "ees"), ("ner", "nes"), ("wer", "wes")]


def rederive_reset(gen, net, cfg, routes, route_lens):
    """RoundaboutGenericEnv._make_vehicles (roundabout_env.py:664-751) with numpy on `gen`: per placed vehicle
    (x, y, heading, speed, delta, closest lane, route, route_len)."""
    ego = net.index[("ser", "ses", 0)]
    lon = net.lanes[ego]["length"] - 2.5
    x, y = net.position(ego, lon, 0.0)
    placed = [(float(x), float(y), float(net.heading_at(ego, lon)), 8.0, 4.0, 4)]
    fd = cfg["incoming_vehicle_destination"]
    for _ in range(int(cfg["vehicles_count"])):
        for _ in range(10):
            f, t = SPAWN_ROADS[gen.integers(0, len(SPAWN_ROADS))]
            lane = net.index[(f, t, int(gen.integers(0, len(net._graph[f][t]))))]
            lon = gen.uniform(5.0, max(5.0, net.lanes[lane]["length"] - 5.0))
            p = np.array(net.position(lane, lon, 0.0), dtype=np.float64)
            if any(np.linalg.norm(p - np.array(q[:2])) < 7.0 for q in placed):
                continue
            speed = 14.0 + gen.normal() * 2.0
            dest = [0, 1, 2, 3][min(fd, 3)] if fd is not None else int(gen.integers(0, 4))
            delta = gen.uniform(3.5, 4.5)
            placed.append((float(p[0]), float(p[1]), float(net.heading_at(lane, lon)), speed, delta, dest))
            break
    xs, ys, hs = (np.array([v[k] for v in placed]) for k in range(3))
    lanes = net.closest_lane(xs, ys, hs)
    dests = [v[5] for v in placed]
    return dict(x=xs, y=ys, heading=hs, speed=np.array([v[3] for v in placed]), delta=np.array([v[4] for v in placed]),
                lane=lanes, route=np.stack([routes[lanes[k], d] for k, d in enumerate(dests)]),
                route_len=np.array([route_lens[lanes[k], d] for k, d in enumerate(dests)]))


@pytest.mark.parametrize("name", CASES)
def test_reset_draws_match_stream_words(name):
    """Every reset of the fixture re-derived from the words before it (the steps draw nothing): stream words,
    population, positions, headings, speeds, DELTA, lanes and routes all exact."""
    from highwayenv_b200.envs.common.vector_env import pcg64_words, set_pcg64_words
    from highwayenv_b200.envs.roundabout_env import GENERIC_DESTINATIONS

    g = load(name)
    cfg = config_of(g)
    net = network_of(cfg)
    routes, route_lens = net.route_table(GENERIC_DESTINATIONS + ["nxs"])
    full = 1 + int(cfg["vehicles_count"])
    n_resets, counts = 0, []
    for i, seed in enumerate(g["seeds"]):
        gen = np.random.Generator(np.random.PCG64(np.random.SeedSequence(int(seed))))
        for words, rec in records(g, i):
            r = rederive_reset(gen, net, cfg, routes, route_lens)
            assert np.array_equal(pcg64_words([gen])[:, 0], words)
            n = len(r["x"])
            assert n == int(rec["count"]), (name, i)
            for k in ("x", "y", "heading", "speed"):
                assert np.array_equal(rec[k][:n], r[k]), (name, i, k)
            assert np.array_equal(rec["delta"][1:n], r["delta"][1:])
            assert np.array_equal(rec["lane"][:n], r["lane"]) and np.array_equal(rec["target_lane"][:n], r["lane"])
            assert np.array_equal(rec["route_len"][:n], r["route_len"])
            for v in range(n):
                assert np.array_equal(rec["route"][v, :r["route_len"][v]], r["route"][v, :r["route_len"][v]])
            counts.append(n)
            n_resets += 1
            set_pcg64_words([gen], words[:, None])
    assert n_resets > len(g["seeds"])
    if name in ("rg_r5_crowded", "rg_32_slots"):  # the population varies: some resets skipped a vehicle
        assert min(counts) < full
    assert max(counts) == full


def test_short_arcs_draw_uniform_5_5():
    """On the radius-5 roundabout some spawn arcs are shorter than 10 m: uniform(5, max(5, length - 5)) still draws."""
    net = network_of({"roundabout_radius": 5, "roundabout_lanes": 2})
    lengths = [net.lanes[net.index[(f, t, k)]]["length"] for f, t in SPAWN_ROADS[:4] for k in range(2)]
    assert min(lengths) < 10.0


def test_struct_layout_matches_gcc():
    from highwayenv_b200 import _native as N

    T = N.HwyRoundaboutGenericSpawn
    names = [f for f, _ in T._fields_]
    assert C.sizeof(T) == 64 and T.route_table.offset == 48
    src = ('#include <stddef.h>\n#include <stdio.h>\n#include "hwyb200.h"\nint main(){'
           + 'printf("%zu\\n", sizeof(HwyRoundaboutGenericSpawn));'
           + "".join(f'printf("%zu\\n", offsetof(HwyRoundaboutGenericSpawn, {f}));' for f in names) + "return 0;}\n")
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    assert got == [C.sizeof(T)] + [getattr(T, f).offset for f in names]


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
    return env


@pytest.mark.parametrize("env_id", ["roundabout-generic-v0", "roundabout-generic-v1"])
@pytest.mark.parametrize("over,exc", [
    ({"roundabout_lanes": 0}, ValueError),
    ({"roundabout_lanes": -1}, ValueError),
    ({"roundabout_lanes": 3}, NotImplementedError),
    ({"roundabout_lanes": 4}, NotImplementedError),
    ({"roundabout_radius": 0}, ValueError),
    ({"roundabout_radius": -5}, ValueError),
    ({"vehicles_count": 32}, NotImplementedError),
    ({"vehicles_count": 50}, NotImplementedError),
    ({"incoming_vehicle_destination": -5}, IndexError),
    ({"action": {"type": "ContinuousAction"}}, NotImplementedError),
    ({"action": {"type": "Nothing"}}, ValueError),
])
def test_rejections(env_id, over, exc):
    """Raised by define_spaces, which __init__ and reset(options={"config": ...}) run before any allocation or
    launch."""
    with pytest.raises(exc):
        _host_env(env_id, over)


def test_host_reset_mode_raises():
    with pytest.raises(NotImplementedError):
        _host_env("roundabout-generic-v0", reset_mode="host")


@pytest.mark.parametrize("over,slots,V,lanes", [
    ({}, 8, 6, 32), ({"vehicles_count": 7}, 8, 8, 32), ({"vehicles_count": 8}, 32, 9, 32),
    ({"vehicles_count": 31, "roundabout_lanes": 1}, 32, 32, 24), ({"vehicles_count": -3}, 8, 1, 32),
    ({"vehicles_count": 0, "roundabout_radius": 5.5}, 8, 1, 32),
])
def test_slots_and_parameters(over, slots, V, lanes):
    env = _host_env("roundabout-generic-v0", over)
    assert (env.SLOTS, env.N_VEHICLES, env._params.n_vehicles, len(env.net.lanes)) == (slots, V, V, lanes)
    assert env._params.reward_type == 0 and env._params.connected_lanes == 0
    assert (env._params.obs_y_lo, env._params.obs_y_hi) == (-100.0, 100.0)  # the roundabout's features_range
    assert _host_env("roundabout-generic-v1", over)._params.connected_lanes == 1


def test_reconfigure_rebuilds_the_lane_table():
    """A new (radius, lanes) rebuilds the table and its device copy; the same pair keeps both."""
    from highwayenv_b200.envs.roundabout_env import roundabout_generic_network

    env = _host_env("roundabout-generic-v0")
    old, old_dev = env.net, env._graph_dev
    env.configure({"vehicles_count": 12})
    env.define_spaces()
    assert env.net is old and env._graph_dev is old_dev and env.SLOTS == 32
    env.configure({"roundabout_radius": 40, "roundabout_lanes": 1})
    env.define_spaces()
    assert env.net is roundabout_generic_network(40, 1) and env.net is not old and env._graph_dev is not old_dev
    assert bytes(env._graph_dev.numpy()) == bytes(env.net.to_struct()) and len(env.net.lanes) == 24


def test_planners_raise():
    from highwayenv_b200 import planning
    from highwayenv_b200.envs.roundabout_env import BatchedRoundaboutGenericEnv

    env = BatchedRoundaboutGenericEnv.__new__(BatchedRoundaboutGenericEnv)
    env.n_agents, env.multi_agent = 1, False
    with pytest.raises(NotImplementedError):
        env.to_finite_mdp()
    for env_id in ("roundabout-generic-v0", "roundabout-generic-v1"):
        assert env_id not in planning.OPD_ENV_IDS and env_id not in planning.MCTS_ENV_IDS
    for policy in (planning.OpdPolicy, planning.MctsPolicy):
        with pytest.raises(NotImplementedError):
            policy(env)


def test_registered():
    import highwayenv_b200 as hb
    from highwayenv_b200 import _native as N
    from highwayenv_b200.config import default_config

    for env_id, cls in [("roundabout-generic-v0", "BatchedRoundaboutGenericEnv"),
                        ("roundabout-generic-v1", "BatchedConnectedLaneRoundaboutGenericEnv")]:
        assert hb.REGISTRY[env_id].endswith(":" + cls)
        assert default_config(env_id)["neighbour_vehicles_connected_lanes"] is env_id.endswith("v1")
    assert N.HWY_ABI_VERSION == 17
    # every network scenario resets and steps through the network entry points with its HwyNetScenario
    hdr = open(os.path.join(ROOT, "include", "hwyb200.h")).read()
    for sym in ("hwy_network_reset", "hwy_network_step", "hwy_network_substeps"):
        assert sym in N.EXPORTS and sym + "(" in hdr
    for sym in ("hwy_roundabout_generic_reset", "hwy_roundabout_reset", "hwy_merge_reset", "hwy_two_way_reset",
                "hwy_u_turn_reset", "hwy_exit_reset", "hwy_intersection_reset", "hwy_intersection_step"):
        assert sym not in N.EXPORTS and sym not in hdr, sym
