"""CPU-only checks: the C-ABI library loads and exports every symbol include/hwyb200.h declares,
the host mirror's config / plugin logic, loud failure without a GPU, and the world_size-2 gloo
path of the env-range sharding."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from highwayenv_b200 import _native as N

    lib = N.load()
    hdr = open(os.path.join(ROOT, "include", "hwyb200.h")).read()
    declared = set(re.findall(r"\b(hwy_[a-z_0-9]+)\s*\(", hdr))
    assert {"hwy_highway_step", "hwy_highway_reset", "hwy_highway_observe", "hwy_highway_substeps",
            "hwy_highway_slot_stride", "hwy_abi_version", "hwy_last_error", "hwy_launch_count",
            "hwy_debug_math", "hwy_debug_pcg64", "hwy_debug_network_lanes",
            "hwy_debug_network_closest_lanes"} <= declared
    assert declared <= set(N.EXPORTS) | {"hwy_debug_phase_cycles"}
    for sym in declared:
        assert getattr(lib, sym) is not None, sym
    assert lib.hwy_abi_version() == N.HWY_ABI_VERSION
    assert lib.hwy_highway_slot_stride(51) == 52 and lib.hwy_highway_slot_stride(20) == 20


def test_network_entries_refuse_bad_scenarios_without_gpu():
    """hwy_network_reset / _step / _substeps refuse an unknown scenario kind, a reset without a scenario or without
    the rng words, and a mask on the racetrack substeps (which run every env) before any device call."""
    import ctypes as C

    from highwayenv_b200 import _native as N

    lib = N.load()
    p, st, sc = N.HwyNetParams(), N.HwyNetState(), N.HwyNetScenario()
    buf = (C.c_double * 64)()
    ptr = C.addressof(buf)
    P, S = C.byref(p), C.byref(st)
    sc.kind = N.HWY_SCENARIO_RACETRACK + 1
    for rc in (lib.hwy_network_reset(P, ptr, C.byref(sc), S, None, None, None, None, None),
               lib.hwy_network_step(P, ptr, C.byref(sc), S, ptr, ptr, ptr, ptr, ptr, None, None, None, None, None),
               lib.hwy_network_substeps(P, ptr, C.byref(sc), S, None, 1, None)):
        assert rc != 0 and b"unknown scenario kind" in lib.hwy_last_error()
    assert lib.hwy_network_reset(P, ptr, None, S, None, None, None, None, None) != 0
    assert b"null scenario" in lib.hwy_last_error()
    sc.kind = N.HWY_SCENARIO_ROUNDABOUT
    assert lib.hwy_network_reset(P, ptr, C.byref(sc), S, None, None, None, None, None) != 0  # st.rng is NULL
    assert b"null rng" in lib.hwy_last_error()
    sc.kind = N.HWY_SCENARIO_RACETRACK
    assert lib.hwy_network_substeps(P, ptr, C.byref(sc), S, ptr, 1, None) != 0
    assert b"mask must be NULL" in lib.hwy_last_error()


def test_struct_layout_matches_header():
    """ctypes mirrors must have the C sizes (gcc as the referee)."""
    import ctypes as C
    import tempfile

    from highwayenv_b200 import _native as N

    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "hwyb200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\\n", '
           'sizeof(HwyHighwayParams), sizeof(HwyHighwayState), sizeof(HwyStraightLane), sizeof(HwyNetLane), '
           'sizeof(HwyNetGraph), sizeof(HwyNetParams), sizeof(HwyNetState), sizeof(HwyIntersectionSpawn), '
           'sizeof(HwyRoundaboutSpawn), sizeof(HwyObsView), sizeof(HwyGridParams), sizeof(HwyTtcParams), '
           'sizeof(HwyLidarParams), sizeof(HwyExitSpawn), sizeof(HwyNetScenario), offsetof(HwyNetScenario, u));'
           'return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", exe])
        sizes = [int(x) for x in subprocess.check_output([exe]).split()]
    assert sizes == [C.sizeof(t) for t in (N.HwyHighwayParams, N.HwyHighwayState, N.HwyStraightLane, N.HwyNetLane,
                                           N.HwyNetGraph, N.HwyNetParams, N.HwyNetState, N.HwyIntersectionSpawn,
                                           N.HwyRoundaboutSpawn, N.HwyObsView, N.HwyGridParams, N.HwyTtcParams,
                                           N.HwyLidarParams, N.HwyExitSpawn, N.HwyNetScenario)] + [N.HwyNetScenario.u.offset]


def test_abi_validation_without_gpu():
    import ctypes as C

    from highwayenv_b200 import _native as N

    lib = N.load()
    assert lib.hwy_highway_step(None, None, None, None, None, None, None, None, None, None, None, 0, None, None) != 0
    assert b"null" in lib.hwy_last_error()
    p, s = N.HwyHighwayParams(), N.HwyHighwayState()
    p.n_vehicles = 500
    assert lib.hwy_highway_observe(C.byref(p), C.byref(s), None, None) != 0
    assert b"n_vehicles" in lib.hwy_last_error()


def test_test_entries_validate_their_arguments():
    """hwy_debug_math / hwy_debug_pcg64 / hwy_debug_network_lanes / hwy_debug_network_closest_lanes refuse bad ops,
    indices, pointers and lane tables before touching the device."""
    import ctypes as C

    from highwayenv_b200 import _native as N

    lib = N.load()
    # host buffers for the pointer arguments a check does not concern: each call fails validation before any launch,
    # and a regression in that order would hand a kernel a host pointer (a launch error), never a made-up address
    buf = (C.c_double * 64)()
    p = C.addressof(buf)
    assert lib.hwy_debug_math(len(N.MATH_OPS), p, p, 4, None) != 0 and b"op" in lib.hwy_last_error()
    assert lib.hwy_debug_math(-1, p, p, 4, None) != 0 and b"op" in lib.hwy_last_error()
    assert lib.hwy_debug_math(0, p, None, 4, None) != 0 and b"null" in lib.hwy_last_error()
    assert lib.hwy_debug_math(0, None, p, 4, None) != 0 and b"null" in lib.hwy_last_error()
    assert lib.hwy_debug_math(0, p, p, -1, None) != 0 and b"n < 0" in lib.hwy_last_error()
    assert lib.hwy_debug_math(0, None, None, 0, None) != 0
    pcg = lib.hwy_debug_pcg64
    assert pcg(len(N.PCG_OPS), 0, 0.0, 0.0, 1, p, p, p, 4, None) != 0 and b"op" in lib.hwy_last_error()
    assert pcg(N.PCG_OPS["pcg_at"], 4 * N.HWY_MAX_VEHICLES + 8, 0.0, 0.0, 0, p, p, None, 4, None) != 0
    assert b"jump table" in lib.hwy_last_error()
    assert pcg(N.PCG_OPS["pcg_at"], -1, 0.0, 0.0, 0, p, p, None, 4, None) != 0
    assert pcg(N.PCG_OPS["choice"], 0, 0.0, 0.0, 1, p, p, p, 4, None) != 0 and b"arg_i" in lib.hwy_last_error()
    assert pcg(N.PCG_OPS["next64"], 0, 0.0, 0.0, -1, p, p, p, 4, None) != 0 and b"count" in lib.hwy_last_error()
    assert pcg(N.PCG_OPS["next64"], 0, 0.0, 0.0, 1, None, p, p, 4, None) != 0 and b"null" in lib.hwy_last_error()
    assert pcg(N.PCG_OPS["next64"], 0, 0.0, 0.0, 1, p, None, p, 4, None) != 0 and b"null" in lib.hwy_last_error()
    assert pcg(N.PCG_OPS["normal"], 0, 0.0, 0.0, 1, p, p, None, 4, None) != 0 and b"null" in lib.hwy_last_error()
    assert pcg(N.PCG_OPS["next64"], 0, 0.0, 0.0, 1, p, p, p, -2, None) != 0 and b"n < 0" in lib.hwy_last_error()
    lanes = lib.hwy_debug_network_lanes
    g = N.HwyNetGraph()
    g.n_lanes, g.n_nodes = 2, 2
    assert lanes(C.byref(g), len(N.LANE_OPS), p, p, 4, None) != 0 and b"op" in lib.hwy_last_error()
    assert lanes(C.byref(g), -1, p, p, 4, None) != 0 and b"op" in lib.hwy_last_error()
    assert lanes(C.byref(g), 0, p, None, 4, None) != 0 and b"null" in lib.hwy_last_error()
    assert lanes(C.byref(g), 0, None, p, 4, None) != 0 and b"null" in lib.hwy_last_error()
    assert lanes(None, 0, p, p, 4, None) != 0 and b"null" in lib.hwy_last_error()
    assert lanes(C.byref(g), 0, p, p, -1, None) != 0 and b"n < 0" in lib.hwy_last_error()
    for n_lanes in (0, N.HWY_NET_MAX_LANES + 1):
        g.n_lanes = n_lanes
        assert lanes(C.byref(g), 0, p, p, 4, None) != 0 and b"n_lanes" in lib.hwy_last_error()
    closest = lib.hwy_debug_network_closest_lanes
    assert closest(None, None, None, p, p, p, None) != 0 and b"null" in lib.hwy_last_error()
    np_, st = N.HwyNetParams(), N.HwyNetState()
    assert closest(C.byref(np_), p, C.byref(st), p, p, p, None) != 0 and b"stride" in lib.hwy_last_error()


def test_default_configs_match_reference_values():
    from highwayenv_b200.config import default_config

    fast, hw = default_config("highway-fast-v0"), default_config("highway-v0")
    # envs/highway_env.py:25-53,162-175 over envs/common/abstract.py:102-125
    assert (fast["simulation_frequency"], fast["lanes_count"], fast["vehicles_count"], fast["duration"],
            fast["ego_spacing"]) == (5, 3, 20, 30, 1.5)
    assert (hw["simulation_frequency"], hw["lanes_count"], hw["vehicles_count"], hw["duration"],
            hw["ego_spacing"]) == (15, 4, 50, 40, 2)
    for c in (fast, hw):
        assert c["policy_frequency"] == 1 and c["collision_reward"] == -1
        assert c["reward_speed_range"] == [20, 30] and c["observation"] == {"type": "Kinematics"}
        assert c["other_vehicles_type"] == "highway_env.vehicle.behavior.IDMVehicle"


def test_golden_config_equals_our_defaults():
    """The defaults restated in config.py equal the reference env's merged config dict."""
    from highwayenv_b200.config import default_config
    from parity_utils import load_golden

    for name, env_id, over in (("highway_fast_v20", "highway-fast-v0", {}),
                               ("highway_fast_v50", "highway-fast-v0", {"vehicles_count": 50}),
                               ("highway_v50", "highway-v0", {})):
        ref = dict(load_golden(name)["config"])
        ref.pop("_env_id"), ref.pop("_others_check_collisions")
        ours = default_config(env_id)
        ours.update(over)
        ours["offscreen_rendering"] = ref["offscreen_rendering"]  # set by configure() from render_mode
        assert ours == ref, name


def test_update_config_validation_rule():
    from highwayenv_b200.config import update_config

    cfg = {"observation": {"type": "Kinematics", "vehicles_count": 5}, "x": 1}
    with pytest.raises(AssertionError):  # nested mapping must redefine every key (utils.py:453-464)
        update_config(cfg, {"observation": {"type": "Kinematics"}})
    update_config(cfg, {"observation": {"type": "Kinematics", "vehicles_count": 7}, "x": 2})
    assert cfg["observation"]["vehicles_count"] == 7 and cfg["x"] == 2


def test_plugin_factories():
    from highwayenv_b200.envs.common.action import action_factory
    from highwayenv_b200.envs.common.observation import observation_factory

    a = action_factory(None, {"type": "DiscreteMetaAction"})
    assert a.space().n == 5 and a.actions[3] == "FASTER"
    c = action_factory(None, {"type": "ContinuousAction"})
    assert c.space().shape == (2,) and c.space().dtype == np.float32
    o = observation_factory(None, {"type": "Kinematics", "vehicles_count": 7})
    assert o.space().shape == (7, 5) and o.space().dtype == np.float32
    with pytest.raises(ValueError, match="Unknown action type"):
        action_factory(None, {"type": "Nope"})
    with pytest.raises(ValueError, match="Unknown observation type"):
        observation_factory(None, {"type": "Nope"})
    with pytest.raises(NotImplementedError):
        observation_factory(None, {"type": "GrayscaleObservation"})  # needs the renderer
    # one registry for every env family (reference observation.py:772-794): the spaces follow the reference's
    g = observation_factory(None, {"type": "OccupancyGrid", "grid_size": [[-300, 300], [-10, 10]], "grid_step": [2, 2]})
    assert g.space().shape == (4, 300, 10) and g.standalone  # the reference's own test (tests/envs/test_observations.py:27-42)
    assert observation_factory(None, {"type": "OccupancyGrid"}).is_default
    assert observation_factory(None, {"type": "OccupancyGrid", "as_image": True}).space().dtype == np.uint8
    assert observation_factory(None, {"type": "TimeToCollision", "horizon": 7}).space().shape == (3, 3, 7)
    li = observation_factory(None, {"type": "LidarObservation", "cells": 24, "normalize": False, "maximum_range": 80})
    assert li.space().shape == (24, 2) and float(li.space().high.max()) == 80.0
    with pytest.raises(NotImplementedError):
        observation_factory(None, {"type": "OccupancyGrid", "absolute": True})  # as the reference's observe()
    # DiscreteAction (action.py:165-196): 3 x 3 grid over [-1, 1]^2 in itertools.product order, float32
    d = action_factory(None, {"type": "DiscreteAction"})
    assert d.space().n == 9 and d.table.dtype == np.float32
    assert d.table.tolist() == [[x, y] for x in (-1.0, 0.0, 1.0) for y in (-1.0, 0.0, 1.0)]
    assert action_factory(None, {"type": "DiscreteAction", "actions_per_axis": 5}).space().n == 25
    # Kinematics feature lists / ranges end up in the kernel parameters
    from highwayenv_b200 import _native as N
    k = observation_factory(None, {"type": "Kinematics", "features": ["presence", "x", "cos_h", "lat_off"],
                                   "features_range": {"x": [-10, 10]}})
    p = N.HwyHighwayParams()
    p.lanes_count = 4
    k.fill_params(p)
    assert k.space().shape == (5, 4) and p.obs_n_features == 4
    assert list(p.obs_feature[:4]) == [0, 1, 6, 11] and list(p.obs_feature_ranged[:4]) == [0, 1, 0, 0]
    assert (p.obs_feature_lo[1], p.obs_feature_hi[1]) == (-10.0, 10.0)
    with pytest.raises(KeyError):
        observation_factory(None, {"type": "Kinematics", "features": ["presence", "nope"]})


def test_network_tables_match_the_reference_dump():
    """road/network.py + the scenario builders against the lane tables dumped from the reference's
    RoadNetwork (graph enumeration order, lane constructor arithmetic, successor lists, priorities)."""
    from highwayenv_b200.envs.intersection_env import make_intersection_network
    from highwayenv_b200.envs.roundabout_env import make_roundabout_network
    from parity_utils import load_golden

    from highwayenv_b200.envs.merge_env import make_merge_network
    from highwayenv_b200.envs.two_way_env import make_two_way_network
    from highwayenv_b200.envs.u_turn_env import make_u_turn_network

    for name, build in (("intersection_kin", make_intersection_network), ("roundabout_kin", make_roundabout_network),
                        ("merge_kin", make_merge_network), ("two_way_ttc", make_two_way_network),
                        ("u_turn_ttc", make_u_turn_network)):
        g, ex = load_golden(name), build().export_arrays()
        assert list(ex["net_node_names"]) == list(g["net_node_names"]), name
        for key, val in ex.items():
            if key != "net_node_names" and key in g:
                assert np.array_equal(val, g[key]), (name, key)
    net = make_intersection_network()
    # plan_route_to (controller.py:71-87): from the south access road to the west exit = right turn
    route = net.plan_route(("o0", "ir0", 0), "o1")
    assert [r[:2] for r in route] == [("o0", "ir0"), ("ir0", "il1"), ("il1", "o1")]
    assert sum(l["exit_lane"] for l in net.lanes) == 4 and sorted({l["priority"] for l in net.lanes}) == [0, 1, 2, 3]


def test_network_env_defaults_match_reference_config():
    """intersection-v0/v2, roundabout-v0/v1 (the v1/v2 ids = ConnectedLaneNeighboursMixin defaults)"""
    import highwayenv_b200 as hb
    from highwayenv_b200.config import default_config
    from parity_utils import load_golden

    for name in ("intersection_kin", "intersection_v2_kin", "roundabout_kin", "roundabout_v1_kin",
                 "intersection_multi_agent", "merge_kin", "merge_v1_kin", "two_way_ttc", "u_turn_ttc", "u_turn_v1_ttc"):
        ref = {k: v for k, v in load_golden(name)["config"].items() if not k.startswith("_") or k == "_env_id"}
        env_id = ref.pop("_env_id")
        assert env_id in hb.REGISTRY
        ours = default_config(env_id)
        ours["offscreen_rendering"] = ref["offscreen_rendering"]
        assert ours == ref, name
    assert default_config("roundabout-v1")["neighbour_vehicles_connected_lanes"] is True


def test_no_silent_cpu_fallback():
    import torch

    import highwayenv_b200 as hb

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        hb.make("highway-fast-v0", num_envs=2)
    with pytest.raises(KeyError):
        hb.make("parking-v0")


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "highwayenv_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dp, f)).read()
                assert "hwy_oracle" not in text and "ref_harness" not in text, f


def test_env_range_and_split():
    from highwayenv_b200.parallel import env_range, split_envs

    assert env_range(0, 8, 8192) == (0, 8192) and env_range(7, 8, 8192) == (57344, 65536)
    assert split_envs(10, 4) == (3, 3, 2, 2) and sum(split_envs(65536, 8)) == 65536
    with pytest.raises(ValueError):
        env_range(8, 8, 1)


_GLOO_WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from highwayenv_b200.parallel import all_gather_batch, env_range
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:" + sys.argv[2], rank=int(sys.argv[3]), world_size=2)
rank = dist.get_rank()
E = 3
lo, hi = env_range(rank, 2, E)
local = (torch.arange(lo, hi, dtype=torch.float32).view(E, 1, 1) * torch.ones(E, 5, 5))
full = all_gather_batch(local)
assert full.shape == (6, 5, 5)
assert torch.equal(full[:, 0, 0], torch.arange(6, dtype=torch.float32)), full[:, 0, 0]
# value = all units / max-over-ranks time, as bench.py computes it
t = torch.tensor([1.0 + rank], dtype=torch.float64)
dist.all_reduce(t, op=dist.ReduceOp.MAX)
assert t.item() == 2.0
dist.barrier(); dist.destroy_process_group()
print("ok", rank)
'''


def test_gloo_world_size_2_gather(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_GLOO_WORKER)
    port = str(29600 + os.getpid() % 300)
    procs = [subprocess.Popen([sys.executable, str(script), ROOT, port, str(r)], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=120)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    assert "ok 0" in outs[0] and "ok 1" in outs[1]


def test_available_actions_mask_matches_reference_rule():
    """DiscreteMetaAction.get_available_actions (action.py:262-299) in tensor form, on CPU tensors"""
    import torch

    from highwayenv_b200.envs.highway_env import available_actions_mask

    table = torch.tensor([[0.0, 4.0 * l, 1.0, 0.0, -0.0, 1.0, 10000.0, 4.0] for l in range(3)], dtype=torch.float64)
    x = torch.tensor([100.0, 100.0, 100.0, -1.0, 10004.9, 10005.0], dtype=torch.float64)
    y = torch.tensor([0.0, 4.0, 8.0, 4.0, 4.0, 4.0], dtype=torch.float64)
    lane = torch.tensor([0, 1, 2, 1, 1, 1])
    si = torch.tensor([0, 1, 2, 1, 1, 1])
    m = available_actions_mask(x, y, lane, si, table, 3).numpy()
    # columns: LANE_LEFT, IDLE, LANE_RIGHT, FASTER, SLOWER
    assert m[0].tolist() == [False, True, True, True, False]   # leftmost lane, lowest speed
    assert m[1].tolist() == [True, True, True, True, True]
    assert m[2].tolist() == [True, True, False, False, True]   # rightmost lane, highest speed
    assert m[3].tolist() == [False, True, False, True, True]   # before the lane start: 0 <= longitudinal fails
    assert m[4].tolist() == [True, True, True, True, True]     # longitudinal < length + VEHICLE_LENGTH
    assert m[5].tolist() == [False, True, False, True, True]


def test_free_running_coverage_of_the_highway_fixtures():
    """The free-running GPU tests compare every well-conditioned (seed, step) of a golden rollout and assert that exact
    count (`parity_utils.comparable_steps`); this pins how much of each rollout that is — at least 95 % — so that a
    fixture regenerated with mostly ill-conditioned states cannot hollow the tests out."""
    from parity_utils import comparable_steps, load_golden

    for name in ("highway_fast_v20", "highway_fast_v50", "highway_v50", "highway_v100_continuous",
                 "highway_discrete_action", "highway_fast_features", "highway_fast_features_range"):
        g = load_golden(name)
        S, T = g["actions"].shape[:2]
        assert comparable_steps(g) >= 0.95 * S * T, (name, comparable_steps(g), S * T)


def test_gymnasium_registration_hook_registers_every_id(monkeypatch):
    """`highwayenv_b200._register_with_gymnasium` (B1 of the boundary): with a gymnasium on the path — here the stub the
    oracle harness runs the reference under — every reference id appears as `hwyb200/<id>` with the single-env facade as
    `entry_point` (gymnasium.make) and the batched class as `vector_entry_point` (gymnasium.make_vec), and every entry
    point resolves to a class of this package."""
    import importlib
    import sys

    import highwayenv_b200 as hb

    shim = os.path.join(ROOT, "oracle", "shim")
    monkeypatch.syspath_prepend(shim)
    for name in [m for m in sys.modules if m == "gymnasium" or m.startswith("gymnasium.")]:
        monkeypatch.delitem(sys.modules, name)
    hb._register_with_gymnasium()
    from gymnasium.envs.registration import registry

    for env_id, entry in hb.REGISTRY.items():
        spec = registry["hwyb200/" + env_id]
        assert spec["entry_point"] == "highwayenv_b200.single:SingleEnv" and spec["kwargs"] == {"env_id": env_id}
        assert spec["vector_entry_point"] == entry
        mod, cls = entry.split(":")
        assert isinstance(getattr(importlib.import_module(mod), cls), type)
    assert len([k for k in registry if k.startswith("hwyb200/")]) == len(hb.REGISTRY)
    for name in [m for m in sys.modules if m == "gymnasium" or m.startswith("gymnasium.")]:
        sys.modules.pop(name, None)  # leave no stub behind for the tests that follow


def test_pcg64_words_round_trip():
    """The generator <-> device-word conversion against numpy's bit_generator.state, with and without a buffered
    32-bit half."""
    from highwayenv_b200.envs.common.vector_env import pcg64_words, set_pcg64_words

    gens = [np.random.Generator(np.random.PCG64(np.random.SeedSequence(s))) for s in (0, 1, 2**63 + 5, 12345)]
    gens[1].integers(0, 7, dtype=np.uint32)  # one 32-bit draw leaves the other half buffered
    gens[2].normal(size=3)
    gens[3].integers(0, 7, size=2, dtype=np.uint32)  # two: the buffer is used up again
    states = [g.bit_generator.state for g in gens]
    assert [st["has_uint32"] for st in states] == [0, 1, 0, 0]
    words = pcg64_words(gens)
    assert words.shape == (5, 4) and words.dtype == np.uint64
    for i, st in enumerate(states):
        w = [int(x) for x in words[:, i]]
        assert (w[0] << 64) | w[1] == st["state"]["state"] and (w[2] << 64) | w[3] == st["state"]["inc"]
        assert w[4] == (st["has_uint32"] << 32) | st["uinteger"]
    fresh = [np.random.Generator(np.random.PCG64(9)) for _ in gens]
    set_pcg64_words(fresh, words)
    for g, h, st in zip(gens, fresh, states):
        assert h.bit_generator.state == st
        assert g.integers(0, 1 << 30, size=5, dtype=np.uint32).tolist() == h.integers(0, 1 << 30, size=5, dtype=np.uint32).tolist()
    assert np.array_equal(pcg64_words(fresh), pcg64_words(gens))


def test_meta_word_pack_round_trip():
    """pack_meta / unpack_meta over every flag combination, lane, target lane and kind."""
    import itertools

    from highwayenv_b200 import _native as N

    flags = tuple(N.META_FLAG_BITS)
    combos = np.array(list(itertools.product([False, True], repeat=len(flags))))
    m = len(combos)
    fields = {"lane": np.arange(m) % 32, "target_lane": (np.arange(m) * 7) % 32, "kind": np.arange(m) % 4}
    fields.update({f: combos[:, k] for k, f in enumerate(flags)})
    meta = N.pack_meta(fields, flags)
    assert meta.dtype == np.int32 and np.all(meta & N.META_PRESENT)
    out = N.unpack_meta(meta, flags)
    for k, v in fields.items():
        assert np.array_equal(out[k], v), k
    bits = [N.META_FLAG_BITS[f] for f in flags]
    assert len(set(bits)) == len(bits) and not any(b & 0xFFFF or b & (3 << N.META_KIND_SHIFT) for b in bits)
    assert not np.any(N.pack_meta(fields, ()) & sum(bits))  # only the named flags are packed


def test_speed_to_index_matches_the_reference_formula():
    """MDPVehicle.speed_to_index at the clip edges and at ties (np.round rounds half to even)."""
    from highwayenv_b200.envs.common.action import speed_to_index

    def reference(ts, v):
        return int(np.clip(np.round((v - ts[0]) / (ts[-1] - ts[0]) * (ts.size - 1)), 0, ts.size - 1))

    ts = np.linspace(20, 30, 3)
    for v, want in ((-5.0, 0), (20.0, 0), (22.5, 0), (22.500001, 1), (25.0, 1), (27.5, 2), (30.0, 2), (99.0, 2)):
        assert speed_to_index(ts, v) == want == reference(ts, v), v
    for ts in (np.linspace(20, 30, 3), np.array([0.0, 10.0]), np.linspace(5, 6, 8), np.array([8.0, 16.0, 24.0, 32.0])):
        for v in np.concatenate([ts, (ts[1:] + ts[:-1]) / 2, [ts[0] - 1, ts[-1] + 1, 8.0, 10.0, 16.0, 25.0, 30.0]]):
            assert speed_to_index(ts, v) == reference(ts, v), (ts, v)
