"""The reference's own known-answer tests (SURVEY.md section 8c; scenarios in kat_scenarios.py) run on the CUDA path
through the C ABI: the device `neighbour_vehicles` / `rotated_rectangles_intersect` via the library's test entries,
vehicle dynamics and control through `hwy_highway_step`."""
import ctypes as C

import numpy as np
import pytest
import torch

import kat_scenarios as K
from test_reference_kats import CONT, META, _cont, _highway, _place

pytestmark = pytest.mark.gpu


def test_rotated_rectangles_intersect():
    """tests/test_utils.py:19-27"""
    from highwayenv_b200 import _native as N

    lib = N.load()
    rects = np.array([[c1[0], c1[1], l1, w1, a1, c2[0], c2[1], l2, w2, a2]
                      for (c1, l1, w1, a1), (c2, l2, w2, a2), _ in K.RECTANGLES], dtype=np.float64)
    d = torch.from_numpy(rects).cuda()
    out = torch.zeros(len(rects), dtype=torch.int32, device="cuda")
    N.check(lib.hwy_debug_rotated_rectangles_intersect(d.data_ptr(), len(rects), out.data_ptr(), None))
    torch.cuda.synchronize()
    assert out.cpu().numpy().astype(bool).tolist() == [w for _, _, w in K.RECTANGLES]


@pytest.mark.parametrize("vp", [8, 32])
@pytest.mark.parametrize("case", K.NEIGHBOURS, ids=[c[0] for c in K.NEIGHBOURS])
def test_neighbour_vehicles(case, vp):
    """tests/road/test_neighbour_vehicles.py on both thread mappings of the network kernels"""
    from highwayenv_b200 import _native as N

    lib = N.load()
    net, x, y, h, lanes, query = K.build_neighbour_case(case)
    V, n, dev = len(x), 3, "cuda"  # three copies of the scene: the middle env is the one checked
    graph = torch.from_numpy(np.frombuffer(bytes(net.to_struct()), dtype=np.uint8).copy()).to(dev)
    z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=dev)  # noqa: E731
    pos, hs, tt, imp = (z(n, vp, 2, dtype=torch.float64) for _ in range(4))
    pos[:, :V, 0], pos[:, :V, 1] = torch.from_numpy(x).to(dev), torch.from_numpy(y).to(dev)
    hs[:, :V, 0], hs[:, :V, 1] = torch.from_numpy(h).to(dev), 10.0
    meta = z(n, vp, dtype=torch.int32)
    m = (lanes.astype(np.int64) << N.META_LANE_SHIFT) | (lanes.astype(np.int64) << N.META_TARGET_SHIFT) | N.META_PRESENT
    meta[:, :V] = torch.from_numpy(m.astype(np.int32)).to(dev)
    delta, route, route_len = z(n, vp, dtype=torch.float64), z(n, vp, N.HWY_NET_MAX_ROUTE, dtype=torch.int32), z(n, vp, dtype=torch.int32)
    speed_index, time_ = z(n, dtype=torch.int32), z(n, dtype=torch.float64)
    count, road_steps, rng = torch.full((n,), V, dtype=torch.int32, device=dev), z(n, dtype=torch.int32), z(5, n, dtype=torch.int64)
    st = N.HwyNetState()
    st.n_envs, st.vp = n, vp
    st.pos, st.hs, st.tt, st.imp = pos.data_ptr(), hs.data_ptr(), tt.data_ptr(), imp.data_ptr()
    st.delta, st.meta, st.route, st.route_len = delta.data_ptr(), meta.data_ptr(), route.data_ptr(), route_len.data_ptr()
    st.speed_index, st.time = speed_index.data_ptr(), time_.data_ptr()
    st.count, st.road_steps, st.rng = count.data_ptr(), road_steps.data_ptr(), rng.data_ptr()
    p = N.HwyNetParams()
    p.n_vehicles, p.simulation_frequency, p.policy_frequency, p.n_target_speeds = V, 15, 1, 3
    p.obs_vehicles_count, p.obs_features = 5, 5
    p.connected_lanes = int(case[3])
    q = z(n, vp, dtype=torch.int32)
    q[:, 0] = int(query)
    front, rear = z(n, vp, dtype=torch.int32), z(n, vp, dtype=torch.int32)
    N.check(lib.hwy_debug_network_neighbours(C.byref(p), graph.data_ptr(), C.byref(st), q.data_ptr(), front.data_ptr(),
                                             rear.data_ptr(), None))
    torch.cuda.synchronize()
    K.check_neighbour_result(case, int(front[1, 0]), int(rear[1, 0]))
    assert torch.equal(front[0], front[2]) and torch.equal(rear[0], rear[2])


# ---------------------------------------------------------------- vehicle dynamics / control through hwy_highway_step
def _env_from(ob, lanes, action, V=1, **over):
    """the same scene as the oracle-side KAT (state built there), loaded into the CUDA env"""
    import highwayenv_b200 as hb

    cfg = {"lanes_count": lanes, "vehicles_count": V - 1, "action": action, "duration": 1000}
    cfg.update(over)
    env = hb.make("highway-v0", num_envs=1, config=cfg, autoreset_mode="Disabled")
    env.reset(seed=0)
    env.load_state_dict({k: ob.a[k].copy() for k in ob.a})
    return env


def _sd(env):
    sd = env.state_dict()
    return {k: v[0] for k, v in sd.items() if k != "rng"}


def test_dynamics_step():
    """vehicle/test_dynamics.py:12-19, vehicle/test_control.py:11-18"""
    ob = _highway(1, CONT)
    _place(ob, 0, 0.0, 0.0, 20.0)
    env = _env_from(ob, 1, CONT)
    for _ in range(2):
        env.step(_cont(0, 0))
    s = _sd(env)
    assert s["x"][0] == pytest.approx(40) and s["y"][0] == pytest.approx(0)
    assert s["speed"][0] == pytest.approx(20) and s["heading"][0] == pytest.approx(0)


def test_dynamics_act():
    """vehicle/test_dynamics.py:22-33"""
    ob = _highway(1, CONT)
    _place(ob, 0, 0.0, 0.0, 20.0)
    env = _env_from(ob, 1, CONT)
    env.step(_cont(1, 0))
    assert _sd(env)["speed"][0] == pytest.approx(21)
    env.step(_cont(0, 0.5))
    s = _sd(env)
    assert s["speed"][0] == pytest.approx(21) and s["y"][0] > 0


def test_dynamics_brake():
    """vehicle/test_dynamics.py:36-41"""
    ob = _highway(1, CONT, policy_frequency=15)
    _place(ob, 0, 0.0, 0.0, 20.0)
    env = _env_from(ob, 1, CONT, policy_frequency=15)
    for _ in range(10 * K.FPS):
        v = float(env._hs[0, 0, 1])
        env.step(_cont(min(max(-1 * v, -5), 5), 0))
    assert _sd(env)["speed"][0] == pytest.approx(0, abs=0.01)


def test_dynamics_front_and_collision():
    """vehicle/test_dynamics.py:44-60: lane_distance_to(v2) = 10 seen through the un-normalised Kinematics row;
    two vehicles 4 m apart are both crashed after the collision sweep"""
    obs_cfg = {"type": "Kinematics", "normalize": False, "see_behind": True}
    ob = _highway(1, CONT, V=2, observation=obs_cfg)
    _place(ob, 0, 0.0, 0.0, 20.0)
    _place(ob, 1, 10.0, 0.0, 10.0)
    env = _env_from(ob, 1, CONT, V=2, observation=obs_cfg)
    o = env.observe().cpu().numpy()
    assert o[0, 1, 0] == 1 and o[0, 1, 1] == pytest.approx(10)
    ob2 = _highway(1, CONT, V=2)
    _place(ob2, 0, 0.0, 0.0, 10.0)
    _place(ob2, 1, 4.0, 0.0, 20.0)
    env2 = _env_from(ob2, 1, CONT, V=2)
    env2.step(_cont(0, 0))
    s = _sd(env2)
    assert s["crashed"][0] and s["crashed"][1]


def test_control_lane_change():
    """vehicle/test_control.py:21-38"""
    ob = _highway(2, META)
    _place(ob, 0, 0.0, 0.0, 20.0)
    ob.a["kind"][0, 0] = 1
    ob.a["speed_index"][0] = 0
    env = _env_from(ob, 2, META)
    env.step(np.array([2], dtype=np.int32))
    for _ in range(2):
        env.step(np.array([1], dtype=np.int32))
    s = _sd(env)
    assert s["speed"][0] == pytest.approx(20)
    assert s["y"][0] == pytest.approx(4.0, abs=1.0) and s["lane"][0] == 1


def test_control_speed():
    """vehicle/test_control.py:41-54"""
    ob = _highway(1, META)
    _place(ob, 0, 0.0, 0.0, 20.0)
    ob.a["kind"][0, 0] = 1
    ob.a["speed_index"][0] = 0
    env = _env_from(ob, 1, META)
    env.step(np.array([3], dtype=np.int32))
    env.step(np.array([1], dtype=np.int32))
    s = _sd(env)
    assert s["speed"][0] == pytest.approx(25, abs=0.5)
    assert s["y"][0] == pytest.approx(0) and s["lane"][0] == 0


def test_road_network_follow_road():
    """road/test_road.py:23-40 test_network on the device (hwy_network_substeps on the diamond network)"""
    from highwayenv_b200 import _native as N

    lib = N.load()
    net = K.diamond_network()
    assert int(net.closest_lane(np.array([5.0]), np.array([0.0]), np.array([0.0]))[0]) == net.index[("0", "1", 0)]
    n, vp, dev = 2, 8, "cuda"
    graph = torch.from_numpy(np.frombuffer(bytes(net.to_struct()), dtype=np.uint8).copy()).to(dev)
    z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=dev)  # noqa: E731
    pos, hs, tt, imp = (z(n, vp, 2, dtype=torch.float64) for _ in range(4))
    pos[:, 0, 0], tt[:, 0, 0] = 5.0, 2.0  # position [5, 0], speed 0, target_speed 2
    delta = torch.full((n, vp), 4.0, dtype=torch.float64, device=dev)
    meta = z(n, vp, dtype=torch.int32)
    meta[:, 0] = (N.KIND_MDP << N.META_KIND_SHIFT) | N.META_PRESENT | N.META_CHECK_COLLISIONS
    route, route_len = z(n, vp, N.HWY_NET_MAX_ROUTE, dtype=torch.int32), z(n, vp, dtype=torch.int32)
    speed_index, time_ = z(n, dtype=torch.int32), z(n, dtype=torch.float64)
    st = N.HwyNetState()
    st.n_envs, st.vp = n, vp
    st.pos, st.hs, st.tt, st.imp = pos.data_ptr(), hs.data_ptr(), tt.data_ptr(), imp.data_ptr()
    st.delta, st.meta, st.route, st.route_len = delta.data_ptr(), meta.data_ptr(), route.data_ptr(), route_len.data_ptr()
    st.speed_index, st.time = speed_index.data_ptr(), time_.data_ptr()
    p = N.HwyNetParams()
    p.n_vehicles, p.simulation_frequency, p.policy_frequency, p.n_target_speeds = 1, 15, 1, 3
    p.obs_vehicles_count, p.obs_features = 5, 5
    p.acc_max, p.comfort_acc_max, p.comfort_acc_min = 6.0, 3.0, -5.0
    p.distance_wanted, p.time_wanted, p.lane_change_delay = 10.0, 1.5, 1.0
    lane, changes = 0, 0
    for _ in range(20 * 15):
        N.check(lib.hwy_network_substeps(C.byref(p), graph.data_ptr(), None, C.byref(st), None, 1, None))
        tgt = (int(meta[1, 0]) >> N.META_TARGET_SHIFT) & 0xFF
        if tgt != lane:
            lane, changes = tgt, changes + 1
    assert changes >= 3
    assert torch.equal(meta[0], meta[1]) and torch.equal(pos[0], pos[1])


@pytest.mark.parametrize("env_id", ["highway-v0", "highway-fast-v0", "roundabout-v0", "roundabout-v1", "intersection-v0",
                                    "intersection-v2", "intersection-multi-agent-v0", "intersection-multi-agent-v1",
                                    "merge-v0", "merge-v1", "two-way-v0", "u-turn-v0"])
def test_env_step_until_done(env_id):
    """envs/test_gym.py:65-90 test_env_step: reset, random actions until the episode ends, observations stay in
    the observation space (shape, dtype, finite; [-1, 1] where the reference normalises and clips)."""
    import highwayenv_b200 as hb

    n = 6
    env = hb.make(env_id, num_envs=n, autoreset_mode="Disabled")
    obs, info = env.reset(seed=42)
    shape = (n,) + tuple(env.single_observation_space.shape)
    assert tuple(obs.shape) == shape and obs.dtype == torch.float32
    rng = np.random.default_rng(0)
    done = np.zeros(n, dtype=bool)
    # merge / two-way have no time limit (they end on a crash or at the end of the road): cap the loop
    horizon = env.config["duration"] * env.config["policy_frequency"]
    duration = int(horizon) if np.isfinite(horizon) else 60
    for t in range(duration + 1):
        sp = env.single_action_space
        hi = sp.n if hasattr(sp, "n") else int(sp.high.max()) + 1
        act = rng.integers(0, hi, size=(n,) + tuple(getattr(sp, "shape", ()) or ())).astype(np.int32)
        obs, reward, terminated, truncated, info = env.step(act)
        o = obs.cpu().numpy()
        assert o.shape == shape and np.isfinite(o).all() and np.abs(o).max() <= 1.0 + 1e-6
        te, tr = terminated.cpu().numpy(), truncated.cpu().numpy()
        done |= te.reshape(n, -1).any(axis=1) | tr
        if done.all():
            break
    if np.isfinite(horizon):
        assert done.all(), "every episode ends by the time limit"
    else:
        assert done.any()


def _single_lane_device(x, speed, kinds):
    """vehicles / objects on RoadNetwork.straight_road_network(1), as raw device state for hwy_network_substeps"""
    from highwayenv_b200 import _native as N

    net = K.single_lane_road()
    n, vp, dev, V = 2, 8, "cuda", len(x)
    graph = torch.from_numpy(np.frombuffer(bytes(net.to_struct()), dtype=np.uint8).copy()).to(dev)
    z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=dev)  # noqa: E731
    t = {k: z(n, vp, 2, dtype=torch.float64) for k in ("pos", "hs", "tt", "imp")}
    t["pos"][:, :V, 0] = torch.tensor(x, dtype=torch.float64, device=dev)
    t["hs"][:, :V, 1] = torch.tensor(speed, dtype=torch.float64, device=dev)
    t["tt"][:, :V, 0] = torch.tensor(speed, dtype=torch.float64, device=dev)
    t["delta"] = torch.full((n, vp), 4.0, dtype=torch.float64, device=dev)
    t["meta"] = z(n, vp, dtype=torch.int32)
    t["meta"][:, :V] = torch.tensor([(k << N.META_KIND_SHIFT) | N.META_PRESENT | N.META_CHECK_COLLISIONS for k in kinds],
                                    dtype=torch.int32, device=dev)
    t["route"], t["route_len"] = z(n, vp, N.HWY_NET_MAX_ROUTE, dtype=torch.int32), z(n, vp, dtype=torch.int32)
    t["speed_index"], t["time"] = z(n, dtype=torch.int32), z(n, dtype=torch.float64)
    st = N.HwyNetState()
    st.n_envs, st.vp = n, vp
    for k in ("pos", "hs", "tt", "imp", "delta", "meta", "route", "route_len", "speed_index", "time"):
        setattr(st, k, t[k].data_ptr())
    p = N.HwyNetParams()
    p.n_vehicles, p.simulation_frequency, p.policy_frequency, p.n_target_speeds = V, 15, 1, 3
    p.obs_vehicles_count, p.obs_features = 5, 5
    p.acc_max, p.comfort_acc_max, p.comfort_acc_min = 6.0, 3.0, -5.0
    p.distance_wanted, p.time_wanted, p.lane_change_delay = 10.0, 1.5, 1.0
    p.lane_change_min_acc_gain, p.lane_change_max_braking_imposed = 0.2, 2.0
    return N, p, graph, st, t


def test_behavior_stop_before_obstacle():
    """vehicle/test_behavior.py:13-27 on the device"""
    N, p, graph, st, t = _single_lane_device([0.0, 80.0], [20.0, 0.0], [0, 3])
    N.check(N.load().hwy_network_substeps(C.byref(p), graph.data_ptr(), None, C.byref(st), None, 10 * K.FPS, None))
    torch.cuda.synchronize()
    x, y = float(t["pos"][1, 0, 0]), float(t["pos"][1, 0, 1])
    assert not (int(t["meta"][1, 0]) & N.META_CRASHED)
    assert x == pytest.approx(70.0, abs=1) and y == pytest.approx(0)
    assert float(t["hs"][1, 0, 1]) == pytest.approx(0, abs=1) and float(t["hs"][1, 0, 0]) == pytest.approx(0)
    assert float(t["pos"][1, 1, 0]) == 80.0  # the object never moves


def test_dynamics_collision_with_obstacle():
    """vehicle/test_dynamics.py:56-60 on the device"""
    N, p, graph, st, t = _single_lane_device([20.0, 23.0], [10.0, 0.0], [0, 3])
    N.check(N.load().hwy_network_substeps(C.byref(p), graph.data_ptr(), None, C.byref(st), None, 1, None))
    torch.cuda.synchronize()
    assert int(t["meta"][1, 0]) & N.META_CRASHED and int(t["meta"][1, 1]) & N.META_CRASHED
