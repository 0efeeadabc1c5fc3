"""`env.copy_envs` (csrc/hwy_copy.cu) on every env family: a copied env behaves as `copy.deepcopy` of its source —
the same observations, rewards, flags and state (streams included) under the same actions, autoresets included —
and every env it did not write is untouched."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LINEAR = "highway_env.vehicle.behavior.LinearVehicle"
FAMILIES = [
    ("highway-fast-v0", None),
    ("highway-fast-v0", {"other_vehicles_type": LINEAR}),
    ("roundabout-v0", None),
    ("merge-v0", None),
    ("two-way-v0", None),
    ("u-turn-v0", None),
    ("exit-v0", None),
    ("intersection-v0", None),
    ("intersection-multi-agent-v0", None),
    ("intersection-v1", None),
]
IDS = [e + ("-linear" if c else "") for e, c in FAMILIES]
N = 8


def make(env_id, config, seed, n=N, **kw):
    import highwayenv_b200 as hb

    env = hb.make(env_id, num_envs=n, config=dict(config or {}), **kw)
    env.reset(seed=seed)
    return env


def random_actions(env, rng):
    sp = env.single_action_space
    if hasattr(sp, "n"):
        return rng.integers(0, sp.n, size=env.num_envs).astype(np.int32)
    shape = (env.num_envs,) + tuple(sp.shape)
    if np.issubdtype(sp.dtype, np.integer):
        return rng.integers(sp.low.min(), sp.high.max() + 1, size=shape).astype(np.int32)
    return rng.uniform(-1, 1, size=shape).astype(np.float32)


def rows(env):
    """Per-env numpy rows of everything observable: state_dict fields with a leading env axis and the streams."""
    sd = env.state_dict()
    out = {k: np.asarray(v) for k, v in sd.items() if k != "rng" and np.ndim(v) >= 1 and np.shape(v)[0] == env.num_envs}
    out["rng"] = env.rng_words().T
    return out


def same_rows(a, ia, b, ib, ctx):
    for k in a:
        x, y = np.ascontiguousarray(a[k][ia]), np.ascontiguousarray(b[k][ib])
        assert x.shape == y.shape and x.tobytes() == y.tobytes(), (ctx, k)


def step_pair(a, b, act_a, act_b, ia, ib, ctx):
    oa, ra, ta, tra, _ = a.step(act_a)
    ob, rb, tb, trb, _ = b.step(act_b)
    for name, x, y in (("obs", oa, ob), ("reward", ra, rb), ("terminated", ta, tb), ("truncated", tra, trb)):
        x, y = x.cpu().numpy()[ia], y.cpu().numpy()[ib]
        assert x.tobytes() == y.tobytes(), (ctx, name)


@pytest.mark.parametrize("env_id,config", FAMILIES, ids=IDS)
def test_copy_from_another_env_then_step(env_id, config):
    rng = np.random.default_rng(3)
    a = make(env_id, config, seed=11)
    for _ in range(3):
        a.step(random_actions(a, rng))
    b, twin = make(env_id, config, seed=500), make(env_id, config, seed=500)
    for _ in range(2):
        act = random_actions(b, rng)
        b.step(act)
        twin.step(act)
    dst, src = np.array([1, 4, 6]), np.array([0, 3, 7])
    keep = np.setdiff1d(np.arange(N), dst)
    b.copy_envs(dst, src, source=a)
    same_rows(rows(a), src, rows(b), dst, "after copy")
    same_rows(rows(twin), keep, rows(b), keep, "uncopied rows after copy")
    assert b.observe().cpu().numpy()[dst].tobytes() == a.observe().cpu().numpy()[src].tobytes()
    for t in range(10):
        act_a = random_actions(a, rng)
        act_b = random_actions(b, rng)
        act_b[dst] = act_a[src]
        step_pair(a, b, act_a, act_b, src, dst, (env_id, t))
        twin.step(act_b)
        same_rows(rows(a), src, rows(b), dst, (env_id, t))
        same_rows(rows(twin), keep, rows(b), keep, (env_id, t, "uncopied"))


@pytest.mark.parametrize("env_id,config", FAMILIES, ids=IDS)
def test_copy_within_one_env_then_step(env_id, config):
    rng = np.random.default_rng(4)
    a, twin = make(env_id, config, seed=21), make(env_id, config, seed=21)
    for _ in range(2):
        act = random_actions(a, rng)
        a.step(act)
        twin.step(act)
    dst, src = [5, 2], [0, 3]
    a.copy_envs(dst, src)
    keep = np.setdiff1d(np.arange(N), dst)
    for t in range(10):
        act = random_actions(a, rng)
        act[dst] = act[src]
        o, r, te, tr, _ = a.step(act)
        twin.step(act)
        for x in (o, r, te, tr):
            x = x.cpu().numpy()
            assert x[dst].tobytes() == x[src].tobytes(), (env_id, t)
        ra = rows(a)
        same_rows(ra, src, ra, dst, (env_id, t))
        same_rows(rows(twin), keep, ra, keep, (env_id, t, "uncopied"))


def test_next_step_pending_reset_is_copied():
    """NextStep autoreset: an env that ended in the last step is reset by the next one; a copy of it is too."""
    rng = np.random.default_rng(5)
    cfg = {"duration": 3}
    a = make("highway-fast-v0", cfg, seed=31, autoreset_mode="NextStep")
    b = make("highway-fast-v0", cfg, seed=900, autoreset_mode="NextStep")
    for _ in range(3):  # every env of a is truncated by this step: its reset is pending
        a.step(random_actions(a, rng))
    assert a._autoreset_envs.bool().all()
    dst, src = np.array([0, 2, 3]), np.array([7, 6, 1])
    b.copy_envs(dst, src, source=a)
    for t in range(10):
        act_a = random_actions(a, rng)
        act_b = random_actions(b, rng)
        act_b[dst] = act_a[src]
        step_pair(a, b, act_a, act_b, src, dst, t)
        same_rows(rows(a), src, rows(b), dst, t)


def test_copy_seeds_a_destination_never_reset_and_replays_in_a_cuda_graph():
    import highwayenv_b200 as hb
    import torch

    a = make("roundabout-v0", None, seed=41)
    a.step(np.zeros(N, np.int32))
    b = hb.make("roundabout-v0", num_envs=N)
    dst = torch.tensor([3, 4], dtype=torch.int64, device="cuda")
    src = torch.tensor([1, 2], dtype=torch.int64, device="cuda")
    b.copy_envs(dst, src, source=a)
    assert b._seeded
    same_rows(rows(a), [1, 2], rows(b), [3, 4], "unseeded destination")
    # captured: the copy reads its indices on the device
    c = make("roundabout-v0", None, seed=42)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c.copy_envs(dst, src, source=a)
    torch.cuda.synchronize()
    graph.replay()
    torch.cuda.synchronize()
    same_rows(rows(a), [1, 2], rows(c), [3, 4], "graph replay")


@pytest.mark.parametrize("env_id,config", FAMILIES, ids=IDS)
def test_every_per_env_tensor_is_copied_or_excluded(env_id, config):
    """Drift guard: a tensor with a leading num_envs axis that copy_envs neither copies nor excludes fails here."""
    import torch

    for mode in ("SameStep", "NextStep"):
        env = make(env_id, config, seed=1, n=7, autoreset_mode=mode)
        env.step(random_actions(env, np.random.default_rng(0)))
        copied = {name for name, t in env._env_rows().items()}
        for name, t in vars(env).items():
            if isinstance(t, torch.Tensor) and t.dim() >= 1 and t.shape[0] in (7, 7 * getattr(env, "n_agents", 1)):
                assert name in copied or name in env.ROW_EXCLUDE, (env_id, mode, name)
        assert "_rng" in copied and "_obs" in copied
        assert ("_autoreset_envs" in copied) == (mode == "NextStep")


def test_rejections_raise_before_any_launch():
    import highwayenv_b200 as hb

    a = make("highway-fast-v0", None, seed=1)
    with pytest.raises(TypeError):
        a.copy_envs([0], [0], source=make("highway-v0", {"vehicles_count": 20, "lanes_count": 3}, seed=1))
    with pytest.raises(ValueError):  # another vehicle count
        a.copy_envs([0], [0], source=make("highway-fast-v0", {"vehicles_count": 30}, seed=1))
    with pytest.raises(ValueError):  # another traffic model
        a.copy_envs([0], [0], source=make("highway-fast-v0", {"other_vehicles_type": LINEAR}, seed=1))
    with pytest.raises(ValueError):  # another observation shape
        a.copy_envs([0], [0], source=make("highway-fast-v0", {"observation": {"type": "Kinematics",
                                                                               "vehicles_count": 7}}, seed=1))
    with pytest.raises(RuntimeError):  # a source never reset
        a.copy_envs([0], [0], source=hb.make("highway-fast-v0", num_envs=N))
    with pytest.raises(ValueError):
        a.copy_envs([0, 1], [2])
    with pytest.raises(IndexError):
        a.copy_envs([N], [0])
    with pytest.raises(IndexError):
        a.copy_envs([0], [-1])
    with pytest.raises(IndexError):
        a.copy_envs([0], [3], source=make("highway-fast-v0", None, seed=2, n=2))
    with pytest.raises(ValueError):
        a.copy_envs([1, 1], [2, 3])
    with pytest.raises(ValueError):
        a.copy_envs([1, 2], [2, 3])
    m = make("intersection-multi-agent-v0", None, seed=1)
    with pytest.raises(TypeError):
        m.copy_envs([0], [0], source=make("intersection-v0", None, seed=1))
    # none of the rejected calls changed anything
    before = rows(a)
    a.copy_envs([], [])
    same_rows(before, np.arange(N), rows(a), np.arange(N), "empty copy")
