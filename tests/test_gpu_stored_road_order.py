"""The road order the highway step kernels leave in the meta words (HWY_META_ORDER_SHIFT) for the first frame of the
next launch is a hint the kernel checks, never state: whatever those bits hold — an older step's order, values that are
no permutation, a permutation in the wrong order — the next steps return bit-identical results to a batch whose bits
were never touched.  And after every step the bits hold the true order, so that the next first frame can use it."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LINEAR = "highway_env.vehicle.behavior.LinearVehicle"
CASES = [  # (env id, config, envs): TPE 64 with dense 5-env blocks (the headline) and with one env per block, TPE 32
    # with linear traffic, TPE 128 (rank repair, every vehicle checks collisions) with continuous actions
    ("highway-fast-v0", {"vehicles_count": 50}, 4096),
    ("highway-fast-v0", {"vehicles_count": 50}, 40),
    ("highway-fast-v0", {"other_vehicles_type": LINEAR}, 64),
    ("highway-v0", {"vehicles_count": 100, "action": {"type": "ContinuousAction"}}, 48),
]
IDS = ["fast50-dense", "fast50", "fast-linear", "v0-100-continuous"]
ORDER_MASK = 0x7F


def order_bits(env):
    import highwayenv_b200._native as N

    return ((env._meta[:, :env.V] >> N.META_ORDER_SHIFT) & ORDER_MASK).cpu().numpy()


def set_order_bits(env, order):
    import torch
    import highwayenv_b200._native as N

    meta = env._meta[:, :env.V]
    bits = torch.from_numpy(np.ascontiguousarray(order, dtype=np.int32)).to(meta.device)
    env._meta[:, :env.V] = (meta & ~(ORDER_MASK << N.META_ORDER_SHIFT)) | (bits << N.META_ORDER_SHIFT)


def true_order(env):
    """Slots by increasing longitudinal position (every lane of these roads starts at x = 0 along +x), ties by slot."""
    x = env.state_dict()["x"]
    slots = np.broadcast_to(np.arange(env.V), x.shape)
    return np.lexsort((slots, x), axis=-1)


def actions(env, rng):
    sp = env.single_action_space
    if hasattr(sp, "n"):
        return rng.integers(0, sp.n, size=env.num_envs).astype(np.int32)
    return rng.uniform(-1, 1, size=(env.num_envs,) + tuple(sp.shape)).astype(np.float32)


def same_step(ra, rb, ctx):
    for k, x, y in zip(("obs", "reward", "terminated", "truncated"), ra[:4], rb[:4]):
        assert x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes(), (ctx, k)


def same_state(a, b, ctx):
    import torch

    sa, sb = a.state_dict(), b.state_dict()
    for k in sa:
        assert np.asarray(sa[k]).tobytes() == np.asarray(sb[k]).tobytes(), (ctx, k)
    assert torch.equal(a._meta, b._meta), (ctx, "meta words with the order bits")


@pytest.mark.parametrize("env_id,config,n", CASES, ids=IDS)
def test_any_stored_order_gives_the_same_steps(env_id, config, n):
    import highwayenv_b200 as hb

    a = hb.make(env_id, num_envs=n, config=config)
    b = hb.make(env_id, num_envs=n, config=config)
    a.reset(seed=7)
    b.reset(seed=7)
    V = a.V
    rng = np.random.default_rng(11)
    corrupt = np.random.default_rng(12)
    history = []
    for t in range(12):
        history.append(order_bits(b))
        kind = t % 4
        if kind == 0:  # stale: the order two steps back (or the reset's)
            set_order_bits(b, history[max(0, t - 2)])
        elif kind == 1:  # no permutation: any 7-bit value, repeats and slots past the vehicles included
            set_order_bits(b, corrupt.integers(0, ORDER_MASK + 1, size=(n, V)))
        elif kind == 2:  # a permutation, but not the order along the road
            set_order_bits(b, corrupt.permuted(np.tile(np.arange(V), (n, 1)), axis=1))
        else:  # all zero: what a state written from the host carries
            set_order_bits(b, np.zeros((n, V)))
        act = actions(a, rng)
        same_step(a.step(act), b.step(act), (env_id, t))
        same_state(a, b, (env_id, t))


@pytest.mark.parametrize("env_id,config,n", CASES, ids=IDS)
def test_each_step_stores_the_order_along_the_road(env_id, config, n):
    import highwayenv_b200 as hb

    env = hb.make(env_id, num_envs=n, config=dict(config, duration=4))  # short episodes: fused autoresets too
    env.reset(seed=3)
    assert np.array_equal(order_bits(env), true_order(env)), "after the reset"
    rng = np.random.default_rng(5)
    resets = 0
    for t in range(10):
        _, _, term, trunc, _ = env.step(actions(env, rng))
        resets += int((term | trunc).sum())
        assert np.array_equal(order_bits(env), true_order(env)), t
    env.road_substeps(3)
    assert np.array_equal(order_bits(env), true_order(env)), "after road_substeps"
    assert resets > 0
