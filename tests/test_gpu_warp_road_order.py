"""Dense env segments of 33 to 64 vehicles find each env's road order with one warp (warp_order: odd-even transposition
passes over the previous permutation); the TPE-thread instantiation of the same kernel counts every vehicle's rank
(rank_count).  Both must give the same bits on states made to leave the sort's easy case: many rank-neighbours swapped
at once, a stored order that is the road order reversed, equal float keys of different doubles, and exact ties
(which switch the env to the linear neighbour scans).  HWYB200_EPB picks the instantiation: with V = 51 (41), 5 (6)
envs per block run dense segments and 4 envs per block TPE-thread segments."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

LINEAR = "highway_env.vehicle.behavior.LinearVehicle"
CASES = [  # (env id, config, dense envs per block): the headline's collision gate, the rank-pruned sweep, linear traffic
    ("highway-fast-v0", {"vehicles_count": 50}, 5),
    ("highway-v0", {"vehicles_count": 40}, 6),
    ("highway-fast-v0", {"vehicles_count": 50, "other_vehicles_type": LINEAR}, 5),
]
IDS = ["fast50", "v0-40-pruned", "fast50-linear"]
KINDS = ["swaps", "reversed", "equal-floats", "ties"]
N_ENVS, STEPS = 40, 4
ORDER_MASK = 0x7F


def set_order_bits(env, order):
    import torch
    import highwayenv_b200._native as N

    meta = env._meta[:, :env.V]
    bits = torch.from_numpy(np.ascontiguousarray(order, dtype=np.int32)).to(meta.device)
    env._meta[:, :env.V] = (meta & ~(ORDER_MASK << N.META_ORDER_SHIFT)) | (bits << N.META_ORDER_SHIFT)


def road_order(x):
    return np.lexsort((np.broadcast_to(np.arange(x.shape[1]), x.shape), x), axis=-1)


def crafted(env, kind):
    """A state of `env` (just reset) and the stored order that goes with it."""
    sd = env.state_dict()
    x, y = sd["x"], sd["y"]
    order = road_order(x)
    rows = np.arange(x.shape[0])
    if kind == "swaps":
        # ranks 2m and 2m + 1 trade places for every m: the stored order has V / 2 inverted boundaries two apart,
        # which frame 0 has to sort all at once
        for k in range(0, x.shape[1] - 1, 2):
            a, b = order[:, k], order[:, k + 1]
            xa, xb = x[rows, a].copy(), x[rows, b].copy()
            x[rows, a], x[rows, b] = xb, xa
    elif kind == "reversed":
        order = order[:, ::-1]
    elif kind in ("equal-floats", "ties"):
        # each vehicle of odd rank moves beside its lower rank-neighbour, on the next lane over: the same double
        # (ties) or a double that rounds to the same float
        for k in range(1, x.shape[1], 2):
            a, b = order[:, k - 1], order[:, k]
            xa = x[rows, a]
            if kind == "ties":
                x[rows, b] = xa
            else:
                up = np.nextafter(xa, np.inf)
                x[rows, b] = np.where(np.float32(up) == np.float32(xa), up, np.nextafter(xa, -np.inf))
                assert (np.float32(x[rows, b]) == np.float32(xa)).all() and (x[rows, b] != xa).all()
            lane_w = 4.0
            y[rows, b] = np.where(y[rows, a] >= lane_w, y[rows, a] - lane_w, y[rows, a] + lane_w)
    sd["x"], sd["y"] = x, y
    return sd, order


def run(env_id, config, kind, epb, monkeypatch):
    import highwayenv_b200 as hb

    monkeypatch.setenv("HWYB200_EPB", str(epb))
    env = hb.make(env_id, num_envs=N_ENVS, config=config)
    env.reset(seed=21)
    sd, order = crafted(env, kind)
    env.load_state_dict(sd)
    set_order_bits(env, order)
    rng = np.random.default_rng(4)
    out = []
    for _ in range(STEPS):
        obs, rew, term, trunc, info = env.step(rng.integers(0, 5, size=N_ENVS).astype(np.int32))
        out += [obs.cpu().numpy(), rew.cpu().numpy(), term.cpu().numpy(), trunc.cpu().numpy()]
        s = env.state_dict()
        out += [np.asarray(s[k]) for k in sorted(s)] + [env._meta.cpu().numpy()]
    return out


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("env_id,config,epb", CASES, ids=IDS)
def test_warp_order_matches_rank_count(env_id, config, epb, kind, monkeypatch):
    dense = run(env_id, config, kind, epb, monkeypatch)
    counted = run(env_id, config, kind, 4, monkeypatch)
    for k, (a, b) in enumerate(zip(dense, counted)):
        assert a.tobytes() == b.tobytes(), (kind, k)
