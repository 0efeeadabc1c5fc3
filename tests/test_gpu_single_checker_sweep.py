"""The collision sweep of highway-fast-v0, where the controlled vehicle (slot 0) is the only vehicle that checks
collisions: each traffic vehicle resolves its own pair with the ego, and the ego takes the OR of the crashes and the
impact of the largest partner with will_intersect (the last writer of the reference's (i < j) loop,
vehicle/objects.py:103-116).  Crafted states put 0 to 3 traffic vehicles on or just ahead of / behind the ego, and
some put the only checking vehicle in another slot (or give two vehicles the check), which takes the general sweep.
One step of each is compared against the C oracle."""
import numpy as np
import pytest

import hwy_oracle as ho
from parity_utils import load_golden

pytestmark = pytest.mark.gpu

N = 512


def crafted_states(ob, rng, checkers):
    """The oracle's reset state with e % 4 traffic vehicles moved next to the ego of env e.  checkers(e, movers)
    gives the slots of env e that check collisions."""
    a = ob.a
    lanes = int(ob.cfg.lanes_count)
    for e in range(ob.n):
        k = e % 4
        movers = rng.choice(np.arange(1, ob.V), size=k, replace=False)
        ex, ey, ev = a["x"][e, 0], a["y"][e, 0], a["speed"][e, 0]
        for j in movers:
            # length 5, width 2: |dx| < 5 and |dy| < 2 overlap now; a little further apart, the ego's (or the other
            # vehicle's) displacement over one substep makes the pair will_intersect
            dx = rng.uniform(-7.0, 7.0)
            dy = rng.choice([0.0, 0.0, rng.uniform(-2.6, 2.6)])
            y = float(np.clip(ey + dy, 0.0, 4.0 * (lanes - 1)))
            a["x"][e, j] = ex + dx
            a["y"][e, j] = y
            a["speed"][e, j] = ev + rng.uniform(-6.0, 6.0) * np.sign(-dx)
            lane = int(np.clip(np.rint(y / 4.0), 0, lanes - 1))
            a["lane"][e, j] = a["target_lane"][e, j] = lane
        a["check_collisions"][e] = 0
        a["check_collisions"][e, checkers(e, movers)] = 1


def step_and_compare(env, ob, rng):
    n = ob.n
    env.load_state_dict({k: ob.a[k].copy() for k in ob.a})
    act = rng.integers(0, 5, size=n).astype(np.int32)
    o_obs, o_rew, o_term, o_trunc = ob.step(act)
    obs, rew, term, trunc, _ = env.step(act)
    sd = env.state_dict()
    for k in ("x", "y", "heading", "speed", "timer", "target_speed"):
        d = np.max(np.abs(sd[k] - ob.a[k]))
        assert d <= 1e-7, (k, d)
    for k in ("lane", "target_lane", "crashed", "has_impact"):
        assert np.array_equal(sd[k].astype(np.int32), ob.a[k].astype(np.int32)), k
    hi = ob.a["has_impact"].astype(bool)
    if hi.any():
        assert np.max(np.abs(sd["impact_x"][hi] - ob.a["impact_x"][hi])) <= 1e-7
        assert np.max(np.abs(sd["impact_y"][hi] - ob.a["impact_y"][hi])) <= 1e-7
    assert np.max(np.abs(rew.cpu().numpy() - o_rew)) <= 1e-9
    assert np.array_equal(term.cpu().numpy(), o_term.astype(bool))
    assert np.array_equal(trunc.cpu().numpy(), o_trunc.astype(bool))
    assert np.max(np.abs(obs.cpu().numpy() - o_obs)) <= 1e-6
    return ob.a["crashed"].astype(bool)


def make_pair(seed):
    import highwayenv_b200 as hb

    cfg = dict(load_golden("highway_fast_v50")["config"])
    env_id = cfg.pop("_env_id")
    ob = ho.OracleBatch(ho.cfg_from_dict(cfg), N, seeds=range(seed, seed + N), threads=8)
    cfg.pop("_others_check_collisions", None)
    env = hb.make(env_id, num_envs=N, config=cfg, autoreset_mode="Disabled")
    env.reset(seed=seed)
    ob.reset()
    return env, ob


def test_ego_only_checker_matches_oracle():
    env, ob = make_pair(700)
    rng = np.random.default_rng(1)
    crafted_states(ob, rng, lambda e, movers: [0])
    crashed = step_and_compare(env, ob, rng)
    traffic_hits = crashed[:, 1:].sum(axis=1)
    ks = np.arange(N) % 4
    # the crafted overlaps happen: crashed egos, and envs where two or three traffic vehicles met the ego
    assert crashed[:, 0].sum() > N // 4
    assert ((ks >= 2) & (traffic_hits >= 2)).sum() > 10


def test_other_checkers_match_oracle():
    """The only checking vehicle in another slot (one next to the ego), or two checking vehicles: the general sweep."""
    env, ob = make_pair(900)
    rng = np.random.default_rng(2)
    crafted_states(ob, rng, lambda e, movers: ([] if e % 2 == 0 else [0]) + [movers[0] if len(movers) else 5])
    crashed = step_and_compare(env, ob, rng)
    assert crashed[0::2, 1:].sum() > N // 8 and not crashed[0::2, 0].all()
