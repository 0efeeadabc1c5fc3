"""The highway step kernel has two instantiations per thread mapping: `AL` (every lane a sideways copy of lane 0, the
general-geometry branches compiled out) and the general one.  On a congruent lane table both must give the same
bits: free-running episodes with SameStep autoreset, same seeds, compared output by output.  Also here: host_stepper() with DiscreteAction."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def rollout(env_id, over, n, T, seed, general=False):
    import highwayenv_b200 as hb

    if general:
        os.environ["HWYB200_GENERAL_LANES"] = "1"
    else:
        os.environ.pop("HWYB200_GENERAL_LANES", None)
    try:
        env = hb.make(env_id, num_envs=n, config=over)
        obs, _ = env.reset(seed=seed)
        out = [obs.cpu().numpy().copy()]
        rng = np.random.default_rng(seed)
        cont = (over or {}).get("action", {}).get("type") == "ContinuousAction"
        for t in range(T):
            if cont:
                act = rng.uniform(-1, 1, size=(n, 2)).astype(np.float32)
            else:
                act = rng.integers(0, 5, size=n).astype(np.int32)
            obs, rew, term, trunc, _ = env.step(act)
            out += [obs.cpu().numpy().copy(), rew.cpu().numpy().copy(), term.cpu().numpy().copy(), trunc.cpu().numpy().copy()]
        sd = env.state_dict()
        out += [sd[k] for k in ("x", "y", "heading", "speed", "timer", "lane", "target_lane", "crashed", "rng")]
        return out
    finally:
        os.environ.pop("HWYB200_GENERAL_LANES", None)


CASES = [
    ("highway-fast-v0", {"vehicles_count": 50}, 64, 40),
    ("highway-fast-v0", None, 64, 40),
    ("highway-v0", {"vehicles_count": 100, "action": {"type": "ContinuousAction"}}, 16, 12),
]


@pytest.mark.parametrize("env_id,over,n,T", CASES)
def test_general_instantiation_is_bit_identical(env_id, over, n, T):
    a = rollout(env_id, over, n, T, 7)
    b = rollout(env_id, over, n, T, 7, general=True)
    for k, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), f"output {k} differs between the AL and the general instantiation"


@pytest.mark.parametrize("env_id,over", [
    ("highway-v0", {"vehicles_count": 30, "action": {"type": "DiscreteAction", "actions_per_axis": 3}}),
    ("intersection-v1", {"action": {"type": "DiscreteAction", "actions_per_axis": 3}}),
])
def test_host_stepper_discrete_action(env_id, over):
    """host_stepper() with DiscreteAction: the index gather is captured with the step; results equal env.step."""
    import highwayenv_b200 as hb

    n = 48
    a = hb.make(env_id, num_envs=n, config=over)
    b = hb.make(env_id, num_envs=n, config=over)
    a.reset(seed=5)
    b.reset(seed=5)
    hs = b.host_stepper()
    rng = np.random.default_rng(2)
    for t in range(20):
        act = rng.integers(0, 9, size=n)
        oa, ra, ta, ua, _ = a.step(act)
        hs.actions[:] = act
        ob, rb, tb, ub = hs.step()
        assert np.array_equal(oa.cpu().numpy(), ob) and np.array_equal(ra.cpu().numpy(), rb), t
        assert np.array_equal(ta.cpu().numpy(), tb) and np.array_equal(ua.cpu().numpy(), ub), t
    hs.actions[0] = 9
    with pytest.raises(IndexError):
        hs.step()
    for bad in (9, -1):  # the eager env.step path checks the index before its device gather
        act = np.zeros(n, dtype=np.int64)
        act[n // 2] = bad
        with pytest.raises(IndexError):
            a.step(act)
