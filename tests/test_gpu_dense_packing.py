"""Dense env packing of the highway step kernels: each env owns V consecutive threads of a block, so env segments
start anywhere in a warp, a warp can hold parts of two or three envs, and the last warp of a block can have threads that
own no env.  The packing must not change a single bit: free-running SameStep-autoreset episodes under two
HWYB200_EPB values (one of them 1 env per block, the other a block of several envs whose last block is only partly
used) give identical states, observations, rewards, flags, info and generator words, and match the C oracle.
V covers segments straddling one and two warp boundaries, exact multiples of a warp and 32, 64 and 128 slots per
env."""
import numpy as np
import pytest

import hwy_linear_oracle as lo
import hwy_oracle as ho
from parity_utils import FLOAT_TOL

pytestmark = pytest.mark.gpu

VS = [17, 21, 32, 33, 51, 63, 64, 65, 101, 128]
LINEAR = "highway_env.vehicle.behavior.LinearVehicle"
# (env id, config, others check collisions): ego-only collisions, the all-pairs pruned sweep, a ContinuousAction
# ego, LinearVehicle traffic
SCENARIOS = {
    "fast": ("highway-fast-v0", {}, 0),
    "all_pairs": ("highway-v0", {}, 1),
    "continuous": ("highway-fast-v0", {"action": {"type": "ContinuousAction"}}, 0),
    "linear": ("highway-fast-v0", {"other_vehicles_type": LINEAR}, 0),
}
F_KEYS = ("x", "y", "heading", "speed", "timer", "target_speed")
I_KEYS = ("lane", "target_lane", "crashed", "has_impact")


def _make(scenario, V, n):
    import highwayenv_b200 as hb

    env_id, extra, _ = SCENARIOS[scenario]
    cfg = dict(extra, vehicles_count=V - 1, duration=4)  # several autoresets per run
    return hb.make(env_id, num_envs=n, config=cfg, device="cuda:0")


def _actions(env, n, T, seed):
    rng = np.random.default_rng(seed)
    if int(env._params.action_type) == 0:
        return [rng.integers(0, 5, size=n).astype(np.int32) for _ in range(T)]
    return [rng.uniform(-1, 1, size=(n, 2)).astype(np.float32) for _ in range(T)]


def _run(monkeypatch, epb, scenario, V, n, acts, seed):
    """One free-running episode set; returns everything the env returned, step by step, and the final state."""
    monkeypatch.setenv("HWYB200_EPB", str(epb))
    env = _make(scenario, V, n)
    out = [env.reset(seed=seed)[0].cpu().numpy()]
    for a in acts:
        obs, rew, term, trunc, info = env.step(a)
        out += [obs.cpu().numpy(), rew.cpu().numpy(), term.cpu().numpy(), trunc.cpu().numpy()]
        out += [v.cpu().numpy() for _, v in sorted(info.items()) if hasattr(v, "cpu")]
        out += [env.state_dict()["rng"]]
    return out, env.state_dict()


def _oracle(scenario, env, n, seed):
    cfg = dict(env.config)
    cfg["_others_check_collisions"] = SCENARIOS[scenario][2]
    if scenario == "linear":
        return lo.LinearOracleBatch(cfg, n, seeds=range(seed, seed + n), threads=8)
    return ho.OracleBatch(ho.cfg_from_dict(cfg), n, seeds=range(seed, seed + n), threads=8)


@pytest.mark.parametrize("scenario", list(SCENARIOS))
@pytest.mark.parametrize("V", VS)
def test_packings_are_bit_identical_and_match_the_oracle(monkeypatch, scenario, V):
    epb = 256 // V
    if epb * (32 if V <= 32 else 64 if V <= 64 else 128) <= 256:
        # the default block keeps TPE-thread segments (V = 32, 64, 101, 128); one env more takes the dense kernel for
        # V = 101, and for V = 32, 64, 128 (V = TPE) a block of one more env, in the same layout
        epb += 1
    n = 3 * epb + 1  # the last block of the packed run holds one env
    seed, T = 4200 + V, 10
    env = _make(scenario, V, n)
    acts = _actions(env, n, T, seed)
    packed, sd_packed = _run(monkeypatch, epb, scenario, V, n, acts, seed)
    single, sd_single = _run(monkeypatch, 1, scenario, V, n, acts, seed)
    assert len(packed) == len(single)
    for k, (a, b) in enumerate(zip(packed, single)):
        assert a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8)), (scenario, V, k)
    for k in sd_packed:
        assert np.array_equal(sd_packed[k], sd_single[k]), (scenario, V, k)

    # the same episodes on the C oracle, free-running, while no live non-crashed vehicle crawls below 1 m/s (the
    # steering law's not_zero(speed) amplifies 1-ulp differences there, tests/parity_utils.py)
    monkeypatch.setenv("HWYB200_EPB", str(epb))
    env = _make(scenario, V, n)
    ob = _oracle(scenario, env, n, seed)
    assert np.array_equal(env.reset(seed=seed)[0].cpu().numpy(), ob.reset())
    tracking = np.ones(n, dtype=bool)
    compared = 0
    for t, a in enumerate(acts):
        o_obs, o_rew, o_term, o_trunc = ob.step(a, autoreset=True)
        obs, rew, term, trunc, _ = env.step(a)
        sd = env.state_dict()
        tracking &= ~((np.abs(ob.a["speed"]) < 1.0) & ~ob.a["crashed"].astype(bool)).any(axis=1)
        m = tracking
        for k in F_KEYS:
            assert np.max(np.abs(sd[k] - ob.a[k])[m], initial=0.0) <= FLOAT_TOL, (scenario, V, t, k)
        for k in I_KEYS:
            assert np.array_equal(sd[k].astype(np.int32)[m], ob.a[k].astype(np.int32)[m]), (scenario, V, t, k)
        assert np.array_equal(term.cpu().numpy()[m], o_term.astype(bool)[m])
        assert np.array_equal(trunc.cpu().numpy()[m], o_trunc.astype(bool)[m])
        assert np.max(np.abs(rew.cpu().numpy() - o_rew)[m], initial=0.0) <= 1e-6
        assert np.max(np.abs(obs.cpu().numpy() - o_obs)[m], initial=0.0) <= 1e-4
        assert np.array_equal(sd["rng"][0][m], ob.rng["state_hi"][m]) and np.array_equal(sd["rng"][1][m],
                                                                                         ob.rng["state_lo"][m])
        compared += int(m.sum())
    assert compared >= n * T // 2, (scenario, V, compared)


@pytest.mark.parametrize("scenario", ["fast", "linear"])
@pytest.mark.parametrize("V", [21, 51, 101])
def test_road_substeps_and_host_stepper_match_the_default_packing(monkeypatch, scenario, V):
    """Enough envs that the default packing is the full one (no small-batch shrink); one env more than a multiple of
    it.  Eager steps + road_substeps, and the host stepper's CUDA graph step by step against the eager steps."""
    import torch

    n = (256 // V) * 2 * torch.cuda.get_device_properties(0).multi_processor_count + 1
    seed = 900 + V
    acts = _actions(_make(scenario, V, n), n, 6, seed)
    runs = {}
    for epb in (None, 1, 256 // V + 1):
        if epb is None:
            monkeypatch.delenv("HWYB200_EPB", raising=False)
        else:
            monkeypatch.setenv("HWYB200_EPB", str(epb))
        eager, graph = _make(scenario, V, n), _make(scenario, V, n)
        eager.reset(seed=seed)
        graph.reset(seed=seed)
        hs = graph.host_stepper()
        outs = []
        for t, a in enumerate(acts):
            o, r, te, tr, _ = eager.step(a)
            hs.actions[:] = a
            ho, hr, hte, htr = hs.step()
            for x, y in ((o, ho), (r, hr), (te, hte), (tr, htr)):
                assert np.array_equal(x.cpu().numpy(), y), (scenario, V, epb, t)
            outs += [ho.copy(), hr.copy(), hte.copy(), htr.copy()]
        eager.road_substeps(7)
        runs[epb] = eager.state_dict(), graph.state_dict(), outs
    want_sd, want_graph_sd, want_outs = runs.pop(None)
    for epb, (sd, graph_sd, outs) in runs.items():
        for k in want_sd:
            assert np.array_equal(sd[k], want_sd[k]), (scenario, V, epb, k)
            assert np.array_equal(graph_sd[k], want_graph_sd[k]), (scenario, V, epb, k)
        for k, (a, b) in enumerate(zip(outs, want_outs)):
            assert np.array_equal(a, b), (scenario, V, epb, k)
