"""intersection ids against the reference on seeds that are not in the fixtures, FREE-RUNNING (no state injection
after the common seed): state, reward, flags, observation and the numpy generator words after every step.  The
reference's episodes are stored in tests/golden/pinned_intersection_*.npz (oracle/gen_pinned.py, one process per
episode: IntersectionEnv._make_vehicles mutates IDMVehicle class constants process-wide)."""
import numpy as np
import pytest

import net_oracle as no
from gen_pinned import INTERSECTION, case_path
from parity_utils import load_pinned
from test_net_oracle_golden import compare_inter


@pytest.mark.parametrize("env_id,obs,seed0,n", INTERSECTION)
def test_intersection_free_running_vs_live_reference(env_id, obs, seed0, n):
    compared = 0
    for seed in range(seed0, seed0 + n):
        cfg, states, ref = load_pinned(case_path("intersection", env_id, obs, seed))
        A = int(cfg.get("controlled_vehicles", 1))
        ob = no.IntersectionOracle(no.graph_from_arrays(ref), no.cfg_from_dict(cfg), 1, ref, cfg)
        ob.reset_env(0, seed=seed)
        compare_inter(states[0], ob.a, 0, f"{env_id} seed {seed} reset", tol=1e-8)
        assert np.max(np.abs(ob.observe().reshape(ref["obs"][0].shape) - ref["obs"][0])) <= 1e-6
        for t in range(len(ref["actions"])):
            a = ref["actions"][t]
            oo, ro, teo, tro = ob.step(a.reshape(1, A) if A > 1 else a)
            ctx = f"{env_id} seed {seed} t={t}"
            st = states[t + 1]
            m = int(st["count"])
            # utils.not_zero(speed) in the steering law (controller.py:166,178) amplifies 1-ulp libm differences by > 1e6
            # per policy step once a non-crashed vehicle crawls below ~1 m/s (tests/parity_utils.py well_conditioned):
            # free-running parity is asserted up to that point, teacher-forced parity (the fixtures) on every state
            if np.any(~st["crashed"][:m].astype(bool) & (np.abs(st["speed"][:m]) < 1.0)):
                break
            compare_inter(st, ob.a, 0, ctx, tol=1e-5)
            assert abs(ref["reward"][t] - ro[0]) <= 1e-6, ctx
            assert bool(ref["terminated"][t]) == bool(teo[0]) and bool(ref["truncated"][t]) == bool(tro[0]), ctx
            o = ref["obs"][t + 1]
            assert np.max(np.abs(o.astype(np.float64).reshape(-1) - oo[0].reshape(-1))) <= 1e-4, ctx
            assert [int(x) for x in ob.rng_words(0)] == [int(x) for x in ref["rng_words"][t]], ctx + " numpy stream"
            compared += 1
    assert compared >= 3 * n
