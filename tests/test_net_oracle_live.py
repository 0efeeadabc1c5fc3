"""Network oracle vs the reference on seeds that are not in the 32-seed fixtures, teacher-forced, one env at a time.
The reference's states, rewards, flags and observations are stored in tests/golden/pinned_network_*.npz
(oracle/gen_pinned.py).  intersection ids: tests/test_intersection_oracle_live.py."""
import numpy as np
import pytest

import net_oracle as no
from gen_pinned import NETWORK, case_path
from parity_utils import compare_state, load_pinned


@pytest.mark.parametrize("env_id,over,T,seeds", NETWORK)
def test_net_oracle_matches_live_reference(env_id, over, T, seeds):
    for seed in seeds:
        cfg, states, ref = load_pinned(case_path("network", env_id, seed))
        V = int(ref["n_vehicles"])
        ob = no.NetOracleBatch(no.graph_from_arrays(ref), no.cfg_from_dict(cfg, n_vehicles=V), 1)
        ob.load_state(0, states[0])
        assert np.max(np.abs(ob.observe().reshape(ref["obs"][0].shape) - ref["obs"][0])) <= 1e-6
        for t in range(T):
            ob.load_state(0, states[t])  # teacher-forced
            oo, ro, teo, tro = ob.step([int(ref["actions"][t])])
            got = {k: ob.a[k][0] for k in ob.a if k not in ("speed_index", "time")}
            got["speed_index"] = ob.a["speed_index"][0]
            ctx = f"{env_id} seed {seed} t={t}"
            assert compare_state(states[t + 1], got, ctx=ctx) < 1e-9
            assert abs(ref["reward"][t] - ro[0]) < 1e-9, ctx
            assert bool(ref["terminated"][t]) == bool(teo[0]) and bool(ref["truncated"][t]) == bool(tro[0]), ctx
            o = ref["obs"][t + 1]
            assert np.max(np.abs(o - oo[0].reshape(o.shape))) <= 1e-6, ctx
