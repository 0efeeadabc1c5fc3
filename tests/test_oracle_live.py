"""Oracle vs the reference on seeds that are in no 32-seed fixture, teacher-forced.  The reference's states, rewards,
flags, observations and available actions are stored in tests/golden/pinned_*.npz (oracle/gen_pinned.py)."""
import os

import numpy as np
import pytest

import hwy_oracle as ho
from gen_pinned import HIGHWAY, OUT, case_path
from parity_utils import compare_state, load_pinned


@pytest.mark.parametrize("env_id,over,T,seed", HIGHWAY)
def test_oracle_matches_live_reference(env_id, over, T, seed):
    cfg, states, ref = load_pinned(case_path("highway", env_id, seed))
    cfg["_others_check_collisions"] = 0 if env_id == "highway-fast-v0" else 1
    oc = ho.cfg_from_dict(cfg)
    ob = ho.OracleBatch(oc, 1, seeds=[seed])
    assert np.array_equal(ob.reset()[0], ref["obs"][0])
    for t in range(T):
        ob.load_state(0, states[t])  # teacher-forced
        act = [int(ref["actions"][t])] if oc.action_type == 0 else ref["actions"][t].astype(np.float32)[None]
        oo, ro, teo, tro = ob.step(act)
        got = {k: ob.a[k][0] for k in ob.a if k not in ("speed_index", "time")}
        got["speed_index"] = ob.a["speed_index"][0]
        assert compare_state(states[t + 1], got, ctx=f"{env_id} t={t}") < 1e-9
        assert abs(ref["reward"][t] - ro[0]) < 1e-12
        assert bool(ref["terminated"][t]) == bool(teo[0]) and bool(ref["truncated"][t]) == bool(tro[0])
        assert np.max(np.abs(ref["obs"][t + 1] - oo[0])) <= 1e-6


def test_available_actions_mask_matches_live_reference():
    """DiscreteMetaAction.get_available_actions (action.py:262-299) vs the product's tensor form (CPU tensors)"""
    import torch

    from highwayenv_b200.envs.highway_env import available_actions_mask

    ref = np.load(os.path.join(OUT, "pinned_available_actions.npz"), allow_pickle=False)
    table = torch.tensor([[0.0, 4.0 * l, 1.0, 0.0, -0.0, 1.0, 10000.0, 4.0] for l in range(3)], dtype=torch.float64)
    m = available_actions_mask(torch.tensor(ref["x"]), torch.tensor(ref["y"]), torch.tensor(ref["lane"]).long(),
                               torch.tensor(ref["speed_index"]).long(), table, 3).numpy().astype(bool)
    for k in range(len(ref["x"])):
        assert np.array_equal(m[k], ref["mask"][k]), (ref["lane"][k], ref["x"][k], ref["y"][k], ref["speed_index"][k])
