"""Generate the OPD tree fixtures from the UNMODIFIED Python reference (needs the reference checkout).

    python oracle/gen_opd.py [name ...]     # writes tests/golden/opd_*.npz

For each case, 8 seeds x 4 decision states (the reset state, then a random action between decisions): the numpy
statement of tests/opd_spec.py planned over `copy.deepcopy(env.unwrapped)` + `env.step(a)` of the reference — the
expansion rl-agents' DeterministicPlannerAgent makes (`AbstractEnv.__deepcopy__`, envs/common/abstract.py:455-465),
expanding only `env.get_available_actions()` (abstract.py:357-358).  Per record: ref_harness.dump_state of the root,
the root's available actions, the whole tree, the selected leaves with their margins over the runner-up, and the
recommended action with its margin.

Before the first case, a deepcopy of a reference env is checked to step bit-identically to its parent.
"""
from __future__ import annotations

import copy
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "tests"))
import ref_harness as rh  # noqa: E402
from opd_spec import N_ACTIONS, opd, reference_expander  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
BUDGET, GAMMA = 50, 0.7  # the reference's planning notebook (scripts/highway_planning.ipynb)
N_DECISIONS = 4

# name -> (env_id, config override, seeds)
CASES = {
    "opd_highway_fast": ("highway-fast-v0", None, list(range(4000, 4008))),
    "opd_highway": ("highway-v0", {"vehicles_count": 30}, list(range(4010, 4018))),
    "opd_roundabout": ("roundabout-v0", None, list(range(4020, 4028))),
    "opd_merge": ("merge-v0", None, list(range(4030, 4038))),
}


def _step(env, a):
    _, r, term, trunc, _ = env.step(int(a))
    return float(r), bool(term), bool(trunc)


def check_deepcopy_is_exact() -> None:
    env = rh.make_reference_env("highway-fast-v0")
    env.reset(seed=1)
    twin = copy.deepcopy(env.unwrapped)
    for a in (3, 0, 1, 2, 4, 1):
        got = [_step(e, a) for e in (env, twin)]
        assert got[0] == got[1], got
        s0, s1 = rh.dump_state(env), rh.dump_state(twin)
        for k in s0:
            assert np.asarray(s0[k]).tobytes() == np.asarray(s1[k]).tobytes(), k


def plan(env) -> dict:
    expand = reference_expander([env], lambda e: copy.deepcopy(e.unwrapped), _step,
                                lambda e: e.unwrapped.get_available_actions())
    tree = opd(1, BUDGET, GAMMA, expand)
    avail = np.zeros(N_ACTIONS, bool)
    avail[env.unwrapped.get_available_actions()] = True
    out = {"opd_" + k: v[0] for k, v in tree.items()}
    out["opd_available"] = avail
    return out


def main(only) -> None:
    rh._ensure_imports()
    check_deepcopy_is_exact()
    for name, (env_id, over, seeds) in CASES.items():
        if only and name not in only:
            continue
        t0 = time.time()
        rng = np.random.default_rng(sum(map(ord, name)))
        states, records = [], []
        for seed in seeds:
            env = rh.make_reference_env(env_id, over)
            env.reset(seed=seed)
            for t in range(N_DECISIONS):
                states.append(rh.dump_state(env))
                records.append(plan(env))
                if t < N_DECISIONS - 1:
                    env.step(int(rng.integers(0, N_ACTIONS)))
        keys = [k for k in states[0].keys() if all(k in s for s in states)]
        out = {k: np.stack([s[k] for s in states]) for k in keys}
        for k in records[0]:
            out[k] = np.stack([r[k] for r in records])
        env = rh.make_reference_env(env_id, over)
        env.reset(seed=0)
        if not env_id.startswith("highway"):
            out.update(rh.dump_network(env))
        cfg = dict(env.config)
        cfg["_env_id"] = env_id
        cfg["_override"] = over or {}
        cfg["_target_speeds"] = [float(x) for x in env.vehicle.target_speeds]
        cfg["_budget"], cfg["_gamma"] = BUDGET, GAMMA
        out["config_json"] = np.array(json.dumps(cfg))
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **out)
        print(f"{name}: {len(states)} decisions in {time.time() - t0:.0f} s -> {path} "
              f"({os.path.getsize(path) / 1e3:.0f} kB)", flush=True)


if __name__ == "__main__":
    if not rh.reference_available():
        raise SystemExit("the reference checkout is not present; the fixtures are generated from it")
    main(sys.argv[1:])
