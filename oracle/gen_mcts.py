"""Generate the MCTS fixtures from the UNMODIFIED Python reference (needs the reference checkout).

    python oracle/gen_mcts.py [name ...]     # writes tests/golden/mcts_*.npz

For each case, 8 seeds x 4 decision states (the reset state, then a random action between decisions), 32 roots: the
numpy statement of tests/mcts_spec.py planned for the 32 roots in lockstep (root k = record k, decision 0) over
`copy.deepcopy(env.unwrapped)` + `env.step(a)` of the reference — the episode copies rl-agents' MCTSAgent makes
(`safe_deepcopy_env`, `AbstractEnv.__deepcopy__`, envs/common/abstract.py:455-465), with the reference's
`get_available_actions()` (abstract.py:357-358) as prior and rollout support.  Per record: ref_harness.dump_state of
the root, the root's available actions, the whole tree, the per-episode leaf / return / descent margin, the
recommended action with its margin, and the trace of every callback (available actions, actions, rewards, done) so the
CPU tests can replay the plan without the reference.
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
from mcts_spec import FIELDS, N_ACTIONS, budget_split, empty_tree, plan, recording, reference_callbacks  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
BUDGET, GAMMA, TEMPERATURE, SEED = 100, 0.7, 1.0, 12345
N_DECISIONS = 4

# name -> (env_id, config override, seeds): the OPD cases' configs (oracle/gen_opd.py) on new seeds
CASES = {
    "mcts_highway_fast": ("highway-fast-v0", None, list(range(6000, 6008))),
    "mcts_highway": ("highway-v0", {"vehicles_count": 30}, list(range(6010, 6018))),
    "mcts_roundabout": ("roundabout-v0", None, list(range(6020, 6028))),
    "mcts_merge": ("merge-v0", None, list(range(6030, 6038))),
}


def _step(env, a):
    _, r, term, trunc, _ = env.step(int(a))
    return float(r), bool(term), bool(trunc)


def callbacks(roots):
    return reference_callbacks(roots, lambda e: copy.deepcopy(e.unwrapped), _step,
                               lambda e: e.unwrapped.get_available_actions())


def run(roots):
    """(tree, out, trace) of the spec over reference root envs, root k keyed as root k of decision 0."""
    episodes, horizon = budget_split(BUDGET, GAMMA)
    tree = empty_tree(len(roots), 1 + N_ACTIONS * episodes)
    cbs, stacked = recording(*callbacks(roots))
    out = plan(tree, episodes, horizon, GAMMA, TEMPERATURE, SEED, 0, *cbs)
    return tree, out, stacked()


def main(only) -> None:
    rh._ensure_imports()
    for name, (env_id, over, seeds) in CASES.items():
        if only and name not in only:
            continue
        t0 = time.time()
        rng = np.random.default_rng(sum(map(ord, name)))
        states, roots, avail = [], [], []
        for seed in seeds:
            env = rh.make_reference_env(env_id, over)
            env.reset(seed=seed)
            for t in range(N_DECISIONS):
                states.append(rh.dump_state(env))
                roots.append(copy.deepcopy(env.unwrapped))
                a = np.zeros(N_ACTIONS, bool)
                a[env.unwrapped.get_available_actions()] = True
                avail.append(a)
                if t < N_DECISIONS - 1:
                    env.step(int(rng.integers(0, N_ACTIONS)))
        tree, res, trace = run(roots)
        keys = [k for k in states[0].keys() if all(k in s for s in states)]
        out = {k: np.stack([s[k] for s in states]) for k in keys}
        out.update({"tree_" + k: tree[k] for k in FIELDS + ("n_nodes", "skipped")})
        out.update({"out_" + k: v for k, v in res.items()})
        out.update({"trace_" + k: v for k, v in trace.items()})
        out["available"] = np.stack(avail)
        env = rh.make_reference_env(env_id, over)
        env.reset(seed=0)
        if not env_id.startswith("highway"):
            out.update(rh.dump_network(env))
        cfg = dict(env.config)
        cfg["_env_id"] = env_id
        cfg["_override"] = over or {}
        cfg["_target_speeds"] = [float(x) for x in env.vehicle.target_speeds]
        cfg["_budget"], cfg["_gamma"], cfg["_temperature"], cfg["_seed"] = BUDGET, GAMMA, TEMPERATURE, SEED
        out["config_json"] = np.array(json.dumps(cfg))
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **out)
        print(f"{name}: {len(states)} roots in {time.time() - t0:.0f} s -> {path} "
              f"({os.path.getsize(path) / 1e3:.0f} kB)", flush=True)


if __name__ == "__main__":
    if not rh.reference_available():
        raise SystemExit("the reference checkout is not present; the fixtures are generated from it")
    main(sys.argv[1:])
