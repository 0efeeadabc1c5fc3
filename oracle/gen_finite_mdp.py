"""Generate the finite-MDP fixtures from the UNMODIFIED Python reference (build container only).

    python oracle/gen_finite_mdp.py [name ...]     # writes tests/golden/finite_mdp_*.npz

For each case, 4 seeds x 9 states (the reset state and 8 steps of random actions): ref_harness.dump_state of the state
and the reference's own `env.unwrapped.to_finite_mdp()` (envs/common/abstract.py:452-453, envs/common/finite_mdp.py:
17-101) on it — grid, state, transition, reward, terminal — padded to the case's largest shape the way the batched
`to_finite_mdp()` pads: lanes past the ego road's count are 0 in the grid; rows past the env's own state count are
self-loops with reward 0, terminal.  `finite_mdp` itself is not installed: oracle/shim/finite_mdp records the arrays.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ref_harness as rh  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
N_STEPS = 8

# name -> (env_id, config override, seeds)
CASES = {
    "finite_mdp_highway": ("highway-v0", {"vehicles_count": 30}, list(range(3000, 3004))),
    "finite_mdp_highway_fast_pf2": ("highway-fast-v0", {"policy_frequency": 2}, list(range(3010, 3014))),  # T = 20
    "finite_mdp_highway_5lanes": ("highway-v0", {"lanes_count": 5}, list(range(3020, 3024))),
    "finite_mdp_roundabout": ("roundabout-v0", None, list(range(3030, 3034))),
    "finite_mdp_merge": ("merge-v0", None, list(range(3040, 3044))),
    "finite_mdp_exit": ("exit-v0", None, list(range(3050, 3054))),
}


def max_road_lanes(env) -> int:
    return max(len(lanes) for tos in env.road.network.graph.values() for lanes in tos.values())


def main(only) -> None:
    rh._ensure_imports()
    try:
        import finite_mdp  # noqa: F401
    except ModuleNotFoundError:
        sys.path.insert(0, rh._SHIM)
    from highway_env.envs.common.finite_mdp import compute_ttc_grid

    for name, (env_id, over, seeds) in CASES.items():
        if only and name not in only:
            continue
        rng = np.random.default_rng(sum(map(ord, name)))
        states, records = [], []
        for seed in seeds:
            env = rh.make_reference_env(env_id, over)
            env.reset(seed=seed)
            l_max = max_road_lanes(env)
            for t in range(N_STEPS + 1):
                states.append(rh.dump_state(env))
                mdp = env.unwrapped.to_finite_mdp()
                # the grid finite_mdp() built (its MDP only carries the raveled arrays): the same call again
                grid = compute_ttc_grid(env.unwrapped, 1 / env.config["policy_frequency"], 10.0)
                records.append(mdp_record(mdp, grid, l_max))
                if t < N_STEPS:
                    env.step(int(rng.integers(0, 5)))
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
        out["config_json"] = np.array(json.dumps(cfg))
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **out)
        print(f"{name}: {len(states)} states, grid {out['mdp_grid'].shape[1:]} -> {path} "
              f"({os.path.getsize(path) / 1e3:.0f} kB)")


def mdp_record(mdp, grid, l_max: int) -> dict:
    V, L, T = grid.shape
    assert tuple(mdp.original_shape) == (V, L, T)
    S, A = mdp.transition.shape
    s_max = V * l_max * T
    transition = np.tile(np.arange(s_max, dtype=np.int64)[:, None], (1, A))
    reward = np.zeros((s_max, A))
    terminal = np.ones(s_max, dtype=bool)
    transition[:S], reward[:S], terminal[:S] = mdp.transition, mdp.reward, mdp.terminal
    g = np.zeros((V, l_max, T))
    g[:, :L] = grid
    return {"mdp_grid": g, "mdp_n_lanes": np.int32(L), "mdp_state": np.int64(mdp.state),
            "mdp_transition": transition.astype(np.int32), "mdp_reward": reward, "mdp_terminal": terminal}


if __name__ == "__main__":
    if not rh.reference_available():
        raise SystemExit("reference not mounted; golden fixtures can only be generated in the build container")
    main(sys.argv[1:])
