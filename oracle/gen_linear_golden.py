"""Golden fixtures of LinearVehicle / AggressiveVehicle / DefensiveVehicle traffic on the highway family, from the
UNMODIFIED Python reference (build container only).

    python oracle/gen_linear_golden.py [case ...]      # writes tests/golden/linear_*.npz

Each fixture is a seeded ref_harness.rollout, as in gen_golden.py, plus ``linear_params`` [seeds, V, 5]: every
vehicle's ACCELERATION_PARAMETERS (3) and STEERING_PARAMETERS (2) after the reset (randomize_behavior,
vehicle/behavior.py:406-415; they never change within an episode).  The controlled vehicle's row is zero.
tests/test_linear_traffic_spec.py pins the C oracle to these, tests/test_gpu_linear_traffic.py the CUDA path.
"""
from __future__ import annotations

import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ref_harness as rh  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
B = "highway_env.vehicle.behavior."

# name -> (env_id, config override, seeds, n_steps, action kind)
CASES = {
    # highway-fast-v0 defaults (V = 21)
    "linear_highway_fast_v20": ("highway-fast-v0", {"other_vehicles_type": B + "LinearVehicle"},
                                list(range(3000, 3032)), 20, "discrete5"),
    # highway-fast-v0 with 50 vehicles (V = 51)
    "linear_aggressive_fast_v50": ("highway-fast-v0", {"other_vehicles_type": B + "AggressiveVehicle",
                                                       "vehicles_count": 50},
                                   list(range(3100, 3132)), 20, "discrete5"),
    # highway-v0 defaults: all-pairs collisions, 15 substeps, 4 lanes
    "linear_defensive_v50": ("highway-v0", {"other_vehicles_type": B + "DefensiveVehicle"},
                             list(range(3200, 3232)), 12, "discrete5"),
    # highway-v0 with 100 vehicles (V = 101, 128 threads per env) and a plain-Vehicle ContinuousAction ego, whose
    # target speed the linear model reads as its own speed
    "linear_highway_v100_continuous": ("highway-v0", {"other_vehicles_type": B + "LinearVehicle", "vehicles_count": 100,
                                                      "action": {"type": "ContinuousAction"}},
                                       list(range(3300, 3332)), 8, "box2"),
}


def _params(env) -> np.ndarray:
    out = np.zeros((len(env.road.vehicles), 5), dtype=np.float64)
    for k, v in enumerate(env.road.vehicles):
        if v in env.controlled_vehicles:
            continue
        out[k, :3] = v.ACCELERATION_PARAMETERS
        out[k, 3:] = v.STEERING_PARAMETERS
    return out


def main() -> None:
    os.makedirs(OUT, exist_ok=True)
    only = sys.argv[1:]
    for name, (env_id, over, seeds, T, akind) in CASES.items():
        if only and name not in only:
            continue
        t0 = time.time()
        rng = np.random.default_rng(sum(map(ord, name)))
        per_seed, params = [], []
        for seed in seeds:
            if akind == "discrete5":
                actions = rng.integers(0, 5, size=T).astype(np.int64)
            else:
                actions = rng.uniform(-1, 1, size=(T, 2)).astype(np.float32)
            got = []
            per_seed.append(rh.rollout(env_id, over, seed, list(actions), mutate=lambda env: got.append(_params(env))))
            params.append(got[0])
        out = {k: np.stack([p[k] for p in per_seed]) for k in per_seed[0].keys()}
        out["seeds"] = np.array(seeds, dtype=np.int64)
        out["linear_params"] = np.stack(params)
        cfg = dict(rh.make_reference_env(env_id, over).config)
        cfg["_others_check_collisions"] = 0 if env_id == "highway-fast-v0" else 1
        cfg["_env_id"] = env_id
        out["config_json"] = np.array(json.dumps(cfg))
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **out)
        print(f"{name}: {len(seeds)} seeds x {T} steps -> {path} "
              f"({os.path.getsize(path)/1e3:.0f} kB, {time.time()-t0:.1f}s)")


if __name__ == "__main__":
    if not rh.reference_available():
        raise SystemExit("reference not mounted; golden fixtures can only be generated in the build container")
    main()
