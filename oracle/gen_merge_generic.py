"""Generate the merge-generic-v0 / v1 fixtures from the UNMODIFIED Python reference (needs the reference checkout).

    python oracle/gen_merge_generic.py [name ...]
    # writes tests/golden/mg_*.npz and pinned_to_config_merge_generic_*.json

For each case, SEEDS x T steps of `MergeGenericEnv` / `ConnectedLaneMergeGenericEnv` (envs/merge_env.py:193-379)
under seeded uniform random actions (integers(0, 5) from a generator keyed by the seed).  When a step ends the
episode, `env.reset()` (no seed) starts the next one on the same stream, as a vector env's autoreset does.  Stored per
seed, in the record format of oracle/gen_roundabout_generic.py:

* on every step: terminated, truncated, crashed (`flags`), the action and the smallest |speed| of a vehicle that has
  not crashed after the step (`min_speed`; tests/parity_utils.py well_conditioned);
* after the seeded reset (`reset_*`), every STRIDE-th step (`steps`, no prefix) and after each autoreset
  (`autoreset_*`, at most MAX_RESETS, `autoreset_step` -1 past the last): the state in ref_harness.dump_state's
  schema padded to the case's slot stride (8 for vehicles_count <= 5, else 32) with `count` and `kind` (3 for the
  Obstacle, which comes after the vehicles), the observation, the stream words and get_available_actions() as a mask
  [5]; on stored steps also the reward and the info["rewards"] terms (collision, right_lane, high_speed, lane_change,
  merging_speed).

Cases:
* mg_default: merge-generic-v0 at its defaults;
* mg_v1_default: merge-generic-v1 (connected-lane neighbour search);
* mg_three_lanes: lanes_count 3, vehicles_count 5 (8 slots full); ("b","c",2) is an ordinary highway lane, so the
  merging term is non-zero on some stored step (asserted);
* mg_one_lane_ttc: lanes_count 1, vehicles_count 4, TimeToCollision (integers(1) draws nothing; no ("b","c",2));
* mg_crowded_32: lanes_count 2, vehicles_count 25, lengths 60 / 40 / 50 / 90 (32 slots, short populations asserted,
  early terminations);
* mg_float_grid: lanes_count 3, lengths 97.5 / 62.25 / 80.5 / 120.5 (end_position 270.75; the sections start at
  non-integer x), OccupancyGrid.

The lane indices are table indices of make_merge_generic_network, whose order the pinned to_config files fix.
"""
from __future__ import annotations

import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import ref_harness as rh  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
SEEDS = list(range(32))
T = 60
STRIDE = 6
MAX_RESETS = 24
TERMS = ("collision_reward", "right_lane_reward", "high_speed_reward", "lane_change_reward", "merging_speed_reward")
FIELDS = ("x", "y", "heading", "speed", "target_speed", "timer", "delta", "lane", "target_lane", "crashed", "impact",
          "check_collisions", "speed_index", "kind")
LENGTHS = ("before_merge_length", "converge_merge_length", "parallel_merge_length", "after_merge_length")

CASES = {
    "mg_default": ("merge-generic-v0", None),
    "mg_v1_default": ("merge-generic-v1", None),
    "mg_three_lanes": ("merge-generic-v0", {"lanes_count": 3, "vehicles_count": 5}),
    "mg_one_lane_ttc": ("merge-generic-v0", {"lanes_count": 1, "vehicles_count": 4,
                                             "observation": {"type": "TimeToCollision"}}),
    "mg_crowded_32": ("merge-generic-v0", {"lanes_count": 2, "vehicles_count": 25, "before_merge_length": 60,
                                           "converge_merge_length": 40, "parallel_merge_length": 50,
                                           "after_merge_length": 90}),
    "mg_float_grid": ("merge-generic-v0", {"lanes_count": 3, "before_merge_length": 97.5,
                                           "converge_merge_length": 62.25, "parallel_merge_length": 80.5,
                                           "after_merge_length": 120.5, "observation": {"type": "OccupancyGrid"}}),
}
SHORT_POPULATIONS = ("mg_crowded_32",)  # must hold at least one reset that skipped a vehicle
MERGING_ON_HIGHWAY = ("mg_three_lanes",)  # must hold a stored step with a non-zero merging term
# to_config of the reference's road per (lanes_count, before, converge, parallel, after)
PINNED = [(2, 150, 80, 80, 150), (1, 150, 80, 80, 150), (3, 97.5, 62.25, 80.5, 120.5), (9, 150, 80, 80, 150)]


def pinned_name(lanes, pre, conv, par, after) -> str:
    return f"pinned_to_config_merge_generic_l{lanes}_{pre}_{conv}_{par}_{after}.json"


def make_env(env_id: str, over):
    rh._ensure_imports()
    from highway_env.envs import merge_env as M

    cls = {"merge-generic-v0": M.MergeGenericEnv, "merge-generic-v1": M.ConnectedLaneMergeGenericEnv}[env_id]
    return cls(config=over)


def slots_of(config) -> int:
    return 8 if int(config["vehicles_count"]) <= 5 else 32


def stream_words(env) -> np.ndarray:
    st = env.np_random.bit_generator.state
    m64 = (1 << 64) - 1
    return np.array([st["state"]["state"] >> 64, st["state"]["state"] & m64, st["state"]["inc"] >> 64,
                     st["state"]["inc"] & m64, (int(st["has_uint32"]) << 32) | int(st["uinteger"])], dtype=np.uint64)


def snapshot(env, obs, pad) -> dict:
    d = rh.dump_state(env, pad)  # vehicles, then the Obstacle (kind 3)
    n = int(d["count"])
    d["kind"][n:] = 0
    out = {k: np.asarray(d[k]) for k in FIELDS}
    avail = np.zeros(5, dtype=np.bool_)
    avail[list(env.get_available_actions())] = True
    out.update(count=np.int32(n), time=np.float64(env.time), obs=np.asarray(obs, dtype=np.float64),
               rng=stream_words(env), available=avail, end_position=np.float64(env.end_position))
    return out


def run_seed(env_id: str, over, seed: int, steps: int = T):
    env = make_env(env_id, over)
    pad = slots_of(env.config)
    g = np.random.default_rng(30_000 + seed)
    obs, _ = env.reset(seed=seed)
    first = snapshot(env, obs, pad)
    actions = g.integers(0, 5, size=steps).astype(np.int32)
    flags = np.zeros((steps, 3), dtype=np.bool_)
    min_speed = np.zeros(steps)
    per_step, resets = {}, []
    for t in range(steps):
        obs, reward, terminated, truncated, info = env.step(int(actions[t]))
        flags[t] = terminated, truncated, env.vehicle.crashed
        min_speed[t] = min((abs(float(v.speed)) for v in env.road.vehicles if not v.crashed), default=np.inf)
        if t % STRIDE == STRIDE - 1:
            per_step[t] = dict(snapshot(env, obs, pad), reward=float(reward),
                               terms=np.array([float(info["rewards"][k]) for k in TERMS]))
        if terminated or truncated:
            obs, _ = env.reset()
            resets.append(dict(snapshot(env, obs, pad), step=t))
    return actions, first, flags, per_step, resets, min_speed


def _run(args):
    return run_seed(*args)


def _json(v):
    return json.dumps(v, default=lambda x: x.tolist() if hasattr(x, "tolist") else str(x))


def main(only) -> None:
    from multiprocessing import Pool

    rh._ensure_imports()
    for name, (env_id, over) in CASES.items():
        if only and name not in only:
            continue
        t0 = time.time()
        with Pool(os.cpu_count() or 1) as pool:
            per = pool.map(_run, [(env_id, over, s) for s in SEEDS])
        keep = np.arange(STRIDE - 1, T, STRIDE)
        out = {"seeds": np.array(SEEDS, dtype=np.int64), "actions": np.stack([p[0] for p in per]), "steps": keep,
               "flags": np.stack([p[2] for p in per]), "min_speed": np.stack([p[5] for p in per])}
        keys = list(per[0][1])
        for k in keys:
            out["reset_" + k] = np.stack([np.asarray(p[1][k]) for p in per])
            out[k] = np.stack([np.stack([np.asarray(p[3][t][k]) for t in keep]) for p in per])
        out["reward"] = np.array([[p[3][t]["reward"] for t in keep] for p in per])
        out["terms"] = np.stack([np.stack([p[3][t]["terms"] for t in keep]) for p in per])
        n_res = max(len(p[4]) for p in per)
        assert n_res <= MAX_RESETS, n_res
        out["autoreset_step"] = np.full((len(SEEDS), MAX_RESETS), -1, dtype=np.int64)
        for k in keys:
            proto = np.asarray(per[0][1][k])
            arr = np.zeros((len(SEEDS), MAX_RESETS) + proto.shape, dtype=proto.dtype)
            for i, p in enumerate(per):
                for j, r in enumerate(p[4]):
                    arr[i, j] = r[k]
                    out["autoreset_step"][i, j] = r["step"]
            out["autoreset_" + k] = arr
        env = make_env(env_id, over)
        full = int(env.config["vehicles_count"]) + 3
        counts = np.concatenate([out["reset_count"].ravel(), out["autoreset_count"][out["autoreset_step"] >= 0]])
        if name in SHORT_POPULATIONS:
            assert (counts < full).any(), f"{name}: no reset with a short population"
        if name in MERGING_ON_HIGHWAY:
            assert (out["terms"][..., 4] != 0).any(), f"{name}: no stored step with a merging term"
        cfg = dict(env.config)
        cfg["_env_id"] = env_id
        cfg["_override"] = over or {}
        out["config_json"] = np.array(_json(cfg))
        out["fields"] = np.array(FIELDS)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **out)
        print(f"{name}: {len(SEEDS)} seeds x {T} steps in {time.time() - t0:.0f} s -> {path} "
              f"({os.path.getsize(path) / 1e3:.0f} kB), {int(out['flags'][..., 0].sum())} terminated, "
              f"{int(out['flags'][..., 1].sum())} truncated, {len(counts)} resets, populations "
              f"{int(counts.min())}..{int(counts.max())} of {full}", flush=True)
    if not only:
        for lanes, *lengths in PINNED:
            env = make_env("merge-generic-v0", {"lanes_count": lanes, **dict(zip(LENGTHS, lengths))})
            env.reset(seed=0)
            path = os.path.join(OUT, pinned_name(lanes, *lengths))
            with open(path, "w") as f:
                f.write(_json(env.road.network.to_config()))
            print("->", path)


if __name__ == "__main__":
    if not rh.reference_available():
        raise SystemExit("the reference checkout is not present; the fixtures are generated from it")
    main(sys.argv[1:])
