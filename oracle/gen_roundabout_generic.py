"""Generate the roundabout-generic-v0 / v1 fixtures from the UNMODIFIED Python reference (needs the reference checkout).

    python oracle/gen_roundabout_generic.py [name ...]
    # writes tests/golden/rg_*.npz and pinned_to_config_roundabout_generic_r*_l*.json

For each case, SEEDS x T steps of `RoundaboutGenericEnv` / `ConnectedLaneRoundaboutGenericEnv`
(envs/roundabout_env.py:398-757) under seeded uniform random actions (integers(0, 5) from a generator keyed by the
seed).  When a step ends the episode, `env.reset()` (no seed) starts the next one on the same stream, as a vector
env's autoreset does.  Stored per seed, in the record format of oracle/gen_racetrack_variants.py:

* on every step: terminated, truncated, crashed (`flags`), the action and the smallest |speed| of a vehicle that has
  not crashed after the step (`min_speed`; the steering law divides by the speed, so below ~1 m/s an ulp of
  difference grows past any fixed tolerance: tests/parity_utils.py well_conditioned);
* after the seeded reset (`reset_*`), every STRIDE-th step (`steps`, no prefix) and after each autoreset
  (`autoreset_*`, at most MAX_RESETS, `autoreset_step` -1 past the last): the state in ref_harness.dump_state's
  schema padded to the case's slot stride (8 for vehicles_count <= 7, else 32) with `count` and `kind`, the
  observation, the stream words and get_available_actions() as a mask [5]; on stored steps also the reward and the
  info["rewards"] terms (collision, high_speed, lane_change, on_road).

Cases:
* rg_default: roundabout-generic-v0 at its defaults;
* rg_v1_default: roundabout-generic-v1 (connected-lane neighbour search);
* rg_r5_crowded: radius 5, vehicles_count 7 (arcs shorter than 10 m draw uniform(5, 5); some resets come out short);
* rg_one_lane_r40_grid: one ring lane (24 lanes), radius 40, vehicles_count 7, the OccupancyGrid observation;
* rg_32_slots: radius 30, vehicles_count 20 (32 slots, populations of 19-21);
* rg_dest_ttc: incoming_vehicle_destination -1 (every vehicle to "wxr", no draw), the TimeToCollision observation.

The lane indices are table indices of make_roundabout_generic_network, whose order the pinned to_config files fix.
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
MAX_RESETS = 16
TERMS = ("collision_reward", "high_speed_reward", "lane_change_reward", "on_road_reward")
FIELDS = ("x", "y", "heading", "speed", "target_speed", "timer", "delta", "lane", "target_lane", "crashed", "impact",
          "check_collisions", "speed_index", "route", "route_len", "kind")

CASES = {
    "rg_default": ("roundabout-generic-v0", None),
    "rg_v1_default": ("roundabout-generic-v1", None),
    "rg_r5_crowded": ("roundabout-generic-v0", {"roundabout_radius": 5, "vehicles_count": 7}),
    "rg_one_lane_r40_grid": ("roundabout-generic-v0", {"roundabout_lanes": 1, "roundabout_radius": 40,
                                                       "vehicles_count": 7, "observation": {"type": "OccupancyGrid"}}),
    "rg_32_slots": ("roundabout-generic-v0", {"roundabout_radius": 30, "vehicles_count": 20}),
    "rg_dest_ttc": ("roundabout-generic-v0", {"incoming_vehicle_destination": -1,
                                              "observation": {"type": "TimeToCollision"}}),
}
SHORT_POPULATIONS = ("rg_r5_crowded", "rg_32_slots")  # each must hold at least one reset that skipped a vehicle
# to_config of the reference's road per (roundabout_radius, roundabout_lanes)
PINNED = [(20, 2), (20, 1), (5, 2), (60, 1)]


def pinned_name(radius, lanes) -> str:
    return f"pinned_to_config_roundabout_generic_r{radius}_l{lanes}.json"


def make_env(env_id: str, over):
    rh._ensure_imports()
    from highway_env.envs import roundabout_env as R

    cls = {"roundabout-generic-v0": R.RoundaboutGenericEnv,
           "roundabout-generic-v1": R.ConnectedLaneRoundaboutGenericEnv}[env_id]
    return cls(config=over)


def slots_of(config) -> int:
    return 8 if int(config["vehicles_count"]) <= 7 else 32


def stream_words(env) -> np.ndarray:
    st = env.np_random.bit_generator.state
    m64 = (1 << 64) - 1
    return np.array([st["state"]["state"] >> 64, st["state"]["state"] & m64, st["state"]["inc"] >> 64,
                     st["state"]["inc"] & m64, (int(st["has_uint32"]) << 32) | int(st["uinteger"])], dtype=np.uint64)


def snapshot(env, obs, pad) -> dict:
    d = rh.dump_state(env, pad)
    n = int(d["count"])
    if "route" not in d:  # no vehicle has a route (never: the ego plans one at reset)
        d["route"], d["route_len"] = np.zeros((pad, rh.NET_MAX_ROUTE), np.int32), np.zeros(pad, np.int32)
    kind = np.zeros(pad, dtype=np.int32)
    kind[0] = 1  # the MDPVehicle ego, then IDM traffic
    d["kind"] = kind
    d["route"][n:], d["route_len"][n:] = 0, 0
    out = {k: np.asarray(d[k]) for k in FIELDS}
    avail = np.zeros(5, dtype=np.bool_)
    avail[list(env.get_available_actions())] = True
    out.update(count=np.int32(n), time=np.float64(env.time), obs=np.asarray(obs, dtype=np.float64),
               rng=stream_words(env), available=avail)
    return out


def run_seed(env_id: str, over, seed: int, steps: int = T):
    env = make_env(env_id, over)
    pad = slots_of(env.config)
    g = np.random.default_rng(20_000 + seed)
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
        full = int(env.config["vehicles_count"]) + 1
        counts = np.concatenate([out["reset_count"].ravel(), out["autoreset_count"][out["autoreset_step"] >= 0]])
        if name in SHORT_POPULATIONS:
            assert (counts < full).any(), f"{name}: no reset with a short population"
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
        for radius, lanes in PINNED:
            env = make_env("roundabout-generic-v0", {"roundabout_radius": radius, "roundabout_lanes": lanes})
            env.reset(seed=0)
            path = os.path.join(OUT, pinned_name(radius, lanes))
            with open(path, "w") as f:
                f.write(_json(env.road.network.to_config()))
            print("->", path)


if __name__ == "__main__":
    if not rh.reference_available():
        raise SystemExit("the reference checkout is not present; the fixtures are generated from it")
    main(sys.argv[1:])
