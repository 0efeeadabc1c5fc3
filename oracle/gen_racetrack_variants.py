"""Generate the racetrack-large / racetrack-oval fixtures from the UNMODIFIED Python reference (needs the reference
checkout).

    python oracle/gen_racetrack_variants.py [name ...]
    # writes tests/golden/racetrack_{large,oval}_*.npz and pinned_to_config_racetrack_{large,oval}_v0*.json

The same recording as oracle/gen_racetrack.py (its state schema, stream words and lane-following controller), on
`RacetrackEnvLarge` / `ConnectedLaneRacetrackEnvLarge` (envs/racetrack_env.py:432-880) and `RacetrackEnvOval` /
`ConnectedLaneRacetrackEnvOval` (:882-1396): 32 seeds x 200 steps per case, flags on every step, and the full state,
stream words, observation and reward every STRIDE-th step and after each reset.  When a step ends the episode,
`env.reset()` (no seed) starts the next one on the same stream, as a vector env's autoreset does.

* racetrack_large_random: large-v0, steering U(-1.2, 1.2);
* racetrack_large_follow: large-v0, the lane-following controller;
* racetrack_large_traffic: large-v0, other_vehicles 6, longitudinal control (throttle U(-0.5, 0.7)), the controller;
* racetrack_large_v1_follow: large-v1, the controller;
* racetrack_large_speed15: large-v0 with speed_limit 15 (every lane's limit, so the ego's spawn speed), the controller;
* racetrack_oval_follow: oval-v0 at its defaults (length 100, no_lanes 3), the controller;
* racetrack_oval_lanes2: oval-v0 with no_lanes 2 and length 150, the controller;
* racetrack_oval_v1_lanes4: oval-v1 with no_lanes 4, other_vehicles 6 and the Kinematics observation, the controller.

The lane indices of the state are table indices of this repository's lane table of the same track
(make_racetrack_large_network / make_racetrack_oval_network), whose order the pinned to_config files fix.
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
import gen_racetrack as gr  # noqa: E402
import ref_harness as rh  # noqa: E402

OUT = gr.OUT
SEEDS, T, STRIDE, MAX_RESETS = gr.SEEDS, gr.T, gr.STRIDE, gr.MAX_RESETS

_TRAFFIC = {"other_vehicles": 6, "action": {"type": "ContinuousAction", "longitudinal": True, "lateral": True,
                                            "target_speeds": [0, 5, 10]}}
CASES = {
    "racetrack_large_random": ("racetrack-large-v0", None, "random"),
    "racetrack_large_follow": ("racetrack-large-v0", None, "follow"),
    "racetrack_large_traffic": ("racetrack-large-v0", _TRAFFIC, "follow"),
    "racetrack_large_v1_follow": ("racetrack-large-v1", None, "follow"),
    "racetrack_large_speed15": ("racetrack-large-v0", {"speed_limit": 15}, "follow"),
    "racetrack_oval_follow": ("racetrack-oval-v0", None, "follow"),
    "racetrack_oval_lanes2": ("racetrack-oval-v0", {"no_lanes": 2, "length": 150}, "follow"),
    "racetrack_oval_v1_lanes4": ("racetrack-oval-v1", {"no_lanes": 4, "other_vehicles": 6,
                                                       "observation": {"type": "Kinematics"}}, "follow"),
}
# to_config of the reference's road, pinned per track: file name -> (env id, config override)
PINNED = {
    "pinned_to_config_racetrack_large_v0.json": ("racetrack-large-v0", None),
    "pinned_to_config_racetrack_oval_v0.json": ("racetrack-oval-v0", None),
    "pinned_to_config_racetrack_oval_v0_lanes2.json": ("racetrack-oval-v0", {"no_lanes": 2}),
    "pinned_to_config_racetrack_oval_v0_lanes4.json": ("racetrack-oval-v0", {"no_lanes": 4}),
}


def make_env(env_id: str, over):
    rh._ensure_imports()
    from highway_env.envs import racetrack_env as R

    cls = {"racetrack-large-v0": R.RacetrackEnvLarge, "racetrack-large-v1": R.ConnectedLaneRacetrackEnvLarge,
           "racetrack-oval-v0": R.RacetrackEnvOval, "racetrack-oval-v1": R.ConnectedLaneRacetrackEnvOval}[env_id]
    return cls(config=over)


def our_network(env_id: str, config: dict):
    from highwayenv_b200.envs.racetrack_env import track_network

    return track_network(env_id, config)


def run_seed(env_id: str, over, policy: str, seed: int, steps: int = T):
    env = make_env(env_id, over)
    net = our_network(env_id, env.config)
    size = env.action_space.shape[0]
    g = np.random.default_rng(20_000 + seed)
    obs, _ = env.reset(seed=seed)
    snap = lambda o: dict(gr.state(env, net), obs=np.asarray(o, dtype=np.float64), rng=gr.stream_words(env))  # noqa: E731
    first = snap(obs)
    actions = np.zeros((steps, size), dtype=np.float32)
    flags = np.zeros((steps, 3), dtype=np.bool_)
    per_step, resets = [], []
    for t in range(steps):
        if policy == "random":
            a = g.uniform(-1.2, 1.2, size=size)
        else:
            steer = np.clip(gr.follow_steering(env) + 0.1 * g.normal(), -1.2, 1.2)
            a = np.array([g.uniform(-0.5, 0.7), steer] if size == 2 else [steer])
        actions[t] = a.astype(np.float32)
        obs, reward, terminated, truncated, info = env.step(actions[t])
        flags[t] = terminated, truncated, env.vehicle.crashed
        terms = np.array([float(info["rewards"][k]) for k in ("lane_centering_reward", "action_reward",
                                                             "collision_reward", "on_road_reward")])
        per_step.append(dict(snap(obs), reward=float(reward), terms=terms))
        if terminated or truncated:
            obs, _ = env.reset()
            resets.append(dict(snap(obs), step=t))
    return env, actions, first, flags, per_step, resets


def _run(args):
    return (None,) + run_seed(*args)[1:]


def _json(v):
    return json.dumps(v, default=lambda x: x.tolist() if hasattr(x, "tolist") else str(x))


def main(only) -> None:
    from multiprocessing import Pool

    rh._ensure_imports()
    for name, (env_id, over, policy) in CASES.items():
        if only and name not in only:
            continue
        t0 = time.time()
        with Pool(min(8, os.cpu_count() or 1)) as pool:
            per = pool.map(_run, [(env_id, over, policy, s) for s in SEEDS])
        keep = np.arange(STRIDE - 1, T, STRIDE)
        out = {"seeds": np.array(SEEDS, dtype=np.int64), "actions": np.stack([p[1] for p in per]), "steps": keep,
               "flags": np.stack([p[3] for p in per])}
        for k in ("state", "count", "obs", "rng"):
            out["reset_" + k] = np.stack([np.asarray(p[2][k]) for p in per])
        for k in ("state", "count", "obs", "rng", "impact", "has_impact", "time"):
            out[k] = np.stack([np.stack([np.asarray(p[4][t][k]) for t in keep]) for p in per])
        out["reward"] = np.array([[p[4][t]["reward"] for t in keep] for p in per])
        out["terms"] = np.stack([np.stack([p[4][t]["terms"] for t in keep]) for p in per])
        n_res = max(len(p[5]) for p in per)
        assert n_res <= MAX_RESETS, n_res
        out["autoreset_step"] = np.full((len(SEEDS), MAX_RESETS), -1, dtype=np.int64)
        for k in ("state", "count", "obs", "rng"):
            proto = np.asarray(per[0][2][k])
            arr = np.zeros((len(SEEDS), MAX_RESETS) + proto.shape, dtype=proto.dtype)
            for i, p in enumerate(per):
                for j, r in enumerate(p[5]):
                    arr[i, j] = r[k]
                    out["autoreset_step"][i, j] = r["step"]
            out["autoreset_" + k] = arr
        env = make_env(env_id, over)
        cfg = {k: v for k, v in env.config.items()}
        cfg["_env_id"] = env_id
        cfg["_override"] = over or {}
        cfg["_policy"] = policy
        out["config_json"] = np.array(_json(cfg))
        out["fields"] = np.array(gr.FIELDS)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **out)
        print(f"{name}: {len(SEEDS)} seeds x {T} steps in {time.time() - t0:.0f} s -> {path} "
              f"({os.path.getsize(path) / 1e3:.0f} kB), {int(out['flags'][..., 0].sum())} terminated, "
              f"{int(out['flags'][..., 1].sum())} truncated, {int((out['autoreset_step'] >= 0).sum())} resets",
              flush=True)
    if not only:
        for fname, (env_id, over) in PINNED.items():
            env = make_env(env_id, over)
            env.reset(seed=0)
            path = os.path.join(OUT, fname)
            with open(path, "w") as f:
                f.write(_json(env.road.network.to_config()))
            print("->", path)


if __name__ == "__main__":
    if not rh.reference_available():
        raise SystemExit("the reference checkout is not present; the fixtures are generated from it")
    main(sys.argv[1:])
