"""Generate the racetrack-v0 / racetrack-v1 fixtures from the UNMODIFIED Python reference (needs the reference checkout).

    python oracle/gen_racetrack.py [name ...]     # writes tests/golden/racetrack_*.npz and pinned_to_config_racetrack_v0.json

For each case, 32 seeds x 200 steps of `RacetrackEnv` / `ConnectedLaneRacetrackEnv` (envs/racetrack_env.py).  When a
step ends the episode (terminated or truncated), `env.reset()` (no seed) starts the next one on the same stream, as a
vector env's autoreset does.  Actions are float32 and are stored:

* racetrack_random: default config, steering U(-1.2, 1.2) from a generator keyed by the seed (short episodes that end
  off the road; values outside [-1, 1] exercise the clip);
* racetrack_follow: default config, a lane-following steering controller computed here from the reference's state plus
  a little noise, so that episodes lap the track (every arc, the front vehicle's lane changes, rear-end contacts);
* racetrack_traffic: other_vehicles 6, longitudinal control (throttle U(-0.5, 0.7)), duration 20 s, the controller
  steering: truncations and resets with up to 6 vehicles;
* racetrack_v1_follow: racetrack-v1 with racetrack_follow's controller;
* racetrack_kinematics: other_vehicles 6 with the Kinematics observation (the step kernel's own observation) and the
  controller.

Stored per seed: the reset state / observation / stream words and the same after each autoreset (at most MAX_RESETS,
zero-padded, `autoreset_step` -1); per step: terminated, truncated, crashed; every STRIDE-th step (`steps`) and after each reset: the
observation, reward, reward terms, the full state, the pending impacts (`impact` [2, 8], `has_impact` [8]: a
will-intersect transition that the vehicle's next step applies), the clock and the stream words in full precision, so
that a test can restart the simulation from any stored step.  The state is in this
repository's slot schema (include/hwyb200.h): slot 0 is the plain ego with its persisting action in
(target_speed, timer); `lane` / `target_lane` are table indices of the lane table (graph enumeration order).
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
T = 200
STRIDE = 10
MAX_RESETS = 40
SLOTS = 8
FIELDS = ("x", "y", "heading", "speed", "target_speed", "timer", "lane", "target_lane", "kind", "crashed")

CASES = {
    "racetrack_random": ("racetrack-v0", None, "random"),
    "racetrack_follow": ("racetrack-v0", None, "follow"),
    "racetrack_traffic": ("racetrack-v0", {"other_vehicles": 6, "duration": 20,
                                           "action": {"type": "ContinuousAction", "longitudinal": True,
                                                      "lateral": True, "target_speeds": [0, 5, 10]}}, "follow"),
    "racetrack_v1_follow": ("racetrack-v1", None, "follow"),
    "racetrack_kinematics": ("racetrack-v0", {"other_vehicles": 6, "observation": {"type": "Kinematics"}}, "follow"),
}


def stream_words(env) -> np.ndarray:
    st = env.np_random.bit_generator.state
    m64 = (1 << 64) - 1
    return np.array([st["state"]["state"] >> 64, st["state"]["state"] & m64, st["state"]["inc"] >> 64,
                     st["state"]["inc"] & m64, (int(st["has_uint32"]) << 32) | int(st["uinteger"])], dtype=np.uint64)


def _net():
    from highwayenv_b200.envs.racetrack_env import make_racetrack_network

    return make_racetrack_network()


def state(env, net) -> dict:
    """The road's vehicles in slot order (the ego first, as in the reference's list)."""
    from highway_env.vehicle.behavior import IDMVehicle

    out = {k: np.zeros(SLOTS, dtype=np.float64) for k in FIELDS}
    impact, has_impact = np.zeros((2, SLOTS)), np.zeros(SLOTS, dtype=np.bool_)
    vs = env.road.vehicles
    assert len(vs) <= SLOTS and vs[0] is env.vehicle
    for k, v in enumerate(vs):
        out["x"][k], out["y"][k] = v.position
        out["heading"][k], out["speed"][k] = v.heading, v.speed
        out["lane"][k] = net.index[(v.lane_index[0], v.lane_index[1], int(v.lane_index[2]))]
        out["crashed"][k] = float(v.crashed)
        if v.impact is not None:
            impact[:, k], has_impact[k] = v.impact, True
        if isinstance(v, IDMVehicle):
            t = v.target_lane_index
            out["target_lane"][k] = net.index[(t[0], t[1], int(t[2]))]
            out["target_speed"][k], out["timer"][k] = v.target_speed, v.timer
        else:
            out["target_lane"][k] = out["lane"][k]
            out["target_speed"][k], out["timer"][k] = v.action["acceleration"], v.action["steering"]
            out["kind"][k] = 2.0
    return {"state": np.stack([out[k] for k in FIELDS]), "count": len(vs), "impact": impact, "has_impact": has_impact,
            "time": float(env.time)}


def follow_steering(env) -> float:
    """A lane-following steering command in [-1, 1] units of the steering range: heading error to the lane 4 m ahead
    and the lateral offset on the vehicle's current lane."""
    from highway_env import utils

    v = env.vehicle
    s, lat = v.lane.local_coordinates(v.position)
    err = utils.wrap_to_pi(v.lane.heading_at(s + 4.0) - v.heading)
    return (1.2 * err - 0.25 * lat) / (np.pi / 4)


def make_env(env_id: str, over):
    rh._ensure_imports()
    from highway_env.envs.racetrack_env import ConnectedLaneRacetrackEnv, RacetrackEnv

    return (ConnectedLaneRacetrackEnv if env_id == "racetrack-v1" else RacetrackEnv)(config=over)


def run_seed(env_id: str, over, policy: str, seed: int, steps: int = T):
    net = _net()
    env = make_env(env_id, over)
    size = env.action_space.shape[0]
    g = np.random.default_rng(20_000 + seed)
    obs, _ = env.reset(seed=seed)
    snap = lambda o: dict(state(env, net), obs=np.asarray(o, dtype=np.float64), rng=stream_words(env))  # noqa: E731
    first = snap(obs)
    actions = np.zeros((steps, size), dtype=np.float32)
    flags = np.zeros((steps, 3), dtype=np.bool_)
    per_step, resets = [], []
    for t in range(steps):
        if policy == "random":
            a = g.uniform(-1.2, 1.2, size=size)
        else:
            steer = np.clip(follow_steering(env) + 0.1 * g.normal(), -1.2, 1.2)
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
        out["config_json"] = np.array(json.dumps(cfg, default=lambda v: v.tolist() if hasattr(v, "tolist") else str(v)))
        out["fields"] = np.array(FIELDS)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **out)
        print(f"{name}: {len(SEEDS)} seeds x {T} steps in {time.time() - t0:.0f} s -> {path} "
              f"({os.path.getsize(path) / 1e3:.0f} kB), {int(out['flags'][..., 0].sum())} terminated, "
              f"{int(out['flags'][..., 1].sum())} truncated", flush=True)
    if not only:
        env = make_env("racetrack-v0", None)
        env.reset(seed=0)
        path = os.path.join(OUT, "pinned_to_config_racetrack_v0.json")
        with open(path, "w") as f:
            json.dump(env.road.network.to_config(), f, default=lambda v: v.tolist() if hasattr(v, "tolist") else str(v))
        print("->", path)


if __name__ == "__main__":
    if not rh.reference_available():
        raise SystemExit("the reference checkout is not present; the fixtures are generated from it")
    main(sys.argv[1:])
