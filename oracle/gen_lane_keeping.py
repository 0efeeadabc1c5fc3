"""Generate the lane-keeping-v0 fixtures from the UNMODIFIED Python reference (needs the reference checkout).

    python oracle/gen_lane_keeping.py [name ...]     # writes tests/golden/lane_keeping_*.npz

For each case, 32 seeds x 420 steps of `LaneKeepingEnv` (envs/lane_keeping_env.py) under the registration's
`TimeLimit(max_episode_steps=200)` (highway_env/__init__.py:89-92), restated here because the env is driven directly:
after the 200th step of an episode `truncated` is True and `env.reset()` (no seed) starts the next episode on the same
stream, as TimeLimit plus a vector env's autoreset do.  420 steps cover two full episodes, both resets and 20 steps of a
third episode.  Actions are float32 draws of U(-1.2, 1.2) from a generator keyed by the seed (values outside [-1, 1]
exercise the action clip).

Stored per seed: the reset observation / vehicle state / lane phase / stream words, and the same after each TimeLimit
reset.  Per step: the lane phase, truncated, and the speed as float32 (enough to tell where the vehicle comes near
zero speed).  Every STRIDE-th step (`steps`, the last step of each block of 20, so both truncation points are among
them): the observation (stacked in attribute order), reward, and the state and stream words after the step, in full
precision.  The stride keeps each fixture a few hundred kB: full-precision floats of all 420 steps would be 2 MB, and a
free-running rollout that drifts shows it at the next stored step.  The stream words of the other steps follow from
the stored ones (every observe draws 4 uniforms per noisy attribute).  The lane phase is 0 while the sine lane is still
queued (`env.lanes` non-empty), 1 after the switch.
"""
from __future__ import annotations

import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_harness as rh  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
SEEDS = list(range(32))
T = 420
MAX_EPISODE_STEPS = 200
STRIDE = 20
_ACTION = {"type": "ContinuousAction", "steering_range": [-np.pi / 3, np.pi / 3], "longitudinal": False,
           "lateral": True, "dynamical": True}

CASES = {
    "lane_keeping_default": None,
    "lane_keeping_pf5": {"policy_frequency": 5},
    "lane_keeping_reference_state": {
        "observation": {"type": "AttributesObservation", "attributes": ["reference_state", "state"]},
        "state_noise": 0.2},
    "lane_keeping_longitudinal": {"action": dict(_ACTION, longitudinal=True)},
}


def stream_words(env) -> np.ndarray:
    st = env.np_random.bit_generator.state
    m64 = (1 << 64) - 1
    return np.array([st["state"]["state"] >> 64, st["state"]["state"] & m64, st["state"]["inc"] >> 64,
                     st["state"]["inc"] & m64, (int(st["has_uint32"]) << 32) | int(st["uinteger"])], dtype=np.uint64)


def snapshot(env, obs) -> tuple:
    """(observation [n_attr, 4, 1], vehicle state [6], lane phase, stream words [5])"""
    o = np.stack([np.asarray(v, dtype=np.float64) for v in obs.values()])
    return o, env.vehicle.state[:, 0].astype(np.float64), int(not env.lanes), stream_words(env)


def run_seed(over, seed: int):
    rh._ensure_imports()
    from highway_env.envs.lane_keeping_env import LaneKeepingEnv

    env = LaneKeepingEnv(config=over)
    size = env.action_space.shape[0]
    actions = np.random.default_rng(10_000 + seed).uniform(-1.2, 1.2, size=(T, size)).astype(np.float32)
    obs, _ = env.reset(seed=seed)
    first = snapshot(env, obs)
    steps = {k: [] for k in ("obs", "state", "phase", "rng")}
    rewards, truncs, resets = [], [], []
    elapsed = 0
    for t in range(T):
        obs, reward, terminated, truncated, info = env.step(actions[t])
        assert not terminated and not truncated and info == {}
        elapsed += 1
        for k, v in zip(steps, snapshot(env, obs)):
            steps[k].append(v)
        rewards.append(float(reward))
        truncs.append(elapsed >= MAX_EPISODE_STEPS)
        if truncs[-1]:
            obs, info = env.reset()
            assert set(info) == {"speed", "crashed", "action"}, info
            resets.append(snapshot(env, obs))
            elapsed = 0
    return env, actions, first, steps, rewards, truncs, resets


def main(only) -> None:
    rh._ensure_imports()
    for name, over in CASES.items():
        if only and name not in only:
            continue
        t0 = time.time()
        per = [run_seed(over, s) for s in SEEDS]
        env = per[0][0]
        out = {"seeds": np.array(SEEDS, dtype=np.int64), "actions": np.stack([p[1] for p in per])}
        keep = np.arange(STRIDE - 1, T, STRIDE)
        out["steps"] = keep
        for j, k in enumerate(("obs", "state", "phase", "rng")):
            out["reset_" + k] = np.stack([p[2][j] for p in per])
            full = np.stack([np.stack(p[3][k]) for p in per])
            out[k] = full.astype(np.uint8) if k == "phase" else full[:, keep]
            if k == "state":
                out["speed"] = full[..., 3].astype(np.float32)
            out["autoreset_" + k] = np.stack([np.stack([r[j] for r in p[6]]) for p in per])
        out["reward"] = np.array([p[4] for p in per], dtype=np.float64)[:, keep]
        out["truncated"] = np.array([p[5] for p in per], dtype=np.bool_)
        out["autoreset_step"] = np.nonzero(out["truncated"][0])[0]
        cfg = {k: v for k, v in env.config.items()}
        cfg["_env_id"] = "lane-keeping-v0"
        cfg["_override"] = over or {}
        out["config_json"] = np.array(json.dumps(cfg))
        out["attributes"] = np.array(list(env.config["observation"]["attributes"]))
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **out)
        print(f"{name}: {len(SEEDS)} seeds x {T} steps in {time.time() - t0:.0f} s -> {path} "
              f"({os.path.getsize(path) / 1e3:.0f} kB)", flush=True)


if __name__ == "__main__":
    if not rh.reference_available():
        raise SystemExit("the reference checkout is not present; the fixtures are generated from it")
    main(sys.argv[1:])
