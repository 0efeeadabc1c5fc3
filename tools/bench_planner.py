"""Throughput of the finite-MDP planner (highwayenv_b200.planning) on one GPU, and its closed-loop driving.

    python tools/bench_planner.py [--envs 4096,16384] [--env-ids highway-v0,roundabout-v0] [--reps 20]

Per (env id, num_envs), after a warm-up, CUDA events time `env.to_finite_mdp()`, `planning.value_iteration()`
(gamma 1, 100 iterations, the rl-agents defaults), `policy.act()` and one closed-loop step `env.step(policy.act())`.
The CPU arm is the numpy statement of the same MDPs (tests/finite_mdp_spec.py: the MDP from the device's grid, then
value iteration) on a sample of the envs, per env and extrapolated to the batch.  The closed loop then drives every
env for --horizon steps with the VI policy and, from the same seeds, with a uniform random policy: the mean return of
each env's first episode and the share of first episodes that end in a crash.  Prints one JSON line per case, with
the card's name and power limit (nvidia-smi --query-gpu, read-only).  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # the numbers still carry the torch device name
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({type(e).__name__})"}


def time_ms(fn, reps: int) -> float:
    """Mean device time of fn() over reps calls (CUDA events around the whole window, after one warm-up call)."""
    fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / reps


def closed_loop(env_id: str, n: int, seed: int, horizon: int, policy_kind: str) -> dict:
    import highwayenv_b200 as hb
    from highwayenv_b200 import planning

    env = hb.make(env_id, num_envs=n, autoreset_mode="Disabled")
    env.reset(seed=seed)
    policy = planning.TtcValueIterationPolicy(env) if policy_kind == "vi" else None
    gen = torch.Generator(device=env.device).manual_seed(seed)
    ret = torch.zeros(n, dtype=torch.float64, device=env.device)
    alive = torch.ones(n, dtype=torch.bool, device=env.device)
    crashed = torch.zeros(n, dtype=torch.bool, device=env.device)
    for _ in range(horizon):
        act = policy.act() if policy is not None else torch.randint(0, 5, (n,), generator=gen, device=env.device)
        _, reward, term, trunc, info = env.step(act)
        ret += torch.where(alive, reward, torch.zeros_like(reward))
        crashed |= alive & info["crashed"]
        alive &= ~(term | trunc)
    return {"mean_return": float(ret.mean()), "crash_rate": float(crashed.float().mean())}


def bench_case(env_id: str, n: int, reps: int, cpu_sample: int) -> dict:
    import highwayenv_b200 as hb
    from finite_mdp_spec import mdp_from_grid, value_iteration as np_value_iteration
    from highwayenv_b200 import planning

    env = hb.make(env_id, num_envs=n)
    env.reset(seed=0)
    rng = np.random.default_rng(0)
    for _ in range(3):
        env.step(rng.integers(0, 5, size=n).astype(np.int32))
    mdp = env.to_finite_mdp()
    policy = planning.TtcValueIterationPolicy(env)
    out = {"env_id": env_id, "num_envs": n, "grid_shape": list(mdp.grid.shape[1:]), "reps": reps}
    out["to_finite_mdp_ms"] = time_ms(env.to_finite_mdp, reps)
    out["value_iteration_ms"] = time_ms(lambda: planning.value_iteration(mdp), reps)
    out["policy_act_ms"] = time_ms(policy.act, reps)
    out["act_plus_step_ms"] = time_ms(lambda: env.step(policy.act()), reps)
    out["closed_loop_env_steps_per_s"] = n / (out["act_plus_step_ms"] / 1e3)
    _, done = planning.value_iteration(mdp)
    out["iterations_done_mean"] = float(done.double().mean())
    # CPU arm: the numpy statement on a sample of the same MDPs (taken after the timed steps)
    mdp = env.to_finite_mdp()
    grid, n_lanes = mdp.grid.cpu().numpy(), mdp.n_lanes.cpu().numpy()
    k = min(cpu_sample, n)
    t0 = time.perf_counter()
    for e in range(k):
        g = grid[e][:, :int(n_lanes[e])]
        tr, rw, te = mdp_from_grid(g, env.config)
        np_value_iteration(tr, rw, te, 1.0, 100)
    per_env = (time.perf_counter() - t0) / k
    out["cpu_numpy_per_env_ms"] = per_env * 1e3
    out["cpu_numpy_batch_ms_extrapolated"] = per_env * n * 1e3
    out["cpu_sample_envs"] = k
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", default="4096,16384")
    ap.add_argument("--env-ids", default="highway-v0,roundabout-v0")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cpu-sample", type=int, default=256)
    ap.add_argument("--horizon", type=int, default=40)
    ap.add_argument("--loop-envs", type=int, default=4096)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_planner.py measures the GPU path and needs a CUDA device")
    info = gpu_info()
    for env_id in args.env_ids.split(","):
        for n in (int(x) for x in args.envs.split(",")):
            print(json.dumps({**info, **bench_case(env_id, n, args.reps, args.cpu_sample)}), flush=True)
        row = {**info, "env_id": env_id, "closed_loop_envs": args.loop_envs, "horizon": args.horizon, "seed": 100}
        row["vi"] = closed_loop(env_id, args.loop_envs, 100, args.horizon, "vi")
        row["random"] = closed_loop(env_id, args.loop_envs, 100, args.horizon, "random")
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
