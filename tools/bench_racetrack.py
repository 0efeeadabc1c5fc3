"""racetrack throughput on one GPU, and the reference's per-core rate on a CPU host.

    python tools/bench_racetrack.py [--env-id racetrack-v0] [--envs 65536 1048576] [--steps 200] [--warmup 50]
                                    [--runs 5] [--out r.json]
    python tools/bench_racetrack.py --reference [--seconds 20]     # CPU host with the reference checkout

GPU mode, per env count, on --env-id (racetrack-v0 by default; racetrack-large-v0 / v1 and racetrack-oval-v0 / v1
run the same kernels on their own lane tables), SameStep autoreset, the default configuration (one front vehicle, the 2 x 12 x 12
OccupancyGrid aligned with the vehicle), seeded uniform steering in [-1, 1] staged on the device beforehand (a pool of
16 tensors, cycled):
  * env-steps/s of `env.step` over --steps steps between two CUDA events on the stream, after --warmup steps; the
    median (min, max) of --runs windows.  The windows span the autoresets, which run inside `env.step`;
  * the step kernel alone: the same windows summed over CUDA events around each launch (`env._kernel_events`);
  * the standalone grid kernel alone (`hwy_observe_grid`, which samples the on_road layer on every lane of the table
    for every cell of every env: 18 on racetrack-v0, 27 on the large track, 24 on the default oval): --steps launches on the current state between two CUDA events, and its time as a share of
    the `env.step` window.
The card's name and power limit are read in the same run; with an --env-id other than racetrack-v0 the JSON line
also names it.  Reference mode times `RacetrackEnv.step` of the unmodified
reference on one core (with `reset()` after each terminated episode), the per-core rate a CPU vector env gets.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def bench_gpu(n: int, steps: int, warmup: int, runs: int, env_id: str = "racetrack-v0") -> dict:
    import torch

    import highwayenv_b200 as hb

    env = hb.make(env_id, num_envs=n, autoreset_mode="SameStep")
    env.reset(seed=0)
    gen = torch.Generator(device=env.device).manual_seed(0)
    pool = [torch.rand(n, 1, device=env.device, generator=gen) * 2 - 1 for _ in range(16)]
    for t in range(warmup):
        env.step(pool[t % 16])
    torch.cuda.synchronize()
    rates, kernel_rates, grid_rates, grid_share, k = [], [], [], [], 0
    for _ in range(runs):
        env._kernel_events = []
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(steps):
            env.step(pool[k % 16])
            k += 1
        e.record()
        e.synchronize()
        step_ms = s.elapsed_time(e)
        rates.append(n * steps / (step_ms / 1e3))
        kernel_ms = sum(a.elapsed_time(b) for a, b in env._kernel_events)
        kernel_rates.append(n * steps / (kernel_ms / 1e3))
        env._kernel_events = None
        s.record()
        for _ in range(steps):
            env._observe_plugin(env._obs)
        e.record()
        e.synchronize()
        grid_ms = s.elapsed_time(e)
        grid_rates.append(n * steps / (grid_ms / 1e3))
        grid_share.append(grid_ms / step_ms)
    med = lambda v: (float(np.median(v)), float(np.min(v)), float(np.max(v)))  # noqa: E731
    return {"num_envs": n, "steps": steps, "runs": runs, "env_steps_per_s": med(rates),
            "step_kernel_env_steps_per_s": med(kernel_rates), "grid_kernel_env_steps_per_s": med(grid_rates),
            "grid_share_of_env_step": med(grid_share)}


def bench_reference(seconds: float) -> dict:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import ref_harness as rh

    rh._ensure_imports()
    from highway_env.envs.racetrack_env import RacetrackEnv

    env = RacetrackEnv()
    env.reset(seed=0)
    actions = np.random.default_rng(0).uniform(-1, 1, (1000, 1)).astype(np.float32)
    steps, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        _, _, terminated, truncated, _ = env.step(actions[steps % 1000])
        steps += 1
        if terminated or truncated:
            env.reset()
    return {"reference_env_steps_per_s_one_core": steps / (time.perf_counter() - t0), "steps": steps}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--env-id", default="racetrack-v0", help="GPU mode: the racetrack id to measure")
    ap.add_argument("--envs", type=int, nargs="+", default=[65536, 1048576])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--out")
    args = ap.parse_args()
    if args.reference:
        import platform

        res = {"host": platform.processor() or platform.machine(), **bench_reference(args.seconds)}
    else:
        import torch

        if not torch.cuda.is_available():
            raise SystemExit("no CUDA device: the GPU numbers are measured on the GPU only")
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        from bench_opd import gpu_info

        res = {"gpu": gpu_info(),
               "results": [bench_gpu(n, args.steps, args.warmup, args.runs, args.env_id) for n in args.envs]}
        if args.env_id != "racetrack-v0":
            res["env_id"] = args.env_id
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
