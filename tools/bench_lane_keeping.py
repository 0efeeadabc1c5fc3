"""lane-keeping-v0 throughput on one GPU, and the reference's per-core rate on a CPU host.

    python tools/bench_lane_keeping.py [--envs 65536 1048576] [--steps 200] [--warmup 50] [--runs 5] [--out r.json]
    python tools/bench_lane_keeping.py --reference [--seconds 20]     # CPU host with the reference checkout

GPU mode, per env count, SameStep autoreset, the default configuration, seeded uniform actions in [-1, 1] staged on
the device beforehand (a pool of 16 tensors, cycled):
  * env-steps/s of `env.step` over --steps steps between two CUDA events on the stream, after --warmup steps; the
    median (min, max) of --runs windows.  The windows span TimeLimit resets, which run inside the step kernel;
  * the step kernel alone: the same windows summed over CUDA events around each launch (`env._kernel_events`);
  * end to end through `env.host_stepper()`: numpy actions in, numpy results out, one CUDA graph and one stream sync
    per step, host clock.
The card's name and power limit are read in the same run.  Reference mode times `LaneKeepingEnv.step` of the unmodified
reference on one core (with the TimeLimit reset every 200 steps), which is the per-core rate a CPU vector env gets.
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


def bench_gpu(n: int, steps: int, warmup: int, runs: int) -> dict:
    import torch

    import highwayenv_b200 as hb

    env = hb.make("lane-keeping-v0", num_envs=n, autoreset_mode="SameStep")
    env.reset(seed=0)
    gen = torch.Generator(device=env.device).manual_seed(0)
    pool = [torch.rand(n, 1, device=env.device, generator=gen) * 2 - 1 for _ in range(16)]
    for t in range(warmup):
        env.step(pool[t % 16])
    torch.cuda.synchronize()
    rates, kernel_rates, k = [], [], 0
    for _ in range(runs):
        env._kernel_events = []
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(steps):
            env.step(pool[k % 16])
            k += 1
        e.record()
        e.synchronize()
        rates.append(n * steps / (s.elapsed_time(e) / 1e3))
        kernel_ms = sum(a.elapsed_time(b) for a, b in env._kernel_events)
        kernel_rates.append(n * steps / (kernel_ms / 1e3))
    env._kernel_events = None
    hs = env.host_stepper()
    rng = np.random.default_rng(0)
    host_actions = [rng.uniform(-1, 1, (n, 1)).astype(np.float32) for _ in range(4)]
    for t in range(warmup):
        hs.actions[:] = host_actions[t % 4]
        hs.step()
    host_rates = []
    for _ in range(runs):
        t0 = time.perf_counter()
        for t in range(steps):
            hs.actions[:] = host_actions[t % 4]
            hs.step()
        host_rates.append(n * steps / (time.perf_counter() - t0))
    med = lambda v: (float(np.median(v)), float(np.min(v)), float(np.max(v)))  # noqa: E731
    return {"num_envs": n, "steps": steps, "runs": runs, "env_steps_per_s": med(rates),
            "kernel_env_steps_per_s": med(kernel_rates), "host_stepper_env_steps_per_s": med(host_rates)}


def bench_reference(seconds: float) -> dict:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import ref_harness as rh

    rh._ensure_imports()
    from highway_env.envs.lane_keeping_env import LaneKeepingEnv

    env = LaneKeepingEnv()
    env.reset(seed=0)
    actions = np.random.default_rng(0).uniform(-1, 1, (1000, 1)).astype(np.float32)
    steps, elapsed, t0 = 0, 0, time.perf_counter()
    while time.perf_counter() - t0 < seconds:
        env.step(actions[steps % 1000])
        steps += 1
        elapsed += 1
        if elapsed == 200:
            env.reset()
            elapsed = 0
    return {"reference_env_steps_per_s_one_core": steps / (time.perf_counter() - t0), "steps": steps}


def main() -> None:
    ap = argparse.ArgumentParser()
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

        res = {"gpu": gpu_info(), "results": [bench_gpu(n, args.steps, args.warmup, args.runs) for n in args.envs]}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
