"""merge-generic-v0 throughput on one GPU, with merge-v0 in the same run for comparison.

    python tools/bench_merge_generic.py [--steps 100] [--warmup 20] [--runs 5] [--out r.json]

Per workload, SameStep autoreset and seeded uniform random DiscreteMetaAction labels staged on the device beforehand
(a pool of 16 tensors, cycled):
  * merge-generic-v0 at its defaults (2 lanes, 3 traffic vehicles, 8 slots) at 65 536 and 1 048 576 envs;
  * merge-generic-v0 with lanes_count 4 and vehicles_count 20 (32 slots) at 65 536 envs;
  * merge-v0 at 65 536 and 1 048 576 envs.
Reported: env-steps/s of `env.step` over --steps steps between two CUDA events on the stream, after --warmup steps, as
the median (min, max) of --runs windows (the windows span the autoresets, which run inside `env.step`), and the reset
kernel alone: --steps masked resets of every env, between two CUDA events.  The card's name and power limit are read in
the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = [("merge-generic-v0", None, 65536), ("merge-generic-v0", None, 1048576),
             ("merge-generic-v0", {"lanes_count": 4, "vehicles_count": 20}, 65536),
             ("merge-v0", None, 65536), ("merge-v0", None, 1048576)]


def bench_gpu(env_id: str, over, n: int, steps: int, warmup: int, runs: int) -> dict:
    import torch

    import highwayenv_b200 as hb

    env = hb.make(env_id, num_envs=n, config=over, autoreset_mode="SameStep")
    env.reset(seed=0)
    gen = torch.Generator(device=env.device).manual_seed(0)
    pool = [torch.randint(0, 5, (n,), device=env.device, generator=gen, dtype=torch.int32) for _ in range(16)]
    for t in range(warmup):
        env.step(pool[t % 16])
    torch.cuda.synchronize()
    rates, reset_rates, k = [], [], 0
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(runs):
        s.record()
        for _ in range(steps):
            env.step(pool[k % 16])
            k += 1
        e.record()
        e.synchronize()
        rates.append(n * steps / (s.elapsed_time(e) / 1e3))
        s.record()
        for _ in range(steps):
            env._device_reset(None, None, None)
        e.record()
        e.synchronize()
        reset_rates.append(n * steps / (s.elapsed_time(e) / 1e3))
    med = lambda v: (float(np.median(v)), float(np.min(v)), float(np.max(v)))  # noqa: E731
    out = {"env_id": env_id, "config": over or {}, "num_envs": n, "slots": env.vp, "steps": steps, "runs": runs,
           "env_steps_per_s": med(rates), "reset_kernel_env_resets_per_s": med(reset_rates)}
    del env
    torch.cuda.empty_cache()
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the GPU numbers are measured on the GPU only")
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from bench_opd import gpu_info

    res = {"gpu": gpu_info(),
           "results": [bench_gpu(i, o, n, args.steps, args.warmup, args.runs) for i, o, n in WORKLOADS]}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
