"""Throughput of multi-agent highway-v0 / highway-fast-v0 (highway_multi_step_kernel) next to the single-agent env at
the same vehicle count, in one process:

    python tools/bench_multi_agent_highway.py [--envs 4096 65536] [--agents 2 4] [--steps 50] [--windows 5]

Each configuration runs MultiAgentAction(DiscreteMetaAction) + MultiAgentObservation(Kinematics) with SameStep
autoreset and random actions; `env.step` is timed with CUDA events over `--windows` windows of `--steps` steps after a
warm-up.  The single-agent env has controlled_vehicles 1 and vehicles_count + A - 1 traffic vehicles, so both step the
same number of vehicles.  Prints the card name and power limit, then one JSON line per configuration with the median
env-steps/s over the windows and their range.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import highwayenv_b200 as hb  # noqa: E402


def rate(env, make_action, steps, windows):
    env.reset(seed=0)
    for _ in range(10):
        env.step(make_action())
    out = []
    for _ in range(windows):
        acts = [make_action() for _ in range(steps)]
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        for a in acts:
            env.step(a)
        end.record()
        end.synchronize()
        out.append(env.num_envs * steps / (start.elapsed_time(end) / 1e3))
    return float(np.median(out)), float(min(out)), float(max(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[4096, 65536])
    ap.add_argument("--agents", type=int, nargs="+", default=[2, 4])
    ap.add_argument("--ids", nargs="+", default=["highway-fast-v0", "highway-v0"])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--windows", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print("card:", card, flush=True)
    for env_id in args.ids:
        count = hb.make(env_id, num_envs=1, device="cuda").config["vehicles_count"]
        for n in args.envs:
            for A in args.agents:
                g = torch.Generator(device="cuda").manual_seed(0)
                cfg = {"controlled_vehicles": A,
                       "action": {"type": "MultiAgentAction", "action_config": {"type": "DiscreteMetaAction"}},
                       "observation": {"type": "MultiAgentObservation", "observation_config": {"type": "Kinematics"}}}
                multi = hb.make(env_id, num_envs=n, config=cfg, device="cuda")
                m = rate(multi, lambda: torch.randint(0, 5, (n, A), device="cuda", dtype=torch.int32, generator=g),
                         args.steps, args.windows)
                del multi
                single = hb.make(env_id, num_envs=n, config={"vehicles_count": count + A - 1}, device="cuda")
                s = rate(single, lambda: torch.randint(0, 5, (n,), device="cuda", dtype=torch.int32, generator=g),
                         args.steps, args.windows)
                del single
                print(json.dumps({"env_id": env_id, "num_envs": n, "agents": A, "vehicles": count + A,
                                  "multi_env_steps_per_s": m[0], "multi_range": m[1:],
                                  "single_env_steps_per_s": s[0], "single_range": s[1:],
                                  "multi_over_single": m[0] / s[0]}), flush=True)
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
