"""Env-steps/s of the highway step kernel with IDMVehicle traffic and with each linear traffic class, on one GPU.

    python tools/bench_linear_traffic.py [--envs 4096] [--steps 50] [--warmup 5] [--reps 3]

Cases: highway-fast-v0 with 50 vehicles (V = 51, 64 threads per env) and highway-v0 with 100 vehicles (V = 101, 128
threads per env), DiscreteMetaAction, SameStep autoreset, a fixed random action batch on the device.  Per (case,
traffic class) CUDA events time --steps env.step calls after --warmup, --reps times, interleaving the classes so that
clock drift hits all of them alike; the median is reported.  Prints one JSON line per case with the card's name and
power limit (nvidia-smi --query-gpu, read-only).  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

B = "highway_env.vehicle.behavior."
TRAFFIC = ("IDMVehicle", "LinearVehicle", "AggressiveVehicle", "DefensiveVehicle")
CASES = (("highway-fast-v0", 50), ("highway-v0", 100))


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return {"gpu": name, "power_limit": power}
    except Exception as e:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({type(e).__name__})"}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import highwayenv_b200 as hb

    info = gpu_info()
    n = args.envs
    for env_id, vehicles in CASES:
        envs = {}
        for cls in TRAFFIC:
            env = hb.make(env_id, num_envs=n, config={"vehicles_count": vehicles, "other_vehicles_type": B + cls})
            env.reset(seed=0)
            envs[cls] = env
        act = torch.randint(0, 5, (n,), dtype=torch.int32, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
        times = {cls: [] for cls in TRAFFIC}
        for _ in range(args.reps):
            for cls, env in envs.items():
                for _ in range(args.warmup):
                    env.step(act)
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                start.record()
                for _ in range(args.steps):
                    env.step(act)
                end.record()
                end.synchronize()
                times[cls].append(start.elapsed_time(end) / 1e3)
        rate = {cls: n * args.steps / statistics.median(t) for cls, t in times.items()}
        line = {"env_id": env_id, "vehicles": vehicles + 1, "num_envs": n, "steps": args.steps, "reps": args.reps,
                "env_steps_per_s": {cls: round(r) for cls, r in rate.items()},
                "relative_to_idm": {cls: round(r / rate["IDMVehicle"], 3) for cls, r in rate.items()},
                "spread": {cls: round((max(t) - min(t)) / statistics.median(t), 3) for cls, t in times.items()}}
        line.update(info)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
