"""OPD planning throughput and closed-loop quality on one GPU.

    python tools/bench_opd.py [--roots 1024 4096] [--envs highway-fast-v0 highway-v0] [--out results.json]

Per env id and root count:
  * `OpdPolicy(env, budget=50, gamma=0.7).act()` (the reference quickstart's planner configuration): ms per call
    (CUDA events, median of --reps calls after warm-up), eager and replayed as one CUDA graph, and decisions/s;
  * a closed loop of --steps steps on the same seeds for OPD, `TtcValueIterationPolicy` and uniform random actions
    (autoreset disabled; an env's episode ends at its first terminated / truncated flag): mean return and crash rate.
The reference for comparison: 1.37 s per highway-fast-v0 decision (50 x deepcopy + step) on one CPU core.
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
from highwayenv_b200 import planning  # noqa: E402

REFERENCE_S_PER_DECISION = 1.37  # unmodified reference, highway-fast-v0, one CPU core


def gpu_info() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        info["power_limit, max_sm_clock"] = out[0] if out else "unavailable"
    except (OSError, subprocess.SubprocessError):
        info["power_limit, max_sm_clock"] = "unavailable"
    return info


def time_act(env_id: str, n: int, reps: int) -> dict:
    env = hb.make(env_id, num_envs=n)
    env.reset(seed=0)
    policy = planning.OpdPolicy(env, budget=50, gamma=0.7)
    for _ in range(3):
        policy.act()
    torch.cuda.synchronize()

    def timed(call):
        ms = []
        for _ in range(reps):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            call()
            e.record()
            e.synchronize()
            ms.append(s.elapsed_time(e))
        return float(np.median(ms)), float(np.min(ms)), float(np.max(ms))

    eager = timed(policy.act)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        policy.act()
    graph.replay()
    torch.cuda.synchronize()
    replay = timed(graph.replay)
    store_bytes = sum(t.numel() * t.element_size() for t in policy.store._env_rows().values())
    return {"ms_per_act": eager[0], "ms_per_act_min_max": eager[1:], "ms_per_act_graph": replay[0],
            "ms_per_act_graph_min_max": replay[1:], "decisions_per_s": n / (eager[0] / 1e3),
            "decisions_per_s_graph": n / (replay[0] / 1e3), "store_state_bytes": store_bytes,
            "store_envs": policy.store.num_envs, "speedup_vs_reference_one_core":
                REFERENCE_S_PER_DECISION * n / (replay[0] / 1e3)}


def closed_loop(env_id: str, n: int, steps: int, kind: str, seed: int) -> dict:
    env = hb.make(env_id, num_envs=n, autoreset_mode="Disabled")
    env.reset(seed=seed)
    if kind == "opd":
        act = planning.OpdPolicy(env, budget=50, gamma=0.7).act
    elif kind == "ttc_vi":
        act = planning.TtcValueIterationPolicy(env).act
    else:
        gen = torch.Generator(device=env.device)
        gen.manual_seed(seed)
        act = lambda: torch.randint(0, 5, (n,), device=env.device, generator=gen, dtype=torch.int32)  # noqa: E731
    ret = torch.zeros(n, dtype=torch.float64, device=env.device)
    crashed = torch.zeros(n, dtype=torch.bool, device=env.device)
    alive = torch.ones(n, dtype=torch.bool, device=env.device)
    for _ in range(steps):
        _, r, term, trunc, info = env.step(act())
        ret += torch.where(alive, r, 0.0)
        crashed |= info["crashed"] & alive
        alive &= ~(term | trunc)
    return {"mean_return": float(ret.mean()), "crash_rate": float(crashed.float().mean())}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--roots", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--envs", nargs="+", default=["highway-fast-v0", "highway-v0"])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--loop-roots", type=int, default=1024)
    ap.add_argument("--out", default="", help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_opd needs a CUDA device")
    result = {"gpu": gpu_info(), "reference_s_per_decision_one_core": REFERENCE_S_PER_DECISION, "act": {}, "loop": {}}
    for env_id in args.envs:
        for n in args.roots:
            r = time_act(env_id, n, args.reps)
            result["act"][f"{env_id} x {n}"] = r
            print(f"{env_id} x {n}: {r['ms_per_act']:.2f} ms/act eager, {r['ms_per_act_graph']:.2f} ms graph, "
                  f"{r['decisions_per_s_graph']:.0f} decisions/s", flush=True)
            torch.cuda.empty_cache()
        for kind in ("opd", "ttc_vi", "random"):
            r = closed_loop(env_id, args.loop_roots, args.steps, kind, seed=2024)
            result["loop"][f"{env_id} {kind}"] = r
            print(f"{env_id} {kind}: return {r['mean_return']:.3f}, crash rate {r['crash_rate']:.3f}", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
