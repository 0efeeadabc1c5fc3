"""MCTS planning throughput and closed-loop quality on one GPU.

    python tools/bench_mcts.py [--roots 1024 4096] [--envs highway-fast-v0 highway-v0] [--out results.json]

Per env id and root count:
  * `MctsPolicy(env, budget=100, gamma=0.7).act()`: ms per call (CUDA events, median of --reps calls after warm-up),
    eager and replayed as one CUDA graph, and decisions/s;
  * a closed loop of --steps steps on the same seeds for MCTS at budgets 50 and 100 (with and without subtree reuse at
    100), OPD at budget 50 and uniform random actions (autoreset disabled; an env's episode ends at its first
    terminated / truncated flag): mean return and crash rate.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import highwayenv_b200 as hb  # noqa: E402
from highwayenv_b200 import planning  # noqa: E402
from tools.bench_opd import gpu_info  # noqa: E402


def _timed(call, reps: int):
    ms = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        call()
        e.record()
        e.synchronize()
        ms.append(s.elapsed_time(e))
    return float(np.median(ms)), float(np.min(ms)), float(np.max(ms))


def time_act(env_id: str, n: int, reps: int, budget: int) -> dict:
    env = hb.make(env_id, num_envs=n)
    env.reset(seed=0)
    policy = planning.MctsPolicy(env, budget=budget, gamma=0.7)
    for _ in range(3):
        policy.act()
    torch.cuda.synchronize()
    launches0 = env._lib.hwy_launch_count()
    policy.act()
    launches = env._lib.hwy_launch_count() - launches0
    eager = _timed(policy.act, reps)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        policy.act()
    graph.replay()
    torch.cuda.synchronize()
    replay = _timed(graph.replay, reps)
    tree_bytes = sum(t.numel() * t.element_size() for t in policy._buffers.values())
    return {"episodes": policy.episodes, "horizon": policy.horizon, "ms_per_act": eager[0],
            "ms_per_act_min_max": eager[1:], "ms_per_act_graph": replay[0], "ms_per_act_graph_min_max": replay[1:],
            "decisions_per_s": n / (eager[0] / 1e3), "decisions_per_s_graph": n / (replay[0] / 1e3),
            "library_launches_per_act": int(launches), "tree_bytes": tree_bytes}


def closed_loop(env_id: str, n: int, steps: int, kind: str, seed: int) -> dict:
    env = hb.make(env_id, num_envs=n, autoreset_mode="Disabled")
    env.reset(seed=seed)
    policy = None
    if kind.startswith("mcts"):
        budget = int(kind.split("_")[1])
        policy = planning.MctsPolicy(env, budget=budget, gamma=0.7, seed=seed, reuse_subtree=kind.endswith("reuse"))
        act = policy.act
    elif kind == "opd_50":
        act = planning.OpdPolicy(env, budget=50, gamma=0.7).act
    else:
        gen = torch.Generator(device=env.device)
        gen.manual_seed(seed)
        act = lambda: torch.randint(0, 5, (n,), device=env.device, generator=gen, dtype=torch.int32)  # noqa: E731
    ret = torch.zeros(n, dtype=torch.float64, device=env.device)
    crashed = torch.zeros(n, dtype=torch.bool, device=env.device)
    alive = torch.ones(n, dtype=torch.bool, device=env.device)
    for _ in range(steps):
        a = act()
        _, r, term, trunc, info = env.step(a)
        if policy is not None:
            policy.advance(a, term | trunc)
        ret += torch.where(alive, r, 0.0)
        crashed |= info["crashed"] & alive
        alive &= ~(term | trunc)
    return {"mean_return": float(ret.mean()), "crash_rate": float(crashed.float().mean())}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--roots", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--envs", nargs="+", default=["highway-fast-v0", "highway-v0"])
    ap.add_argument("--budget", type=int, default=100)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--loop-roots", type=int, default=1024)
    ap.add_argument("--loops", nargs="+", default=["mcts_50", "mcts_100", "mcts_100_reuse", "opd_50", "random"])
    ap.add_argument("--out", default="", help="also write the JSON result to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mcts needs a CUDA device")
    result = {"gpu": gpu_info(), "budget": args.budget, "act": {}, "loop": {}}
    for env_id in args.envs:
        for n in args.roots:
            r = time_act(env_id, n, args.reps, args.budget)
            result["act"][f"{env_id} x {n}"] = r
            print(f"{env_id} x {n}: {r['ms_per_act']:.2f} ms/act eager, {r['ms_per_act_graph']:.2f} ms graph, "
                  f"{r['decisions_per_s_graph']:.0f} decisions/s", flush=True)
            torch.cuda.empty_cache()
        for kind in args.loops:
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
