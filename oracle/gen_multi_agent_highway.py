"""Generate the multi-agent highway fixtures from the UNMODIFIED Python reference (needs the reference checkout).

    python oracle/gen_multi_agent_highway.py [name ...]     # writes tests/golden/multi_highway_*.npz

Each step case resets `SEEDS` seeds and applies `T` seeded random actions with `ref_harness.rollout` (stepping goes on
after a termination, as the reference allows).  MultiAgentAction takes a tuple: integer actions [A] become a tuple of
ints in `rollout`, ContinuousAction actions are passed here as a tuple of float32 [2] arrays.

* multi_highway_v0_a2: highway-v0, A = 2, MultiAgentAction(DiscreteMetaAction) + MultiAgentObservation(Kinematics);
* multi_highway_fast_a3: highway-fast-v0, A = 3, both switches on (the controlled vehicles collide with each other);
* multi_highway_fast_plain_action: highway-fast-v0, A = 2, plain DiscreteMetaAction + MultiAgentObservation (the
  second controlled vehicle acts as act(None));
* multi_highway_v0_continuous: highway-v0, vehicles_count 40, A = 4, MultiAgentAction(ContinuousAction) + plain
  Kinematics;
* multi_highway_fast_ttc: highway-fast-v0, A = 2, MultiAgentAction(DiscreteMetaAction) +
  MultiAgentObservation(TimeToCollision);
* multi_highway_resets: reset only, 8 configurations of (A, vehicles_count, initial_lane_id) x 8 seeds, including
  A = 8 and vehicles_count < A (empty near_split bins).

Stored per step case, stacked over seeds [S, T + 1, ...] (index 0 = the reset): the per-vehicle state of
`ref_harness.dump_state` (list order), the stream words, the observation; per step [S, T]: actions, reward,
terminated, truncated.  The reset case stores one group per configuration, `c{k}_*`, with the same state fields.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_harness as rh  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
FIELDS = ("x", "y", "heading", "speed", "target_speed", "timer", "delta", "lane", "target_lane", "crashed", "impact",
          "check_collisions", "speed_index", "time")


def multi(A, action, observation, multi_action=True, multi_obs=True, **extra):
    act = {"type": "MultiAgentAction", "action_config": action} if multi_action else action
    obs = {"type": "MultiAgentObservation", "observation_config": observation} if multi_obs else observation
    return dict({"controlled_vehicles": A, "action": act, "observation": obs}, **extra)


DMA, CONT, KIN, TTC = ({"type": "DiscreteMetaAction"}, {"type": "ContinuousAction"}, {"type": "Kinematics"},
                       {"type": "TimeToCollision"})
# name: (env id, config, A, action kind, seeds, steps)
CASES = {
    "multi_highway_v0_a2": ("highway-v0", multi(2, DMA, KIN), 2, "meta", 4, 30),
    "multi_highway_fast_a3": ("highway-fast-v0", multi(3, DMA, KIN), 3, "meta", 6, 30),
    "multi_highway_fast_plain_action": ("highway-fast-v0", multi(2, DMA, KIN, multi_action=False), 2, "meta1", 6, 30),
    "multi_highway_v0_continuous": ("highway-v0", multi(4, CONT, KIN, multi_obs=False, vehicles_count=40), 4, "cont", 4,
                                    20),
    "multi_highway_fast_ttc": ("highway-fast-v0", multi(2, DMA, TTC), 2, "meta", 6, 30),
}
RESET_CONFIGS = [  # (A, vehicles_count, initial_lane_id, env id)
    (2, 50, None, "highway-v0"), (3, 20, None, "highway-fast-v0"), (8, 50, None, "highway-v0"),
    (5, 3, None, "highway-fast-v0"), (4, 30, 1, "highway-v0"), (3, 2, 0, "highway-fast-v0"),
    (8, 119, None, "highway-v0"), (6, 25, 2, "highway-fast-v0")]
RESET_SEEDS = 8


def actions_for(kind, A, seed, T):
    g = np.random.default_rng(1000 + seed)
    if kind == "meta":
        return [g.integers(0, 5, size=A).astype(np.int64) for _ in range(T)]
    if kind == "meta1":
        return [int(g.integers(0, 5)) for _ in range(T)]
    return [tuple(g.uniform(-1, 1, size=2).astype(np.float32) for _ in range(A)) for _ in range(T)]


def gen_case(name):
    env_id, cfg, A, kind, S, T = CASES[name]
    runs = []
    for seed in range(S):
        acts = actions_for(kind, A, seed, T)
        runs.append(rh.rollout(env_id, cfg, seed, acts))
    out = {k: np.stack([np.asarray(r[k]) for r in runs]) for k in FIELDS + ("obs", "reward", "terminated", "truncated",
                                                                            "rng_words")}
    if kind == "cont":
        out["actions"] = np.stack([np.asarray([np.stack(a) for a in actions_for(kind, A, s, T)], dtype=np.float32)
                                   for s in range(S)])
    else:
        out["actions"] = np.stack([np.asarray(actions_for(kind, A, s, T)) for s in range(S)])
    out["config"] = np.array(json.dumps(cfg))
    out["env_id"] = np.array(env_id)
    out["seeds"] = np.arange(S)
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **out)
    print(name, {k: v.shape for k, v in out.items()})


def gen_resets():
    out = {}
    for c, (A, count, lane_id, env_id) in enumerate(RESET_CONFIGS):
        cfg = multi(A, DMA, KIN, vehicles_count=count, initial_lane_id=lane_id)
        runs = [rh.rollout(env_id, cfg, 100 * c + s, []) for s in range(RESET_SEEDS)]
        for k in FIELDS + ("obs", "rng_words"):
            out[f"c{c}_{k}"] = np.stack([np.asarray(r[k])[0] for r in runs])
        out[f"c{c}_config"] = np.array(json.dumps(cfg))
        out[f"c{c}_env_id"] = np.array(env_id)
        out[f"c{c}_seeds"] = 100 * c + np.arange(RESET_SEEDS)
    out["n_configs"] = np.array(len(RESET_CONFIGS))
    np.savez_compressed(os.path.join(OUT, "multi_highway_resets.npz"), **out)
    print("multi_highway_resets", len(out), "arrays")


if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES) + ["multi_highway_resets"]
    for n in names:
        gen_resets() if n == "multi_highway_resets" else gen_case(n)
