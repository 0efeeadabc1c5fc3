"""Shared helpers for parity tests (golden fixtures <-> oracle <-> CUDA path)."""
from __future__ import annotations

import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

FLOAT_TOL = 1e-5  # BASELINE.json north_star: <= 1e-5 abs on positions / headings / speeds
STATE_F = ("x", "y", "heading", "speed")


def load_golden(name: str) -> dict:
    z = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
    d = {k: z[k] for k in z.files}
    if "config_json" in d:
        d["config"] = json.loads(str(d["config_json"]))
    return d


def load_pinned(path: str):
    """A tests/golden/pinned_*.npz case of oracle/gen_pinned.py: (config, [state after t steps], other arrays)."""
    z = np.load(path, allow_pickle=False)
    d = {k: z[k] for k in z.files}
    cfg = json.loads(str(d.pop("config_json")))
    keys = [k for k in d if k.startswith("s_")]
    states = [{k[2:]: d[k][t] for k in keys} for t in range(d[keys[0]].shape[0])]
    return cfg, states, {k: v for k, v in d.items() if not k.startswith("s_")}


def golden_state(g: dict, i: int, t: int) -> dict:
    """State of seed-slot i after t steps, in ref_harness.dump_state layout."""
    keys = ("x", "y", "heading", "speed", "target_speed", "timer", "delta", "lane", "target_lane",
            "crashed", "impact", "check_collisions", "speed_index", "time")
    return {k: g[k][i, t] for k in keys}


def well_conditioned(st: dict, min_speed: float = 1.0) -> bool:
    """The reference's steering law divides by not_zero(speed) (controller.py:166,178): for a
    NON-crashed vehicle crawling at |v| < ~1 m/s it amplifies 1-ulp libm differences by
    > 1e6 per policy step, so free-running trajectories of two correct implementations
    diverge there.  Free-running parity is asserted on the prefix before that happens;
    teacher-forced (one-step) parity is asserted on every state."""
    alive = ~st["crashed"].astype(bool)
    return bool(np.all(np.abs(st["speed"][alive]) >= min_speed))


def comparable_steps(g: dict) -> int:
    """How many (seed, step) pairs of a golden rollout a free-running comparison covers: for every seed the prefix of
    steps whose golden state is well conditioned.  A property of the fixture alone, so the free-running tests assert
    this exact count instead of a floor (round-1 verdict: `compared >= 3 * S` was 10 % of the steps)."""
    S, T = g["actions"].shape[:2]
    n = 0
    for i in range(S):
        for t in range(T):
            if not well_conditioned(golden_state(g, i, t + 1)):
                break
            n += 1
    return n


def compare_state(st: dict, got: dict, tol: float = FLOAT_TOL, ctx: str = "") -> float:
    """st: golden (dump_state layout); got: dict of arrays with the same schema where
    target_lane mirrors lane for vehicles without one and impact is (has_impact, ix, iy)."""
    worst = 0.0
    for k in STATE_F:
        d = float(np.max(np.abs(st[k] - got[k])))
        assert d <= tol, f"{ctx} {k} diff {d}"
        worst = max(worst, d)
    idm = slice(1, None)
    d = float(np.max(np.abs(np.nan_to_num(st["timer"][idm]) - got["timer"][idm])))
    assert d <= tol, f"{ctx} timer diff {d}"
    worst = max(worst, d)
    ts = ~np.isnan(st["target_speed"])
    d = float(np.max(np.abs(st["target_speed"][ts] - got["target_speed"][ts]))) if ts.any() else 0.0
    assert d <= tol, f"{ctx} target_speed diff {d}"
    assert np.array_equal(st["lane"], got["lane"]), f"{ctx} lane {st['lane']} vs {got['lane']}"
    tl = np.where(st["target_lane"] < 0, st["lane"], st["target_lane"])
    assert np.array_equal(tl, got["target_lane"]), f"{ctx} target_lane"
    assert np.array_equal(st["crashed"].astype(bool), got["crashed"].astype(bool)), f"{ctx} crashed"
    has = ~np.isnan(st["impact"][:, 0])
    assert np.array_equal(has, got["has_impact"].astype(bool)), f"{ctx} has_impact"
    if has.any():
        d = max(
            float(np.max(np.abs(st["impact"][has, 0] - got["impact_x"][has]))),
            float(np.max(np.abs(st["impact"][has, 1] - got["impact_y"][has]))),
        )
        assert d <= tol, f"{ctx} impact diff {d}"
        worst = max(worst, d)
    if st["speed_index"][0] >= 0:
        assert int(st["speed_index"][0]) == int(got["speed_index"]), f"{ctx} speed_index"
    return worst
