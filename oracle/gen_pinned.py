"""Record the reference's outputs for the cases of the pinned-reference tests into tests/golden/pinned_*.npz / .json.

    python oracle/gen_pinned.py          (needs the unmodified reference: see ref_harness.REFERENCE_ROOT)

Unlike gen_golden.py (32-seed rollouts), this stores exactly what tests/test_oracle_live.py, test_net_oracle_live.py,
test_intersection_oracle_live.py and test_network_config_live.py compare against: teacher-forced steps on seeds that
are in no other fixture, free-running intersection episodes with the numpy generator words, the reference's
`RoadNetwork.to_config()` dicts and `DiscreteMetaAction.get_available_actions` on sampled ego states.  Each case is
generated in its own process: IntersectionEnv._make_vehicles rewrites IDMVehicle class constants process-wide."""
from __future__ import annotations

import json
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")
sys.path.insert(0, HERE)

HIGHWAY = [("highway-fast-v0", {"vehicles_count": 50}, 12, 4242),
           ("highway-v0", {"vehicles_count": 30, "lanes_count": 5, "action": {"type": "ContinuousAction"}}, 6, 77)]
NETWORK = [("roundabout-v0", {"observation": {"type": "TimeToCollision", "horizon": 10}}, 11, (31, 32)),
           ("roundabout-v1", None, 11, (33,)), ("merge-v0", None, 14, (34, 35)), ("merge-v1", None, 14, (36,)),
           ("two-way-v0", None, 10, (37, 38)), ("u-turn-v0", None, 10, (39, 40)), ("u-turn-v1", None, 10, (41,))]
INTERSECTION = [("intersection-v0", "default", 5000, 6), ("intersection-v0", "OccupancyGrid", 5100, 6),
                ("intersection-v2", "default", 5200, 4), ("intersection-multi-agent-v0", "default", 5300, 4)]
NETWORK_CONFIG = ["intersection-v0", "merge-v0", "roundabout-v0", "two-way-v0", "u-turn-v0"]


def case_path(kind: str, *parts) -> str:
    name = "_".join([kind] + [str(p) for p in parts]).replace("-", "_").replace(".", "_")
    return os.path.join(OUT, "pinned_" + name + ".npz")


def _json(o):
    return json.dumps(o, default=lambda v: v.tolist() if hasattr(v, "tolist") else str(v))


def _save(path: str, cfg: dict, states: list, **arrays) -> None:
    """states: list of dump_state-like dicts, stacked per key under 's_<key>'."""
    out = {"config_json": np.array(_json(cfg))}
    for k in states[0]:
        out["s_" + k] = np.stack([np.asarray(s[k]) for s in states])
    out.update({k: np.asarray(v) for k, v in arrays.items()})
    np.savez_compressed(path, **out)


def rng_words(env) -> list:
    w, m64 = env.np_random.bit_generator.state, (1 << 64) - 1
    return [w["state"]["state"] >> 64, w["state"]["state"] & m64, w["state"]["inc"] >> 64, w["state"]["inc"] & m64,
            (int(w["has_uint32"]) << 32) | int(w["uinteger"])]


def gen_highway(i: int) -> None:
    import ref_harness as rh

    env_id, over, T, seed = HIGHWAY[i]
    env = rh.make_reference_env(env_id, over)
    obs0, _ = env.reset(seed=seed)
    cfg = dict(env.config)
    rng = np.random.default_rng(seed)
    states, obs, acts, rew, term, trunc = [rh.dump_state(env)], [np.asarray(obs0)], [], [], [], []
    for _ in range(T):
        a = int(rng.integers(5)) if cfg["action"]["type"] != "ContinuousAction" else rng.uniform(-1, 1, 2).astype(np.float32)
        o, r, te, tr, _ = env.step(a)
        states.append(rh.dump_state(env))
        obs.append(np.asarray(o)), acts.append(np.asarray(a, dtype=np.float64)), rew.append(r), term.append(te), trunc.append(tr)
    _save(case_path("highway", env_id, seed), cfg, states, obs=np.stack(obs), actions=np.stack(acts),
          reward=np.array(rew, dtype=np.float64), terminated=np.array(term), truncated=np.array(trunc))


def gen_actions_mask() -> None:
    """the 200 ego states of test_available_actions_mask and the reference's available actions for each"""
    import ref_harness as rh

    env = rh.make_reference_env("highway-fast-v0", {"lanes_count": 3})
    env.reset(seed=0)
    rng = np.random.default_rng(0)
    rows, mask = [], np.zeros((200, 5), dtype=bool)
    for k in range(200):
        v = env.vehicle
        lane, si = int(rng.integers(3)), int(rng.integers(3))
        x = float(rng.choice([-3.0, 0.0, 50.0, 9999.0, 10004.99, 10005.0, 10010.0]))
        y = 4.0 * lane + float(rng.uniform(-2, 2))
        v.position, v.lane_index, v.speed_index = np.array([x, y]), ("0", "1", lane), si
        v.lane = env.road.network.get_lane(v.lane_index)
        mask[k, sorted(set(env.action_type.get_available_actions()))] = True
        rows.append((x, y, lane, si))
    r = np.array(rows, dtype=np.float64)
    np.savez_compressed(os.path.join(OUT, "pinned_available_actions.npz"), x=r[:, 0], y=r[:, 1],
                        lane=r[:, 2].astype(np.int32), speed_index=r[:, 3].astype(np.int32), mask=mask)


def _net_state(env, V) -> dict:
    import net_oracle as no
    import ref_harness as rh

    st = rh.dump_state(env)
    st["target_lane"] = np.where(st["target_lane"] < 0, st["lane"], st["target_lane"])
    if "route" not in st:
        st["route"], st["route_len"] = np.zeros((V, no.NET_MAX_ROUTE), dtype=np.int32), np.zeros(V, dtype=np.int32)
    if "kind" in st:
        st["impact"] = np.where((st["kind"] == 3)[:, None], np.nan, st["impact"])  # objects: inert zeros
    else:
        st["kind"] = np.array([1] + [0] * (V - 1), dtype=np.int32)
    st.setdefault("count", np.int32(V))
    st.setdefault("is_yielding", np.zeros(V, dtype=np.int32))
    st.setdefault("road_steps", np.int64(0))
    return st


def gen_network(i: int, seed: int) -> None:
    import ref_harness as rh

    env_id, over, T, _ = NETWORK[i]
    env = rh.make_reference_env(env_id, over)
    obs0, _ = env.reset(seed=seed)
    cfg = dict(env.config)
    cfg["_env_id"] = env_id
    if env_id.startswith("merge"):
        lanes = [li for li, _ in rh.lane_list(env)]
        cfg["_merge_lane"] = lanes.index(("b", "c", 2))
        cfg["_default_side_lanes"] = len(env.road.network.all_side_lanes(env.vehicle.lane_index))
    V = len(env.road.vehicles) + len(env.road.objects)
    net = rh.dump_network(env)
    rng = np.random.default_rng(seed)
    states, obs, acts, rew, term, trunc = [_net_state(env, V)], [np.asarray(obs0)], [], [], [], []
    for _ in range(T):
        a = int(rng.integers(5))
        o, r, te, tr, _ = env.step(a)
        states.append(_net_state(env, V))
        obs.append(np.asarray(o)), acts.append(a), rew.append(r), term.append(te), trunc.append(tr)
    _save(case_path("network", env_id, seed), cfg, states, obs=np.stack(obs), actions=np.array(acts, dtype=np.int32),
          reward=np.array(rew, dtype=np.float64), terminated=np.array(term), truncated=np.array(trunc),
          n_vehicles=np.int32(V), **net)


def gen_intersection(i: int, seed: int) -> None:
    """free-running episode: reference state / obs / reward / flags / generator words after every step"""
    import ref_harness as rh

    env_id, obs_type, _, _ = INTERSECTION[i]
    over = None if obs_type == "default" else {"observation": {"type": obs_type}}
    env = rh.make_reference_env(env_id, over)
    obs0, _ = env.reset(seed=seed)
    cfg = dict(env.config)
    net = rh.dump_network(env)
    A = int(cfg.get("controlled_vehicles", 1))
    rng = np.random.default_rng(seed)
    states, obs, acts, rew, term, trunc, words = [rh.dump_state(env, 32)], [np.asarray(obs0)], [], [], [], [], []
    for _ in range(int(cfg["duration"] * cfg["policy_frequency"]) + 1):
        a = rng.integers(0, 3, size=A)
        o, r, te, tr, _ = env.step(tuple(int(x) for x in a) if A > 1 else int(a[0]))
        states.append(rh.dump_state(env, 32))
        obs.append(np.asarray(o)), acts.append(a.astype(np.int32)), rew.append(r), term.append(te), trunc.append(tr)
        words.append(rng_words(env))
        if te or tr:
            break
    _save(case_path("intersection", env_id, obs_type, seed), cfg, states, obs=np.stack(obs), actions=np.stack(acts),
          reward=np.array(rew, dtype=np.float64), terminated=np.array(term), truncated=np.array(trunc),
          rng_words=np.array(words, dtype=np.uint64), **net)


def gen_network_config(env_id: str) -> None:
    import ref_harness as rh

    env = rh.make_reference_env(env_id, None)
    env.reset(seed=0)
    path = os.path.join(OUT, "pinned_to_config_" + env_id.replace("-", "_") + ".json")
    with open(path, "w") as f:
        f.write(_json(env.road.network.to_config()))


def jobs() -> list:
    out = [["highway", str(i)] for i in range(len(HIGHWAY))] + [["actions_mask"]]
    out += [["network", str(i), str(s)] for i, c in enumerate(NETWORK) for s in c[3]]
    out += [["intersection", str(i), str(s)] for i, c in enumerate(INTERSECTION) for s in range(c[2], c[2] + c[3])]
    return out + [["network_config", e] for e in NETWORK_CONFIG]


def run(job: list) -> None:
    kind, args = job[0], job[1:]
    if kind == "highway":
        gen_highway(int(args[0]))
    elif kind == "actions_mask":
        gen_actions_mask()
    elif kind == "network":
        gen_network(int(args[0]), int(args[1]))
    elif kind == "intersection":
        gen_intersection(int(args[0]), int(args[1]))
    else:
        gen_network_config(args[0])


if __name__ == "__main__":
    import ref_harness as rh

    if not rh.reference_available():
        raise SystemExit("the reference is not available (ref_harness.REFERENCE_ROOT)")
    if len(sys.argv) > 1:
        run(sys.argv[1:])
    else:
        for job in jobs():
            subprocess.check_call([sys.executable, os.path.abspath(__file__)] + job)
