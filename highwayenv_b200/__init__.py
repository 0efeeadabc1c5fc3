"""highwayenv_b200 — H100-native batched backend for HighwayEnv's simulation hot path.

Drop-in for the path ``AbstractEnv._simulate -> Road.act / Road.step -> observe / reward``
of Farama-Foundation/HighwayEnv 1.12.1, for thousands of independent envs at once:

    import highwayenv_b200 as hb
    env = hb.make("highway-fast-v0", num_envs=4096, config={"vehicles_count": 50})
    obs, info = env.reset(seed=0)
    obs, reward, terminated, truncated, info = env.step(actions)   # device tensors

The env ids, ``config`` keys and observation/action plugin names are the reference's
(highway_env/__init__.py:36-184).  Kernels are hand-written CUDA for sm_90a behind the C
ABI of include/hwyb200.h; there is no CPU fallback.
"""
from __future__ import annotations

import importlib
from typing import Any, Optional

__version__ = "0.1.0"

# id -> "module:Class" (same ids as the reference registers, highway_env/__init__.py:46-54)
REGISTRY = {
    "highway-v0": "highwayenv_b200.envs.highway_env:BatchedHighwayEnv",
    "highway-fast-v0": "highwayenv_b200.envs.highway_env:BatchedHighwayEnvFast",
    "roundabout-v0": "highwayenv_b200.envs.roundabout_env:BatchedRoundaboutEnv",
    "intersection-v0": "highwayenv_b200.envs.intersection_env:BatchedIntersectionEnv",
    "intersection-v1": "highwayenv_b200.envs.intersection_env:BatchedContinuousIntersectionEnv",
    # ConnectedLaneNeighboursMixin variants (neighbour search across lane segments)
    "roundabout-v1": "highwayenv_b200.envs.roundabout_env:BatchedConnectedLaneRoundaboutEnv",
    "intersection-v2": "highwayenv_b200.envs.intersection_env:BatchedConnectedLaneIntersectionEnv",
    "two-way-v0": "highwayenv_b200.envs.two_way_env:BatchedTwoWayEnv",
    "u-turn-v0": "highwayenv_b200.envs.u_turn_env:BatchedUTurnEnv",
    "u-turn-v1": "highwayenv_b200.envs.u_turn_env:BatchedConnectedLaneUTurnEnv",
    "exit-v0": "highwayenv_b200.envs.exit_env:BatchedExitEnv",
    "exit-v1": "highwayenv_b200.envs.exit_env:BatchedConnectedLaneExitEnv",
    "merge-v0": "highwayenv_b200.envs.merge_env:BatchedMergeEnv",
    "merge-v1": "highwayenv_b200.envs.merge_env:BatchedConnectedLaneMergeEnv",
    # MultiAgentAction / MultiAgentObservation (v1, v2: behind MultiAgentWrapper)
    "intersection-multi-agent-v0": "highwayenv_b200.envs.intersection_env:BatchedMultiAgentIntersectionEnv",
    "intersection-multi-agent-v1": "highwayenv_b200.envs.intersection_env:BatchedMultiAgentWrappedIntersectionEnv",
    "intersection-multi-agent-v2": "highwayenv_b200.envs.intersection_env:BatchedConnectedLaneMultiAgentIntersectionEnv",
}


def make(env_id: str, num_envs: int = 1, config: Optional[dict] = None, device: Any = None,
         render_mode: Optional[str] = None, **kwargs):
    """``gym.make`` equivalent for the batched backend (``"highwayenv_b200:highway-v0"`` and
    ``"highway_env:highway-v0"`` module-prefixed ids are accepted too)."""
    if ":" in env_id:
        env_id = env_id.split(":", 1)[1]
    if env_id not in REGISTRY:
        raise KeyError(f"{env_id!r} is not on the accelerated path; available: {sorted(REGISTRY)}")
    mod, cls = REGISTRY[env_id].split(":")
    env_cls = getattr(importlib.import_module(mod), cls)
    return env_cls(config=config, render_mode=render_mode, num_envs=num_envs, device=device, **kwargs)


def make_single(env_id: str, config: Optional[dict] = None, **kwargs):
    """`gym.make(env_id, config=...)` equivalent: ONE env with the gymnasium.Env surface (numpy observation, python
    float / bool returns, no autoreset) over the same kernels — see highwayenv_b200/single.py."""
    from .single import SingleEnv

    if ":" in env_id:
        env_id = env_id.split(":", 1)[1]
    return SingleEnv(env_id, config=config, **kwargs)


def _register_with_gymnasium() -> None:
    """When gymnasium is installed, expose the ids as vector envs:
    ``gymnasium.make_vec("hwyb200/highway-fast-v0", num_envs=4096)``."""
    try:
        from gymnasium.envs.registration import register, registry  # type: ignore
    except Exception:
        return
    for env_id, entry in REGISTRY.items():
        gid = f"hwyb200/{env_id}"  # hwyb200/<reference id>: gymnasium.make -> SingleEnv, gymnasium.make_vec -> batched env
        if gid not in registry:
            try:
                register(id=gid, entry_point="highwayenv_b200.single:SingleEnv", vector_entry_point=entry,
                         kwargs={"env_id": env_id})
            except Exception:
                pass


_register_with_gymnasium()
