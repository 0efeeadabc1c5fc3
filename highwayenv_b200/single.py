"""A single-env, `gymnasium.Env`-shaped facade over the batched backend (SURVEY §7 step 1; reference surface:
`AbstractEnv.reset / step`, envs/common/abstract.py:219-285): numpy observation, python float / bool returns, an `info`
dict of python scalars with the reference's keys (`speed`, `crashed`, `action`, `rewards`), no autoreset.

    env = highwayenv_b200.make_single("highway-fast-v0", config={"vehicles_count": 50})
    obs, info = env.reset(seed=0)
    obs, reward, terminated, truncated, info = env.step(env.action_space.sample())

It is the batched env with `num_envs=1` (same kernels, same seeds: `reset(seed=s)` gives the reference env's episode
for seed `s`); one step costs a kernel launch plus a device->host read, so use the batched interface for throughput.
"""
from __future__ import annotations

from typing import Any, Optional

import numpy as np

try:  # a real gymnasium.Env when gymnasium is installed (wrappers and checkers then accept it)
    import gymnasium as _gym

    _Base = _gym.Env
except Exception:  # pragma: no cover - gymnasium is not in this image
    _Base = object


def _obs_row(obs):
    """Env 0's observation as numpy; a Dict observation (lane-keeping-v0) as a dict of float64 arrays."""
    if isinstance(obs, dict):
        return {k: v[0].cpu().numpy().copy() for k, v in obs.items()}
    return obs[0].cpu().numpy().copy()


def _scalar(v):
    a = v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)
    a = a.reshape(a.shape[1:]) if a.ndim >= 1 and a.shape[0] == 1 else a
    return a.item() if a.ndim == 0 else a


class SingleEnv(_Base):
    metadata = {"render_modes": []}

    def __init__(self, env_id: str, config: Optional[dict] = None, render_mode: Optional[str] = None, **kwargs: Any):
        from . import make

        kwargs.pop("num_envs", None)
        self.batched = make(env_id, num_envs=1, config=config, render_mode=render_mode, autoreset_mode="Disabled", **kwargs)
        self.observation_space = self.batched.single_observation_space
        self.action_space = self.batched.single_action_space
        self.render_mode = None

    @property
    def config(self) -> dict:
        return self.batched.config

    @property
    def unwrapped(self):
        return self

    def _info(self, info: dict) -> dict:
        out = {}
        for k, v in info.items():
            if k == "final_obs":
                continue
            out[k] = {n: _scalar(t) for n, t in v.items()} if isinstance(v, dict) else _scalar(v)
        return out

    def reset(self, *, seed: Optional[int] = None, options: Optional[dict] = None):
        obs, info = self.batched.reset(seed=seed, options=options)
        return _obs_row(obs), self._info(info)

    def step(self, action):
        a = np.asarray(action)
        buf = self.batched._action_buf
        a = a.reshape((1,) + tuple(buf.shape[1:])).astype(np.float32 if buf.dtype.is_floating_point else np.int64)
        obs, reward, terminated, truncated, info = self.batched.step(a)
        return (_obs_row(obs), float(_scalar(reward)), bool(_scalar(terminated)), bool(_scalar(truncated)),
                self._info(info))

    def get_available_actions(self):
        """DiscreteMetaAction.get_available_actions (envs/common/action.py:262-299) as a list of action indices."""
        mask = self.batched.get_available_actions()[0].cpu().numpy()
        return [int(i) for i in np.nonzero(mask)[0]]

    def to_finite_mdp(self):
        """AbstractEnv.to_finite_mdp() (envs/common/abstract.py:452-453): the time-to-collision MDP of the current
        state with finite_mdp's DeterministicMDP attributes (transition, reward, terminal, state, original_shape,
        mode), as rl-agents' ValueIterationAgent reads it from `env.unwrapped`."""
        return self.batched.to_finite_mdp().env(0)

    def close(self) -> None:
        self.batched.close()
