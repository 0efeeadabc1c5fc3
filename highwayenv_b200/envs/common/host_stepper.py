"""`env.host_stepper()`: one CUDA graph per env.step for callers that live on the host (any env family)."""
from __future__ import annotations

import numpy as np
import torch


class HostStepper:
    """`env.step` for callers that live on the host (a CPU policy, a gymnasium wrapper stack): pinned host
    buffers for the actions and the results, and ONE CUDA graph holding the action upload, the step kernel
    and the result downloads, so a step costs one graph launch + one stream sync instead of six API calls.

        hs = env.host_stepper()
        hs.actions[:] = policy(hs.obs)            # numpy views of pinned memory
        obs, reward, terminated, truncated = hs.step()

    The arrays returned are the stepper's own pinned buffers (overwritten by the next step).  State, RNG
    streams and autoreset behave exactly as with `env.step` (same kernels, same buffers).  Every env family
    qualifies: the highway step is one kernel; a network step (intersection: classify + 16-slot + 32-slot step
    kernels + compaction + reset kernel, plus a standalone observation plugin if one is configured) is captured
    as a whole, so the host pays one launch for all of them."""

    def __init__(self, env) -> None:
        if not env._seeded:
            raise RuntimeError("call reset() before host_stepper()")
        if env.reset_mode != "device":
            raise NotImplementedError("host_stepper needs the device reset path (reset_mode='device')")
        self.env = env
        dev = env.device
        table = getattr(env.action_type, "table", None)
        # DiscreteAction (action.py:165-196): the host hands over indices; the gather into the (throttle, steering)
        # buffer is a device op of env.step and is captured with it.  The range check of `all_actions[action]` cannot
        # run inside a graph (it reads the device), so step() makes it on the host array instead.
        self._n_table = 0 if table is None else int(table.shape[0])
        if env.autoreset_mode == "NextStep":
            # NextStep runs host-side control flow per call (which envs ended last time); a captured graph would
            # replay one frozen decision
            raise NotImplementedError("host_stepper with autoreset_mode='NextStep' — use SameStep or Disabled")
        pin = lambda t: torch.empty(tuple(t.shape), dtype=t.dtype).pin_memory()  # noqa: E731
        if self._n_table:
            if getattr(env, "_action_table", None) is None or env._action_table.device != dev:
                env._action_table = torch.from_numpy(table).to(dev)  # env.step builds it lazily; not under capture
            self._h_actions = torch.empty((env.num_envs,), dtype=torch.int64).pin_memory()
            self._d_actions = torch.empty((env.num_envs,), dtype=torch.int64, device=dev)
        else:
            self._h_actions = pin(env._action_buf)
            self._d_actions = env._action_buf
        self._h_obs, self._h_reward = pin(env._obs), pin(env._reward)
        self._h_term, self._h_trunc = pin(env._terminated), pin(env._truncated)
        self.actions = self._h_actions.numpy()
        self.obs, self.reward = self._h_obs.numpy(), self._h_reward.numpy()
        self.terminated, self.truncated = self._h_term.numpy().view(np.bool_), self._h_trunc.numpy().view(np.bool_)
        self._h_obs.copy_(env._obs)
        self._stream = torch.cuda.Stream(device=dev)
        self._graph = torch.cuda.CUDAGraph()
        with torch.cuda.device(dev):
            torch.cuda.synchronize(dev)
            with torch.cuda.graph(self._graph, stream=self._stream):
                self._d_actions.copy_(self._h_actions, non_blocking=True)
                obs, reward, term, trunc, _ = env.step(self._d_actions)
                self._h_obs.copy_(obs, non_blocking=True)
                self._h_reward.copy_(env._reward, non_blocking=True)
                self._h_term.copy_(env._terminated, non_blocking=True)
                self._h_trunc.copy_(env._truncated, non_blocking=True)

    def step(self):
        if self._n_table and (self.actions.min() < 0 or self.actions.max() >= self._n_table):
            raise IndexError("list index out of range")  # all_actions[action] in the reference
        self._graph.replay()
        self._stream.synchronize()
        return self.obs, self.reward, self.terminated, self.truncated
