"""Numpy statement of the batched finite MDP and of value iteration — the specification the device kernels
(csrc/hwy_observe.cu finite_mdp_kernel, csrc/hwy_plan.cu) follow bit for bit, and the helpers of its tests.

* `mdp_from_grid` restates finite_mdp() (reference envs/common/finite_mdp.py:17-101, 166-203) from a TTC grid;
* `value_iteration` restates rl-agents' ValueIterationAgent (Q_0 = 0; Bellman backups whose terminal rows do not
  bootstrap; stop at the first np.allclose(Q_k, Q_{k+1}) and keep Q_k).

Fixtures tests/golden/finite_mdp_*.npz come from `python oracle/gen_finite_mdp.py` (the unmodified reference)."""
from __future__ import annotations

import numpy as np

from parity_utils import load_golden

FIXTURES = ["finite_mdp_highway", "finite_mdp_highway_fast_pf2", "finite_mdp_highway_5lanes", "finite_mdp_roundabout",
            "finite_mdp_merge", "finite_mdp_exit"]
N_ACTIONS = 5


def mdp_from_grid(grid: np.ndarray, cfg: dict):
    """(transition int64 [S, 5], reward float64 [S, 5], terminal bool [S]) of the grid [V, L, T]."""
    V, L, T = grid.shape
    h, i, j = np.meshgrid(np.arange(V), np.arange(L), np.arange(T), indexing="ij")
    h, i, j = h.ravel(), i.ravel(), j.ravel()

    def ravel(hh, ii, jj):
        return np.ravel_multi_index((np.clip(hh, 0, V - 1), np.clip(ii, 0, L - 1), np.clip(jj, 0, T - 1)), (V, L, T))

    first = j == 0
    transition = np.stack([ravel(h, i - 1, j + 1), ravel(h, i, j + 1), ravel(h, i + 1, j + 1),
                           ravel(np.where(first, h + 1, h), i, j + 1), ravel(np.where(first, h - 1, h), i, j + 1)],
                          axis=1).astype(np.int64)
    lanes = np.arange(L) / max(L - 1, 1)
    speeds = np.arange(V) / max(V - 1, 1)
    state_reward = (cfg["collision_reward"] * grid + cfg["right_lane_reward"] * lanes[None, :, None]
                    + cfg["high_speed_reward"] * speeds[:, None, None]).ravel()
    action_reward = np.array([cfg["lane_change_reward"], 0, cfg["lane_change_reward"], 0, 0], dtype=np.float64)
    reward = state_reward[:, None] + action_reward[None, :]
    terminal = ((grid == 1) | (np.arange(T)[None, None, :] == T - 1)).ravel()
    return transition, reward, terminal


def value_iteration(transition, reward, terminal, gamma: float = 1.0, iterations: int = 100):
    """-> (q [S, A], iterations_done) for one deterministic MDP (its own S rows)."""
    q = np.zeros(reward.shape)
    for k in range(iterations):
        next_v = q.max(axis=1)[transition]
        next_v[terminal] = 0
        q_new = reward + gamma * next_v
        if np.allclose(q, q_new):
            return q, k
        q = q_new
    return q, iterations


def value_iteration_batch(transition, reward, terminal, n_states, gamma=1.0, iterations=100):
    """The padded batch layout: [N, S_max, A] q (rows past n_states 0) and [N] iterations_done."""
    n, s_max, a = reward.shape
    q = np.zeros((n, s_max, a))
    done = np.zeros(n, dtype=np.int32)
    for e in range(n):
        S = int(n_states[e])
        q[e, :S], done[e] = value_iteration(transition[e, :S], reward[e, :S], terminal[e, :S], gamma, iterations)
    return q, done


def random_mdps(rng, n: int, s_max: int, a: int, reward_levels: int = 3):
    """Seeded random deterministic MDPs in the padded layout, with ragged n_states and many reward ties."""
    n_states = rng.integers(1, s_max + 1, size=n).astype(np.int32)
    transition = np.tile(np.arange(s_max, dtype=np.int32)[None, :, None], (n, 1, a))
    reward = np.zeros((n, s_max, a))
    terminal = np.ones((n, s_max), dtype=bool)
    for e in range(n):
        S = int(n_states[e])
        transition[e, :S] = rng.integers(0, S, size=(S, a))
        reward[e, :S] = rng.integers(-reward_levels, reward_levels + 1, size=(S, a)) * 0.25
        terminal[e, :S] = rng.random(S) < 0.1
    return transition, reward, terminal, n_states


def load(name: str):
    return load_golden(name)
