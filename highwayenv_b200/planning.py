"""Model-based planning on the device: the batched finite MDP of the reference's `AbstractEnv.to_finite_mdp()`
(envs/common/abstract.py:452-453, envs/common/finite_mdp.py:17-203), batched value iteration with the semantics of
rl-agents' `ValueIterationAgent`, and the policy that rebuilds and solves the MDP at every step.

    env = highwayenv_b200.make("highway-v0", num_envs=4096)
    env.reset(seed=0)
    policy = TtcValueIterationPolicy(env)
    for _ in range(40):
        env.step(policy.act())          # no host round trip

`env.to_finite_mdp()` (csrc/hwy_observe.cu finite_mdp_kernel) builds, per env, the time-to-collision grid over every
lane of the ego's road and the deterministic MDP on its (speed, lane, time) cells; `value_iteration()`
(csrc/hwy_plan.cu) solves any batch of deterministic MDPs in that layout.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _native as N

HORIZON = 10.0  # finite_mdp(env, time_quantization=1 / policy_frequency, horizon=10.0)
N_ACTIONS = 5   # LANE_LEFT, IDLE, LANE_RIGHT, FASTER, SLOWER
MAX_LANES, MAX_T = 8, 64  # the TTC grid kernels' limits (csrc/hwy_observe.cu)


class DeterministicMdp:
    """One env's MDP under the attribute names of finite_mdp's `DeterministicMDP`, as numpy arrays:
    `transition` int64 [S, A], `reward` float64 [S, A], `terminal` bool [S], `state` (int), `original_shape`
    (speeds, lanes, time) and `mode = "deterministic"`."""

    mode = "deterministic"

    def __init__(self, transition, reward, terminal, state, original_shape):
        self.transition, self.reward, self.terminal = transition, reward, terminal
        self.state, self.original_shape = state, original_shape


class FiniteMdp:
    """The finite MDPs of a batch of envs, device tensors padded to the largest shape:

    ============  ===============================  ==========================================================
    grid          [N, n_speeds, L_max, T] float64  compute_ttc_grid; lanes >= n_lanes[e] are 0
    n_lanes       [N] int32                        lanes of the ego's road
    n_states      [N] int32                        n_speeds * n_lanes * T
    state         [N] int64                        ravel_multi_index((speed_index, lane id, 0), grid shape)
    transition    [N, S_max, 5] int32              raveled in each env's own (n_speeds, n_lanes, T) shape
    reward        [N, S_max, 5] float64
    terminal      [N, S_max] bool
    ============  ===============================  ==========================================================

    S_max = n_speeds * L_max * T; rows s >= n_states[e] point to themselves, have reward 0 and are terminal."""

    def __init__(self, n: int, n_speeds: int, l_max: int, n_t: int, device):
        s_max = n_speeds * l_max * n_t
        z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=device)  # noqa: E731
        self.grid = z(n, n_speeds, l_max, n_t, dtype=torch.float64)
        self.n_lanes, self.n_states = z(n, dtype=torch.int32), z(n, dtype=torch.int32)
        self.state = z(n, dtype=torch.int64)
        self.transition = z(n, s_max, N_ACTIONS, dtype=torch.int32)
        self.reward = z(n, s_max, N_ACTIONS, dtype=torch.float64)
        self.terminal = z(n, s_max, dtype=torch.bool)

    def env(self, i: int) -> DeterministicMdp:
        """Env `i` as the reference's `env.to_finite_mdp()` returns it (rows sliced to that env's own states)."""
        V, _, T = self.grid.shape[1:]
        L = int(self.n_lanes[i])
        S = V * L * T
        return DeterministicMdp(self.transition[i, :S].cpu().numpy().astype(np.int64),
                                self.reward[i, :S].cpu().numpy().copy(), self.terminal[i, :S].cpu().numpy().copy(),
                                int(self.state[i]), (V, L, T))


def _ego_target_speeds(env) -> np.ndarray:
    """MDPVehicle.target_speeds of the controlled vehicle; compute_ttc_grid needs an MDPVehicle."""
    from .envs.common.action import DiscreteMetaAction

    at = getattr(env, "action_type", None)
    if at is None and hasattr(env, "target_speeds"):  # the intersection family keeps DiscreteMetaAction implicit
        return np.asarray(env.target_speeds, dtype=np.float64)
    if not isinstance(at, DiscreteMetaAction):
        raise ValueError("to_finite_mdp needs an MDPVehicle ego (DiscreteMetaAction): compute_ttc_grid reads "
                         "vehicle.target_speeds (finite_mdp.py:104-163)")
    return np.asarray(at.target_speeds, dtype=np.float64)


def _max_road_lanes(env) -> int:
    net = getattr(env, "net", None)
    if net is not None:
        return max(int(lane["road_count"]) for lane in net.lanes)
    return int(env._params.lanes_count)


def mdp_params(env) -> N.HwyFiniteMdpParams:
    """The kernel parameters of env.to_finite_mdp(); every unsupported configuration raises here, before any launch:
    multi-agent (NotImplementedError), a non-MDPVehicle ego (ValueError), a reward key the env's config lacks
    (the reference's KeyError), an action set other than the 5 meta-actions (NotImplementedError: the reference's
    transition model reads actions 0 and 2 as lane changes whatever the set is), T > 64 or roads wider than 8 lanes
    (ValueError)."""
    if getattr(env, "multi_agent", False) or getattr(env, "n_agents", 1) > 1:
        raise NotImplementedError("to_finite_mdp of a multi-agent env")
    ts = _ego_target_speeds(env)
    cfg = env.config
    rewards = [float(cfg[k]) for k in ("collision_reward", "right_lane_reward", "high_speed_reward",
                                       "lane_change_reward")]  # finite_mdp.py:63-78, in the reference's order
    if getattr(env.single_action_space, "n", None) != N_ACTIONS:
        raise NotImplementedError("to_finite_mdp with an action set other than the 5 DiscreteMetaAction actions")
    pf = int(cfg["policy_frequency"])
    n_t = int(HORIZON / (1 / pf))
    if not 1 <= n_t <= MAX_T:
        raise ValueError(f"to_finite_mdp: T = int(10 / (1 / policy_frequency)) = {n_t} is outside 1..{MAX_T}")
    l_max = _max_road_lanes(env)
    if not 1 <= l_max <= MAX_LANES:
        raise ValueError(f"to_finite_mdp: roads of up to {MAX_LANES} lanes")
    p = N.HwyFiniteMdpParams()
    p.policy_frequency, p.n_target_speeds, p.l_max, p.n_t, p.horizon = pf, int(ts.size), l_max, n_t, HORIZON
    for k, t in enumerate(ts):
        p.target_speeds[k] = float(t)
    p.collision_reward, p.right_lane_reward, p.high_speed_reward, p.lane_change_reward = rewards
    return p


def _launch_finite_mdp(env, p: N.HwyFiniteMdpParams, out: FiniteMdp) -> None:
    view, graph = env._obs_view()
    with torch.cuda.device(env.device):
        N.check(env._lib.hwy_finite_mdp(graph, C.byref(view), C.byref(p), out.grid.data_ptr(), out.n_lanes.data_ptr(),
                                        out.n_states.data_ptr(), out.state.data_ptr(), out.transition.data_ptr(),
                                        out.reward.data_ptr(), out.terminal.data_ptr(), env._stream()))


def _shape(p: N.HwyFiniteMdpParams):
    return int(p.n_target_speeds), int(p.l_max), int(p.n_t)


def to_finite_mdp(env) -> FiniteMdp:
    """`env.to_finite_mdp()` of every env of a batched env (see FiniteMdp)."""
    if not env._seeded:
        raise RuntimeError("call reset() before to_finite_mdp()")
    p = mdp_params(env)
    out = FiniteMdp(env.num_envs, *_shape(p), env.device)
    _launch_finite_mdp(env, p, out)
    return out


def _check_vi_args(transition, reward, terminal, n_states, gamma, iterations):
    if not isinstance(transition, torch.Tensor) or transition.dim() != 3:
        raise ValueError("transition must be an int32 tensor [N, S_max, A]")
    n, s_max, a = transition.shape
    dev = transition.device
    if dev.type != "cuda":
        raise ValueError("value_iteration runs on CUDA tensors")
    for name, t, dtypes, shape in (("transition", transition, (torch.int32,), (n, s_max, a)),
                                   ("reward", reward, (torch.float64,), (n, s_max, a)),
                                   ("terminal", terminal, (torch.bool, torch.uint8), (n, s_max)),
                                   ("n_states", n_states, (torch.int32,), (n,))):
        if not isinstance(t, torch.Tensor) or t.dtype not in dtypes or tuple(t.shape) != shape or t.device != dev:
            raise ValueError(f"{name} must be a {'/'.join(map(str, dtypes))} tensor of shape {shape} on {dev}")
    if n < 1 or not 1 <= s_max <= N.HWY_VI_MAX_STATES or not 1 <= a <= N.HWY_VI_MAX_ACTIONS:
        raise ValueError(f"value_iteration: N >= 1, 1 <= S_max <= {N.HWY_VI_MAX_STATES}, "
                         f"1 <= A <= {N.HWY_VI_MAX_ACTIONS}")
    if not 0.0 <= float(gamma) <= 1.0:
        raise ValueError("gamma must be in [0, 1]")
    if int(iterations) != iterations or iterations < 0 or iterations > 2**31 - 1:
        raise ValueError("iterations must be an int >= 0")


def _launch_value_iteration(transition, reward, terminal, n_states, gamma, iterations, q, done, state=None,
                            action=None) -> None:
    n, s_max, a = transition.shape
    p = N.HwyValueIterationParams()
    p.n_envs, p.s_max, p.n_actions, p.iterations, p.gamma = n, s_max, a, int(iterations), float(gamma)
    p.state = None if state is None else state.data_ptr()
    p.action = None if action is None else action.data_ptr()
    with torch.cuda.device(transition.device):
        N.check(N.load().hwy_value_iteration(C.byref(p), transition.data_ptr(), reward.data_ptr(),
                                             terminal.data_ptr(), n_states.data_ptr(), q.data_ptr(), done.data_ptr(),
                                             torch.cuda.current_stream(transition.device).cuda_stream))


def value_iteration(mdp, gamma: float = 1.0, iterations: int = 100):
    """Value iteration of a batch of deterministic MDPs (`transition` int32 [N, S_max, A], `reward` float64
    [N, S_max, A], `terminal` bool [N, S_max], `n_states` int32 [N], as `to_finite_mdp()` returns them or built by
    the caller), one CUDA block per env.  Per env, over its own n_states rows:

        Q_0 = 0
        for k in range(iterations):
            next_v = Q_k.max(axis=1)[transition]; next_v[terminal] = 0
            Q_new = reward + gamma * next_v
            if np.allclose(Q_k, Q_new): break          # Q_k is returned
            Q_{k+1} = Q_new

    Returns `(q [N, S_max, A] float64, iterations_done [N] int32)`; rows past n_states are 0.  An env whose
    n_states is outside 0..S_max or that has a successor outside its own rows gets iterations_done = -1 and q = 0;
    the other envs are unaffected."""
    transition, reward, terminal, n_states = (t.contiguous() if isinstance(t, torch.Tensor) else t for t in (
        mdp.transition, mdp.reward, mdp.terminal, mdp.n_states))
    _check_vi_args(transition, reward, terminal, n_states, gamma, iterations)
    q = torch.empty(transition.shape, dtype=torch.float64, device=transition.device)
    done = torch.empty(transition.shape[0], dtype=torch.int32, device=transition.device)
    _launch_value_iteration(transition, reward, terminal, n_states, gamma, iterations, q, done)
    return q, done


class TtcValueIterationPolicy:
    """rl-agents' `ValueIterationAgent.act()` for every env of a batched env: rebuild `env.to_finite_mdp()`, solve
    it with `value_iteration(gamma, iterations)` and take the first argmax of `q[e, state[e]]` (np.argmax).
    `act()` returns int64 actions [N] on the env's device, for `env.step`.  Buffers are allocated at the first
    call (and again only if the env's MDP shape changes); later calls make no host synchronisation and no
    allocation, so `act()` can be captured in a CUDA graph."""

    def __init__(self, env, gamma: float = 1.0, iterations: int = 100):
        if not 0.0 <= float(gamma) <= 1.0:
            raise ValueError("gamma must be in [0, 1]")
        if int(iterations) != iterations or iterations < 0:
            raise ValueError("iterations must be an int >= 0")
        mdp_params(env)  # unsupported envs fail here
        self.env, self.gamma, self.iterations = env, float(gamma), int(iterations)
        self._key = None
        self.mdp = self.q = self.iterations_done = self.actions = None

    def act(self) -> torch.Tensor:
        env = self.env
        if not env._seeded:
            raise RuntimeError("call reset() before act()")
        p = mdp_params(env)
        key = (env.num_envs, env.device) + _shape(p)
        if key != self._key:
            self.mdp = FiniteMdp(env.num_envs, *_shape(p), env.device)
            self.q = torch.zeros(self.mdp.reward.shape, dtype=torch.float64, device=env.device)
            self.iterations_done = torch.zeros(env.num_envs, dtype=torch.int32, device=env.device)
            self.actions = torch.zeros(env.num_envs, dtype=torch.int64, device=env.device)
            self._key = key
        m = self.mdp
        _launch_finite_mdp(env, p, m)
        _launch_value_iteration(m.transition, m.reward, m.terminal, m.n_states, self.gamma, self.iterations, self.q,
                                self.iterations_done, m.state, self.actions)
        return self.actions
