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

`OpdPolicy` plans on the simulator itself instead of the TTC abstraction: optimistic deterministic planning over
clones of every env (`env.copy_envs`, csrc/hwy_copy.cu), with its tree kernels in csrc/hwy_plan.cu.

    policy = OpdPolicy(env, budget=50, gamma=0.7)
    env.step(policy.act())

`MctsPolicy` is open-loop Monte-Carlo tree search on the same clones, optionally keeping the subtree of the action
taken across decisions:

    policy = MctsPolicy(env, budget=100, gamma=0.7, reuse_subtree=True)
    a = policy.act()
    _, _, term, trunc, _ = env.step(a)
    policy.advance(a, term | trunc)
"""
from __future__ import annotations

import copy
import ctypes as C
from types import SimpleNamespace

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


OPD_ENV_IDS = ("highway-v0", "highway-fast-v0", "roundabout-v0", "roundabout-v1", "merge-v0", "merge-v1", "exit-v0",
               "exit-v1")


def opd_discount_tables(gamma: float, expansions: int):
    """(g, t) float64 [expansions + 2]: g[d] = gamma ** d and the optimistic bound t[d] = g[d] / (1 - gamma) of the
    discounted rewards past depth d (rewards <= 1)."""
    g = np.float64(gamma) ** np.arange(expansions + 2, dtype=np.float64)
    return g, g / (np.float64(1.0) - np.float64(gamma))


def _check_tree_search_env(env, planner: str) -> None:
    """The envs the tree-search planners run on: one MDPVehicle ego on an id whose `step` draws nothing from the env's
    stream (OPD_ENV_IDS), so a row copy steps exactly like `copy.deepcopy` of the env."""
    from .envs.common.action import DiscreteMetaAction

    if getattr(env, "multi_agent", False) or getattr(env, "n_agents", 1) > 1:
        raise NotImplementedError(f"{planner} of a multi-agent env")
    if env.ENV_ID not in OPD_ENV_IDS:
        raise NotImplementedError(f"{planner} on {env.ENV_ID} (supported: {', '.join(OPD_ENV_IDS)})")
    if not isinstance(getattr(env, "action_type", None), DiscreteMetaAction):
        raise ValueError(f"{planner} plans over the 5 DiscreteMetaAction actions of an MDPVehicle ego")


class OpdPolicy:
    """Optimistic deterministic planning (Hren & Munos 2008; rl-agents' `DeterministicPlannerAgent`, which the
    reference's quickstart runs on highway-fast-v0 with `budget: 50, gamma: 0.7`) on the simulator itself, for every
    env of a batched env at once.  The statement it follows is tests/opd_spec.py.

    Per root env, a tree of M = 1 + 5 E nodes (E = budget // 5 expansions) lives in a *store* env of N * M rows, one
    per node; a *work* env of N * 5 rows steps a leaf's state once per action.  Expansion k:

      1. hwy_opd_select picks, per root, the open leaf with the largest upper bound;
      2. work.copy_envs: the leaf's store row into the root's 5 work rows;
      3. the leaf's available actions (hwy_available_actions) and work.step(0..4);
      4. store.copy_envs: the work rows into the child rows 1 + 5 k + a;
      5. hwy_opd_record writes the children's records.

    `act()` returns int64 actions [N] on the env's device: the root child whose subtree holds the largest value.
    Buffers and the two envs are built at the first call (and again only if the env's size changes); later calls make
    no host synchronisation and no allocation, so `act()` can be captured in a CUDA graph.  `tree` holds the last
    decision's trees as [N, M] device tensors (exists, parent, action, depth, reward, value, upper, terminal,
    expanded) and `selected` [N, E]."""

    def __init__(self, env, budget: int = 50, gamma: float = 0.7):
        _check_tree_search_env(env, "OPD")
        if not 0.0 <= float(gamma) < 1.0:
            raise ValueError("gamma must be in [0, 1)")
        if int(budget) != budget or budget < N_ACTIONS:
            raise ValueError(f"budget must be an int >= {N_ACTIONS} (the number of actions)")
        self.env, self.budget, self.gamma = env, int(budget), float(gamma)
        self.expansions = self.budget // N_ACTIONS
        self.max_nodes = 1 + N_ACTIONS * self.expansions
        self._key = None
        self.store = self.work = self.tree = self.selected = self.actions = None

    def _allocate(self) -> None:
        env, n, M, E, dev = self.env, self.env.num_envs, self.max_nodes, self.expansions, self.env.device
        cls, cfg = type(env), copy.deepcopy(env.config)
        self.store = cls(config=cfg, num_envs=n * M, device=dev, autoreset_mode="Disabled")
        self.work = cls(config=copy.deepcopy(cfg), num_envs=n * N_ACTIONS, device=dev, autoreset_mode="Disabled")
        # every row is written by copy_envs before anything reads it: no streams to seed
        self.store._seeded = self.work._seeded = True
        z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=dev)  # noqa: E731
        g, t = opd_discount_tables(self.gamma, E)
        self._g, self._t = torch.from_numpy(g).to(dev), torch.from_numpy(t).to(dev)
        tr = {name: z(n, M, dtype=torch.uint8) for name in ("exists", "expanded", "terminal")}
        tr.update({name: z(n, M, dtype=torch.int32) for name in ("parent", "action", "depth", "branch")})
        tr.update({name: z(n, M, dtype=torch.float64) for name in ("reward", "value", "upper")})
        self._buffers = tr
        self.selected = z(n, E, dtype=torch.int32)
        self.actions = z(n, dtype=torch.int64)
        self._leaf_row = z(n * N_ACTIONS, dtype=torch.int64)
        self._available = z(n * N_ACTIONS, N_ACTIONS, dtype=torch.uint8)
        T = N.HwyOpdTree()
        T.n_roots, T.max_nodes, T.expansions, T.n_actions = n, M, E, N_ACTIONS
        T.discount, T.bound = self._g.data_ptr(), self._t.data_ptr()
        for name, buf in tr.items():
            setattr(T, name, buf.data_ptr())
        T.selected, T.leaf_row, T.recommended = self.selected.data_ptr(), self._leaf_row.data_ptr(), self.actions.data_ptr()
        self._T = T
        self.tree = SimpleNamespace(**{k: (v.view(torch.bool) if v.dtype == torch.uint8 else v) for k, v in tr.items()},
                                    selected=self.selected)
        # row indices: root r -> store row r M; work row r 5 + a; child of expansion k -> store row r M + 1 + 5 k + a
        roots = torch.arange(n, dtype=torch.int64, device=dev)
        self._root_src, self._root_dst = roots, roots * M
        self._work_rows = torch.arange(n * N_ACTIONS, dtype=torch.int64, device=dev)
        a = torch.arange(N_ACTIONS, dtype=torch.int64, device=dev)
        self._child_rows = [((roots * M)[:, None] + 1 + N_ACTIONS * k + a[None, :]).reshape(-1).contiguous()
                            for k in range(E)]
        self._work_actions = a.to(torch.int32).repeat(n)
        self._leaf_table = self.work._row_copy_table(self.store)
        self._child_table = self.store._row_copy_table(self.work)
        self._key = (n, dev, env.V, str(env._row_layout()))

    def act(self) -> torch.Tensor:
        env = self.env
        if not env._seeded:
            raise RuntimeError("call reset() before act()")
        if (env.num_envs, env.device, env.V, str(env._row_layout())) != self._key:
            self._allocate()
        store, work, lib, T = self.store, self.work, env._lib, C.byref(self._T)
        # the root states into node 0, unchecked (the checks of copy_envs read the indices back); the env's buffers may
        # have been re-allocated since the last call, so its table is built again
        store._copy_rows(store._row_copy_table(env), self._root_dst, self._root_src)
        stream = env._stream()
        with torch.cuda.device(env.device):
            for k in range(self.expansions):
                N.check(lib.hwy_opd_select(T, k, stream))
                work._copy_rows(self._leaf_table, self._work_rows, self._leaf_row)
                work._available_actions(self._available)
                work.step(self._work_actions)
                store._copy_rows(self._child_table, self._child_rows[k], self._work_rows)
                N.check(lib.hwy_opd_record(T, k, self._available.data_ptr(), work._reward.data_ptr(),
                                           work._terminated.data_ptr(), work._truncated.data_ptr(), stream))
            N.check(lib.hwy_opd_recommend(T, stream))
        return self.actions


MCTS_ENV_IDS = OPD_ENV_IDS


def mcts_budget(budget: int, gamma: float):
    """(episodes, horizon) of a budget, rl-agents' `AbstractPlanner.allocate_budget`:
    horizon(E) = max(ceil(ln E / (2 ln(1 / gamma))), 1) and episodes = the largest E >= 1 with E * horizon(E) <= budget
    (100 at gamma 0.7 is 20 x 5).  gamma must lie in (0, 1); a budget with no split raises ValueError."""
    if not 0.0 < float(gamma) < 1.0:
        raise ValueError("gamma must be in (0, 1)")
    if int(budget) != budget or budget < 1:
        raise ValueError(f"budget {budget} has no split into episodes x horizon (it must be an int >= 1)")

    def horizon(e: int) -> int:
        return max(int(np.ceil(np.log(np.float64(e)) / (2 * np.log(1 / np.float64(gamma))))), 1)

    e = 1
    while (e + 1) * horizon(e + 1) <= budget:
        e += 1
    return e, horizon(e)


class MctsPolicy:
    """Open-loop Monte-Carlo tree search (rl-agents' `MCTSAgent` with its `random_available` prior and rollout
    policies) on the simulator itself, for every env of a batched env at once.  The statement it follows, with its
    deviations from rl-agents, is tests/mcts_spec.py.

    `budget` is split into `episodes` x `horizon` (`mcts_budget`).  Each episode of each root re-simulates from a copy
    of the root's state in a *work* env of N rows (the caller's class and config, autoreset disabled): it descends the
    tree by `value + T * n_children * prior / (count + 1)` (exact ties by a draw), expands the leaf over its available
    actions, rolls out uniformly random available actions to the horizon, and backs the discounted return up to the
    root.  `act()` returns int64 actions [N] on the env's device: the root child with the most visits (ties by value,
    then the lowest action).  `temperature = 1.0` is this library's default; rl-agents' own default is not restated
    here because it cannot be checked against the reference.

    Draws come from a counter-based generator keyed by (seed, decision, root, episode, depth); `decision` counts
    `act()` calls on the device, so a replayed CUDA graph draws fresh numbers.  A tree holds M = 1 + 5 *
    max_expansions slots (default: `episodes`, or 4 * `episodes` with `reuse_subtree`); an expansion that does not fit
    is skipped and counted in `tree.skipped`.

    With `reuse_subtree=True`, `advance(actions, done)` after each `env.step` keeps the subtree under the action taken
    (rl-agents' `step_strategy: "subtree"`) and clears the trees of rows that are done or whose action has no child;
    `act()` twice without `advance()` in between raises.  Without it every `act()` starts from a bare root and
    `advance()` does nothing.  Buffers and the work env are built at the first call (and again, with a fresh tree and
    decision counter, only if the env's size changes); later `act()` / `advance()` calls make no host synchronisation
    and can be captured in a CUDA graph.  The caller's env is only read.

    `tree` holds [N, M] device tensors (exists, expanded, parent, action, child_base, n_children, prior, count, value),
    `n_nodes` and `skipped` [N], and the last decision's `leaf` / `returns` [N, episodes] (the node each episode backed
    up from and its discounted return)."""

    FIELDS = ("exists", "expanded", "parent", "action", "child_base", "n_children", "prior", "count", "value")

    def __init__(self, env, budget: int = 100, gamma: float = 0.7, temperature: float = 1.0, seed: int = 0,
                 reuse_subtree: bool = False, max_expansions=None):
        _check_tree_search_env(env, "MCTS")
        self.episodes, self.horizon = mcts_budget(budget, gamma)
        temperature = float(temperature)
        if not (np.isfinite(temperature) and temperature >= 0.0):
            raise ValueError("temperature must be finite and >= 0")
        if max_expansions is None:
            max_expansions = self.episodes * (4 if reuse_subtree else 1)
        if int(max_expansions) != max_expansions or max_expansions < 1:
            raise ValueError("max_expansions must be an int >= 1")
        self.env, self.budget, self.gamma, self.temperature = env, int(budget), float(gamma), temperature
        self.seed, self.reuse_subtree = int(seed) & (2**64 - 1), bool(reuse_subtree)
        self.max_expansions = int(max_expansions)
        self.max_nodes = 1 + N_ACTIONS * self.max_expansions
        self._key = None
        self._awaiting_advance = False
        self.work = self.tree = self.actions = self.decision = None

    def _allocate(self) -> None:
        env, n, M, E, dev = self.env, self.env.num_envs, self.max_nodes, self.episodes, self.env.device
        self.work = type(env)(config=copy.deepcopy(env.config), num_envs=n, device=dev, autoreset_mode="Disabled")
        self.work._seeded = True  # every row is written by a row copy before anything reads it
        z = lambda *shape, dtype: torch.zeros(*shape, dtype=dtype, device=dev)  # noqa: E731
        self._g = torch.from_numpy(np.float64(self.gamma) ** np.arange(self.horizon, dtype=np.float64)).to(dev)
        self.decision = z(1, dtype=torch.int64)
        tr = {name: z(n, M, dtype=torch.uint8) for name in ("exists", "expanded")}
        tr.update({name: z(n, M, dtype=torch.int32) for name in ("parent", "action", "child_base", "n_children",
                                                                 "count")})
        tr.update({name: z(n, M, dtype=torch.float64) for name in ("prior", "value")})
        per_root = {"n_nodes": z(n, dtype=torch.int32), "skipped": z(n, dtype=torch.int32),
                    "walk_node": z(n, dtype=torch.int32), "walk_return": z(n, dtype=torch.float64),
                    "walk_flags": z(n, dtype=torch.uint8), "leaf": z(n, E, dtype=torch.int32),
                    "returns": z(n, E, dtype=torch.float64), "remap": z(n, M, dtype=torch.int32)}
        self._work_actions = z(n, dtype=torch.int32)
        self.actions = z(n, dtype=torch.int64)
        self._adv_actions, self._adv_done = z(n, dtype=torch.int64), z(n, dtype=torch.uint8)
        self._available = z(n, N_ACTIONS, dtype=torch.uint8)
        self._buffers = {**tr, **per_root}
        T = N.HwyMctsTree()
        T.n_roots, T.max_nodes, T.episodes, T.horizon = n, M, E, self.horizon
        T.temperature, T.seed = self.temperature, self.seed
        T.discount, T.decision = self._g.data_ptr(), self.decision.data_ptr()
        for name, buf in self._buffers.items():
            setattr(T, name, buf.data_ptr())
        T.actions, T.recommended = self._work_actions.data_ptr(), self.actions.data_ptr()
        self._T = T
        self.tree = SimpleNamespace(**{k: (v.view(torch.bool) if v.dtype == torch.uint8 else v) for k, v in tr.items()},
                                    n_nodes=per_root["n_nodes"], skipped=per_root["skipped"], leaf=per_root["leaf"],
                                    returns=per_root["returns"])
        self._rows = torch.arange(n, dtype=torch.int64, device=dev)
        self._key = (n, dev, env.V, str(env._row_layout()))
        self._reroot(None, None)  # bare roots
        self._awaiting_advance = False

    def _reroot(self, actions, done) -> None:
        with torch.cuda.device(self.env.device):
            N.check(self.env._lib.hwy_mcts_reroot(C.byref(self._T), None if actions is None else actions.data_ptr(),
                                                  None if done is None else done.data_ptr(), self.env._stream()))

    def act(self) -> torch.Tensor:
        env = self.env
        if not env._seeded:
            raise RuntimeError("call reset() before act()")
        if (env.num_envs, env.device, env.V, str(env._row_layout())) != self._key:
            self._allocate()
        if self._awaiting_advance:
            raise RuntimeError("reuse_subtree: call advance(actions, done) after env.step and before the next act()")
        if not self.reuse_subtree:
            self._reroot(None, None)
        work, lib, T, stream = self.work, env._lib, C.byref(self._T), env._stream()
        # the env's buffers may have been re-allocated since the last call: its table is built again
        table = work._row_copy_table(env)
        with torch.cuda.device(env.device):
            for e in range(self.episodes):
                work._copy_rows(table, self._rows, self._rows)
                for d in range(self.horizon):
                    work._available_actions(self._available)
                    N.check(lib.hwy_mcts_advance(T, e, d, self._available.data_ptr(), work._reward.data_ptr(),
                                                 work._terminated.data_ptr(), work._truncated.data_ptr(), stream))
                    work.step(self._work_actions)
                N.check(lib.hwy_mcts_backup(T, e, work._reward.data_ptr(), stream))
            N.check(lib.hwy_mcts_recommend(T, stream))
        self._awaiting_advance = self.reuse_subtree
        return self.actions

    def advance(self, actions, done) -> None:
        """After `env.step(actions)`: re-root every tree at the child of the action taken (`reuse_subtree`), clearing
        the rows where `done` (bool [N], e.g. terminated | truncated) or the action has no child.  A no-op without
        `reuse_subtree`.  Device tensors keep it free of host synchronisation."""
        if not self.reuse_subtree:
            return
        if self._key is None:
            raise RuntimeError("advance() before the first act()")
        n = self.env.num_envs
        actions, done = torch.as_tensor(actions), torch.as_tensor(done)
        if actions.numel() != n or done.numel() != n:
            raise ValueError(f"advance() takes one action and one done flag per env ({n})")
        self._adv_actions.copy_(actions.reshape(n), non_blocking=True)
        self._adv_done.copy_(done.reshape(n), non_blocking=True)
        self._reroot(self._adv_actions, self._adv_done)
        self._awaiting_advance = False
