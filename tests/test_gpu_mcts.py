"""`planning.MctsPolicy`: open-loop MCTS over env clones (a work env stepped through `copy_envs`' row copies, tree
kernels in csrc/hwy_plan.cu), against the numpy statement of tests/mcts_spec.py — run over the unmodified reference
(fixtures mcts_*.npz, `copy.deepcopy` + `step`) and over this library's own `copy_envs`, `get_available_actions` and
`step` — plus subtree reuse, the caller's env left untouched, sync-free calls, CUDA-graph replay and rejections."""
import numpy as np
import pytest

from mcts_spec import FIELDS, FIXTURES, N_ACTIONS, advance, budget_split, empty_tree, load, plan
from test_gpu_opd import make_from_fixture

pytestmark = pytest.mark.gpu

MARGIN = 1e-9  # descent choices and recommendations closer than this are ties up to rounding: not compared
VALUE_TOL = 1e-6  # returns accumulated over up to 5 free-running steps (positions agree to 1e-5)
TREE_EXACT = ("exists", "expanded", "parent", "action", "child_base", "n_children", "prior", "count")
LINEAR = {"other_vehicles_type": "highway_env.vehicle.behavior.LinearVehicle"}


def host_tree(policy):
    t = {k: getattr(policy.tree, k).cpu().numpy() for k in FIELDS + ("n_nodes", "skipped", "leaf", "returns")}
    t["recommended"] = policy.actions.cpu().numpy()
    return t


@pytest.mark.parametrize("name", FIXTURES)
def test_mcts_trees_equal_the_reference(name):
    from highwayenv_b200 import planning

    g = load(name)
    cfg = g["config"]
    ref, out = g["tree"], g["out"]
    env = make_from_fixture(g)
    policy = planning.MctsPolicy(env, budget=cfg["_budget"], gamma=cfg["_gamma"], temperature=cfg["_temperature"],
                                 seed=cfg["_seed"])
    policy.act()
    got = host_tree(policy)
    n, E = out["margin"].shape
    compared_recs, whole_trees, worst = 0, 0, 0.0
    for i in range(n):
        # the walks agree up to the first episode whose descent had a runner-up within rounding of the choice
        close = np.nonzero(out["margin"][i] < MARGIN)[0]
        k_star = int(close[0]) if close.size else E
        assert np.array_equal(got["leaf"][i, :k_star], out["leaf"][i, :k_star]), (name, i)
        d = np.abs(got["returns"][i, :k_star] - out["ret"][i, :k_star])
        worst = max(worst, float(d.max(initial=0.0)))
        assert d.max(initial=0.0) <= VALUE_TOL, (name, i, d.max())
        if k_star < E:
            continue
        whole_trees += 1
        for k in TREE_EXACT + ("n_nodes", "skipped"):
            assert np.array_equal(got[k][i], ref[k][i]), (name, i, k)
        d = np.abs(got["value"][i] - ref["value"][i])
        worst = max(worst, float(d.max()))
        assert d.max() <= VALUE_TOL, (name, i, d.max())
        if out["recommended_margin"][i] >= MARGIN:
            assert got["recommended"][i] == out["recommended"][i], (name, i)
            compared_recs += 1
    print(f"{name}: whole trees compared on {whole_trees} of {n} roots, recommended action on {compared_recs} "
          f"(the rest hold a choice within {MARGIN}); worst value difference {worst:.3g}")
    assert compared_recs >= n // 2


def library_callbacks(env, n):
    """The spec's callbacks over this library: a work env of n rows and the public `copy_envs`,
    `get_available_actions` and `step`."""
    import highwayenv_b200 as hb
    import torch

    work = hb.make(env.ENV_ID, num_envs=n, config=dict(env.config), autoreset_mode="Disabled")
    rows = np.arange(n)

    def begin_episode():
        work.copy_envs(rows, rows, source=env)

    def available():
        return work.get_available_actions().cpu().numpy()

    def step(actions):
        _, r, te, tr, _ = work.step(torch.as_tensor(actions, dtype=torch.int32, device=env.device))
        return r.cpu().numpy(), (te | tr).cpu().numpy()

    return begin_episode, available, step


def assert_equal_to_spec(policy, tree, out, tag):
    got = host_tree(policy)
    for k in FIELDS + ("n_nodes", "skipped"):
        assert np.ascontiguousarray(got[k]).tobytes() == np.ascontiguousarray(
            tree[k].astype(got[k].dtype)).tobytes(), (tag, k)
    assert got["leaf"].tobytes() == out["leaf"].tobytes(), tag
    assert got["returns"].tobytes() == out["ret"].tobytes(), tag
    assert np.array_equal(got["recommended"], out["recommended"]), tag


def _rolled_env(env_id, config, n, seed=77):
    import highwayenv_b200 as hb

    env = hb.make(env_id, num_envs=n, config=dict(config or {}))
    env.reset(seed=seed)
    rng = np.random.default_rng(0)
    for _ in range(3):
        env.step(rng.integers(0, N_ACTIONS, size=n).astype(np.int32))
    return env


@pytest.mark.parametrize("env_id,config", [("highway-fast-v0", None), ("roundabout-v0", None),
                                           ("highway-v0", LINEAR)])
def test_mcts_equals_the_spec_over_the_library(env_id, config):
    from highwayenv_b200 import planning

    n = 64
    env = _rolled_env(env_id, config, n)
    # budget 100 at gamma 0.7 (20 x 5), and 23 at gamma 0.5 (11 x 2: 1 unused) with another temperature and seed
    for budget, gamma, temperature, seed in ((100, 0.7, 1.0, 0), (23, 0.5, 0.3, 99)):
        policy = planning.MctsPolicy(env, budget=budget, gamma=gamma, temperature=temperature, seed=seed)
        policy.act()
        episodes, horizon = budget_split(budget, gamma)
        assert (policy.episodes, policy.horizon) == (episodes, horizon)
        tree = empty_tree(n, 1 + N_ACTIONS * episodes)
        out = plan(tree, episodes, horizon, gamma, temperature, seed, 0, *library_callbacks(env, n))
        assert_equal_to_spec(policy, tree, out, (env_id, budget))


@pytest.mark.parametrize("max_expansions", [None, 3])
@pytest.mark.parametrize("env_id,config", [("highway-fast-v0", None), ("roundabout-v0", None),
                                           ("highway-v0", LINEAR)])
def test_subtree_reuse_equals_the_spec_over_the_library(env_id, config, max_expansions):
    """4 consecutive decisions with reuse_subtree: the policy's trees, re-rooted by advance(), equal the spec's at
    every decision; some rows are cleared by done and some by an action without a child.  With room for 3 expansions
    the trees fill up (a chain from the root to the horizon alone takes 4 at budget 50) and expansions are skipped."""
    import torch
    from highwayenv_b200 import planning

    n, budget, gamma, seed = 64, 50, 0.7, 5
    env = _rolled_env(env_id, config, n, seed=78)
    policy = planning.MctsPolicy(env, budget=budget, gamma=gamma, seed=seed, reuse_subtree=True,
                                 max_expansions=max_expansions)
    episodes, horizon = budget_split(budget, gamma)
    tree = empty_tree(n, policy.max_nodes)
    cleared = skipped = 0
    for decision in range(4):
        policy.act()
        out = plan(tree, episodes, horizon, gamma, 1.0, seed, decision, *library_callbacks(env, n))
        assert_equal_to_spec(policy, tree, out, (env_id, decision))
        skipped += int(tree["skipped"].sum())
        actions = out["recommended"].copy()
        actions[decision::7] = 0  # LANE_LEFT: no child where it is not available
        _, _, term, trunc, _ = env.step(torch.as_tensor(actions, dtype=torch.int32, device=env.device))
        done = (term | trunc).cpu().numpy()
        done[3::11] = True
        base = tree["child_base"][:, 0]
        cleared += int(sum(done[i] or not tree["exists"][i, base[i] + actions[i]] for i in range(n)))
        policy.advance(torch.as_tensor(actions, device=env.device), torch.as_tensor(done, device=env.device))
        advance(tree, actions, done)
        got = host_tree(policy)
        for k in FIELDS + ("n_nodes",):
            assert np.ascontiguousarray(got[k]).tobytes() == np.ascontiguousarray(
                tree[k].astype(got[k].dtype)).tobytes(), (env_id, decision, k)
    print(f"{env_id}: {cleared} trees cleared and {skipped} expansions skipped over 4 decisions")
    assert cleared > 0 and (skipped > 0 or max_expansions is None)


def test_the_callers_env_is_untouched():
    from highwayenv_b200 import planning

    env = _rolled_env("roundabout-v0", None, 96)
    before_sd, before_rng = env.state_dict(), env.rng_words()
    before_obs = env._obs.clone()
    policy = planning.MctsPolicy(env, reuse_subtree=True)
    policy.act()
    after_sd = env.state_dict()
    for k in before_sd:
        assert np.asarray(before_sd[k]).tobytes() == np.asarray(after_sd[k]).tobytes(), k
    assert env.rng_words().tobytes() == before_rng.tobytes()
    assert env._obs.equal(before_obs)


def test_calls_do_not_sync_and_replay_in_cuda_graphs():
    import highwayenv_b200 as hb
    import torch
    from highwayenv_b200 import planning

    n = 128
    env_a = hb.make("highway-fast-v0", num_envs=n, autoreset_mode="Disabled")
    env_a.reset(seed=3)
    env_b = hb.make("highway-fast-v0", num_envs=n, autoreset_mode="Disabled")
    env_b.reset(seed=4)
    env_b.copy_envs(np.arange(n), np.arange(n), source=env_a)
    eager = planning.MctsPolicy(env_a, budget=50, seed=11, reuse_subtree=True)
    graphed = planning.MctsPolicy(env_b, budget=50, seed=11, reuse_subtree=True)
    done_a = torch.zeros(n, dtype=torch.bool, device="cuda")
    eager.act()
    eager.advance(eager.actions, done_a)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:  # the second act() and advance()
        eager.act()
        eager.advance(eager.actions, done_a)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    # the graphed policy catches up eagerly (2 decisions), then captures one act() and one advance()
    for _ in range(2):
        graphed.act()
        graphed.advance(graphed.actions, done_a)
    static_actions = torch.zeros(n, dtype=torch.int64, device="cuda")
    static_done = torch.zeros(n, dtype=torch.bool, device="cuda")
    g_act, g_adv = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g_act):  # capture records the launches without running them
        graphed.act()
    with torch.cuda.graph(g_adv):
        graphed.advance(static_actions, static_done)
    for step in range(4):
        a = eager.act().clone()
        g_act.replay()
        torch.cuda.synchronize()
        assert torch.equal(a, graphed.actions), step
        for k in FIELDS:
            assert torch.equal(getattr(eager.tree, k), getattr(graphed.tree, k)), (step, k)
        _, _, te, tr, _ = env_a.step(a)
        done = (te | tr).clone()
        _, _, te_b, tr_b, _ = env_b.step(a)
        assert torch.equal(done, te_b | tr_b)
        eager.advance(a, done)
        static_actions.copy_(a)
        static_done.copy_(done)
        g_adv.replay()
        torch.cuda.synchronize()
        for k in FIELDS + ("n_nodes",):
            assert torch.equal(getattr(eager.tree, k), getattr(graphed.tree, k)), (step, k)
    assert int(eager.decision) == int(graphed.decision) == 6


def test_reuse_needs_advance_between_decisions():
    import highwayenv_b200 as hb
    from highwayenv_b200 import planning

    env = hb.make("highway-fast-v0", num_envs=4)
    env.reset(seed=1)
    policy = planning.MctsPolicy(env, budget=10, reuse_subtree=True)
    policy.act()
    with pytest.raises(RuntimeError):
        policy.act()
    policy.advance(policy.actions, np.zeros(4, bool))
    policy.act()
    plain = planning.MctsPolicy(env, budget=10)
    plain.act()
    plain.act()  # without reuse every act() starts from a bare root
    assert int(plain.tree.count[:, 0].max()) == plain.episodes


@pytest.mark.parametrize("env_id,config,kw,error", [
    ("intersection-multi-agent-v0", None, {}, NotImplementedError),
    ("intersection-v0", None, {}, NotImplementedError),
    ("two-way-v0", None, {}, NotImplementedError),
    ("highway-fast-v0", {"action": {"type": "ContinuousAction"}}, {}, ValueError),
    ("highway-fast-v0", None, {"gamma": 1.0}, ValueError),
    ("highway-fast-v0", None, {"gamma": 0.0}, ValueError),
    ("highway-fast-v0", None, {"budget": 0}, ValueError),
    ("highway-fast-v0", None, {"temperature": -1.0}, ValueError),
    ("highway-fast-v0", None, {"temperature": float("inf")}, ValueError),
    ("highway-fast-v0", None, {"temperature": float("nan")}, ValueError),
    ("highway-fast-v0", None, {"max_expansions": 0}, ValueError),
])
def test_rejected_configurations(env_id, config, kw, error):
    import highwayenv_b200 as hb
    from highwayenv_b200 import planning

    env = hb.make(env_id, num_envs=2, config=dict(config or {}))
    with pytest.raises(error):
        planning.MctsPolicy(env, **kw)
