"""Masked device resets of the scripted network families (roundabout, merge, two-way, u-turn, exit): a reset writes
exactly the envs its masks select, and a selected env comes out byte-identical to the same env under an unmasked
reset."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ENV_IDS = ["roundabout-v0", "merge-v0", "two-way-v0", "u-turn-v0", "exit-v0"]
N = 257  # the warp-per-env (roundabout) and thread-per-env kernels both end in a partial block


def rows(env):
    """Every per-env tensor the env reads later, and the streams, as host arrays with a leading env axis."""
    out = {k: t.cpu().contiguous().numpy() for k, t in env._env_rows().items()}
    out["rng_words"] = env.rng_words().T
    return out


def assert_rows(a, ia, b, ib, ctx):
    for k in a:
        x, y = np.ascontiguousarray(a[k][ia]), np.ascontiguousarray(b[k][ib])
        assert x.shape == y.shape and x.tobytes() == y.tobytes(), (ctx, k)


def stepped_env(env_id):
    import highwayenv_b200 as hb

    env = hb.make(env_id, num_envs=N, autoreset_mode="Disabled")
    env.reset(seed=[1000 + 7 * i for i in range(N)])
    rng = np.random.default_rng(5)
    for _ in range(3):
        env.step(rng.integers(0, env.single_action_space.n, size=N).astype(np.int32))
    return env


def reset_mask(env, sel):
    env.reset(options={"reset_mask": sel.astype(np.uint8)})


def two_masks(env, sel):
    """The gate SameStep autoreset uses: two device masks (terminated, truncated), either selects an env."""
    import torch

    i = np.arange(N)
    a = torch.from_numpy((sel & (i % 2 == 0)).astype(np.uint8)).cuda()
    b = torch.from_numpy((sel & ((i % 2 == 1) | (i % 3 == 0))).astype(np.uint8)).cuda()  # overlaps a on i % 6 == 0
    assert ((a.cpu().numpy() | b.cpu().numpy()) == sel).all()
    env._device_reset(a.data_ptr(), b.data_ptr(), env._fused_out.data_ptr())
    if env._plugin_standalone:
        env._observe_plugin(env._obs, a, b)
    torch.cuda.synchronize()


@pytest.mark.parametrize("gate", [reset_mask, two_masks], ids=["reset_mask", "two_masks"])
@pytest.mark.parametrize("env_id", ENV_IDS)
def test_masked_reset_writes_the_selected_envs_as_a_full_reset(env_id, gate):
    import highwayenv_b200 as hb

    a = stepped_env(env_id)
    a.observe()
    before = rows(a)
    b = hb.make(env_id, num_envs=N, autoreset_mode="Disabled")
    b.copy_envs(np.arange(N), np.arange(N), source=a)
    assert_rows(before, slice(None), rows(b), slice(None), (env_id, "copy"))

    i = np.arange(N)
    sel = (i % 5 == 0) | (i % 7 == 3) | (i >= N - 2)  # the last envs sit in the last, partial block
    gate(a, sel)
    b.reset()  # every env, from the same streams
    after, full = rows(a), rows(b)
    assert_rows(before, ~sel, after, ~sel, (env_id, gate.__name__, "unselected"))
    assert_rows(full, sel, after, sel, (env_id, gate.__name__, "selected"))
    assert (after["_time"][sel] == 0).all() and (before["_time"][sel] > 0).all()
