"""The batched gym surface every env family shares (envs/common/vector_env.py): argument checks that must fail on the
host before any kernel launch, and how the env streams carry over state_dict loads and re-allocations."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FAMILIES = ["highway-fast-v0", "roundabout-v0", "merge-v0", "exit-v0", "intersection-v0"]


@pytest.mark.parametrize("env_id", FAMILIES)
def test_bad_arguments_raise_before_any_launch(env_id):
    import highwayenv_b200 as hb
    from highwayenv_b200 import _native as N

    lib = N.load()
    n = 4
    with pytest.raises(ValueError):
        hb.make(env_id, num_envs=0)
    with pytest.raises(RuntimeError):
        hb.make(env_id, num_envs=n, device="cpu")
    env = hb.make(env_id, num_envs=n)
    launches = lib.hwy_launch_count()
    for seeds in ([1, 2, 3], [1, 2, 3, 4, 5]):
        with pytest.raises(ValueError):
            env.reset(seed=seeds)
    for m in (3, 5):
        with pytest.raises(ValueError):
            env.reset(seed=0, options={"reset_mask": np.ones(m, dtype=bool)})
    with pytest.raises(ValueError):
        env.reset(seed=0, options={"reset_mask": np.ones((n, 1), dtype=bool)})
    assert lib.hwy_launch_count() == launches
    env.reset(seed=[10, 11, 12, 13], options={"reset_mask": np.ones(n, dtype=bool)})  # the right shapes pass


@pytest.mark.parametrize("env_id", ["highway-fast-v0", "intersection-v0"])
def test_loaded_streams_survive_an_unseeded_reset(env_id):
    """load_state_dict(rng) then reset() without a seed continues the loaded streams, like the reference's np_random;
    an env never seeded takes the streams reset(seed=0) would give it."""
    import highwayenv_b200 as hb
    from highwayenv_b200.envs.common.vector_env import pcg64_words

    n = 16
    ref = hb.make(env_id, num_envs=n)
    ref.reset(seed=11)
    sd = ref.state_dict()
    obs_ref, _ = ref.reset()
    env = hb.make(env_id, num_envs=n)
    env.load_state_dict(sd)
    obs, _ = env.reset()
    assert np.array_equal(env.rng_words(), ref.rng_words())
    assert np.array_equal(obs.cpu().numpy(), obs_ref.cpu().numpy())

    unseeded = hb.make(env_id, num_envs=n)
    unseeded.load_state_dict({k: v for k, v in sd.items() if k != "rng"})
    want = pcg64_words([np.random.Generator(np.random.PCG64(np.random.SeedSequence(i))) for i in range(n)])
    assert np.array_equal(unseeded.rng_words(), want)


def test_streams_survive_a_reallocating_config_reset():
    """reset(options={"config": ...}) re-allocates the device buffers; the env streams carry over, so two envs with
    the same seed stay identical."""
    import highwayenv_b200 as hb

    envs = [hb.make("highway-fast-v0", num_envs=8) for _ in range(2)]
    for e in envs:
        e.reset(seed=3)
    a, b = (e.reset(options={"config": {"vehicles_count": 30}})[0].cpu().numpy() for e in envs)
    assert np.array_equal(a, b)
    assert np.array_equal(envs[0].rng_words(), envs[1].rng_words())
