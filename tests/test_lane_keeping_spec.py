"""lane-keeping-v0 without a GPU: the fixtures of oracle/gen_lane_keeping.py checked against themselves (stream use per
observe, the exact noise draws of the `state` attribute at the resets, spawn, reward, TimeLimit points), one seed rerun
against the live reference when it is present, the C structs against gcc, and the configuration checks that run before
any launch."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = ["lane_keeping_default", "lane_keeping_pf5", "lane_keeping_reference_state", "lane_keeping_longitudinal"]


def load(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    g["config"] = json.loads(str(g.pop("config_json")))
    return g


def config_of(g):
    return {k: v for k, v in g["config"].items() if not k.startswith("_")}


def generator(words):
    from highwayenv_b200.envs.common.vector_env import set_pcg64_words

    gen = np.random.Generator(np.random.PCG64(0))
    set_pcg64_words([gen], np.asarray(words, dtype=np.uint64).reshape(5, 1))
    return gen


def words(gen):
    from highwayenv_b200.envs.common.vector_env import pcg64_words

    return pcg64_words([gen])[:, 0]


def stream_per_step(g):
    """The stream words after every step ([S, T, 5]) and after each TimeLimit reset ([S, 2, 5]), from the reset's words:
    each observe draws 4 uniforms per noisy attribute (one per word), a reset observes three times."""
    noisy = sum(a != "reference_state" for a in g["attributes"])
    S, T = g["truncated"].shape
    out, resets = np.zeros((S, T, 5), np.uint64), np.zeros((S, 2, 5), np.uint64)
    for i in range(S):
        gen = generator(g["reset_rng"][i])
        for t in range(T):
            gen.random(4 * noisy)
            out[i, t] = words(gen)
            if g["truncated"][i, t]:
                gen.random(3 * 4 * noisy)
                resets[i, (t + 1) // 200 - 1] = words(gen)
    return out, resets


def state_noise(words_before, n_skip, lim):
    """The `state` attribute's noise of the observe that starts after `n_skip` draws from `words_before`."""
    gen = generator(words_before)
    gen.random(n_skip)
    return gen.uniform(-lim, lim, size=(4, 1))


@pytest.mark.parametrize("name", CASES)
def test_fixture_self_consistency(name):
    from highwayenv_b200.envs.lane_keeping_env import lane_keeping_params, make_lane_keeping_network

    g = load(name)
    cfg = config_of(g)
    attrs = list(g["attributes"])
    noisy = sum(a != "reference_state" for a in attrs)
    S, T = g["actions"].shape[:2]
    steps = g["steps"]
    assert (S, T) == (32, 420) and steps.tolist() == list(range(19, 420, 20))
    assert g["obs"].shape == (S, len(steps), len(attrs), 4, 1) and g["state"].shape == (S, len(steps), 6)
    assert g["phase"].shape == g["truncated"].shape == g["speed"].shape == (S, T)
    assert np.array_equal(g["speed"][:, steps], g["state"][..., 3].astype(np.float32))
    # TimeLimit(max_episode_steps=200): truncated after steps 200 and 400, never terminated
    assert g["autoreset_step"].tolist() == [199, 399]
    assert np.array_equal(g["truncated"], np.broadcast_to(np.isin(np.arange(T), [199, 399]), (S, T)))
    # the spawn, in the reset and at both autoresets; the lane phase only moves forward within an episode
    p = lane_keeping_params(cfg)
    spawn = np.array([p.x0, p.y0, p.heading0, p.speed0, 0.0, 0.0])
    assert np.array_equal(g["reset_state"], np.broadcast_to(spawn, (S, 6)))
    assert np.array_equal(g["autoreset_state"], np.broadcast_to(spawn, (S, 2, 6)))
    assert not g["reset_phase"].any() and not g["autoreset_phase"].any()
    d = np.diff(g["phase"].astype(np.int64), axis=1)
    assert (d >= 0).all() or set(np.nonzero(d < 0)[1]) <= {199, 399}
    # stream use: 4 words per noisy attribute per observe, 3 observes per reset (24 words by default)
    per_step, resets = stream_per_step(g)
    assert np.array_equal(per_step[:, steps], g["rng"]) and np.array_equal(resets, g["autoreset_rng"])
    for i, seed in enumerate(g["seeds"]):
        gen = np.random.Generator(np.random.PCG64(np.random.SeedSequence(int(seed))))
        gen.random(3 * 4 * noisy)
        assert np.array_equal(words(gen), g["reset_rng"][i])
    # the returned reset observation: `state` is the spawn plus the noise drawn after the two discarded observes
    if "state" in attrs:
        k, lim = attrs.index("state"), cfg["state_noise"]
        for i, seed in enumerate(g["seeds"]):
            w0 = words(np.random.Generator(np.random.PCG64(np.random.SeedSequence(int(seed)))))
            want = spawn[[1, 2, 4, 5]].reshape(4, 1) + state_noise(w0, 2 * 4 * noisy, lim)
            assert np.array_equal(g["reset_obs"][i, k], want)
            for r, t in enumerate((199, 399)):
                want = spawn[[1, 2, 4, 5]].reshape(4, 1) + state_noise(per_step[i, t], 2 * 4 * noisy, lim)
                assert np.array_equal(g["autoreset_obs"][i, r, k], want)
    # reward 1 - (lat / width) ** 2 on the lane after the step's switch
    net = make_lane_keeping_network()
    lanes = [net.index[("c", "d", 0)], net.index[("a", "b", 0)]]
    for i in range(S):
        for j, t in enumerate(steps):
            st = g["state"][i, j]
            _, lat = net.local_coordinates(lanes[int(g["phase"][i, t])], np.array([st[0]]), np.array([st[1]]))
            assert abs(g["reward"][i, j] - (1 - (float(lat[0]) / 10.0) ** 2)) <= 1e-12, (name, i, t)


def test_defaults_match_reference_config():
    from highwayenv_b200.config import default_config

    import highwayenv_b200 as hb

    assert "lane-keeping-v0" in hb.REGISTRY
    ref = config_of(load("lane_keeping_default"))
    ours = default_config("lane-keeping-v0")
    ours["offscreen_rendering"] = ref["offscreen_rendering"]
    assert ours == ref


@pytest.mark.skipif(not os.path.isdir(os.path.join(os.environ.get("HWY_REFERENCE_ROOT", "/root/reference"),
                                                   "highway_env")), reason="needs the reference checkout")
@pytest.mark.parametrize("name", ["lane_keeping_default", "lane_keeping_longitudinal"])
def test_one_seed_against_live_reference(name):
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import gen_lane_keeping as gl

    g = load(name)
    i = 5
    _, actions, first, steps, rewards, truncs, resets = gl.run_seed(gl.CASES[name], int(g["seeds"][i]))
    keep = g["steps"]
    assert np.array_equal(actions, g["actions"][i])
    assert np.array_equal(first[0], g["reset_obs"][i]) and np.array_equal(first[3], g["reset_rng"][i])
    for k in ("obs", "state", "rng"):
        assert np.array_equal(np.stack(steps[k])[keep], g[k][i]), k
    assert np.array_equal(np.array(steps["phase"]), g["phase"][i])
    assert np.array_equal(np.stack(steps["rng"]), stream_per_step(g)[0][i])  # every step's words
    assert np.array_equal(np.array(rewards)[keep], g["reward"][i])
    assert np.array_equal(np.array(truncs), g["truncated"][i])
    assert np.array_equal(np.stack([r[0] for r in resets]), g["autoreset_obs"][i])


def test_struct_layout_matches_gcc():
    import ctypes as C

    from highwayenv_b200 import _native as N

    fields = {"HwyLaneKeepingParams": ("frames", "attr", "longitudinal", "autoreset", "dt", "speed0", "lanes"),
              "HwyLaneKeepingState": ("state", "lane_phase", "elapsed", "rng")}
    exprs = []
    for struct, names in fields.items():
        exprs.append(f"sizeof({struct})")
        exprs += [f"offsetof({struct}, {f})" for f in names]
    src = ('#include <stddef.h>\n#include <stdio.h>\n#include "hwyb200.h"\nint main(){'
           + "".join(f'printf("%zu\\n", (size_t){e});' for e in exprs) + "return 0;}\n")
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    want = []
    for struct, names in fields.items():
        t = getattr(N, struct)
        want.append(C.sizeof(t))
        want += [getattr(t, f).offset for f in names]
    assert got == want
    hdr = open(os.path.join(ROOT, "include", "hwyb200.h")).read()
    assert "#define HWY_ABI_VERSION 17" in hdr and N.HWY_ABI_VERSION == 17
    assert {"hwy_lane_keeping_reset", "hwy_lane_keeping_step"} <= set(N.EXPORTS)


def _cfg(**over):
    from highwayenv_b200.config import default_config

    cfg = default_config("lane-keeping-v0")
    for k, v in over.items():
        if k in ("observation", "action"):
            cfg[k] = {**cfg[k], **v}
        else:
            cfg[k] = v
    return cfg


def test_supported_configuration_parameters():
    from highwayenv_b200 import _native as N
    from highwayenv_b200.envs.lane_keeping_env import lane_keeping_params

    p = lane_keeping_params(_cfg())
    assert (p.frames, p.n_attr, list(p.attr), p.longitudinal, p.lateral, p.act_clip) == (1, 3, [0, 1, 2], 0, 1, 1)
    assert p.max_episode_steps == 200 and p.autoreset == N.AUTORESET_SAME_STEP and p.dt == 0.1
    assert (p.steer_lo, p.steer_hi, p.acc_lo, p.acc_hi) == (-np.pi / 3, np.pi / 3, -5.0, 5.0)
    assert (p.lanes[0].type, p.lanes[1].type, p.lanes[1].amplitude) == (N.LANE_STRAIGHT, N.LANE_SINE, 5.0)
    p = lane_keeping_params(_cfg(policy_frequency=5, observation={"attributes": ["reference_state", "state"]},
                                 action={"longitudinal": True, "acceleration_range": [-2, 3], "clip": False}),
                            autoreset_mode="NextStep")
    assert (p.frames, p.n_attr, list(p.attr)[:2], p.longitudinal, p.act_clip) == (2, 2, [2, 0], 1, 0)
    assert (p.acc_lo, p.acc_hi, p.autoreset) == (-2.0, 3.0, N.AUTORESET_DISABLED)


@pytest.mark.parametrize("over,exc", [
    ({"observation": {"type": "Kinematics"}}, NotImplementedError),
    ({"observation": {"attributes": ["state", "heading"]}}, ValueError),
    ({"observation": {"attributes": []}}, ValueError),
    ({"observation": {"attributes": ["state", "state"]}}, ValueError),
    ({"action": {"dynamical": False}}, NotImplementedError),
    ({"action": {"type": "DiscreteMetaAction"}}, NotImplementedError),
    ({"action": {"lateral": False, "longitudinal": False}}, ValueError),
    ({"action": {"speed_range": [0, 10]}}, NotImplementedError),
    ({"policy_frequency": 20}, ValueError),
    ({"manual_control": True}, NotImplementedError),
])
def test_unsupported_configuration_raises(over, exc):
    from highwayenv_b200.envs.lane_keeping_env import lane_keeping_params

    with pytest.raises(exc):
        lane_keeping_params(_cfg(**over))


def test_dict_space_fallback_and_batching():
    from highwayenv_b200.spaces import Box, Dict, batch_space

    sp = Dict({"state": Box(-np.inf, np.inf, shape=(4, 1), dtype=np.float64),
               "derivative": Box(-np.inf, np.inf, shape=(4, 1), dtype=np.float64)})
    assert list(sp.spaces) == ["derivative", "state"]  # gymnasium's Dict sorts a plain dict's keys
    b = batch_space(sp, 3)
    assert isinstance(b, Dict) and b["state"].shape == (3, 4, 1) and b["state"].dtype == np.float64
    x = sp.sample()
    assert set(x) == {"state", "derivative"} and sp.contains(x)
