"""bench.py --dump-outputs: every array as float32 / float64 .npy, whole outputs whenever they fit the budget together,
a fixed seeded row sample (with its row list) only beyond that, and never more bytes than the budget."""
import os

import numpy as np

import bench


def _outputs(n_small, n_big, width):
    rng = np.random.default_rng(5)
    return {
        "cfgA": {"cfgA_obs": rng.random((n_small, 4), dtype=np.float32), "cfgA_reward": rng.random(n_small),
                 "cfgA_terminated": rng.random(n_small) < 0.5},
        "cfgB": {"cfgB_obs": rng.random((n_big, width), dtype=np.float32), "cfgB_reward": rng.random(n_big),
                 "cfgB_terminated": rng.random(n_big) < 0.5},
    }


def _dir_bytes(d):
    return sum(os.path.getsize(os.path.join(d, f)) for f in os.listdir(d))


def test_dump_keeps_whole_outputs_when_they_fit_together(tmp_path):
    out = _outputs(100, 2000, 16)  # cfgB alone is more than half of the budget, both fit
    bench.dump_outputs(out, str(tmp_path), budget=200_000)
    assert not any(f.endswith("_rows.npy") for f in os.listdir(tmp_path))
    for arrays in out.values():
        for k, v in arrays.items():
            got = np.load(tmp_path / (k + ".npy"))
            assert got.dtype == (np.float64 if v.dtype == np.float64 else np.float32)
            assert np.array_equal(got, v.astype(got.dtype))
    assert _dir_bytes(tmp_path) <= 200_000


def test_dump_samples_fixed_rows_within_the_budget(tmp_path):
    out = _outputs(100, 20000, 16)
    for d in ("a", "b"):
        bench.dump_outputs(out, str(tmp_path / d), budget=200_000)
        assert _dir_bytes(tmp_path / d) <= 200_000
    a, b = tmp_path / "a", tmp_path / "b"
    assert sorted(os.listdir(a)) == sorted(os.listdir(b))
    for f in os.listdir(a):
        assert np.array_equal(np.load(a / f), np.load(b / f))
    assert not (a / "cfgA_rows.npy").exists() and np.array_equal(np.load(a / "cfgA_obs.npy"), out["cfgA"]["cfgA_obs"])
    rows = np.load(a / "cfgB_rows.npy").astype(np.int64)
    assert 0 < len(rows) < 20000 and np.all(np.diff(rows) > 0)
    assert np.array_equal(np.load(a / "cfgB_obs.npy"), out["cfgB"]["cfgB_obs"][rows])
    assert np.array_equal(np.load(a / "cfgB_terminated.npy"), out["cfgB"]["cfgB_terminated"][rows].astype(np.float32))
