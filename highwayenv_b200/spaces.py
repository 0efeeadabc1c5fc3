"""Observation/action space descriptors.

gymnasium (pinned 1.3.0 by the reference, uv.lock) is not installed in this image; when it
is importable its ``spaces`` are used so the envs plug into RL libraries unchanged,
otherwise these minimal stand-ins with the same attributes (shape, dtype, low/high, n,
sample, contains) are used.
"""
from __future__ import annotations

import numpy as np

try:  # pragma: no cover - depends on the image
    from gymnasium.spaces import Box, Dict, Discrete  # type: ignore

    HAVE_GYMNASIUM = True
except Exception:  # ModuleNotFoundError in this image
    HAVE_GYMNASIUM = False

    class _Space:
        def __init__(self, shape, dtype, seed=None):
            self.shape = tuple(shape)
            self.dtype = np.dtype(dtype)
            self._np_random = np.random.default_rng(seed)

        def seed(self, seed=None):
            self._np_random = np.random.default_rng(seed)

    class Box(_Space):
        def __init__(self, low, high, shape=None, dtype=np.float32, seed=None):
            if shape is None:
                shape = np.broadcast(np.asarray(low), np.asarray(high)).shape
            super().__init__(shape, dtype, seed)
            self.low = np.broadcast_to(np.asarray(low, dtype=self.dtype), self.shape).copy()
            self.high = np.broadcast_to(np.asarray(high, dtype=self.dtype), self.shape).copy()

        def sample(self):
            lo = np.where(np.isfinite(self.low), self.low, -1.0)
            hi = np.where(np.isfinite(self.high), self.high, 1.0)
            return self._np_random.uniform(lo, hi).astype(self.dtype)

        def contains(self, x):
            x = np.asarray(x)
            return x.shape == self.shape and bool(np.all(x >= self.low) and np.all(x <= self.high))

        def __repr__(self):
            return f"Box({self.low.min()}, {self.high.max()}, {self.shape}, {self.dtype})"

    class Discrete(_Space):
        def __init__(self, n, seed=None, start=0):
            super().__init__((), np.int64, seed)
            self.n = int(n)
            self.start = int(start)

        def sample(self):
            return int(self._np_random.integers(self.n)) + self.start

        def contains(self, x):
            return self.start <= int(x) < self.start + self.n

        def __repr__(self):
            return f"Discrete({self.n})"

    class Dict(_Space):
        """A mapping of named spaces; keys sorted as gymnasium's Dict sorts a plain dict."""

        def __init__(self, spaces, seed=None):
            super().__init__((), None, seed)
            self.shape, self.dtype = None, None
            self.spaces = dict(sorted(dict(spaces).items()))

        def __getitem__(self, key):
            return self.spaces[key]

        def keys(self):
            return self.spaces.keys()

        def sample(self):
            return {k: s.sample() for k, s in self.spaces.items()}

        def contains(self, x):
            return (isinstance(x, dict) and set(x) == set(self.spaces)
                    and all(s.contains(x[k]) for k, s in self.spaces.items()))

        def __repr__(self):
            return "Dict(" + ", ".join(f"{k!r}: {s}" for k, s in self.spaces.items()) + ")"


def batch_space(space, n: int):
    """gymnasium.vector.utils.batch_space for the space kinds used here."""
    if isinstance(space, Box):
        return Box(
            low=np.broadcast_to(space.low, (n,) + space.shape).copy(),
            high=np.broadcast_to(space.high, (n,) + space.shape).copy(),
            dtype=space.dtype,
        )
    if isinstance(space, Discrete):
        try:
            from gymnasium.spaces import MultiDiscrete  # type: ignore

            return MultiDiscrete(np.full((n,), space.n, dtype=np.int64))
        except Exception:
            return Box(low=0, high=space.n - 1, shape=(n,), dtype=np.int64)
    if isinstance(space, Dict):
        return Dict({k: batch_space(s, n) for k, s in space.spaces.items()})
    raise TypeError(space)
