"""The kernels' restatement of numpy's Generator(PCG64) (csrc/hwy_math.cuh Pcg64, the jump table of the fused
autoreset in csrc/hwy_highway.cu), called through `hwy_debug_pcg64`, against numpy itself: every draw and the 5
generator words afterwards bit for bit, from seeded states and from crafted states (tests/rng_craft.py) that reach the
rare branches — Lemire rejections and the ziggurat's wedge and tail."""
import numpy as np
import pytest
import torch

import rng_craft as rc

pytestmark = pytest.mark.gpu

JUMP_N = 4 * 128 + 8  # kPcgJumpN = 4 * HWY_MAX_VEHICLES + 8


def run(op, words, count=0, arg_i=0, lo=0.0, hi=0.0):
    """words [n][5] (uint64) -> (draws [n][count] or [n][count][2] uint64, words after [n][5])"""
    from highwayenv_b200 import _native as N

    w = np.ascontiguousarray(np.asarray(words, dtype=np.uint64).T)  # [5][n], the HwyHighwayState.rng layout
    n = w.shape[1]
    d_in = torch.from_numpy(w.view(np.int64)).cuda()
    d_out = torch.zeros_like(d_in)
    per = 2 if op == "normal" else 1
    d_draws = torch.zeros((n, max(count, 1) * per), dtype=torch.int64, device="cuda")
    N.check(N.load().hwy_debug_pcg64(N.PCG_OPS[op], int(arg_i), float(lo), float(hi), int(count), d_in.data_ptr(),
                                     d_out.data_ptr(), d_draws.data_ptr(), n, None))
    torch.cuda.synchronize()
    draws = d_draws.cpu().numpy().view(np.uint64)[:, :count * per]
    if op == "normal":
        draws = draws.reshape(n, count, 2)
    return draws, d_out.cpu().numpy().view(np.uint64).T.copy()


def seeded(seeds, has=0, u=0):
    return [rc.words_of(*rc.seeded_state(s), has, u) for s in seeds]


def crafted_zero_halves(seeds):
    """states whose buffered half, fresh low half or the following high half is 0"""
    out = []
    for s in seeds:
        st, inc = rc.seeded_state(s)
        out += [rc.words_of(st, inc, 1, 0),
                rc.words_of(rc.crafted_state(0x5A5A5A5A << 32, inc, m=0, seed=s), inc, 0, 0),   # low half 0
                rc.words_of(rc.crafted_state(0x5A5A5A5A, inc, m=0, seed=s), inc, 0, 0),         # high half 0
                rc.words_of(rc.crafted_state(0, inc, m=1, seed=s), inc, 1, 0xFFFFFFFF)]          # both, 2nd output
    return out


def assert_words(got, gens, what):
    want = np.stack([rc.words_of(g) for g in gens])
    assert np.array_equal(got, want), f"{what}: generator words differ in {np.nonzero((got != want).any(1))[0][:8]}"


@pytest.mark.parametrize("has", [0, 1])
def test_next64_next32_next_double(has):
    states = seeded(range(64), has, 0x13579BDF) + crafted_zero_halves(range(8))
    for op, count in (("next64", 257), ("next32", 257), ("next_double", 100)):
        draws, words = run(op, states, count)
        gens = [rc.generator_of(w) for w in states]
        for k, g in enumerate(gens):
            if op == "next64":
                want = g.bit_generator.random_raw(count)
            elif op == "next32":
                want = g.integers(0, 1 << 32, size=count, dtype=np.uint32).astype(np.uint64)
            else:
                want = g.random(count).view(np.uint64)
            assert np.array_equal(draws[k], want), (op, k)
        assert_words(words, gens, op)


def test_uniform():
    states = seeded(range(100, 164)) + seeded(range(3), 1, 77)
    for lo, hi in ((0.0, 1.0), (0.9, 1.1), (3.5, 4.5), (21.0, 24.0), (-5.0, 5.0), (1e-300, 1e300)):
        draws, words = run("uniform", states, 50, lo=lo, hi=hi)
        gens = [rc.generator_of(w) for w in states]
        for k, g in enumerate(gens):
            assert np.array_equal(draws[k], g.uniform(lo, hi, 50).view(np.uint64)), (lo, hi, k)
        assert_words(words, gens, "uniform")


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 20, (1 << 30) + 1])
def test_choice(n):
    """Generator.choice(n) = integers(0, n): Lemire's method on buffered 32-bit halves.  2^30 + 1 rejects with
    p ~ 1/4, so seeded states run the rejection loop; the small n get crafted zero words in the buffered and in the
    fresh position (rejected for every n that is not a power of two)."""
    states = seeded(range(200, 328)) + seeded(range(4), 1, 0) + crafted_zero_halves(range(300, 316))
    count = 40
    draws, words = run("choice", states, count, arg_i=n)
    gens = [rc.generator_of(w) for w in states]
    rejected = 0
    for k, g in enumerate(gens):
        probe = rc.generator_of(states[k])
        r32 = [int(v) for v in probe.integers(0, 1 << 32, size=2 * count, dtype=np.uint32)]
        rejected += any(rc.lemire_rejects(v, n) for v in r32[:count]) if n > 1 else 0
        want = [g.choice(n) for _ in range(count)]
        assert draws[k].astype(np.int64).tolist() == want, (n, k)
    assert_words(words, gens, f"choice({n})")
    if n & (n - 1):
        assert rejected > 0, "no rejection was exercised"


def test_normal_ten_million_draws_with_wedge_and_tail():
    """random_standard_normal: the 256-layer ziggurat.  The fast path is exact arithmetic; the wedge (exp) and tail
    (log1p) decide with CUDA's libm, so a flipped accept/reject would desynchronise the stream words."""
    n, count = 4096, 2500
    states = seeded(range(10_000, 10_000 + n))
    draws, words = run("normal", states, count)
    vals, used = draws[..., 0].view(np.float64), draws[..., 1].astype(np.int64)
    gens = [rc.generator_of(w) for w in states]
    want = np.stack([g.standard_normal(count) for g in gens])
    assert_words(words, gens, "normal")  # every accept/reject decision matched numpy's
    assert used.min() >= 1, "a draw consumed more than 16 outputs"
    tail = np.abs(want) >= rc.ZIGGURAT_NOR_R
    wedge = (used > 1) & ~tail
    fast = used == 1
    n_tail, n_wedge = int(tail.sum()), int(wedge.sum())
    print(f"\n[normal] {n * count} draws: fast {int(fast.sum())}, wedge {n_wedge}, tail {n_tail}", end="")
    assert n_tail > 0 and n_wedge > 0
    assert np.array_equal(vals[~tail].view(np.uint64), want[~tail].view(np.uint64))
    _assert_tail_values(vals[tail], want[tail])


def _assert_tail_values(got, want):
    """The tail value R + (-log1p(-u) / R) goes through CUDA's log1p: equal to numpy's, or at most 1 ulp apart —
    reported explicitly, because the stream itself stays exact either way."""
    diff = np.abs(got.view(np.int64) - want.view(np.int64))
    if diff.any():
        print(f"\n[normal] {int((diff > 0).sum())} of {len(got)} tail values differ from numpy's "
              f"by up to {int(diff.max())} ulp (CUDA log1p)", end="")
    assert diff.max(initial=0) <= 1


@pytest.mark.parametrize("kind", ["tail+", "tail-", "wedge"])
def test_normal_crafted_tail_and_wedge(kind):
    states = []
    for s in range(64):
        st, inc = rc.seeded_state(20_000 + s)
        word = {"tail+": rc.ziggurat_tail_word(False), "tail-": rc.ziggurat_tail_word(True),
                "wedge": rc.ziggurat_word(1 + s * 4 % 255)}[kind]
        states.append(rc.words_of(rc.crafted_state(word, inc, m=0, seed=s), inc, s & 1, 5))
    draws, words = run("normal", states, 3)
    gens = [rc.generator_of(w) for w in states]
    want = np.stack([g.standard_normal(3) for g in gens])
    assert_words(words, gens, kind)
    vals, used = draws[..., 0].view(np.float64), draws[..., 1].astype(np.int64)
    assert (used[:, 0] >= (3 if kind.startswith("tail") else 2)).all()
    tail = np.abs(want) >= rc.ZIGGURAT_NOR_R
    if kind.startswith("tail"):
        assert tail[:, 0].all() and ((want[:, 0] < 0) == (kind == "tail-")).all()
    else:
        assert not tail[:, 0].any()
    assert np.array_equal(vals[~tail].view(np.uint64), want[~tail].view(np.uint64))
    _assert_tail_values(vals[tail], want[tail])


def test_pcg_at_every_jump_index():
    """pcg_at(n) positions a generator at output n of its stream (state A^n s + G_n inc): equal to numpy's
    bit_generator.advance(n) for every n of the table, seeded and crafted increments."""
    base = seeded(range(30_000, 30_008), 1, 99)
    for inc in (1, (1 << 128) - 1, (0x0123456789ABCDEF << 64) | 0xFEDCBA9876543211):
        base.append(rc.words_of(rc.crafted_state(rc.M64, inc, m=3), inc, 1, 12345))
    for n in range(JUMP_N):
        _, words = run("pcg_at", base, arg_i=n)
        gens = [rc.generator_of(w) for w in base]
        for g in gens:
            g.bit_generator.advance(n)
        assert_words(words, gens, f"pcg_at({n})")
