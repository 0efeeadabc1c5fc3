"""The crafted-generator helpers (tests/rng_craft.py) against numpy's own Generator(PCG64), and the C oracle's Lemire
rejection against numpy's: the GPU tests that inject these states rely on both."""
import copy
import ctypes as C

import numpy as np
import pytest

import hwy_oracle as ho
import rng_craft as rc

INCS = [rc.seeded_state(s)[1] for s in (0, 7, 123456)] + [1, (1 << 128) - 1]


def _u32_stream(g, k):
    return [int(v) for v in g.integers(0, 1 << 32, size=k, dtype=np.uint32)]


@pytest.mark.parametrize("inc", INCS)
def test_crafted_state_emits_the_chosen_word(inc):
    r = np.random.default_rng(inc & 0xFFFF)
    for m in (0, 1, 5, 63, 200):
        for x in (0, 1, rc.M64, 0xFFFFFFFF, 0xFFFFFFFF << 32, int(r.integers(0, 1 << 63)) * 2 + 1):
            for hi in (0, 1 << 63, int(r.integers(0, 1 << 63))):
                g = rc.make_generator(rc.crafted_state(x, inc, m=m, hi=hi), inc)
                raw = g.bit_generator.random_raw(m + 1)
                assert int(raw[-1]) == x, (m, hex(x), hex(hi))


def test_step_back_inverts_a_step():
    state, inc = rc.seeded_state(99)
    g = rc.make_generator(state, inc)
    g.bit_generator.random_raw(37)
    after = g.bit_generator.state["state"]["state"]
    assert rc.step_back(after, inc, 37) == state
    assert rc.output_of(rc.step_back(after, inc, 0)) == int(rc.make_generator(
        rc.step_back(after, inc, 1), inc).bit_generator.random_raw())


@pytest.mark.parametrize("has", [0, 1])
def test_next32_is_low_then_buffered_high_half(has):
    """integers(0, 2**32, uint32) serves next_uint32 unchanged: the low half of a fresh output, then its buffered high
    half (what the GPU stream test uses as numpy's next32)."""
    state, inc = rc.seeded_state(5)
    u = 0xDEADBEEF
    g = rc.make_generator(state, inc, has, u)
    got = _u32_stream(g, 9)
    raw = [int(v) for v in rc.make_generator(state, inc).bit_generator.random_raw(5)]
    halves = [h for w in raw for h in (w & 0xFFFFFFFF, w >> 32)]
    assert got == ([u] if has else []) + halves[:9 - has]
    w = rc.words_of(g)
    assert int(w[4]) >> 32 == (1 if (9 - has) % 2 else 0)


def _consumed(state, inc, after_state, limit=64):
    g = rc.make_generator(state, inc)
    for k in range(limit + 1):
        if g.bit_generator.state["state"]["state"] == after_state:
            return k
        g.bit_generator.random_raw()
    raise AssertionError("more than %d outputs" % limit)


@pytest.mark.parametrize("n", [3, 5, 7, 20, (1 << 30) + 1])
def test_zero_words_force_a_lemire_rejection(n):
    state, inc = rc.seeded_state(11)
    assert rc.lemire_rejects(0, n)
    # buffered half 0: choice redraws from a fresh output
    for call in ("choice", "integers"):
        g = rc.make_generator(state, inc, 1, 0)
        v = g.choice(n) if call == "choice" else int(g.integers(0, n))
        after = g.bit_generator.state
        assert _consumed(state, inc, after["state"]["state"]) == 1 and after["has_uint32"] == 1
        lo = int(rc.make_generator(state, inc).bit_generator.random_raw()) & 0xFFFFFFFF
        assert v == (lo * n) >> 32
    # fresh output with low half 0: the redraw takes that output's high half (which is not 0 here)
    hi_half = 0x9E3779B9
    st = rc.crafted_state(hi_half << 32, inc, m=0)
    g = rc.make_generator(st, inc)
    v = g.choice(n)
    after = g.bit_generator.state
    assert _consumed(st, inc, after["state"]["state"]) == 1 and after["has_uint32"] == 0
    assert v == (hi_half * n) >> 32
    # without the zero the same call keeps the high half buffered
    g = rc.make_generator(rc.crafted_state((hi_half << 32) | 12345, inc, m=0), inc)
    g.choice(n)
    assert g.bit_generator.state["has_uint32"] == 1


def _orc(words):
    w = [int(v) for v in words]
    return ho.OrcPcg64(w[0], w[1], w[2], w[3], w[4] >> 32, w[4] & 0xFFFFFFFF)


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 20, (1 << 30) + 1])
def test_oracle_choice_rejects_where_numpy_does(n):
    lib = ho.lib()
    states = []
    for s in range(4):
        state, inc = rc.seeded_state(300 + s)
        states += [(state, inc, 1, 0), (state, inc, 0, 0), (state, inc, 1, 0xFFFFFFFF),
                   (rc.crafted_state(0x12345678 << 32, inc, m=0), inc, 0, 0),
                   (rc.crafted_state(0x00000000FFFF0000, inc, m=0), inc, 1, 7),
                   (rc.crafted_state(0xABCDEF01, inc, m=0), inc, 0, 0)]  # high half 0: the 2nd request rejects
    for st in states:
        g = rc.make_generator(*st)
        o = _orc(rc.words_of(*st))
        for _ in range(6):
            assert lib.orc_rng_choice(C.byref(o), n) == g.choice(n)
        ws = rc.words_of(g)
        assert [o.state_hi, o.state_lo, o.inc_hi, o.inc_lo] == [int(v) for v in ws[:4]]
        assert (o.has_uint32, o.uinteger) == (int(ws[4]) >> 32, int(ws[4]) & 0xFFFFFFFF)


@pytest.mark.parametrize("negative", [False, True])
def test_ziggurat_tail_word(negative):
    hits = 0
    for s in range(8):
        state, inc = rc.seeded_state(500 + s)
        st = rc.crafted_state(rc.ziggurat_tail_word(negative), inc, m=0)
        g = rc.make_generator(st, inc)
        x = g.standard_normal()
        assert abs(x) >= rc.ZIGGURAT_NOR_R and (x < 0) == negative
        hits += _consumed(st, inc, g.bit_generator.state["state"]["state"]) >= 3  # word + 2 doubles per try
    assert hits == 8


@pytest.mark.parametrize("layer", [1, 2, 100, 254, 255])
def test_ziggurat_wedge_word(layer):
    for s in range(8):
        state, inc = rc.seeded_state(600 + s)
        st = rc.crafted_state(rc.ziggurat_word(layer), inc, m=0)
        g = rc.make_generator(st, inc)
        x = g.standard_normal()
        assert _consumed(st, inc, g.bit_generator.state["state"]["state"]) >= 2
        assert abs(x) < rc.ZIGGURAT_NOR_R or layer == 0
        if layer == 1:
            continue  # ki[1] = 0: every draw of layer 1 goes through the wedge
        # the fast path of the same layer (magnitude 0) consumes one output
        g2 = rc.make_generator(rc.crafted_state(rc.ziggurat_word(layer, magnitude=0), inc, m=0), inc)
        assert g2.standard_normal() == 0.0
        assert _consumed(rc.crafted_state(rc.ziggurat_word(layer, magnitude=0), inc, m=0), inc,
                         g2.bit_generator.state["state"]["state"]) == 1


@pytest.mark.parametrize("V,L,has,ego", [(21, 3, 0, True), (21, 3, 1, True), (51, 4, 1, True), (21, 3, 0, False),
                                         (8, 2, 1, False)])
def test_spawn_requests_locate_every_lane_choice(V, L, has, ego):
    """spawn_requests names the output (and half) behind every lane choice of the highway spawn: a zero crafted there
    is the very word that choice(L) reads, replayed on numpy in the draw order of Vehicle.create_random."""
    state, inc = rc.seeded_state(77)
    reqs = rc.spawn_requests(V, L, has, ego)
    assert len(reqs) == (V - 1) + int(ego)
    for v, out, half in reqs:
        if half == "buffered":
            st, u = state, 0
        else:
            word = 0x5A5A5A5A << 32 if half == "low" else 0x5A5A5A5A  # this half 0, the other not
            st, u = rc.crafted_state(word, inc, m=out), 0x77777777
        g = rc.make_generator(st, inc, has, u)
        for w in range(V):
            if L > 1 and (w > 0 or ego):
                if w == v:
                    assert _u32_stream(copy.deepcopy(g), 1) == [0], (v, out, half)
                    break
                g.choice(L)
            g.uniform(0, 1, size=1 if w == 0 else 3)
        else:
            raise AssertionError("vehicle %d never drew" % v)


def test_numpy_dot_of_2_vectors_is_one_fma():
    """The kernels model numpy's np.dot / np.linalg.norm of 2-vectors as fma(a1, b1, round(a0 * b0)) (hwy_math.cuh
    dot2).  If this numpy build computes it another way, the GPU parity tests would drift for no visible reason."""
    from fractions import Fraction

    r = np.random.default_rng(2024)
    a = r.standard_normal((3000, 2)) * np.exp2(r.integers(-20, 20, size=(3000, 2)))
    b = r.standard_normal((3000, 2)) * np.exp2(r.integers(-20, 20, size=(3000, 2)))
    b[:500, 1] = -a[:500, 0] * b[:500, 0] / a[:500, 1] * (1 + r.uniform(-1e-12, 1e-12, 500))  # cancellation
    for (a0, a1), (b0, b1) in zip(a.tolist(), b.tolist()):
        want = float(Fraction(a1) * Fraction(b1) + Fraction(a0 * b0))
        assert float(np.dot(np.array([a0, a1]), np.array([b0, b1]))) == want
        n_want = float(np.sqrt(float(Fraction(a1) * Fraction(a1) + Fraction(a0 * a0))))
        assert float(np.linalg.norm(np.array([a0, a1]))) == n_want
