"""The scalar device functions of the step kernels (csrc/hwy_math.cuh, csrc/hwy_device.cuh), called through
`hwy_debug_math`, against exact references built here: mpmath at 60 digits for the transcendental ones,
`fractions.Fraction` (correctly rounded) for the fused dot product, and CPython / numpy float arithmetic for the
operations that are meant to be bit-identical.  The trajectory tests cannot see errors of an ulp; these can.

Run with `-s` to see the measured maxima."""
import math
import sys
from fractions import Fraction

import mpmath as mp
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DBL_MIN = sys.float_info.min
SUB = 5e-324  # spacing of the subnormals


def run(op, rows):
    from highwayenv_b200 import _native as N

    code, k_in, k_out = N.MATH_OPS[op]
    a = np.ascontiguousarray(np.asarray(rows, dtype=np.float64).reshape(-1, k_in))
    d_in = torch.from_numpy(a).cuda()
    d_out = torch.full((len(a), k_out), np.nan, dtype=torch.float64, device="cuda")
    N.check(N.load().hwy_debug_math(code, d_in.data_ptr(), d_out.data_ptr(), len(a), None))
    torch.cuda.synchronize()
    out = d_out.cpu().numpy()
    return out[:, 0] if k_out == 1 else out


def ulp_of(ref):
    """spacing of the doubles in the binade of the exact value `ref` (an mpf), never below the subnormal spacing"""
    if ref == 0:
        return mp.mpf(SUB)
    _, e = mp.frexp(ref)
    return max(mp.ldexp(1, int(e) - 53), mp.mpf(SUB))


def ulp_err(got, ref):
    return float(abs(mp.mpf(float(got)) - ref) / ulp_of(ref))


def report(name, v):
    print(f"\n[device math] {name}: {v:.3g}", end="")


def bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


def neighbours(xs):
    return [y for x in xs for y in (np.nextafter(x, -np.inf), x, np.nextafter(x, np.inf))]


# ------------------------------------------------------------------ m_sincos
def test_sincos_fast_path_within_one_ulp():
    r = np.random.default_rng(1)
    pi4 = 0.7853981633974483
    hw = lambda w: float(np.array([w << 32], dtype=np.uint64).view(np.float64)[0])  # noqa: E731
    # fdlibm's branch points; 2^-27 is where the (x, 1) shortcut ends
    edges = neighbours([0.3, 0.78125, pi4, hw(0x3FD33333), hw(0x3FE90000), 1e-8, 0.1, 0.5, 2.0 ** -26, 2.0 ** -27])
    edges = [x for x in edges if abs(x) <= pi4]
    xs = np.concatenate([r.uniform(-pi4, pi4, 20000), edges, -np.array(edges), [SUB, -SUB, DBL_MIN, 1e-310, -1e-320]])
    out = run("sincos", xs)
    worst_s = worst_c = 0.0
    with mp.workdps(60):
        for x, (s, c) in zip(xs.tolist(), out.tolist()):
            worst_s = max(worst_s, ulp_err(s, mp.sin(mp.mpf(x))))
            worst_c = max(worst_c, ulp_err(c, mp.cos(mp.mpf(x))))
    report("m_sincos |x| <= pi/4: max sin error (ulp)", worst_s)
    report("m_sincos |x| <= pi/4: max cos error (ulp)", worst_c)
    assert worst_s <= 1.0 and worst_c <= 1.0
    z = run("sincos", [0.0, -0.0])
    assert bits(z[:, 0]).tolist() == bits([0.0, -0.0]).tolist() and z[:, 1].tolist() == [1.0, 1.0]
    # either side of the shortcut the polynomial and the shortcut agree: sin = x, cos = 1 exactly
    t = [np.nextafter(2.0 ** -27, 0), 2.0 ** -27, np.nextafter(2.0 ** -27, 1)]
    z = run("sincos", t + [-x for x in t])
    assert bits(z[:, 0]).tolist() == bits(t + [-x for x in t]).tolist() and (z[:, 1] == 1.0).all()


def test_sincos_library_path_within_two_ulp():
    r = np.random.default_rng(2)
    pi4 = 0.7853981633974483
    xs = np.concatenate([r.uniform(pi4, 50.0, 2000) * r.choice([-1, 1], 2000), neighbours([np.nextafter(pi4, 1.0)]),
                         [1.0, -1.0, math.pi, -math.pi, 1e5, 1e22, -3e300]])
    xs = xs[np.abs(xs) > pi4]
    out = run("sincos", xs)
    worst = 0.0
    with mp.workdps(60):
        for x, (s, c) in zip(xs.tolist(), out.tolist()):
            worst = max(worst, ulp_err(s, mp.sin(mp.mpf(x))), ulp_err(c, mp.cos(mp.mpf(x))))
    report("m_sincos |x| > pi/4 (library sincos): max error (ulp)", worst)
    assert worst <= 2.0


# ------------------------------------------------------------------ idm_pow
def _pow_errors(xs, ds):
    out = run("idm_pow", np.stack([xs, ds], axis=1))
    errs = []
    with mp.workdps(60):
        for x, d, g in zip(xs.tolist(), ds.tolist(), out.tolist()):
            ref = mp.power(mp.mpf(x), mp.mpf(d)) if x > 0 else mp.mpf(0)
            errs.append((x, d, g, ref))
    return errs


def test_idm_pow_delta_4():
    r = np.random.default_rng(3)
    xs = np.concatenate([r.uniform(0, 3, 20000), [0.0, 1.0, 2.0, 3.0, 0.5, 1e-30, 1e-76, 1e-77],
                         np.geomspace(1e-73, 1e-70, 300),     # x^4 around 2^-968
                         np.geomspace(2.0 ** -255.5, 2.0 ** -242, 3000),  # x^4 across [DBL_MIN, 2^-968)
                         np.geomspace(1.2e-77, 2e-77, 300),   # x^4 around DBL_MIN
                         np.geomspace(1e-80, 1.1e-77, 300),   # x^4 subnormal
                         neighbours([1e60]), [1e61, 1e70, 1e76, 1e77, 1e100, 1e300, np.inf]])
    worst_n = worst_low = worst_s = worst_lib = 0.0
    for x, d, g, ref in _pow_errors(xs, np.full(len(xs), 4.0)):
        if ref > sys.float_info.max:
            assert g == np.inf, x
        elif x >= 1e60:  # the library pow
            worst_lib = max(worst_lib, ulp_err(g, ref))
        elif ref < DBL_MIN:
            worst_s = max(worst_s, float(abs(mp.mpf(g) - ref) / SUB))
        elif ref < 2.0 ** -968:
            # the residuals f (of p*p) and 2pe fall below the subnormal spacing: each rounds by up to 0.5 and 1
            # spacing, on top of the final 0.5 ulp (<= 2 ulp in the lowest binade, less above)
            assert abs(mp.mpf(g) - ref) <= ulp_of(ref) / 2 + mp.mpf(1.5) * SUB, x
            worst_low = max(worst_low, ulp_err(g, ref))
        else:
            worst_n = max(worst_n, ulp_err(g, ref))
    report("idm_pow delta=4, results >= 2^-968: max error (ulp)", worst_n)
    report("idm_pow delta=4, results in [DBL_MIN, 2^-968): max error (ulp)", worst_low)
    report("idm_pow delta=4, results below DBL_MIN: max error (subnormal spacings)", worst_s)
    report("idm_pow delta=4, x >= 1e60 (library pow): max error (ulp)", worst_lib)
    assert worst_n <= 0.51 and worst_s <= 1.0 and worst_lib <= 2.0
    assert run("idm_pow", [[0.0, 4.0]]).tolist() == [0.0] and run("idm_pow", [[np.inf, 4.0]]).tolist() == [np.inf]


def test_idm_pow_randomized_delta():
    r = np.random.default_rng(4)
    n = 20000
    xs, ds = r.uniform(0.5, 2.0, n), r.uniform(3.5, 4.5, n)
    edge_x = np.concatenate([[0.5, 2.0, 1.0, np.nextafter(1.0, 0), np.nextafter(1.0, 2)], r.uniform(0.5, 2, 45)])
    xs = np.concatenate([xs, np.repeat(edge_x, 2)])
    ds = np.concatenate([ds, np.tile([3.5, 4.5], len(edge_x))])
    worst = max(ulp_err(g, ref) for _, _, g, ref in _pow_errors(xs, ds))
    report("idm_pow delta in [3.5, 4.5], x in [0.5, 2]: max error (ulp)", worst)
    assert worst <= 2.5
    # small ratios: the rounding of (delta - 4) log x (|.| <= 69) dominates; relative error below 1e-14
    xs = np.exp(r.uniform(np.log(1e-60), np.log(0.5), 5000))
    xs = np.concatenate([xs, [np.nextafter(1e-60, 1.0)]])
    ds = r.uniform(3.5, 4.5, len(xs))
    rel = max(float(abs(mp.mpf(g) - ref) / ref) for _, _, g, ref in _pow_errors(xs, ds))
    report("idm_pow delta in [3.5, 4.5], x in (1e-60, 0.5): max relative error", rel)
    assert rel < 1e-14


def test_idm_pow_library_side_of_the_branches():
    """|delta - 4| > 0.5 and x <= 1e-60 take the library pow (<= 2 ulp); x = 0 gives 0."""
    r = np.random.default_rng(5)
    xs = r.uniform(0.5, 2.0, 200)
    lo, hi = np.nextafter(3.5, 0), np.nextafter(4.5, 9)
    xs = np.concatenate([xs, xs, [1e-60, np.nextafter(1e-60, 0)] * 3])
    ds = np.concatenate([np.full(200, lo), np.full(200, hi), [3.5, 3.5, 4.2, 4.2, 4.5, 4.5]])
    worst = max(ulp_err(g, ref) for _, _, g, ref in _pow_errors(xs, ds))
    report("idm_pow library branches: max error (ulp)", worst)
    assert worst <= 2.0
    assert run("idm_pow", [[0.0, 3.5], [0.0, 4.2], [0.0, 4.5]]).tolist() == [0.0, 0.0, 0.0]


def test_exp_dlog():
    r = np.random.default_rng(6)
    d, x = r.uniform(-0.5, 0.5, 20000), r.uniform(0.5, 2.0, 20000)
    out = run("exp_dlog", np.stack([d, x], axis=1))
    with mp.workdps(60):
        worst = max(ulp_err(g, mp.power(mp.mpf(xx), mp.mpf(dd))) for dd, xx, g in zip(d.tolist(), x.tolist(), out.tolist()))
    report("m_exp_dlog |d| <= 0.5, x in [0.5, 2]: max error (ulp)", worst)
    assert worst <= 2.0


# ------------------------------------------------------------------ floored modulo
def _same(got, want):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    nan = np.isnan(want)
    return bool(np.array_equal(np.isnan(got), nan) and np.array_equal(bits(got[~nan]), bits(want[~nan])))


@pytest.mark.parametrize("b", [2 * np.pi, 1.0, 0.7, 0.5, 3.0])
def test_py_mod_pos_is_bit_identical_to_python(b):
    r = np.random.default_rng(7)
    base = [0.0, -0.0, b, 2 * b, -b, 3 * b, -2 * b, 0.5 * b, -0.5 * b]
    a = (neighbours(base) + [-SUB, -1e-300, -1e-17, SUB, 1e300, -1e300, 1e20, -1e20, 2.0 ** 52, 2.0 ** 52 - 1,
                             2.0 ** 52 + 2, 2.0 ** 53, -(2.0 ** 52), np.nan, np.inf, -np.inf]
         + list(r.uniform(-10 * b, 10 * b, 3000)) + list(r.uniform(-1e6, 1e6, 500)))
    a = np.array(a)
    got = run("py_mod_pos", np.stack([a, np.full(len(a), b)], axis=1))
    want_py = [x % b for x in a.tolist()]
    with np.errstate(invalid="ignore"):
        want_np = np.float64(1.0) * (a % np.float64(b))
    assert _same(got, want_py), [(x, g, w) for x, g, w in zip(a, got, want_py) if not _same([g], [w])][:5]
    assert _same(got, want_np)
    assert bits(run("py_mod_pos", [[-0.0, b]]))[0] == bits(0.0)  # +0.0, as CPython and numpy


def test_wrap_to_pi_is_bit_identical_to_python():
    r = np.random.default_rng(8)
    pi = np.pi
    base = [0.0, -0.0, pi, -pi, 2 * pi, -2 * pi, 3 * pi, -3 * pi, pi / 2, -pi / 2, 1e-17, -1e-17]
    xs = np.array(neighbours(base) + [1e300, -1e300, 1e16, np.nan, np.inf, -np.inf]
                  + list(r.uniform(-20, 20, 4000)))
    got = run("wrap_to_pi", xs)
    want = [((x + pi) % (2 * pi)) - pi for x in xs.tolist()]  # utils.py:59-60
    assert _same(got, want)


# ------------------------------------------------------------------ not_zero, div_finite
def _not_zero(x, eps=1e-2):  # utils.py:50-56
    if abs(x) > eps:
        return x
    elif x >= 0:
        return eps
    else:
        return -eps


def test_not_zero_and_div_finite_are_bit_identical():
    xs = np.array(neighbours([0.0, -0.0, 0.01, -0.01, 1.0, -1.0]) + [np.nan, np.inf, -np.inf, 1e-300, -1e-300])
    assert _same(run("not_zero", xs), [_not_zero(x) for x in xs.tolist()])
    r = np.random.default_rng(9)
    nums = [0.0, -0.0, 1.0, -1.0, SUB, -3.5, 1e300] + list(r.standard_normal(50))
    dens = [1.0, -1.0, 0.01, -0.01, 3.7, -1e300, 1e-300, -SUB, SUB, 1e308, -2.5] + list(r.standard_normal(30))
    pairs = np.array([(n, d) for n in nums for d in dens])
    assert _same(run("div_finite", pairs), [n / d for n, d in pairs.tolist()])


# ------------------------------------------------------------------ dot2 / norm2
def test_dot2_and_norm2_are_the_correctly_rounded_single_fma():
    r = np.random.default_rng(10)
    n = 6000
    a = r.standard_normal((n, 2)) * np.exp2(r.integers(-30, 30, size=(n, 2)))
    b = r.standard_normal((n, 2)) * np.exp2(r.integers(-30, 30, size=(n, 2)))
    k = n // 3  # cancellation: a0 b0 ~ -a1 b1
    b[:k, 1] = -a[:k, 0] * b[:k, 0] / a[:k, 1] * (1 + r.uniform(-1e-10, 1e-10, k))
    b[k:k + 50, 1] = -a[k:k + 50, 0] * b[k:k + 50, 0] / a[k:k + 50, 1]
    got = run("dot2", np.concatenate([a, b], axis=1))
    want = [float(Fraction(a1) * Fraction(b1) + Fraction(a0 * b0)) for (a0, a1), (b0, b1) in zip(a.tolist(), b.tolist())]
    assert _same(got, want)
    got_n = run("norm2", a)
    want_n = [math.sqrt(float(Fraction(a1) ** 2 + Fraction(a0 * a0))) for a0, a1 in a.tolist()]
    assert _same(got_n, want_n)


# ------------------------------------------------------------------ slip angle
MAX_STEER = float(np.pi / 3)


def _beta_ref_controlled(x):
    """the reference's chain: arcsin, arctan(2 tan), clip to +-np.pi/3, arctan(tan / 2) (controller.py:176-186,
    kinematics.py:141-142), evaluated exactly"""
    s = mp.asin(mp.mpf(x))
    d = mp.atan(2 * mp.tan(s))
    d = min(max(d, -mp.mpf(MAX_STEER)), mp.mpf(MAX_STEER))
    beta = mp.atan(mp.tan(d) / 2)
    return mp.sin(beta), mp.cos(beta)


def _beta_errors(op, xs, ref):
    out = run(op, xs)
    worst, worst_abs0 = 0.0, 0.0
    with mp.workdps(60):
        for x, (s, c) in zip(xs.tolist(), out.tolist()):
            rs, rc_ = ref(x)
            worst = max(worst, ulp_err(s, rs), ulp_err(c, rc_))
            if abs(x) < 1e-3:
                worst_abs0 = max(worst_abs0, float(abs(mp.mpf(s) - rs)))
    return worst, worst_abs0


def test_beta_of_controlled():
    r = np.random.default_rng(11)
    xstar = math.sqrt(3 / 7)  # 2|x| = tan(pi/3) sqrt(1 - x^2): where the steering saturates
    near = [xstar]
    for _ in range(6):
        near += [np.nextafter(near[-1], 1.0)]
    lo = [xstar]
    for _ in range(6):
        lo += [np.nextafter(lo[-1], 0.0)]
    edges = near + lo + [1.0, np.nextafter(1.0, 0), 0.0, -0.0, 1e-300, 1e-8, 1e-4]
    xs = np.concatenate([r.uniform(-1, 1, 20000), edges, -np.array(edges), r.uniform(-1e-3, 1e-3, 500)])
    worst, near0 = _beta_errors("beta_of_controlled", xs, _beta_ref_controlled)
    report("beta_of_controlled: max error vs the reference chain (ulp)", worst)
    report("beta_of_controlled |x| < 1e-3: max abs error of sin(beta)", near0)
    assert worst <= 4.0 and near0 <= 1e-16


def test_beta_of_angle():
    r = np.random.default_rng(12)
    edges = neighbours([np.pi / 4, np.pi / 2, np.pi / 3, 1e-8]) + [0.0, -0.0]
    xs = np.concatenate([r.uniform(-np.pi / 2, np.pi / 2, 20000), edges, -np.array(edges), r.uniform(-1e-3, 1e-3, 500)])

    def ref(d):
        beta = mp.atan(mp.tan(mp.mpf(d)) / 2)  # kinematics.py:141-142
        return mp.sin(beta), mp.cos(beta)

    worst, near0 = _beta_errors("beta_of_angle", xs, ref)
    report("beta_of_angle: max error (ulp)", worst)
    report("beta_of_angle |delta| < 1e-3: max abs error of sin(beta)", near0)
    assert worst <= 4.0 and near0 <= 1e-16


# ------------------------------------------------------------------ speed_to_index
@pytest.mark.parametrize("ts", [[20.0, 25.0, 30.0], [18.0, 21.5, 30.0, 31.0], [0.0, 10.0], list(np.linspace(5, 40, 8))])
def test_speed_to_index_matches_numpy_round_and_clip(ts):
    ts = np.array(ts)
    n = len(ts)
    half = [ts[0] + (k + 0.5) / (n - 1) * (ts[-1] - ts[0]) for k in range(n - 1)]
    speeds = np.array(neighbours(half + list(ts)) + [-1e9, 1e9, ts[0] - 100, ts[-1] + 100, -0.0]
                      + list(np.random.default_rng(13).uniform(ts[0] - 10, ts[-1] + 10, 2000)))
    table = np.zeros(8)
    table[:n] = ts
    rows = np.concatenate([speeds[:, None], np.full((len(speeds), 1), n), np.tile(table, (len(speeds), 1))], axis=1)
    got = run("speed_to_index", rows)
    x = (speeds - ts[0]) / (ts[-1] - ts[0])  # controller.py:326-344
    want = np.clip(np.round(x * (n - 1)), 0, n - 1).astype(np.int64)
    assert np.array_equal(got.astype(np.int64), want)


def test_speed_to_index_refuses_a_table_size_outside_1_to_8():
    rows = np.zeros((4, 10))
    rows[:, 1] = [0, 9, -1, np.nan]
    assert np.isnan(run("speed_to_index", rows)).all()
