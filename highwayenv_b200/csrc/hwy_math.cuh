// hwy_math.cuh — scalar helpers shared by the sm_90a kernels.
//
// The simulation arithmetic is fp64 and follows the reference's operation order; the
// translation unit is compiled with -fmad=false so the compiler never contracts a*b+c.
// The only fused operations are the explicit fma() below, which reproduce what numpy
// itself does for 2-vector np.dot / np.linalg.norm (see DESIGN.md "numerics").
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "hwy_ziggurat_tables.h"

namespace hwy {

constexpr double kPi = 3.141592653589793;        // np.pi
constexpr double kTwoPi = 2 * 3.141592653589793;  // 2 * np.pi
constexpr double kVehLength = 5.0;                // vehicle/kinematics.py:21
constexpr double kVehWidth = 2.0;                 // vehicle/kinematics.py:23
constexpr double kMaxSpeed = 40.0;                // vehicle/kinematics.py:27
constexpr double kMinSpeed = -40.0;               // vehicle/kinematics.py:29
constexpr double kLaneVehLength = 5.0;            // road/lane.py:17
// ControlledVehicle gains, vehicle/controller.py:24-33
constexpr double kTauAcc = 0.6, kTauHeading = 0.2, kTauLateral = 0.6;
constexpr double kTauPursuit = 0.5 * kTauHeading;
constexpr double kKpA = 1 / kTauAcc;
constexpr double kKpHeading = 1 / kTauHeading;
constexpr double kKpLateral = 1 / kTauLateral;
constexpr double kMaxSteer = kPi / 3;

// np.dot on 2-vectors: fma(a1*b1 + round(a0*b0))
__device__ __forceinline__ double dot2(double a0, double a1, double b0, double b1) {
    return fma(a1, b1, a0 * b0);
}
__device__ __forceinline__ double norm2(double a0, double a1) { return sqrt(dot2(a0, a1, a0, a1)); }
__device__ __forceinline__ double clipd(double x, double lo, double hi) {
    return fmin(fmax(x, lo), hi);
}
// utils.py:50-56
__device__ __forceinline__ double not_zero(double x) {
    const double eps = 1e-2;
    if (fabs(x) > eps) return x;
    return x >= 0 ? eps : -eps;
}
// Out-of-line copies of the fp64 libm routines: every call site shares one body, which keeps
// the step kernel inside the instruction cache (the inlined versions made it > 140 KB and
// ~half of all issue slots stalled on instruction fetch).
static __device__ __noinline__ double m_asin(double x) { return asin(x); }
static __device__ __noinline__ double m_tan(double x) { return tan(x); }
static __device__ __noinline__ double m_atan(double x) { return atan(x); }
static __device__ __noinline__ double m_sin(double x) { return sin(x); }
// sin and cos together.  Headings and lane phases are almost always within +-pi/4 (a vehicle following its lane),
// where no argument reduction is needed: the fdlibm kernel polynomials (__kernel_sin / __kernel_cos, < 1 ulp, the
// same accuracy class as numpy's and CUDA's own routines) cost ~30 fp64 operations instead of the ~300 issued
// instructions of the general sincos(), which had become the largest single item of the step kernel's
// instructions.  Larger arguments take the library routine.  Returned by
// value: pointer results through a non-inlined call would live in local memory.
static __device__ __noinline__ double2 m_sincos_impl(double x) {
    const double ax = fabs(x);
    if (ax <= 0.7853981633974483) {
        // fdlibm's |x| < 2^-27 shortcut: the polynomials round to (x, 1) there too, but would turn sin(-0.0) into +0.0
        if (ax < 7.450580596923828e-09) return make_double2(x, 1.0);
        const double z = x * x;
        double r = fma(z, 1.58969099521155010221e-10, -2.50507602534068634195e-08);
        r = fma(z, r, 2.75573137070700676789e-06);
        r = fma(z, r, -1.98412698298579493134e-04);
        r = fma(z, r, 8.33333333332248946124e-03);
        const double v = z * x;
        const double sn = fma(v, fma(z, r, -1.66666666666666324348e-01), x);
        double q = fma(z, -1.13596475577881948265e-11, 2.08757232129817482790e-09);
        q = fma(z, q, -2.75573143513906633035e-07);
        q = fma(z, q, 2.48015872894767294178e-05);
        q = fma(z, q, -1.38888888888741095749e-03);
        q = fma(z, q, 4.16666666666666019037e-02);
        const double zr = z * (z * q);
        double cs;
        if (ax < 0.3) {
            cs = 1.0 - (0.5 * z - zr);
        } else {  // split 1 - z/2 around qx ~ |x|/4 so that the subtraction from 1 is exact
            const double qx = ax > 0.78125 ? 0.28125 : __hiloint2double(__double2hiint(ax) - 0x00200000, 0);
            const double hz = 0.5 * z - qx;
            cs = (1.0 - qx) - (hz - zr);
        }
        return make_double2(sn, cs);
    }
    double sn, cs;
    sincos(x, &sn, &cs);
    return make_double2(sn, cs);
}
__device__ __forceinline__ void m_sincos(double x, double* s, double* c) {
    const double2 r = m_sincos_impl(x);
    *s = r.x;
    *c = r.y;
}
static __device__ __noinline__ double m_pow(double x, double y) { return pow(x, y); }
static __device__ __noinline__ double m_fmod(double a, double b) { return fmod(a, b); }
// n / d for a finite non-zero d.  An exactly zero numerator (a vehicle that sits on its lane centre with the lane's
// heading: most of a highway) sends the compiler's fp64 division to its out-of-line slow path (~100 instructions);
// (+-0) / d = (+-0) * d for every finite non-zero d, sign included.
__device__ __forceinline__ double div_finite(double n, double d) { return n == 0.0 ? n * d : n / d; }
// x ** delta of IDMVehicle.acceleration (behavior.py:183-186) for x >= 0.  DELTA = 4.0 unless randomize_behavior was
// called: x^4 from two exact squarings (x*x = p + e and p*p = q + f with fma residuals), (p + e)^2 = q + f + 2pe + e^2
// rounded once — within 0.51 ulp of the exact power, the quality of glibc's pow behind numpy's `**` (CUDA's pow is a
// ~200-instruction routine with a 2 ulp bound).  Below x^4 ~ 2^-968 (x < ~1e-73) the residuals are no longer exact
// doubles: there the error is at most 0.5 ulp + 1.5 * 2^-1074 (<= 2 ulp in the lowest binade).  Any other exponent, huge or
// non-finite x: the library pow.  tests/test_gpu_device_math.py measures these bounds on the device.
//
// randomize_behavior (highway-v0 / highway-fast-v0 traffic) draws DELTA from U(3.5, 4.5): then x^delta = x^4 * x^d with
// |d| = |delta - 4| <= 0.5, the first factor as above and the second as exp(d * log(x)).  The usual weakness of
// exp(y log x) — the error of log(x) is multiplied by y log x — is small here because |d log x| <= 0.35 for x in
// [0.5, 2] (ratios of a speed to its target): ~1.5 ulp on top of the two functions' own 1 ulp, the same class as the
// library pow's 2 ulp bound.  For small x the rounding of d * log(x) (|d log x| <= 69 down to x = 1e-60) dominates:
// a relative error below 1e-14, irrelevant where (1 - x^delta) is what is used.  It replaces ~175 issued instructions per call by ~80.  HWY_LIBRARY_POW restores the library call.
static __device__ __noinline__ double m_exp_dlog(double d, double x) { return exp(d * log(x)); }
__device__ __forceinline__ double idm_pow(double x, double delta) {
#ifndef HWY_LIBRARY_POW
    if (x < 1e60 && fabs(delta - 4.0) <= 0.5) {
#else
    if (delta == 4.0 && x < 1e70) {
#endif
        const double p = x * x, e = fma(x, x, -p);
        const double q = p * p, f = fma(p, p, -q);
        const double x4 = q + (f + 2.0 * (p * e));
#ifndef HWY_LIBRARY_POW
        if (delta == 4.0) return x4;
        if (x > 1e-60) return x4 * m_exp_dlog(delta - 4.0, x);
        if (x == 0.0) return 0.0;  // 0 ** delta, delta > 0
#else
        return x4;
#endif
    }
    return m_pow(x, delta);
}


// Python floored float modulo (b > 0 here).  fmod() is exact, so the cases around the principal range need no call:
//   0 <= a < b      -> |a|          (-0.0 % b is +0.0: fmod gives -0.0, then CPython's copysign(0, b))
//   b <= a < 2b     -> a - b        (exact by Sterbenz: b <= a <= 2b)
//   -b <= a < 0     -> fmod = a, then the sign fix-up `+= b` (one rounded add, as CPython's float_rem does)
//   b == 1          -> a - floor(a) (exact) for a >= 0
// Everything else takes the library fmod (a bit-serial loop).
static __device__ __noinline__ double py_mod_slow(double a, double b) {
    double m = m_fmod(a, b);
    if (m != 0.0) {
        if (m < 0) m += b;
    } else {
        m = 0.0;
    }
    return m;
}
__device__ __forceinline__ double py_mod_pos(double a, double b) {
    if (a >= 0.0) {
        if (a < b) return fabs(a);
        if (a < b + b) return a - b;
        if (b == 1.0 && a < 4503599627370496.0) return a - floor(a);
    } else if (a >= -b) {
        return a + b;
    }
    return py_mod_slow(a, b);
}
// utils.py:59-60
__device__ __forceinline__ double wrap_to_pi(double x) { return py_mod_pos(x + kPi, kTwoPi) - kPi; }
// utils.py:31-33
__device__ __forceinline__ double lmap(double v, double x0, double x1, double y0, double y1) {
    return y0 + (v - x0) * (y1 - y0) / (x1 - x0);
}

// numpy Generator(PCG64): 128-bit LCG, XSL-RR output (numpy/random/src/pcg64/pcg64.h)
struct Pcg64 {
    uint64_t s_hi, s_lo, i_hi, i_lo;
    uint32_t has32, u32;

    __device__ __forceinline__ uint64_t next64() {
        const uint64_t m_hi = 0x2360ed051fc65da4ULL, m_lo = 0x4385df649fccf645ULL;
        uint64_t lo = s_lo * m_lo;
        uint64_t hi = __umul64hi(s_lo, m_lo) + s_hi * m_lo + s_lo * m_hi;
        uint64_t nlo = lo + i_lo;
        uint64_t carry = nlo < lo ? 1 : 0;
        s_lo = nlo;
        s_hi = hi + i_hi + carry;
        uint64_t x = s_hi ^ s_lo;
        unsigned rot = (unsigned)(s_hi >> 58);
        return (x >> rot) | (x << ((64 - rot) & 63));
    }
    __device__ __forceinline__ uint32_t next32() {
        if (has32) {
            has32 = 0;
            return u32;
        }
        uint64_t n = next64();
        has32 = 1;
        u32 = (uint32_t)(n >> 32);
        return (uint32_t)n;
    }
    __device__ __forceinline__ double next_double() {
        return (double)(next64() >> 11) * (1.0 / 9007199254740992.0);
    }
    // Generator.uniform (distributions.c random_uniform)
    __device__ __forceinline__ double uniform(double lo, double hi) {
        double range = hi - lo;
        return lo + range * next_double();
    }
    // Generator.normal() = random_standard_normal (distributions.c): 256-layer ziggurat on one
    // 64-bit output (8 bits layer, 1 bit sign, 52 bits magnitude); wedge and tail are rejection
    // sampled with further doubles.  Bit-exact on the fast path (99.2 %); the wedge/tail paths
    // use CUDA's exp/log1p, which may differ from numpy's by an ulp.
    __device__ __noinline__ double normal() {
        for (;;) {
            uint64_t r = next64();
            int idx = (int)(r & 0xff);
            r >>= 8;
            int sign = (int)(r & 0x1);
            uint64_t rabs = (r >> 1) & 0x000fffffffffffffULL;
            double x = (double)rabs * __longlong_as_double((long long)k_wi_double_bits[idx]);
            if (sign & 0x1) x = -x;
            if (rabs < k_ki_double_bits[idx]) return x;
            if (idx == 0) {
                for (;;) {
                    double xx = -kZigguratNorInvR * log1p(-next_double());
                    double yy = -log1p(-next_double());
                    if (yy + yy > xx * xx)
                        return ((rabs >> 8) & 0x1) ? -(kZigguratNorR + xx) : kZigguratNorR + xx;
                }
            } else {
                double f1 = __longlong_as_double((long long)k_fi_double_bits[idx - 1]);
                double f0 = __longlong_as_double((long long)k_fi_double_bits[idx]);
                if ((f1 - f0) * next_double() + f0 < exp(-0.5 * x * x)) return x;
            }
        }
    }
    // Generator.choice(n) / integers(0, n): Lemire rejection on buffered 32-bit draws
    __device__ __forceinline__ int choice(int n) {
        uint32_t rng = (uint32_t)(n - 1);
        if (rng == 0) return 0;
        uint32_t rng_excl = rng + 1;
        uint64_t m = (uint64_t)next32() * rng_excl;
        uint32_t leftover = (uint32_t)m;
        if (leftover < rng_excl) {
            uint32_t threshold = (0xffffffffu - rng) % rng_excl;
            while (leftover < threshold) {
                m = (uint64_t)next32() * rng_excl;
                leftover = (uint32_t)m;
            }
        }
        return (int)(m >> 32);
    }
};

// The stream words of env e in a [5][n] table (HwyHighwayState.rng, HwyNetState.rng): state hi / lo, increment
// hi / lo, has32 << 32 | u32.
__device__ __forceinline__ Pcg64 load_rng(const uint64_t* rng, size_t n, int e) {
    Pcg64 g;
    g.s_hi = rng[0 * n + e];
    g.s_lo = rng[1 * n + e];
    g.i_hi = rng[2 * n + e];
    g.i_lo = rng[3 * n + e];
    uint64_t w4 = rng[4 * n + e];
    g.has32 = (uint32_t)(w4 >> 32);
    g.u32 = (uint32_t)w4;
    return g;
}
// the words a draw changes: the state and the buffered 32-bit half (the increment is constant)
__device__ __forceinline__ void store_rng(uint64_t* rng, size_t n, int e, const Pcg64& g) {
    rng[0 * n + e] = g.s_hi;
    rng[1 * n + e] = g.s_lo;
    rng[4 * n + e] = ((uint64_t)g.has32 << 32) | g.u32;
}
// all five words
__device__ __forceinline__ void store_rng_all(uint64_t* rng, size_t n, int e, const Pcg64& g) {
    store_rng(rng, n, e, g);
    rng[2 * n + e] = g.i_hi;
    rng[3 * n + e] = g.i_lo;
}

}  // namespace hwy
