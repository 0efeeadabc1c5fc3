// hwy_highway.cu — sm_90a kernels + C ABI for the straight-highway family
// (highway-v0 / highway-fast-v0) of the batched HighwayEnv hot path.
//
// Thread mapping of the step kernel: one (env, vehicle) pair per thread, each env a dense segment of V = n_vehicles
// consecutive threads of the block (segments start anywhere in a warp); TPE (32/64/128, the next power of two >= V)
// sizes the per-env shared arrays.  The whole AbstractEnv.step — every substep of
// Road.act/Road.step, then observe/reward/termination — runs in ONE kernel, so the SoA state
// makes one HBM round trip per env-step (128-bit loads/stores per vehicle).
//
// Per substep each env stages its vehicles in shared memory ("Frame", double buffered) and
// derives, in parallel and without divergence:
//   * the rank of every vehicle along the road and per-lane membership bit-masks in rank
//     order, which turn Road.neighbour_vehicles (the reference's 65 % hot spot, an O(V) scan
//     per query) into two bit-scans;
//   * per-lane target / lane bit-masks that prune IDMVehicle.change_lane_policy's abort scan
//     to the handful of vehicles that can matter;
//   * the collision sweep as a pair-parallel pass (sphere pre-check per pair, SAT only for
//     the rare close pairs) reduced per vehicle with shared-memory atomics.
// The reference's sequential semantics (Gauss-Seidel target-lane updates in Road.act,
// last-writer-wins impacts in Road.step, tie rules of the neighbour search) are preserved:
// see DESIGN.md "ordering".  Reference paths are relative to /root/reference/highway_env.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <atomic>
#include <cstddef>
#include <mutex>

#include <cuda_runtime.h>

#include "../../include/hwyb200.h"
#include "hwy_device.cuh"
#include "hwy_math.cuh"

namespace hwy {

// Optional per-phase cycle accounting (-DHWY_PHASE_TIMING): warp-level clock64() deltas summed
// into g_phase_cycles; read with hwy_debug_phase_cycles().  Off in the shipped build.
#ifdef HWY_PHASE_TIMING
__device__ unsigned long long g_phase_cycles[16];
#define PHASE_INIT() long long _pt = clock64()
#define PHASE_MARK(k)                                                                 \
    do {                                                                              \
        long long _n = clock64();                                                     \
        if ((threadIdx.x & 31) == 0) atomicAdd(&g_phase_cycles[k], (unsigned long long)(_n - _pt)); \
        _pt = _n;                                                                     \
    } while (0)
#else
#define PHASE_INIT()
#define PHASE_MARK(k)
#endif

// ------------------------------------------------------------------ shared staging
template <int TPE>
struct Frame {
    static constexpr int NW = TPE / 32;
    double x[TPE], y[TPE], c[TPE], s[TPE], v[TPE], ts[TPE];
    double ls[TPE];                          // longitudinal coordinate on lane 0
    __align__(16) float lsf[TPE];            // the same rounded to float (monotone): rank pre-sort key
    uint32_t smask[HWY_MAX_LANES][NW];       // rank-ordered on_lane(margin=1) membership of lane l
    uint32_t tm[HWY_MAX_LANES][NW];          // vehicles whose target lane is l   (slot order)
    uint32_t lane_is[HWY_MAX_LANES][NW];     // vehicles whose lane_index is l    (slot order)
    uint32_t fired[NW];                      // IDM vehicles whose lane-change timer will fire
    unsigned char lane[TPE], tgt[TPE], perm[TPE], rank[TPE];
    int slow;                                // ties in ls or unaligned lanes: use the linear scans
    unsigned vmax_bits;                      // max(0, max speed) of the env, float bits rounded up (pruned sweep bound)
};

template <int TPE>
struct EnvShared {
    static constexpr int NW = TPE / 32;
    Frame<TPE> f[2];
    double key[TPE];                         // observation sort keys
    uint32_t geo[TPE][NW];                   // abort-scan hits (0 < d < d*) of mid-change vehicles
    uint32_t mid[NW];                        // active mid-change IDM vehicles (lane != target)
    // MOBIL work list: (vehicle, candidate lane) items pushed by the vehicles whose timer fired
    // and evaluated densely by the env's first threads; accepted candidates set ok_left/ok_right.
    uint32_t ok_left[NW], ok_right[NW];
    int n_items;
    unsigned short items[2 * TPE];
    double free_t[TPE], acc_own[TPE], delta[TPE];  // own IDM free-road term / own-lane acceleration / DELTA
    signed char f_own[TPE], r_own[TPE];      // own-lane preceding / following vehicle (-1: none)
    uint32_t ctrl[NW], cc[NW];               // ControlledVehicle instances / check_collisions
    int last_will[TPE];                      // collision sweep: largest partner with will_intersect
    unsigned char crash_hit[TPE];
    // fused autoreset staging (Vehicle.create_random chain): per-vehicle spawn increment / position
    double sp_x[TPE];
    int done, sp_fallback;
};

// All envs of a block advance in lock-step (block-wide barriers): besides ordering the shared
// staging it keeps the block's warps on the same code at the same time, which is what the
// instruction cache wants from a ~100 KB kernel (per-env barriers were slower).
template <int TPE>
__device__ __forceinline__ void env_sync() {
    __syncthreads();
}
template <int TPE, int LEVEL>
__device__ __forceinline__ void env_sync_phase() {
    __syncthreads();
}

template <int NW>
__device__ __forceinline__ bool test_bit(const uint32_t (&m)[NW], int i) {
    return (m[i >> 5] >> (i & 31)) & 1u;
}

// Hardware lane, read afresh at each use: a lane index held in a register across the substep loop costs a spill.
__device__ __forceinline__ int lane_id() {
    int l;
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
    return l;
}

// Dense env segments (DENSE step kernels) in a warp.  A warp ballot is indexed by hardware lane, an env's mask words
// by vehicle (bit i & 31 of word i >> 5), and a dense segment starts anywhere in a warp, so a warp holds parts of up
// to three envs.  The first lane of each env's part (vehicle i, lane 0 or i == 0) ORs the part's bits, vehicles
// [i, i + n), into the at most two words they straddle, which must be zero before.  Threads that own no vehicle
// (i >= V) are never a first lane.
__device__ __forceinline__ void segment_or(uint32_t* words, uint32_t ballot, int i, int V) {
    const int lane = lane_id();
    if (i >= V || (i != 0 && lane != 0)) return;
    const int n = min(V - i, 32 - lane);
    const uint32_t m = (ballot >> lane) & (0xffffffffu >> (32 - n));
    if (!m) return;
    const int sh = i & 31;
    atomicOr(&words[i >> 5], m << sh);
    const uint32_t hi = __funnelshift_l(m, 0u, sh);  // m >> (32 - sh), 0 for sh == 0
    if (hi) atomicOr(&words[(i >> 5) + 1], hi);
}
// The env segments of the calling warp as a ballot of their first lanes, and the index of the caller's segment among
// them (threads past the last env count as part of the last segment).  Warp-wide.
__device__ __forceinline__ uint32_t segment_leads(int i, bool active, int& mine) {
    const int lane = lane_id();
    const uint32_t lead = __ballot_sync(0xffffffffu, active && (i == 0 || lane == 0));
    mine = __popc(lead & (0xffffffffu >> (31 - lane))) - 1;
    return lead;
}

// ------------------------------------------------------------------ neighbour search
// road/road.py:483-547 neighbour_vehicles, same-segment search, exact linear form (used when
// two vehicles share a longitudinal coordinate or the lanes are not axis aligned).
// Ties: front `<=` keeps the later index, rear `>` keeps the earlier one.
template <int TPE>
__device__ __noinline__ void neighbours_linear(const Frame<TPE>& F, const HwyStraightLane L, int V,
                                               int self, int& front, int& rear) {
    double s = lane_s(L, F.x[self], F.y[self]);
    double s_front = 0, s_rear = 0;
    front = -1;
    rear = -1;
    for (int v = 0; v < V; ++v) {
        if (v == self) continue;
        double s_v, lat_v;
        lane_local(L, F.x[v], F.y[v], s_v, lat_v);
        if (!lane_on(L, s_v, lat_v, 1.0)) continue;
        if (s <= s_v && (front < 0 || s_v <= s_front)) {
            s_front = s_v;
            front = v;
        }
        if (s_v < s && (rear < 0 || s_v > s_rear)) {
            s_rear = s_v;
            rear = v;
        }
    }
}

// Same query through the rank-ordered membership mask: the preceding vehicle is the member of
// lane l with the lowest rank above ours, the following one the highest rank below.
template <int TPE>
__device__ __forceinline__ void neighbours(const HwyHighwayParams& P, const Frame<TPE>& F, int V, int l,
                                           int self, int& front, int& rear) {
    constexpr int NW = TPE / 32;
    if (F.slow) {
        neighbours_linear(F, P.lanes[l], V, self, front, rear);
        return;
    }
    const int r = F.rank[self];
    const int w0 = r >> 5, b = r & 31;
    front = -1;
    rear = -1;
    uint32_t m = F.smask[l][w0] & (b == 31 ? 0u : (~0u << (b + 1)));
    int w = w0;
    while (m == 0 && ++w < NW) m = F.smask[l][w];
    if (m) front = F.perm[w * 32 + __ffs(m) - 1];
    m = F.smask[l][w0] & ((1u << b) - 1u);
    w = w0;
    while (m == 0 && --w >= 0) m = F.smask[l][w];
    if (m) rear = F.perm[w * 32 + 31 - __clz(m)];
}

// The same query as a real call (front | rear << 8, 0xff = none) for the places that are not on every thread's path
// (MOBIL items, the target-lane query of a vehicle that is changing lanes): three inlined copies of the bit scans cost
// 5 KB of the per-substep loop.
template <int TPE>
__device__ __noinline__ int neighbours_packed(const uint32_t* __restrict__ smask_l, const Frame<TPE>& F, int self) {
    constexpr int NW = TPE / 32;
    const int r = F.rank[self];
    const int w0 = r >> 5, b = r & 31;
    int front = 0xff, rear = 0xff;
    uint32_t m = smask_l[w0] & (b == 31 ? 0u : (~0u << (b + 1)));
    int w = w0;
    while (m == 0 && ++w < NW) m = smask_l[w];
    if (m) front = F.perm[w * 32 + __ffs(m) - 1];
    m = smask_l[w0] & ((1u << b) - 1u);
    w = w0;
    while (m == 0 && --w >= 0) m = smask_l[w];
    if (m) rear = F.perm[w * 32 + 31 - __clz(m)];
    return front | (rear << 8);
}
template <int TPE>
__device__ __forceinline__ void neighbours_cold(const HwyHighwayParams& P, const Frame<TPE>& F, int V, int l,
                                                int self, int& front, int& rear) {
    if (F.slow) {
        neighbours_linear(F, P.lanes[l], V, self, front, rear);
        return;
    }
    const int fr = neighbours_packed(F.smask[l], F, self);
    front = (fr & 0xff) == 0xff ? -1 : (fr & 0xff);
    rear = (fr >> 8) == 0xff ? -1 : (fr >> 8);
}

// ------------------------------------------------------------------ IDM (vehicle/behavior.py)
// Scalars of the IDM the out-of-line helpers need (passing the kernel-parameter struct by
// reference to a __noinline__ function would force a per-thread local copy of it).
struct IdmK {
    double comfort_acc_max, distance_wanted, time_wanted, two_sqrt_ab;
};
__device__ __forceinline__ IdmK make_idm(const HwyHighwayParams& P) {
    IdmK k;
    k.comfort_acc_max = P.comfort_acc_max;
    k.distance_wanted = P.distance_wanted;
    k.time_wanted = P.time_wanted;
    k.two_sqrt_ab = 2 * sqrt(-P.comfort_acc_max * P.comfort_acc_min);  // 2 * np.sqrt(ab)
    return k;
}
// :192-217 desired_gap(ego, front), projected
template <int TPE>
__device__ __forceinline__ double desired_gap(const IdmK& K, const Frame<TPE>& F, int ego, int front) {
    double dvx = F.v[ego] * F.c[ego] - F.v[front] * F.c[front];
    double dvy = F.v[ego] * F.s[ego] - F.v[front] * F.s[front];
    double dv = dot2(dvx, dvy, F.c[ego], F.s[ego]);
    return K.distance_wanted + F.v[ego] * K.time_wanted + F.v[ego] * dv / K.two_sqrt_ab;
}
// lane_distance_to on the ego's own lane (vehicle/objects.py:183-198)
template <int TPE>
__device__ __forceinline__ double lane_distance(const HwyHighwayParams& P, const Frame<TPE>& F,
                                                bool aligned, int ego, int other) {
    if (aligned) return F.ls[other] - F.ls[ego];
    const HwyStraightLane& L = P.lanes[F.lane[ego]];
    return lane_s(L, F.x[other], F.y[other]) - lane_s(L, F.x[ego], F.y[ego]);
}
// :150-190 acceleration(): free-road term with the CALLER's DELTA ...
__device__ __noinline__ double idm_free_term(double comfort_acc_max, double speed, double target_speed,
                                             double speed_limit, double delta) {
    double ego_target_speed = clipd(target_speed, 0.0, speed_limit);
    return comfort_acc_max * (1 - idm_pow(fmax(speed, 0.0) / fabs(not_zero(ego_target_speed)), delta));
}
// ... and the interaction term COMFORT_ACC_MAX * (d* / not_zero(d))^2 for a given gap d
template <int TPE>
__device__ __noinline__ double idm_gap_core(const IdmK K, const Frame<TPE>& F, int ego, int front, double d) {
    double q = desired_gap(K, F, ego, front) / not_zero(d);
    return K.comfort_acc_max * (q * q);  // np.power(q, 2)
}
template <int TPE>
__device__ __forceinline__ double idm_gap_term(const HwyHighwayParams& P, const IdmK& K,
                                               const Frame<TPE>& F, bool aligned, int ego, int front) {
    return idm_gap_core(K, F, ego, front, lane_distance(P, F, aligned, ego, front));
}
// acceleration(ego_vehicle=ego, front_vehicle=front) for an `ego` other than the caller
template <int TPE>
__device__ __forceinline__ double idm_acceleration_of(const HwyHighwayParams& P, const IdmK& K,
                                                      const Frame<TPE>& F, bool aligned, double delta,
                                                      int ego, int front) {
    if (ego < 0) return 0.0;
    double acc = idm_free_term(K.comfort_acc_max, F.v[ego], F.ts[ego],
                               P.lanes[F.lane[ego]].speed_limit, delta);
    if (front >= 0) acc -= idm_gap_term(P, K, F, aligned, ego, front);
    return acc;
}

// ------------------------------------------------------------------ LinearVehicle (vehicle/behavior.py:350-583)
// Per-env shared staging of the traffic's linear parameters, placed after the block's EnvShared array by the linear
// kernel only (so EnvShared and the IDM kernel keep their layout): MOBIL items read the item owner's parameters.
template <int TPE>
struct LinearShared {
    double acc[3][TPE];    // ACCELERATION_PARAMETERS
    double steer[2][TPE];  // STEERING_PARAMETERS
};

// python min(x, 0): x unless 0 < x
__device__ __forceinline__ double py_min0(double x) { return 0.0 < x ? 0.0 : x; }

// :417-465 acceleration(ego_vehicle=ego, front_vehicle=front) with the CALLER's parameters (a0, a1, a2):
// np.dot(ACCELERATION_PARAMETERS, [vt, dv, dp]), which numpy's BLAS evaluates as fma(a2, dp, fma(a1, dv, a0 * vt)).
// F.ts holds getattr(ego, "target_speed", ego.speed) (publish<..., true>).
template <int TPE>
__device__ __forceinline__ double linear_acceleration(const HwyHighwayParams& P, const IdmK& K, const Frame<TPE>& F,
                                                      bool aligned, double a0, double a1, double a2, int ego,
                                                      int front) {
    if (ego < 0) return 0.0;
    const double v = F.v[ego];
    const double vt = F.ts[ego] - v;
    double dv = 0.0, dp = 0.0;
    if (front >= 0) {
        const double d_safe = K.distance_wanted + fmax(v, 0.0) * K.time_wanted;
        const double d = lane_distance(P, F, aligned, ego, front);
        dv = py_min0(F.v[front] - v);
        dp = py_min0(d - d_safe);
    }
    return __fma_rn(a2, dp, __fma_rn(a1, dv, a0 * vt));
}

// :467-502 steering_control(target_lane) on a StraightLane (heading_at is the lane heading), then IDMVehicle.act's
// clip to +-MAX_STEERING_ANGLE (:107-110); np.dot on the 2 features is fma(s1, f1, s0 * f0).
static __device__ __noinline__ double linear_steering(const HwyStraightLane L, double x, double y, double heading,
                                                      double speed, double s0, double s1) {
    double lc_s, lc_lat;
    lane_local(L, x, y, lc_s, lc_lat);
    const double nz = not_zero(speed);
    const double f0 = wrap_to_pi(L.heading - heading) * kVehLength / nz;
    // (not_zero(v) ** 2 is the host libm's pow there, which can differ from the exact-rounded nz * nz by 1 ulp)
    const double f1 = -lc_lat * kVehLength / (nz * nz);
    return clipd(__fma_rn(s1, f1, s0 * f0), -kMaxSteer, kMaxSteer);
}

// ------------------------------------------------------------------ observation
// envs/common/observation.py:234-276 KinematicObservation.observe (presence,x,y,vx,vy; order
// "sorted") with road/road.py:421-450 close_objects_to and kinematics.py:237-261 to_dict.
__device__ __forceinline__ int obs_columns(const HwyHighwayParams& P) {
    return P.obs_n_features > 0 ? P.obs_n_features : 5;
}

// One observation row with a configured feature list (Vehicle.to_dict, vehicle/kinematics.py:237-261;
// normalize_obs, observation.py:207-232).  Out of line: the default five columns never come here.
__device__ __noinline__ void kinematics_row_features(const HwyHighwayParams& P, int lane, double x, double y,
                                                     double heading, double c, double s, double dx, double dy,
                                                     double dvx, double dvy, float* __restrict__ o,
                                                     float* __restrict__ o2) {
    const HwyStraightLane L = P.lanes[lane];
    double lon, lat;
    lane_local(L, x, y, lon, lat);  // Vehicle.lane_offset :228-235
    for (int col = 0; col < P.obs_n_features; ++col) {
        double v = 0.0;
        switch (P.obs_feature[col]) {
            case HWY_FEAT_PRESENCE: v = 1.0; break;
            case HWY_FEAT_X: v = dx; break;
            case HWY_FEAT_Y: v = dy; break;
            case HWY_FEAT_VX: v = dvx; break;
            case HWY_FEAT_VY: v = dvy; break;
            case HWY_FEAT_HEADING: v = heading; break;
            case HWY_FEAT_COS_H: v = c; break;
            case HWY_FEAT_SIN_H: v = s; break;
            case HWY_FEAT_LONG_OFF: v = lon; break;
            case HWY_FEAT_LAT_OFF: v = lat; break;
            case HWY_FEAT_ANG_OFF: v = wrap_to_pi(heading - L.heading); break;  // lane.local_angle (lane.py:145-147)
            default: v = 0.0; break;  // cos_d / sin_d: no route on this road family => destination == position
        }
        if (P.obs_normalize && P.obs_feature_ranged[col]) {
            v = lmap(v, P.obs_feature_lo[col], P.obs_feature_hi[col], -1.0, 1.0);
            if (P.obs_clip) v = clipd(v, -1.0, 1.0);
        }
        o[col] = (float)v;
        if (o2) o2[col] = (float)v;
    }
}

// DENSE (dense step kernels): threads i >= V own no vehicle and store nothing; the V threads pad the missing rows.
template <int TPE, bool DENSE = false>
__device__ __forceinline__ void kinematics_observe(const HwyHighwayParams& P, const Frame<TPE>& F,
                                                   double* key_scratch, int i, double heading,
                                                   float* __restrict__ obs_env,
                                                   float* __restrict__ obs_env2 = nullptr) {
    const int V = P.n_vehicles, K = P.obs_vehicles_count;
    const HwyStraightLane& Le = P.lanes[F.lane[0]];
    const double ex = F.x[0], ey = F.y[0];
    const double evx = F.v[0] * F.c[0], evy = F.v[0] * F.s[0];
    double key = INFINITY;
    if (i > 0 && i < V) {
        bool ok = norm2(F.x[i] - ex, F.y[i] - ey) < P.perception_distance;
        double d = lane_s(Le, F.x[i], F.y[i]) - lane_s(Le, ex, ey);
        ok = ok && (P.obs_see_behind || -2 * kVehLength < d);
        if (ok) key = fabs(d);
    }
    if (!DENSE || i < V) key_scratch[i] = key;
    env_sync<TPE>();
    // stable rank among the valid candidates (python sorted() on |lane_distance_to|)
    int rank = 0, n_valid = 0;
    for (int u = 1; u < V; ++u) {
        double ku = key_scratch[u];
        n_valid += ku < INFINITY;
        rank += (ku < key) || (ku == key && u < i);
    }
    // obs_env == nullptr: an env of the block that is not observed (masked out, a surplus slot of the last block, not
    // re-spawned), or in a dense kernel a thread that owns no vehicle.  It still runs to here so that every thread of
    // the block meets the same barrier instruction.
    if (!obs_env) return;
    const double xr = 5.0 * kMaxSpeed, yr = 4.0 * P.lanes_count, vr = 2 * kMaxSpeed;
    int row = -1;
    double r1 = 0, r2 = 0, r3 = 0, r4 = 0;
    if (i == 0) {
        row = 0;
        r1 = ex;
        r2 = ey;
        r3 = evx;
        r4 = evy;
    } else if (key < INFINITY && rank < K - 1) {
        row = rank + 1;
        r1 = F.x[i];
        r2 = F.y[i];
        r3 = F.v[i] * F.c[i];
        r4 = F.v[i] * F.s[i];
        if (!P.obs_absolute) {
            r1 -= ex;
            r2 -= ey;
            r3 -= evx;
            r4 -= evy;
        }
    }
    const int NF = obs_columns(P);
    if (row >= 0 && P.obs_n_features > 0) {
        kinematics_row_features(P, F.lane[i], F.x[i], F.y[i], heading, F.c[i], F.s[i], r1, r2, r3, r4,
                                obs_env + NF * row, obs_env2 ? obs_env2 + NF * row : nullptr);
    } else if (row >= 0) {
        if (P.obs_normalize) {  // normalize_obs :207-232
            r1 = lmap(r1, -xr, xr, -1.0, 1.0);
            r2 = lmap(r2, -yr, yr, -1.0, 1.0);
            r3 = lmap(r3, -vr, vr, -1.0, 1.0);
            r4 = lmap(r4, -vr, vr, -1.0, 1.0);
            if (P.obs_clip) {
                r1 = clipd(r1, -1.0, 1.0);
                r2 = clipd(r2, -1.0, 1.0);
                r3 = clipd(r3, -1.0, 1.0);
                r4 = clipd(r4, -1.0, 1.0);
            }
        }
        float* o = obs_env + 5 * row;
        o[0] = 1.0f;
        o[1] = (float)r1;
        o[2] = (float)r2;
        o[3] = (float)r3;
        o[4] = (float)r4;
        if (obs_env2) {
            o = obs_env2 + 5 * row;
            o[0] = 1.0f;
            o[1] = (float)r1;
            o[2] = (float)r2;
            o[3] = (float)r3;
            o[4] = (float)r4;
        }
    }
    int filled = 1 + (n_valid < K - 1 ? n_valid : K - 1);  // zero padding of missing rows
    if constexpr (DENSE) {
        for (int pad = i; i < V && pad < K; pad += V) {  // (K may exceed V)
            if (pad < filled) continue;
            for (int col = 0; col < NF; ++col) {
                obs_env[NF * pad + col] = 0.0f;
                if (obs_env2) obs_env2[NF * pad + col] = 0.0f;
            }
        }
    } else if (i < K && i >= filled) {
        for (int col = 0; col < NF; ++col) {
            obs_env[NF * i + col] = 0.0f;
            if (obs_env2) obs_env2[NF * i + col] = 0.0f;
        }
    }
}

// ------------------------------------------------------------------ state I/O
struct VehicleRegs {
    double x, y, heading, speed, target_speed, timer, delta, imp_x, imp_y;
    int meta;
};

__device__ __forceinline__ void load_vehicle(const HwyHighwayState& S, size_t slot, VehicleRegs& r) {
    double2 a = reinterpret_cast<const double2*>(S.pos)[slot];
    double2 b = reinterpret_cast<const double2*>(S.hs)[slot];
    double2 c = reinterpret_cast<const double2*>(S.tt)[slot];
    double2 d = reinterpret_cast<const double2*>(S.imp)[slot];
    r.x = a.x;
    r.y = a.y;
    r.heading = b.x;
    r.speed = b.y;
    r.target_speed = c.x;
    r.timer = c.y;
    r.imp_x = d.x;
    r.imp_y = d.y;
    r.delta = S.delta[slot];
    r.meta = S.meta[slot];
}
__device__ __forceinline__ void store_vehicle(const HwyHighwayState& S, size_t slot,
                                              const VehicleRegs& r) {
    reinterpret_cast<double2*>(S.pos)[slot] = make_double2(r.x, r.y);
    reinterpret_cast<double2*>(S.hs)[slot] = make_double2(r.heading, r.speed);
    reinterpret_cast<double2*>(S.tt)[slot] = make_double2(r.target_speed, r.timer);
    reinterpret_cast<double2*>(S.imp)[slot] = make_double2(r.imp_x, r.imp_y);
    S.meta[slot] = r.meta;  // delta never changes during a step
}

// Stage one vehicle into frame F (plain stores) and clear the words of F that build_frame fills
// with atomics (DENSE: the caller does, clear_masks).  Callers put a barrier between publish() and build_frame().
template <int TPE, bool LINEAR = false, bool DENSE = false>
__device__ __forceinline__ void publish(const HwyHighwayParams& P, Frame<TPE>& F, int i, bool active,
                                        const VehicleRegs& r) {
    constexpr int NW = TPE / 32;
    if (active) {
        double sn, cs;
        m_sincos(r.heading, &sn, &cs);
        F.x[i] = r.x;
        F.y[i] = r.y;
        F.c[i] = cs;
        F.s[i] = sn;
        F.v[i] = r.speed;
        // getattr(ego_vehicle, "target_speed", 0): a plain Vehicle has none (behavior.py:172); the linear model's
        // default is the vehicle's own speed (behavior.py:449-452)
        F.ts[i] = meta_kind(r.meta) == HWY_KIND_VEHICLE ? (LINEAR ? r.speed : 0.0) : r.target_speed;
        F.ls[i] = lane_s(P.lanes[0], r.x, r.y);
        F.lsf[i] = (float)F.ls[i];
        F.lane[i] = (unsigned char)meta_lane(r.meta);
        F.tgt[i] = (unsigned char)meta_target(r.meta);
    }
    if (!DENSE && i < HWY_MAX_LANES * NW) (&F.smask[0][0])[i] = 0;
    if (i == 0) {
        F.slow = 0;
        F.vmax_bits = 0u;
    }
}

// Dense step kernels: zero the words build_frame ORs into (smask, tm, lane_is, fired: adjacent in Frame), spread over
// the env's V threads.
template <int TPE>
__device__ __forceinline__ void clear_masks(Frame<TPE>& F, int i, int V) {
    constexpr int kWords = (3 * HWY_MAX_LANES + 1) * (TPE / 32);
    static_assert(offsetof(Frame<TPE>, fired) + sizeof(F.fired) - offsetof(Frame<TPE>, smask) == 4 * kWords,
                  "mask words of Frame are not adjacent");
#pragma unroll 1  // (unrolled, it costs the step kernel 70 B of spills)
    for (int k = i; k < kWords; k += V) (&F.smask[0][0])[k] = 0;
}

// Collision test of the pair a < b on the staged positions (vehicle/objects.py:92-138):
// handle_collisions' gate is applied by the caller, _is_colliding here.
// The sphere pre-check is split: the squared-distance reject (the vast majority of the pairs) is inline, the exact
// `dist > thr` of the reference with its square root sits at the top of the out-of-line pair_sat.
template <int TPE>
__device__ __forceinline__ bool pair_precheck(const Frame<TPE>& F, int a, int b, double dt) {
    const double diag = sqrt(kVehLength * kVehLength + kVehWidth * kVehWidth);
    const double thr = (diag + diag) / 2 + F.v[a] * dt;
    const double dx = F.x[b] - F.x[a], dy = F.y[b] - F.y[a];
    // far pairs: d^2 clearly above thr^2 => the exact test in pair_sat is true too
    return !(thr >= 0.0 && dx * dx + dy * dy > thr * thr * 1.000001 + 1e-9);
}
template <int TPE>
__device__ __noinline__ void pair_sat(const Frame<TPE>& F, int a, int b, double dt, bool& inter,
                                      bool& will, double& trx, double& try_) {
    {
        const double diag = sqrt(kVehLength * kVehLength + kVehWidth * kVehWidth);
        const double thr = (diag + diag) / 2 + F.v[a] * dt;
        const double dist = norm2(F.x[b] - F.x[a], F.y[b] - F.y[a]);
        if (dist > thr) {  // vehicle/objects.py:122-126
            inter = false;
            will = false;
            trx = try_ = 0.0;
            return;
        }
    }
    // Conservative shortcut.  The reference's flags are sticky ANDs over the visited edge
    // normals and its `break` only triggers once both are False, so if ONE of the four distinct
    // rectangle axes separates the rectangles statically AND after the relative-displacement
    // extension, the result is (False, False, None) whatever the other axes say.  We test that
    // in closed form with a 1e-6 m safety margin (>> the ~1e-12 rounding of either evaluation);
    // anything closer runs the exact SAT below.
    {
        const double hl = kVehLength / 2, hw = kVehWidth / 2, margin = 1e-6;
        const double ca = F.c[a], sa = F.s[a], cb = F.c[b], sb = F.s[b];
        const double dx = F.x[b] - F.x[a], dy = F.y[b] - F.y[a];
        const double rvx = (F.v[a] * ca - F.v[b] * cb) * dt, rvy = (F.v[a] * sa - F.v[b] * sb) * dt;
        const double cd = fabs(ca * cb + sa * sb), sd = fabs(sa * cb - ca * sb);  // |cos|, |sin| of the heading difference
        bool separated = false;
        // axes of a: longitudinal (ca, sa) and lateral (-sa, ca); of b likewise
        separated |= fabs(dx * ca + dy * sa) - (hl + hl * cd + hw * sd) - fabs(rvx * ca + rvy * sa) > margin;
        separated |= fabs(-dx * sa + dy * ca) - (hw + hl * sd + hw * cd) - fabs(-rvx * sa + rvy * ca) > margin;
        separated |= fabs(dx * cb + dy * sb) - (hl + hl * cd + hw * sd) - fabs(rvx * cb + rvy * sb) > margin;
        separated |= fabs(-dx * sb + dy * cb) - (hw + hl * sd + hw * cd) - fabs(-rvx * sb + rvy * cb) > margin;
        if (separated) {
            inter = false;
            will = false;
            trx = try_ = 0.0;
            return;
        }
    }
    Quad pa = make_polygon(F.x[a], F.y[a], F.c[a], F.s[a]);
    Quad pb = make_polygon(F.x[b], F.y[b], F.c[b], F.s[b]);
    polygons_intersecting(pa, pb, F.v[a] * F.c[a] * dt, F.v[a] * F.s[a] * dt, F.v[b] * F.c[b] * dt,
                          F.v[b] * F.s[b] * dt, inter, will, trx, try_);
}

// Rank of vehicle i along the road by counting (O(V) per thread), out of line: it runs on the first frame of a launch
// and when the previous order broke (see build_frame), and its unrolled loops are 8 KB of code that the per-substep
// loop should not carry.  Returns rank | tie << 8.
template <int TPE>
__device__ __noinline__ int rank_count(const Frame<TPE>& F, int V, int i, bool active) {
    const double si = active ? F.ls[i] : 0.0;
    const float fi = active ? F.lsf[i] : 0.0f;
    int rank = 0;
    bool ambiguous = false;
    const float4* lsf4 = reinterpret_cast<const float4*>(F.lsf);
    const int n4 = V >> 2;
    for (int q = 0; q < n4; ++q) {
        float4 f = lsf4[q];
        const int u = q << 2;
        rank += (f.x < fi) + (f.y < fi) + (f.z < fi) + (f.w < fi);
        ambiguous = ambiguous || (f.x == fi && u != i) || (f.y == fi && u + 1 != i) ||
                    (f.z == fi && u + 2 != i) || (f.w == fi && u + 3 != i);
    }
    for (int u = n4 << 2; u < V; ++u) {
        float fu = F.lsf[u];
        rank += fu < fi;
        ambiguous = ambiguous || (fu == fi && u != i);
    }
    bool tie = false;
    if (ambiguous) {
        rank = 0;
#pragma unroll 1
        for (int u = 0; u < V; ++u) {
            double su = F.ls[u];
            rank += (su < si) || (su == si && u < i);
            tie = tie || (su == si && u != i);
        }
    }
    return rank | ((int)tie << 8);
}

// When the chain check of build_frame fails it is almost always because one vehicle overtook its rank-neighbour during
// the substep: boundary k of the previous permutation (between positions k-1 and k) is inverted.  If every inverted
// boundary is strictly inverted (no equal float keys), at least three boundaries away from the next inverted one, and
// swapping its two vehicles leaves them in order with their unmoved outer neighbours, the swapped permutation is again
// a strictly increasing chain of float keys — hence of the doubles — and every vehicle's rank is its old one, +-1 for
// the swapped ones.  Like the chain check this runs redundantly in every warp of the env on shared data (ballots, no
// barrier, no shared-memory writes), ~70 instructions instead of the ~400 of rank_count.  Returns the rank, or -1 when
// the pattern is anything else (rank_count decides).  Boundary k = 32 w + b + 1 is bit b of word w.  DENSE: the warp
// evaluates each env segment it holds in turn, lane b taking boundaries 32 w + b + 1 of that env.
template <int TPE, bool DENSE>
__device__ __noinline__ int rank_repair(const Frame<TPE>& F, const Frame<TPE>& prev, int V, int i, bool active) {
    constexpr int NW = TPE / 32;
    uint32_t inv[NW];
    uint32_t bad = 0;
    if constexpr (!DENSE) {
        const int wl = i & 31;
#pragma unroll
        for (int w = 0; w < NW; ++w) {
            const int k = w * 32 + wl + 1;
            const bool in = k < V;
            const float a = in ? F.lsf[prev.perm[k - 1]] : 0.0f, c = in ? F.lsf[prev.perm[k]] : 1.0f;
            bool wrong = in && !(a < c) && !(a > c);  // equal (or NaN) keys: not this path
            if (in && a > c) {
                // the swapped pair against its outer neighbours (positions k-2 and k+1 are unmoved, see the spacing
                // rule)
                if (k >= 2 && !(F.lsf[prev.perm[k - 2]] < c)) wrong = true;
                if (k + 1 < V && !(a < F.lsf[prev.perm[k + 1]])) wrong = true;
            }
            inv[w] = __ballot_sync(0xffffffffu, in && a > c);
            bad |= __ballot_sync(0xffffffffu, wrong);
        }
    } else {
        const int lane = lane_id();
        int mine;
        int s = 0;
        for (uint32_t lead = segment_leads(i, active, mine); lead; lead &= lead - 1, ++s) {
            // env of segment s: the envs of a block are consecutive EnvShared records
            const ptrdiff_t d = (ptrdiff_t)(s - mine) * (ptrdiff_t)sizeof(EnvShared<TPE>);
            const Frame<TPE>& Fs = *reinterpret_cast<const Frame<TPE>*>(reinterpret_cast<const char*>(&F) + d);
            const Frame<TPE>& Ps = *reinterpret_cast<const Frame<TPE>*>(reinterpret_cast<const char*>(&prev) + d);
            uint32_t s_inv[NW];
            uint32_t s_bad = 0;
#pragma unroll
            for (int w = 0; w < NW; ++w) {
                const int k = w * 32 + lane + 1;
                const bool in = k < V;
                const float a = in ? Fs.lsf[Ps.perm[k - 1]] : 0.0f, c = in ? Fs.lsf[Ps.perm[k]] : 1.0f;
                bool wrong = in && !(a < c) && !(a > c);  // equal (or NaN) keys: not this path
                if (in && a > c) {
                    // the swapped pair against its outer neighbours (positions k-2 and k+1 are unmoved, see the spacing
                    // rule)
                    if (k >= 2 && !(Fs.lsf[Ps.perm[k - 2]] < c)) wrong = true;
                    if (k + 1 < V && !(a < Fs.lsf[Ps.perm[k + 1]])) wrong = true;
                }
                s_inv[w] = __ballot_sync(0xffffffffu, in && a > c);
                s_bad |= __ballot_sync(0xffffffffu, wrong);
            }
            if (s == mine) {
#pragma unroll
                for (int w = 0; w < NW; ++w) inv[w] = s_inv[w];
                bad = s_bad;
            }
        }
    }
    // spacing: no other inverted boundary within two boundaries of an inverted one (also across the word seam)
#pragma unroll
    for (int w = 0; w < NW; ++w) {
        uint32_t near = (inv[w] << 1) | (inv[w] << 2);
        if (w > 0) near |= (inv[w - 1] >> 31) | (inv[w - 1] >> 30);
        bad |= inv[w] & near;
    }
    if (bad) return -1;
    if (!active) return 0;
    const int r0 = prev.rank[i];
    // upper vehicle of an inverted boundary r0 moves down, lower vehicle of an inverted boundary r0 + 1 moves up
    // (static indices only: a dynamically indexed register array would live in local memory)
    uint32_t w_dn = 0, w_up = 0;
#pragma unroll
    for (int w = 0; w < NW; ++w) {
        if (r0 >= 1 && w == ((r0 - 1) >> 5)) w_dn = inv[w];
        if (w == (r0 >> 5)) w_up = inv[w];
    }
    if (r0 >= 1 && ((w_dn >> ((r0 - 1) & 31)) & 1u)) return r0 - 1;
    if (r0 + 1 < V && ((w_up >> (r0 & 31)) & 1u)) return r0 + 1;
    return r0;
}

// After a barrier that follows publish(): ranks, rank-ordered membership masks, lane / target
// masks (warp ballots) and the first pass of the collision sweep of Road.step
// (road/road.py:477-481).  All threads of the env call this convergently.
template <int TPE, bool DENSE>
__device__ __forceinline__ void build_frame(const HwyHighwayParams& P, EnvShared<TPE>& sm, Frame<TPE>& F,
                                            int i, bool active, bool aligned, const VehicleRegs& r,
                                            double dt, bool do_sweep, bool pruned, const Frame<TPE>* prev) {
    const int V = P.n_vehicles;
    const int wie = i >> 5;  // warp within the env (TPE-thread segments)
    const int lane = meta_lane(r.meta), tgt = meta_target(r.meta);
    // -- rank along the road (s, slot) and tie detection.  Float keys first: rounding to float
    // is monotone, so fu < fi implies su < si; only equal float keys need the doubles.
    int rank = 0;
    // The order along the road rarely changes within one substep: with the previous frame of the same launch at hand
    // (`prev`, uniform), every warp checks the whole chain key[perm[k-1]] < key[perm[k]] under the previous permutation
    // of each env segment it holds, one with TPE-thread segments (V - 1 float comparisons spread over its 32 lanes, no
    // communication between the warps: each warp of an env reaches the same verdict).  A strictly increasing chain of
    // float keys is a strictly increasing chain of the doubles they were rounded from, so the ranks are the previous
    // ones and there is neither a tie nor an ambiguity — the O(V) scan per thread (14 % of the kernel's instructions
    // at V = 51) runs only when some pair swapped or drew level.
    bool reuse = false;
    if (prev && !DENSE) {
        bool ok = true;
#pragma unroll 1
        for (int k = (i & 31) + 1; k < V; k += 32) ok = ok && (F.lsf[prev->perm[k - 1]] < F.lsf[prev->perm[k]]);
        reuse = __all_sync(0xffffffffu, ok);
    } else if (prev) {
        int mine, s = 0;
#pragma unroll 1
        for (uint32_t lead = segment_leads(i, active, mine); lead; lead &= lead - 1, ++s) {
            // env of segment s: the envs of a block are consecutive EnvShared records
            const ptrdiff_t d = (ptrdiff_t)(s - mine) * (ptrdiff_t)sizeof(EnvShared<TPE>);
            const Frame<TPE>& Fs = *reinterpret_cast<const Frame<TPE>*>(reinterpret_cast<const char*>(&F) + d);
            const Frame<TPE>& Ps = *reinterpret_cast<const Frame<TPE>*>(reinterpret_cast<const char*>(prev) + d);
            bool ok = true;
#pragma unroll 1
            for (int k = lane_id() + 1; k < V; k += 32)
                ok = ok && (Fs.lsf[Ps.perm[k - 1]] < Fs.lsf[Ps.perm[k]]);
            ok = __all_sync(0xffffffffu, ok);
            if (s == mine) reuse = ok;
        }
    }
    bool tie = false;
    if constexpr (!DENSE) {
        if (reuse) {
            rank = active ? prev->rank[i] : 0;
        } else {
            // (the repair pays for itself only where the count is long, so only the 128-slot kernel uses it)
            int rt = (TPE >= 128 && prev) ? rank_repair<TPE, DENSE>(F, *prev, V, i, active) : -1;
            if (rt < 0) rt = rank_count(F, V, i, active);  // first frame of a launch, ties, or more than isolated swaps
            rank = rt & 0xff;
            tie = (rt >> 8) != 0;
        }
    } else {
        // the verdict differs between the segments of a warp, and the repair is warp-wide
        int rt = -1;
        if (TPE >= 128 && prev && __any_sync(0xffffffffu, !reuse)) rt = rank_repair<TPE, DENSE>(F, *prev, V, i, active);
        if (reuse) {
            rank = active ? prev->rank[i] : 0;
        } else if (active) {
            if (rt < 0) rt = rank_count(F, V, i, active);
            rank = rt & 0xff;
            tie = (rt >> 8) != 0;
        }
    }
    if (active) {
        F.perm[rank] = (unsigned char)i;
        F.rank[i] = (unsigned char)rank;
        if (tie || !aligned) F.slow = 1;
#pragma unroll 1
        for (int l = 0; l < P.lanes_count; ++l) {
            double s_l, lat_l;
            lane_local(P.lanes[l], r.x, r.y, s_l, lat_l);
            if (lane_on(P.lanes[l], s_l, lat_l, 1.0)) atomicOr(&F.smask[l][rank >> 5], 1u << (rank & 31));
        }
    }
    // -- slot-ordered masks by ballot
    const bool is_idm = meta_kind(r.meta) == HWY_KIND_IDM;
#pragma unroll 1
    for (int l = 0; l < P.lanes_count; ++l) {
        uint32_t b_lane = __ballot_sync(0xffffffffu, active && lane == l);
        uint32_t b_tgt = __ballot_sync(0xffffffffu, active && tgt == l);
        if constexpr (DENSE) {
            segment_or(F.lane_is[l], b_lane, i, V);
            segment_or(F.tm[l], b_tgt, i, V);
        } else if ((i & 31) == 0) {
            F.lane_is[l][wie] = b_lane;
            F.tm[l][wie] = b_tgt;
        }
    }
    // superset of the vehicles whose MOBIL decision may fire in the coming act (the crashed
    // flag may still be stale here; crashed vehicles never fire, so this only over-approximates)
    uint32_t b_fired = __ballot_sync(0xffffffffu, active && is_idm && lane == tgt && P.lane_change_delay < r.timer);
    if constexpr (DENSE)
        segment_or(F.fired, b_fired, i, V);
    else if ((i & 31) == 0)
        F.fired[wie] = b_fired;

    // -- collision sweep, pass 1: every gated pair once.  A pair with exactly one
    // check_collisions side is taken by the other side's thread (so the controlled vehicle's
    // pairs are spread over the block); pairs of two checking vehicles are dealt round-robin.
    if (do_sweep && pruned) {
        // many checking vehicles (highway-v0: all of them): the sweep runs after the next barrier over the
        // rank-neighbours only (sweep_pruned); here just the env's speed bound.  Non-negative floats order
        // like their bit patterns.  DENSE: the reduction runs over the lanes of the caller's env segment in this warp.
        if constexpr (DENSE) {
            if (active) {
                const int lane = lane_id(), lo = max(lane - i, 0), hi = min(lane - i + V, 32);
                const unsigned vb = __reduce_max_sync((0xffffffffu >> (32 - (hi - lo))) << lo,
                                                      __float_as_uint(fmaxf(__double2float_ru(r.speed), 0.0f)));
                if (lane == lo) atomicMax(&F.vmax_bits, vb);
            }
        } else {
            unsigned vb = __float_as_uint(active ? fmaxf(__double2float_ru(r.speed), 0.0f) : 0.0f);
            vb = __reduce_max_sync(0xffffffffu, vb);
            if ((i & 31) == 0) atomicMax(&F.vmax_bits, vb);
        }
    } else if (active && do_sweep) {
        const bool cc_i = test_bit(sm.cc, i);
        auto do_pair = [&](int a, int b) {
            if (!pair_precheck(F, a, b, dt)) return;
            bool inter, will;
            double trx, try_;
            pair_sat(F, a, b, dt, inter, will, trx, try_);
            if (will) {
                atomicMax(&sm.last_will[a], b);
                atomicMax(&sm.last_will[b], a);
            }
            if (inter) sm.crash_hit[a] = sm.crash_hit[b] = 1;
        };
        // partners = vehicles that check collisions; a pair of two checking vehicles is dealt
        // round-robin (thread i takes j = i+k mod V, k <= V/2), a pair with one checking side is
        // taken by the other side's thread.
#pragma unroll
        for (int w = 0; w < TPE / 32; ++w) {
            uint32_t m = sm.cc[w];
            if (w == (i >> 5)) m &= ~(1u << (i & 31));
            while (m) {
                int j = w * 32 + __ffs(m) - 1;
                m &= m - 1;
                if (cc_i) {
                    int k = j - i;
                    if (k < 0) k += V;
                    if (2 * k > V || (2 * k == V && i > j)) continue;
                }
                do_pair(i < j ? i : j, i < j ? j : i);
            }
        }
    }
}

// Collision sweep, pass 1, rank-pruned form (after the barrier that follows build_frame).  The frame holds every
// vehicle's rank along the road (s = projection on lane 0's unit direction, ties broken by slot), and
// |s_b - s_a| <= ||p_b - p_a||, so a pair whose s-gap exceeds the largest possible reject threshold
// diag + max(v) dt of vehicle/objects.py:122-138 fails that sphere pre-check too: scanning the rank-neighbours
// upwards until the gap exceeds the bound visits exactly the pairs the all-pairs sweep can accept (plus a few it
// rejects itself).  Every unordered pair is met once, from its lower-ranked member.
template <int TPE>
__device__ __forceinline__ void sweep_pruned(EnvShared<TPE>& sm, const Frame<TPE>& F, int V, int i, bool active,
                                             double dt) {
    if (!active) return;
    const double diag = sqrt(kVehLength * kVehLength + kVehWidth * kVehWidth);
    const double bound = diag + (double)__uint_as_float(F.vmax_bits) * dt + 1e-6;  // >= thr of any pair, + rounding of s
    const bool cc_i = test_bit(sm.cc, i);
    const double si = F.ls[i];
    for (int q = F.rank[i] + 1; q < V; ++q) {
        const int j = F.perm[q];
        if (F.ls[j] - si > bound) break;
        if (!(cc_i || test_bit(sm.cc, j))) continue;  // handle_collisions' gate (objects.py:99-100)
        const int a = i < j ? i : j, b = i < j ? j : i;
        if (!pair_precheck(F, a, b, dt)) continue;
        bool inter, will;
        double trx, try_;
        pair_sat(F, a, b, dt, inter, will, trx, try_);
        if (will) {
            atomicMax(&sm.last_will[a], b);
            atomicMax(&sm.last_will[b], a);
        }
        if (inter) sm.crash_hit[a] = sm.crash_hit[b] = 1;
    }
}

// Collision sweep, pass 2 (own slot): `crashed` is an OR over the intersecting partners, the
// impact is the one of the LAST writer in the reference's (i < j) double loop = the largest
// partner index with will_intersect (vehicle/objects.py:103-116).  SAT is recomputed for that
// one pair (deterministic, rare).
template <int TPE>
__device__ __forceinline__ void apply_collisions(EnvShared<TPE>& sm, const Frame<TPE>& F, int i,
                                                 VehicleRegs& r, double dt) {
    if (sm.crash_hit[i]) {
        r.meta |= HWY_META_CRASHED;
        sm.crash_hit[i] = 0;
    }
    int j = sm.last_will[i];
    if (j >= 0) {
        int a = i < j ? i : j, b = i < j ? j : i;
        bool inter, will;
        double trx, try_;
        pair_sat(F, a, b, dt, inter, will, trx, try_);
        r.imp_x = i == a ? trx / 2 : -trx / 2;
        r.imp_y = i == a ? try_ / 2 : -try_ / 2;
        r.meta |= HWY_META_HAS_IMPACT;
        sm.last_will[i] = -1;
    }
}

// ------------------------------------------------------------------ fused autoreset
// PCG64 jump table: state_n = A^n * state_0 + G_n * inc (mod 2^128), G_n = sum_{j<n} A^j, so a
// thread can enter the env's numpy stream at any output index with two 128-bit multiplies.
constexpr int kPcgJumpN = 4 * HWY_MAX_VEHICLES + 8;
__device__ uint64_t g_pcg_jump[kPcgJumpN][4];  // A^n hi, lo, G_n hi, lo

struct U128 {
    uint64_t hi, lo;
};
__device__ __forceinline__ U128 mul128(U128 a, U128 b) {
    U128 r;
    r.lo = a.lo * b.lo;
    r.hi = __umul64hi(a.lo, b.lo) + a.hi * b.lo + a.lo * b.hi;
    return r;
}
__device__ __forceinline__ U128 add128(U128 a, U128 b) {
    U128 r;
    r.lo = a.lo + b.lo;
    r.hi = a.hi + b.hi + (r.lo < a.lo ? 1 : 0);
    return r;
}
// generator positioned so that its next next64() returns output number n of the stream `g0`
__device__ __forceinline__ Pcg64 pcg_at(const Pcg64& g0, int n) {
    U128 an = {g_pcg_jump[n][0], g_pcg_jump[n][1]}, gn = {g_pcg_jump[n][2], g_pcg_jump[n][3]};
    U128 st = add128(mul128(an, U128{g0.s_hi, g0.s_lo}), mul128(gn, U128{g0.i_hi, g0.i_lo}));
    Pcg64 g = g0;
    g.s_hi = st.hi;
    g.s_lo = st.lo;
    g.has32 = 0;
    g.u32 = 0;
    return g;
}
// the same for any n >= 0: jumps of at most kPcgJumpN - 1 outputs (the linear traffic's spawn reaches ~1 100)
__device__ __forceinline__ Pcg64 pcg_at_far(const Pcg64& g0, int n) {
    Pcg64 g = g0;
    while (n >= kPcgJumpN) {
        g = pcg_at(g, kPcgJumpN - 1);
        n -= kPcgJumpN - 1;
    }
    return pcg_at(g, n);
}

// LinearVehicle.randomize_behavior (behavior.py:406-415) before the inherited DELTA draw: uniform(size=3), then
// uniform(size=2) — each element 0.0 + 1.0 * next_double — mapped by RANGE[0] + u * (RANGE[1] - RANGE[0]).
__device__ __forceinline__ void draw_linear_params(Pcg64& g, const HwyLinearTraffic& T, double (&p)[HWY_LINEAR_PARAMS]) {
    for (int k = 0; k < 3; ++k) p[k] = T.acc_lo[k] + g.next_double() * T.acc_span[k];
    for (int k = 0; k < 2; ++k) p[3 + k] = T.steer_lo[k] + g.next_double() * T.steer_span[k];
}

// HighwayEnv._create_vehicles (envs/highway_env.py:72-98,177-182) for one env inside the step
// kernel, one vehicle per thread.  Vehicle.create_random (vehicle/kinematics.py:50-104) draws,
// per vehicle and in list order, [choice(lanes): one 32-bit word][uniform: 64 bit] for the ego
// and [32][64 speed][64 position][64 DELTA] for traffic; numpy serves 32-bit words as the low
// then the buffered high half of one 64-bit output.  Absent a Lemire rejection (p = 2^-32 per
// draw) every vehicle's position in the stream is therefore known in closed form; the only
// sequential part is the running sum of the longitudinal positions (kept sequential so it
// rounds like the reference).  Rejections, or lanes that are not the x-aligned highway, fall
// back to the serial draw order on one thread.  All threads of the BLOCK must call this
// (barriers); only envs with do_reset do work.  On return r/speed_index hold the new state.
// LINEAR: LinearVehicle traffic draws its 5 parameters between the position and DELTA (8 outputs per
// vehicle instead of 3) and stores them in T->params.
template <int TPE, bool LINEAR = false>
__device__ __forceinline__ void spawn_fused(const HwyHighwayParams& P, const HwyHighwayState& S,
                                            EnvShared<TPE>& sm, int e, int i, bool active,
                                            bool do_reset, bool simple_geometry, VehicleRegs& r,
                                            int& speed_index, const HwyLinearTraffic* T = nullptr) {
    const int V = P.n_vehicles, L = P.lanes_count;
    const size_t n = (size_t)S.n_envs;
    constexpr int kPer = LINEAR ? 3 + HWY_LINEAR_PARAMS : 3;  // 64-bit outputs per traffic vehicle
    auto jump = [](const Pcg64& g, int k) { return LINEAR ? pcg_at_far(g, k) : pcg_at(g, k); };
    Pcg64 g0;
    double speed = 0.0, delta = 4.0, incr = 0.0;
    double lin[HWY_LINEAR_PARAMS] = {0.0, 0.0, 0.0, 0.0, 0.0};
    int lane_id = 0;
    if (do_reset) {
        g0.s_hi = S.rng[0 * n + e];
        g0.s_lo = S.rng[1 * n + e];
        g0.i_hi = S.rng[2 * n + e];
        g0.i_lo = S.rng[3 * n + e];
        uint64_t w4 = S.rng[4 * n + e];
        g0.has32 = (uint32_t)(w4 >> 32);
        g0.u32 = (uint32_t)w4;
    }
    const int h0 = do_reset ? (int)g0.has32 : 0;
    const int n32 = L > 1 ? 1 : 0;                            // choice(1) draws nothing
    const int ego32 = (n32 && P.initial_lane_id < 0) ? 1 : 0;
    auto q_before = [&](int k) { return k == 0 ? 0 : ego32 + (k - 1) * n32; };       // 32-bit requests before k
    auto n64_before = [&](int k) { return k == 0 ? 0 : 1 + kPer * (k - 1); };         // 64-bit outputs before k
    auto fresh_before = [&](int q) { return h0 == 0 ? (q + 1) / 2 : q / 2; };         // outputs used by requests < q
    auto base_of = [&](int k) { return fresh_before(q_before(k)) + n64_before(k); };  // outputs before vehicle k
    if (do_reset && active && simple_geometry) {
        const int k = i;
        const bool has32 = k == 0 ? ego32 : n32;
        Pcg64 g = jump(g0, base_of(k));
        uint32_t r32 = 0;
        if (has32) {
            const int rq = q_before(k);
            if (((h0 + rq) & 1) == 0) {
                r32 = (uint32_t)g.next64();  // fresh output: low half (the high half stays buffered)
            } else if (rq == 0) {
                r32 = g0.u32;                // the half buffered before this reset
            } else {
                // high half of the output the previous requester opened: vehicle k-1
                Pcg64 gp = jump(g0, base_of(k - 1));
                r32 = (uint32_t)(gp.next64() >> 32);
            }
            // Lemire (random_bounded_uint64, rng = L-1): rejection => serial fallback
            uint64_t m = (uint64_t)r32 * (uint32_t)L;
            uint32_t leftover = (uint32_t)m;
            if (leftover < (uint32_t)L && leftover < (0xffffffffu - (uint32_t)(L - 1)) % (uint32_t)L)
                sm.sp_fallback = 1;
            lane_id = (int)(m >> 32);
        }
        if (k == 0 && P.initial_lane_id >= 0) lane_id = P.initial_lane_id;
        const HwyStraightLane& Ln = P.lanes[lane_id];
        const bool is_ego = k == 0;
        speed = is_ego ? P.ego_speed : g.uniform(0.7 * Ln.speed_limit, 0.8 * Ln.speed_limit);
        double spacing = is_ego ? P.ego_spacing : 1 / P.vehicles_density;
        double default_spacing = 12 + 1.0 * speed;
        double offset = spacing * default_spacing * P.spawn_exp;
        incr = offset * g.uniform(0.9, 1.1);
        if constexpr (LINEAR) {
            if (!is_ego) draw_linear_params(g, *T, lin);
        }
        if (!is_ego) delta = g.uniform(P.delta_lo, P.delta_hi);
        sm.sp_x[k] = is_ego ? 3 * offset + incr : incr;  // x0 = 3 * offset; x0 += offset * U
    }
    env_sync<TPE>();
    if (do_reset && i == 0) {
        if (simple_geometry && !sm.sp_fallback) {
            // x_k = max_j<k s_j + incr_k; positions increase strictly, so the max is x_{k-1}
            double x = sm.sp_x[0];
            for (int k = 1; k < V; ++k) {
                x = x + sm.sp_x[k];
                sm.sp_x[k] = x;
            }
            // stream position after the reset
            const int Q = ego32 + (V - 1) * n32;
            Pcg64 ge = jump(g0, fresh_before(Q) + n64_before(V));
            uint32_t has_f = (uint32_t)((h0 + Q) & 1), u_f = g0.u32;
            if (Q > 0) {
                int rf = Q - 1;  // last fresh request
                if (((h0 + rf) & 1) != 0) rf -= 1;
                if (rf >= 0) {
                    int kf = ego32 ? rf : rf + 1;  // vehicle issuing request rf
                    Pcg64 gp = jump(g0, base_of(kf));
                    u_f = (uint32_t)(gp.next64() >> 32);
                }
            }
            S.rng[0 * n + e] = ge.s_hi;
            S.rng[1 * n + e] = ge.s_lo;
            S.rng[4 * n + e] = ((uint64_t)has_f << 32) | u_f;
        }
    }
    env_sync<TPE>();
    const bool fallback = do_reset && (!simple_geometry || sm.sp_fallback);
    if (fallback && i == 0) {
        // serial draw order, results staged through HBM (rare path)
        Pcg64 g = g0;
        double2* pos = reinterpret_cast<double2*>(S.pos);
        double2* hs = reinterpret_cast<double2*>(S.hs);
        const size_t base = (size_t)e * S.vp;
        for (int v = 0; v < V; ++v) {
            const bool is_ego = v == 0;
            int id = (is_ego && P.initial_lane_id >= 0) ? P.initial_lane_id : g.choice(L);
            const HwyStraightLane& Lv = P.lanes[id];
            double sp = is_ego ? P.ego_speed : g.uniform(0.7 * Lv.speed_limit, 0.8 * Lv.speed_limit);
            double spacing = is_ego ? P.ego_spacing : 1 / P.vehicles_density;
            double offset = spacing * (12 + 1.0 * sp) * P.spawn_exp;
            double x0;
            if (v > 0) {
                x0 = lane_s(Lv, pos[base].x, pos[base].y);
                for (int j = 1; j < v; ++j) x0 = fmax(x0, lane_s(Lv, pos[base + j].x, pos[base + j].y));
            } else {
                x0 = 3 * offset;
            }
            x0 += offset * g.uniform(0.9, 1.1);
            double px = (Lv.start_x + x0 * Lv.dir_x) + 0.0 * Lv.lat_x;
            double py = (Lv.start_y + x0 * Lv.dir_y) + 0.0 * Lv.lat_y;
            pos[base + v] = make_double2(px, py);
            hs[base + v] = make_double2(Lv.heading, sp);
            if constexpr (LINEAR) {
                double p[HWY_LINEAR_PARAMS] = {0.0, 0.0, 0.0, 0.0, 0.0};
                if (!is_ego) draw_linear_params(g, *T, p);
                for (int k = 0; k < HWY_LINEAR_PARAMS; ++k) T->params[(base + v) * HWY_LINEAR_PARAMS + k] = p[k];
            }
            S.delta[base + v] = is_ego ? 4.0 : g.uniform(P.delta_lo, P.delta_hi);
        }
        S.rng[0 * n + e] = g.s_hi;
        S.rng[1 * n + e] = g.s_lo;
        S.rng[4 * n + e] = ((uint64_t)g.has32 << 32) | g.u32;
        __threadfence_block();
    }
    env_sync<TPE>();
    if (do_reset && active) {
        const bool is_ego = i == 0;
        double px, py, heading;
        if (fallback) {
            const size_t slot = (size_t)e * S.vp + i;  // staged by thread 0 before the barrier
            px = S.pos[2 * slot];
            py = S.pos[2 * slot + 1];
            heading = S.hs[2 * slot];
            speed = S.hs[2 * slot + 1];
            delta = S.delta[slot];
        } else {
            const HwyStraightLane& Ln = P.lanes[lane_id];
            double x0 = sm.sp_x[i];
            px = (Ln.start_x + x0 * Ln.dir_x) + 0.0 * Ln.lat_x;  // lane.position(x0, 0)
            py = (Ln.start_y + x0 * Ln.dir_y) + 0.0 * Ln.lat_y;
            heading = Ln.heading;
            if constexpr (LINEAR) {  // (the serial path stored them itself)
                const size_t slot = (size_t)e * S.vp + i;
                for (int k = 0; k < HWY_LINEAR_PARAMS; ++k) T->params[slot * HWY_LINEAR_PARAMS + k] = lin[k];
            }
        }
        int lane = closest_lane(P, px, py, heading);  // RoadObject.__init__ objects.py:46-50
        double target_speed = speed;                   // `target_speed or self.speed`
        double timer = 0.0;
        int kind, cc;
        if (is_ego) {
            cc = 1;
            delta = 4.0;
            if (P.action_type == 0) {
                kind = HWY_KIND_MDP;
                speed_index = speed_to_index(P, target_speed);
                target_speed = P.target_speeds[speed_index];
            } else {
                kind = HWY_KIND_VEHICLE;
                speed_index = -1;
            }
        } else {
            kind = HWY_KIND_IDM;
            cc = P.others_check_collisions;
            timer = py_mod_pos((px + py) * kPi, P.lane_change_delay);  // behavior.py:64
        }
        r.x = px;
        r.y = py;
        r.heading = heading;
        r.speed = speed;
        r.target_speed = target_speed;
        r.timer = timer;
        r.delta = delta;
        r.imp_x = r.imp_y = 0.0;
        r.meta = (lane << HWY_META_LANE_SHIFT) | (lane << HWY_META_TARGET_SHIFT) |
                 (cc ? HWY_META_CHECK_COLLISIONS : 0) | (kind << HWY_META_KIND_SHIFT) | HWY_META_PRESENT;
    }
}

// ------------------------------------------------------------------ the step kernel
constexpr int kMaxBlockThreads = 512;  // 128 registers/thread => one full register file
// Register budget of the step kernel = 65536 / (HWY_STEP_BOUND_THREADS * HWY_STEP_BOUND_BLOCKS); the launcher never
// uses more than HWY_STEP_BOUND_THREADS threads per block.  (512, 1): 128 registers, two 256-thread blocks per SM.
#ifndef HWY_STEP_BOUND_THREADS
#define HWY_STEP_BOUND_THREADS 512
#endif
#ifndef HWY_STEP_BOUND_BLOCKS
#define HWY_STEP_BOUND_BLOCKS 1
#endif

// blockDim.x = TPE * (envs per block); dynamic shared memory = envs per block * sizeof(EnvShared).
// DENSE (see launch_step): `dense_epb` envs per block, env `sub` on the V threads from sub * V, vehicle
// i = threadIdx.x - sub * V; blockDim.x = dense_epb * V rounded up to whole warps, and the threads past dense_epb * V
// own no vehicle: they meet every barrier and warp collective and do nothing else.
// AL (host-checked, lanes_congruent): every lane is a copy of lane 0 shifted sideways — what
// RoadNetwork.straight_road_network builds (road/road.py:291-321) — so the general-geometry branches (per-lane
// projections in lane_distance / closest_lane, F.slow for unaligned lanes) are compiled out.  The per-substep loop
// of this kernel is about as large as the SM's instruction cache, so code bytes on the hot path are a first-order
// cost.
//
// The kernel body (hwy_highway_step.cuh) is compiled twice: highway_step_kernel (IDMVehicle traffic, LINEAR = false)
// and highway_linear_step_kernel (LinearVehicle traffic, LINEAR = true, `T` its parameters; the block's LinearShared
// staging follows its EnvShared array in dynamic shared memory).  Only `if constexpr (LINEAR)` branches differ, and
// each kernel keeps the body in its own scope (an inlined device function changes the IDM kernel's code schedule).
template <int TPE, bool AL, bool DENSE>
__global__ void __launch_bounds__(HWY_STEP_BOUND_THREADS, HWY_STEP_BOUND_BLOCKS)
highway_step_kernel(const __grid_constant__ HwyHighwayParams P, const HwyHighwayState S,
                    const int32_t* __restrict__ action_i, const float* __restrict__ action_f,
                    float* __restrict__ obs, double* __restrict__ reward,
                    uint8_t* __restrict__ terminated, uint8_t* __restrict__ truncated,
                    double* __restrict__ info_speed, uint8_t* __restrict__ info_crashed,
                    const int autoreset, float* __restrict__ final_obs, const int dense_epb) {
    constexpr bool LINEAR = false;
    const HwyLinearTraffic* T = nullptr;
#include "hwy_highway_step.cuh"
}

// LinearVehicle / AggressiveVehicle / DefensiveVehicle traffic (vehicle/behavior.py:350-583)
template <int TPE, bool AL, bool DENSE>
__global__ void __launch_bounds__(HWY_STEP_BOUND_THREADS, HWY_STEP_BOUND_BLOCKS)
highway_linear_step_kernel(const __grid_constant__ HwyHighwayParams P, const HwyHighwayState S,
                           const __grid_constant__ HwyLinearTraffic T_, const int32_t* __restrict__ action_i,
                           const float* __restrict__ action_f, float* __restrict__ obs, double* __restrict__ reward,
                           uint8_t* __restrict__ terminated, uint8_t* __restrict__ truncated,
                           double* __restrict__ info_speed, uint8_t* __restrict__ info_crashed,
                           const int autoreset, float* __restrict__ final_obs, const int dense_epb) {
    constexpr bool LINEAR = true;
    const HwyLinearTraffic* T = &T_;
#include "hwy_highway_step.cuh"
}

// ------------------------------------------------------------------ observe-only kernel
template <int TPE>
struct ObsShared {
    Frame<TPE> f;
    double key[TPE];
};

template <int TPE>
__global__ void __launch_bounds__(TPE == 32 ? 128 : TPE)
highway_observe_kernel(const __grid_constant__ HwyHighwayParams P, const HwyHighwayState S,
                       const uint8_t* __restrict__ mask_a, const uint8_t* __restrict__ mask_b,
                       float* __restrict__ obs) {
    constexpr int EPB = TPE == 32 ? 4 : 1;
    __shared__ ObsShared<TPE> smem[EPB];
    const int sub = threadIdx.x / TPE, i = threadIdx.x % TPE;
    const int env = blockIdx.x * EPB + sub;
    const bool env_ok = env < S.n_envs;
    const int e = env_ok ? env : S.n_envs - 1;
    ObsShared<TPE>& sm = smem[sub];
    const bool active = i < P.n_vehicles;
    VehicleRegs r;
    load_vehicle(S, (size_t)e * S.vp + (active ? i : 0), r);
    publish(P, sm.f, i, active, r);
    env_sync<TPE>();
    const bool wanted = env_ok && env_selected(mask_a, mask_b, e);
    kinematics_observe(P, sm.f, sm.key, i, r.heading,
                       wanted ? obs + (size_t)e * P.obs_vehicles_count * obs_columns(P) : nullptr);
}

// ------------------------------------------------------------------ reset kernel
// HighwayEnv._create_road/_create_vehicles (envs/highway_env.py:55-98,177-182) with
// Vehicle.create_random (vehicle/kinematics.py:50-104), IDMVehicle.__init__ timer and
// randomize_behavior (behavior.py:64-69), MDPVehicle.__init__ (controller.py:284-293).
// The spawn is a sequential chain on the env's PCG64 stream => one thread per env.
// LINEAR: LinearVehicle.randomize_behavior (behavior.py:406-415) draws the traffic's parameters into T->params.
__global__ void __launch_bounds__(128)
highway_reset_kernel(const __grid_constant__ HwyHighwayParams P, const HwyHighwayState S,
                     const uint8_t* __restrict__ mask_a, const uint8_t* __restrict__ mask_b) {
    constexpr bool LINEAR = false;
    const HwyLinearTraffic* T = nullptr;
#include "hwy_highway_reset.cuh"
}

__global__ void __launch_bounds__(128)
highway_linear_reset_kernel(const __grid_constant__ HwyHighwayParams P, const HwyHighwayState S,
                            const __grid_constant__ HwyLinearTraffic T_, const uint8_t* __restrict__ mask_a,
                            const uint8_t* __restrict__ mask_b) {
    constexpr bool LINEAR = true;
    const HwyLinearTraffic* T = &T_;
#include "hwy_highway_reset.cuh"
}

// ------------------------------------------------------------------ test entries
// The production device functions on one input per thread (hwy_debug_math); the operands of each HWY_MATH_* op
// are listed in include/hwyb200.h.
__host__ __device__ inline int math_in_width(int op) {
    switch (op) {
        case HWY_MATH_DOT2: return 4;
        case HWY_MATH_SPEED_TO_INDEX: return 2 + HWY_MAX_TARGET_SPEEDS;
        case HWY_MATH_IDM_POW: case HWY_MATH_EXP_DLOG: case HWY_MATH_PY_MOD_POS: case HWY_MATH_DIV_FINITE:
        case HWY_MATH_NORM2: return 2;
        default: return 1;
    }
}
__host__ __device__ inline int math_out_width(int op) {
    return op == HWY_MATH_SINCOS || op == HWY_MATH_BETA_CONTROLLED || op == HWY_MATH_BETA_ANGLE ? 2 : 1;
}
__global__ void debug_math_kernel(int op, const double* __restrict__ in, double* __restrict__ out, int n) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const double* a = in + (size_t)k * math_in_width(op);
    double* o = out + (size_t)k * math_out_width(op);
    switch (op) {
        case HWY_MATH_SINCOS: m_sincos(a[0], &o[0], &o[1]); break;
        case HWY_MATH_IDM_POW: o[0] = idm_pow(a[0], a[1]); break;
        case HWY_MATH_EXP_DLOG: o[0] = m_exp_dlog(a[0], a[1]); break;
        case HWY_MATH_PY_MOD_POS: o[0] = py_mod_pos(a[0], a[1]); break;
        case HWY_MATH_WRAP_TO_PI: o[0] = wrap_to_pi(a[0]); break;
        case HWY_MATH_NOT_ZERO: o[0] = not_zero(a[0]); break;
        case HWY_MATH_DIV_FINITE: o[0] = div_finite(a[0], a[1]); break;
        case HWY_MATH_DOT2: o[0] = dot2(a[0], a[1], a[2], a[3]); break;
        case HWY_MATH_NORM2: o[0] = norm2(a[0], a[1]); break;
        case HWY_MATH_BETA_CONTROLLED: beta_of_controlled(a[0], o[0], o[1]); break;
        case HWY_MATH_BETA_ANGLE: beta_of_angle(a[0], o[0], o[1]); break;
        case HWY_MATH_SPEED_TO_INDEX: {
            if (!(a[1] >= 1.0 && a[1] <= (double)HWY_MAX_TARGET_SPEEDS)) {  // outside the table: no index
                o[0] = __longlong_as_double(0x7ff8000000000000LL);
                break;
            }
            HwyHighwayParams P;
            P.n_target_speeds = (int)a[1];
            for (int j = 0; j < HWY_MAX_TARGET_SPEEDS; ++j) P.target_speeds[j] = a[2 + j];
            o[0] = (double)speed_to_index(P, a[0]);
            break;
        }
    }
}

// count draws of one kind from the generator of each thread (words [5][n], the HwyHighwayState.rng layout);
// draws [n][count] (doubles as their bits), for HWY_PCG_NORMAL [n][count][2] = (value bits, 64-bit outputs consumed).
__global__ void debug_pcg64_kernel(int op, int arg_i, double arg_lo, double arg_hi, int count,
                                   const uint64_t* __restrict__ words_in, uint64_t* __restrict__ words_out,
                                   uint64_t* __restrict__ draws, int n) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    Pcg64 g = load_rng(words_in, (size_t)n, e);
    if (op == HWY_PCG_AT) {
        g = pcg_at(g, arg_i);
    } else {
        uint64_t* d = draws + (size_t)e * count * (op == HWY_PCG_NORMAL ? 2 : 1);
        for (int j = 0; j < count; ++j) {
            switch (op) {
                case HWY_PCG_NEXT64: d[j] = g.next64(); break;
                case HWY_PCG_NEXT32: d[j] = g.next32(); break;
                case HWY_PCG_NEXT_DOUBLE: d[j] = (uint64_t)__double_as_longlong(g.next_double()); break;
                case HWY_PCG_UNIFORM: d[j] = (uint64_t)__double_as_longlong(g.uniform(arg_lo, arg_hi)); break;
                case HWY_PCG_CHOICE: d[j] = (uint64_t)g.choice(arg_i); break;
                case HWY_PCG_NORMAL: {
                    const Pcg64 before = g;
                    d[2 * j] = (uint64_t)__double_as_longlong(g.normal());
                    // outputs consumed: the smallest k with before advanced by k == after (0: more than 16)
                    uint64_t used = 0;
                    for (int k = 1; k <= 16 && !used; ++k) {
                        const Pcg64 a = pcg_at(before, k);
                        if (a.s_hi == g.s_hi && a.s_lo == g.s_lo) used = k;
                    }
                    d[2 * j + 1] = used;
                    break;
                }
            }
        }
    }
    store_rng_all(words_out, (size_t)n, e, g);
}

}  // namespace hwy

// ====================================================================== C ABI
// error text / launch counter shared by the translation units of the library (hwy_abi.h)
namespace hwy_abi {
thread_local char g_err[512] = "";
thread_local unsigned long long g_launches = 0;

int fail(const char* fmt, const char* detail) {
    snprintf(g_err, sizeof(g_err), fmt, detail);
    return 1;
}
int check_launch(const char* what) {
    ++g_launches;
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) {
        snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(err));
        return 1;
    }
    return 0;
}
}  // namespace hwy_abi

namespace {
using hwy_abi::check_launch;
using hwy_abi::fail;
using hwy_abi::g_err;
using hwy_abi::g_launches;
int validate(const HwyHighwayParams* p, const HwyHighwayState* s) {
    if (!p || !s) return fail("%s", "null params/state");
    if (p->n_vehicles < 1 || p->n_vehicles > HWY_MAX_VEHICLES) return fail("%s", "n_vehicles out of range");
    if (p->lanes_count < 1 || p->lanes_count > HWY_MAX_LANES) return fail("%s", "lanes_count out of range");
    if (p->obs_vehicles_count < 1 || p->obs_vehicles_count > HWY_MAX_OBS_VEHICLES)
        return fail("%s", "obs_vehicles_count out of range");
    if (p->obs_n_features < 0 || p->obs_n_features > HWY_MAX_OBS_FEATURES)
        return fail("%s", "obs_n_features out of range");
    for (int c = 0; c < p->obs_n_features; ++c)
        if (p->obs_feature[c] < HWY_FEAT_PRESENCE || p->obs_feature[c] > HWY_FEAT_ANG_OFF)
            return fail("%s", "unknown observation feature code");
    if (p->n_target_speeds < 1 || p->n_target_speeds > HWY_MAX_TARGET_SPEEDS)
        return fail("%s", "n_target_speeds out of range");
    if (p->simulation_frequency < 1 || p->policy_frequency < 1 ||
        p->simulation_frequency < p->policy_frequency)
        return fail("%s", "bad simulation/policy frequency");
    if (s->n_envs < 1) return fail("%s", "n_envs < 1");
    if (s->vp < p->n_vehicles || (s->vp & 1)) return fail("%s", "slot stride must be even and >= n_vehicles");
    if (!s->pos || !s->hs || !s->tt || !s->imp || !s->delta || !s->meta || !s->speed_index ||
        !s->time || !s->rng)
        return fail("%s", "null state pointer");
    int dev_count = 0;
    if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count < 1) {
        cudaGetLastError();
        return fail("%s", "no CUDA device: this library has no CPU fallback");
    }
    return 0;
}
int tpe_for(int n_vehicles) { return n_vehicles <= 32 ? 32 : (n_vehicles <= 64 ? 64 : 128); }

struct Grid {
    int blocks, threads;
};
Grid grid_for(int tpe, int n_envs) {
    int epb = tpe == 32 ? 4 : 1;
    return Grid{(n_envs + epb - 1) / epb, tpe * epb};
}

int step_block_thread_limit() {
    return hwy::kMaxBlockThreads < HWY_STEP_BOUND_THREADS ? hwy::kMaxBlockThreads : HWY_STEP_BOUND_THREADS;
}
int step_half_block_threads() { return step_block_thread_limit() / 2; }
// Envs per block of the step kernel: as many V-thread envs as fit half the block-thread limit (two blocks per SM),
// reduced when that leaves the last wave of blocks mostly empty.  HWYB200_EPB overrides, up to the whole limit.  Both
// are also bounded by shared memory (env_bytes per env), which only binds below V = 17.
struct StepDevice {
    int n_sm, smem_sm, smem_block;  // SMs, shared memory per SM, opt-in shared memory per block
};
// read once per device
const StepDevice& step_device(int dev) {
    static StepDevice info[64];
    static std::atomic<bool> ready[64];
    static std::mutex mu;
    if (!ready[dev].load(std::memory_order_acquire)) {
        std::lock_guard<std::mutex> lock(mu);
        if (!ready[dev].load(std::memory_order_relaxed)) {
            StepDevice d{132, 228 * 1024, 227 * 1024};
            cudaDeviceGetAttribute(&d.n_sm, cudaDevAttrMultiProcessorCount, dev);
            cudaDeviceGetAttribute(&d.smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
            cudaDeviceGetAttribute(&d.smem_block, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
            info[dev] = d;
            ready[dev].store(true, std::memory_order_release);
        }
    }
    return info[dev];
}
int step_envs_per_block(int n_vehicles, size_t env_bytes, int n_envs, const StepDevice& d) {
    const int limit = step_block_thread_limit();
    int max_epb = std::min<long>(limit / n_vehicles, d.smem_block / (long)env_bytes);
    if (max_epb < 1) max_epb = 1;
    if (const char* e = getenv("HWYB200_EPB")) {
        int v = atoi(e);
        if (v >= 1 && v <= max_epb) return v;
    }
    // Two resident blocks per SM (rather than one block of max_epb envs or many 1-env blocks): the blocks cover each other's
    // barrier stalls.  Small batches shrink the block so every SM still gets work.
    int epb = std::min<long>(step_half_block_threads() / n_vehicles, (d.smem_sm / 2 - 1024) / (long)env_bytes);
    if (epb < 1) epb = 1;
    while (epb > 1 && (long)n_envs < (long)epb * 2 * d.n_sm) --epb;
    return epb;
}

// One-time (per device) fill of the PCG64 jump table used by the fused autoreset.  The table is computed on
// the host and copied with a synchronous cudaMemcpyToSymbol under a mutex, so it is complete before any kernel
// of any stream that is launched afterwards; hwy_highway_reset calls this too, i.e. the table exists before the
// first step.  A first call from a capturing stream is refused (the copy cannot be captured).
int ensure_pcg_jump(cudaStream_t st) {
    static std::mutex mu;
    static bool ready[64] = {false};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return fail("%s", "cudaGetDevice failed");
    std::lock_guard<std::mutex> lock(mu);
    if (ready[dev]) return 0;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (st && cudaStreamIsCapturing(st, &cap) == cudaSuccess && cap != cudaStreamCaptureStatusNone)
        return fail("%s", "PCG64 jump table not initialised on this device: call hwy_highway_reset (or one eager "
                          "step) before capturing a step into a CUDA graph");
    static uint64_t table[hwy::kPcgJumpN][4];
    typedef unsigned __int128 u128;
    const u128 A = ((u128)0x2360ed051fc65da4ULL << 64) | 0x4385df649fccf645ULL;
    u128 an = 1, gn = 0;
    for (int n = 0; n < hwy::kPcgJumpN; ++n) {
        table[n][0] = (uint64_t)(an >> 64);
        table[n][1] = (uint64_t)an;
        table[n][2] = (uint64_t)(gn >> 64);
        table[n][3] = (uint64_t)gn;
        gn = gn * A + 1;  // G_{n+1} = G_n * A + 1
        an = an * A;
    }
    cudaError_t err = cudaMemcpyToSymbol(hwy::g_pcg_jump, table, sizeof(table));
    if (err != cudaSuccess) return fail("cudaMemcpyToSymbol(g_pcg_jump): %s", cudaGetErrorString(err));
    ready[dev] = true;
    return 0;
}

// host copy of hwy::lanes_congruent (hwy_device.cuh)
bool lanes_congruent_host(const HwyHighwayParams* p) {
    const HwyStraightLane* L = p->lanes;
    bool ok = L[0].dir_y == 0.0;
    for (int l = 1; l < p->lanes_count; ++l)
        ok = ok && L[l].start_x == L[0].start_x && L[l].dir_x == L[0].dir_x && L[l].dir_y == 0.0 &&
             L[l].heading == L[0].heading && L[l].length == L[0].length && L[l].lat_x == L[0].lat_x &&
             L[l].lat_y == L[0].lat_y;
    return ok;
}

template <int TPE, bool AL, bool DENSE>
int launch_step_kernel(const HwyHighwayParams* p, const HwyHighwayState* s, const HwyLinearTraffic* t,
                       const int32_t* action_i, const float* action_f, float* obs, double* reward,
                       uint8_t* terminated, uint8_t* truncated, double* info_speed, uint8_t* info_crashed,
                       int autoreset, float* final_obs, int epb, size_t env_bytes, int dev, cudaStream_t st) {
    const int blocks = (s->n_envs + epb - 1) / epb;
    const size_t smem = (size_t)epb * env_bytes;
    // the attribute is per device (and per template instance): cache it by device ordinal
    static std::atomic<size_t> configured[2][64];
    if (smem > configured[t != nullptr][dev].load(std::memory_order_relaxed)) {
        cudaError_t err = t ? cudaFuncSetAttribute(hwy::highway_linear_step_kernel<TPE, AL, DENSE>,
                                                   cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                            : cudaFuncSetAttribute(hwy::highway_step_kernel<TPE, AL, DENSE>,
                                                   cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (err != cudaSuccess) return fail("cudaFuncSetAttribute: %s", cudaGetErrorString(err));
        configured[t != nullptr][dev].store(smem, std::memory_order_relaxed);
    }
    const int threads = DENSE ? (epb * p->n_vehicles + 31) & ~31 : epb * TPE;
    if (t)
        hwy::highway_linear_step_kernel<TPE, AL, DENSE><<<blocks, threads, smem, st>>>(
            *p, *s, *t, action_i, action_f, obs, reward, terminated, truncated, info_speed, info_crashed,
            autoreset, final_obs, epb);
    else
        hwy::highway_step_kernel<TPE, AL, DENSE><<<blocks, threads, smem, st>>>(
            *p, *s, action_i, action_f, obs, reward, terminated, truncated, info_speed, info_crashed,
            autoreset, final_obs, epb);
    return 0;
}

// t == nullptr: IDMVehicle traffic (highway_step_kernel); else LinearVehicle traffic (highway_linear_step_kernel)
template <int TPE, bool AL>
int launch_step(const HwyHighwayParams* p, const HwyHighwayState* s, const HwyLinearTraffic* t,
                const int32_t* action_i, const float* action_f, float* obs, double* reward, uint8_t* terminated,
                uint8_t* truncated, double* info_speed, uint8_t* info_crashed, int autoreset,
                float* final_obs, cudaStream_t st) {
    if (autoreset > 0 && ensure_pcg_jump(st)) return 1;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return fail("%s", "cudaGetDevice failed");
    const size_t env_bytes = sizeof(hwy::EnvShared<TPE>) + (t ? sizeof(hwy::LinearShared<TPE>) : 0);
    const int epb = step_envs_per_block(p->n_vehicles, env_bytes, s->n_envs, step_device(dev));
    // Dense segments (V threads per env, the DENSE kernels) only where they put more envs into a block than TPE-thread
    // segments; otherwise the TPE-thread kernel runs, which carries none of the segment bookkeeping.
    const bool dense = epb * TPE > step_half_block_threads();
    if (dense)
        return launch_step_kernel<TPE, AL, true>(p, s, t, action_i, action_f, obs, reward, terminated, truncated,
                                                 info_speed, info_crashed, autoreset, final_obs, epb, env_bytes, dev,
                                                 st);
    return launch_step_kernel<TPE, AL, false>(p, s, t, action_i, action_f, obs, reward, terminated, truncated,
                                              info_speed, info_crashed, autoreset, final_obs, epb, env_bytes, dev, st);
}

int launch_observe(const HwyHighwayParams* p, const HwyHighwayState* s, const uint8_t* mask_a,
                   const uint8_t* mask_b, float* obs, cudaStream_t st) {
    int tpe = tpe_for(p->n_vehicles);
    Grid g = grid_for(tpe, s->n_envs);
    if (tpe == 32)
        hwy::highway_observe_kernel<32><<<g.blocks, g.threads, 0, st>>>(*p, *s, mask_a, mask_b, obs);
    else if (tpe == 64)
        hwy::highway_observe_kernel<64><<<g.blocks, g.threads, 0, st>>>(*p, *s, mask_a, mask_b, obs);
    else
        hwy::highway_observe_kernel<128><<<g.blocks, g.threads, 0, st>>>(*p, *s, mask_a, mask_b, obs);
    return check_launch("highway_observe_kernel");
}

int launch_reset(const HwyHighwayParams* p, const HwyHighwayState* s, const uint8_t* mask_a,
                 const uint8_t* mask_b, cudaStream_t st) {
    int blocks = (s->n_envs + 127) / 128;
    hwy::highway_reset_kernel<<<blocks, 128, 0, st>>>(*p, *s, mask_a, mask_b);
    return check_launch("highway_reset_kernel");
}

int launch_linear_reset(const HwyHighwayParams* p, const HwyHighwayState* s, const HwyLinearTraffic* t,
                        const uint8_t* mask_a, const uint8_t* mask_b, cudaStream_t st) {
    int blocks = (s->n_envs + 127) / 128;
    hwy::highway_linear_reset_kernel<<<blocks, 128, 0, st>>>(*p, *s, *t, mask_a, mask_b);
    return check_launch("highway_linear_reset_kernel");
}

int validate_linear(const HwyLinearTraffic* t) {
    if (!t || !t->params) return fail("%s", "null linear traffic parameters");
    return 0;
}
}  // namespace

namespace {
int dispatch_step(const HwyHighwayParams* p, const HwyHighwayState* s, const HwyLinearTraffic* t,
                  const int32_t* action_i, const float* action_f, float* obs, double* reward, uint8_t* terminated,
                  uint8_t* truncated, double* info_speed, uint8_t* info_crashed, int autoreset, float* final_obs,
                  cudaStream_t st);
int check_step_args(const HwyHighwayParams* p, const HwyHighwayState* s, const int32_t* action_i,
                    const float* action_f, float* obs, double* reward, uint8_t* terminated, uint8_t* truncated,
                    int autoreset);
}

extern "C" {

int hwy_abi_version(void) { return HWY_ABI_VERSION; }
const char* hwy_last_error(void) { return g_err; }
uint64_t hwy_launch_count(void) { return g_launches; }
int hwy_highway_slot_stride(int n_vehicles) { return (n_vehicles + 1) & ~1; }

int hwy_highway_observe(const HwyHighwayParams* p, const HwyHighwayState* s, float* obs, void* stream) {
    if (validate(p, s)) return 1;
    if (!obs) return fail("%s", "obs is null");
    return launch_observe(p, s, nullptr, nullptr, obs, (cudaStream_t)stream);
}

int hwy_highway_reset(const HwyHighwayParams* p, const HwyHighwayState* s, const uint8_t* mask,
                      float* obs, void* stream) {
    if (validate(p, s)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    if (ensure_pcg_jump(st)) return 1;  // the fused autoreset of later steps reads the table
    if (launch_reset(p, s, mask, nullptr, st)) return 1;
    if (obs) return launch_observe(p, s, mask, nullptr, obs, st);
    return 0;
}

// debug: read and clear the per-phase cycle counters (all zero unless built with HWY_PHASE_TIMING)
int hwy_debug_phase_cycles(unsigned long long* out16) {
#ifdef HWY_PHASE_TIMING
    unsigned long long zero[16] = {0};
    if (cudaMemcpyFromSymbol(out16, hwy::g_phase_cycles, sizeof(zero)) != cudaSuccess) return 1;
    if (cudaMemcpyToSymbol(hwy::g_phase_cycles, zero, sizeof(zero)) != cudaSuccess) return 1;
    return 0;
#else
    for (int k = 0; k < 16; ++k) out16[k] = 0;
    return 0;
#endif
}

int hwy_debug_math(int op, const double* in, double* out, int n, void* stream) {
    if (op < HWY_MATH_SINCOS || op > HWY_MATH_SPEED_TO_INDEX) return fail("%s", "hwy_debug_math: unknown op");
    if (n < 0) return fail("%s", "hwy_debug_math: n < 0");
    if (!in || !out) return fail("%s", "hwy_debug_math: null pointer");
    if (n == 0) return 0;
    hwy::debug_math_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(op, in, out, n);
    return check_launch("debug_math_kernel");
}

int hwy_debug_pcg64(int op, int arg_i, double arg_lo, double arg_hi, int count, const uint64_t* words_in,
                    uint64_t* words_out, uint64_t* draws, int n, void* stream) {
    if (op < HWY_PCG_NEXT64 || op > HWY_PCG_AT) return fail("%s", "hwy_debug_pcg64: unknown op");
    if (n < 0) return fail("%s", "hwy_debug_pcg64: n < 0");
    if (op == HWY_PCG_CHOICE && arg_i < 1) return fail("%s", "hwy_debug_pcg64: choice needs arg_i >= 1");
    if (op == HWY_PCG_AT && (arg_i < 0 || arg_i >= hwy::kPcgJumpN))
        return fail("%s", "hwy_debug_pcg64: pcg_at index outside the jump table");
    if (op != HWY_PCG_AT && (count < 0 || count > (1 << 20))) return fail("%s", "hwy_debug_pcg64: count outside 0..2^20");
    if (!words_in || !words_out || (op != HWY_PCG_AT && count > 0 && !draws))
        return fail("%s", "hwy_debug_pcg64: null pointer");
    if (n == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    if ((op == HWY_PCG_AT || op == HWY_PCG_NORMAL) && ensure_pcg_jump(st)) return 1;
    hwy::debug_pcg64_kernel<<<(n + 127) / 128, 128, 0, st>>>(op, arg_i, arg_lo, arg_hi, op == HWY_PCG_AT ? 0 : count,
                                                              words_in, words_out, draws, n);
    return check_launch("debug_pcg64_kernel");
}

int hwy_highway_autoreset(const HwyHighwayParams* p, const HwyHighwayState* s,
                          const uint8_t* terminated, const uint8_t* truncated, float* obs,
                          void* stream) {
    if (validate(p, s)) return 1;
    if (!terminated || !truncated || !obs) return fail("%s", "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (launch_reset(p, s, terminated, truncated, st)) return 1;
    return launch_observe(p, s, terminated, truncated, obs, st);
}

int hwy_highway_step(const HwyHighwayParams* p, const HwyHighwayState* s, const int32_t* action_i,
                     const float* action_f, float* obs, double* reward, uint8_t* terminated,
                     uint8_t* truncated, double* info_speed, uint8_t* info_crashed, int autoreset,
                     float* final_obs, void* stream) {
    if (check_step_args(p, s, action_i, action_f, obs, reward, terminated, truncated, autoreset)) return 1;
    return dispatch_step(p, s, nullptr, action_i, action_f, obs, reward, terminated, truncated, info_speed, info_crashed,
                         autoreset, final_obs, (cudaStream_t)stream);
}

/* B4 seam of the reference (abstract.py:304-307 minus action_type.act): n_substeps x (Road.act(); Road.step(dt)). */
int hwy_highway_substeps(const HwyHighwayParams* p, const HwyHighwayState* s, int n_substeps, const float* action_f,
                         void* stream) {
    if (validate(p, s)) return 1;
    if (n_substeps < 1 || n_substeps > 4096) return fail("%s", "n_substeps must be in 1..4096");
    return dispatch_step(p, s, nullptr, nullptr, action_f, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                         -n_substeps, nullptr, (cudaStream_t)stream);
}

// ---- LinearVehicle traffic: the same four entry points on the linear kernels
int hwy_highway_linear_reset(const HwyHighwayParams* p, const HwyHighwayState* s, const HwyLinearTraffic* t,
                             const uint8_t* mask, float* obs, void* stream) {
    if (validate(p, s) || validate_linear(t)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    if (ensure_pcg_jump(st)) return 1;
    if (launch_linear_reset(p, s, t, mask, nullptr, st)) return 1;
    if (obs) return launch_observe(p, s, mask, nullptr, obs, st);
    return 0;
}

int hwy_highway_linear_autoreset(const HwyHighwayParams* p, const HwyHighwayState* s, const HwyLinearTraffic* t,
                                 const uint8_t* terminated, const uint8_t* truncated, float* obs, void* stream) {
    if (validate(p, s) || validate_linear(t)) return 1;
    if (!terminated || !truncated || !obs) return fail("%s", "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (launch_linear_reset(p, s, t, terminated, truncated, st)) return 1;
    return launch_observe(p, s, terminated, truncated, obs, st);
}

int hwy_highway_linear_step(const HwyHighwayParams* p, const HwyHighwayState* s, const HwyLinearTraffic* t,
                            const int32_t* action_i, const float* action_f, float* obs, double* reward,
                            uint8_t* terminated, uint8_t* truncated, double* info_speed, uint8_t* info_crashed,
                            int autoreset, float* final_obs, void* stream) {
    if (check_step_args(p, s, action_i, action_f, obs, reward, terminated, truncated, autoreset)) return 1;
    if (validate_linear(t)) return 1;
    return dispatch_step(p, s, t, action_i, action_f, obs, reward, terminated, truncated, info_speed, info_crashed,
                         autoreset, final_obs, (cudaStream_t)stream);
}

int hwy_highway_linear_substeps(const HwyHighwayParams* p, const HwyHighwayState* s, const HwyLinearTraffic* t,
                                int n_substeps, const float* action_f, void* stream) {
    if (validate(p, s) || validate_linear(t)) return 1;
    if (n_substeps < 1 || n_substeps > 4096) return fail("%s", "n_substeps must be in 1..4096");
    return dispatch_step(p, s, t, nullptr, action_f, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                         -n_substeps, nullptr, (cudaStream_t)stream);
}

}  // extern "C"

namespace {
int check_step_args(const HwyHighwayParams* p, const HwyHighwayState* s, const int32_t* action_i,
                    const float* action_f, float* obs, double* reward, uint8_t* terminated, uint8_t* truncated,
                    int autoreset) {
    if (validate(p, s)) return 1;
    if (!obs || !reward || !terminated || !truncated) return fail("%s", "null output pointer");
    if (p->action_type == 0 && !action_i) return fail("%s", "DiscreteMetaAction needs action_i");
    if (p->action_type == 1 && !action_f) return fail("%s", "ContinuousAction needs action_f");
    if (autoreset != HWY_AUTORESET_DISABLED && autoreset != HWY_AUTORESET_SAME_STEP)
        return fail("%s", "unknown autoreset mode");
    return 0;
}

int dispatch_step(const HwyHighwayParams* p, const HwyHighwayState* s, const HwyLinearTraffic* t,
                  const int32_t* action_i, const float* action_f, float* obs, double* reward, uint8_t* terminated,
                  uint8_t* truncated, double* info_speed, uint8_t* info_crashed, int autoreset, float* final_obs,
                  cudaStream_t st) {
    int tpe = tpe_for(p->n_vehicles);
    // HWYB200_GENERAL_LANES=1 (tests): run the general-geometry instantiation on a congruent lane table too
    const char* force_general = getenv("HWYB200_GENERAL_LANES");
    const bool al = lanes_congruent_host(p) && !(force_general && force_general[0] == '1');
#define HWY_LAUNCH_STEP(T, A)                                                                              \
    launch_step<T, A>(p, s, t, action_i, action_f, obs, reward, terminated, truncated, info_speed, info_crashed, \
                      autoreset, final_obs, st)
    int rc;
    if (tpe == 32)
        rc = al ? HWY_LAUNCH_STEP(32, true) : HWY_LAUNCH_STEP(32, false);
    else if (tpe == 64)
        rc = al ? HWY_LAUNCH_STEP(64, true) : HWY_LAUNCH_STEP(64, false);
    else
        rc = al ? HWY_LAUNCH_STEP(128, true) : HWY_LAUNCH_STEP(128, false);
#undef HWY_LAUNCH_STEP
    if (rc) return 1;
    if (check_launch(t ? "highway_linear_step_kernel" : "highway_step_kernel")) return 1;
    return 0;
}
}  // namespace
