// hwy_highway.cu — sm_90a kernels + C ABI for the straight-highway family
// (highway-v0 / highway-fast-v0) of the batched HighwayEnv hot path.
//
// Thread mapping: one (env, vehicle) pair per thread, TPE threads per env (32/64/128, the
// next power of two >= n_vehicles).  The whole AbstractEnv.step — every substep of
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
#include <atomic>
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

template <int TPE>
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
    key_scratch[i] = key;
    env_sync<TPE>();
    // stable rank among the valid candidates (python sorted() on |lane_distance_to|)
    int rank = 0, n_valid = 0;
    for (int u = 1; u < V; ++u) {
        double ku = key_scratch[u];
        n_valid += ku < INFINITY;
        rank += (ku < key) || (ku == key && u < i);
    }
    // obs_env == nullptr: an env of the block that is not observed (masked out, a surplus slot of the last block, not
    // re-spawned).  It still runs to here so that every thread of the block meets the same barrier instruction.
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
    if (i < K && i >= filled) {
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
// with atomics.  Callers put a barrier between publish() and build_frame().
template <int TPE>
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
        // getattr(ego_vehicle, "target_speed", 0): a plain Vehicle has none (behavior.py:172)
        F.ts[i] = meta_kind(r.meta) == HWY_KIND_VEHICLE ? 0.0 : r.target_speed;
        F.ls[i] = lane_s(P.lanes[0], r.x, r.y);
        F.lsf[i] = (float)F.ls[i];
        F.lane[i] = (unsigned char)meta_lane(r.meta);
        F.tgt[i] = (unsigned char)meta_target(r.meta);
    }
    if (i < HWY_MAX_LANES * NW) (&F.smask[0][0])[i] = 0;
    if (i == 0) {
        F.slow = 0;
        F.vmax_bits = 0u;
    }
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
// the pattern is anything else (rank_count decides).  Boundary k = 32 w + b + 1 is bit b of word w.
template <int TPE>
__device__ __noinline__ int rank_repair(const Frame<TPE>& F, const Frame<TPE>& prev, int V, int i, bool active) {
    constexpr int NW = TPE / 32;
    const int wl = i & 31;
    uint32_t inv[NW];
    uint32_t bad = 0;
#pragma unroll
    for (int w = 0; w < NW; ++w) {
        const int k = w * 32 + wl + 1;
        const bool in = k < V;
        const float a = in ? F.lsf[prev.perm[k - 1]] : 0.0f, c = in ? F.lsf[prev.perm[k]] : 1.0f;
        bool wrong = in && !(a < c) && !(a > c);  // equal (or NaN) keys: not this path
        if (in && a > c) {
            // the swapped pair against its outer neighbours (positions k-2 and k+1 are unmoved, see the spacing rule)
            if (k >= 2 && !(F.lsf[prev.perm[k - 2]] < c)) wrong = true;
            if (k + 1 < V && !(a < F.lsf[prev.perm[k + 1]])) wrong = true;
        }
        inv[w] = __ballot_sync(0xffffffffu, in && a > c);
        bad |= __ballot_sync(0xffffffffu, wrong);
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
template <int TPE>
__device__ __forceinline__ void build_frame(const HwyHighwayParams& P, EnvShared<TPE>& sm, Frame<TPE>& F,
                                            int i, bool active, bool aligned, const VehicleRegs& r,
                                            double dt, bool do_sweep, bool pruned, const Frame<TPE>* prev) {
    const int V = P.n_vehicles;
    const int wie = i >> 5;  // warp within the env
    const int lane = meta_lane(r.meta), tgt = meta_target(r.meta);
    // -- rank along the road (s, slot) and tie detection.  Float keys first: rounding to float
    // is monotone, so fu < fi implies su < si; only equal float keys need the doubles.
    int rank = 0;
    // The order along the road rarely changes within one substep: with the previous frame of the same launch at hand
    // (`prev`, uniform), every warp of the env checks the whole chain key[perm[k-1]] < key[perm[k]] under the previous
    // permutation (V - 1 float comparisons spread over its 32 lanes, no communication between the warps: each reaches
    // the same verdict).  A strictly increasing chain of float keys is a strictly increasing chain of the doubles they
    // were rounded from, so the ranks are the previous ones and there is neither a tie nor an ambiguity — the O(V)
    // scan per thread (14 % of the kernel's instructions at V = 51) runs only when some pair swapped or drew level.
    bool reuse = false;
    if (prev) {
        bool ok = true;
#pragma unroll 1
        for (int k = (i & 31) + 1; k < V; k += 32) ok = ok && (F.lsf[prev->perm[k - 1]] < F.lsf[prev->perm[k]]);
        reuse = __all_sync(0xffffffffu, ok);
    }
    bool tie = false;
    if (reuse) {
        rank = active ? prev->rank[i] : 0;
    } else {
        // (the repair pays for itself only where the count is long, so only the 128-slot kernel uses it)
        int rt = (TPE >= 128 && prev) ? rank_repair(F, *prev, V, i, active) : -1;
        if (rt < 0) rt = rank_count(F, V, i, active);  // first frame of a launch, ties, or more than isolated swaps
        rank = rt & 0xff;
        tie = (rt >> 8) != 0;
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
        if ((i & 31) == 0) {
            F.lane_is[l][wie] = b_lane;
            F.tm[l][wie] = b_tgt;
        }
    }
    // superset of the vehicles whose MOBIL decision may fire in the coming act (the crashed
    // flag may still be stale here; crashed vehicles never fire, so this only over-approximates)
    uint32_t b_fired = __ballot_sync(0xffffffffu, active && is_idm && lane == tgt && P.lane_change_delay < r.timer);
    if ((i & 31) == 0) F.fired[wie] = b_fired;

    // -- collision sweep, pass 1: every gated pair once.  A pair with exactly one
    // check_collisions side is taken by the other side's thread (so the controlled vehicle's
    // pairs are spread over the block); pairs of two checking vehicles are dealt round-robin.
    if (do_sweep && pruned) {
        // many checking vehicles (highway-v0: all of them): the sweep runs after the next barrier over the
        // rank-neighbours only (sweep_pruned); here just the env's speed bound.  Non-negative floats order
        // like their bit patterns.
        unsigned vb = __float_as_uint(active ? fmaxf(__double2float_ru(r.speed), 0.0f) : 0.0f);
        vb = __reduce_max_sync(0xffffffffu, vb);
        if ((i & 31) == 0) atomicMax(&F.vmax_bits, vb);
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
template <int TPE>
__device__ __forceinline__ void spawn_fused(const HwyHighwayParams& P, const HwyHighwayState& S,
                                            EnvShared<TPE>& sm, int e, int i, bool active,
                                            bool do_reset, bool simple_geometry, VehicleRegs& r,
                                            int& speed_index) {
    const int V = P.n_vehicles, L = P.lanes_count;
    const size_t n = (size_t)S.n_envs;
    Pcg64 g0;
    double speed = 0.0, delta = 4.0, incr = 0.0;
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
    auto n64_before = [&](int k) { return k == 0 ? 0 : 1 + 3 * (k - 1); };            // 64-bit outputs before k
    auto fresh_before = [&](int q) { return h0 == 0 ? (q + 1) / 2 : q / 2; };         // outputs used by requests < q
    auto base_of = [&](int k) { return fresh_before(q_before(k)) + n64_before(k); };  // outputs before vehicle k
    if (do_reset && active && simple_geometry) {
        const int k = i;
        const bool has32 = k == 0 ? ego32 : n32;
        Pcg64 g = pcg_at(g0, base_of(k));
        uint32_t r32 = 0;
        if (has32) {
            const int rq = q_before(k);
            if (((h0 + rq) & 1) == 0) {
                r32 = (uint32_t)g.next64();  // fresh output: low half (the high half stays buffered)
            } else if (rq == 0) {
                r32 = g0.u32;                // the half buffered before this reset
            } else {
                // high half of the output the previous requester opened: vehicle k-1
                Pcg64 gp = pcg_at(g0, base_of(k - 1));
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
            Pcg64 ge = pcg_at(g0, fresh_before(Q) + n64_before(V));
            uint32_t has_f = (uint32_t)((h0 + Q) & 1), u_f = g0.u32;
            if (Q > 0) {
                int rf = Q - 1;  // last fresh request
                if (((h0 + rf) & 1) != 0) rf -= 1;
                if (rf >= 0) {
                    int kf = ego32 ? rf : rf + 1;  // vehicle issuing request rf
                    Pcg64 gp = pcg_at(g0, base_of(kf));
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
// AL (host-checked, lanes_congruent): every lane is a copy of lane 0 shifted sideways — what
// RoadNetwork.straight_road_network builds (road/road.py:291-321) — so the general-geometry branches (per-lane
// projections in lane_distance / closest_lane, F.slow for unaligned lanes) are compiled out.  The per-substep loop
// of this kernel is about as large as the SM's instruction cache, so code bytes on the hot path are a first-order
// cost.
template <int TPE, bool AL>
__global__ void __launch_bounds__(HWY_STEP_BOUND_THREADS, HWY_STEP_BOUND_BLOCKS)
highway_step_kernel(const __grid_constant__ HwyHighwayParams P, const HwyHighwayState S,
                    const int32_t* __restrict__ action_i, const float* __restrict__ action_f,
                    float* __restrict__ obs, double* __restrict__ reward,
                    uint8_t* __restrict__ terminated, uint8_t* __restrict__ truncated,
                    double* __restrict__ info_speed, uint8_t* __restrict__ info_crashed,
                    const int autoreset, float* __restrict__ final_obs) {
    constexpr int NW = TPE / 32;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    EnvShared<TPE>* smem = reinterpret_cast<EnvShared<TPE>*>(smem_raw);
    const int EPB = blockDim.x / TPE;
    const int sub = threadIdx.x / TPE;
    const int i = threadIdx.x % TPE;
    const int env = blockIdx.x * EPB + sub;
    const bool env_ok = env < S.n_envs;  // surplus envs of the last block mirror the last env
    const int e = env_ok ? env : S.n_envs - 1;
    EnvShared<TPE>& sm = smem[sub];
    const int V = P.n_vehicles;
    const bool active = i < V;
    const size_t slot = (size_t)e * S.vp + (active ? i : 0);
    const bool aligned = AL || lanes_aligned(P);
    const bool congruent = AL || lanes_congruent(P);

    VehicleRegs r;
    load_vehicle(S, slot, r);
    const int kind = meta_kind(r.meta);
    int speed_index = (i == 0) ? S.speed_index[e] : 0;
    double act_steer = 0.0, act_accel = 0.0;
    // autoreset < 0 (hwy_highway_substeps): -autoreset times Road.act() + Road.step(dt) and nothing else — no
    // action_type.act, no observation / reward / clock; the controlled vehicle acts like ControlledVehicle.act(None)
    const int substeps_only = autoreset < 0 ? -autoreset : 0;
    const int frames = substeps_only ? substeps_only : P.simulation_frequency / P.policy_frequency;
    const double dt = 1.0 / P.simulation_frequency;

    // ---- static masks
    {
        uint32_t b_cc = __ballot_sync(0xffffffffu, active && (r.meta & HWY_META_CHECK_COLLISIONS));
        uint32_t b_ctrl = __ballot_sync(0xffffffffu, active && kind != HWY_KIND_VEHICLE);
        if ((i & 31) == 0) {
            sm.cc[i >> 5] = b_cc;
            sm.ctrl[i >> 5] = b_ctrl;
            sm.mid[i >> 5] = 0;
        }
        sm.last_will[i] = -1;
        sm.crash_hit[i] = 0;
        if (i < NW) sm.ok_left[i] = sm.ok_right[i] = 0;
        if (i == 0) sm.n_items = 0;
        if (active) sm.delta[i] = r.delta;
    }
    const IdmK K = make_idm(P);
    // all-pairs gate (every vehicle checks collisions): rank-pruned sweep; a single checking vehicle (highway-fast)
    // already costs one pre-check per thread
    const bool pruned = P.others_check_collisions != 0;
    int p = 1;
    PHASE_INIT();
    PHASE_MARK(0);  // load + static masks

    // One iteration = stage the current state, derive its masks (+ the collision sweep of the
    // substep that produced it), then — except after the last substep — act and integrate.
    for (int frame = 0;; ++frame) {
        p ^= 1;
        Frame<TPE>& F = sm.f[p];
        publish(P, F, i, active, r);
        PHASE_MARK(1);  // publish
        env_sync<TPE>();
        PHASE_MARK(2);  // barrier after publish
        if (i < NW) sm.mid[i] = sm.ok_left[i] = sm.ok_right[i] = 0;  // all readers are past phase B
        if (i == 0) sm.n_items = 0;
        // frame 0: masks only — the sweep of the stored state ran at the end of the substep that
        // produced it (previous launch).  Later: Road.step's sweep (road/road.py:477-481).
        build_frame(P, sm, F, i, active, aligned, r, dt, frame > 0, pruned, frame > 0 ? &sm.f[p ^ 1] : nullptr);
        PHASE_MARK(3);  // ranks, masks, sweep pass 1
        if (pruned && frame > 0) {  // uniform over the grid
            env_sync_phase<TPE, 3>();
            sweep_pruned(sm, F, V, i, active, dt);
        }
        env_sync_phase<TPE, 3>();
        PHASE_MARK(4);  // barrier after build
        if (active && frame > 0) apply_collisions(sm, F, i, r, dt);
        PHASE_MARK(5);  // sweep pass 2
        if (frame == frames) break;

        // ---- action_type.act(action) on the first frame (abstract.py:294-304)
        if (frame == 0) {
            if (i == 0) {
                if (kind == HWY_KIND_MDP) {
                    // MDPVehicle.act (controller.py:295-315) + ControlledVehicle.act lane part
                    // (:99-124); labels action.py:204.  follow_road (:135-143) cannot change the
                    // target on the single-road highway graph (next_lane hits KeyError,
                    // road/road.py:129-130).
                    int a = substeps_only ? 1 : action_i[e];  // substeps only: act(None) = IDLE
                    if (a == 3 || a == 4) {
                        int idx = speed_to_index(P, r.speed) + (a == 3 ? 1 : -1);
                        idx = max(0, min(idx, P.n_target_speeds - 1));
                        speed_index = idx;
                        r.target_speed = P.target_speeds[idx];
                        F.ts[0] = r.target_speed;
                    } else if (a == 0 || a == 2) {
                        int old = meta_target(r.meta);
                        int id = old + (a == 2 ? 1 : -1);
                        id = max(0, min(id, P.lanes_count - 1));
                        if (lane_reachable(P.lanes[id], r.x, r.y)) {
                            r.meta = meta_set_target(r.meta, id);
                            F.tgt[0] = (unsigned char)id;
                            F.tm[old][0] &= ~1u;
                            F.tm[id][0] |= 1u;
                        }
                    }
                } else {
                    // ContinuousAction.get_action/act (action.py:136-162): Box is float32 and
                    // lmap (utils.py:31-33) stays in float32 (NEP 50 weak python scalars)
                    // (substeps only: the vehicle's current action dict, or the default {0, 0} when none is given —
                    // lmap(0) of the symmetric default ranges)
                    float a0 = action_f ? action_f[2 * (size_t)e] : 0.0f, a1 = action_f ? action_f[2 * (size_t)e + 1] : 0.0f;
                    if (P.act_clip) {
                        a0 = fminf(fmaxf(a0, -1.0f), 1.0f);
                        a1 = fminf(fmaxf(a1, -1.0f), 1.0f);
                    }
                    float acc = __fadd_rn((float)P.acc_lo,
                                          __fdiv_rn(__fmul_rn(__fsub_rn(a0, -1.0f),
                                                              (float)(P.acc_hi - P.acc_lo)), 2.0f));
                    float st = __fadd_rn((float)P.steer_lo,
                                         __fdiv_rn(__fmul_rn(__fsub_rn(a1, -1.0f),
                                                             (float)(P.steer_hi - P.steer_lo)), 2.0f));
                    act_accel = (double)acc;
                    act_steer = (double)st;
                }
            }
            env_sync<TPE>();
        }

        PHASE_MARK(6);  // ego action (+ barrier on frame 0)
        // ---- Road.act() (road/road.py:464-467), phase A1: own-lane IDM; lane-change policy set-up
        const int lane = meta_lane(r.meta);
        const int tgt0 = meta_target(r.meta);
        const bool crashed = (r.meta & HWY_META_CRASHED) != 0;
        const bool idm_active = active && kind == HWY_KIND_IDM && !crashed;  // behavior.py:102-103
        bool is_mid = false, fired = false;
        double acc = 0.0, free_i = 0.0;
        if (idm_active) {
            free_i = idm_free_term(K.comfort_acc_max, r.speed, r.target_speed, P.lanes[lane].speed_limit, r.delta);
            int f_own, r_own;
            neighbours(P, F, V, lane, i, f_own, r_own);
            acc = free_i;  // behavior.py:115-120
            if (f_own >= 0) acc -= idm_gap_term(P, K, F, aligned, i, f_own);
            if (lane != tgt0) {
                // change_lane_policy, ongoing change (behavior.py:229-244).  Only a controlled
                // vehicle v that is not on our target lane T and whose target is T when we act
                // can abort us: candidates = (target is T now) or (may switch to T this act).
                is_mid = true;
                uint32_t g[NW];
#pragma unroll
                for (int w = 0; w < NW; ++w) {
                    uint32_t may = F.tm[tgt0][w];
                    uint32_t adj = (tgt0 > 0 ? F.lane_is[tgt0 - 1][w] : 0u) |
                                   (tgt0 < P.lanes_count - 1 ? F.lane_is[tgt0 + 1][w] : 0u);
                    may |= F.fired[w] & adj;
                    uint32_t cand = may & sm.ctrl[w] & ~F.lane_is[tgt0][w];
                    if (w == (i >> 5)) cand &= ~(1u << (i & 31));
                    g[w] = 0;
                    while (cand) {
                        int b = __ffs(cand) - 1;
                        cand &= cand - 1;
                        int v = w * 32 + b;
                        double d = lane_distance(P, F, aligned, i, v);
                        double d_star = desired_gap(K, F, i, v);
                        if (0 < d && d < d_star) g[w] |= 1u << b;
                    }
                    sm.geo[i][w] = g[w];
                }
                atomicOr(&sm.mid[i >> 5], 1u << (i & 31));
            } else if (P.lane_change_delay < r.timer) {  // utils.do_every (utils.py:27-28)
                r.timer = 0.0;
                fired = true;
                // side_lanes (road/road.py:200-211): id-1 then id+1.  Each admissible candidate
                // becomes a work item; mobil() itself runs in phase A2 on a dense set of threads.
                sm.free_t[i] = free_i;
                sm.acc_own[i] = acc;
                sm.f_own[i] = (signed char)f_own;
                sm.r_own[i] = (signed char)r_own;
                if (!(fabs(r.speed) < 1)) {
                    for (int k = 0; k < 2; ++k) {
                        int cand = k == 0 ? lane - 1 : lane + 1;
                        if (cand < 0 || cand > P.lanes_count - 1) continue;
                        if (!lane_reachable(P.lanes[cand], r.x, r.y)) continue;
                        int slot_ = atomicAdd(&sm.n_items, 1);
                        sm.items[slot_] = (unsigned short)(i | (cand << 8) | (k << 15));
                    }
                }
            }
        }
        PHASE_MARK(7);  // phase A1
        env_sync_phase<TPE, 2>();
        PHASE_MARK(8);  // barrier after phase A1

        // ---- phase A2: mobil(lane_index) (behavior.py:265-324; route None => acceleration-gain
        // branch) for the queued (vehicle, candidate) items, one item per thread.
        for (int t = i; t < sm.n_items; t += TPE) {
            const int it = sm.items[t];
            const int v = it & 0xff, cand = (it >> 8) & 0x7f, right = it >> 15;
            const double delta_v = sm.delta[v];
            int new_preceding, new_following;
            neighbours_cold(P, F, V, cand, v, new_preceding, new_following);
            double new_following_pred_a = idm_acceleration_of(P, K, F, aligned, delta_v, new_following, v);
            if (new_following_pred_a < -P.lane_change_max_braking_imposed) continue;
            double self_pred_a = sm.free_t[v];
            if (new_preceding >= 0) self_pred_a -= idm_gap_term(P, K, F, aligned, v, new_preceding);
            double self_a = sm.acc_own[v];  // acceleration(self, old_preceding)
            double jerk = self_pred_a - self_a;
            if (P.politeness != 0.0) {
                const int f_o = sm.f_own[v], r_o = sm.r_own[v];
                double new_following_a =
                    idm_acceleration_of(P, K, F, aligned, delta_v, new_following, new_preceding);
                double old_following_a = idm_acceleration_of(P, K, F, aligned, delta_v, r_o, v);
                double old_following_pred_a = idm_acceleration_of(P, K, F, aligned, delta_v, r_o, f_o);
                jerk = self_pred_a - self_a +
                       P.politeness * (new_following_pred_a - new_following_a + old_following_pred_a -
                                       old_following_a);
            }
            if (jerk < P.lane_change_min_acc_gain) continue;
            atomicOr(right ? &sm.ok_right[v >> 5] : &sm.ok_left[v >> 5], 1u << (v & 31));
        }
        PHASE_MARK(13);  // phase A2
        env_sync_phase<TPE, 2>();
        PHASE_MARK(14);  // barrier after phase A2

        // ---- Road.act() phase B (steering + target-lane IDM with the final target), then
        // Road.step(dt): Vehicle.step (kinematics.py:130-177; IDMVehicle.step behavior.py:139-148).
        // The new state goes to the other frame, so no barrier is needed before staging it.
        if (active) {
            // both side lanes may pass mobil(); the later one (id+1) wins (behavior.py:252-263)
            int tgt = tgt0;
            if (fired) {
                if (test_bit(sm.ok_right, i))
                    tgt = lane + 1;
                else if (test_bit(sm.ok_left, i))
                    tgt = lane - 1;
            }
            if (is_mid) {
                // Ordered resolution of the Gauss-Seidel abort scan (behavior.py:229-244).  Vehicles
                // act in list order: vehicle j sees the NEW target of every earlier vehicle and the
                // OLD one of every later vehicle.  Only events on our target lane T matter (a
                // vehicle leaving T, or an aborting vehicle returning to its own lane, sits ON the
                // lane it now targets and is excluded by `lane_index != T`), so each mid-change
                // vehicle replays, redundantly and in registers, the decisions of the earlier
                // mid-change vehicles that share its target.
                const int T = tgt0, iw = i >> 5, ib = i & 31;
                uint32_t tmT[NW], lneT[NW], chgT[NW], ab[NW];
#pragma unroll
                for (int w = 0; w < NW; ++w) {
                    tmT[w] = F.tm[T][w];
                    lneT[w] = ~F.lane_is[T][w];
                    // vehicles whose MOBIL decision just switched their target to T
                    chgT[w] = (T > 0 ? sm.ok_right[w] & F.lane_is[T - 1][w] : 0u) |
                              (T < P.lanes_count - 1 ? sm.ok_left[w] & ~sm.ok_right[w] & F.lane_is[T + 1][w] : 0u);
                    ab[w] = 0;
                }
#pragma unroll
                for (int w = 0; w < NW; ++w) {
                    uint32_t m = sm.mid[w] & tmT[w];
                    if (w > iw) m = 0;
                    if (w == iw) m &= (2u << ib) - 1u;  // mids up to and including ourselves
                    while (m) {
                        int b = __ffs(m) - 1;
                        m &= m - 1;
                        int j = w * 32 + b;
                        uint32_t hit = 0;
#pragma unroll
                        for (int w2 = 0; w2 < NW; ++w2) {
                            uint32_t below = w2 < w ? ~0u : (w2 == w ? (1u << b) - 1u : 0u);
                            uint32_t cur = (tmT[w2] & ~ab[w2]) | (chgT[w2] & below);
                            hit |= sm.geo[j][w2] & lneT[w2] & cur;
                        }
                        if (hit) ab[w] |= 1u << b;  // behavior.py:241-243: target := current lane
                    }
                }
                if ((ab[iw] >> ib) & 1u) tgt = lane;
            }
            // IDMVehicle.act (behavior.py:109-112) and ControlledVehicle.act(None)
            // (controller.py:126-133, runs even when crashed) share the steering law
            double sin_beta = 0.0, cos_beta = 1.0;  // crashed: steering 0 (clip_actions :155-158)
            if (idm_active || (kind == HWY_KIND_MDP && !crashed)) {
                double xs = steering_sin_slip(P.lanes[tgt], r.x, r.y, r.heading, r.speed);
                beta_of_controlled(xs, sin_beta, cos_beta);
            } else if (kind == HWY_KIND_VEHICLE && !crashed) {
                beta_of_angle(act_steer, sin_beta, cos_beta);
            }
            if (idm_active) {
                if (lane != tgt) {  // behavior.py:121-131
                    int f_t, r_t;
                    neighbours_cold(P, F, V, tgt, i, f_t, r_t);
                    double tacc = free_i;
                    if (f_t >= 0) tacc -= idm_gap_term(P, K, F, aligned, i, f_t);
                    acc = fmin(acc, tacc);
                }
                act_accel = clipd(acc, -P.acc_max, P.acc_max);
            } else if (kind == HWY_KIND_MDP) {
                act_accel = kKpA * (r.target_speed - r.speed);  // speed_control :189-198
            }
            r.meta = meta_set_target(r.meta, tgt);

            PHASE_MARK(9);  // phase B
            if (kind == HWY_KIND_IDM) r.timer += dt;
            if (crashed) {  // clip_actions :155-168
                act_steer = 0.0;
                act_accel = -1.0 * r.speed;
            }
            if (r.speed > kMaxSpeed)
                act_accel = fmin(act_accel, 1.0 * (kMaxSpeed - r.speed));
            else if (r.speed < kMinSpeed)
                act_accel = fmax(act_accel, 1.0 * (kMinSpeed - r.speed));
            // cos/sin(heading + beta) by angle addition from the staged cos/sin(heading)
            const double ch = F.c[i], sh = F.s[i];
            double cs = ch * cos_beta - sh * sin_beta, sn = sh * cos_beta + ch * sin_beta;
            double vx = r.speed * cs, vy = r.speed * sn;
            r.x += vx * dt;
            r.y += vy * dt;
            if (r.meta & HWY_META_HAS_IMPACT) {
                r.x += r.imp_x;
                r.y += r.imp_y;
                r.meta = (r.meta | HWY_META_CRASHED) & ~HWY_META_HAS_IMPACT;
            }
            r.heading += div_finite(r.speed * sin_beta, kVehLength / 2) * dt;
            r.speed += act_accel * dt;
            int nl = closest_lane(P, r.x, r.y, r.heading, congruent);  // on_state_update :170-177
            r.meta = meta_set_lane(r.meta, nl);
            if (kind == HWY_KIND_VEHICLE) r.meta = meta_set_target(r.meta, nl);  // schema: mirrors lane
        }
        PHASE_MARK(10);  // integrate
    }

    PHASE_MARK(11);
    if (substeps_only) {  // uniform over the grid
        if (active && env_ok) store_vehicle(S, slot, r);
        return;
    }
    // ---- epilogue: state back to HBM, observation, reward, termination
    const Frame<TPE>& F = sm.f[p];
    const size_t obs_off = (size_t)e * P.obs_vehicles_count * obs_columns(P);
    float* obs_env = obs + obs_off;
    kinematics_observe(P, F, sm.key, i, r.heading, env_ok ? obs_env : nullptr,
                       (autoreset && final_obs) ? final_obs + obs_off : nullptr);
    if (i == 0) {
        sm.done = 0;
        sm.sp_fallback = 0;
    }
    if (i == 0 && env_ok) {
        // envs/highway_env.py:100-151
        const int lane = meta_lane(r.meta);
        const HwyStraightLane& L = P.lanes[lane];
        int rl = kind == HWY_KIND_VEHICLE ? lane : meta_target(r.meta);
        double forward_speed = r.speed * F.c[0];
        double scaled_speed = lmap(forward_speed, P.reward_speed_lo, P.reward_speed_hi, 0.0, 1.0);
        double es, elat;
        lane_local(L, r.x, r.y, es, elat);
        bool on_road = lane_on(L, es, elat, 0.0);
        bool is_crashed = (r.meta & HWY_META_CRASHED) != 0;
        int nl1 = P.lanes_count - 1 > 1 ? P.lanes_count - 1 : 1;
        double rew = 0.0;
        rew = rew + P.collision_reward * (is_crashed ? 1.0 : 0.0);
        rew = rew + P.right_lane_reward * ((double)rl / (double)nl1);
        rew = rew + P.high_speed_reward * clipd(scaled_speed, 0.0, 1.0);
        rew = rew + 0.0 * (on_road ? 1.0 : 0.0);
        if (P.normalize_reward)
            rew = lmap(rew, P.collision_reward, P.high_speed_reward + P.right_lane_reward, 0.0, 1.0);
        rew *= on_road ? 1.0 : 0.0;
        double t = S.time[e] + 1.0 / P.policy_frequency;  // abstract.py:274
        S.time[e] = t;
        S.speed_index[e] = speed_index;
        reward[e] = rew;
        terminated[e] = (uint8_t)(is_crashed || (P.offroad_terminal && !on_road));
        truncated[e] = (uint8_t)(t >= P.duration);
        if (info_speed) info_speed[e] = r.speed;  // abstract.py:200-217 _info
        if (info_crashed) info_crashed[e] = (uint8_t)is_crashed;
        if (S.reward_terms) {  // _rewards (highway_env.py:118-137): info["rewards"]
            double* rt = S.reward_terms + (size_t)e * HWY_REWARD_TERMS;
            rt[0] = is_crashed ? 1.0 : 0.0;
            rt[1] = (double)rl / (double)nl1;
            rt[2] = clipd(scaled_speed, 0.0, 1.0);
            rt[3] = on_road ? 1.0 : 0.0;
            rt[4] = 0.0;
        }
        sm.done = autoreset && (is_crashed || (P.offroad_terminal && !on_road) || t >= P.duration);
    }
    if (autoreset) {
        // ---- SameStep autoreset fused into the step: envs that ended re-spawn from their own
        // numpy stream and return the reset observation (gymnasium AutoresetMode.SAME_STEP)
        env_sync<TPE>();
        const bool do_reset = env_ok && sm.done;
        const bool simple_geometry = aligned && P.lanes[0].start_x == 0.0 && P.lanes[0].dir_x == 1.0;
        spawn_fused(P, S, sm, e, i, active, do_reset, simple_geometry, r, speed_index);
        Frame<TPE>& G = sm.f[p ^ 1];
        if (do_reset) publish(P, G, i, active, r);
        // barrier + "does any env of this block re-spawn?": the second observation runs under a block-uniform
        // condition, so that all threads of the block meet the same barrier instructions (a per-env condition around
        // __syncthreads() is what compute-sanitizer's synccheck rejects, even though the arrival counts match)
        const bool any_reset = __syncthreads_or(do_reset) != 0;
        if (any_reset) {
            kinematics_observe(P, G, sm.key, i, r.heading, do_reset ? obs_env : nullptr);
            if (do_reset && i == 0) {
                S.time[e] = 0.0;
                S.speed_index[e] = speed_index;
            }
        }
    }
    if (active && env_ok) store_vehicle(S, slot, r);
    if (autoreset && active && env_ok && sm.done) S.delta[slot] = r.delta;
    PHASE_MARK(12);  // epilogue
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
                       int use_mask, float* __restrict__ obs) {
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
    const bool wanted = env_ok && (!use_mask || (mask_a && mask_a[e]) || (mask_b && mask_b[e]));
    kinematics_observe(P, sm.f, sm.key, i, r.heading,
                       wanted ? obs + (size_t)e * P.obs_vehicles_count * obs_columns(P) : nullptr);
}

// ------------------------------------------------------------------ reset kernel
// HighwayEnv._create_road/_create_vehicles (envs/highway_env.py:55-98,177-182) with
// Vehicle.create_random (vehicle/kinematics.py:50-104), IDMVehicle.__init__ timer and
// randomize_behavior (behavior.py:64-69), MDPVehicle.__init__ (controller.py:284-293).
// The spawn is a sequential chain on the env's PCG64 stream => one thread per env.
__global__ void __launch_bounds__(128)
highway_reset_kernel(const __grid_constant__ HwyHighwayParams P, const HwyHighwayState S,
                     const uint8_t* __restrict__ mask_a, const uint8_t* __restrict__ mask_b,
                     int use_mask) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= S.n_envs) return;
    if (use_mask && !((mask_a && mask_a[e]) || (mask_b && mask_b[e]))) return;
    const int n = S.n_envs;
    Pcg64 g;
    g.s_hi = S.rng[0 * (size_t)n + e];
    g.s_lo = S.rng[1 * (size_t)n + e];
    g.i_hi = S.rng[2 * (size_t)n + e];
    g.i_lo = S.rng[3 * (size_t)n + e];
    u64 w4 = S.rng[4 * (size_t)n + e];
    g.has32 = (uint32_t)(w4 >> 32);
    g.u32 = (uint32_t)w4;

    double x_max = 0.0;  // running max of the longitudinal coordinates of spawned vehicles
    bool aligned = true;  // all lanes share origin-x and direction => s is lane independent
    for (int l = 1; l < P.lanes_count; ++l)
        aligned = aligned && P.lanes[l].start_x == P.lanes[0].start_x &&
                        P.lanes[l].dir_x == P.lanes[0].dir_x && P.lanes[l].dir_y == 0.0 &&
                        P.lanes[0].dir_y == 0.0;
    double2* pos = reinterpret_cast<double2*>(S.pos);
    double2* hs = reinterpret_cast<double2*>(S.hs);
    double2* tt = reinterpret_cast<double2*>(S.tt);
    double2* imp = reinterpret_cast<double2*>(S.imp);
    const size_t base = (size_t)e * S.vp;
    int ego_speed_index = -1;
    for (int v = 0; v < P.n_vehicles; ++v) {
        const bool is_ego = v == 0;
        // choice(list(graph.keys())) / choice(list(graph[_from].keys())): single element => no draw
        int id = (is_ego && P.initial_lane_id >= 0) ? P.initial_lane_id : g.choice(P.lanes_count);
        const HwyStraightLane& L = P.lanes[id];
        double speed = is_ego ? P.ego_speed : g.uniform(0.7 * L.speed_limit, 0.8 * L.speed_limit);
        double spacing = is_ego ? P.ego_spacing : 1 / P.vehicles_density;
        double default_spacing = 12 + 1.0 * speed;
        double offset = spacing * default_spacing * P.spawn_exp;
        double x0;
        if (v > 0) {
            if (aligned) {
                x0 = x_max;
            } else {  // np.max over lane.local_coordinates(v.position)[0] on the chosen lane
                x0 = lane_s(L, pos[base].x, pos[base].y);
                for (int j = 1; j < v; ++j) x0 = fmax(x0, lane_s(L, pos[base + j].x, pos[base + j].y));
            }
        } else {
            x0 = 3 * offset;
        }
        x0 += offset * g.uniform(0.9, 1.1);
        // lane.position(x0, 0), lane.heading_at(x0)  (road/lane.py:192-200)
        double px = (L.start_x + x0 * L.dir_x) + 0.0 * L.lat_x;
        double py = (L.start_y + x0 * L.dir_y) + 0.0 * L.lat_y;
        double heading = L.heading;
        double s_here = lane_s(L, px, py);
        x_max = v == 0 ? s_here : fmax(x_max, s_here);
        int lane = closest_lane(P, px, py, heading);  // RoadObject.__init__ objects.py:46-50
        double target_speed = speed;                   // `target_speed or self.speed`
        double timer = 0.0, delta = 4.0;
        int kind, cc;
        if (is_ego) {
            cc = 1;
            if (P.action_type == 0) {
                kind = HWY_KIND_MDP;
                ego_speed_index = speed_to_index(P, target_speed);
                target_speed = P.target_speeds[ego_speed_index];
            } else {
                kind = HWY_KIND_VEHICLE;
            }
        } else {
            kind = HWY_KIND_IDM;
            cc = P.others_check_collisions;
            timer = py_mod_pos((px + py) * kPi, P.lane_change_delay);  // behavior.py:64
            delta = g.uniform(P.delta_lo, P.delta_hi);                 // behavior.py:66-69
        }
        pos[base + v] = make_double2(px, py);
        hs[base + v] = make_double2(heading, speed);
        tt[base + v] = make_double2(target_speed, timer);
        imp[base + v] = make_double2(0.0, 0.0);
        S.delta[base + v] = delta;
        S.meta[base + v] = (lane << HWY_META_LANE_SHIFT) | (lane << HWY_META_TARGET_SHIFT) |
                           (cc ? HWY_META_CHECK_COLLISIONS : 0) | (kind << HWY_META_KIND_SHIFT) |
                           HWY_META_PRESENT;
    }
    S.speed_index[e] = ego_speed_index;
    S.time[e] = 0.0;
    S.rng[0 * (size_t)n + e] = g.s_hi;
    S.rng[1 * (size_t)n + e] = g.s_lo;
    S.rng[2 * (size_t)n + e] = g.i_hi;
    S.rng[3 * (size_t)n + e] = g.i_lo;
    S.rng[4 * (size_t)n + e] = ((u64)g.has32 << 32) | g.u32;
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

// Envs per block of the step kernel: as many as fit 512 threads (lock-step, see env_sync),
// reduced when that leaves the last wave of blocks mostly empty.  HWYB200_EPB overrides.
int step_envs_per_block(int tpe, int n_envs) {
    int max_epb = (hwy::kMaxBlockThreads < HWY_STEP_BOUND_THREADS ? hwy::kMaxBlockThreads : HWY_STEP_BOUND_THREADS) / tpe;
    if (max_epb < 1) max_epb = 1;
    if (const char* e = getenv("HWYB200_EPB")) {
        int v = atoi(e);
        if (v >= 1 && v <= max_epb) return v;
    }
    // Two resident blocks per SM (rather than one block of max_epb envs or many 1-env blocks): the blocks cover each other's
    // barrier stalls.  Small batches shrink the block so every SM still gets work.
    int n_sm = 132;
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev);
    int epb = max_epb >= 2 ? max_epb / 2 : 1;
    while (epb > 1 && (long)n_envs < (long)epb * 2 * n_sm) --epb;
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

template <int TPE, bool AL>
int launch_step(const HwyHighwayParams* p, const HwyHighwayState* s, const int32_t* action_i,
                const float* action_f, float* obs, double* reward, uint8_t* terminated,
                uint8_t* truncated, double* info_speed, uint8_t* info_crashed, int autoreset,
                float* final_obs, int blocks, int epb, cudaStream_t st) {
    if (autoreset > 0 && ensure_pcg_jump(st)) return 1;
    size_t smem = (size_t)epb * sizeof(hwy::EnvShared<TPE>);
    // the attribute is per device (and per template instance): cache it by device ordinal
    static std::atomic<size_t> configured[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return fail("%s", "cudaGetDevice failed");
    if (smem > configured[dev].load(std::memory_order_relaxed)) {
        cudaError_t err = cudaFuncSetAttribute(hwy::highway_step_kernel<TPE, AL>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (err != cudaSuccess) return fail("cudaFuncSetAttribute: %s", cudaGetErrorString(err));
        configured[dev].store(smem, std::memory_order_relaxed);
    }
    hwy::highway_step_kernel<TPE, AL><<<blocks, TPE * epb, smem, st>>>(
        *p, *s, action_i, action_f, obs, reward, terminated, truncated, info_speed, info_crashed,
        autoreset, final_obs);
    return 0;
}

int launch_observe(const HwyHighwayParams* p, const HwyHighwayState* s, const uint8_t* mask_a,
                   const uint8_t* mask_b, int use_mask, float* obs, cudaStream_t st) {
    int tpe = tpe_for(p->n_vehicles);
    Grid g = grid_for(tpe, s->n_envs);
    if (tpe == 32)
        hwy::highway_observe_kernel<32><<<g.blocks, g.threads, 0, st>>>(*p, *s, mask_a, mask_b, use_mask, obs);
    else if (tpe == 64)
        hwy::highway_observe_kernel<64><<<g.blocks, g.threads, 0, st>>>(*p, *s, mask_a, mask_b, use_mask, obs);
    else
        hwy::highway_observe_kernel<128><<<g.blocks, g.threads, 0, st>>>(*p, *s, mask_a, mask_b, use_mask, obs);
    return check_launch("highway_observe_kernel");
}

int launch_reset(const HwyHighwayParams* p, const HwyHighwayState* s, const uint8_t* mask_a,
                 const uint8_t* mask_b, int use_mask, cudaStream_t st) {
    int blocks = (s->n_envs + 127) / 128;
    hwy::highway_reset_kernel<<<blocks, 128, 0, st>>>(*p, *s, mask_a, mask_b, use_mask);
    return check_launch("highway_reset_kernel");
}
}  // namespace

namespace {
int dispatch_step(const HwyHighwayParams* p, const HwyHighwayState* s, const int32_t* action_i, const float* action_f,
                  float* obs, double* reward, uint8_t* terminated, uint8_t* truncated, double* info_speed,
                  uint8_t* info_crashed, int autoreset, float* final_obs, cudaStream_t st);
}

extern "C" {

int hwy_abi_version(void) { return HWY_ABI_VERSION; }
const char* hwy_last_error(void) { return g_err; }
uint64_t hwy_launch_count(void) { return g_launches; }
int hwy_highway_slot_stride(int n_vehicles) { return (n_vehicles + 1) & ~1; }

int hwy_highway_observe(const HwyHighwayParams* p, const HwyHighwayState* s, float* obs, void* stream) {
    if (validate(p, s)) return 1;
    if (!obs) return fail("%s", "obs is null");
    return launch_observe(p, s, nullptr, nullptr, 0, obs, (cudaStream_t)stream);
}

int hwy_highway_reset(const HwyHighwayParams* p, const HwyHighwayState* s, const uint8_t* mask,
                      float* obs, void* stream) {
    if (validate(p, s)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    int use_mask = mask != nullptr;
    if (ensure_pcg_jump(st)) return 1;  // the fused autoreset of later steps reads the table
    if (launch_reset(p, s, mask, nullptr, use_mask, st)) return 1;
    if (obs) return launch_observe(p, s, mask, nullptr, use_mask, obs, st);
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

int hwy_highway_autoreset(const HwyHighwayParams* p, const HwyHighwayState* s,
                          const uint8_t* terminated, const uint8_t* truncated, float* obs,
                          void* stream) {
    if (validate(p, s)) return 1;
    if (!terminated || !truncated || !obs) return fail("%s", "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (launch_reset(p, s, terminated, truncated, 1, st)) return 1;
    return launch_observe(p, s, terminated, truncated, 1, obs, st);
}

int hwy_highway_step(const HwyHighwayParams* p, const HwyHighwayState* s, const int32_t* action_i,
                     const float* action_f, float* obs, double* reward, uint8_t* terminated,
                     uint8_t* truncated, double* info_speed, uint8_t* info_crashed, int autoreset,
                     float* final_obs, void* stream) {
    if (validate(p, s)) return 1;
    if (!obs || !reward || !terminated || !truncated) return fail("%s", "null output pointer");
    if (p->action_type == 0 && !action_i) return fail("%s", "DiscreteMetaAction needs action_i");
    if (p->action_type == 1 && !action_f) return fail("%s", "ContinuousAction needs action_f");
    if (autoreset != HWY_AUTORESET_DISABLED && autoreset != HWY_AUTORESET_SAME_STEP)
        return fail("%s", "unknown autoreset mode");
    return dispatch_step(p, s, action_i, action_f, obs, reward, terminated, truncated, info_speed, info_crashed, autoreset,
                         final_obs, (cudaStream_t)stream);
}

/* B4 seam of the reference (abstract.py:304-307 minus action_type.act): n_substeps x (Road.act(); Road.step(dt)). */
int hwy_highway_substeps(const HwyHighwayParams* p, const HwyHighwayState* s, int n_substeps, const float* action_f,
                         void* stream) {
    if (validate(p, s)) return 1;
    if (n_substeps < 1 || n_substeps > 4096) return fail("%s", "n_substeps must be in 1..4096");
    return dispatch_step(p, s, nullptr, action_f, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, -n_substeps, nullptr,
                         (cudaStream_t)stream);
}

}  // extern "C"

namespace {
int dispatch_step(const HwyHighwayParams* p, const HwyHighwayState* s, const int32_t* action_i, const float* action_f,
                  float* obs, double* reward, uint8_t* terminated, uint8_t* truncated, double* info_speed,
                  uint8_t* info_crashed, int autoreset, float* final_obs, cudaStream_t st) {
    int tpe = tpe_for(p->n_vehicles);
    int epb = step_envs_per_block(tpe, s->n_envs);
    int blocks = (s->n_envs + epb - 1) / epb;
    // HWYB200_GENERAL_LANES=1 (tests): run the general-geometry instantiation on a congruent lane table too
    const char* force_general = getenv("HWYB200_GENERAL_LANES");
    const bool al = lanes_congruent_host(p) && !(force_general && force_general[0] == '1');
#define HWY_LAUNCH_STEP(T, A)                                                                              \
    launch_step<T, A>(p, s, action_i, action_f, obs, reward, terminated, truncated, info_speed, info_crashed, \
                      autoreset, final_obs, blocks, epb, st)
    int rc;
    if (tpe == 32)
        rc = al ? HWY_LAUNCH_STEP(32, true) : HWY_LAUNCH_STEP(32, false);
    else if (tpe == 64)
        rc = al ? HWY_LAUNCH_STEP(64, true) : HWY_LAUNCH_STEP(64, false);
    else
        rc = al ? HWY_LAUNCH_STEP(128, true) : HWY_LAUNCH_STEP(128, false);
#undef HWY_LAUNCH_STEP
    if (rc) return 1;
    if (check_launch("highway_step_kernel")) return 1;
    return 0;
}
}  // namespace
