// hwy_observe.cu — the observation plugin registry on the device: OccupancyGrid (every constructor option),
// TimeToCollision and LidarObservation for ANY env family (the reference's observation_factory,
// envs/common/observation.py:772-794, builds any ObservationType on any env).  The kernels read the state of
// either family through a HwyObsView; the lane table is a HwyNetGraph (the highway family passes the table of
// RoadNetwork.straight_road_network).  One block per (env, controlled vehicle).
//
// These are standalone epilogues: the fused step kernels keep their specialised observations (Kinematics on the
// highway family; Kinematics / default OccupancyGrid / TimeToCollision on the network family); any other
// (env, observation) pair runs the step and then one of these kernels — one extra read of a few KB of state per env.
//
// Reference paths are relative to /root/reference/highway_env.
#include <cstdio>
#include <cuda_runtime.h>

#include "../../include/hwyb200.h"
#include "hwy_abi.h"
#include "hwy_lanes.cuh"

namespace hwyobs {
using namespace hwy;
using namespace hwynet;

constexpr int kThreads = 128;
constexpr int R = HWY_NET_MAX_ROUTE;

struct Veh {
    double x, y, heading, speed;
    int lane, kind;
};
__device__ __forceinline__ Veh load_veh(const HwyObsView& v, int e, int slot) {
    const size_t k = (size_t)e * v.vp + slot;
    double2 p = reinterpret_cast<const double2*>(v.pos)[k];
    double2 h = reinterpret_cast<const double2*>(v.hs)[k];
    const int m = v.meta[k];
    return Veh{p.x, p.y, h.x, h.y, meta_lane(m), meta_kind(m)};
}
__device__ __forceinline__ bool is_controlled(int kind) { return kind == HWY_KIND_MDP || kind == HWY_KIND_VEHICLE; }

// slot of the a-th controlled vehicle of env e in list order (0 when there is none)
__device__ int find_ego(const HwyObsView& v, int e, int count, int agent) {
    int seen = 0;
    for (int s = 0; s < count; ++s) {
        if (is_controlled(meta_kind(v.meta[(size_t)e * v.vp + s]))) {
            if (seen == agent) return s;
            ++seen;
        }
    }
    return 0;
}

// Vehicle.to_dict (vehicle/kinematics.py:237-261) relative to the observer; road objects are not in road.vehicles
__device__ double vehicle_feature(const GraphShared& g, const HwyObsView& view, int e, int slot, const Veh& o,
                                  const Veh& ego, int feat, int observe_intentions) {
    double sn, cs;
    m_sincos(o.heading, &sn, &cs);
    switch (feat) {
        case HWY_FEAT_PRESENCE: return 1.0;
        case HWY_FEAT_X: return o.x - ego.x;
        case HWY_FEAT_Y: return o.y - ego.y;
        case HWY_FEAT_VX:
        case HWY_FEAT_VY: {
            double es, ec;
            m_sincos(ego.heading, &es, &ec);
            return feat == HWY_FEAT_VX ? o.speed * cs - ego.speed * ec : o.speed * sn - ego.speed * es;
        }
        case HWY_FEAT_HEADING: return o.heading;
        case HWY_FEAT_COS_H: return cs;
        case HWY_FEAT_SIN_H: return sn;
        case HWY_FEAT_COS_D:
        case HWY_FEAT_SIN_D: {
            // destination (:203-215): the end of the last route lane (lane id None -> 0); no route: the position
            const int rl = view.route_len ? view.route_len[(size_t)e * view.vp + slot] : 0;
            if (!observe_intentions || rl == 0) return 0.0;
            const int en = view.route[((size_t)e * view.vp + slot) * R + rl - 1];
            const int first = road_first(g, RT_FROM(en), RT_TO(en));
            const int id = RT_ID(en) < 0 ? 0 : RT_ID(en);
            const HwyNetLane& L = g.lanes[first + id];
            double dx, dy;
            lane_position(L, L.length, 0.0, dx, dy);
            dx -= o.x;
            dy -= o.y;
            if (dx == 0.0 && dy == 0.0) return 0.0;
            const double n = sqrt(dx * dx + dy * dy);
            return feat == HWY_FEAT_COS_D ? dx / n : dy / n;
        }
        case HWY_FEAT_LONG_OFF:
        case HWY_FEAT_LAT_OFF:
        case HWY_FEAT_ANG_OFF: {
            const HwyNetLane& L = g.lanes[o.lane];
            double lon, lat;
            lane_local(L, o.x, o.y, lon, lat);
            if (feat == HWY_FEAT_LONG_OFF) return lon;
            if (feat == HWY_FEAT_LAT_OFF) return lat;
            return wrap_to_pi(o.heading - lane_heading_at(L, lon));  // lane.local_angle (road/lane.py:145-147)
        }
        default: return NAN;
    }
}

// OccupancyGridObservation.pos_to_index (observation.py:422-444), position relative to the observer
__device__ __forceinline__ void grid_index(const HwyGridParams& P, double px, double py, double ce, double se,
                                           int& ci, int& cj) {
    if (P.align_to_vehicle_axes) {
        // np.array([[c, s], [-s, c]]) @ position: numpy rounds each row as fma(M[i][0], p[0], M[i][1] * p[1])
        const double rx = fma(ce, px, se * py), ry = fma(-se, px, ce * py);
        px = rx;
        py = ry;
    }
    ci = (int)floor((px - P.grid_lo[0]) / P.grid_step[0]);
    cj = (int)floor((py - P.grid_lo[1]) / P.grid_step[1]);
}

// ------------------------------------------------------------------ OccupancyGrid (observation.py:354-420)
// dynamic shared memory: GraphShared | owner[cells] (int) | road[cells] (unsigned char)
__global__ void __launch_bounds__(kThreads)
grid_kernel(const HwyNetGraph* __restrict__ graph, const __grid_constant__ HwyObsView view,
            const __grid_constant__ HwyGridParams P, const uint8_t* __restrict__ mask_a,
            const uint8_t* __restrict__ mask_b, float* __restrict__ obs) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    GraphShared& g = *reinterpret_cast<GraphShared*>(smem_raw);
    const int NX = P.shape[0], NY = P.shape[1], cells = NX * NY, F = P.n_features;
    int* owner = reinterpret_cast<int*>(smem_raw + ((sizeof(GraphShared) + 15) & ~size_t(15)));
    unsigned char* road = reinterpret_cast<unsigned char*>(owner + cells);
    const int A = view.n_agents > 1 ? view.n_agents : 1;
    const int e = blockIdx.x / A, agent = blockIdx.x % A;
    if (!env_selected(mask_a, mask_b, e)) return;
    stage_graph(g, graph);
    const int tid = threadIdx.x;
    const int count = view.count ? view.count[e] : view.n_vehicles;
    __shared__ int s_ego;
    if (tid == 0) s_ego = find_ego(view, e, count, agent);
    for (int k = tid; k < cells; k += kThreads) {
        owner[k] = 0x7fffffff;
        road[k] = 0;
    }
    __syncthreads();
    const Veh ego = load_veh(view, e, s_ego);
    double se, ce;
    m_sincos(ego.heading, &se, &ce);
    // vehicles are written in REVERSED list order (df[::-1]): the lowest index owns a shared cell
    for (int s = tid; s < count; s += kThreads) {
        const Veh o = load_veh(view, e, s);
        if (o.kind == HWY_KIND_OBSTACLE) continue;  // road.vehicles only
        double x = o.x - ego.x, y = o.y - ego.y;
        if (P.x_ranged) x = lmap(lmap(x, P.x_lo, P.x_hi, -1.0, 1.0), -1.0, 1.0, P.x_lo, P.x_hi);
        if (P.y_ranged) y = lmap(lmap(y, P.y_lo, P.y_hi, -1.0, 1.0), -1.0, 1.0, P.y_lo, P.y_hi);
        int ci, cj;
        grid_index(P, x, y, ce, se, ci, cj);
        if (0 <= ci && ci < NX && 0 <= cj && cj < NY) atomicMin(&owner[ci * NY + cj], s);
    }
    bool want_road = false;
    for (int l = 0; l < F; ++l) want_road = want_road || P.features[l] == HWY_FEAT_ON_ROAD;
    if (want_road) {
        // fill_road_layer_by_lanes (:466-499): waypoints every min(grid_step) within +-100 m of the observer's
        // longitudinal coordinate on each lane, clipped to the lane
        const double spacing = fmin(P.grid_step[0], P.grid_step[1]);
        for (int l = 0; l < g.n_lanes; ++l) {
            const HwyNetLane& L = g.lanes[l];
            const double origin = lane_s_of(L, ego.x, ego.y);
            const double start = origin - 100, stop = origin + 100;
            const int n = (int)ceil((stop - start) / spacing);  // np.arange length
            for (int k = tid; k < n; k += kThreads) {
                const double wp = clipd(start + k * spacing, 0.0, L.length);
                double px, py;
                lane_position(L, wp, 0.0, px, py);
                int ci, cj;
                grid_index(P, px - ego.x, py - ego.y, ce, se, ci, cj);
                if (0 <= ci && ci < NX && 0 <= cj && cj < NY) road[ci * NY + cj] = 1;
            }
        }
    }
    __syncthreads();
    float* out = obs + ((size_t)e * A + agent) * (size_t)F * cells;
    for (int k = tid; k < F * cells; k += kThreads) {
        const int layer = k / cells, cell = k - layer * cells;
        const int feat = P.features[layer];
        double val = NAN;
        if (feat == HWY_FEAT_ON_ROAD) {
            if (road[cell]) val = 1.0;
        } else if (feat != HWY_FEAT_UNKNOWN && owner[cell] != 0x7fffffff) {
            const int s = owner[cell];
            const Veh o = load_veh(view, e, s);
            val = vehicle_feature(g, view, e, s, o, ego, feat, P.observe_intentions);
            if (P.ranged[layer]) val = lmap(val, P.range_lo[layer], P.range_hi[layer], -1.0, 1.0);
        }
        float f = 0.0f;  // np.clip keeps NaN; astype(uint8) of NaN and nan_to_num both give 0
        if (!isnan(val)) {
            if (P.clip) val = clipd(val, -1.0, 1.0);
            if (P.as_image) val = (double)(unsigned char)(long long)((clipd(val, -1.0, 1.0) + 1) / 2 * 255);
            f = (float)val;
        }
        out[k] = f;
    }
}

// ------------------------------------------------------------------ TimeToCollision
// road/road.py:231-276 is_connected_road(l1, l2, route, same_lane=False, depth): the two route-following cases are
// tail calls (a loop here); the "all roads at the junction" case branches onto a small explicit stack.
__device__ bool is_connected_road(const GraphShared& g, int f1, int t1, int f2, int t2, const int* route, int rlen,
                                  int depth) {
    struct Item {
        short f, t, ro, d;
    };
    Item stack[24];
    int sp = 0;
    stack[sp++] = Item{(short)f1, (short)t1, 0, (short)depth};
    while (sp > 0) {
        Item it = stack[--sp];
        int f = it.f, t = it.t, ro = it.ro, d = it.d;
        for (;;) {
            if ((f2 == f && t2 == t) || t2 == f) return true;
            if (d <= 0) break;
            if (ro < rlen && RT_FROM(route[ro]) == f && RT_TO(route[ro]) == t) {
                ++ro;
                continue;
            }
            if (ro < rlen && RT_FROM(route[ro]) == t) {
                f = RT_FROM(route[ro]);
                t = RT_TO(route[ro]);
                ++ro;
                --d;
                continue;
            }
            for (int k = 0; k < g.succ_count[t] && sp < 24; ++k)
                stack[sp++] = Item{(short)t, (short)g.lanes[g.succ[t][k]].to_node, (short)ro, (short)(d - 1)};
            break;
        }
    }
    return false;
}

constexpr int kTtcMaxLanes = 8, kTtcMaxT = 64;
typedef int TtcCost2[HWY_MAX_TARGET_SPEEDS][kTtcMaxLanes][kTtcMaxT];  // 2 * cost (0, 1 = 0.5, 2 = 1.0)

// envs/common/finite_mdp.py:104-163 compute_ttc_grid of env e, observed by the vehicle in `ego_slot`, into the
// zeroed shared `cost2` with n_t cells of tq seconds; all lanes of the ego's road (EL).  Called by every thread of
// the block; the caller synchronises before reading cost2.
__device__ void ttc_grid_accumulate(const GraphShared& g, const HwyObsView& view, int e, int count, int ego_slot,
                                    const Veh& ego, const HwyNetLane& EL, int n_speeds, const double* target_speeds,
                                    double tq, int n_t, TtcCost2& cost2) {
    const int n_lanes = EL.road_count;
    double es, ec;
    m_sincos(ego.heading, &es, &ec);
    const double ego_s = lane_s_of(EL, ego.x, ego.y);
    const int* route = view.route ? view.route + ((size_t)e * view.vp + ego_slot) * R : nullptr;
    const int rlen = view.route_len ? view.route_len[(size_t)e * view.vp + ego_slot] : 0;
    for (int s = threadIdx.x; s < count; s += blockDim.x) {
        if (s == ego_slot) continue;
        const Veh o = load_veh(view, e, s);
        if (o.kind == HWY_KIND_OBSTACLE) continue;  // road.vehicles only
        const HwyNetLane& OL = g.lanes[o.lane];
        const bool connected = is_connected_road(g, EL.from_node, EL.to_node, OL.from_node, OL.to_node, route, rlen, 3);
        const double margin = kVehLength / 2 + kVehLength / 2;
        const double base = lane_s_of(EL, o.x, o.y) - ego_s;  // lane_distance_to (vehicle/objects.py:183-198)
        double os, oc;
        m_sincos(o.heading, &os, &oc);
        const double other_projected_speed = o.speed * dot2(oc, os, ec, es);
        for (int si = 0; si < n_speeds; ++si) {
            const double ego_speed = target_speeds[si];
            if (ego_speed == o.speed) continue;
            for (int k = 0; k < 3; ++k) {
                const double m = k == 0 ? 0.0 : (k == 1 ? -margin : margin);
                const double ttc = (base + m) / not_zero(ego_speed - other_projected_speed);
                if (ttc < 0 || !connected) continue;
                int l0 = 0, l1 = n_lanes;
                if (OL.road_count == EL.road_count) {
                    l0 = OL.lane_id;
                    l1 = l0 + 1;
                }
                const int times[2] = {(int)(ttc / tq), (int)ceil(ttc / tq)};
                for (int q = 0; q < 2; ++q) {
                    const int t = times[q];
                    if (0 <= t && t < n_t)
                        for (int l = l0; l < l1 && l < kTtcMaxLanes; ++l) atomicMax(&cost2[si][l][t], k == 0 ? 2 : 1);
                }
            }
        }
    }
}

// compute_ttc_grid + observation.py:128-152 (pad with ones, crop 3 x 3)
__global__ void __launch_bounds__(kThreads)
ttc_kernel(const HwyNetGraph* __restrict__ graph, const __grid_constant__ HwyObsView view,
           const __grid_constant__ HwyTtcParams P, const uint8_t* __restrict__ mask_a,
           const uint8_t* __restrict__ mask_b, float* __restrict__ obs) {
    __shared__ GraphShared g;
    __shared__ TtcCost2 cost2;
    __shared__ int s_ego;
    const int A = view.n_agents > 1 ? view.n_agents : 1;
    const int e = blockIdx.x / A, agent = blockIdx.x % A;
    if (!env_selected(mask_a, mask_b, e)) return;
    stage_graph(g, graph);
    const int tid = threadIdx.x;
    const int count = view.count ? view.count[e] : view.n_vehicles;
    if (tid == 0) s_ego = find_ego(view, e, count, agent);
    for (int k = tid; k < HWY_MAX_TARGET_SPEEDS * kTtcMaxLanes * kTtcMaxT; k += kThreads) (&cost2[0][0][0])[k] = 0;
    __syncthreads();
    const int ego_slot = s_ego;
    const Veh ego = load_veh(view, e, ego_slot);
    const HwyNetLane& EL = g.lanes[ego.lane];
    const int n_speeds = P.n_target_speeds, n_lanes = EL.road_count;
    const double tq = 1.0 / P.policy_frequency;
    const int n_t = (int)(P.horizon / tq);
    ttc_grid_accumulate(g, view, e, count, ego_slot, ego, EL, n_speeds, P.target_speeds, tq, n_t, cost2);
    __syncthreads();
    const int speed_index = view.speed_index ? view.speed_index[(size_t)e * A + agent] : 0;
    float* out = obs + ((size_t)e * A + agent) * (size_t)(9 * n_t);
    for (int k = tid; k < 9 * n_t; k += kThreads) {
        const int a = k / (3 * n_t), b = (k / n_t) % 3, t = k % n_t;
        const int vrow = n_speeds + speed_index - 1 + a;
        int src = vrow < 1 + n_speeds ? 0 : (vrow < 1 + n_speeds + (n_speeds - 2) ? 1 + (vrow - (1 + n_speeds)) : n_speeds - 1);
        if (n_speeds == 1) src = 0;
        const int lcol = n_lanes + EL.lane_id - 1 + b;
        const float val = (lcol < n_lanes || lcol >= 2 * n_lanes) ? 1.0f : 0.5f * (float)cost2[src][lcol - n_lanes][t];
        out[k] = val;
    }
}

// ------------------------------------------------------------------ finite MDP (finite_mdp.py:17-101, 166-203)
// finite_mdp(env, time_quantization=1/policy_frequency, horizon) of every env: the uncropped TTC grid of the first
// controlled vehicle over the n_lanes = road_count lanes of its road, and the deterministic MDP on the raveled
// (speed, lane, time) cells of that grid.  Rows s >= n_states of the [s_max] padding are absorbing: self-loops,
// reward 0, terminal.
__global__ void __launch_bounds__(kThreads)
finite_mdp_kernel(const HwyNetGraph* __restrict__ graph, const __grid_constant__ HwyObsView view,
                  const __grid_constant__ HwyFiniteMdpParams P, double* __restrict__ grid_out,
                  int32_t* __restrict__ n_lanes_out, int32_t* __restrict__ n_states_out, int64_t* __restrict__ state_out,
                  int32_t* __restrict__ transition, double* __restrict__ reward, uint8_t* __restrict__ terminal) {
    __shared__ GraphShared g;
    __shared__ TtcCost2 cost2;
    __shared__ int s_ego;
    const int e = blockIdx.x;
    stage_graph(g, graph);
    const int tid = threadIdx.x;
    const int count = view.count ? view.count[e] : view.n_vehicles;
    if (tid == 0) s_ego = find_ego(view, e, count, 0);
    for (int k = tid; k < HWY_MAX_TARGET_SPEEDS * kTtcMaxLanes * kTtcMaxT; k += kThreads) (&cost2[0][0][0])[k] = 0;
    __syncthreads();
    const int ego_slot = s_ego;
    const Veh ego = load_veh(view, e, ego_slot);
    const HwyNetLane& EL = g.lanes[ego.lane];
    const int V = P.n_target_speeds, T = P.n_t, LM = P.l_max;
    const int L = EL.road_count < LM ? EL.road_count : LM;  // l_max covers every road of the graph (host-checked)
    ttc_grid_accumulate(g, view, e, count, ego_slot, ego, EL, V, P.target_speeds, 1.0 / P.policy_frequency, T, cost2);
    __syncthreads();
    const int S = V * L * T, s_max = V * LM * T;
    if (tid == 0) {
        const int speed_index = view.speed_index ? view.speed_index[e] : 0;
        n_lanes_out[e] = L;
        n_states_out[e] = S;
        state_out[e] = ((long long)speed_index * L + EL.lane_id) * T;  // ravel_multi_index((h, lane_index[2], 0))
    }
    double* ge = grid_out + (size_t)e * s_max;
    for (int k = tid; k < s_max; k += kThreads) {
        const int h = k / (LM * T), l = (k / T) % LM, t = k % T;
        ge[k] = l < L ? 0.5 * cost2[h][l][t] : 0.0;
    }
    // state_reward = (collision * grid + right_lane * lanes) + high_speed * speeds;  reward = state_reward[s] +
    // [lane_change, 0, lane_change, 0, 0][a]  (the reference's operation order; -fmad=false keeps each rounding)
    const double lane_den = (double)(L - 1 > 1 ? L - 1 : 1), speed_den = (double)(V - 1 > 1 ? V - 1 : 1);
    int32_t* tr = transition + (size_t)e * s_max * 5;
    double* rw = reward + (size_t)e * s_max * 5;
    uint8_t* te = terminal + (size_t)e * s_max;
    for (int s = tid; s < s_max; s += kThreads) {
        if (s >= S) {
            for (int a = 0; a < 5; ++a) {
                tr[s * 5 + a] = s;
                rw[s * 5 + a] = 0.0;
            }
            te[s] = 1;
            continue;
        }
        const int h = s / (L * T), i = (s / T) % L, j = s % T;
        const double cell = 0.5 * cost2[h][i][j];
        const double sr = (P.collision_reward * cell + P.right_lane_reward * ((double)i / lane_den)) +
                          P.high_speed_reward * ((double)h / speed_den);
        te[s] = cell == 1.0 || j == T - 1;
        // transition_model / clip_position: every action advances time; LANE_LEFT / LANE_RIGHT move one lane,
        // FASTER / SLOWER one speed only from the first time cell
        const int jn = j + 1 < T ? j + 1 : T - 1;
        const int il = i > 0 ? i - 1 : 0, ir = i + 1 < L ? i + 1 : L - 1;
        const int hf = j == 0 && h + 1 < V ? h + 1 : h, hs = j == 0 && h > 0 ? h - 1 : h;
        const int next[5] = {(h * L + il) * T + jn, (h * L + i) * T + jn, (h * L + ir) * T + jn, (hf * L + i) * T + jn,
                             (hs * L + i) * T + jn};
        for (int a = 0; a < 5; ++a) {
            tr[s * 5 + a] = next[a];
            rw[s * 5 + a] = sr + ((a == 0 || a == 2) ? P.lane_change_reward : 0.0);
        }
    }
}

// ------------------------------------------------------------------ LidarObservation (observation.py:678-769)
// utils.distance_to_rect (utils.py:388-416)
__device__ double distance_to_rect(double rx, double ry, double qx, double qy, const double (&c)[4][2]) {
    double ux = c[1][0] - c[0][0], uy = c[1][1] - c[0][1], vx = c[3][0] - c[0][0], vy = c[3][1] - c[0][1];
    const double un = norm2(ux, uy), vn = norm2(vx, vy);
    ux /= un;
    uy /= un;
    vx /= vn;
    vy /= vn;
    const double rqu = dot2(qx - rx, qy - ry, ux, uy), rqv = dot2(qx - rx, qy - ry, vx, vy);
    double i10 = dot2(c[0][0] - rx, c[0][1] - ry, ux, uy) / rqu, i11 = dot2(c[1][0] - rx, c[1][1] - ry, ux, uy) / rqu;
    double i20 = dot2(c[0][0] - rx, c[0][1] - ry, vx, vy) / rqv, i21 = dot2(c[3][0] - rx, c[3][1] - ry, vx, vy) / rqv;
    if (!(rqu >= 0)) {
        const double t = i10;
        i10 = i11;
        i11 = t;
    }
    if (!(rqv >= 0)) {
        const double t = i20;
        i20 = i21;
        i21 = t;
    }
    if (interval_distance(i10, i11, i20, i21) <= 0 && interval_distance(0.0, 1.0, i10, i11) <= 0 &&
        interval_distance(0.0, 1.0, i20, i21) <= 0)
        return fmax(i10, i20) * norm2(qx - rx, qy - ry);
    return INFINITY;
}

// One thread per (env, agent, cell): trace() visits the obstacles in list order and every cell keeps a running
// (float32!) minimum with `<=`, so a cell's final value only depends on the sequence of candidates for THAT cell.
__global__ void __launch_bounds__(kThreads)
lidar_kernel(const __grid_constant__ HwyObsView view, const __grid_constant__ HwyLidarParams P,
             const uint8_t* __restrict__ mask_a, const uint8_t* __restrict__ mask_b, float* __restrict__ obs) {
    const int A = view.n_agents > 1 ? view.n_agents : 1;
    const int cells = P.cells;
    const long long gid = (long long)blockIdx.x * kThreads + threadIdx.x;
    const long long total = (long long)view.n_envs * A * cells;
    if (gid >= total) return;
    const int cell = (int)(gid % cells);
    const int agent = (int)((gid / cells) % A);
    const int e = (int)(gid / ((long long)cells * A));
    if (!env_selected(mask_a, mask_b, e)) return;
    const int count = view.count ? view.count[e] : view.n_vehicles;
    const int ego_slot = find_ego(view, e, count, agent);
    const Veh ego = load_veh(view, e, ego_slot);
    double es, ec;
    m_sincos(ego.heading, &es, &ec);
    const double ovx = ego.speed * ec, ovy = ego.speed * es;
    const double angle = 2 * kPi / cells;
    const double range = P.maximum_range;
    float dist_f = (float)range, vel_f = (float)range;
    double dirs, dirc;
    m_sincos(cell * angle, &dirs, &dirc);
    // sector of an angle; the angles come from CUDA's atan2, which is not numpy's: within a few ulp of a sector
    // boundary either side is a faithful answer (numpy's own choice there depends on its SIMD dispatch)
    auto to_index = [&](double a) { return (int)py_mod_pos(floor(a / angle), (double)cells); };
    for (int s = 0; s < count; ++s) {
        if (s == ego_slot) continue;
        const Veh o = load_veh(view, e, s);
        const bool is_object = o.kind == HWY_KIND_OBSTACLE;
        const double len = is_object ? 2.0 : kVehLength, wid = 2.0;
        const double center_distance = norm2(o.x - ego.x, o.y - ego.y);
        if (center_distance > range) continue;
        double sh, ch;
        m_sincos(o.heading, &sh, &ch);
        const double vx = is_object ? 0.0 : o.speed * ch, vy = is_object ? 0.0 : o.speed * sh;
        const double rel_v = dot2(vx - ovx, vy - ovy, dirc, dirs);
        const int center_index = to_index(atan2(o.y - ego.y, o.x - ego.x) + angle / 2);
        if (center_index == cell) {
            const double distance = center_distance - wid / 2;
            if (distance <= (double)dist_f) {
                dist_f = (float)distance;
                vel_f = (float)rel_v;
            }
        }
        // utils.rect_corners (utils.py:128-157) and the angular sector they cover
        const double cl[4][2] = {{-len / 2, -wid / 2}, {-len / 2, wid / 2}, {len / 2, wid / 2}, {len / 2, -wid / 2}};
        double corners[4][2], amin = 0, amax = 0;
        for (int k = 0; k < 4; ++k) {
            corners[k][0] = (ch * cl[k][0] + (-sh) * cl[k][1]) + o.x;
            corners[k][1] = (sh * cl[k][0] + ch * cl[k][1]) + o.y;
            const double a = atan2(corners[k][1] - ego.y, corners[k][0] - ego.x) + angle / 2;
            if (k == 0 || a < amin) amin = a;
            if (k == 0 || a > amax) amax = a;
        }
        if (amin < -kPi / 2 && kPi / 2 < amax) {  // the corners wrap around +pi
            const double t = amin;
            amin = amax;
            amax = t + 2 * kPi;
        }
        const int start = to_index(amin), end = to_index(amax);
        // indexes: start..end, or start..cells-1 then 0..end (twice through `start` when start == end)
        int visits = 0;
        if (start < end)
            visits = (start <= cell && cell <= end) ? 1 : 0;
        else
            visits = (cell >= start ? 1 : 0) + (cell <= end ? 1 : 0);
        if (visits) {
            const double d = distance_to_rect(ego.x, ego.y, ego.x + range * dirc, ego.y + range * dirs, corners);
            if (d <= (double)dist_f) {  // a second visit compares the value with itself: no change
                dist_f = (float)d;
                vel_f = (float)rel_v;
            }
        }
    }
    if (P.normalize) {
        dist_f = dist_f / (float)range;
        vel_f = vel_f / (float)range;
    }
    float* out = obs + (((size_t)e * A + agent) * cells + cell) * 2;
    out[0] = dist_f;
    out[1] = vel_f;
}

}  // namespace hwyobs

// ====================================================================== C ABI
namespace {
using hwy_abi::check_launch;
using hwy_abi::fail;

int validate_view(const HwyObsView* v) {
    if (!v) return fail("%s", "null view");
    if (v->n_envs < 1 || v->vp < 1) return fail("%s", "bad view sizes");
    if (!v->pos || !v->hs || !v->meta) return fail("%s", "null state pointer in view");
    if (!v->count && (v->n_vehicles < 1 || v->n_vehicles > v->vp)) return fail("%s", "n_vehicles out of range");
    if (v->n_agents < 0 || v->n_agents > 8) return fail("%s", "n_agents out of range");
    return hwy_abi::require_device();
}
int agents_of(const HwyObsView* v) { return v->n_agents > 1 ? v->n_agents : 1; }
}  // namespace

extern "C" {

int hwy_observe_grid(const HwyNetGraph* graph, const HwyObsView* view, const HwyGridParams* p, const uint8_t* mask_a,
                     const uint8_t* mask_b, float* obs, void* stream) {
    if (validate_view(view)) return 1;
    if (!graph || !p || !obs) return fail("%s", "null pointer");
    if (p->n_features < 1 || p->n_features > HWY_MAX_OBS_FEATURES) return fail("%s", "n_features out of range");
    for (int k = 0; k < p->n_features; ++k)
        if (p->features[k] < 0 || p->features[k] > HWY_FEAT_UNKNOWN) return fail("%s", "unknown grid feature code");
    if (p->shape[0] < 1 || p->shape[1] < 1) return fail("%s", "empty grid");
    const long long cells = (long long)p->shape[0] * p->shape[1];
    const size_t smem = ((sizeof(hwynet::GraphShared) + 15) & ~size_t(15)) + (size_t)cells * 5 + 16;
    if (smem > 200 * 1024) return fail("%s", "OccupancyGrid too large for one block's shared memory (cells <= ~38000)");
    if (!(p->grid_step[0] > 0) || !(p->grid_step[1] > 0)) return fail("%s", "grid_step must be positive");
    if (hwy_abi::opt_in_smem((const void*)hwyobs::grid_kernel, smem)) return 1;
    hwyobs::grid_kernel<<<view->n_envs * agents_of(view), hwyobs::kThreads, smem, (cudaStream_t)stream>>>(
        graph, *view, *p, mask_a, mask_b, obs);
    return check_launch("observe grid_kernel");
}

int hwy_observe_ttc(const HwyNetGraph* graph, const HwyObsView* view, const HwyTtcParams* p, const uint8_t* mask_a,
                    const uint8_t* mask_b, float* obs, void* stream) {
    if (validate_view(view)) return 1;
    if (!graph || !p || !obs) return fail("%s", "null pointer");
    if (p->n_target_speeds < 1 || p->n_target_speeds > HWY_MAX_TARGET_SPEEDS) return fail("%s", "n_target_speeds out of range");
    if (p->policy_frequency < 1 || p->horizon < 1) return fail("%s", "bad horizon / policy_frequency");
    if ((long long)p->horizon * p->policy_frequency > hwyobs::kTtcMaxT) return fail("%s", "horizon * policy_frequency > 64");
    hwyobs::ttc_kernel<<<view->n_envs * agents_of(view), hwyobs::kThreads, 0, (cudaStream_t)stream>>>(
        graph, *view, *p, mask_a, mask_b, obs);
    return check_launch("observe ttc_kernel");
}

int hwy_finite_mdp(const HwyNetGraph* graph, const HwyObsView* view, const HwyFiniteMdpParams* p, double* grid,
                   int32_t* n_lanes, int32_t* n_states, int64_t* state, int32_t* transition, double* reward,
                   uint8_t* terminal, void* stream) {
    if (validate_view(view)) return 1;
    if (!graph || !p || !grid || !n_lanes || !n_states || !state || !transition || !reward || !terminal)
        return fail("%s", "null pointer");
    if (view->n_agents > 1) return fail("%s", "finite MDP of a multi-agent env");
    if (p->n_target_speeds < 1 || p->n_target_speeds > HWY_MAX_TARGET_SPEEDS) return fail("%s", "n_target_speeds out of range");
    if (p->l_max < 1 || p->l_max > hwyobs::kTtcMaxLanes) return fail("%s", "l_max out of range (1..8)");
    if (p->policy_frequency < 1 || !(p->horizon > 0)) return fail("%s", "bad horizon / policy_frequency");
    if (p->n_t != (int)(p->horizon / (1.0 / p->policy_frequency))) return fail("%s", "n_t != int(horizon / (1 / policy_frequency))");
    if (p->n_t < 1 || p->n_t > hwyobs::kTtcMaxT) return fail("%s", "n_t out of range (1..64)");
    hwyobs::finite_mdp_kernel<<<view->n_envs, hwyobs::kThreads, 0, (cudaStream_t)stream>>>(
        graph, *view, *p, grid, n_lanes, n_states, state, transition, reward, terminal);
    return check_launch("finite_mdp_kernel");
}

int hwy_observe_lidar(const HwyObsView* view, const HwyLidarParams* p, const uint8_t* mask_a, const uint8_t* mask_b,
                      float* obs, void* stream) {
    if (validate_view(view)) return 1;
    if (!p || !obs) return fail("%s", "null pointer");
    if (p->cells < 1 || p->cells > 4096) return fail("%s", "cells out of range");
    if (!(p->maximum_range > 0)) return fail("%s", "maximum_range must be positive");
    const long long total = (long long)view->n_envs * agents_of(view) * p->cells;
    const int blocks = (int)((total + hwyobs::kThreads - 1) / hwyobs::kThreads);
    hwyobs::lidar_kernel<<<blocks, hwyobs::kThreads, 0, (cudaStream_t)stream>>>(*view, *p, mask_a, mask_b, obs);
    return check_launch("observe lidar_kernel");
}

}  // extern "C"
