// hwy_network.cu — sm_90a kernels + C ABI for envs on a GENERAL road network: roundabout-v0|v1, merge-v0|v1,
// two-way-v0, u-turn-v0|v1 (8 vehicle slots per env) and intersection-v0|v2, intersection-multi-agent-v0|v1|v2
// (16 / 32 slots, RegulatedRoad, a population that changes every step).
// StraightLane / SineLane / CircularLane geometry, planned routes with RoadNetwork.next_lane, IDM + MOBIL with the
// route branch, all-pairs SAT collisions incl. road objects (Obstacle), connected-lane neighbour search, Kinematics /
// TimeToCollision / OccupancyGrid observations, the scenarios' rewards, and their resets on the env's numpy stream.
//
// Thread mapping: template <int G, bool REG> — G threads per env (vehicle slot = thread), 256-thread blocks; the
// groups of a block advance through the phases of a substep together (block-wide `barrier.sync`): the kernels are
// several times the instruction cache, and warps left to drift apart stalled on instruction fetch.
//  * Each vehicle's local coordinates on its own lane are computed once per substep and reused by every query.
//  * Vehicle.on_state_update's get_closest_lane_index over ALL lanes (47 % of the reference's step on networks) is
//    pruned exactly by a lateral lower bound; the surviving (vehicle, lane) pairs form a work list for the group.
//  * Road.act's Gauss-Seidel part: follow_road runs for all vehicles at once; only vehicles whose lane-change
//    policy can read or move a target lane take turns in list order.
//  * Steering, IDM acceleration, integration and the collision sweep run one vehicle per thread.
// The lane table lives in HBM (HwyNetGraph) and is staged into shared memory once per block.  DESIGN.md 3.5-3.9.
//
// Reference paths are relative to /root/reference/highway_env.
#include <atomic>
#include <cstdio>
#include <mutex>

#include <cuda_runtime.h>

#include "../../include/hwyb200.h"
#include "hwy_abi.h"
#include "hwy_device.cuh"
#include "hwy_math.cuh"
#include "hwy_lanes.cuh"

namespace hwynet {
using namespace hwy;

constexpr int R = HWY_NET_MAX_ROUTE;
constexpr int kBlockThreads = 256;  // observe / substeps / debug kernels
// The step kernels run ONE block per SM (128 registers x 512 threads): one instruction stream per SM.  The step body is
// ~110 KB of SASS against a much smaller instruction cache, and two co-resident blocks in different phases evict each
// other: 512 x 1 was faster than 256 x 2 (same warps per SM) and 128 x 4.  The
// launch uses fewer threads per block when that spreads the envs over all SMs (step_plan).
#ifndef HWY_NET_STEP_THREADS
#define HWY_NET_STEP_THREADS 512
#endif
constexpr int kStepThreads = HWY_NET_STEP_THREADS;
constexpr int kPred = 11;  // np.arange(0.25, 3, 0.25) prediction points of RegulatedRoad.is_conflict_possible
constexpr int kPredChunk = 4;  // horizon points staged in shared memory at a time

template <int G>
__host__ __device__ constexpr int kCand() {
    return G >= 32 ? 48 : 40;
}

// Per-env shared staging for G vehicle slots.  REG adds the RegulatedRoad prediction buffers.
template <int G, bool REG>
struct EnvStage {
    double x[G], y[G], heading[G], c[G], s[G], v[G], ts[G];
    int lane[G], tgt[G], kind[G];
    int tgt_prev[G];  // target lanes before the current Road.act (Gauss-Seidel view of later vehicles)
    int route[G][R];
    int route_len[G];
    int count, ego, speed_index, road_steps;
    unsigned agent_mask;    // the controlled (MDP) vehicles among the first `count` slots, list order = agent order
    double agent_reward[4];  // per-agent rewards of the step (MultiAgent: summed in agent order)
    double agent_terms[4][4];  // per-agent _agent_rewards terms (collision, high_speed, arrived, on_road)
    unsigned yield_mask;
    // spawn record (dynamic population): written by the group's first thread, adopted by the new slot
    double sp_x, sp_y, sp_h, sp_speed, sp_delta, sp_ts;
    int sp_ok, sp_lane, sp_dest, sp_kind;
    double key[G];
    // local coordinates of every vehicle on its OWN lane (st.lane), refreshed together with the lane index:
    // what local_coordinates() returns for (vehicle.lane, vehicle.position), reused by every query on that lane
    double own_s[G], own_lat[G];
    int n_cand;
    union {
        double ttc[3][4][16];  // TimeToCollision grid [speed][lane on road][time] (u-turn-v0: 16 s horizon)
        struct {
            int owner[121];           // OccupancyGrid: lowest vehicle index in the cell
            unsigned char road[121];  // on_road layer
        } cells;
        struct {  // closest-lane search: (vehicle, lane) pairs that survive the lateral lower bound
            double d[kCand<G>()], s[kCand<G>()], lat[kCand<G>()];
            unsigned short vl[kCand<G>()];
        } cand;
    } o;
    // RegulatedRoad: predicted (x, y, heading) of every vehicle at kPredChunk horizon points at a time
    double pred[REG ? G : 1][REG ? kPredChunk : 1][3];
};

// road/road.py:138-157 next_lane_given_next_road (next_id < 0 == None)
__device__ __forceinline__ int next_lane_given_next_road(const GraphShared& g, int cur, int next_first,
                                                         int next_id, double px, double py, double& dist) {
    const HwyNetLane& C = g.lanes[cur];
    int n_next = g.lanes[next_first].road_count;
    if (C.road_count == n_next) {
        if (next_id < 0) next_id = C.lane_id;
    } else {
        int best = 0;
        double bd = 0;
        for (int l = 0; l < n_next; ++l) {
            double d = lane_distance(g.lanes[next_first + l], px, py);
            if (l == 0 || d < bd) {
                bd = d;
                best = l;
            }
        }
        next_id = best;
    }
    dist = lane_distance(g.lanes[next_first + next_id], px, py);
    return next_id;
}

// road/road.py:73-136 next_lane: pops the vehicle's route in place
template <int G, bool REG>
__device__ __noinline__ int next_lane(const GraphShared& g, EnvStage<G, REG>& st, int v, int cur) {
    const HwyNetLane& C = g.lanes[cur];
    int* route = st.route[v];
    int rlen = st.route_len[v];
    int next_first = -1, next_id = -1;
    if (rlen > 0) {
        if (RT_FROM(route[0]) == C.from_node && RT_TO(route[0]) == C.to_node) {
            for (int k = 1; k < rlen; ++k) route[k - 1] = route[k];
            --rlen;
            st.route_len[v] = rlen;
        }
        if (rlen > 0 && RT_FROM(route[0]) == C.to_node) {
            next_first = road_first(g, RT_FROM(route[0]), RT_TO(route[0]));
            next_id = RT_ID(route[0]);
        }
    }
    double lon, lat, px, py;
    lane_local(C, st.x[v], st.y[v], lon, lat);
    lane_position(C, lon, 0.0, px, py);
    if (next_first < 0) {
        int n_succ = g.succ_count[C.to_node];
        if (n_succ == 0) return cur;  // KeyError on graph[_to]: keep the current lane
        int best = -1;
        double bd = 0;
        for (int k = 0; k < n_succ; ++k) {
            int nf = g.succ[C.to_node][k];
            double d;
            int nid = next_lane_given_next_road(g, cur, nf, next_id, px, py, d);
            if (k == 0 || d < bd) {
                bd = d;
                best = nf + nid;
            }
        }
        return best;
    }
    double d;
    next_id = next_lane_given_next_road(g, cur, next_first, next_id, px, py, d);
    return next_first + next_id;
}

// vehicle/controller.py:135-143 follow_road
template <int G, bool REG>
__device__ __forceinline__ void follow_road(const GraphShared& g, EnvStage<G, REG>& st, int v) {
    const HwyNetLane& T = g.lanes[st.tgt[v]];
    const double s = st.tgt[v] == st.lane[v] ? st.own_s[v] : lane_s_of(T, st.x[v], st.y[v]);
    if (s > T.length - kLaneVehLength / 2)  // after_end (lane.py:120-125)
        st.tgt[v] = next_lane(g, st, v, st.tgt[v]);
}

// road/road.py:483-547 neighbour_vehicles.  `connected` = config["neighbour_vehicles_connected_lanes"]
// (ConnectedLaneNeighboursMixin, abstract.py:26-37; road.py:509-529): the lanes continuing `lane_idx` (every road
// leaving its end node: lane _id, or lane 0 when that road has fewer lanes) are searched with offset +length and
// the lanes leading into its start node (from-nodes in graph order = table order) with offset -their length; a
// vehicle counts on the FIRST lane of that list it is on.
template <int G, bool REG>
__device__ __noinline__ void neighbours(const GraphShared& g, const EnvStage<G, REG>& st, int V, int veh,
                                        int lane_idx, bool connected, int& front, int& rear) {
    constexpr int kMaxSearch = 16;
    const HwyNetLane& L = g.lanes[lane_idx];
    const double s = lane_idx == st.lane[veh] ? st.own_s[veh] : lane_s_of(L, st.x[veh], st.y[veh]);
    if (!connected) {  // same-segment search: one lane, no list
        double s_front = 0, s_rear = 0;
        front = -1;
        rear = -1;
        // The reference scans the vehicles in list order: the front neighbour is the smallest s_v >= s with ties going
        // to the LATER vehicle (`<=`), the rear one the largest s_v < s with ties going to the EARLIER vehicle (`>`).
        // Stated as an order on (s_v, index) the scan can be split: vehicles on the query lane use their cached
        // coordinates at once; the others take the sqrt / atan2 / sin-free pre-test (lane_maybe_on) and only the
        // survivors — gathered in a mask so that the lanes of a warp evaluate theirs together — get exact coordinates.
        unsigned pending = 0;
        for (int v = 0; v < V; ++v) {
            if (v == veh) continue;
            if (st.lane[v] != lane_idx) {
                if (lane_maybe_on(L, st.x[v], st.y[v])) pending |= 1u << v;
                continue;
            }
            const double s_v = st.own_s[v];
            if (!lane_on(L, s_v, st.own_lat[v], 1.0)) continue;
            if (s <= s_v && (front < 0 || s_v < s_front || (s_v == s_front && v > front))) {
                s_front = s_v;
                front = v;
            }
            if (s_v < s && (rear < 0 || s_v > s_rear || (s_v == s_rear && v < rear))) {
                s_rear = s_v;
                rear = v;
            }
        }
        while (pending) {
            const int v = __ffs(pending) - 1;
            pending &= pending - 1;
            double s_v, lat_v;
            lane_local(L, st.x[v], st.y[v], s_v, lat_v);
            if (!lane_on(L, s_v, lat_v, 1.0)) continue;
            if (s <= s_v && (front < 0 || s_v < s_front || (s_v == s_front && v > front))) {
                s_front = s_v;
                front = v;
            }
            if (s_v < s && (rear < 0 || s_v > s_rear || (s_v == s_rear && v < rear))) {
                s_rear = s_v;
                rear = v;
            }
        }
        return;
    }
    unsigned char lanes[kMaxSearch];
    int n_l = 1;
    lanes[0] = (unsigned char)lane_idx;
    int n_next = 0;
    if (connected) {
        for (int k = 0; k < g.succ_count[L.to_node] && n_l < kMaxSearch; ++k) {
            const int f = g.succ[L.to_node][k];
            lanes[n_l++] = (unsigned char)(f + (L.lane_id < g.lanes[f].road_count ? L.lane_id : 0));
        }
        n_next = n_l - 1;
        for (int l = 0; l < g.n_lanes && n_l < kMaxSearch; ++l) {
            const HwyNetLane& P0 = g.lanes[l];
            if (P0.lane_id != 0 || P0.to_node != L.from_node) continue;
            lanes[n_l++] = (unsigned char)(l + (L.lane_id < P0.road_count ? L.lane_id : 0));
        }
    }
    double s_front = 0, s_rear = 0;
    front = -1;
    rear = -1;
    for (int v = 0; v < V; ++v) {
        if (v == veh) continue;
        for (int k = 0; k < n_l; ++k) {
            const int sl = lanes[k];
            const HwyNetLane& SL = g.lanes[sl];
            double s_v, lat_v;
            if (st.lane[v] == sl) {
                s_v = st.own_s[v];
                lat_v = st.own_lat[v];
            } else {
                if (!lane_maybe_on(SL, st.x[v], st.y[v])) continue;  // on_lane(margin=1) cannot hold
                lane_local(SL, st.x[v], st.y[v], s_v, lat_v);
            }
            if (!lane_on(SL, s_v, lat_v, 1.0)) continue;
            if (k > 0) s_v += k <= n_next ? L.length : -SL.length;
            if (s <= s_v && (front < 0 || s_v <= s_front)) {
                s_front = s_v;
                front = v;
            }
            if (s_v < s && (rear < 0 || s_v > s_rear)) {
                s_rear = s_v;
                rear = v;
            }
            break;  // matched on this lane
        }
    }
}

template <int G, bool REG>
__device__ __forceinline__ double lane_distance_to(const GraphShared& g, const EnvStage<G, REG>& st, int self,
                                                   int other) {
    const HwyNetLane& L = g.lanes[st.lane[self]];
    const double s_other = st.lane[other] == st.lane[self] ? st.own_s[other] : lane_s_of(L, st.x[other], st.y[other]);
    return s_other - st.own_s[self];
}
// vehicle/behavior.py:192-217
template <int G, bool REG>
__device__ __forceinline__ double desired_gap(const HwyNetParams& P, const EnvStage<G, REG>& st, int ego, int front) {
    double ab = -P.comfort_acc_max * P.comfort_acc_min;
    double dvx = st.v[ego] * st.c[ego] - st.v[front] * st.c[front];
    double dvy = st.v[ego] * st.s[ego] - st.v[front] * st.s[front];
    double dv = dot2(dvx, dvy, st.c[ego], st.s[ego]);
    return P.distance_wanted + st.v[ego] * P.time_wanted + st.v[ego] * dv / (2 * sqrt(ab));
}
// vehicle/behavior.py:150-190 with the caller's DELTA
template <int G, bool REG>
__device__ __noinline__ double idm_acceleration(const HwyNetParams& P, const GraphShared& g,
                                                const EnvStage<G, REG>& st, double delta, int ego, int front) {
    if (ego < 0 || st.kind[ego] == HWY_KIND_OBSTACLE) return 0.0;  // `not isinstance(ego_vehicle, Vehicle)`
    double ego_target_speed = clipd(st.ts[ego], 0.0, g.lanes[st.lane[ego]].speed_limit);
    double acc = P.comfort_acc_max *
                 (1 - idm_pow(fmax(st.v[ego], 0.0) / fabs(not_zero(ego_target_speed)), delta));
    if (front >= 0) {
        double d = lane_distance_to(g, st, ego, front);
        double q = desired_gap(P, st, ego, front) / not_zero(d);
        acc -= P.comfort_acc_max * (q * q);
    }
    return acc;
}

__device__ __forceinline__ int isign(int a) { return (a > 0) - (a < 0); }
// env.controlled_vehicles: MDPVehicle (DiscreteMetaAction) or a plain Vehicle / BicycleVehicle (ContinuousAction)
__device__ __forceinline__ bool is_controlled_kind(int kind) { return kind == HWY_KIND_MDP || kind == HWY_KIND_VEHICLE; }

// vehicle/behavior.py:265-324 mobil(lane_index), incl. the planned-route branch
template <int G, bool REG>
__device__ __noinline__ bool mobil(const HwyNetParams& P, const GraphShared& g, const EnvStage<G, REG>& st, int V,
                                   int v, double delta, int lane_index) {
    int new_preceding, new_following;
    neighbours(g, st, V, v, lane_index, P.connected_lanes != 0, new_preceding, new_following);
    double new_following_pred_a = idm_acceleration(P, g, st, delta, new_following, v);
    if (new_following_pred_a < -P.lane_change_max_braking_imposed) return false;
    int old_preceding, old_following;
    neighbours(g, st, V, v, st.lane[v], P.connected_lanes != 0, old_preceding, old_following);
    double self_pred_a = idm_acceleration(P, g, st, delta, v, new_preceding);
    if (st.route_len[v] > 0 && RT_ID(st.route[v][0]) >= 0) {
        int tid = g.lanes[st.tgt[v]].lane_id, cid = g.lanes[lane_index].lane_id;
        if (isign(cid - tid) != isign(RT_ID(st.route[v][0]) - tid)) return false;  // wrong direction
        if (self_pred_a < -P.lane_change_max_braking_imposed) return false;
    } else {
        double self_a = idm_acceleration(P, g, st, delta, v, old_preceding);
        double jerk = self_pred_a - self_a;
        if (P.politeness != 0.0) {
            double new_following_a = idm_acceleration(P, g, st, delta, new_following, new_preceding);
            double old_following_a = idm_acceleration(P, g, st, delta, old_following, v);
            double old_following_pred_a = idm_acceleration(P, g, st, delta, old_following, old_preceding);
            jerk = self_pred_a - self_a + P.politeness * (new_following_pred_a - new_following_a +
                                                          old_following_pred_a - old_following_a);
        }
        if (jerk < P.lane_change_min_acc_gain) return false;
    }
    return true;
}

// vehicle/behavior.py:219-263 change_lane_policy; returns the (possibly reset) timer
template <int G, bool REG>
__device__ __forceinline__ double change_lane_policy(const HwyNetParams& P, const GraphShared& g,
                                                     EnvStage<G, REG>& st, int V, int v, double delta,
                                                     double timer) {
    const int lane = st.lane[v];
    if (lane != st.tgt[v]) {
        const HwyNetLane &A = g.lanes[lane], &B = g.lanes[st.tgt[v]];
        if (A.from_node == B.from_node && A.to_node == B.to_node) {
            for (int o = 0; o < V; ++o) {
                // vehicles later in the list have not acted yet: their target lane of before this Road.act
                const int tgt_o = o < v ? st.tgt[o] : st.tgt_prev[o];
                if (o != v && st.lane[o] != st.tgt[v] && tgt_o == st.tgt[v]) {
                    double d = lane_distance_to(g, st, v, o);
                    double d_star = desired_gap(P, st, v, o);
                    if (0 < d && d < d_star) {
                        st.tgt[v] = lane;
                        break;
                    }
                }
            }
        }
        return timer;
    }
    if (!(P.lane_change_delay < timer)) return timer;
    const HwyNetLane& A = g.lanes[lane];
    for (int k = 0; k < 2; ++k) {  // side_lanes: id-1 then id+1 (road/road.py:200-211)
        if (k == 0 && !(A.lane_id > 0)) continue;
        if (k == 1 && !(A.lane_id < A.road_count - 1)) continue;
        int cand = k == 0 ? lane - 1 : lane + 1;
        if (!lane_reachable(g.lanes[cand], st.x[v], st.y[v])) continue;
        if (fabs(st.v[v]) < 1) continue;
        if (mobil(P, g, st, V, v, delta, cand)) st.tgt[v] = cand;
    }
    return 0.0;
}

// vehicle/controller.py:145-187 steering_control up to the argument of the last arcsin
__device__ __noinline__ double steering_sin_slip(const HwyNetLane& L, double lc_s, double lc_lat, double heading,
                                                 double speed) {
    double lane_future_heading = lane_heading_at(L, lc_s + speed * kTauPursuit);
    double lateral_speed_command = -kKpLateral * lc_lat;
    double heading_command = m_asin(clipd(div_finite(lateral_speed_command, not_zero(speed)), -1.0, 1.0));
    double heading_ref = lane_future_heading + clipd(heading_command, -kPi / 4, kPi / 4);
    double heading_rate_command = kKpHeading * wrap_to_pi(heading_ref - heading);
    return clipd(kVehLength / 2 / not_zero(speed) * heading_rate_command, -1.0, 1.0);
}

__device__ __forceinline__ int speed_to_index(const HwyNetParams& P, double speed) {
    int n = P.n_target_speeds;
    double x = (speed - P.target_speeds[0]) / (P.target_speeds[n - 1] - P.target_speeds[0]);
    return (int)clipd(rint(x * (n - 1)), 0.0, (double)(n - 1));
}

// group-wide helpers (G consecutive lanes of a warp)
template <int G>
__device__ __forceinline__ unsigned group_mask() {
    return G == 32 ? 0xffffffffu : (((1u << (G & 31)) - 1u) << ((threadIdx.x & 31) & ~(G - 1)));
}
template <int G>
__device__ __forceinline__ void group_sync() {
    __syncwarp(group_mask<G>());
}
// Block-wide variant for the unconditional phase boundaries of a substep.  Only the G threads of an env exchange
// data, but the kernels' code is several times the 32 KB instruction cache: keeping the block's warps in the same
// phase lets them share the fetched lines instead of each streaming the whole body (stall_no_instruction).
template <int G>
__device__ __forceinline__ void phase_sync() {
#ifdef HWY_NET_WARP_PHASES
    __syncwarp(group_mask<G>());
#else
    // NOT __syncthreads(): that is barrier.sync.ALIGNED, which requires the whole warp to arrive converged — the
    // compiler does not guarantee that here (per-vehicle branches around the call sites; synccheck flagged it).
    // The unaligned form counts threads individually and is also the intra-group memory fence the callers need.
    asm volatile("barrier.sync 0;" ::: "memory");
#endif
}

// road/road.py:55-71 get_closest_lane_index for every vehicle of the group; also refreshes the own-lane
// coordinate cache.  np.argmin over distance_with_heading of all lanes keeps the FIRST minimum.  Exact pruning:
// the distance to the lane the vehicle was on is an upper bound of the minimum, and
// distance_with_heading >= |lateral offset| (all its terms are >= 0 and rounding is monotone), so a lane whose
// |lateral| — no atan2 needed — exceeds that bound can never win.  The surviving (vehicle, lane) pairs go to a
// shared work list that the whole group evaluates, then every vehicle reduces its own entries by (d, lane).
template <int G, bool REG>
__device__ __forceinline__ void closest_lane_group(const GraphShared& g, EnvStage<G, REG>& st, int V, int i,
                                                   bool mobile) {
    const bool active = i < V && mobile;  // a road object keeps the lane it was created on
    constexpr int K = kCand<G>();
    double x = 0, y = 0, h = 0, bd = 0, bs = 0, blat = 0;
    int bl = 0;
    if (i == 0) st.n_cand = 0;
    if (active) {
        x = st.x[i];
        y = st.y[i];
        h = st.heading[i];
        bl = st.lane[i];
        bd = lane_distance_with_heading(g.lanes[bl], x, y, h, bs, blat);
    }
    // (this barrier and the one that ends the function are not needed for memory ordering — n_cand could be re-armed in
    // the reduce phase and nothing after the function reads another vehicle's lane before the next barrier — but removing
    // them was slower: the block-wide barriers keep the block's warps on the same instruction-cache lines)
    phase_sync<G>();
    if (active) {
        const int hint = bl;
        CircleCache cc = {0.0, 0.0, 0.0, false};
        for (int l = 0; l < g.n_lanes; ++l) {
            if (l == hint) continue;
            const HwyNetLane& L = g.lanes[l];
            if (closest_lane_prunable(L, x, y, bd, cc)) continue;
            int slot = atomicAdd(&st.n_cand, 1);
            if (slot < K) {
                st.o.cand.vl[slot] = (unsigned short)((i << 8) | l);
            } else {  // list full: evaluate in place
                double s_, r_;
                double d = lane_distance_with_heading(L, x, y, h, s_, r_);
                if (d < bd || (d == bd && l < bl)) {
                    bd = d;
                    bl = l;
                    bs = s_;
                    blat = r_;
                }
            }
        }
    }
    phase_sync<G>();
    const int n = min(st.n_cand, K);
    for (int p = i; p < n; p += G) {
        const int v = st.o.cand.vl[p] >> 8, l = st.o.cand.vl[p] & 0xff;
        st.o.cand.d[p] = lane_distance_with_heading(g.lanes[l], st.x[v], st.y[v], st.heading[v], st.o.cand.s[p],
                                                    st.o.cand.lat[p]);
    }
    phase_sync<G>();
    if (active) {
        for (int p = 0; p < n; ++p) {
            const int vl = st.o.cand.vl[p];
            if ((vl >> 8) != i) continue;
            const int l = vl & 0xff;
            const double d = st.o.cand.d[p];
            if (d < bd || (d == bd && l < bl)) {
                bd = d;
                bl = l;
                bs = st.o.cand.s[p];
                blat = st.o.cand.lat[p];
            }
        }
        st.lane[i] = bl;
        st.own_s[i] = bs;
        st.own_lat[i] = blat;
    }
    phase_sync<G>();
}

// ------------------------------------------------------------------ observations
// road/road.py:231-276 is_connected_road(l1, l2, route, same_lane=False, depth).  The two
// route-following cases are tail calls (a loop here); the "all roads at the intersection" case
// branches, so pending (road, route offset, depth) items sit on a small explicit stack.
__device__ __noinline__ bool is_connected_road(const GraphShared& g, int f1, int t1, int f2, int t2,
                                               const int* route, int rlen, int depth) {
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
            if ((f2 == f && t2 == t) || t2 == f) return true;  // is_same_road or is_leading_to_road
            if (d <= 0) break;
            if (ro < rlen && RT_FROM(route[ro]) == f && RT_TO(route[ro]) == t) {
                ++ro;  // route starts at the current road: skip it
                continue;
            }
            if (ro < rlen && RT_FROM(route[ro]) == t) {
                f = RT_FROM(route[ro]);  // route continues from the current road: follow it
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

// envs/common/finite_mdp.py:104-163 compute_ttc_grid + observation.py:128-152 (pad / crop)
template <int G, bool REG>
__device__ __forceinline__ void observe_ttc(const HwyNetParams& P, const GraphShared& g, EnvStage<G, REG>& st,
                                            int V, int i, int speed_index, float* __restrict__ obs_env) {
    const int ego = st.ego;
    const HwyNetLane& EL = g.lanes[st.lane[ego]];
    const int n_speeds = P.n_target_speeds, n_lanes = EL.road_count;
    const double tq = 1.0 / P.policy_frequency;
    const int n_t = (int)(P.ttc_horizon / tq);
    for (int k = i; k < 3 * 4 * 16; k += G) (&st.o.ttc[0][0][0])[k] = 0.0;
    group_sync<G>();
    if (i != ego && i < V && st.kind[i] != HWY_KIND_OBSTACLE) {  // one thread per other VEHICLE; cells take the max cost
        const int o = i;
        const HwyNetLane& OL = g.lanes[st.lane[o]];
        const bool connected = is_connected_road(g, EL.from_node, EL.to_node, OL.from_node, OL.to_node,
                                                 st.route[ego], st.route_len[ego], 3);
        const double margin = kVehLength / 2 + kVehLength / 2;
        const double base = lane_distance_to(g, st, ego, o);
        const double other_projected_speed = st.v[o] * dot2(st.c[o], st.s[o], st.c[ego], st.s[ego]);
        for (int si = 0; si < n_speeds; ++si) {
            const double ego_speed = P.target_speeds[si];
            if (ego_speed == st.v[o]) continue;
            for (int k = 0; k < 3; ++k) {
                const double m = k == 0 ? 0.0 : (k == 1 ? -margin : margin);
                const double cost = k == 0 ? 1.0 : 0.5;
                double ttc = (base + m) / not_zero(ego_speed - other_projected_speed);
                if (ttc < 0 || !connected) continue;
                int l0 = 0, l1 = n_lanes;
                if (OL.road_count == EL.road_count) {
                    l0 = OL.lane_id;
                    l1 = l0 + 1;
                }
                int times[2] = {(int)(ttc / tq), (int)ceil(ttc / tq)};
                for (int q = 0; q < 2; ++q) {
                    int t = times[q];
                    if (0 <= t && t < n_t)
                        for (int l = l0; l < l1; ++l)  // positive doubles order like their bit patterns
                            atomicMax(reinterpret_cast<unsigned long long*>(&st.o.ttc[si][l][t]),
                                      (unsigned long long)__double_as_longlong(cost));
                }
            }
        }
    }
    group_sync<G>();
    const int ego_lane_id = EL.lane_id;
    for (int k = i; k < 9 * n_t; k += G) {
        int a = k / (3 * n_t), b = (k / n_t) % 3, t = k % n_t;
        int vrow = n_speeds + speed_index - 1 + a;
        int src = vrow < 1 + n_speeds ? 0 : (vrow < 1 + n_speeds + (n_speeds - 2) ? 1 + (vrow - (1 + n_speeds)) : n_speeds - 1);
        if (n_speeds == 1) src = 0;
        int lcol = n_lanes + ego_lane_id - 1 + b;
        double val = (lcol < n_lanes || lcol >= 2 * n_lanes) ? 1.0 : st.o.ttc[src][lcol - n_lanes][t];
        obs_env[k] = (float)val;
    }
}

// envs/common/observation.py:234-276 with explicit features_range (absolute or relative);
// F = 5 (presence, x, y, vx, vy) or 7 (+ cos_h, sin_h, vehicle/kinematics.py:247-248)
template <int G, bool REG>
__device__ __forceinline__ void observe_kinematics(const HwyNetParams& P, const GraphShared& g,
                                                   EnvStage<G, REG>& st, int V, int i,
                                                   float* __restrict__ obs_env) {
    const int K = P.obs_vehicles_count, F = P.obs_n_feat > 0 ? P.obs_n_feat : (P.obs_features == 7 ? 7 : 5);
    const int ego = st.ego;
    const double ex = st.x[ego], ey = st.y[ego];
    const double evx = st.v[ego] * st.c[ego], evy = st.v[ego] * st.s[ego];
    double key = INFINITY;
    if (i != ego && i < V) {
        bool ok = norm2(st.x[i] - ex, st.y[i] - ey) < P.perception_distance;
        double d = lane_distance_to(g, st, ego, i);
        // close_objects_to (road/road.py:421-450): obstacles are always filtered like see_behind=False
        ok = ok && ((P.obs_see_behind && st.kind[i] != HWY_KIND_OBSTACLE) || -2 * kVehLength < d);
        if (ok) key = fabs(d);
    }
    st.key[i] = key;
    group_sync<G>();
    int rank = 0, n_valid = 0;
    for (int u = 0; u < V; ++u) {
        double ku = st.key[u];
        n_valid += ku < INFINITY;
        rank += (ku < key) || (ku == key && u < i);
    }
    int row = -1;
    double r1 = 0, r2 = 0, r3 = 0, r4 = 0;
    if (i == ego && i < V) {
        row = 0;
        r1 = ex;
        r2 = ey;
        r3 = evx;
        r4 = evy;
        // ExitObservation.observe (observation.py:632-636): ego_dict["x"] = exit_lane.local_coordinates(position)[0]
        if (P.obs_exit_lane > 0) r1 = lane_s_of(g.lanes[P.obs_exit_lane], ex, ey);
    } else if (key < INFINITY && rank < K - 1) {
        row = rank + 1;
        r1 = st.x[i];
        r2 = st.y[i];
        r3 = st.v[i] * st.c[i];
        r4 = st.v[i] * st.s[i];
        if (!P.obs_absolute) {
            r1 -= ex;
            r2 -= ey;
            r3 -= evx;
            r4 -= evy;
        }
    }
    if (row >= 0 && P.obs_n_feat > 0) {
        // configured column list (any Vehicle.to_dict key, vehicle/kinematics.py:237-261) with per-column ranges
        // (normalize_obs, observation.py:207-232); road objects lack the vehicle-only columns (NaN in the frame -> 0)
        const int NF = P.obs_n_feat;
        const bool object = st.kind[i] == HWY_KIND_OBSTACLE;
        const HwyNetLane& L = g.lanes[st.lane[i]];
        float* o = obs_env + NF * row;
        for (int col = 0; col < NF; ++col) {
            double v = 0.0;
            switch (P.obs_feat[col]) {
                case HWY_FEAT_PRESENCE: v = 1.0; break;
                case HWY_FEAT_X: v = r1; break;
                case HWY_FEAT_Y: v = r2; break;
                case HWY_FEAT_VX: v = object ? r3 - st.v[i] * st.c[i] : r3; break;  // objects: vx = vy = 0 (objects.py:146)
                case HWY_FEAT_VY: v = object ? r4 - st.v[i] * st.s[i] : r4; break;
                case HWY_FEAT_HEADING: v = object ? 0.0 : st.heading[i]; break;
                case HWY_FEAT_COS_H: v = st.c[i]; break;
                case HWY_FEAT_SIN_H: v = st.s[i]; break;
                case HWY_FEAT_LONG_OFF: v = object ? 0.0 : st.own_s[i]; break;  // Vehicle.lane_offset (:228-235)
                case HWY_FEAT_LAT_OFF: v = object ? 0.0 : st.own_lat[i]; break;
                case HWY_FEAT_ANG_OFF: v = object ? 0.0 : wrap_to_pi(st.heading[i] - lane_heading_at(L, st.own_s[i])); break;
                default: v = 0.0; break;  // cos_d / sin_d with observe_intentions=False (the only supported setting)
            }
            if (P.obs_normalize && P.obs_feat_ranged[col]) {
                v = lmap(v, P.obs_feat_lo[col], P.obs_feat_hi[col], -1.0, 1.0);
                if (P.obs_clip) v = clipd(v, -1.0, 1.0);
            }
            o[col] = (float)v;
        }
    } else if (row >= 0) {
        if (P.obs_normalize) {
            r1 = lmap(r1, P.obs_x_lo, P.obs_x_hi, -1.0, 1.0);
            r2 = lmap(r2, P.obs_y_lo, P.obs_y_hi, -1.0, 1.0);
            r3 = lmap(r3, P.obs_vx_lo, P.obs_vx_hi, -1.0, 1.0);
            r4 = lmap(r4, P.obs_vy_lo, P.obs_vy_hi, -1.0, 1.0);
            if (P.obs_clip) {
                r1 = clipd(r1, -1.0, 1.0);
                r2 = clipd(r2, -1.0, 1.0);
                r3 = clipd(r3, -1.0, 1.0);
                r4 = clipd(r4, -1.0, 1.0);
            }
        }
        float* o = obs_env + F * row;
        o[0] = 1.0f;
        o[1] = (float)r1;
        o[2] = (float)r2;
        o[3] = (float)r3;
        o[4] = (float)r4;
        if (F == 7) {
            o[5] = (float)st.c[i];
            o[6] = (float)st.s[i];
        }
    }
    int filled = 1 + (n_valid < K - 1 ? n_valid : K - 1);
    for (int k = i; k < K; k += G)
        if (k >= filled)
            for (int f = 0; f < F; ++f) obs_env[F * k + f] = 0.0f;
}

// envs/common/observation.py:354-484 OccupancyGridObservation.observe with the defaults of :282-284
// (presence, vx, vy, on_road; 11 x 11 cells of 5 m; world axes; relative to the observer)
template <int G, bool REG>
__device__ __forceinline__ void observe_occupancy(const HwyNetParams& P, const GraphShared& g,
                                                  EnvStage<G, REG>& st, int V, int i,
                                                  float* __restrict__ obs_env) {
    const int ego = st.ego;
    const double lo = -5.5 * 5, step = 5;
    const double ex = st.x[ego], ey = st.y[ego];
    const double evx = st.v[ego] * st.c[ego], evy = st.v[ego] * st.s[ego];
    for (int k = i; k < 121; k += G) {
        st.o.cells.owner[k] = 0x7fffffff;
        st.o.cells.road[k] = 0;
    }
    group_sync<G>();
    int cell = -1;
    if (i < V) {  // vehicles are written in REVERSED list order: the lowest index owns a shared cell
        double x = st.x[i] - ex, y = st.y[i] - ey;
        int ci = (int)floor((x - lo) / step), cj = (int)floor((y - lo) / step);
        if (0 <= ci && ci < 11 && 0 <= cj && cj < 11) {
            cell = ci * 11 + cj;
            atomicMin(&st.o.cells.owner[cell], i);
        }
    }
    // fill_road_layer_by_lanes (:446-484): waypoints every 5 m within +-100 m of the observer's
    // longitudinal coordinate on each lane, clipped to the lane
    for (int l = 0; l < g.n_lanes; ++l) {
        const HwyNetLane& L = g.lanes[l];
        const double origin = lane_s_of(L, ex, ey);
        const double start = origin - 100, stop = origin + 100;
        const int n = (int)ceil((stop - start) / 5.0);  // np.arange length
        for (int k = i; k < n; k += G) {
            double wp = clipd(start + k * 5.0, 0.0, L.length);
            double px, py;
            lane_position(L, wp, 0.0, px, py);
            px -= ex;
            py -= ey;
            int ci = (int)floor((px - lo) / step), cj = (int)floor((py - lo) / step);
            if (0 <= ci && ci < 11 && 0 <= cj && cj < 11) st.o.cells.road[ci * 11 + cj] = 1;
        }
    }
    group_sync<G>();
    for (int k = i; k < 121; k += G) {
        obs_env[k] = 0.0f;        // nan_to_num of the untouched cells
        obs_env[121 + k] = 0.0f;
        obs_env[242 + k] = 0.0f;
        obs_env[363 + k] = st.o.cells.road[k] ? 1.0f : 0.0f;
    }
    group_sync<G>();
    if (cell >= 0 && st.o.cells.owner[cell] == i) {
        double vx = st.v[i] * st.c[i] - evx, vy = st.v[i] * st.s[i] - evy;
        vx = lmap(vx, -2 * kMaxSpeed, 2 * kMaxSpeed, -1.0, 1.0);  // normalize :340-352 (x, y not normalised)
        vy = lmap(vy, -2 * kMaxSpeed, 2 * kMaxSpeed, -1.0, 1.0);
        obs_env[cell] = 1.0f;
        obs_env[121 + cell] = (float)clipd(vx, -1.0, 1.0);
        obs_env[242 + cell] = (float)clipd(vy, -1.0, 1.0);
    }
}

__device__ __forceinline__ int obs_size(const HwyNetParams& P) {
    if (P.obs_type == HWY_OBS_OCCUPANCY) return 4 * 11 * 11;
    if (P.obs_type == HWY_OBS_TTC) return 9 * (int)(P.ttc_horizon / (1.0 / P.policy_frequency));
    return P.obs_vehicles_count * (P.obs_n_feat > 0 ? P.obs_n_feat : (P.obs_features == 7 ? 7 : 5));
}

template <int G, bool REG>
__device__ __forceinline__ void observe_any(const HwyNetParams& P, const GraphShared& g, EnvStage<G, REG>& st,
                                            int V, int i, float* __restrict__ obs_env) {
    if (P.obs_type == HWY_OBS_TTC)
        observe_ttc(P, g, st, V, i, st.speed_index, obs_env);
    else if (P.obs_type == HWY_OBS_OCCUPANCY)
        observe_occupancy(P, g, st, V, i, obs_env);
    else
        observe_kinematics(P, g, st, V, i, obs_env);
}

// ------------------------------------------------------------------ state I/O
struct Regs {
    double x, y, heading, speed, target_speed, timer, delta, imp_x, imp_y;
    int meta;
};
__device__ __forceinline__ void load_regs(const HwyNetState& S, size_t slot, Regs& r) {
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
__device__ __forceinline__ void store_regs(const HwyNetState& S, size_t slot, const Regs& r) {
    reinterpret_cast<double2*>(S.pos)[slot] = make_double2(r.x, r.y);
    reinterpret_cast<double2*>(S.hs)[slot] = make_double2(r.heading, r.speed);
    reinterpret_cast<double2*>(S.tt)[slot] = make_double2(r.target_speed, r.timer);
    reinterpret_cast<double2*>(S.imp)[slot] = make_double2(r.imp_x, r.imp_y);
    S.delta[slot] = r.delta;
    S.meta[slot] = r.meta;
}
template <int G, bool REG>
__device__ __forceinline__ void publish(EnvStage<G, REG>& st, int i, const Regs& r) {
    double sn, cs;
    m_sincos(r.heading, &sn, &cs);
    st.x[i] = r.x;
    st.y[i] = r.y;
    st.heading[i] = r.heading;
    st.c[i] = cs;
    st.s[i] = sn;
    st.v[i] = r.speed;
    // getattr(ego_vehicle, "target_speed", 0) (behavior.py:172): a plain Vehicle has none (its tt pair holds the
    // BicycleVehicle's lateral_speed / yaw_rate)
    st.ts[i] = meta_kind(r.meta) == HWY_KIND_VEHICLE ? 0.0 : r.target_speed;
}


// ------------------------------------------------------------------ the ContinuousAction ego (plain Vehicle / BicycleVehicle)
// BicycleVehicle.derivative_func (vehicle/dynamics.py:73-111) on (x, y, heading, speed, lateral_speed, yaw_rate)
__device__ __noinline__ void bicycle_derivative(const double (&st)[6], double steering, double acceleration,
                                                double (&d)[6]) {
    const double mass = 1.0, len_a = kVehLength / 2, len_b = kVehLength / 2;
    const double inertia_z = 1.0 / 12 * mass * (kVehLength * kVehLength + kVehWidth * kVehWidth);
    const double friction_front = 15.0 * mass, friction_rear = 15.0 * mass;
    const double heading = st[2], speed = st[3], lateral_speed = st[4], yaw_rate = st[5];
    const double theta_vf = atan2(lateral_speed + len_a * yaw_rate, speed);
    const double theta_vr = atan2(lateral_speed - len_b * yaw_rate, speed);
    double f_yf = 2 * friction_front * (steering - theta_vf);
    double f_yr = 2 * friction_rear * (0.0 - theta_vr);
    if (fabs(speed) < 1) {  // low speed dynamics: damping of lateral speed and yaw rate
        f_yf = -mass * lateral_speed - inertia_z / len_a * yaw_rate;
        f_yr = -mass * lateral_speed + inertia_z / len_a * yaw_rate;
    }
    const double d_lateral_speed = 1 / mass * (f_yf + f_yr) - yaw_rate * speed;
    const double d_yaw_rate = 1 / inertia_z * (len_a * f_yf - len_b * f_yr);
    double sn, cs;
    sincos(heading, &sn, &cs);
    d[0] = cs * speed + (-sn) * lateral_speed;
    d[1] = sn * speed + cs * lateral_speed;
    d[2] = yaw_rate;
    d[3] = acceleration;
    d[4] = d_lateral_speed;
    d[5] = d_yaw_rate;
}
// Vehicle.clip_actions (kinematics.py:155-168), shared by both vehicle classes
__device__ __forceinline__ void clip_plain_actions(double speed, bool crashed, double& steering, double& acceleration) {
    if (crashed) {
        steering = 0.0;
        acceleration = -1.0 * speed;
    }
    if (speed > kMaxSpeed)
        acceleration = fmin(acceleration, 1.0 * (kMaxSpeed - speed));
    else if (speed < kMinSpeed)
        acceleration = fmax(acceleration, 1.0 * (kMinSpeed - speed));
}
// BicycleVehicle.step (dynamics.py:142-161): clip_actions, then one rk4 step (:13-30)
__device__ __noinline__ void bicycle_advance(double (&st)[6], bool crashed, double& steering, double& acceleration,
                                             double dt) {
    clip_plain_actions(st[3], crashed, steering, acceleration);
    steering = clipd(steering, -kPi / 2, kPi / 2);
    st[5] = clipd(st[5], -2 * kPi, 2 * kPi);  // MAX_ANGULAR_SPEED
    double f1[6], f2[6], f3[6], f4[6], tmp[6];
    bicycle_derivative(st, steering, acceleration, f1);
    for (int k = 0; k < 6; ++k) tmp[k] = st[k] + (f1[k] * (dt / 2));
    bicycle_derivative(tmp, steering, acceleration, f2);
    for (int k = 0; k < 6; ++k) tmp[k] = st[k] + (f2[k] * (dt / 2));
    bicycle_derivative(tmp, steering, acceleration, f3);
    for (int k = 0; k < 6; ++k) tmp[k] = st[k] + (f3[k] * dt);
    bicycle_derivative(tmp, steering, acceleration, f4);
    for (int k = 0; k < 6; ++k) st[k] = st[k] + (dt / 6) * (f1[k] + (2 * f2[k]) + (2 * f3[k]) + f4[k]);
}
// Vehicle.step (kinematics.py:130-153) on an explicit state; the pending impact is the caller's
__device__ __noinline__ void kinematic_advance(double (&st)[6], bool crashed, double& steering, double& acceleration,
                                               double dt) {
    clip_plain_actions(st[3], crashed, steering, acceleration);
    const double beta = atan(1.0 / 2 * tan(steering));
    double sn, cs;
    sincos(st[2] + beta, &sn, &cs);
    st[0] += (st[3] * cs) * dt;
    st[1] += (st[3] * sn) * dt;
    st[2] += st[3] * sin(beta) / (kVehLength / 2) * dt;
    st[3] += acceleration * dt;
}

// ------------------------------------------------------------------ RegulatedRoad (road/regulation.py)
__device__ __forceinline__ int HwyNetLane_route(const HwyNetLane& L) {
    return L.from_node | (L.to_node << 8) | ((L.lane_id + 1) << 16);
}

// road/road.py:323-362 position_heading_along_route(route, longitudinal, 0, current_lane_index)
template <int G, bool REG>
__device__ __noinline__ void position_heading_along_route(const GraphShared& g, const EnvStage<G, REG>& st, int v,
                                                          double longitudinal, double& px, double& py,
                                                          double& heading) {
    const int cur = st.lane[v];
    const int* route = st.route[v];
    int rlen = st.route_len[v];
    int own = HwyNetLane_route(g.lanes[cur]);
    if (rlen == 0) {  // `self.route or [self.lane_index]`
        route = &own;
        rlen = 1;
    }
    int k = 0;
    for (;;) {
        int first = road_first(g, RT_FROM(route[k]), RT_TO(route[k]));
        int id = RT_ID(route[k]);
        if (id < 0) id = g.lanes[cur].lane_id;
        const HwyNetLane& L = g.lanes[first + id];
        if (k < rlen - 1 && longitudinal > L.length) {
            longitudinal -= L.length;
            ++k;
            continue;
        }
        lane_position(L, longitudinal, 0.0, px, py);
        heading = lane_heading_at(L, longitudinal);
        return;
    }
}

// utils.py:77-174 rotated_rectangles_intersect: 9 points (corners, centre, edge midpoints) of one
// rectangle inside the other, both ways, with the reference's rotation convention
// One direction of utils.py:77-174 rotated_rectangles_intersect with the sines / cosines of both headings given:
// the 9 points (corners, centre, edge midpoints, the reference's order) of rectangle 1 tested inside rectangle 2.
__device__ __forceinline__ bool corner_inside(double c1x, double c1y, double s1, double c1, double c2x, double c2y,
                                              double s2, double c2, double l, double w) {
    const double hl = l / 2, hw = w / 2;
    const double pxs[9] = {-hl, -hl, hl, hl, 0, -hl, hl, 0, 0};
    const double pys[9] = {-hw, hw, hw, -hw, 0, 0, 0, -hw, hw};
#pragma unroll
    for (int k = 0; k < 9; ++k) {
        double px = c1 * pxs[k] + (-s1) * pys[k] + c1x;
        double py = s1 * pxs[k] + c1 * pys[k] + c1y;
        double dx = px - c2x, dy = py - c2y;
        double rx = c2 * dx + (-s2) * dy, ry = s2 * dx + c2 * dy;
        if (-l / 2 <= rx && rx <= l / 2 && -w / 2 <= ry && ry <= w / 2) return true;
    }
    return false;
}
// Both directions for two rectangles of the same size.  Inlined into enforce_road_rules, which is itself a real call
// from the substep loop (enforce_road_rules_call): its two unrolled copies used to be 13 KB in the middle of that
// loop; rolled loops and a call per pair were both slower on cfg 3 than this form.
__device__ __forceinline__ bool rotated_rectangles_intersect(double c1x, double c1y, double a1, double c2x, double c2y,
                                                          double a2, double l, double w) {
    double s1, c1, s2, c2;
    m_sincos(a1, &s1, &c1);
    m_sincos(a2, &s2, &c2);
    return corner_inside(c1x, c1y, s1, c1, c2x, c2y, s2, c2, l, w) ||
           corner_inside(c2x, c2y, s2, c2, c1x, c1y, s1, c1, l, w);
}

// general form (two sizes) for the known-answer hook debug_rectangles_kernel
__device__ __forceinline__ bool has_corner_inside(double c1x, double c1y, double l1, double w1, double a1,
                                                  double c2x, double c2y, double l2, double w2, double a2) {
    const double hl = l1 / 2, hw = w1 / 2;
    const double pxs[9] = {-hl, -hl, hl, hl, 0, -hl, hl, 0, 0};
    const double pys[9] = {-hw, hw, hw, -hw, 0, 0, 0, -hw, hw};
    double s1, c1, s2, c2;
    m_sincos(a1, &s1, &c1);
    m_sincos(a2, &s2, &c2);
#ifdef HWY_NET_INLINE_RECT
#pragma unroll
#else
#pragma unroll 1
#endif
    for (int k = 0; k < 9; ++k) {
        double px = c1 * pxs[k] + (-s1) * pys[k] + c1x;
        double py = s1 * pxs[k] + c1 * pys[k] + c1y;
        double dx = px - c2x, dy = py - c2y;
        double rx = c2 * dx + (-s2) * dy, ry = s2 * dx + c2 * dy;
        if (-l2 / 2 <= rx && rx <= l2 / 2 && -w2 / 2 <= ry && ry <= w2 / 2) return true;
    }
    return false;
}

// regulation.py:42-111: enforce_road_rules with is_conflict_possible / respect_priorities.
// All threads of the group call this; r is the caller's vehicle.
// PLAIN: the env may hold a ContinuousAction ego (kind HWY_KIND_VEHICLE); compiled out otherwise so that the
// DiscreteMetaAction kernels keep their register budget
template <int G, bool REG, bool PLAIN>
__device__ __forceinline__ void enforce_road_rules(const bool dynamical, const GraphShared& g,
                                                   EnvStage<G, REG>& st, int V, int i, Regs& r, double act_steer) {
    const bool active = i < V;
    // un-freeze (YIELD_DURATION = 0: every yielding vehicle is released at the next regulation tick)
    if (active && (r.meta & HWY_META_YIELDING)) {
        r.target_speed = g.lanes[st.lane[i]].speed_limit;
        r.meta &= ~HWY_META_YIELDING;
        st.ts[i] = r.target_speed;
    }
    if (i == 0) st.yield_mask = 0;
    // Pairs (a < b) are dealt round-robin over the group: this thread owns pairs i, i + G, ... (<= 16 of the
    // 32 * 31 / 2); bit q of `conflict` = its q-th pair conflicts at some horizon point.  The horizon
    // (predict_trajectory_constant_speed, vehicle/controller.py:236-253, t = 0.25 .. 2.75 s) is staged
    // kPredChunk points at a time.
    const int n_pairs = V * (V - 1) / 2;
    auto row_start = [V](int a) { return a * (2 * V - a - 1) / 2; };
    auto decode = [&](int p, int& a, int& b) {
        const int w = 2 * V - 1;
        a = (int)(((float)w - sqrtf((float)(w * w - 8 * p))) * 0.5f);
        a = max(0, min(a, V - 2));
        while (a > 0 && row_start(a) > p) --a;
        while (row_start(a + 1) <= p) ++a;
        b = a + 1 + (p - row_start(a));
    };
    unsigned conflict = 0;
    const double s0 = active ? st.own_s[i] : 0.0;
    // A plain Vehicle / BicycleVehicle (ContinuousAction ego) is not a ControlledVehicle: its
    // predict_trajectory_constant_speed (vehicle/kinematics.py:179-198) steps a copy 11 x 0.25 s with acceleration 0
    // and its current steering; the copy's state is carried across the horizon chunks.
    const bool plain = PLAIN && active && meta_kind(r.meta) == HWY_KIND_VEHICLE;
    double sim[PLAIN ? 6 : 1];
    double sim_steer = act_steer, sim_acc = 0.0;
    bool sim_crashed = (r.meta & HWY_META_CRASHED) != 0, sim_impact = (r.meta & HWY_META_HAS_IMPACT) != 0;
    if constexpr (PLAIN) {
        sim[0] = r.x, sim[1] = r.y, sim[2] = r.heading, sim[3] = r.speed, sim[4] = r.target_speed, sim[5] = r.timer;
    }
    for (int k0 = 0; k0 < kPred; k0 += kPredChunk) {
        const int nk = min(kPredChunk, kPred - k0);
        if (active) {
            for (int k = 0; k < nk; ++k) {
                double px, py, ph;
                bool simulated = false;
                if constexpr (PLAIN) {
                    if (plain) {
                        if (dynamical) {
                            bicycle_advance(sim, sim_crashed, sim_steer, sim_acc, 0.25);
                        } else {
                            kinematic_advance(sim, sim_crashed, sim_steer, sim_acc, 0.25);
                            if (sim_impact) {  // kinematics.py:147-150
                                sim[0] += r.imp_x;
                                sim[1] += r.imp_y;
                                sim_crashed = true;
                                sim_impact = false;
                            }
                        }
                        px = sim[0];
                        py = sim[1];
                        ph = sim[2];
                        simulated = true;
                    }
                }
                if (!simulated)
                    position_heading_along_route(g, st, i, s0 + r.speed * (0.25 * (k0 + k + 1)), px, py, ph);
                st.pred[i][k][0] = px;
                st.pred[i][k][1] = py;
                st.pred[i][k][2] = ph;
            }
        }
        group_sync<G>();
        int q = 0;
        for (int p = i; p < n_pairs; p += G, ++q) {
            if ((conflict >> q) & 1u) continue;
            int a, b;
            decode(p, a, b);
            bool hit = false;
            for (int k = 0; k < nk && !hit; ++k) {
                double p1x = st.pred[a][k][0], p1y = st.pred[a][k][1], p2x = st.pred[b][k][0], p2y = st.pred[b][k][1];
                if (norm2(p2x - p1x, p2y - p1y) > kVehLength) continue;
                double h1 = st.pred[a][k][2], h2 = st.pred[b][k][2];
#ifdef HWY_NET_INLINE_RECT
                hit = has_corner_inside(p1x, p1y, 1.5 * kVehLength, 0.9 * kVehWidth, h1, p2x, p2y, 1.5 * kVehLength,
                                        0.9 * kVehWidth, h2) ||
                      has_corner_inside(p2x, p2y, 1.5 * kVehLength, 0.9 * kVehWidth, h2, p1x, p1y, 1.5 * kVehLength,
                                        0.9 * kVehWidth, h1);
#else
                hit = rotated_rectangles_intersect(p1x, p1y, h1, p2x, p2y, h2, 1.5 * kVehLength, 0.9 * kVehWidth);
#endif
            }
            if (hit) conflict |= 1u << q;
        }
        group_sync<G>();
    }
    for (int q = 0; conflict >> q; ++q) {
        if (!((conflict >> q) & 1u)) continue;
        int a, b;
        decode(i + q * G, a, b);
        const int pa = g.lanes[st.lane[a]].priority, pb = g.lanes[st.lane[b]].priority;
        int y;
        if (pa > pb)
            y = b;
        else if (pa < pb)
            y = a;
        else {  // the vehicle behind yields (front_distance_to, vehicle/objects.py:205-206)
            double fab = dot2(st.c[a], st.s[a], st.x[b] - st.x[a], st.y[b] - st.y[a]);
            double fba = dot2(st.c[b], st.s[b], st.x[a] - st.x[b], st.y[a] - st.y[b]);
            y = fab > fba ? a : b;
        }
        if (st.kind[y] == HWY_KIND_IDM) atomicOr(&st.yield_mask, 1u << y);  // never an MDPVehicle
    }
    group_sync<G>();
    if (active && ((st.yield_mask >> i) & 1u)) {
        r.target_speed = 0.0;
        r.meta |= HWY_META_YIELDING;
        st.ts[i] = 0.0;
    }
    group_sync<G>();
}

// Out-of-line form for the kernels without a ContinuousAction ego: 1 = released (target speed back to the lane's
// limit, YIELDING cleared), 2 = yields (target speed 0, YIELDING set), 0 = unchanged.
template <int G, bool REG>
__device__ __noinline__ int enforce_road_rules_call(const GraphShared& g, EnvStage<G, REG>& st, int V, int i,
                                                    int meta, double speed) {
    Regs r;
    r.x = r.y = r.heading = r.target_speed = r.timer = r.delta = r.imp_x = r.imp_y = 0.0;
    r.speed = speed;
    r.meta = meta;
    enforce_road_rules<G, REG, false>(false, g, st, V, i, r, 0.0);
    if (r.meta & HWY_META_YIELDING) return 2;
    return (meta & HWY_META_YIELDING) ? 1 : 0;
}

__device__ __forceinline__ int n_agents_of(const HwyNetParams& P) { return P.n_agents > 1 ? P.n_agents : 1; }
// slot of the a-th controlled vehicle (-1: none)
__device__ __forceinline__ int agent_slot(unsigned agent_mask, int a) {
    for (int k = 0; k < a; ++k) agent_mask &= agent_mask - 1;
    return agent_mask ? __ffs(agent_mask) - 1 : -1;
}
// observation_type.observe(): one observation per controlled vehicle (MultiAgentObservation, observation.py:588-604)
template <int G, bool REG>
__device__ __forceinline__ void observe_agents(const HwyNetParams& P, const GraphShared& g, EnvStage<G, REG>& st, int i,
                                               float* __restrict__ obs_env) {
    const int A = n_agents_of(P);
    if (A == 1) {
        observe_any(P, g, st, st.count, i, obs_env);
        return;
    }
    const int first = st.ego;
    for (int a = 0; a < A; ++a) {
        group_sync<G>();
        if (i == 0) st.ego = max(agent_slot(st.agent_mask, a), 0);
        group_sync<G>();
        observe_any(P, g, st, st.count, i, obs_env + (size_t)a * obs_size(P));
    }
    group_sync<G>();
    if (i == 0) st.ego = first;
    group_sync<G>();
}

// The exact half of _is_colliding (vehicle/objects.py:118-138) for a pair that survived the squared-distance reject:
// the sphere pre-check with its square root, then the separating-axis test.  Out of line — a few pairs per env-step
// get here, and inlined it was 6 KB of the substep loop.  Returns will_intersect | intersecting << 1; tr = transition.
__device__ __noinline__ int collide_exact(double xa, double ya, double ca, double sa, double va, double xb, double yb,
                                          double cb, double sb, double vb, bool b_object, double dt, double* tr) {
    const double diag_v = 0x1.58a68a4a8d9f3p+2, diag_o = 0x1.6a09e667f3bcdp+1;
    const double dist = norm2(xb - xa, yb - ya);
    if (dist > (diag_v + (b_object ? diag_o : diag_v)) / 2 + va * dt) return 0;
    const double len_b = b_object ? 2.0 : kVehLength;
    Quad pa = make_polygon(xa, ya, ca, sa);
    Quad pb = make_polygon(xb, yb, cb, sb, len_b);
    bool inter, will;
    double trx, try_;
    polygons_intersecting(pa, pb, va * ca * dt, va * sa * dt, vb * cb * dt, vb * sb * dt, inter, will, trx, try_);
    tr[0] = trx;
    tr[1] = try_;
    return (will ? 1 : 0) | (inter ? 2 : 0);
}

// ------------------------------------------------------------------ one simulation substep
// Road.act() then [RegulatedRoad rules] Road.step(dt) for one env; all threads of the group call it.
// `ego_label` >= 0 on the first frame of a policy step: the meta-action label of the controlled vehicle.
template <int G, bool REG, bool PLAIN = false>
__device__ __forceinline__ void substep(const HwyNetParams& P, const GraphShared& g, EnvStage<G, REG>& st, int i,
                                        Regs& r, double& act_accel, double& act_steer, double dt, int ego_label,
                                        int* my_speed_index = nullptr, const float* act_f = nullptr) {
    const int V = st.count;
    const bool active = i < V;
    const int kind = meta_kind(r.meta);
    // ---- ContinuousAction.get_action / act on the first frame (envs/common/action.py:136-162): the Box is float32
    // and NEP 50 keeps utils.lmap (utils.py:31-33) in float32; the vehicle's action dict persists until the next act
    if (PLAIN && act_f && active && kind == HWY_KIND_VEHICLE) {
        float a0 = act_f[0], a1 = act_f[1];
        if (P.act_clip) {
            a0 = fminf(fmaxf(a0, -1.0f), 1.0f);
            a1 = fminf(fmaxf(a1, -1.0f), 1.0f);
        }
        const float acc = __fadd_rn((float)P.acc_lo, __fdiv_rn(__fmul_rn(__fsub_rn(a0, -1.0f), (float)(P.acc_hi - P.acc_lo)), 2.0f));
        const float stf = __fadd_rn((float)P.steer_lo, __fdiv_rn(__fmul_rn(__fsub_rn(a1, -1.0f), (float)(P.steer_hi - P.steer_lo)), 2.0f));
        act_accel = (double)acc;
        act_steer = (double)stf;
    }
    // ---- action_type.act on the first frame: MDPVehicle.act (controller.py:295-315)
    // (every controlled vehicle has its own label: MultiAgentAction.act, action.py:316-321)
    if (ego_label >= 0 && active && kind == HWY_KIND_MDP) {
        follow_road(g, st, i);
        if (ego_label == 3 || ego_label == 4) {
            int idx = speed_to_index(P, r.speed) + (ego_label == 3 ? 1 : -1);
            idx = max(0, min(idx, P.n_target_speeds - 1));
            if (i == st.ego) st.speed_index = idx;
            if (my_speed_index) *my_speed_index = idx;
            r.target_speed = P.target_speeds[idx];
            st.ts[i] = r.target_speed;
        } else if (ego_label == 0 || ego_label == 2) {
            const HwyNetLane& T = g.lanes[st.tgt[i]];
            int id = max(0, min(T.lane_id + (ego_label == 2 ? 1 : -1), T.road_count - 1));
            int cand = T.road_first + id;
            if (lane_reachable(g.lanes[cand], r.x, r.y)) st.tgt[i] = cand;
        }
    }
    phase_sync<G>();
    // ---- Road.act (road/road.py:464-467): vehicle.act() in list order.  follow_road only touches the vehicle's
    // own target lane and route, so all of them run at once; what must stay ordered is the lane-change policy of the
    // vehicles whose policy can read another vehicle's target lane or move their own (a pending change on the same
    // road, or a decision tick on a multi-lane road).  Those take turns; when it is u's turn it sees the final
    // target lanes of the vehicles before it and the pre-act ones (tgt_prev) of the vehicles after it.
    const bool crashed = (r.meta & HWY_META_CRASHED) != 0;
    bool ordered = false;
    if (active) {
        st.tgt_prev[i] = st.tgt[i];
        // road.objects neither act nor step (road/road.py:464-476)
        // (nor does a plain Vehicle: Vehicle.act(None) keeps its action, kinematics.py:119-128)
        if (kind != HWY_KIND_OBSTACLE && kind != HWY_KIND_VEHICLE && (kind != HWY_KIND_IDM || !crashed))
            follow_road(g, st, i);  // behavior.py:102-103, controller.py:98
        // IDMVehicle(enable_lane_change=False) never runs change_lane_policy (behavior.py:104-105)
        if (kind == HWY_KIND_IDM && !crashed && !(r.meta & HWY_META_NO_LANE_CHANGE)) {
            const int lane = st.lane[i], tgt = st.tgt[i];
            const HwyNetLane &A = g.lanes[lane], &B = g.lanes[tgt];
            if (lane != tgt) {
                ordered = A.from_node == B.from_node && A.to_node == B.to_node;
            } else if (P.lane_change_delay < r.timer) {  // do_every (utils.py:16-17)
                if (A.road_count > 1)
                    ordered = true;
                else
                    r.timer = 0.0;  // decision tick with no side lane
            }
        }
    }
    phase_sync<G>();
    unsigned turn = __ballot_sync(group_mask<G>(), ordered) >> ((threadIdx.x & 31) & ~(G - 1));
    while (turn) {
        const int v = __ffs(turn) - 1;
        turn &= turn - 1;
        if (i == v) r.timer = change_lane_policy(P, g, st, V, v, r.delta, r.timer);
        group_sync<G>();
    }
    // ---- parallel part: steering + acceleration
    const bool mobile = active && kind != HWY_KIND_OBSTACLE;  // road.objects neither act nor step
    double sin_beta = 0.0, cos_beta = 1.0;
    const bool plain = PLAIN && mobile && kind == HWY_KIND_VEHICLE;  // the ContinuousAction ego: its action dict persists
    if (mobile && !plain) {
        const int lane = st.lane[i], tgt = st.tgt[i];
        if (!crashed) {
            double lc_s = st.own_s[i], lc_lat = st.own_lat[i];
            if (tgt != lane) lane_local(g.lanes[tgt], r.x, r.y, lc_s, lc_lat);
            double xs = steering_sin_slip(g.lanes[tgt], lc_s, lc_lat, r.heading, r.speed);
            beta_of_controlled(xs, sin_beta, cos_beta);
        }
        if (kind == HWY_KIND_IDM) {
            if (!crashed) {
                int f, rr;
                neighbours(g, st, V, i, lane, P.connected_lanes != 0, f, rr);
                double acc = idm_acceleration(P, g, st, r.delta, i, f);
                if (lane != tgt) {
                    neighbours(g, st, V, i, tgt, P.connected_lanes != 0, f, rr);
                    acc = fmin(acc, idm_acceleration(P, g, st, r.delta, i, f));
                }
                act_accel = clipd(acc, -P.acc_max, P.acc_max);
            }
        } else {
            act_accel = kKpA * (r.target_speed - r.speed);
        }
    }
    // ---- RegulatedRoad.step (regulation.py:36-40): rules every int(1/dt/2) substeps, before Road.step
    if (REG) {
        if (i == 0) st.road_steps += 1;
        group_sync<G>();
        if (P.regulated && st.road_steps % (int)(1 / dt / 2) == 0)
        {
#ifdef HWY_NET_INLINE_RULES
            if constexpr (true) {
                enforce_road_rules<G, REG, PLAIN>(P.dynamical != 0, g, st, V, i, r, act_steer);
            } else {
#else
            if constexpr (PLAIN) {
                enforce_road_rules<G, REG, true>(P.dynamical != 0, g, st, V, i, r, act_steer);
            } else {
#endif
                // the rules only read this vehicle's flags and speed and only move its target speed and YIELDING bit:
                // a real call with those in registers keeps 10 KB that run every 7th substep out of the loop body
                const int code = enforce_road_rules_call<G, REG>(g, st, V, i, r.meta, r.speed);
                if (code == 1) {
                    r.target_speed = g.lanes[st.lane[i]].speed_limit;
                    r.meta &= ~HWY_META_YIELDING;
                } else if (code == 2) {
                    r.target_speed = 0.0;
                    r.meta |= HWY_META_YIELDING;
                }
            }
        }
    }
    // ---- Road.step: Vehicle.step (kinematics.py:130-177), IDMVehicle.step timer (behavior.py:139-148)
    if (PLAIN && plain && P.dynamical) {
        // BicycleVehicle.step (dynamics.py:142-150): rk4 over (x, y, heading, speed, lateral_speed, yaw_rate); it never
        // consumes Vehicle.impact (crashed is set by the collision test itself)
        double bs[6] = {r.x, r.y, r.heading, r.speed, r.target_speed, r.timer};
        bicycle_advance(bs, crashed, act_steer, act_accel, dt);
        r.x = bs[0];
        r.y = bs[1];
        r.heading = bs[2];
        r.speed = bs[3];
        r.target_speed = bs[4];
        r.timer = bs[5];
    } else if (mobile) {
        if (plain) {  // Vehicle.step with the action's steering angle: beta = arctan(1/2 tan(delta_f))
            if (crashed) act_steer = 0.0;
            beta_of_angle(act_steer, sin_beta, cos_beta);
        }
        if (kind == HWY_KIND_IDM) r.timer += dt;
        if (crashed) act_accel = -1.0 * r.speed;
        if (r.speed > kMaxSpeed)
            act_accel = fmin(act_accel, 1.0 * (kMaxSpeed - r.speed));
        else if (r.speed < kMinSpeed)
            act_accel = fmax(act_accel, 1.0 * (kMinSpeed - r.speed));
        const double ch = st.c[i], sh = st.s[i];
        double cs = ch * cos_beta - sh * sin_beta, sn = sh * cos_beta + ch * sin_beta;
        r.x += (r.speed * cs) * dt;
        r.y += (r.speed * sn) * dt;
        if (r.meta & HWY_META_HAS_IMPACT) {
            r.x += r.imp_x;
            r.y += r.imp_y;
            r.meta = (r.meta | HWY_META_CRASHED) & ~HWY_META_HAS_IMPACT;
        }
        r.heading += div_finite(r.speed * sin_beta, kVehLength / 2) * dt;
        r.speed += act_accel * dt;
    }
    phase_sync<G>();  // everyone is done reading the pre-step staging
    if (active) publish(st, i, r);
    phase_sync<G>();
    closest_lane_group(g, st, V, i, mobile);  // on_state_update
    if (plain) st.tgt[i] = st.lane[i];  // schema: a plain Vehicle has no target lane of its own
    // ---- collision sweep (road/road.py:477-481): partners in ascending order => the surviving impact is
    // the one of the largest partner index
    // Road objects (Obstacle: 2 x 2 m, kind 3) sit in the slots after the vehicles, so vehicle i meets its vehicle
    // partners first and the objects last, as in the reference; only vehicles call handle_collisions; against an
    // Obstacle the vehicle takes the WHOLE transition (vehicle/objects.py:104-107).
    // The reference's sphere pre-check (vehicle/objects.py:122-126) first runs on squared distances with a 1e-9 m slack
    // (no sqrt) and the partners that survive are gathered in a mask, so that the lanes of a warp run the exact pre-check
    // and the separating-axis test together instead of one at a time.
    if (active) {
        // RoadObject.diagonal = sqrt(LENGTH^2 + WIDTH^2) (objects.py:63): sqrt(29) and sqrt(8), correctly rounded
        const double diag_v = 0x1.58a68a4a8d9f3p+2, diag_o = 0x1.6a09e667f3bcdp+1;
        unsigned pending = 0;
#pragma unroll 1
        for (int j = 0; j < V; ++j) {
            if (j == i) continue;
            const int a = i < j ? i : j, b = i < j ? j : i;
            if (st.kind[a] == HWY_KIND_OBSTACLE) continue;
            const double reach = (diag_v + (st.kind[b] == HWY_KIND_OBSTACLE ? diag_o : diag_v)) / 2 + st.v[a] * dt + 1e-9;
            const double dx = st.x[b] - st.x[a], dy = st.y[b] - st.y[a];
            const bool far = reach <= 0.0 || dot2(dx, dy, dx, dy) > reach * reach * (1.0 + 1e-12);
            if (!far) pending |= 1u << j;  // (a NaN distance stays pending, as it passes the reference's `>` test)
        }
        while (pending) {
            const int j = __ffs(pending) - 1;
            pending &= pending - 1;
            const int a = i < j ? i : j, b = i < j ? j : i;
            const bool b_object = st.kind[b] == HWY_KIND_OBSTACLE;
            double tr[2];
#ifdef HWY_NET_INLINE_COLLIDE
            int flags = 0;
            {
                const double len_b = b_object ? 2.0 : kVehLength;
                const double dist = norm2(st.x[b] - st.x[a], st.y[b] - st.y[a]);
                if (dist > (diag_v + (b_object ? diag_o : diag_v)) / 2 + st.v[a] * dt) continue;
                Quad pa = make_polygon(st.x[a], st.y[a], st.c[a], st.s[a]);
                Quad pb = make_polygon(st.x[b], st.y[b], st.c[b], st.s[b], len_b);
                bool inter, will;
                polygons_intersecting(pa, pb, st.v[a] * st.c[a] * dt, st.v[a] * st.s[a] * dt, st.v[b] * st.c[b] * dt,
                                      st.v[b] * st.s[b] * dt, inter, will, tr[0], tr[1]);
                flags = (will ? 1 : 0) | (inter ? 2 : 0);
            }
#else
            const int flags = collide_exact(st.x[a], st.y[a], st.c[a], st.s[a], st.v[a], st.x[b], st.y[b], st.c[b], st.s[b],
                                            st.v[b], b_object, dt, tr);
#endif
            if ((flags & 1) && !(b_object && i == b)) {
                const double share = b_object ? 1.0 : 0.5;
                r.imp_x = i == a ? tr[0] * share : -tr[0] * share;
                r.imp_y = i == a ? tr[1] * share : -tr[1] * share;
                r.meta |= HWY_META_HAS_IMPACT;
            }
            if (flags & 2) r.meta |= HWY_META_CRASHED;
        }
    }
}

// load one env into the group's stage (count, ego, routes, staged kinematics)
template <int G, bool REG>
__device__ __forceinline__ void load_env(const HwyNetParams& P, const GraphShared& g, const HwyNetState& S,
                                         EnvStage<G, REG>& st, int e, int i, Regs& r) {
    const size_t slot = (size_t)e * S.vp + i;
    load_regs(S, slot, r);
    const int* src = S.route + slot * R;
    for (int k = 0; k < R; ++k) st.route[i][k] = src[k];
    st.route_len[i] = S.route_len[slot];
    const int count = S.count ? S.count[e] : P.n_vehicles;
    if (i == 0) {
        st.n_cand = 0;
        st.count = count;
        st.speed_index = S.speed_index[e];
        st.road_steps = S.road_steps ? S.road_steps[e] : 0;
    }
    publish(st, i, r);
    st.lane[i] = meta_lane(r.meta);
    st.tgt[i] = meta_target(r.meta);
    st.kind[i] = meta_kind(r.meta);
    if (i < count) lane_local(g.lanes[st.lane[i]], r.x, r.y, st.own_s[i], st.own_lat[i]);
    // the controlled vehicle: first MDPVehicle of the list
    unsigned is_mdp = __ballot_sync(group_mask<G>(), i < count && is_controlled_kind(meta_kind(r.meta)));
    is_mdp >>= ((threadIdx.x & 31) & ~(G - 1));
    if (i == 0) {
        st.ego = is_mdp ? __ffs(is_mdp) - 1 : 0;
        st.agent_mask = is_mdp;
    }
    group_sync<G>();
}

template <int G, bool REG>
__device__ __forceinline__ void store_env(const HwyNetState& S, EnvStage<G, REG>& st, int e, int i, int dst,
                                          Regs& r) {
    // dst: destination slot of this vehicle (-1: dropped)
    if (dst >= 0) {
        r.meta = meta_set_target(meta_set_lane(r.meta, st.lane[i]), st.tgt[i]);
        const size_t slot = (size_t)e * S.vp + dst;
        store_regs(S, slot, r);
        int* d = S.route + slot * R;
        for (int k = 0; k < R; ++k) d[k] = st.route[i][k];
        S.route_len[slot] = st.route_len[i];
    }
}

// ------------------------------------------------------------------ intersection population
// envs/intersection_env.py:325-352 _spawn_vehicle, executed by ONE thread: consumes the env's numpy
// stream (uniform; choice(range(4), size=2, replace=False) = Floyd's algorithm + tail shuffle;
// normal; normal; uniform) and leaves the accepted vehicle in the stage's spawn record.
template <int G, bool REG>
__device__ __noinline__ void spawn_vehicle(const HwyNetParams& P, const HwyIntersectionSpawn& SP,
                                           const GraphShared& g, EnvStage<G, REG>& st, Pcg64& rng,
                                           unsigned keep_mask, double longitudinal, double position_deviation,
                                           double speed_deviation, double spawn_probability, bool go_straight) {
    st.sp_ok = 0;
    if (rng.next_double() > spawn_probability) return;  // np_random.uniform()
    int a = rng.choice(3), b = rng.choice(4);            // Floyd: j = 2, 3
    if (b == a) b = 3;
    int route2[2] = {a, b};
    int j = rng.choice(2);                               // _shuffle_int(n = 2): swap [1] <-> [j]
    int tmp = route2[1];
    route2[1] = route2[j];
    route2[j] = tmp;
    const int r0 = route2[0];
    const int r1 = go_straight ? (r0 + 2) % 4 : route2[1];
    const int lane = SP.spawn_lane[r0];
    const double lon = longitudinal + 5.0 + rng.normal() * position_deviation;
    const double speed = 8.0 + rng.normal() * speed_deviation;
    double px, py;
    lane_position(g.lanes[lane], lon, 0.0, px, py);  // make_on_lane (vehicle/objects.py:68-90)
    const double heading = lane_heading_at(g.lanes[lane], lon);
    for (int v = 0; v < st.count; ++v) {
        if (!((keep_mask >> v) & 1u)) continue;
        if (norm2(st.x[v] - px, st.y[v] - py) < 15) return;
    }
    st.sp_delta = rng.uniform(3.5, 4.5);  // randomize_behavior
    st.sp_x = px;
    st.sp_y = py;
    st.sp_h = heading;
    st.sp_speed = speed;
    st.sp_dest = r1;
    st.sp_ok = 1;  // sp_lane: spawn_closest_lane, by the whole group
}

// RoadObject.__init__'s closest-lane search (objects.py:46-50) for the spawn record, by ALL threads of the group after
// a group_sync that follows the spawning thread: lane l of the network goes to thread l mod G, then a (distance, index)
// minimum over the group = np.argmin's first minimum.  (One thread used to walk all 20 lanes, atan2 included, while
// the other slots of the env waited: every step in the step kernel, ten times in a reset.)
template <int G, bool REG>
__device__ __forceinline__ void spawn_closest_lane(const GraphShared& g, EnvStage<G, REG>& st, int i) {
    if (!st.sp_ok) return;  // uniform over the group
    const double px = st.sp_x, py = st.sp_y, h = st.sp_h;
    double bd = INFINITY;
    int bl = 0x7fffffff;
    for (int l = i; l < g.n_lanes; l += G) {
        const double d = lane_distance_with_heading(g.lanes[l], px, py, h);
        if (bl == 0x7fffffff || d < bd) {
            bd = d;
            bl = l;
        }
    }
#pragma unroll
    for (int off = G / 2; off > 0; off >>= 1) {
        const double d2 = __shfl_xor_sync(group_mask<G>(), bd, off);
        const int l2 = __shfl_xor_sync(group_mask<G>(), bl, off);
        if (l2 != 0x7fffffff && (bl == 0x7fffffff || d2 < bd || (d2 == bd && l2 < bl))) {
            bd = d2;
            bl = l2;
        }
    }
    if (i == 0) st.sp_lane = bl;
    group_sync<G>();
}

// the thread owning the new slot adopts the spawn record: an IDMVehicle, or the MDPVehicle of _make_vehicles
template <int G, bool REG>
__device__ __forceinline__ void adopt_spawn(const HwyNetParams& P, const HwyIntersectionSpawn& SP,
                                            const GraphShared& g, EnvStage<G, REG>& st, int i, Regs& r,
                                            int kind = HWY_KIND_IDM) {
    r.x = st.sp_x;
    r.y = st.sp_y;
    r.heading = st.sp_h;
    r.speed = st.sp_speed;
    if (kind == HWY_KIND_IDM) {
        r.target_speed = st.sp_speed;
        r.timer = py_mod_pos((st.sp_x + st.sp_y) * kPi, P.lane_change_delay);  // behavior.py:59
        r.delta = st.sp_delta;
    } else if (kind == HWY_KIND_VEHICLE) {  // no target speed; (lateral_speed, yaw_rate) = 0 (dynamics.py:52-53)
        r.target_speed = 0.0;
        r.timer = 0.0;
        r.delta = 4.0;
    } else {
        r.target_speed = st.sp_ts;
        r.timer = 0.0;
        r.delta = 4.0;
    }
    r.imp_x = r.imp_y = 0.0;
    r.meta = (st.sp_lane << HWY_META_LANE_SHIFT) | (st.sp_lane << HWY_META_TARGET_SHIFT) | HWY_META_CHECK_COLLISIONS |
             (kind << HWY_META_KIND_SHIFT) | HWY_META_PRESENT;
    const int* rs = SP.route_table + ((size_t)st.sp_lane * 4 + st.sp_dest) * R;
    for (int k = 0; k < R; ++k) st.route[i][k] = rs[k];
    // plan_route_to raises AttributeError on a plain Vehicle: no route (intersection_env.py:309-315)
    st.route_len[i] = kind == HWY_KIND_VEHICLE ? 0 : SP.route_len[(size_t)st.sp_lane * 4 + st.sp_dest];
    st.lane[i] = st.tgt[i] = st.sp_lane;
    st.kind[i] = kind;
    lane_local(g.lanes[st.sp_lane], r.x, r.y, st.own_s[i], st.own_lat[i]);
    publish(st, i, r);
}

// ------------------------------------------------------------------ the step kernel
template <int G, bool REG, bool PLAIN>
__global__ void __launch_bounds__(kStepThreads, 1)
network_step_kernel(const __grid_constant__ HwyNetParams P, const HwyNetGraph* __restrict__ graph, const __grid_constant__ HwyNetState S,
                    const __grid_constant__ HwyIntersectionSpawn SP, const int32_t* __restrict__ action, float* __restrict__ obs,
                    double* __restrict__ reward, uint8_t* __restrict__ terminated,
                    uint8_t* __restrict__ truncated, double* __restrict__ info_speed,
                    uint8_t* __restrict__ info_crashed, const int* __restrict__ list,
                    double* __restrict__ agents_reward, uint8_t* __restrict__ agents_terminated) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    GraphShared& g = *reinterpret_cast<GraphShared*>(smem_raw);
    EnvStage<G, REG>* stages =
        reinterpret_cast<EnvStage<G, REG>*>(smem_raw + ((sizeof(GraphShared) + 15) & ~size_t(15)));
    const int kEnvs = blockDim.x / G;  // the launch sizes the block (step_plan)
    // with a work list (list[0] = how many, list[1..] = env ids) the grid is dense over the list and the
    // blocks past its end leave as a whole; partial blocks let the spare groups ride along on the last entry
    const int n_work = list ? list[0] : S.n_envs;
    if (blockIdx.x * kEnvs >= n_work) return;
    stage_graph(g, graph);

    const int sub = threadIdx.x / G, i = threadIdx.x % G;
    const int idx = blockIdx.x * kEnvs + sub;
    const bool env_ok = idx < n_work;
    const int pick = env_ok ? idx : n_work - 1;
    const int e = list ? list[1 + pick] : pick;
    EnvStage<G, REG>& st = stages[sub];

    Regs r;
    load_env(P, g, S, st, e, i, r);
    const int frames = P.simulation_frequency / P.policy_frequency;
    const double dt = 1.0 / P.simulation_frequency;
    const int A = n_agents_of(P);
    // this thread's agent number (controlled vehicles in list order), its action and its MDPVehicle.speed_index
    const bool is_agent = i < st.count && is_controlled_kind(meta_kind(r.meta));
    const int my_agent = is_agent ? min(__popc(st.agent_mask & ((1u << i) - 1u)), A - 1) : 0;
    // ContinuousAction (P.action_type == 1): `action` holds float32 (throttle, steering) pairs, one per controlled vehicle
    const bool continuous = P.action_type == 1;
    const float* act_f = continuous ? reinterpret_cast<const float*>(action) + 2 * ((size_t)e * A + my_agent) : nullptr;
    const int act = continuous ? 1 : action[(size_t)e * A + my_agent];
    // action label: DiscreteMetaAction.ACTIONS_ALL, or ACTIONS_LONGI {0 SLOWER, 1 IDLE, 2 FASTER} (action.py:204-206)
    const int label = continuous ? -1 : (P.action_mode == 1 ? (act == 0 ? 4 : (act == 2 ? 3 : 1)) : act);
    int my_speed_index = is_agent ? S.speed_index[(size_t)e * A + my_agent] : 0;
    double act_accel = 0.0, act_steer = 0.0;

    for (int frame = 0; frame < frames; ++frame)
        substep<G, REG, PLAIN>(P, g, st, i, r, act_accel, act_steer, dt, frame == 0 ? label : -1, &my_speed_index,
                               frame == 0 ? act_f : nullptr);
    group_sync<G>();

    // ---- epilogue: observation, reward, termination (before any population change)
    const int V = st.count, ego = st.ego;
    float* obs_env = obs + (size_t)e * A * obs_size(P);
    observe_agents(P, g, st, i, obs_env);
    if (A > 1) {
        // ---- several controlled vehicles (envs/intersection_env.py:62-134): mean of the agents' rewards, terminated
        // when ANY crashed or ALL arrived; per-agent rewards / terminal flags for _info
        bool is_crashed = false, arrived = false, on_road = true;
        if (is_agent) {
            const HwyNetLane& L = g.lanes[st.lane[i]];
            const double es = st.own_s[i], elat = st.own_lat[i];
            on_road = lane_on(L, es, elat, 0.0);
            is_crashed = (r.meta & HWY_META_CRASHED) != 0;
            arrived = L.exit_lane && es >= 25;
            double scaled_speed = lmap(r.speed, P.reward_speed_lo, P.reward_speed_hi, 0.0, 1.0);
            double rew = 0.0;
            rew = rew + P.collision_reward * (is_crashed ? 1.0 : 0.0);
            rew = rew + P.high_speed_reward * clipd(scaled_speed, 0.0, 1.0);
            rew = rew + P.arrived_reward * (arrived ? 1.0 : 0.0);
            rew = rew + 0.0 * (on_road ? 1.0 : 0.0);
            if (arrived) rew = P.arrived_reward;
            rew *= on_road ? 1.0 : 0.0;
            if (P.normalize_reward) rew = lmap(rew, P.collision_reward, P.arrived_reward, 0.0, 1.0);
            st.agent_reward[my_agent] = rew;
            st.agent_terms[my_agent][0] = is_crashed ? 1.0 : 0.0;
            st.agent_terms[my_agent][1] = clipd(scaled_speed, 0.0, 1.0);
            st.agent_terms[my_agent][2] = arrived ? 1.0 : 0.0;
            st.agent_terms[my_agent][3] = on_road ? 1.0 : 0.0;
            if (env_ok) {
                if (agents_reward) agents_reward[(size_t)e * A + my_agent] = rew;
                if (agents_terminated) agents_terminated[(size_t)e * A + my_agent] = (uint8_t)(is_crashed || arrived);
                S.speed_index[(size_t)e * A + my_agent] = my_speed_index;
            }
        }
        const unsigned gm = group_mask<G>();
        const bool any_crashed = __ballot_sync(gm, is_agent && is_crashed) != 0;
        const bool all_arrived = __ballot_sync(gm, is_agent && !arrived) == 0;
        group_sync<G>();
        if (i == ego && env_ok) {
            double sum = 0.0;
            for (int a = 0; a < A; ++a) sum = sum + st.agent_reward[a];
            double t = S.time[e] + 1.0 / P.policy_frequency;
            S.time[e] = t;
            reward[e] = sum / (double)A;
            if (S.reward_terms) {  // _rewards (intersection_env.py:67-77): every term averaged over the agents
                for (int k = 0; k < 4; ++k) {
                    double tk = 0.0;
                    for (int a = 0; a < A; ++a) tk = tk + st.agent_terms[a][k];
                    S.reward_terms[(size_t)e * HWY_REWARD_TERMS + k] = tk / (double)A;
                }
                S.reward_terms[(size_t)e * HWY_REWARD_TERMS + 4] = 0.0;
            }
            terminated[e] = (uint8_t)(any_crashed || all_arrived || (P.offroad_terminal && !on_road));
            truncated[e] = (uint8_t)(t >= P.duration);
            if (info_speed) info_speed[e] = r.speed;
            if (info_crashed) info_crashed[e] = (uint8_t)is_crashed;
        }
    } else if (i == ego && i < V && env_ok) {
        const HwyNetLane& L = g.lanes[st.lane[i]];
        const double es = st.own_s[i], elat = st.own_lat[i];
        const bool on_road = lane_on(L, es, elat, 0.0);
        const bool is_crashed = (r.meta & HWY_META_CRASHED) != 0;
        double rew = 0.0;
        bool term;
        double rt[HWY_REWARD_TERMS] = {0.0, 0.0, 0.0, 0.0, 0.0};  // un-weighted terms of _rewards (info["rewards"])
        if (P.reward_type == 1) {
            // envs/intersection_env.py:79-117,368-373 (one controlled vehicle)
            const bool arrived = L.exit_lane && es >= 25;
            double scaled_speed = lmap(r.speed, P.reward_speed_lo, P.reward_speed_hi, 0.0, 1.0);
            rew = rew + P.collision_reward * (is_crashed ? 1.0 : 0.0);
            rew = rew + P.high_speed_reward * clipd(scaled_speed, 0.0, 1.0);
            rew = rew + P.arrived_reward * (arrived ? 1.0 : 0.0);
            rew = rew + 0.0 * (on_road ? 1.0 : 0.0);
            if (arrived) rew = P.arrived_reward;
            rew *= on_road ? 1.0 : 0.0;
            if (P.normalize_reward) rew = lmap(rew, P.collision_reward, P.arrived_reward, 0.0, 1.0);
            term = is_crashed || arrived || (P.offroad_terminal && !on_road);
            rt[0] = is_crashed ? 1.0 : 0.0;
            rt[1] = clipd(scaled_speed, 0.0, 1.0);
            rt[2] = arrived ? 1.0 : 0.0;
            rt[3] = on_road ? 1.0 : 0.0;
        } else if (P.reward_type == 2) {
            // envs/merge_env.py:39-84: unclipped speed term, lane id of the CURRENT lane, altruistic penalty over the
            // ControlledVehicles on the merging lane ("b", "c", 2); never truncated, terminated past x = 370
            double scaled_speed = lmap(r.speed, P.reward_speed_lo, P.reward_speed_hi, 0.0, 1.0);
            double merging = 0.0;
            for (int v = 0; v < V; ++v)
                if (st.lane[v] == P.merge_lane && st.kind[v] != HWY_KIND_OBSTACLE)
                    merging = merging + (st.ts[v] - st.v[v]) / st.ts[v];
            rew = rew + P.collision_reward * (is_crashed ? 1.0 : 0.0);
            rew = rew + P.right_lane_reward * ((double)L.lane_id / 1.0);
            rew = rew + P.high_speed_reward * scaled_speed;
            rew = rew + P.lane_change_reward * ((act == 0 || act == 2) ? 1.0 : 0.0);
            rew = rew + P.merging_speed_reward * merging;
            rew = lmap(rew, P.collision_reward + P.merging_speed_reward, P.high_speed_reward + P.right_lane_reward, 0.0,
                       1.0);
            term = is_crashed || r.x > 370;
            rt[0] = is_crashed ? 1.0 : 0.0;
            rt[1] = (double)L.lane_id / 1.0;
            rt[2] = scaled_speed;
            rt[3] = (act == 0 || act == 2) ? 1.0 : 0.0;
            rt[4] = merging;
        } else if (P.reward_type == 5) {
            // envs/exit_env.py:147-198: collision, goal (the TARGET lane is the exit lane), clipped speed term, target
            // lane id; normalised to [collision_reward, goal_reward] and clipped to [0, 1]
            const int tl = st.tgt[i];
            const bool success = tl == P.exit_lane_a || tl == P.exit_lane_b;
            double scaled_speed = lmap(r.speed, P.reward_speed_lo, P.reward_speed_hi, 0.0, 1.0);
            rew = rew + P.collision_reward * (is_crashed ? 1.0 : 0.0);
            rew = rew + P.goal_reward * (success ? 1.0 : 0.0);
            rew = rew + P.high_speed_reward * clipd(scaled_speed, 0.0, 1.0);
            rew = rew + P.right_lane_reward * (double)g.lanes[tl].lane_id;
            if (P.normalize_reward) rew = clipd(lmap(rew, P.collision_reward, P.goal_reward, 0.0, 1.0), 0.0, 1.0);
            term = is_crashed;
            rt[0] = is_crashed ? 1.0 : 0.0;
            rt[1] = success ? 1.0 : 0.0;
            rt[2] = clipd(scaled_speed, 0.0, 1.0);
            rt[3] = (double)g.lanes[tl].lane_id;
        } else if (P.reward_type == 4) {
            // envs/u_turn_env.py:36-82: collision, current lane id (left-most = highest), clipped speed term;
            // normalised, then multiplied by on_road; truncated at `duration`
            const int n1 = L.road_count - 1 > 1 ? L.road_count - 1 : 1;
            double scaled_speed = lmap(r.speed, P.reward_speed_lo, P.reward_speed_hi, 0.0, 1.0);
            rew = rew + P.collision_reward * (is_crashed ? 1.0 : 0.0);
            rew = rew + P.left_lane_reward * ((double)L.lane_id / (double)n1);
            rew = rew + P.high_speed_reward * clipd(scaled_speed, 0.0, 1.0);
            rew = rew + 0.0 * (on_road ? 1.0 : 0.0);
            if (P.normalize_reward)
                rew = lmap(rew, P.collision_reward, P.high_speed_reward + P.left_lane_reward, 0.0, 1.0);
            rew *= on_road ? 1.0 : 0.0;
            term = is_crashed;
            rt[0] = is_crashed ? 1.0 : 0.0;
            rt[1] = (double)L.lane_id / (double)n1;
            rt[2] = clipd(scaled_speed, 0.0, 1.0);
            rt[3] = on_road ? 1.0 : 0.0;
        } else if (P.reward_type == 3) {
            // envs/two_way_env.py:35-62: speed index and how far left the TARGET lane is; never truncated
            const int n_side = L.road_count;  // all_side_lanes(vehicle.lane_index)
            rew = rew + P.high_speed_reward * ((double)st.speed_index / (double)(P.n_target_speeds - 1));
            rew = rew + P.left_lane_reward *
                            ((double)(n_side - 1 - g.lanes[st.tgt[i]].lane_id) / (double)(n_side - 1));
            term = is_crashed;
            rt[0] = (double)st.speed_index / (double)(P.n_target_speeds - 1);
            rt[1] = (double)(n_side - 1 - g.lanes[st.tgt[i]].lane_id) / (double)(n_side - 1);
        } else {
            // envs/roundabout_env.py:44-71
            rew = rew + P.collision_reward * (is_crashed ? 1.0 : 0.0);
            rew = rew + P.high_speed_reward * ((double)st.speed_index / (double)(3 - 1));
            rew = rew + P.lane_change_reward * ((act == 0 || act == 2) ? 1.0 : 0.0);
            rew = rew + 0.0 * (on_road ? 1.0 : 0.0);
            if (P.normalize_reward) rew = lmap(rew, P.collision_reward, P.high_speed_reward, 0.0, 1.0);
            rew *= on_road ? 1.0 : 0.0;
            term = is_crashed;
            rt[0] = is_crashed ? 1.0 : 0.0;
            rt[1] = (double)st.speed_index / (double)(3 - 1);
            rt[2] = (act == 0 || act == 2) ? 1.0 : 0.0;
            rt[3] = on_road ? 1.0 : 0.0;
        }
        if (S.reward_terms)
            for (int k = 0; k < HWY_REWARD_TERMS; ++k) S.reward_terms[(size_t)e * HWY_REWARD_TERMS + k] = rt[k];
        double t = S.time[e] + 1.0 / P.policy_frequency;
        S.time[e] = t;
        S.speed_index[e] = st.speed_index;
        reward[e] = rew;
        terminated[e] = (uint8_t)term;
        truncated[e] = (uint8_t)(t >= P.duration);
        if (info_speed) info_speed[e] = r.speed;
        if (info_crashed) info_crashed[e] = (uint8_t)is_crashed;
    }
    group_sync<G>();

    // ---- IntersectionEnv.step (intersection_env.py:136-140): _clear_vehicles, then _spawn_vehicle(p)
    int dst = i < V ? i : -1;
    if (REG && P.dynamic_population) {
        bool keep = i < V;
        if (keep && !is_controlled_kind(meta_kind(r.meta))) {  // _clear_vehicles :354-366
            const HwyNetLane& L = g.lanes[st.lane[i]];
            if (L.exit_lane && st.own_s[i] >= L.length - 4 * kVehLength) keep = false;
        }
        unsigned keep_mask = __ballot_sync(group_mask<G>(), keep) >> ((threadIdx.x & 31) & ~(G - 1));
        const int n_keep = __popc(keep_mask);
        dst = keep ? __popc(keep_mask & ((1u << i) - 1u)) : -1;
        if (i == 0) {
            Pcg64 rng = load_rng(S.rng, (size_t)S.n_envs, e);
            spawn_vehicle(P, SP, g, st, rng, keep_mask, 0.0, 1.0, 1.0, SP.spawn_probability, false);
            if (n_keep >= G && st.sp_ok) {  // every slot taken: the spawn is dropped, LOUDLY (the reference's list
                st.sp_ok = 0;               // is unbounded; it peaks at ~15-23 vehicles within the default 13 s)
                if (env_ok && S.overflow) S.overflow[e] += 1;
            }
            if (env_ok) store_rng(S.rng, (size_t)S.n_envs, e, rng);
        }
        group_sync<G>();
        if (env_ok) store_env(S, st, e, i, dst, r);
        group_sync<G>();
        spawn_closest_lane(g, st, i);
        if (st.sp_ok && i == n_keep) {
            adopt_spawn(P, SP, g, st, i, r);
            if (env_ok) store_env(S, st, e, i, i, r);
        }
        if (i == 0 && env_ok) {
            S.count[e] = n_keep + st.sp_ok;
            S.road_steps[e] = st.road_steps;
        }
    } else {
        if (env_ok) store_env(S, st, e, i, dst, r);
        if (REG && i == 0 && env_ok && S.road_steps) S.road_steps[e] = st.road_steps;
    }
}

template <int G, bool REG>
__global__ void __launch_bounds__(kBlockThreads)
network_observe_kernel(const __grid_constant__ HwyNetParams P, const HwyNetGraph* __restrict__ graph, const __grid_constant__ HwyNetState S,
                       const uint8_t* __restrict__ mask_a, const uint8_t* __restrict__ mask_b,
                       float* __restrict__ obs) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    GraphShared& g = *reinterpret_cast<GraphShared*>(smem_raw);
    EnvStage<G, REG>* stages =
        reinterpret_cast<EnvStage<G, REG>*>(smem_raw + ((sizeof(GraphShared) + 15) & ~size_t(15)));
    stage_graph(g, graph);
    constexpr int kEnvs = kBlockThreads / G;
    const int sub = threadIdx.x / G, i = threadIdx.x % G;
    const int env = blockIdx.x * kEnvs + sub;
    const bool env_ok = env < S.n_envs;
    const int e = env_ok ? env : S.n_envs - 1;
    EnvStage<G, REG>& st = stages[sub];
    Regs r;
    load_env(P, g, S, st, e, i, r);
    if (!env_selected(mask_a, mask_b, e)) return;  // whole group leaves together (selection is per env)
    observe_agents(P, g, st, i, obs + (size_t)e * n_agents_of(P) * obs_size(P));
}

// Test entries for the reference's own known-answer tests: Road.neighbour_vehicles(vehicle, lane) of every vehicle
// (tests/road/test_neighbour_vehicles.py) and utils.rotated_rectangles_intersect (tests/test_utils.py:19-27).
template <int G, bool REG>
__global__ void __launch_bounds__(kBlockThreads)
debug_neighbours_kernel(const __grid_constant__ HwyNetParams P, const HwyNetGraph* __restrict__ graph,
                        const __grid_constant__ HwyNetState S, const int32_t* __restrict__ query_lane,
                        int32_t* __restrict__ front, int32_t* __restrict__ rear) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    GraphShared& g = *reinterpret_cast<GraphShared*>(smem_raw);
    EnvStage<G, REG>* stages =
        reinterpret_cast<EnvStage<G, REG>*>(smem_raw + ((sizeof(GraphShared) + 15) & ~size_t(15)));
    stage_graph(g, graph);
    constexpr int kEnvs = kBlockThreads / G;
    const int sub = threadIdx.x / G, i = threadIdx.x % G;
    const int env = blockIdx.x * kEnvs + sub;
    const bool env_ok = env < S.n_envs;
    const int e = env_ok ? env : S.n_envs - 1;
    EnvStage<G, REG>& st = stages[sub];
    Regs r;
    load_env(P, g, S, st, e, i, r);
    int f = -1, rr = -1;
    const size_t slot = (size_t)e * S.vp + i;
    if (i < st.count) neighbours(g, st, st.count, i, query_lane ? query_lane[slot] : st.lane[i], P.connected_lanes != 0, f, rr);
    if (env_ok) {
        front[slot] = f;
        rear[slot] = rr;
    }
}
__global__ void debug_rectangles_kernel(const double* __restrict__ rects, int n, int32_t* __restrict__ out) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const double* q = rects + 10 * k;
    if (q[2] == q[7] && q[3] == q[8])  // equal sizes: the function the regulation step calls
        out[k] = rotated_rectangles_intersect(q[0], q[1], q[4], q[5], q[6], q[9], q[2], q[3]);
    else
        out[k] = has_corner_inside(q[0], q[1], q[2], q[3], q[4], q[5], q[6], q[7], q[8], q[9]) ||
                 has_corner_inside(q[5], q[6], q[7], q[8], q[9], q[0], q[1], q[2], q[3], q[4]);
}

// Road.act + Road.step `n_substeps` times with no ego action (IntersectionEnv._make_vehicles warm-up)
template <int G, bool REG>
__global__ void __launch_bounds__(kBlockThreads)
network_substeps_kernel(const __grid_constant__ HwyNetParams P, const HwyNetGraph* __restrict__ graph, const __grid_constant__ HwyNetState S,
                        const uint8_t* __restrict__ mask, int n_substeps) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    GraphShared& g = *reinterpret_cast<GraphShared*>(smem_raw);
    EnvStage<G, REG>* stages =
        reinterpret_cast<EnvStage<G, REG>*>(smem_raw + ((sizeof(GraphShared) + 15) & ~size_t(15)));
    stage_graph(g, graph);
    constexpr int kEnvs = kBlockThreads / G;
    const int sub = threadIdx.x / G, i = threadIdx.x % G;
    const int env_raw = blockIdx.x * kEnvs + sub;
    // substep() has block-wide phase barriers: a block leaves only as a whole; envs that are not selected ride
    // along (on a valid env's data) and store nothing
    const bool selected = env_raw < S.n_envs && (!mask || mask[env_raw]);
    if (!__syncthreads_or(selected)) return;
    const int env = env_raw < S.n_envs ? env_raw : S.n_envs - 1;
    EnvStage<G, REG>& st = stages[sub];
    Regs r;
    load_env(P, g, S, st, env, i, r);
    const double dt = 1.0 / P.simulation_frequency;
    double act_accel = 0.0, act_steer = 0.0;
    for (int k = 0; k < n_substeps; ++k) substep(P, g, st, i, r, act_accel, act_steer, dt, -1);
    group_sync<G>();
    if (!selected) return;
    store_env(S, st, env, i, i < st.count ? i : -1, r);
    if (i == 0 && S.road_steps) S.road_steps[env] = st.road_steps;
}

// work list of the envs to reset: list[0] = how many, list[1..] = env ids (any order)
__global__ void compact_envs_kernel(const uint8_t* __restrict__ mask_a, const uint8_t* __restrict__ mask_b, int n_envs,
                                    int* __restrict__ list) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    const bool sel = e < n_envs && env_selected(mask_a, mask_b, e);
    const unsigned m = __ballot_sync(0xffffffffu, sel);
    if (!m) return;
    const int lane = threadIdx.x & 31;
    int base = 0;
    if (lane == __ffs(m) - 1) base = atomicAdd(&list[0], __popc(m));
    base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
    if (sel) list[1 + base + __popc(m & ((1u << lane) - 1u))] = e;
}

// Two work lists for the step: envs whose population fits 16 slots even after this step's spawn (count <= 15)
// run two per warp; the rest use 32 slots.  small / large: [n_envs + 1] each, [0] = count (zeroed by the caller).
__global__ void classify_envs_kernel(const int* __restrict__ count, int n_envs, int* __restrict__ small,
                                     int* __restrict__ large) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    const bool ok = e < n_envs;
    const bool is_small = ok && count[e] <= 15;
    const int lane = threadIdx.x & 31;
    for (int pass = 0; pass < 2; ++pass) {
        const bool sel = ok && (pass == 0 ? is_small : !is_small);
        int* list = pass == 0 ? small : large;
        const unsigned m = __ballot_sync(0xffffffffu, sel);
        if (!m) continue;
        int base = 0;
        if (lane == __ffs(m) - 1) base = atomicAdd(&list[0], __popc(m));
        base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
        if (sel) list[1 + base + __popc(m & ((1u << lane) - 1u))] = e;
    }
}

// IntersectionEnv._make_vehicles (envs/intersection_env.py:245-323) for the listed envs, one 32-slot group each:
// n-1 _spawn_vehicle draws along the access roads, the 3 s warm-up simulation, the straight-going challenger, the
// controlled vehicle, and the 20 m pruning around it; then the fresh observation.  Dense over the work list: block
// b serves entries [8b, 8b+8) and leaves as a whole when there are none.
template <int G, bool REG>
__global__ void __launch_bounds__(kBlockThreads)
intersection_reset_kernel(const __grid_constant__ HwyNetParams P, const HwyNetGraph* __restrict__ graph, const __grid_constant__ HwyNetState S,
                          const __grid_constant__ HwyIntersectionSpawn SP, const int* __restrict__ list, float* __restrict__ obs) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    GraphShared& g = *reinterpret_cast<GraphShared*>(smem_raw);
    EnvStage<G, REG>* stages =
        reinterpret_cast<EnvStage<G, REG>*>(smem_raw + ((sizeof(GraphShared) + 15) & ~size_t(15)));
    const int kEnvs = blockDim.x / G;
    const int n_sel = list[0];
    if (blockIdx.x * kEnvs >= n_sel) return;  // uniform per block
    stage_graph(g, graph);
    const int sub = threadIdx.x / G, i = threadIdx.x % G;
    const int idx = blockIdx.x * kEnvs + sub;
    const bool selected = idx < n_sel;  // the others ride along on the last entry and store nothing
    const int e = list[1 + (selected ? idx : n_sel - 1)];
    EnvStage<G, REG>& st = stages[sub];

    Regs r = {};
    st.x[i] = st.y[i] = st.heading[i] = st.s[i] = st.v[i] = st.ts[i] = 0.0;
    st.c[i] = 1.0;
    st.lane[i] = st.tgt[i] = st.tgt_prev[i] = 0;
    st.kind[i] = HWY_KIND_IDM;
    st.route_len[i] = 0;
    st.own_s[i] = st.own_lat[i] = 0.0;
    Pcg64 rng;
    if (i == 0) {
        st.n_cand = 0;
        st.count = 0;
        st.ego = 0;
        st.speed_index = 0;
        st.road_steps = 0;
        st.sp_ok = 0;
        rng = load_rng(S.rng, (size_t)S.n_envs, e);
    }
    group_sync<G>();
    auto commit = [&](int kind) {  // the spawn record (if accepted) becomes vehicle number `count`
        group_sync<G>();
        spawn_closest_lane(g, st, i);
        if (st.sp_ok && i == st.count) adopt_spawn(P, SP, g, st, i, r, kind);
        group_sync<G>();
        if (i == 0 && st.sp_ok) st.count += 1;
        group_sync<G>();
    };
    // ---- :266-270  n_vehicles - 1 draws at np.linspace(0, 80, n_vehicles)[t]
    const int n0 = SP.initial_vehicle_count;
    for (int t = 0; t < n0 - 1; ++t) {
        if (i == 0) {
            const unsigned present = st.count >= 32 ? 0xffffffffu : ((1u << st.count) - 1u);
            // _make_vehicles calls _spawn_vehicle(longitudinal) with the FUNCTION default spawn_probability = 0.6
            // (intersection_env.py:268,331), not config["spawn_probability"] (used by the per-step spawn, :139)
            spawn_vehicle(P, SP, g, st, rng, present, (double)t * (80.0 / (double)(n0 - 1)), 1.0, 1.0, 0.6, false);
            if (st.count >= G && st.sp_ok) {
                st.sp_ok = 0;
                if (selected && S.overflow) S.overflow[e] += 1;
            }
        }
        commit(HWY_KIND_IDM);
    }
    // ---- :271-278  3 s of simulation under the RegulatedRoad rules
    const double dt = 1.0 / P.simulation_frequency;
    double act_accel = 0.0, act_steer = 0.0;
    for (int k = 0; k < 3 * P.simulation_frequency; ++k) substep(P, g, st, i, r, act_accel, act_steer, dt, -1);
    group_sync<G>();
    // ---- :281-288  the challenger: certain, going straight, tight deviations
    if (i == 0) {
        const unsigned present = st.count >= 32 ? 0xffffffffu : ((1u << st.count) - 1u);
        spawn_vehicle(P, SP, g, st, rng, present, 60.0, 0.1, 0.0, 1.0, true);
        if (st.count >= G && st.sp_ok) {
            st.sp_ok = 0;
            if (selected && S.overflow) S.overflow[e] += 1;
        }
    }
    commit(HWY_KIND_IDM);
    // ---- :291-315  the controlled vehicles, one per access road ("o{k}", "ir{k}", 0), k = agent % 4
    const int A = n_agents_of(P);
    for (int agent = 0; agent < A; ++agent) {
        if (i == 0) {
            const int dest = SP.ego_destination >= 0 ? SP.ego_destination : 1 + rng.choice(3);  // "o" + integers(1, 4)
            const HwyNetLane& EL = g.lanes[SP.spawn_lane[agent % 4]];
            const double lon = 60.0 + 5.0 * (1.0 + 1.0 * rng.normal());  // 60 + 5 * np_random.normal(1)
            lane_position(EL, lon, 0.0, st.sp_x, st.sp_y);
            st.sp_h = lane_heading_at(EL, 60.0);
            st.sp_speed = EL.speed_limit;
            st.sp_dest = dest;  // sp_lane: spawn_closest_lane inside commit()
            // MDPVehicle.__init__ (controller.py:283-293); a plain Vehicle has no speed index (-1 in the state)
            const int si0 = speed_to_index(P, st.sp_speed);
            st.speed_index = P.action_type == 1 ? -1 : si0;
            st.sp_ts = P.target_speeds[si0];
            st.sp_ok = st.count < G ? 1 : 0;
            if (!st.sp_ok && selected && S.overflow) S.overflow[e] += 1;
            if (agent == 0) st.ego = st.count;
        }
        // action_type.vehicle_class (:291-300): MDPVehicle, or Vehicle / BicycleVehicle for a ContinuousAction
        commit(P.action_type == 1 ? HWY_KIND_VEHICLE : HWY_KIND_MDP);
    }
    // ---- :317-323  after each controlled vehicle the TRAFFIC within 20 m of it is dropped; controlled vehicles are
    // never dropped and their creation does not look at the others, so all prunings can run at the end
    const int V = st.count;
    bool keep = i < V;
    if (keep && !is_controlled_kind(st.kind[i])) {
        for (int v = 0; v < V; ++v)
            if (is_controlled_kind(st.kind[v]) && norm2(st.x[i] - st.x[v], st.y[i] - st.y[v]) < 20) keep = false;
    }
    const unsigned keep_mask = __ballot_sync(group_mask<G>(), keep) >> ((threadIdx.x & 31) & ~(G - 1));
    const int dst = keep ? __popc(keep_mask & ((1u << i) - 1u)) : -1;
    if (!selected) return;  // no block-wide barrier below this line
    store_env(S, st, e, i, dst, r);
    if (i == 0) {
        S.count[e] = __popc(keep_mask);
        S.road_steps[e] = st.road_steps;
        for (int agent = 0; agent < A; ++agent) S.speed_index[(size_t)e * A + agent] = st.speed_index;
        S.time[e] = 0.0;
        store_rng(S.rng, (size_t)S.n_envs, e, rng);
    }
    if (!obs) return;
    group_sync<G>();  // the stored state is re-read by other threads of the group
    load_env(P, g, S, st, e, i, r);
    observe_agents(P, g, st, i, obs + (size_t)e * A * obs_size(P));
}

// ------------------------------------------------------------------ the scripted resets
// The _make_vehicles of roundabout, merge, exit, u-turn and two-way: a fixed placement drawn from the env's numpy
// stream, for the envs the masks select.  Each family kernel keeps its own placement and draw order; the helpers
// below are the rest.

// RoadObject.__init__ (objects.py:46-50): the closest lane, first minimum in graph-enumeration order
__device__ __forceinline__ int closest_lane(const HwyNetGraph* graph, double x, double y, double heading) {
    int lane = 0;
    double bd = 0;
    for (int l = 0; l < graph->n_lanes; ++l) {
        const double d = lane_distance_with_heading(graph->lanes[l], x, y, heading);
        if (l == 0 || d < bd) {
            bd = d;
            lane = l;
        }
    }
    return lane;
}

// One placed vehicle into slot k, with no impact; IDM vehicles get IDMVehicle.__init__'s lane-change timer
// (behavior.py:64).  `flags`: further meta bits (HWY_META_NO_LANE_CHANGE).
__device__ __forceinline__ void store_vehicle(const HwyNetParams& P, const HwyNetState& S, size_t k, double px,
                                              double py, double heading, double speed, double target_speed,
                                              double delta, int lane, int target, int kind, int flags = 0) {
    const double timer = kind == HWY_KIND_IDM ? py_mod_pos((px + py) * kPi, P.lane_change_delay) : 0.0;
    reinterpret_cast<double2*>(S.pos)[k] = make_double2(px, py);
    reinterpret_cast<double2*>(S.hs)[k] = make_double2(heading, speed);
    reinterpret_cast<double2*>(S.tt)[k] = make_double2(target_speed, timer);
    reinterpret_cast<double2*>(S.imp)[k] = make_double2(0.0, 0.0);
    S.delta[k] = delta;
    S.meta[k] = (lane << HWY_META_LANE_SHIFT) | (target << HWY_META_TARGET_SHIFT) | HWY_META_CHECK_COLLISIONS |
                (kind << HWY_META_KIND_SHIFT) | HWY_META_PRESENT | flags;
}

// The per-env end of a scripted reset: the ego's speed index, the clock, the advanced stream, and the population
// and RegulatedRoad clock where the state has them (the 32-slot state of exit-v0)
__device__ __forceinline__ void store_env_tail(const HwyNetState& S, uint64_t* rng, int e, int speed_index, int count,
                                               const Pcg64& g) {
    S.speed_index[e] = speed_index;
    S.time[e] = 0.0;
    if (S.count) S.count[e] = count;
    if (S.road_steps) S.road_steps[e] = 0;
    store_rng(rng, (size_t)S.n_envs, e, g);
}

// RoundaboutEnv._make_vehicles (envs/roundabout_env.py:317-391), one env per WARP.  The draws are a sequential chain
// on the env's numpy stream: every lane of the warp walks it redundantly (same instructions, same values — no
// shuffles), and the expensive part, RoadObject.__init__'s closest-lane search over all 32 lanes of the network for
// each of the 5 vehicles (objects.py:46-50), is spread over the warp: lane l evaluates graph lane l, then a
// (distance, index) minimum over the warp = np.argmin's first minimum (one thread per env made the reset a large share
// of a cfg 4 step).
__global__ void __launch_bounds__(128)
roundabout_reset_kernel(const __grid_constant__ HwyNetParams P, const HwyNetGraph* __restrict__ graph, const __grid_constant__ HwyRoundaboutSpawn SP,
                        const __grid_constant__ HwyNetState S, uint64_t* __restrict__ rng, const uint8_t* __restrict__ mask_a,
                        const uint8_t* __restrict__ mask_b) {
    const int e = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int wl = threadIdx.x & 31;
    if (e >= S.n_envs || !env_selected(mask_a, mask_b, e)) return;  // warp-uniform
    Pcg64 g = load_rng(rng, (size_t)S.n_envs, e);
    const size_t base = (size_t)e * S.vp;
    for (int v = 0; v < P.n_vehicles; ++v) {
        const bool is_ego = v == 0;
        double px, py, heading, speed, delta = 4.0;
        int dest = 3;
        if (is_ego) {
            const HwyNetLane& L = graph->lanes[SP.ego_lane];
            lane_position(L, SP.ego_longitudinal, 0.0, px, py);
            heading = lane_heading_at(L, SP.ego_heading_longitudinal);
            speed = SP.ego_speed;
        } else {
            const int j = v - 1;
            const HwyNetLane& L = graph->lanes[SP.spawn_lane[j]];
            double lon = SP.base_longitudinal[j] + g.normal() * SP.position_deviation;
            speed = SP.traffic_speed + g.normal() * SP.speed_deviation;
            dest = (j == 0 && SP.fixed_destination >= 0) ? SP.fixed_destination : g.choice(3);
            delta = g.uniform(SP.delta_lo, SP.delta_hi);
            lane_position(L, lon, 0.0, px, py);  // make_on_lane (vehicle/objects.py:68-90)
            heading = lane_heading_at(L, lon);
        }
        // closest_lane over the warp
        double bd = INFINITY;
        int lane = 0x7fffffff;
        for (int l = wl; l < graph->n_lanes; l += 32) {
            const double d = lane_distance_with_heading(graph->lanes[l], px, py, heading);
            if (lane == 0x7fffffff || d < bd) {
                bd = d;
                lane = l;
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const double d2 = __shfl_xor_sync(0xffffffffu, bd, off);
            const int l2 = __shfl_xor_sync(0xffffffffu, lane, off);
            if (l2 != 0x7fffffff && (lane == 0x7fffffff || d2 < bd || (d2 == bd && l2 < lane))) {
                bd = d2;
                lane = l2;
            }
        }
        if (wl == 0) {
            store_vehicle(P, S, base + v, px, py, heading, speed, is_ego ? P.target_speeds[SP.ego_speed_index] : speed,
                          delta, lane, lane, is_ego ? HWY_KIND_MDP : HWY_KIND_IDM);
            S.route_len[base + v] = SP.route_len[(size_t)lane * 4 + dest];
        }
        const int* rsrc = SP.route_table + ((size_t)lane * 4 + dest) * R;
        int* rdst = S.route + (base + v) * R;
        for (int k = wl; k < R; k += 32) rdst[k] = rsrc[k];
    }
    if (wl == 0) store_env_tail(S, rng, e, SP.ego_speed_index, P.n_vehicles, g);
}

// MergeEnv._make_vehicles and the ramp's Obstacle (envs/merge_env.py:150-190), one env per thread
__global__ void __launch_bounds__(128)
merge_reset_kernel(const __grid_constant__ HwyNetParams P, const HwyNetGraph* __restrict__ graph,
                   const __grid_constant__ HwyMergeSpawn SP, const __grid_constant__ HwyNetState S,
                   uint64_t* __restrict__ rng, const uint8_t* __restrict__ mask_a, const uint8_t* __restrict__ mask_b) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= S.n_envs || !env_selected(mask_a, mask_b, e)) return;
    Pcg64 g = load_rng(rng, (size_t)S.n_envs, e);
    const size_t base = (size_t)e * S.vp;
    const double base_position[3] = {90.0, 70.0, 5.0}, base_speed[3] = {29.0, 31.0, 31.5};
    for (int v = 0; v < 6; ++v) {
        double px, py, speed, target_speed;
        int kind = HWY_KIND_IDM;
        if (v == 0) {  // :158-161 ego = action_type.vehicle_class(road, ("a","b",1).position(30, 0), speed=30)
            lane_position(graph->lanes[SP.lane_ab[1]], 30.0, 0.0, px, py);
            speed = 30.0;
            kind = HWY_KIND_MDP;
            target_speed = P.target_speeds[SP.ego_speed_index];
        } else if (v <= 3) {  // :165-169
            const HwyNetLane& L = graph->lanes[SP.lane_ab[g.choice(2)]];  // np_random.integers(2)
            lane_position(L, base_position[v - 1] + g.uniform(-5.0, 5.0), 0.0, px, py);
            speed = base_speed[v - 1] + g.uniform(-1.0, 1.0);
            target_speed = speed;
        } else if (v == 4) {  // :171-175 the merging vehicle
            lane_position(graph->lanes[SP.lane_jk], 110.0, 0.0, px, py);
            speed = 20.0;
            target_speed = 30.0;
        } else {  // _make_road :147: Obstacle(road, lbc.position(ends[2], 0))
            px = SP.obstacle_x;
            py = SP.obstacle_y;
            speed = target_speed = 0.0;
            kind = HWY_KIND_OBSTACLE;
        }
        const int lane = closest_lane(graph, px, py, 0.0);  // at heading 0
        // DELTA 4: randomize_behavior is not called here
        store_vehicle(P, S, base + v, px, py, 0.0, speed, target_speed, 4.0, lane, lane, kind);
        S.route_len[base + v] = 0;
    }
    store_env_tail(S, rng, e, SP.ego_speed_index, P.n_vehicles, g);
}

// ExitEnv._create_vehicles (envs/exit_env.py:107-145), one env per thread (the longitudinal positions are a running
// maximum over the vehicles created so far).  Draws per traffic vehicle: Generator.choice(lanes, p=lanes / lanes.sum())
// = one random() searched in the normalised cumulative sum (numpy's legacy-free choice with p), then create_random's
// uniform(0.9, 1.1); the ego draws only the latter.  No randomize_behavior: DELTA stays 4.
__global__ void __launch_bounds__(128)
exit_reset_kernel(const __grid_constant__ HwyNetParams P, const HwyNetGraph* __restrict__ graph,
                  const __grid_constant__ HwyExitSpawn SP, const __grid_constant__ HwyNetState S,
                  uint64_t* __restrict__ rng, const uint8_t* __restrict__ mask_a, const uint8_t* __restrict__ mask_b) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= S.n_envs || !env_selected(mask_a, mask_b, e)) return;
    Pcg64 g = load_rng(rng, (size_t)S.n_envs, e);
    const size_t base = (size_t)e * S.vp;
    double x_max = 0.0;
    for (int v = 0; v < SP.n_vehicles; ++v) {
        const bool is_ego = v == 0;
        int lane_id = 0;
        if (!is_ego) {  // cdf.searchsorted(random(), side="right")
            const double u = g.next_double();
            lane_id = 0;
            for (int k = 0; k < SP.lanes_count; ++k) lane_id += SP.cdf[k] <= u;
            lane_id = min(lane_id, SP.lanes_count - 1);
        }
        const HwyNetLane& L = graph->lanes[lane_id];  // ("0", "1", lane_id): the first road of the table
        const double speed = is_ego ? SP.ego_speed : L.speed_limit;
        const double spacing = is_ego ? SP.ego_spacing : 1 / SP.vehicles_density;
        const double default_spacing = 12 + 1.0 * speed;
        const double offset = spacing * default_spacing * SP.spawn_exp;
        double x0 = v > 0 ? x_max : 3 * offset;  // np.max of the local longitudinal coordinates (the lanes are aligned)
        x0 += offset * g.uniform(0.9, 1.1);
        double px, py;
        lane_position(L, x0, 0.0, px, py);
        const double heading = L.heading;
        const double s_here = lane_s_of(graph->lanes[0], px, py);
        x_max = v == 0 ? s_here : fmax(x_max, s_here);
        const int lane = closest_lane(graph, px, py, heading);
        if (is_ego) {  // MDPVehicle.__init__ (controller.py:283-293); no route
            store_vehicle(P, S, base + v, px, py, heading, speed, P.target_speeds[SP.ego_speed_index], 4.0, lane, lane,
                          HWY_KIND_MDP);
            S.route_len[base + v] = 0;
        } else {  // vehicle.enable_lane_change = False (:143)
            store_vehicle(P, S, base + v, px, py, heading, speed, speed, 4.0, lane, lane, HWY_KIND_IDM,
                          HWY_META_NO_LANE_CHANGE);
            const HwyNetLane& CL = graph->lanes[lane];  // plan_route_to("3") (controller.py:71-87)
            int* route = S.route + (base + v) * R;
            route[0] = CL.from_node | (CL.to_node << 8) | ((CL.lane_id + 1) << 16);
            route[1] = SP.route_12;
            route[2] = SP.route_23;
            S.route_len[base + v] = 3;
        }
    }
    store_env_tail(S, rng, e, SP.ego_speed_index, SP.n_vehicles, g);
}

// UTurnEnv._make_vehicles (envs/u_turn_env.py:179-275), one env per thread: the MDPVehicle at the start of
// ("a","b",0) and six IDM vehicles made on fixed lanes with normal-jittered longitudinal / speed, all routed to "d"
__global__ void __launch_bounds__(128)
u_turn_reset_kernel(const __grid_constant__ HwyNetParams P, const HwyNetGraph* __restrict__ graph,
                    const __grid_constant__ HwyUTurnSpawn SP, const __grid_constant__ HwyNetState S,
                    uint64_t* __restrict__ rng, const uint8_t* __restrict__ mask_a, const uint8_t* __restrict__ mask_b) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= S.n_envs || !env_selected(mask_a, mask_b, e)) return;
    Pcg64 g = load_rng(rng, (size_t)S.n_envs, e);
    const size_t base = (size_t)e * S.vp;
    for (int v = 0; v < 7; ++v) {
        double px, py, heading, speed, target_speed, delta = 4.0;
        int kind = HWY_KIND_IDM;
        if (v == 0) {  // :189-201 ego = vehicle_class(road, ("a","b",0).position(0, 0), speed=16)
            lane_position(graph->lanes[SP.lane[0]], 0.0, 0.0, px, py);
            heading = 0.0;
            speed = 16.0;
            kind = HWY_KIND_MDP;
            target_speed = P.target_speeds[SP.ego_speed_index];
        } else {  // make_on_lane (vehicle/objects.py:68-90) with longitudinal + normal * 2, speed + normal * 2
            const HwyNetLane& L = graph->lanes[SP.lane[v]];
            const double lon = SP.longitudinal[v] + g.normal() * 2.0;
            speed = SP.speed[v] + g.normal() * 2.0;
            lane_position(L, lon, 0.0, px, py);
            heading = lane_heading_at(L, lon);
            target_speed = speed;
            if (v == 1) delta = g.uniform(3.5, 4.5);  // only vehicle 1 calls randomize_behavior (:218)
        }
        const int lane = closest_lane(graph, px, py, heading);
        store_vehicle(P, S, base + v, px, py, heading, speed, target_speed, delta, lane, lane, kind);
        const int* rsrc = SP.route_table + (size_t)lane * R;  // plan_route_to("d") from the closest lane
        int* rdst = S.route + (base + v) * R;
        for (int k = 0; k < R; ++k) rdst[k] = rsrc[k];
        S.route_len[base + v] = SP.route_len[lane];
    }
    store_env_tail(S, rng, e, SP.ego_speed_index, P.n_vehicles, g);
}

// TwoWayEnv._make_vehicles (envs/two_way_env.py:113-158), one env per thread
__global__ void __launch_bounds__(128)
two_way_reset_kernel(const __grid_constant__ HwyNetParams P, const HwyNetGraph* __restrict__ graph,
                     const __grid_constant__ HwyTwoWaySpawn SP, const __grid_constant__ HwyNetState S,
                     uint64_t* __restrict__ rng, const uint8_t* __restrict__ mask_a, const uint8_t* __restrict__ mask_b) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= S.n_envs || !env_selected(mask_a, mask_b, e)) return;
    Pcg64 g = load_rng(rng, (size_t)S.n_envs, e);
    const size_t base = (size_t)e * S.vp;
    for (int v = 0; v < 6; ++v) {
        double px, py, heading, speed, target_speed;
        int kind = HWY_KIND_IDM, flags = HWY_META_NO_LANE_CHANGE;
        if (v == 0) {  // :120-123 ego on ("a","b",1) at s = 30, speed 30
            const HwyNetLane& L = graph->lanes[SP.lane_ab1];
            lane_position(L, 30.0, 0.0, px, py);
            heading = 0.0;
            speed = 30.0;
            kind = HWY_KIND_MDP;
            flags = 0;
            target_speed = P.target_speeds[SP.ego_speed_index];
        } else if (v <= 3) {  // :126-144 three vehicles ahead on the same lane
            const HwyNetLane& L = graph->lanes[SP.lane_ab1];
            const double i = (double)(v - 1);
            lane_position(L, 70.0 + 40.0 * i + 10.0 * g.normal(), 0.0, px, py);
            heading = lane_heading_at(L, 70.0 + 40.0 * i);
            speed = 24.0 + 2.0 * g.normal();
            target_speed = speed;
        } else {  // :145-158 two oncoming vehicles on ("b","a",0)
            const HwyNetLane& L = graph->lanes[SP.lane_ba0];
            const double i = (double)(v - 4);
            lane_position(L, 200.0 + 100.0 * i + 10.0 * g.normal(), 0.0, px, py);
            heading = lane_heading_at(L, 200.0 + 100.0 * i);
            speed = 20.0 + 5.0 * g.normal();
            target_speed = speed;
        }
        const int lane = closest_lane(graph, px, py, heading);
        const int target = v >= 4 ? SP.lane_ba0 : lane;  // :157 v.target_lane_index = ("b", "a", 0)
        store_vehicle(P, S, base + v, px, py, heading, speed, target_speed, 4.0, lane, target, kind, flags);
        S.route_len[base + v] = 0;
    }
    store_env_tail(S, rng, e, SP.ego_speed_index, P.n_vehicles, g);
}

}  // namespace hwynet

// ====================================================================== C ABI
namespace {
using hwy_abi::check_launch;
using hwy_abi::fail;

int validate_net(const HwyNetParams* p, const HwyNetGraph* graph, const HwyNetState* s) {
    if (!p || !graph || !s) return fail("%s", "null params/graph/state");
    if (s->vp != HWY_NET_GROUP && s->vp != HWY_NET_GROUP_LARGE) return fail("%s", "slot stride must be 8 or 32");
    if (p->n_vehicles < 1 || p->n_vehicles > s->vp) return fail("%s", "n_vehicles out of range for the network kernels");
    if (p->n_target_speeds < 1 || p->n_target_speeds > 3) return fail("%s", "network kernels support up to 3 target speeds");
    if (p->obs_type != HWY_OBS_KINEMATICS && p->obs_type != HWY_OBS_TTC && p->obs_type != HWY_OBS_OCCUPANCY)
        return fail("%s", "unknown obs_type");
    if (p->obs_type == HWY_OBS_TTC && (p->ttc_horizon * p->policy_frequency < 1 || p->ttc_horizon * p->policy_frequency > 16))
        return fail("%s", "ttc horizon out of range");
    if (p->obs_type == HWY_OBS_KINEMATICS && (p->obs_vehicles_count < 1 || p->obs_vehicles_count > 32))
        return fail("%s", "obs_vehicles_count out of range");
    if (p->simulation_frequency < 1 || p->policy_frequency < 1 || p->simulation_frequency < p->policy_frequency)
        return fail("%s", "bad simulation/policy frequency");
    if (s->n_envs < 1) return fail("%s", "n_envs < 1");
    if (!s->pos || !s->hs || !s->tt || !s->imp || !s->delta || !s->meta || !s->route || !s->route_len ||
        !s->speed_index || !s->time)
        return fail("%s", "null state pointer");
    if (s->vp == HWY_NET_GROUP_LARGE && (!s->count || !s->road_steps)) return fail("%s", "count / road_steps required");
    if (p->n_agents < 0 || p->n_agents > 4) return fail("%s", "n_agents out of range (0..4)");
    int dev_count = 0;
    if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count < 1) {
        cudaGetLastError();
        return fail("%s", "no CUDA device: this library has no CPU fallback");
    }
    return 0;
}

// one side stream (+ fork / join events) per device, created on first use
struct SideStream {
    cudaStream_t stream;
    cudaEvent_t fork, join;
};
SideStream* side_stream() {
    static std::mutex mu;
    static SideStream* table[64] = {nullptr};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) {
        fail("%s", "cudaGetDevice failed");
        return nullptr;
    }
    std::lock_guard<std::mutex> lock(mu);
    if (!table[dev]) {
        SideStream* s = new SideStream;
        if (cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaEventCreateWithFlags(&s->fork, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&s->join, cudaEventDisableTiming) != cudaSuccess) {
            fail("%s", "side stream creation failed");
            delete s;
            return nullptr;
        }
        table[dev] = s;
    }
    return table[dev];
}

// Dynamic shared memory of a block of `per` envs on G slots: the staged lane table, then one EnvStage per env
template <int G, bool REG>
size_t stage_smem_bytes(int per) {
    return ((sizeof(hwynet::GraphShared) + 15) & ~size_t(15)) + (size_t)per * sizeof(hwynet::EnvStage<G, REG>);
}
template <typename K>
int configure_smem(K kernel, size_t bytes) {
    cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (err != cudaSuccess) return fail("cudaFuncSetAttribute: %s", cudaGetErrorString(err));
    return 0;
}
int blocks_for(int n_envs, int g) {
    int per = hwynet::kBlockThreads / g;
    return (n_envs + per - 1) / per;
}

// Block shape of a step launch: the fewest whole waves of one block per SM that cover n_envs, the envs spread evenly
// over waves x SMs blocks (6 336 roundabout envs, 8 slots, 132 SMs: 132 blocks of 48 envs = 384 threads instead of 99
// blocks of 64 envs).  Work-list launches (16- / 32-slot intersection kernels) are planned for n_envs, the upper
// bound of a list known only on the device; blocks past the list's end leave at once.
struct StepPlan {
    int threads, blocks, per;
    size_t smem;
};
int sm_count() {
    static std::atomic<int> cached[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    int n = cached[dev].load(std::memory_order_relaxed);
    if (n == 0) {
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        cached[dev].store(n, std::memory_order_relaxed);
    }
    return n;
}
template <int G, bool REG>
StepPlan step_plan(int n_envs) {
    const int per_max = hwynet::kStepThreads / G, sms = sm_count();
    const int waves = (n_envs + sms * per_max - 1) / (sms * per_max);
    int per = (n_envs + waves * sms - 1) / (waves * sms);
    int threads = ((per * G + 31) / 32) * 32;
    if (threads > hwynet::kStepThreads) threads = hwynet::kStepThreads;
    per = threads / G;
    StepPlan plan;
    plan.threads = threads;
    plan.per = per;
    plan.blocks = (n_envs + per - 1) / per;
    plan.smem = stage_smem_bytes<G, REG>(per);
    return plan;
}

template <int G, bool REG>
int launch_step(const HwyNetParams* p, const HwyNetGraph* graph, const HwyIntersectionSpawn& sp, const HwyNetState* s,
                const int32_t* action, float* obs, double* reward, uint8_t* terminated, uint8_t* truncated,
                double* info_speed, uint8_t* info_crashed, cudaStream_t st, const int* list = nullptr,
                double* agents_reward = nullptr, uint8_t* agents_terminated = nullptr) {
    const StepPlan plan = step_plan<G, REG>(s->n_envs);
    const size_t smem_max = stage_smem_bytes<G, REG>(hwynet::kStepThreads / G);
    if constexpr (REG) {
        if (p->action_type == 1) {  // a ContinuousAction ego (plain Vehicle / BicycleVehicle): its own instantiation
            if (configure_smem(hwynet::network_step_kernel<G, REG, true>, smem_max)) return 1;
            hwynet::network_step_kernel<G, REG, true><<<plan.blocks, plan.threads, plan.smem, st>>>(
                *p, graph, *s, sp, action, obs, reward, terminated, truncated, info_speed, info_crashed, list,
                agents_reward, agents_terminated);
            return check_launch("network_step_kernel");
        }
    }
    if (p->action_type == 1) return fail("%s", "ContinuousAction is implemented on the intersection family (32-slot state)");
    if (configure_smem(hwynet::network_step_kernel<G, REG, false>, smem_max)) return 1;
    hwynet::network_step_kernel<G, REG, false><<<plan.blocks, plan.threads, plan.smem, st>>>(
        *p, graph, *s, sp, action, obs, reward, terminated, truncated, info_speed, info_crashed, list, agents_reward,
        agents_terminated);
    return check_launch("network_step_kernel");
}

template <int G_, bool REG_>
struct Slots {
    static constexpr int G = G_;
    static constexpr bool REG = REG_;
};
// One launch of a 256-thread group kernel (observe, substeps, debug neighbours) on the state's slot stride:
// kernel_for(Slots<G, REG>{}) names the kernel's <G, REG> instantiation, <8, false> for the 8-slot state and
// <32, true> for the 32-slot one.
template <typename KernelFor, typename... Args>
int launch_groups(KernelFor kernel_for, const char* name, const HwyNetState* s, cudaStream_t st, const Args&... args) {
    auto launch = [&](auto slots) {
        using T = decltype(slots);
        const auto kernel = kernel_for(slots);
        const size_t smem = stage_smem_bytes<T::G, T::REG>(hwynet::kBlockThreads / T::G);
        if (configure_smem(kernel, smem)) return 1;
        kernel<<<blocks_for(s->n_envs, T::G), hwynet::kBlockThreads, smem, st>>>(args...);
        return check_launch(name);
    };
    if (s->vp == HWY_NET_GROUP) return launch(Slots<HWY_NET_GROUP, false>{});
    return launch(Slots<HWY_NET_GROUP_LARGE, true>{});
}
int observe_dispatch(const HwyNetParams* p, const HwyNetGraph* graph, const HwyNetState* s, const uint8_t* mask_a,
                     const uint8_t* mask_b, float* obs, cudaStream_t st) {
    return launch_groups([](auto t) { return hwynet::network_observe_kernel<decltype(t)::G, decltype(t)::REG>; },
                         "network_observe_kernel", s, st, *p, graph, *s, mask_a, mask_b, obs);
}

// The reset is a long dependent chain per env (9 spawn attempts, 45 warm-up substeps, ...) for the few envs that
// ended (~8 % per step): 64-thread blocks (4 envs on 16 slots, 2 on 32) spread them over all SMs and shorten the
// lock-step waits.
template <int G>
int launch_intersection_reset(const HwyNetParams* p, const HwyNetGraph* graph, const HwyIntersectionSpawn* spawn,
                              const HwyNetState* s, float* obs, cudaStream_t st) {
    constexpr int kThreads = 64, per = kThreads / G;
    const size_t smem = stage_smem_bytes<G, true>(per);
    if (configure_smem(hwynet::intersection_reset_kernel<G, true>, smem)) return 1;
    hwynet::intersection_reset_kernel<G, true>
        <<<(s->n_envs + per - 1) / per, kThreads, smem, st>>>(*p, graph, *s, *spawn, spawn->scratch, obs);
    return check_launch("intersection_reset_kernel");
}

// A scripted reset: the family kernel over 128-thread blocks, `threads_per_env` (1, or 32 for roundabout) per env,
// then the fresh observation of the envs it reset
template <typename K, typename Spawn>
int scripted_reset(K kernel, const char* name, int threads_per_env, const HwyNetParams* p, const HwyNetGraph* graph,
                   const Spawn* spawn, const HwyNetState* s, uint64_t* rng, const uint8_t* mask_a,
                   const uint8_t* mask_b, float* obs, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    const int per = 128 / threads_per_env;
    kernel<<<(s->n_envs + per - 1) / per, 128, 0, st>>>(*p, graph, *spawn, *s, rng, mask_a, mask_b);
    if (check_launch(name)) return 1;
    return obs ? observe_dispatch(p, graph, s, mask_a, mask_b, obs, st) : 0;
}
}  // namespace

extern "C" {

int hwy_network_obs_size(const HwyNetParams* p) {
    if (!p) return 0;
    const int agents = p->n_agents > 1 ? p->n_agents : 1;  // one observation per controlled vehicle
    if (p->obs_type == HWY_OBS_OCCUPANCY) return agents * 4 * 11 * 11;
    if (p->obs_type == HWY_OBS_TTC) return agents * 9 * (int)(p->ttc_horizon / (1.0 / p->policy_frequency));
    return agents * p->obs_vehicles_count * (p->obs_n_feat > 0 ? p->obs_n_feat : (p->obs_features == 7 ? 7 : 5));
}

int hwy_network_step(const HwyNetParams* p, const HwyNetGraph* graph, const HwyNetState* s,
                     const int32_t* action, float* obs, double* reward, uint8_t* terminated,
                     uint8_t* truncated, double* info_speed, uint8_t* info_crashed, void* stream) {
    if (validate_net(p, graph, s)) return 1;
    if (!action || !obs || !reward || !terminated || !truncated) return fail("%s", "null pointer");
    if (s->vp != HWY_NET_GROUP) return fail("%s", "hwy_network_step expects slot stride 8 (use hwy_intersection_step)");
    HwyIntersectionSpawn none = {};
    return launch_step<HWY_NET_GROUP, false>(p, graph, none, s, action, obs, reward, terminated, truncated,
                                             info_speed, info_crashed, (cudaStream_t)stream);
}

int hwy_intersection_step(const HwyNetParams* p, const HwyNetGraph* graph, const HwyIntersectionSpawn* spawn,
                          const HwyNetState* s, const int32_t* action, float* obs, double* reward,
                          uint8_t* terminated, uint8_t* truncated, double* info_speed, uint8_t* info_crashed,
                          void* stream) {
    return hwy_intersection_step_agents(p, graph, spawn, s, action, obs, reward, terminated, truncated, info_speed,
                                        info_crashed, nullptr, nullptr, stream);
}

int hwy_intersection_step_agents(const HwyNetParams* p, const HwyNetGraph* graph, const HwyIntersectionSpawn* spawn,
                                 const HwyNetState* s, const int32_t* action, float* obs, double* reward,
                                 uint8_t* terminated, uint8_t* truncated, double* info_speed, uint8_t* info_crashed,
                                 double* agents_reward, uint8_t* agents_terminated, void* stream) {
    if (validate_net(p, graph, s)) return 1;
    if (p->n_agents > 1 && (p->obs_type != HWY_OBS_KINEMATICS || p->reward_type != 1))
        return fail("%s", "several controlled vehicles: Kinematics observation on intersection envs only");
    if (!action || !obs || !reward || !terminated || !truncated) return fail("%s", "null pointer");
    if (s->vp != HWY_NET_GROUP_LARGE) return fail("%s", "hwy_intersection_step expects slot stride 32");
    if (p->dynamic_population && (!spawn || !spawn->route_table || !spawn->route_len || !s->rng))
        return fail("%s", "dynamic population needs the spawn tables and the rng words");
    HwyIntersectionSpawn none = {};
    cudaStream_t st = (cudaStream_t)stream;
    if (spawn && spawn->scratch && s->count) {
        // populations of <= 15 vehicles (nearly all envs) step two per warp on 16 slots, the others on 32
        int* small = spawn->scratch;
        int* large = spawn->scratch + (s->n_envs + 1);
        cudaMemsetAsync(small, 0, sizeof(int), st);
        cudaMemsetAsync(large, 0, sizeof(int), st);
        hwynet::classify_envs_kernel<<<(s->n_envs + 255) / 256, 256, 0, st>>>(s->count, s->n_envs, small, large);
        if (check_launch("classify_envs_kernel")) return 1;
        // The two kernels serve disjoint envs, and the 32-slot one rarely fills the GPU (the few envs that hold more
        // than 15 vehicles): it runs on a side stream forked from and joined back into the caller's stream (under a
        // CUDA-graph capture the fork / join become graph edges), so it overlaps the 16-slot kernel instead of
        // following it with most SMs idle.
        SideStream* side = side_stream();
        if (!side) return 1;
        cudaEventRecord(side->fork, st);
        cudaStreamWaitEvent(side->stream, side->fork, 0);
        if (launch_step<HWY_NET_GROUP_LARGE, true>(p, graph, *spawn, s, action, obs, reward, terminated, truncated,
                                                   info_speed, info_crashed, side->stream, large, agents_reward,
                                                   agents_terminated))
            return 1;
        cudaEventRecord(side->join, side->stream);
        if (launch_step<16, true>(p, graph, *spawn, s, action, obs, reward, terminated, truncated, info_speed,
                                  info_crashed, st, small, agents_reward, agents_terminated))
            return 1;
        cudaStreamWaitEvent(st, side->join, 0);
        return 0;
    }
    return launch_step<HWY_NET_GROUP_LARGE, true>(p, graph, spawn ? *spawn : none, s, action, obs, reward, terminated,
                                                  truncated, info_speed, info_crashed, st, nullptr, agents_reward,
                                                  agents_terminated);
}

int hwy_intersection_reset(const HwyNetParams* p, const HwyNetGraph* graph, const HwyIntersectionSpawn* spawn,
                           const HwyNetState* s, const uint8_t* mask_a, const uint8_t* mask_b, float* obs,
                           float* final_obs, void* stream) {
    if (validate_net(p, graph, s)) return 1;
    if (s->vp != HWY_NET_GROUP_LARGE) return fail("%s", "hwy_intersection_reset expects slot stride 32");
    if (!spawn || !spawn->route_table || !spawn->route_len || !spawn->scratch || !s->rng)
        return fail("%s", "reset needs the spawn tables, the scratch list and the rng words");
    if (spawn->initial_vehicle_count < 1 || spawn->initial_vehicle_count > HWY_NET_GROUP_LARGE - 2)
        return fail("%s", "initial_vehicle_count out of range");
    if (final_obs && !obs) return fail("%s", "final_obs without obs");
    cudaStream_t st = (cudaStream_t)stream;
    cudaMemsetAsync(spawn->scratch, 0, sizeof(int), st);
    hwynet::compact_envs_kernel<<<(s->n_envs + 255) / 256, 256, 0, st>>>(mask_a, mask_b, s->n_envs, spawn->scratch);
    if (final_obs)
        cudaMemcpyAsync(final_obs, obs, (size_t)s->n_envs * hwy_network_obs_size(p) * sizeof(float),
                        cudaMemcpyDeviceToDevice, st);
    if (check_launch("compact_envs_kernel")) return 1;
    if (spawn->initial_vehicle_count + 1 <= 16)  // n-1 draws + challenger + controlled vehicle fit 16 slots
        return launch_intersection_reset<16>(p, graph, spawn, s, obs, st);
    return launch_intersection_reset<HWY_NET_GROUP_LARGE>(p, graph, spawn, s, obs, st);
}

int hwy_debug_network_neighbours(const HwyNetParams* p, const HwyNetGraph* graph, const HwyNetState* s,
                                 const int32_t* query_lane, int32_t* front, int32_t* rear, void* stream) {
    if (validate_net(p, graph, s)) return 1;
    if (!front || !rear) return fail("%s", "null pointer");
    return launch_groups([](auto t) { return hwynet::debug_neighbours_kernel<decltype(t)::G, decltype(t)::REG>; },
                         "debug_neighbours_kernel", s, (cudaStream_t)stream, *p, graph, *s, query_lane, front, rear);
}

int hwy_debug_rotated_rectangles_intersect(const double* rects, int n, int32_t* out, void* stream) {
    if (!rects || !out || n < 0) return fail("%s", "bad arguments");
    if (n == 0) return 0;
    hwynet::debug_rectangles_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(rects, n, out);
    return check_launch("debug_rectangles_kernel");
}

int hwy_merge_reset(const HwyNetParams* p, const HwyNetGraph* graph, const HwyMergeSpawn* spawn, const HwyNetState* s,
                    uint64_t* rng, const uint8_t* mask_a, const uint8_t* mask_b, float* obs, void* stream) {
    if (validate_net(p, graph, s)) return 1;
    if (!spawn || !rng) return fail("%s", "null spawn / rng");
    if (s->vp != HWY_NET_GROUP || p->n_vehicles != 6) return fail("%s", "merge-v0: 5 vehicles + 1 obstacle on 8 slots");
    return scripted_reset(hwynet::merge_reset_kernel, "merge_reset_kernel", 1,
                          p, graph, spawn, s, rng, mask_a, mask_b, obs, stream);
}

int hwy_exit_reset(const HwyNetParams* p, const HwyNetGraph* graph, const HwyExitSpawn* spawn, const HwyNetState* s,
                   uint64_t* rng, const uint8_t* mask_a, const uint8_t* mask_b, float* obs, void* stream) {
    if (validate_net(p, graph, s)) return 1;
    if (!spawn || !rng) return fail("%s", "null spawn / rng");
    if (s->vp != HWY_NET_GROUP_LARGE || spawn->n_vehicles < 1 || spawn->n_vehicles > HWY_NET_GROUP_LARGE)
        return fail("%s", "exit-v0: 1..32 vehicles on 32 slots");
    if (spawn->lanes_count < 1 || spawn->lanes_count > HWY_MAX_LANES) return fail("%s", "lanes_count out of range");
    return scripted_reset(hwynet::exit_reset_kernel, "exit_reset_kernel", 1,
                          p, graph, spawn, s, rng, mask_a, mask_b, obs, stream);
}

int hwy_u_turn_reset(const HwyNetParams* p, const HwyNetGraph* graph, const HwyUTurnSpawn* spawn, const HwyNetState* s,
                     uint64_t* rng, const uint8_t* mask_a, const uint8_t* mask_b, float* obs, void* stream) {
    if (validate_net(p, graph, s)) return 1;
    if (!spawn || !rng || !spawn->route_table || !spawn->route_len) return fail("%s", "null spawn / rng / route table");
    if (s->vp != HWY_NET_GROUP || p->n_vehicles != 7) return fail("%s", "u-turn-v0: 7 vehicles on 8 slots");
    return scripted_reset(hwynet::u_turn_reset_kernel, "u_turn_reset_kernel", 1,
                          p, graph, spawn, s, rng, mask_a, mask_b, obs, stream);
}

int hwy_two_way_reset(const HwyNetParams* p, const HwyNetGraph* graph, const HwyTwoWaySpawn* spawn, const HwyNetState* s,
                      uint64_t* rng, const uint8_t* mask_a, const uint8_t* mask_b, float* obs, void* stream) {
    if (validate_net(p, graph, s)) return 1;
    if (!spawn || !rng) return fail("%s", "null spawn / rng");
    if (s->vp != HWY_NET_GROUP || p->n_vehicles != 6) return fail("%s", "two-way-v0: 6 vehicles on 8 slots");
    return scripted_reset(hwynet::two_way_reset_kernel, "two_way_reset_kernel", 1,
                          p, graph, spawn, s, rng, mask_a, mask_b, obs, stream);
}

int hwy_network_substeps(const HwyNetParams* p, const HwyNetGraph* graph, const HwyNetState* s, const uint8_t* mask,
                         int n_substeps, void* stream) {
    if (validate_net(p, graph, s)) return 1;
    if (n_substeps < 0) return fail("%s", "n_substeps < 0");
    return launch_groups([](auto t) { return hwynet::network_substeps_kernel<decltype(t)::G, decltype(t)::REG>; },
                         "network_substeps_kernel", s, (cudaStream_t)stream, *p, graph, *s, mask, n_substeps);
}

int hwy_network_observe(const HwyNetParams* p, const HwyNetGraph* graph, const HwyNetState* s, float* obs,
                        void* stream) {
    if (validate_net(p, graph, s)) return 1;
    if (!obs) return fail("%s", "obs is null");
    return observe_dispatch(p, graph, s, nullptr, nullptr, obs, (cudaStream_t)stream);
}

int hwy_roundabout_reset(const HwyNetParams* p, const HwyNetGraph* graph, const HwyRoundaboutSpawn* spawn,
                         const HwyNetState* s, uint64_t* rng, const uint8_t* mask_a, const uint8_t* mask_b,
                         float* obs, void* stream) {
    if (validate_net(p, graph, s)) return 1;
    if (!spawn || !rng || !spawn->route_table || !spawn->route_len) return fail("%s", "null spawn / rng pointer");
    if (p->n_vehicles != 5 || s->vp != HWY_NET_GROUP) return fail("%s", "roundabout spawn places exactly 5 vehicles in 8 slots");
    return scripted_reset(hwynet::roundabout_reset_kernel, "roundabout_reset_kernel", 32,  // a warp per env
                          p, graph, spawn, s, rng, mask_a, mask_b, obs, stream);
}

}  // extern "C"
