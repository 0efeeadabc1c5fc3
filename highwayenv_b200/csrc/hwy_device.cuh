// hwy_device.cuh — device functions of the highway hot path that do not depend on the
// kernel's thread mapping: StraightLane geometry, the steering law, the SAT collision test,
// MDPVehicle speed indexing.  Reference paths are relative to /root/reference/highway_env.
#pragma once
#include "../../include/hwyb200.h"
#include "hwy_math.cuh"

namespace hwy {

typedef unsigned long long u64;

// env e takes part in a masked launch: one of the two masks selects it, or there is no mask at all
__device__ __forceinline__ bool env_selected(const uint8_t* mask_a, const uint8_t* mask_b, int e) {
    return (!mask_a && !mask_b) || (mask_a && mask_a[e]) || (mask_b && mask_b[e]);
}

// ------------------------------------------------------------------ lane geometry
// road/lane.py:205-209 StraightLane.local_coordinates
__device__ __forceinline__ void lane_local(const HwyStraightLane& L, double x, double y, double& s,
                                           double& lat) {
    double ddx = x - L.start_x, ddy = y - L.start_y;
    s = dot2(ddx, ddy, L.dir_x, L.dir_y);
    lat = dot2(ddx, ddy, L.lat_x, L.lat_y);
}
__device__ __forceinline__ double lane_s(const HwyStraightLane& L, double x, double y) {
    return dot2(x - L.start_x, y - L.start_y, L.dir_x, L.dir_y);
}
// road/lane.py:80-102 on_lane
__device__ __forceinline__ bool lane_on(const HwyStraightLane& L, double s, double lat, double margin) {
    return fabs(lat) <= L.width / 2 + margin && -kLaneVehLength <= s && s < L.length + kLaneVehLength;
}
// road/lane.py:104-118 is_reachable_from (forbidden is False on the highway)
__device__ __forceinline__ bool lane_reachable(const HwyStraightLane& L, double x, double y) {
    double s, lat;
    lane_local(L, x, y, s, lat);
    return fabs(lat) <= 2 * L.width && 0 <= s && s < L.length + kLaneVehLength;
}
// road/road.py:55-71 get_closest_lane_index with lane.py:132-143 distance_with_heading:
// first minimum in graph-enumeration order.
// `aligned` (lanes_aligned below, uniform): every lane has the direction, origin-x, heading and length of lane 0, so
// s, the two longitudinal terms and the angle term are bitwise the same for every lane and only the lateral offset
// (dy of the lane origin; dir = (1, 0), lat = (-0, 1) make both dot products exact) is per lane.
__device__ __forceinline__ int closest_lane(const HwyHighwayParams& P, double x, double y, double h, bool aligned = false) {
    int best = 0;
    double bd = 0;
    if (aligned) {
        const HwyStraightLane& L0 = P.lanes[0];
        const double s = dot2(x - L0.start_x, y - L0.start_y, L0.dir_x, L0.dir_y);
        const double t1 = fmax(s - L0.length, 0.0), t2 = fmax(0.0 - s, 0.0);
        const double angle = 1.0 * fabs(wrap_to_pi(h - L0.heading));
#pragma unroll 1
        for (int l = 0; l < P.lanes_count; ++l) {
            const HwyStraightLane& L = P.lanes[l];
            const double r = dot2(x - L.start_x, y - L.start_y, L.lat_x, L.lat_y);
            const double d = fabs(r) + t1 + t2 + angle;
            if (l == 0 || d < bd) {
                bd = d;
                best = l;
            }
        }
        return best;
    }
    for (int l = 0; l < P.lanes_count; ++l) {
        const HwyStraightLane& L = P.lanes[l];
        double s, r;
        lane_local(L, x, y, s, r);
        double angle = fabs(wrap_to_pi(h - L.heading));
        double d = fabs(r) + fmax(s - L.length, 0.0) + fmax(0.0 - s, 0.0) + 1.0 * angle;
        if (l == 0 || d < bd) {
            bd = d;
            best = l;
        }
    }
    return best;
}
// All lanes share origin-x and an x-aligned direction (RoadNetwork.straight_road_network with
// angle 0, road/road.py:291-321): the longitudinal coordinate is then bitwise lane independent.
// stricter: also the same heading, length and lateral direction (what closest_lane's shared terms need)
__device__ __forceinline__ bool lanes_congruent(const HwyHighwayParams& P) {
    bool ok = P.lanes[0].dir_y == 0.0;
    for (int l = 1; l < P.lanes_count; ++l)
        ok = ok && P.lanes[l].start_x == P.lanes[0].start_x && P.lanes[l].dir_x == P.lanes[0].dir_x &&
             P.lanes[l].dir_y == 0.0 && P.lanes[l].heading == P.lanes[0].heading &&
             P.lanes[l].length == P.lanes[0].length && P.lanes[l].lat_x == P.lanes[0].lat_x &&
             P.lanes[l].lat_y == P.lanes[0].lat_y;
    return ok;
}
__device__ __forceinline__ bool lanes_aligned(const HwyHighwayParams& P) {
    bool ok = P.lanes[0].dir_y == 0.0;
    for (int l = 1; l < P.lanes_count; ++l)
        ok = ok && P.lanes[l].start_x == P.lanes[0].start_x && P.lanes[l].dir_x == P.lanes[0].dir_x &&
             P.lanes[l].dir_y == 0.0;
    return ok;
}

// vehicle/controller.py:145-187 steering_control on a StraightLane, up to the argument of the
// last arcsin: returns x = clip(LENGTH/2/not_zero(speed) * heading_rate_command, -1, 1), i.e.
// the SINE of the commanded slip angle.
static __device__ __noinline__ double steering_sin_slip(const HwyStraightLane L, double x, double y,
                                                 double heading, double speed) {
    double lc_s, lc_lat;
    lane_local(L, x, y, lc_s, lc_lat);
    double lane_future_heading = L.heading;  // StraightLane.heading_at
    double lateral_speed_command = -kKpLateral * lc_lat;
    double heading_command = m_asin(clipd(div_finite(lateral_speed_command, not_zero(speed)), -1.0, 1.0));
    double heading_ref = lane_future_heading + clipd(heading_command, -kPi / 4, kPi / 4);
    double heading_rate_command = kKpHeading * wrap_to_pi(heading_ref - heading);
    return clipd(kVehLength / 2 / not_zero(speed) * heading_rate_command, -1.0, 1.0);
}

// The reference then computes  delta = clip(arctan(2 tan(arcsin(x))), +-pi/3)  (controller.py:
// 176-186) and, in Vehicle.step,  beta = arctan(1/2 tan(delta))  (kinematics.py:141-142), of which
// only sin(beta) and cos(beta) are used.  When delta is not clipped the two maps cancel:
// beta = arcsin(x), so sin(beta) = x and cos(beta) = sqrt(1 - x^2); when it is clipped
// (2 |tan(arcsin x)| > tan(pi/3)) beta = +-arctan(tan(pi/3)/2).  Evaluating that closed form
// replaces six libm calls per vehicle-substep by two square roots; it differs from the
// reference's rounded chain by a few ulp (same order as CUDA-vs-glibc libm differences).
__device__ __forceinline__ void beta_of_controlled(double x, double& sin_beta, double& cos_beta) {
    const double T3 = 1.7320508075688767;  // np.tan(np.pi / 3)
    double c = sqrt(1.0 - x * x);          // cos(arcsin x) >= 0
    if (2.0 * fabs(x) > T3 * c) {          // steering saturated at MAX_STEERING_ANGLE
        // t = +-T3/2: 1/sqrt(1 + t*t) does not depend on the sign and (-t)*inv = -(t*inv), so the constants fold
        const double t0 = 0.5 * T3;
        const double inv = 1.0 / sqrt(1.0 + t0 * t0);
        sin_beta = copysign(t0 * inv, x);
        cos_beta = inv;
    } else {
        sin_beta = x;
        cos_beta = c;
    }
}
// beta = arctan(1/2 tan(delta)) for an explicit steering angle (ContinuousAction ego)
static __device__ __noinline__ void beta_of_angle(double delta, double& sin_beta, double& cos_beta) {
    double t = 0.5 * m_tan(delta);
    double inv = 1.0 / sqrt(1.0 + t * t);
    sin_beta = t * inv;
    cos_beta = inv;
}

// vehicle/controller.py:326-344 speed_to_index (np.round: half to even)
__device__ __forceinline__ int speed_to_index(const HwyHighwayParams& P, double speed) {
    int n = P.n_target_speeds;
    double x = (speed - P.target_speeds[0]) / (P.target_speeds[n - 1] - P.target_speeds[0]);
    return (int)clipd(rint(x * (n - 1)), 0.0, (double)(n - 1));
}

// ------------------------------------------------------------------ collision (SAT)
// A vehicle rectangle as RoadObject.polygon() builds it (vehicle/objects.py:169-181): the 4
// corners (rotation @ points).T + position; the closing 5th point repeats the first and adds
// nothing to projections (same value), so it is not materialised.
struct Quad {
    double x[4], y[4];
};
__device__ __forceinline__ Quad make_polygon(double px, double py, double c, double s, double length = kVehLength) {
    const double hl = length / 2, hw = kVehWidth / 2;
    const double lx[4] = {-hl, -hl, +hl, +hl};
    const double ly[4] = {-hw, +hw, +hw, -hw};
    Quad q;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        q.x[k] = (c * lx[k] + (-s) * ly[k]) + px;
        q.y[k] = (s * lx[k] + c * ly[k]) + py;
    }
    return q;
}
// utils.py:177-185 project_polygon
__device__ __forceinline__ void project_polygon(const Quad& p, double ax, double ay, double& mn,
                                                double& mx) {
    mn = mx = dot2(p.x[0], p.y[0], ax, ay);
#pragma unroll
    for (int k = 1; k < 4; ++k) {
        double pr = dot2(p.x[k], p.y[k], ax, ay);
        if (pr < mn) mn = pr;
        if (pr > mx) mx = pr;
    }
}
// utils.py:188-193
__device__ __forceinline__ double interval_distance(double min_a, double max_a, double min_b,
                                                    double max_b) {
    return min_a < min_b ? min_b - max_a : min_a - max_b;
}

// utils.py:196-241 are_polygons_intersecting: SAT over the 4+4 edge normals with the relative
// displacement extension; returns (intersecting, will_intersect, translation).  One rolled
// loop over the 8 edges: the polygon whose edges are being visited is rotated in registers so
// the current edge is always (point 0 -> point 1); projections are order independent.
__device__ __forceinline__ void rotate_quad(Quad& q) {
    double tx = q.x[0], ty = q.y[0];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        q.x[k] = q.x[k + 1];
        q.y[k] = q.y[k + 1];
    }
    q.x[3] = tx;
    q.y[3] = ty;
}
__device__ __forceinline__ void polygons_intersecting(Quad a, Quad b, double dax, double day,
                                                      double dbx, double dby, bool& intersecting_out,
                                                      bool& will_intersect_out, double& trx,
                                                      double& try_) {
    bool intersecting = true, will_intersect = true;
    double min_distance = INFINITY, tax = 0.0, tay = 0.0;
    // centre difference a[:-1].mean(axis=0) - b[:-1].mean(axis=0): sequential row sums / 4
    const double dcx = (((a.x[0] + a.x[1]) + a.x[2]) + a.x[3]) / 4.0 - (((b.x[0] + b.x[1]) + b.x[2]) + b.x[3]) / 4.0;
    const double dcy = (((a.y[0] + a.y[1]) + a.y[2]) + a.y[3]) / 4.0 - (((b.y[0] + b.y[1]) + b.y[2]) + b.y[3]) / 4.0;
    const double rdx = dax - dbx, rdy = day - dby;
    bool brk = false;
#pragma unroll 1
    for (int e = 0; e < 8; ++e) {
        if (e == 4) brk = false;  // the `break` leaves only the inner loop (utils.py:232-233)
        if (brk) continue;
        const bool on_a = e < 4;
        double p1x = on_a ? a.x[0] : b.x[0], p1y = on_a ? a.y[0] : b.y[0];
        double p2x = on_a ? a.x[1] : b.x[1], p2y = on_a ? a.y[1] : b.y[1];
        double nx = -p2y + p1y, ny = p2x - p1x;
        double nn = norm2(nx, ny);
        nx /= nn;
        ny /= nn;
        double min_a, max_a, min_b, max_b;
        project_polygon(a, nx, ny, min_a, max_a);
        project_polygon(b, nx, ny, min_b, max_b);
        if (interval_distance(min_a, max_a, min_b, max_b) > 0) intersecting = false;
        double vp = dot2(nx, ny, rdx, rdy);
        if (vp < 0)
            min_a += vp;
        else
            max_a += vp;
        double distance = interval_distance(min_a, max_a, min_b, max_b);
        if (distance > 0) will_intersect = false;
        if (!intersecting && !will_intersect) {
            brk = true;
            continue;
        }
        if (fabs(distance) < min_distance) {
            min_distance = fabs(distance);
            bool pos = dot2(dcx, dcy, nx, ny) > 0;
            tax = pos ? nx : -nx;
            tay = pos ? ny : -ny;
        }
        if (on_a)
            rotate_quad(a);
        else
            rotate_quad(b);
    }
    intersecting_out = intersecting;
    will_intersect_out = will_intersect;
    trx = will_intersect ? min_distance * tax : 0.0;
    try_ = will_intersect ? min_distance * tay : 0.0;
}

// ------------------------------------------------------------------ packed meta word
__device__ __forceinline__ int meta_lane(int m) { return (m >> HWY_META_LANE_SHIFT) & 0xff; }
__device__ __forceinline__ int meta_target(int m) { return (m >> HWY_META_TARGET_SHIFT) & 0xff; }
__device__ __forceinline__ int meta_kind(int m) { return (m >> HWY_META_KIND_SHIFT) & 3; }
__device__ __forceinline__ int meta_set_lane(int m, int l) {
    return (m & ~(0xff << HWY_META_LANE_SHIFT)) | (l << HWY_META_LANE_SHIFT);
}
__device__ __forceinline__ int meta_set_target(int m, int l) {
    return (m & ~(0xff << HWY_META_TARGET_SHIFT)) | (l << HWY_META_TARGET_SHIFT);
}

}  // namespace hwy
