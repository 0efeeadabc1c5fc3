// hwy_bicycle.cuh — the dynamical BicycleVehicle (vehicle/dynamics.py) and Vehicle.clip_actions, shared by the
// intersection-v1 ego (hwy_network.cu) and lane-keeping-v0 (hwy_lane_keeping.cu).  Reference paths are relative to
// /root/reference/highway_env.  The two out-of-line functions are `inline` so that both translation units may define
// them.
#pragma once
#include <cuda_runtime.h>

#include "hwy_math.cuh"

namespace hwynet {
using namespace hwy;

// BicycleVehicle.derivative_func (vehicle/dynamics.py:73-111) on (x, y, heading, speed, lateral_speed, yaw_rate)
inline __device__ __noinline__ void bicycle_derivative(const double (&st)[6], double steering, double acceleration,
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
inline __device__ __noinline__ void bicycle_advance(double (&st)[6], bool crashed, double& steering,
                                                    double& acceleration, double dt) {
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

}  // namespace hwynet
