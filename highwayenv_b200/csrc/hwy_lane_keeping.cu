// hwy_lane_keeping.cu — sm_90a kernels + C ABI of lane-keeping-v0 (LaneKeepingEnv, envs/lane_keeping_env.py): one
// dynamical BicycleVehicle per env steering along a SineLane, no traffic, a noisy AttributesObservation drawn from the
// env's numpy stream, and the registration's TimeLimit(max_episode_steps=200) as the only end of an episode.
//
// Thread mapping: one thread per env.  The state is structure-of-arrays fp64 ([6][n_envs]), so every load and store of
// a warp is one contiguous run; the observation row of an env ([n_attr][4] f64) is written by its thread straight to
// the output buffer.  The two lanes are read from the kernel parameter (__grid_constant__: referenced in place, not
// copied to local memory).
// DESIGN.md 3.16.
//
// Reference paths are relative to /root/reference/highway_env.
#include <cstdint>
#include <cstdio>

#include <cuda_runtime.h>

#include "../../include/hwyb200.h"
#include "hwy_abi.h"
#include "hwy_math.cuh"
#include "hwy_lanes.cuh"
#include "hwy_bicycle.cuh"

namespace hwylk {
using namespace hwy;
using namespace hwynet;

constexpr int kBlockThreads = 256;
enum { ATTR_STATE = 0, ATTR_DERIVATIVE = 1, ATTR_REFERENCE_STATE = 2 };

// AttributesObservation.observe (envs/common/observation.py:582-585) over LaneKeepingEnv's properties
// (lane_keeping_env.py:144-171): the state and derivative columns [1, 2, 4, 5] plus uniform(-noise, noise, (4, 1)),
// drawn in attribute order; reference_state = [y - lat, lane.heading_at(longi), 0, 0] on the env's current lane.
// `steering` / `acceleration` are the vehicle's action dict as act() left it (not yet clipped by step()).
// `o` is the env's row of the observation buffer.
__device__ __forceinline__ void observe(const HwyLaneKeepingParams& P, const double (&st)[6], double steering,
                                       double acceleration, int phase, Pcg64& g, double* __restrict__ o) {
    for (int k = 0; k < P.n_attr; ++k) {
        double* c = o + 4 * k;
        const int a = P.attr[k];
        if (a == ATTR_REFERENCE_STATE) {
            double s, lat;
            lane_local(P.lanes[phase], st[0], st[1], s, lat);
            c[0] = st[1] - lat;
            c[1] = lane_heading_at(P.lanes[phase], s);
            c[2] = 0.0;
            c[3] = 0.0;
            continue;
        }
        double v[6];
        if (a == ATTR_DERIVATIVE)
            bicycle_derivative(st, steering, acceleration, v);
        else
            for (int j = 0; j < 6; ++j) v[j] = st[j];
        const double noise = a == ATTR_DERIVATIVE ? P.derivative_noise : P.state_noise;
        c[0] = v[1] + g.uniform(-noise, noise);
        c[1] = v[2] + g.uniform(-noise, noise);
        c[2] = v[4] + g.uniform(-noise, noise);
        c[3] = v[5] + g.uniform(-noise, noise);
    }
}

// AbstractEnv.reset (envs/common/abstract.py:219-249) after the seeding: LaneKeepingEnv._reset builds the scene
// without draws; define_spaces observes twice (AttributesObservation.space) and the returned observation is the third.
// Only the draws of the first two matter: 4 per noisy attribute each.
__device__ __forceinline__ void reset_env(const HwyLaneKeepingParams& P, double (&st)[6], int& phase, int& elapsed,
                                          Pcg64& g, double* __restrict__ o) {
    int noisy = 0;
    for (int k = 0; k < P.n_attr; ++k) noisy += P.attr[k] != ATTR_REFERENCE_STATE;
    for (int d = 0; d < 2 * 4 * noisy; ++d) g.next64();
    st[0] = P.x0;
    st[1] = P.y0;
    st[2] = P.heading0;
    st[3] = P.speed0;
    st[4] = 0.0;
    st[5] = 0.0;
    phase = 0;
    elapsed = 0;
    observe(P, st, 0.0, 0.0, phase, g, o);  // Vehicle.__init__: action = {steering: 0, acceleration: 0}
}

__device__ __forceinline__ void load_state(const HwyLaneKeepingState& S, int e, double (&st)[6]) {
    const size_t n = (size_t)S.n_envs;
    for (int j = 0; j < 6; ++j) st[j] = S.state[j * n + e];
}
__device__ __forceinline__ void store_state(const HwyLaneKeepingState& S, int e, const double (&st)[6]) {
    const size_t n = (size_t)S.n_envs;
    for (int j = 0; j < 6; ++j) S.state[j * n + e] = st[j];
}

__global__ void __launch_bounds__(kBlockThreads)
lane_keeping_reset_kernel(const __grid_constant__ HwyLaneKeepingParams P, const __grid_constant__ HwyLaneKeepingState S,
                          const uint8_t* __restrict__ mask_a, const uint8_t* __restrict__ mask_b,
                          double* __restrict__ obs) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= S.n_envs) return;
    if ((mask_a || mask_b) && !((mask_a && mask_a[e]) || (mask_b && mask_b[e]))) return;
    Pcg64 g = load_rng(S.rng, S.n_envs, e);
    double st[6];
    int phase, elapsed;
    reset_env(P, st, phase, elapsed, g, obs + (size_t)e * 4 * P.n_attr);
    store_state(S, e, st);
    S.lane_phase[e] = phase;
    S.elapsed[e] = elapsed;
    store_rng(S.rng, S.n_envs, e, g);
}

// LaneKeepingEnv.step (lane_keeping_env.py:54-72) under TimeLimit(max_episode_steps=200) (highway_env/__init__.py:89)
__global__ void __launch_bounds__(kBlockThreads)
lane_keeping_step_kernel(const __grid_constant__ HwyLaneKeepingParams P, const __grid_constant__ HwyLaneKeepingState S,
                         const float* __restrict__ actions, double* __restrict__ obs, double* __restrict__ final_obs,
                         double* __restrict__ reward, uint8_t* __restrict__ terminated,
                         uint8_t* __restrict__ truncated) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= S.n_envs) return;
    const int n_obs = 4 * P.n_attr;
    double* o = obs + (size_t)e * n_obs;
    Pcg64 g = load_rng(S.rng, S.n_envs, e);
    double st[6];
    load_state(S, e, st);
    int phase = S.lane_phase[e], elapsed = S.elapsed[e];
    // 1. the queued lane takes over once the vehicle has left the first one: `not self.lane.on_lane(position)`
    if (phase == 0) {
        double s, lat;
        lane_local(P.lanes[0], st[0], st[1], s, lat);
        if (!lane_on(P.lanes[0], s, lat, 0.0)) phase = 1;
    }
    // 2. ContinuousAction.get_action (envs/common/action.py:136-162): the Box is float32 and NEP 50 keeps utils.lmap
    // (utils.py:31-33) in float32; a disabled axis is the int 0
    const int na = P.longitudinal + P.lateral;
    double acc0 = 0.0, steer0 = 0.0;
    for (int k = 0; k < na; ++k) {
        float a = actions[(size_t)e * na + k];
        if (P.act_clip) a = fminf(fmaxf(a, -1.0f), 1.0f);
        const bool is_acc = P.longitudinal && k == 0;
        const double lo = is_acc ? P.acc_lo : P.steer_lo, hi = is_acc ? P.acc_hi : P.steer_hi;
        const double v = (double)__fadd_rn((float)lo, __fdiv_rn(__fmul_rn(__fsub_rn(a, -1.0f), (float)(hi - lo)), 2.0f));
        if (is_acc)
            acc0 = v;
        else
            steer0 = v;
    }
    // 3. observe before simulating: the state from before the step, the derivative with the new action
    observe(P, st, steer0, acc0, phase, g, o);
    // 4. _simulate (abstract.py:288-316): act again on frame 0; BicycleVehicle.step clips the action dict in place,
    // and the clipped values carry over to the following frames; the yaw rate clip is kept in the state
    double steer = steer0, acc = acc0;
    for (int f = 0; f < P.frames; ++f) bicycle_advance(st, false, steer, acc, P.dt);
    // 5. reward on the env's current lane (the switch of this step's start only: it can be stale)
    {
        double s, lat;
        lane_local(P.lanes[phase], st[0], st[1], s, lat);
        const double q = lat / P.lanes[phase].width;
        reward[e] = 1 - q * q;
    }
    ++elapsed;
    const bool trunc = elapsed >= P.max_episode_steps;
    terminated[e] = 0;
    truncated[e] = trunc;
    if (P.autoreset == HWY_AUTORESET_SAME_STEP && trunc) {
        double* fo = final_obs + (size_t)e * n_obs;
        for (int j = 0; j < n_obs; ++j) fo[j] = o[j];
        reset_env(P, st, phase, elapsed, g, o);
    }
    store_state(S, e, st);
    S.lane_phase[e] = phase;
    S.elapsed[e] = elapsed;
    store_rng(S.rng, S.n_envs, e, g);
}

}  // namespace hwylk

// ====================================================================== C ABI
namespace {
using hwy_abi::fail;

int validate(const HwyLaneKeepingParams* p, const HwyLaneKeepingState* s) {
    if (!p || !s) return fail("%s", "null params / state");
    if (s->n_envs < 0) return fail("%s", "n_envs must be >= 0");
    if (s->n_envs > 0 && (!s->state || !s->lane_phase || !s->elapsed || !s->rng)) return fail("%s", "null state buffer");
    if (p->frames < 1) return fail("%s", "frames (simulation_frequency // policy_frequency) must be >= 1");
    if (p->n_attr < 1 || p->n_attr > HWY_LK_MAX_ATTR) return fail("%s", "n_attr must be in 1..3");
    for (int k = 0; k < p->n_attr; ++k)
        if (p->attr[k] < 0 || p->attr[k] > 2) return fail("%s", "attr must be 0 (state), 1 (derivative) or 2 (reference_state)");
    if ((p->longitudinal != 0 && p->longitudinal != 1) || (p->lateral != 0 && p->lateral != 1) ||
        p->longitudinal + p->lateral == 0)
        return fail("%s", "longitudinal / lateral must be 0 or 1, and not both 0");
    if (p->autoreset != HWY_AUTORESET_DISABLED && p->autoreset != HWY_AUTORESET_SAME_STEP)
        return fail("%s", "autoreset must be HWY_AUTORESET_DISABLED or HWY_AUTORESET_SAME_STEP");
    for (int l = 0; l < 2; ++l)
        if (p->lanes[l].type != HWY_LANE_STRAIGHT && p->lanes[l].type != HWY_LANE_SINE)
            return fail("%s", "lanes must be straight or sine lanes");
    return 0;
}
unsigned grid_for(int n) { return (unsigned)((n + hwylk::kBlockThreads - 1) / hwylk::kBlockThreads); }
}  // namespace

extern "C" {

int hwy_lane_keeping_reset(const HwyLaneKeepingParams* p, const HwyLaneKeepingState* s, const uint8_t* mask_a,
                           const uint8_t* mask_b, double* obs, void* stream) {
    if (validate(p, s)) return 1;
    if (s->n_envs == 0) return 0;
    if (!obs) return fail("%s", "null obs");
    hwylk::lane_keeping_reset_kernel<<<grid_for(s->n_envs), hwylk::kBlockThreads, 0, (cudaStream_t)stream>>>(
        *p, *s, mask_a, mask_b, obs);
    return hwy_abi::check_launch("lane_keeping_reset_kernel");
}

int hwy_lane_keeping_step(const HwyLaneKeepingParams* p, const HwyLaneKeepingState* s, const float* actions,
                          double* obs, double* final_obs, double* reward, uint8_t* terminated, uint8_t* truncated,
                          void* stream) {
    if (validate(p, s)) return 1;
    if (s->n_envs == 0) return 0;
    if (!actions || !obs || !reward || !terminated || !truncated) return fail("%s", "null step buffer");
    if (p->autoreset == HWY_AUTORESET_SAME_STEP && !final_obs) return fail("%s", "null final_obs with SameStep autoreset");
    hwylk::lane_keeping_step_kernel<<<grid_for(s->n_envs), hwylk::kBlockThreads, 0, (cudaStream_t)stream>>>(
        *p, *s, actions, obs, final_obs, reward, terminated, truncated);
    return hwy_abi::check_launch("lane_keeping_step_kernel");
}

}  // extern "C"
