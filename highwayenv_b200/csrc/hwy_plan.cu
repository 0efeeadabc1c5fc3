// hwy_plan.cu — planning on the device: batched value iteration of deterministic finite MDPs (the solver of
// rl-agents' ValueIterationAgent, which the reference's docs run on env.to_finite_mdp(), docs/content/algorithms.md).
// One block per env, a synchronous (Jacobi) sweep over the env's states per iteration, so every update is the
// numpy expression  reward + gamma * next_v  evaluated elementwise.  The per-state values live in shared memory.
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/hwyb200.h"
#include "hwy_abi.h"

namespace hwyplan {

constexpr int kThreads = 128;

// np.isclose(x, y) with the defaults of np.allclose (rtol 1e-5, atol 1e-8):
//   (|x - y| <= atol + rtol * |y|) & isfinite(y) | (x == y)
__device__ __forceinline__ bool np_isclose(double x, double y) {
    return (fabs(x - y) <= 1e-8 + 1e-5 * fabs(y) && isfinite(y)) || x == y;
}

// one Bellman backup of Q(s, a) from the state values v (rows of terminal states do not bootstrap)
__device__ __forceinline__ double backup(double r, double gamma, bool term, const double* v, int t) {
    return r + gamma * (term ? 0.0 : v[t]);
}

// dynamic shared memory: three value buffers of s_max doubles.  After iteration k (Q_{k+1} computed) `vprev` holds
// V_k = max_a Q_k and `vcur` V_{k+1}; Q_k is recomputed from V_{k-1} for the allclose test instead of being stored.
__global__ void __launch_bounds__(kThreads)
value_iteration_kernel(const __grid_constant__ HwyValueIterationParams P, const int32_t* __restrict__ transition,
                       const double* __restrict__ reward, const uint8_t* __restrict__ terminal,
                       const int32_t* __restrict__ n_states, double* __restrict__ q,
                       int32_t* __restrict__ iterations_done) {
    extern __shared__ double vbuf[];
    const int e = blockIdx.x, tid = threadIdx.x, A = P.n_actions, SM = P.s_max;
    const size_t row0 = (size_t)e * SM;
    const int32_t* tr = transition + row0 * A;
    const double* rw = reward + row0 * A;
    const uint8_t* te = terminal + row0;
    double* qe = q + row0 * A;
    const int S = n_states[e];
    // the successors come from the caller: an env with one outside its own rows is not iterated at all
    bool bad = S < 0 || S > SM;
    if (!bad)
        for (int k = tid; k < S * A; k += kThreads) bad = bad || tr[k] < 0 || tr[k] >= S;
    if (__syncthreads_or(bad)) {
        for (int k = tid; k < SM * A; k += kThreads) qe[k] = 0.0;
        if (tid == 0) {
            iterations_done[e] = -1;
            if (P.action) P.action[e] = -1;
        }
        return;
    }
    double *vprev = vbuf, *vcur = vbuf + SM, *vnext = vbuf + 2 * SM;
    for (int s = tid; s < S; s += kThreads) vcur[s] = 0.0;  // V_0 = max_a Q_0 = 0
    __syncthreads();
    const double gamma = P.gamma;
    int done = P.iterations;
    for (int k = 0; k < P.iterations; ++k) {
        bool differs = false;
        for (int s = tid; s < S; s += kThreads) {
            const bool term = te[s];
            double m = 0.0;
            for (int a = 0; a < A; ++a) {
                const int t = tr[s * A + a];
                const double r = rw[s * A + a];
                const double qn = backup(r, gamma, term, vcur, t);
                const double qo = k == 0 ? 0.0 : backup(r, gamma, term, vprev, t);
                differs = differs || !np_isclose(qo, qn);
                if (a == 0 || qn > m || isnan(qn)) m = isnan(m) ? m : qn;  // ndarray.max: NaN propagates
            }
            vnext[s] = m;
        }
        if (!__syncthreads_or(differs)) {  // np.allclose(Q_k, Q_{k+1}): keep Q_k
            done = k;
            break;
        }
        double* t = vprev;
        vprev = vcur;
        vcur = vnext;
        vnext = t;
    }
    // Q_done = reward + gamma * next_v(V_{done-1}), V_{done-1} in vprev (Q_0 = 0)
    for (int k = tid; k < SM * A; k += kThreads) {
        const int s = k / A;
        qe[k] = (done == 0 || s >= S) ? 0.0 : backup(rw[k], gamma, te[s], vprev, tr[k]);
    }
    if (P.action) {
        __syncthreads();
        if (tid == 0) {  // np.argmax(q[state]): the first maximum (the first NaN if any)
            const long long st = P.state[e];
            long long best = -1;
            if (st >= 0 && st < S) {
                const double* row = qe + st * A;
                best = 0;
                for (int a = 1; a < A && !isnan(row[best]); ++a)
                    if (row[a] > row[best] || isnan(row[a])) best = a;
            }
            P.action[e] = best;
        }
    }
    if (tid == 0) iterations_done[e] = done;
}

}  // namespace hwyplan

// ====================================================================== C ABI
extern "C" int hwy_value_iteration(const HwyValueIterationParams* p, const int32_t* transition, const double* reward,
                                   const uint8_t* terminal, const int32_t* n_states, double* q,
                                   int32_t* iterations_done, void* stream) {
    using hwy_abi::fail;
    if (!p || !transition || !reward || !terminal || !n_states || !q || !iterations_done) return fail("%s", "null pointer");
    if (p->n_envs < 1) return fail("%s", "n_envs must be >= 1");
    if (p->s_max < 1 || p->s_max > HWY_VI_MAX_STATES) return fail("%s", "s_max out of range (1..4096)");
    if (p->n_actions < 1 || p->n_actions > HWY_VI_MAX_ACTIONS) return fail("%s", "n_actions out of range (1..8)");
    if (p->iterations < 0) return fail("%s", "iterations must be >= 0");
    if (!(p->gamma >= 0.0 && p->gamma <= 1.0)) return fail("%s", "gamma must be in [0, 1]");
    if ((p->state == nullptr) != (p->action == nullptr)) return fail("%s", "state and action go together");
    int dev_count = 0;
    if (cudaGetDeviceCount(&dev_count) != cudaSuccess || dev_count < 1) {
        cudaGetLastError();
        return fail("%s", "no CUDA device: this library has no CPU fallback");
    }
    // the opt-in to the largest size is made once (a later call may be under CUDA-graph capture); every launch passes
    // its own 3 * s_max doubles.  Per device.
    static bool opted_in[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return fail("%s", "cudaGetDevice failed");
    if (!opted_in[dev]) {
        cudaError_t err = cudaFuncSetAttribute(hwyplan::value_iteration_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               3 * HWY_VI_MAX_STATES * (int)sizeof(double));
        if (err != cudaSuccess) return fail("cudaFuncSetAttribute: %s", cudaGetErrorString(err));
        opted_in[dev] = true;
    }
    const int smem = 3 * p->s_max * (int)sizeof(double);
    hwyplan::value_iteration_kernel<<<p->n_envs, hwyplan::kThreads, smem, (cudaStream_t)stream>>>(
        *p, transition, reward, terminal, n_states, q, iterations_done);
    return hwy_abi::check_launch("value_iteration_kernel");
}
