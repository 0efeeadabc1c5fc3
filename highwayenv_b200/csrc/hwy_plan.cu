// hwy_plan.cu — planning on the device: batched value iteration of deterministic finite MDPs (the solver of
// rl-agents' ValueIterationAgent, which the reference's docs run on env.to_finite_mdp(), docs/content/algorithms.md).
// One block per env, a synchronous (Jacobi) sweep over the env's states per iteration, so every update is the
// numpy expression  reward + gamma * next_v  evaluated elementwise.  The per-state values live in shared memory.
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/hwyb200.h"
#include "hwy_abi.h"
#include "hwy_lanes.cuh"

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

// ------------------------------------------------------------------ available meta-actions
// DiscreteMetaAction.get_available_actions of the first controlled vehicle (slot 0), one thread per env
__global__ void available_actions_kernel(const HwyNetGraph* __restrict__ graph, const __grid_constant__ HwyObsView V,
                                         int n_speeds, uint8_t* __restrict__ mask) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= V.n_envs) return;
    const size_t v0 = (size_t)e * V.vp;
    const double x = V.pos[2 * v0], y = V.pos[2 * v0 + 1];
    const int lane = (V.meta[v0] >> HWY_META_LANE_SHIFT) & 0xFF;
    const int si = V.speed_index[(size_t)e * (V.n_agents > 1 ? V.n_agents : 1)];
    const HwyNetLane& L = graph->lanes[lane];
    uint8_t* m = mask + (size_t)e * 5;
    // side_lanes (road/road.py:200-211): id - 1, id + 1 of the same road, which the lane table stores consecutively
    m[0] = L.lane_id > 0 && hwynet::lane_reachable(graph->lanes[lane - 1], x, y);
    m[1] = 1;
    m[2] = L.lane_id < L.road_count - 1 && hwynet::lane_reachable(graph->lanes[lane + 1], x, y);
    m[3] = si < n_speeds - 1;
    m[4] = si > 0;
}

// ------------------------------------------------------------------ optimistic deterministic planning
// One thread per root; a tree is at most 1 + 5 * expansions nodes, scanned in node order.
constexpr int kOpdThreads = 128;

__global__ void __launch_bounds__(kOpdThreads) opd_select_kernel(const __grid_constant__ HwyOpdTree T, int k) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= T.n_roots) return;
    const size_t row = (size_t)r * T.max_nodes;
    if (k == 0) {  // root: node 0, depth 0, value 0, not terminal; no other node exists
        for (int c = 0; c < T.max_nodes; ++c) {
            T.exists[row + c] = c == 0;
            T.expanded[row + c] = 0;
            T.terminal[row + c] = 0;
            T.parent[row + c] = -1;
            T.action[row + c] = -1;
            T.depth[row + c] = 0;
            T.branch[row + c] = -1;
            T.reward[row + c] = 0.0;
            T.value[row + c] = 0.0;
            T.upper[row + c] = c == 0 ? T.bound[0] : 0.0;
        }
    }
    // open leaves created so far: the root and the children of expansions 0..k-1
    const int last = k == 0 ? 1 : 1 + T.n_actions * k;
    int best = -1;
    double best_upper = 0.0;
    for (int c = 0; c < last; ++c) {
        if (!T.exists[row + c] || T.expanded[row + c] || T.terminal[row + c]) continue;
        const double u = T.upper[row + c];
        if (best < 0 || u > best_upper) {
            best = c;
            best_upper = u;
        }
    }
    T.selected[(size_t)r * T.expansions + k] = best;
    const int64_t leaf = (int64_t)r * T.max_nodes + (best < 0 ? 0 : best);
    for (int a = 0; a < T.n_actions; ++a) T.leaf_row[(size_t)r * T.n_actions + a] = leaf;
}

__global__ void __launch_bounds__(kOpdThreads)
opd_record_kernel(const __grid_constant__ HwyOpdTree T, int k, const uint8_t* __restrict__ available,
                  const double* __restrict__ reward, const uint8_t* __restrict__ terminated,
                  const uint8_t* __restrict__ truncated) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= T.n_roots) return;
    const size_t row = (size_t)r * T.max_nodes;
    const int p = T.selected[(size_t)r * T.expansions + k];
    if (p < 0) return;  // no open leaf: the expansion is a no-op
    T.expanded[row + p] = 1;
    const int dp = T.depth[row + p];
    const double vp = T.value[row + p], g = T.discount[dp], bound = T.bound[dp + 1];
    for (int a = 0; a < T.n_actions; ++a) {
        const size_t w = (size_t)r * T.n_actions + a;
        // the leaf's available actions: the mask of work row r * n_actions (every work row holds the leaf's state)
        if (!available[(size_t)r * T.n_actions * 5 + a]) continue;
        const size_t c = row + 1 + (size_t)T.n_actions * k + a;
        const bool term = terminated[w] || truncated[w];
        const double rw = reward[w];
        const double v = vp + g * rw;
        T.exists[c] = 1;
        T.parent[c] = p;
        T.action[c] = a;
        T.depth[c] = dp + 1;
        T.branch[c] = p == 0 ? a : T.branch[row + p];
        T.reward[c] = rw;
        T.value[c] = v;
        T.terminal[c] = term;
        T.upper[c] = term ? v : v + bound;
    }
}

__global__ void __launch_bounds__(kOpdThreads) opd_recommend_kernel(const __grid_constant__ HwyOpdTree T) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= T.n_roots) return;
    const size_t row = (size_t)r * T.max_nodes;
    double best[HWY_VI_MAX_ACTIONS];
    bool seen[HWY_VI_MAX_ACTIONS];
    for (int a = 0; a < T.n_actions; ++a) seen[a] = false;
    for (int c = 1; c < T.max_nodes; ++c) {
        if (!T.exists[row + c]) continue;
        const int b = T.branch[row + c];
        const double v = T.value[row + c];
        if (!seen[b] || v > best[b]) best[b] = v;
        seen[b] = true;
    }
    int64_t rec = -1;
    for (int a = 0; a < T.n_actions; ++a)
        if (seen[a] && (rec < 0 || best[a] > best[rec])) rec = a;
    T.recommended[r] = rec;
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

extern "C" int hwy_available_actions(const HwyNetGraph* graph, const HwyObsView* view, int n_target_speeds,
                                     uint8_t* mask, void* stream) {
    using hwy_abi::fail;
    if (!graph || !view || !mask || !view->pos || !view->meta || !view->speed_index) return fail("%s", "null pointer");
    if (view->n_envs < 1) return fail("%s", "n_envs must be >= 1");
    if (n_target_speeds < 1 || n_target_speeds > HWY_MAX_TARGET_SPEEDS) return fail("%s", "n_target_speeds out of range");
    const int threads = 128;
    hwyplan::available_actions_kernel<<<(view->n_envs + threads - 1) / threads, threads, 0, (cudaStream_t)stream>>>(
        graph, *view, n_target_speeds, mask);
    return hwy_abi::check_launch("available_actions_kernel");
}

namespace {
int validate_opd(const HwyOpdTree* t) {
    using hwy_abi::fail;
    if (!t) return fail("%s", "null tree");
    if (t->n_roots < 1) return fail("%s", "n_roots must be >= 1");
    if (t->n_actions != 5) return fail("%s", "n_actions must be 5 (the meta-actions)");
    if (t->expansions < 1 || t->max_nodes != 1 + t->n_actions * t->expansions)
        return fail("%s", "max_nodes must be 1 + n_actions * expansions, expansions >= 1");
    if (!t->discount || !t->bound || !t->exists || !t->expanded || !t->terminal || !t->parent || !t->action ||
        !t->depth || !t->branch || !t->reward || !t->value || !t->upper || !t->selected || !t->leaf_row ||
        !t->recommended)
        return fail("%s", "null tree buffer");
    return 0;
}
unsigned opd_blocks(const HwyOpdTree* t) { return (t->n_roots + hwyplan::kOpdThreads - 1) / hwyplan::kOpdThreads; }
}  // namespace

extern "C" int hwy_opd_select(const HwyOpdTree* t, int k, void* stream) {
    if (validate_opd(t)) return 1;
    if (k < 0 || k >= t->expansions) return hwy_abi::fail("%s", "expansion index out of range");
    hwyplan::opd_select_kernel<<<opd_blocks(t), hwyplan::kOpdThreads, 0, (cudaStream_t)stream>>>(*t, k);
    return hwy_abi::check_launch("opd_select_kernel");
}

extern "C" int hwy_opd_record(const HwyOpdTree* t, int k, const uint8_t* available, const double* reward,
                              const uint8_t* terminated, const uint8_t* truncated, void* stream) {
    if (validate_opd(t)) return 1;
    if (k < 0 || k >= t->expansions) return hwy_abi::fail("%s", "expansion index out of range");
    if (!available || !reward || !terminated || !truncated) return hwy_abi::fail("%s", "null pointer");
    hwyplan::opd_record_kernel<<<opd_blocks(t), hwyplan::kOpdThreads, 0, (cudaStream_t)stream>>>(
        *t, k, available, reward, terminated, truncated);
    return hwy_abi::check_launch("opd_record_kernel");
}

extern "C" int hwy_opd_recommend(const HwyOpdTree* t, void* stream) {
    if (validate_opd(t)) return 1;
    hwyplan::opd_recommend_kernel<<<opd_blocks(t), hwyplan::kOpdThreads, 0, (cudaStream_t)stream>>>(*t);
    return hwy_abi::check_launch("opd_recommend_kernel");
}
