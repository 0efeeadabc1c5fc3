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

// ------------------------------------------------------------------ Monte-Carlo tree search
// One thread per root, tests/mcts_spec.py step for step.  fp64 arithmetic is spelled with _rn intrinsics so that no
// contraction can round differently from numpy.
constexpr int kMctsThreads = 128;
constexpr uint8_t kWalkDone = 1, kWalkRolling = 2;
constexpr int kIdle = 1;

__device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// mcts_spec.draw: the finaliser chained over (seed, decision, root, episode, depth, purpose)
__device__ __forceinline__ uint64_t mcts_draw(const HwyMctsTree& T, int r, int e, int d, int purpose) {
    const uint64_t words[6] = {T.seed, (uint64_t)*T.decision, (uint64_t)r, (uint64_t)e, (uint64_t)d,
                               (uint64_t)purpose};
    uint64_t x = 0;
    for (int k = 0; k < 6; ++k) x = splitmix64(x + 0x9E3779B97F4A7C15ull + words[k]);
    return x;
}

// mcts_spec.pick: floor(u * k), u = (x >> 11) 2^-53, exactly ((x >> 11) * k < 2^56)
__device__ __forceinline__ int mcts_pick(uint64_t x, int k) { return (int)(((x >> 11) * (uint64_t)k) >> 53); }

// the j-th set bit of a 5-bit mask in ascending order
__device__ __forceinline__ int nth_set(unsigned mask, int j) {
    for (int a = 0; a < 5; ++a)
        if (mask >> a & 1u) {
            if (j == 0) return a;
            --j;
        }
    return kIdle;
}

__device__ void mcts_clear(const HwyMctsTree& T, size_t row, int start) {
    for (int c = start; c < T.max_nodes; ++c) {
        T.exists[row + c] = 0;
        T.expanded[row + c] = 0;
        T.parent[row + c] = -1;
        T.action[row + c] = -1;
        T.child_base[row + c] = -1;
        T.n_children[row + c] = 0;
        T.count[row + c] = 0;
        T.prior[row + c] = 0.0;
        T.value[row + c] = 0.0;
    }
    if (start == 0) {
        T.exists[row] = 1;
        T.prior[row] = 1.0;
    }
}

__global__ void __launch_bounds__(kMctsThreads)
mcts_advance_kernel(const __grid_constant__ HwyMctsTree T, int e, int d, const uint8_t* __restrict__ available,
                    const double* __restrict__ reward, const uint8_t* __restrict__ terminated,
                    const uint8_t* __restrict__ truncated) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= T.n_roots) return;
    const size_t row = (size_t)r * T.max_nodes;
    int node = 0;
    double ret = 0.0;
    uint8_t flags = 0;
    if (d == 0) {
        if (e == 0) T.skipped[r] = 0;
    } else {
        node = T.walk_node[r];
        ret = T.walk_return[r];
        flags = T.walk_flags[r];
        if (!(flags & kWalkDone)) {
            ret = __dadd_rn(ret, __dmul_rn(T.discount[d - 1], reward[r]));
            if (terminated[r] || truncated[r]) flags |= kWalkDone;
        }
    }
    unsigned avail = 0;
    for (int a = 0; a < 5; ++a) avail |= (available[(size_t)r * 5 + a] ? 1u : 0u) << a;
    int act = kIdle;
    if (!(flags & kWalkDone)) {
        bool descended = false;
        if (!(flags & kWalkRolling)) {
            if (T.expanded[row + node]) {  // descent: the best score, exact ties by a draw
                const int base = T.child_base[row + node];
                const double tn = __dmul_rn(T.temperature, (double)T.n_children[row + node]);
                double score[5], best = 0.0;
                unsigned cand = 0;
                for (int a = 0; a < 5; ++a) {
                    const size_t c = row + base + a;
                    if (!T.exists[c]) continue;
                    score[a] = __dadd_rn(T.value[c], __ddiv_rn(__dmul_rn(tn, T.prior[c]), (double)(T.count[c] + 1)));
                    if (!cand || score[a] > best) best = score[a];
                    cand |= 1u << a;
                }
                unsigned ties = 0;
                for (int a = 0; a < 5; ++a)
                    if ((cand >> a & 1u) && score[a] == best) ties |= 1u << a;
                act = nth_set(ties, mcts_pick(mcts_draw(T, r, e, d, 0), __popc(ties)));
                node = base + act;
                descended = true;
            } else {  // expansion of the leaf, unless the tree is full
                const int base = T.n_nodes[r];
                if (base + 5 > T.max_nodes) {
                    T.skipped[r] += 1;
                } else {
                    const int k = __popc(avail);
                    T.n_nodes[r] = base + 5;
                    T.expanded[row + node] = 1;
                    T.child_base[row + node] = base;
                    T.n_children[row + node] = k;
                    for (int a = 0; a < 5; ++a) {
                        const size_t c = row + base + a;
                        const bool ok = avail >> a & 1u;
                        T.parent[c] = node;
                        T.action[c] = a;
                        T.exists[c] = ok;
                        T.prior[c] = ok ? __ddiv_rn(1.0, (double)k) : 0.0;
                    }
                }
                flags |= kWalkRolling;
            }
        }
        if (!descended) act = nth_set(avail, mcts_pick(mcts_draw(T, r, e, d, 1), __popc(avail)));
    }
    T.actions[r] = act;
    T.walk_node[r] = node;
    T.walk_return[r] = ret;
    T.walk_flags[r] = flags;
}

__global__ void __launch_bounds__(kMctsThreads)
mcts_backup_kernel(const __grid_constant__ HwyMctsTree T, int e, const double* __restrict__ reward) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= T.n_roots) return;
    const size_t row = (size_t)r * T.max_nodes;
    const int node = T.walk_node[r];
    double ret = T.walk_return[r];
    // the last step's flags end nothing: only its reward counts
    if (!(T.walk_flags[r] & kWalkDone)) ret = __dadd_rn(ret, __dmul_rn(T.discount[T.horizon - 1], reward[r]));
    for (int c = node; c >= 0; c = T.parent[row + c]) {
        const int n = T.count[row + c] + 1;
        const double v = T.value[row + c];
        T.count[row + c] = n;
        T.value[row + c] = __dadd_rn(v, __dmul_rn(__ddiv_rn(1.0, (double)n), __dsub_rn(ret, v)));
    }
    T.leaf[(size_t)r * T.episodes + e] = node;
    T.returns[(size_t)r * T.episodes + e] = ret;
}

__global__ void __launch_bounds__(kMctsThreads) mcts_recommend_kernel(const __grid_constant__ HwyMctsTree T) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r == 0) *T.decision += 1;  // no thread of this kernel draws
    if (r >= T.n_roots) return;
    const size_t row = (size_t)r * T.max_nodes;
    int64_t rec = -1;
    if (T.expanded[row]) {
        const int base = T.child_base[row];
        for (int a = 0; a < 5; ++a) {
            const size_t c = row + base + a;
            if (!T.exists[c]) continue;
            const size_t b = row + base + rec;
            if (rec < 0 || T.count[c] > T.count[b] || (T.count[c] == T.count[b] && T.value[c] > T.value[b])) rec = a;
        }
    }
    T.recommended[r] = rec;
}

__global__ void __launch_bounds__(kMctsThreads)
mcts_reroot_kernel(const __grid_constant__ HwyMctsTree T, const int64_t* __restrict__ actions,
                   const uint8_t* __restrict__ done) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= T.n_roots) return;
    const size_t row = (size_t)r * T.max_nodes;
    int c = -1;
    if (actions && !done[r] && T.expanded[row]) {
        const int64_t a = actions[r];
        if (a >= 0 && a < 5 && T.exists[row + T.child_base[row] + a]) c = T.child_base[row] + (int)a;
    }
    if (c < 0) {
        mcts_clear(T, row, 0);
        T.n_nodes[r] = 1;
        return;
    }
    // the kept slots: c, then every slot whose parent is kept (parents precede children); new indices in order
    int32_t* remap = T.remap + row;
    for (int j = 0; j < T.max_nodes; ++j) remap[j] = -1;
    remap[c] = 0;
    int k = 1;
    for (int j = c + 1; j < T.max_nodes; ++j) {
        const int p = T.parent[row + j];
        if (p >= 0 && remap[p] >= 0) remap[j] = k++;
    }
    for (int j = c; j < T.max_nodes; ++j) {  // remap[j] <= j: in place, ascending
        const int n = remap[j];
        if (n < 0) continue;
        const size_t s = row + j, t = row + n;
        const int p = T.parent[s], cb = T.child_base[s];
        T.exists[t] = T.exists[s];
        T.expanded[t] = T.expanded[s];
        T.action[t] = T.action[s];
        T.n_children[t] = T.n_children[s];
        T.count[t] = T.count[s];
        T.prior[t] = T.prior[s];
        T.value[t] = T.value[s];
        T.parent[t] = j == c ? -1 : remap[p];
        T.child_base[t] = cb < 0 ? -1 : remap[cb];
    }
    mcts_clear(T, row, k);
    T.n_nodes[r] = k;
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
    if (hwy_abi::require_device()) return 1;
    // The opt-in is to the largest size, made by the first call on a device, so that no later call has to raise it (a
    // later call may be under CUDA-graph capture); every launch passes its own 3 * s_max doubles.
    if (hwy_abi::opt_in_smem((const void*)hwyplan::value_iteration_kernel, 3 * HWY_VI_MAX_STATES * sizeof(double)))
        return 1;
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

namespace {
int validate_mcts(const HwyMctsTree* t) {
    using hwy_abi::fail;
    if (!t) return fail("%s", "null tree");
    if (t->n_roots < 1) return fail("%s", "n_roots must be >= 1");
    if (t->max_nodes < 6 || (t->max_nodes - 1) % 5 != 0) return fail("%s", "max_nodes must be 1 + 5 k, k >= 1");
    if (t->episodes < 1 || t->horizon < 1) return fail("%s", "episodes and horizon must be >= 1");
    if (!(t->temperature >= 0.0 && t->temperature <= 1.7976931348623157e308))
        return fail("%s", "temperature must be finite and >= 0");
    if (!t->discount || !t->decision || !t->exists || !t->expanded || !t->parent || !t->action || !t->child_base ||
        !t->n_children || !t->count || !t->prior || !t->value || !t->n_nodes || !t->skipped || !t->walk_node ||
        !t->walk_return || !t->walk_flags || !t->leaf || !t->returns || !t->remap || !t->actions || !t->recommended)
        return fail("%s", "null tree buffer");
    return 0;
}
unsigned mcts_blocks(const HwyMctsTree* t) { return (t->n_roots + hwyplan::kMctsThreads - 1) / hwyplan::kMctsThreads; }
}  // namespace

extern "C" int hwy_mcts_advance(const HwyMctsTree* t, int e, int d, const uint8_t* available, const double* reward,
                                const uint8_t* terminated, const uint8_t* truncated, void* stream) {
    if (validate_mcts(t)) return 1;
    if (e < 0 || e >= t->episodes || d < 0 || d >= t->horizon) return hwy_abi::fail("%s", "episode or step out of range");
    if (!available || !reward || !terminated || !truncated) return hwy_abi::fail("%s", "null pointer");
    hwyplan::mcts_advance_kernel<<<mcts_blocks(t), hwyplan::kMctsThreads, 0, (cudaStream_t)stream>>>(
        *t, e, d, available, reward, terminated, truncated);
    return hwy_abi::check_launch("mcts_advance_kernel");
}

extern "C" int hwy_mcts_backup(const HwyMctsTree* t, int e, const double* reward, void* stream) {
    if (validate_mcts(t)) return 1;
    if (e < 0 || e >= t->episodes) return hwy_abi::fail("%s", "episode out of range");
    if (!reward) return hwy_abi::fail("%s", "null pointer");
    hwyplan::mcts_backup_kernel<<<mcts_blocks(t), hwyplan::kMctsThreads, 0, (cudaStream_t)stream>>>(*t, e, reward);
    return hwy_abi::check_launch("mcts_backup_kernel");
}

extern "C" int hwy_mcts_recommend(const HwyMctsTree* t, void* stream) {
    if (validate_mcts(t)) return 1;
    hwyplan::mcts_recommend_kernel<<<mcts_blocks(t), hwyplan::kMctsThreads, 0, (cudaStream_t)stream>>>(*t);
    return hwy_abi::check_launch("mcts_recommend_kernel");
}

extern "C" int hwy_mcts_reroot(const HwyMctsTree* t, const int64_t* actions, const uint8_t* done, void* stream) {
    if (validate_mcts(t)) return 1;
    if ((actions == nullptr) != (done == nullptr)) return hwy_abi::fail("%s", "actions and done go together");
    hwyplan::mcts_reroot_kernel<<<mcts_blocks(t), hwyplan::kMctsThreads, 0, (cudaStream_t)stream>>>(*t, actions, done);
    return hwy_abi::check_launch("mcts_reroot_kernel");
}
