// hwy_lanes_debug.cu — the test entry hwy_debug_network_lanes: the lane functions of the network kernels
// (hwy_lanes.cuh) on one input per thread, on the lane table as the kernels stage it.  A translation unit of its own:
// the lane functions are noinline, and a new caller in hwy_network.cu would change how the step kernels call them.
#include <cuda_runtime.h>

#include "../../include/hwyb200.h"
#include "hwy_abi.h"
#include "hwy_lanes.cuh"

namespace hwylanes {
using namespace hwynet;

constexpr int kThreads = 256;

// The lane functions on one input per thread (hwy_debug_network_lanes; operands in include/hwyb200.h)
__host__ __device__ inline int lanes_out_width(int op) {
    switch (op) {
        case HWY_LANES_LOCAL: case HWY_LANES_POSITION: return 2;
        case HWY_LANES_DISTANCE_WITH_HEADING: return 3;
        case HWY_LANES_PRUNABLE_SCAN: return HWY_NET_MAX_LANES;
        default: return 1;
    }
}
__global__ void __launch_bounds__(kThreads)
debug_lanes_kernel(const HwyNetGraph* __restrict__ graph, int op, const double* __restrict__ in,
                   double* __restrict__ out, int n) {
    __shared__ GraphShared g;
    stage_graph(g, graph);
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const double* a = in + (size_t)k * HWY_LANES_IN;
    double* o = out + (size_t)k * lanes_out_width(op);
    const int l = (int)fmin(fmax(a[0], -1.0), (double)HWY_NET_MAX_LANES);
    if (!(a[0] == (double)l && l >= 0 && l < g.n_lanes)) {
        for (int j = 0; j < lanes_out_width(op); ++j) o[j] = __longlong_as_double(0x7ff8000000000000LL);
        return;
    }
    const HwyNetLane& L = g.lanes[l];
    switch (op) {
        case HWY_LANES_LOCAL: lane_local(L, a[1], a[2], o[0], o[1]); break;
        case HWY_LANES_POSITION: lane_position(L, a[1], a[2], o[0], o[1]); break;
        case HWY_LANES_HEADING_AT: o[0] = lane_heading_at(L, a[1]); break;
        case HWY_LANES_DISTANCE_WITH_HEADING: {
            double s, lat;
            o[0] = lane_distance_with_heading(L, a[1], a[2], a[3], s, lat);
            o[1] = s;
            o[2] = lat;
            break;
        }
        case HWY_LANES_ON: {
            double s, lat;
            lane_local(L, a[1], a[2], s, lat);
            o[0] = lane_on(L, s, lat, 1.0) ? 1.0 : 0.0;
            break;
        }
        case HWY_LANES_MAYBE_ON: o[0] = lane_maybe_on(L, a[1], a[2]) ? 1.0 : 0.0; break;
        case HWY_LANES_PRUNABLE: {
            CircleCache cc = {0.0, 0.0, 0.0, false};
            o[0] = closest_lane_prunable(L, a[1], a[2], a[3], cc) ? 1.0 : 0.0;
            break;
        }
        case HWY_LANES_PRUNABLE_SCAN: {
            CircleCache cc = {0.0, 0.0, 0.0, false};
            for (int m = 0; m < HWY_NET_MAX_LANES; ++m) {
                const bool scanned = m < g.n_lanes && m != l;
                o[m] = scanned && closest_lane_prunable(g.lanes[m], a[1], a[2], a[3], cc) ? 1.0 : 0.0;
            }
            break;
        }
    }
}

}  // namespace hwylanes

using hwy_abi::check_launch;
using hwy_abi::fail;

extern "C" {

int hwy_debug_network_lanes(const HwyNetGraph* graph, int op, const double* in, double* out, int n, void* stream) {
    if (op < HWY_LANES_LOCAL || op > HWY_LANES_PRUNABLE_SCAN) return fail("%s", "hwy_debug_network_lanes: unknown op");
    if (n < 0) return fail("%s", "hwy_debug_network_lanes: n < 0");
    if (!graph || !in || !out) return fail("%s", "hwy_debug_network_lanes: null pointer");
    if (graph->n_lanes < 1 || graph->n_lanes > HWY_NET_MAX_LANES)
        return fail("%s", "hwy_debug_network_lanes: n_lanes outside 1..HWY_NET_MAX_LANES");
    if (n == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    HwyNetGraph* d_graph = nullptr;
    cudaError_t err = cudaMallocAsync((void**)&d_graph, sizeof(HwyNetGraph), st);
    if (err != cudaSuccess) {
        cudaGetLastError();
        return fail("hwy_debug_network_lanes: %s", cudaGetErrorString(err));
    }
    cudaMemcpyAsync(d_graph, graph, sizeof(HwyNetGraph), cudaMemcpyHostToDevice, st);
    hwylanes::debug_lanes_kernel<<<(n + hwylanes::kThreads - 1) / hwylanes::kThreads, hwylanes::kThreads, 0, st>>>(
        d_graph, op, in, out, n);
    const int rc = check_launch("debug_lanes_kernel");
    cudaFreeAsync(d_graph, st);
    return rc;
}

}  // extern "C"
