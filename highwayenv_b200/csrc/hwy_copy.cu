// hwy_copy.cu — env cloning: copy the per-env rows of a set of buffers from source rows to destination rows, the device
// side of `copy.deepcopy(env)` for a batch of envs (BatchedVectorEnv.copy_envs).  One launch covers every buffer of the
// env; a warp copies one (pair, buffer) row, with 16-byte accesses where the row's alignment allows.
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/hwyb200.h"
#include "hwy_abi.h"

namespace hwycopy {

constexpr int kWarps = 8;  // warps per block: one row each

struct RowCopyTable {
    HwyRowCopy buf[HWY_COPY_MAX_BUFS];
};

template <typename T>
__device__ __forceinline__ void copy_row(const char* __restrict__ s, char* __restrict__ d, int64_t n, int lane) {
    const T* src = reinterpret_cast<const T*>(s);
    T* dst = reinterpret_cast<T*>(d);
    for (int64_t k = lane; k < n; k += 32) dst[k] = src[k];
}

// grid (ceil(n_pairs / kWarps), n_bufs): warp w of block (x, b) copies row src[x * kWarps + w] of buffer b
__global__ void __launch_bounds__(kWarps * 32)
copy_env_rows_kernel(const __grid_constant__ RowCopyTable T, const int64_t* __restrict__ dst,
                     const int64_t* __restrict__ src, int n_pairs) {
    const int pair = blockIdx.x * kWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (pair >= n_pairs) return;
    const HwyRowCopy& B = T.buf[blockIdx.y];
    const int64_t bytes = B.row_bytes;
    const char* s = static_cast<const char*>(B.src) + src[pair] * bytes;
    char* d = static_cast<char*>(B.dst) + dst[pair] * bytes;
    const uintptr_t align = reinterpret_cast<uintptr_t>(B.src) | reinterpret_cast<uintptr_t>(B.dst) | (uintptr_t)bytes;
    if ((align & 15) == 0)
        copy_row<int4>(s, d, bytes / 16, lane);
    else if ((align & 3) == 0)
        copy_row<int32_t>(s, d, bytes / 4, lane);
    else
        copy_row<char>(s, d, bytes, lane);
}

}  // namespace hwycopy

// ====================================================================== C ABI
extern "C" int hwy_copy_env_rows(const HwyRowCopy* bufs, int n_bufs, const int64_t* dst, const int64_t* src,
                                 int n_pairs, void* stream) {
    using hwy_abi::fail;
    if (n_pairs < 0 || n_bufs < 0) return fail("%s", "n_pairs and n_bufs must be >= 0");
    if (n_bufs > HWY_COPY_MAX_BUFS) return fail("%s", "more than HWY_COPY_MAX_BUFS buffers");
    if (n_pairs == 0 || n_bufs == 0) return 0;
    if (!bufs || !dst || !src) return fail("%s", "null pointer");
    hwycopy::RowCopyTable table = {};
    for (int b = 0; b < n_bufs; ++b) {
        if (!bufs[b].src || !bufs[b].dst) return fail("%s", "null buffer");
        if (bufs[b].row_bytes <= 0) return fail("%s", "row_bytes must be > 0");
        table.buf[b] = bufs[b];
    }
    const dim3 grid((n_pairs + hwycopy::kWarps - 1) / hwycopy::kWarps, n_bufs);
    hwycopy::copy_env_rows_kernel<<<grid, hwycopy::kWarps * 32, 0, (cudaStream_t)stream>>>(table, dst, src, n_pairs);
    return hwy_abi::check_launch("copy_env_rows_kernel");
}
