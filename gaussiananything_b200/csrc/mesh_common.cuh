// Shared pieces of the mesh-extraction kernels (mesh_tsdf.cu, mesh_extract.cu): the device-wide exclusive scan that
// turns per-item counts into output offsets, and the status read-back of include/ga_b200.h Part 4.
#pragma once
#include "../../include/ga_b200.h"
#include <cuda_runtime.h>

// both mesh .cu files include this: the kernels are static (internal linkage)
namespace ga_mesh {

constexpr int SCAN_BLOCK = 1024;

static inline int scan_partials(int64_t n) { return (int)((n + SCAN_BLOCK - 1) / SCAN_BLOCK); }

// exclusive scan of x over the 1024 threads of the block; *total = the block's sum (every thread)
static __device__ __forceinline__ int block_exclusive_scan(int x, int *total)
{
    __shared__ int warp_sum[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) warp_sum[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        int s = warp_sum[lane], si = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, si, o);
            if (lane >= o) si += y;
        }
        warp_sum[lane] = si - s;                       // exclusive prefix of the warp sums
    }
    __syncthreads();
    const int r = inc - x + warp_sum[warp];
    // the block total: the last warp's exclusive prefix plus its own sum
    __shared__ int tot;
    if (threadIdx.x == SCAN_BLOCK - 1) tot = warp_sum[31] + inc;
    __syncthreads();
    *total = tot;
    __syncthreads();                                   // warp_sum / tot may be reused by the next call
    return r;
}

static __global__ void __launch_bounds__(SCAN_BLOCK) scan_blocks_kernel(int *a, int64_t n, int *partials)
{
    const int64_t i = (int64_t)blockIdx.x * SCAN_BLOCK + threadIdx.x;
    const int x = i < n ? a[i] : 0;
    int tot;
    const int e = block_exclusive_scan(x, &tot);
    if (i < n) a[i] = e;
    if (threadIdx.x == 0) partials[blockIdx.x] = tot;
}

static __global__ void __launch_bounds__(SCAN_BLOCK) scan_partials_kernel(int *partials, int nb, int *total)
{
    int carry = 0;
    for (int base = 0; base < nb; base += SCAN_BLOCK) {
        const int i = base + threadIdx.x;
        const int x = i < nb ? partials[i] : 0;
        int tot;
        const int e = block_exclusive_scan(x, &tot);
        if (i < nb) partials[i] = e + carry;
        carry += tot;
    }
    if (threadIdx.x == 0) *total = carry;
}

static __global__ void __launch_bounds__(256) scan_add_kernel(int *a, int64_t n, const int *partials)
{
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i < n) a[i] += partials[i / SCAN_BLOCK];
}

// a[0..n) <- exclusive prefix sums of a (int32, in place); *total (device) <- the sum.
// partials: int32[scan_partials(n)].
static inline cudaError_t scan_exclusive(int *a, int64_t n, int *partials, int *total, cudaStream_t s)
{
    if (n <= 0) return cudaMemsetAsync(total, 0, sizeof(int), s);
    const int nb = scan_partials(n);
    scan_blocks_kernel<<<nb, SCAN_BLOCK, 0, s>>>(a, n, partials);
    scan_partials_kernel<<<1, SCAN_BLOCK, 0, s>>>(partials, nb, total);
    scan_add_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(a, n, partials);
    return cudaGetLastError();
}

// status_host / status_event: both NULL or both set; when set, copy the status words and record the event
static inline cudaError_t publish_status(const int32_t *status, int32_t *status_host, void *status_event,
                                         cudaStream_t s)
{
    if (status_host == nullptr) return cudaSuccess;
    cudaError_t e = cudaMemcpyAsync(status_host, status, GA_MESH_STATUS_INTS * sizeof(int32_t),
                                    cudaMemcpyDeviceToHost, s);
    if (e != cudaSuccess) return e;
    return cudaEventRecord((cudaEvent_t)status_event, s);
}

}  // namespace ga_mesh
