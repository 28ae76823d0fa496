// Surface point clouds (include/ga_b200.h Part 10):
//   chunk_surface_points : a G-buffer chunk's depth maps -> the kept surface points of the chosen views, compacted in
//                          view-major, row-major order (count, scan, emit; the pixels are unprojected twice rather
//                          than stored)
//   fps_ex               : farthest-point sampling of clouds too large for one CTA.  A cooperative grid: every CTA
//                          keeps a slice of its cloud in registers (the rest in global memory), each round ends in one
//                          64-bit atomicMax per CTA into the round's slot and one grid.sync().
// This file is compiled without FMA contraction: the unprojection is gbuffer_pack_kernel's to the bit, and the FPS
// distance is (dx*dx + dy*dy) + dz*dz with each operation rounded on its own.
#include "../../include/ga_b200.h"
#include "device_once.cuh"
#include "gbuffer_common.cuh"
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace cg = cooperative_groups;

namespace {

// ---------------------------------------------------------------------------------------------------------------
// Chunk surface points.  A block takes 1024 pixels of one view (256 threads x 4 consecutive pixels of a row).
// ---------------------------------------------------------------------------------------------------------------
constexpr int kSpThreads = 256, kSpPix = 4 * kSpThreads, kScanThreads = 1024;

struct SurfArgs {
    const uint8_t *alpha;
    const float *depth, *cams;
    const int32_t *views;
    int n_chunk, H, W, blocks_per_view;
    int alpha_min;
    float min_depth;
    int32_t *block_off;   // [n_views * blocks_per_view]: kept pixels per block, then (scan) their exclusive offsets
    int32_t *count;
    float *points;
};

// keep[i] and xyz[i] of the thread's four pixels; returns how many are kept
__device__ __forceinline__ int surf_pixels(const SurfArgs &a, const float *cam, int view, int p0, bool keep[4],
                                           float xyz[4][3])
{
    const int H = a.H, W = a.W, HW = H * W;
    int n = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) keep[i] = false;
    if (p0 >= HW) return 0;
    const int y = p0 / W, x0 = p0 - y * W;
    const float4 dep = __ldg(reinterpret_cast<const float4 *>(a.depth + (size_t)view * HW + p0));
    const float d4[4] = {dep.x, dep.y, dep.z, dep.w};
    const uint32_t aw = __ldg(reinterpret_cast<const uint32_t *>(a.alpha + ((size_t)y * a.n_chunk + view) * W + x0));
    const float v_cam = ((float)y + 0.5f) / (float)H;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const float u_cam = ((float)(x0 + i) + 0.5f) / (float)W;
        gbuf::unproject(cam, u_cam, v_cam, d4[i], xyz[i]);
        const int al = (int)((aw >> (8 * i)) & 0xffu);
        keep[i] = al >= a.alpha_min && d4[i] >= a.min_depth && xyz[i][0] != 0.0f && xyz[i][1] != 0.0f &&
                  xyz[i][2] != 0.0f;
        n += keep[i];
    }
    return n;
}

// grid (blocks_per_view, n_views): the kept count of each block
__global__ void __launch_bounds__(kSpThreads) surf_count_kernel(SurfArgs a)
{
    __shared__ float cam[25];
    __shared__ int wsum[kSpThreads / 32];
    const int slot = blockIdx.y, view = a.views[slot];
    for (int i = threadIdx.x; i < 25; i += blockDim.x) cam[i] = a.cams[view * 25 + i];
    __syncthreads();
    bool keep[4];
    float xyz[4][3];
    int n = surf_pixels(a, cam, view, blockIdx.x * kSpPix + threadIdx.x * 4, keep, xyz);
#pragma unroll
    for (int o = 16; o; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < kSpThreads / 32; w++) t += wsum[w];
        a.block_off[slot * a.blocks_per_view + blockIdx.x] = t;
    }
}

// one block: exclusive scan of the block counts in place, total to *count
__global__ void __launch_bounds__(kScanThreads) surf_scan_kernel(int32_t *__restrict__ off, int n, int32_t *__restrict__ count)
{
    __shared__ int wsum[kScanThreads / 32];
    __shared__ int carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += kScanThreads) {
        const int i = base + threadIdx.x;
        const int v = i < n ? off[i] : 0;
        int x = v;                                                       // inclusive warp scan
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) wsum[warp] = x;
        __syncthreads();
        if (warp == 0) {
            int s = wsum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, s, o);
                if (lane >= o) s += y;
            }
            wsum[lane] = s;                                              // inclusive over warps
        }
        __syncthreads();
        const int c = carry;
        const int excl = c + (warp ? wsum[warp - 1] : 0) + x - v;
        if (i < n) off[i] = excl;
        __syncthreads();
        if (threadIdx.x == kScanThreads - 1) carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) *count = carry;
}

// grid (blocks_per_view, n_views): the kept points of each block at its offset, in pixel order
__global__ void __launch_bounds__(kSpThreads) surf_emit_kernel(SurfArgs a)
{
    __shared__ float cam[25];
    __shared__ int wsum[kSpThreads / 32];
    const int slot = blockIdx.y, view = a.views[slot], lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < 25; i += blockDim.x) cam[i] = a.cams[view * 25 + i];
    __syncthreads();
    bool keep[4];
    float xyz[4][3];
    const int n = surf_pixels(a, cam, view, blockIdx.x * kSpPix + threadIdx.x * 4, keep, xyz);
    int x = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    int pos = a.block_off[slot * a.blocks_per_view + blockIdx.x] + x - n;
    for (int w = 0; w < warp; w++) pos += wsum[w];
    float *out = a.points + (size_t)pos * 3;
#pragma unroll
    for (int i = 0; i < 4; i++)
        if (keep[i]) {
            out[0] = xyz[i][0];
            out[1] = xyz[i][1];
            out[2] = xyz[i][2];
            out += 3;
        }
}

// ---------------------------------------------------------------------------------------------------------------
// Farthest-point sampling on a cooperative grid.  Cloud b has `cpc` CTAs; CTA j of it owns the points
// p = j * T + t + i * (cpc * T): i < kFxReg in registers, the rest (p >= kFxReg * cpc * T) with their running minimum
// in global memory.  A thread visits its points in increasing p, so a strict > keeps its lowest index among equal
// distances; across threads and CTAs the key (distance bits << 32 | ~p) makes atomicMax do the same.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kFxThreads = 512, kFxReg = 14;   // 14 points per thread: 126 registers, no spill

struct FpsArgs {
    const float *pcd;
    const int32_t *lengths, *start;
    int batch, N, K, cpc;
    int32_t *idx_out;
    float *xyz_out;
    unsigned long long *slots;   // [batch, K]
    float *md;                   // [batch, N]: running minimum of the points beyond the registers
};

__device__ __forceinline__ int cloud_len(const FpsArgs &a, int b)
{
    return a.lengths ? min(max(__ldg(a.lengths + b), 0), a.N) : a.N;
}

__device__ __forceinline__ float sq_dist(float px, float py, float pz, float sx, float sy, float sz)
{
    const float dx = __fsub_rn(px, sx), dy = __fsub_rn(py, sy), dz = __fsub_rn(pz, sz);
    return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__global__ void __launch_bounds__(kFxThreads, 1) fps_grid_kernel(FpsArgs a)
{
    __shared__ unsigned long long wkey[kFxThreads / 32];
    cg::grid_group grid = cg::this_grid();
    const int b = blockIdx.x / a.cpc, j = blockIdx.x - b * a.cpc, tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5, K = a.K;
    const int stride = a.cpc * kFxThreads, first = j * kFxThreads + tid;
    const int len = cloud_len(a, b), kb = min(K, len);
    int rounds = 0;                                                      // the grid runs the longest cloud's rounds
    for (int c = 0; c < a.batch; c++) rounds = max(rounds, min(K, cloud_len(a, c)));
    const float *P = a.pcd + (size_t)b * a.N * 3;
    float *md_g = a.md + (size_t)b * a.N;
    unsigned long long *slot = a.slots + (size_t)b * K;

    for (size_t i = (size_t)blockIdx.x * kFxThreads + tid; i < (size_t)a.batch * K; i += (size_t)gridDim.x * kFxThreads)
        a.slots[i] = 0ull;
    float px[kFxReg], py[kFxReg], pz[kFxReg], md[kFxReg];
#pragma unroll
    for (int i = 0; i < kFxReg; i++) {
        const int p = first + i * stride;
        const bool in = p < len;
        px[i] = in ? __ldg(P + 3 * p) : 0.f;
        py[i] = in ? __ldg(P + 3 * p + 1) : 0.f;
        pz[i] = in ? __ldg(P + 3 * p + 2) : 0.f;
        md[i] = INFINITY;
    }
    for (int p = first + kFxReg * stride; p < len; p += stride) md_g[p] = INFINITY;
    if (j == 0)                                                          // slots past the cloud's length
        for (int k = kb + tid; k < K; k += kFxThreads) {
            a.idx_out[(size_t)b * K + k] = -1;
            float *o = a.xyz_out + ((size_t)b * K + k) * 3;
            o[0] = o[1] = o[2] = 0.f;
        }
    grid.sync();

    int cur = kb > 0 ? __ldg(a.start + b) : 0;
    for (int k = 0; k < rounds; k++) {
        const bool active = k + 1 < kb;                                  // this cloud selects point k + 1
        if (k < kb) {
            const float sx = __ldg(P + 3 * cur), sy = __ldg(P + 3 * cur + 1), sz = __ldg(P + 3 * cur + 2);
            if (j == 0 && tid == 0) {
                a.idx_out[(size_t)b * K + k] = cur;
                float *o = a.xyz_out + ((size_t)b * K + k) * 3;
                o[0] = sx; o[1] = sy; o[2] = sz;
            }
            if (active) {
                float best = -1.f;
                int bi = -1;
#pragma unroll
                for (int i = 0; i < kFxReg; i++) {
                    const int p = first + i * stride;
                    if (p < len) {
                        md[i] = fminf(md[i], sq_dist(px[i], py[i], pz[i], sx, sy, sz));
                        if (md[i] > best) { best = md[i]; bi = p; }
                    }
                }
                for (int p = first + kFxReg * stride; p < len; p += stride) {
                    const float d = fminf(__ldcg(md_g + p),
                                          sq_dist(__ldg(P + 3 * p), __ldg(P + 3 * p + 1), __ldg(P + 3 * p + 2), sx, sy, sz));
                    __stcg(md_g + p, d);
                    if (d > best) { best = d; bi = p; }
                }
                unsigned long long key = bi < 0 ? 0ull
                    : ((unsigned long long)__float_as_uint(best) << 32) | (unsigned long long)(~(uint32_t)bi);
#pragma unroll
                for (int o = 16; o; o >>= 1) {
                    const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, o);
                    key = other > key ? other : key;
                }
                if (lane == 0) wkey[warp] = key;
                __syncthreads();
                if (tid == 0) {
                    for (int w = 1; w < kFxThreads / 32; w++) key = wkey[w] > key ? wkey[w] : key;
                    atomicMax(slot + k + 1, key);
                }
            }
        }
        if (k + 1 == rounds) break;
        grid.sync();
        if (active) cur = (int)~(uint32_t)__ldcg(slot + k + 1);
    }
}

struct FpsGrid {
    int max_ctas;       // co-resident CTAs of fps_grid_kernel on the current device
};

FpsGrid fps_grid()
{
    static GaPerDevice f;
    int dev = 0;
    if (ga_first_use_on_device(f, &dev) || dev < 0 || dev >= 64) {
        int per_sm = 0, coop = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fps_grid_kernel, kFxThreads, 0);
        cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
        const int n = coop ? per_sm * ga_sm_count() : 0;
        if (dev < 0 || dev >= 64) return {n};
        f.value[dev] = n;
    }
    return {f.value[dev]};
}

constexpr size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

}  // namespace

extern "C" size_t ga_chunk_surface_points_scratch_bytes(int n_views, int H, int W)
{
    if (n_views <= 0 || H <= 0 || W <= 0) return 0;
    return (size_t)n_views * (((size_t)H * W + kSpPix - 1) / kSpPix) * sizeof(int32_t);
}

extern "C" int ga_chunk_surface_points(const uint8_t *alpha, const float *depth, const float *cams, int n_chunk, int H,
                                       int W, const int32_t *views, int n_views, int alpha_min, float min_depth,
                                       float *points, int32_t *count, void *scratch, size_t scratch_bytes,
                                       void *stream)
{
    if (!alpha || !depth || !cams || !views || !points || !count || !scratch || n_chunk <= 0 || n_views <= 0 ||
        n_views > 65535 || H <= 0 || W <= 0 || W % 4 != 0 || (int64_t)H * W > (1 << 26) ||
        (int64_t)n_views * H * W > INT32_MAX)
        return GA_ERR_BADARG;
    if (scratch_bytes < ga_chunk_surface_points_scratch_bytes(n_views, H, W)) return GA_ERR_WORKSPACE;
    const int bpv = (H * W + kSpPix - 1) / kSpPix;
    SurfArgs a{alpha, depth, cams, views, n_chunk, H, W, bpv, alpha_min, min_depth,
               reinterpret_cast<int32_t *>(scratch), count, points};
    cudaStream_t s = (cudaStream_t)stream;
    surf_count_kernel<<<dim3(bpv, n_views), kSpThreads, 0, s>>>(a);
    surf_scan_kernel<<<1, kScanThreads, 0, s>>>(a.block_off, bpv * n_views, count);
    surf_emit_kernel<<<dim3(bpv, n_views), kSpThreads, 0, s>>>(a);
    return (int)cudaGetLastError();
}

extern "C" size_t ga_fps_ex_workspace_bytes(int batch, int N, int K)
{
    if (batch <= 0 || N <= 0 || K <= 0) return 0;
    return align256((size_t)batch * K * sizeof(unsigned long long)) + (size_t)batch * N * sizeof(float);
}

extern "C" int ga_fps_ex(const float *pcd, const int32_t *lengths, int batch, int N, int K, const int32_t *start_idx,
                         int32_t *idx_out, float *xyz_out, void *workspace, size_t workspace_bytes, void *stream)
{
    if (!pcd || !start_idx || !idx_out || !xyz_out || batch <= 0 || N <= 0 || K <= 0) return GA_ERR_BADARG;
    if (N > GA_FPS_EX_MAX_N || K > GA_FPS_EX_MAX_K) return GA_ERR_SIZE;
    // Every cloud has N points and the one-CTA kernel holds them: it is the faster of the two there
    // (profiles/pcd_h100.md), and needs no workspace.
    if (!lengths && N <= GA_FPS_MAX_N && K <= GA_FPS_MAX_K && K <= N)
        return ga_fps(pcd, batch, N, K, start_idx, idx_out, xyz_out, stream);
    if (!workspace) return GA_ERR_BADARG;
    if (workspace_bytes < ga_fps_ex_workspace_bytes(batch, N, K)) return GA_ERR_WORKSPACE;
    const int max_ctas = fps_grid().max_ctas;
    if (batch > max_ctas) return GA_ERR_SIZE;
    // CTAs per cloud: at least 2048 points each where the grid allows it (a wider grid makes each round's
    // grid.sync() dearer than the distance updates it spreads)
    const int want = (int)(((int64_t)N + 4 * kFxThreads - 1) / (4 * kFxThreads));
    const int cpc = max(1, min(want, max_ctas / batch));
    char *ws = static_cast<char *>(workspace);
    FpsArgs a{pcd, lengths, start_idx, batch, N, K, cpc, idx_out, xyz_out,
              reinterpret_cast<unsigned long long *>(ws),
              reinterpret_cast<float *>(ws + align256((size_t)batch * K * sizeof(unsigned long long)))};
    void *args[] = {&a};
    return (int)cudaLaunchCooperativeKernel((const void *)fps_grid_kernel, dim3(batch * cpc), dim3(kFxThreads), args, 0,
                                            (cudaStream_t)stream);
}
