// LPIPS (VGG) backward, input gradients only (the network is frozen).  The 3x3 convolutions' dgrad runs on the wgmma
// implicit GEMM of vae_encoder.cu (flipped weights, ga_conv3x3_mask_bf16 / ga_conv3x3_bf16); this file holds the rest:
//   lpips_tap_backward   : at one tap, the head's gradient plus the 2x2 max pool's routed gradient, through the tap's
//                          ReLU mask, rounded to bf16 once
//   lpips_input_backward : the dgrad of features.0 (64 -> 3 channels) fused with the backward of lpips_pack
// Formulas and roundings are stated in include/ga_b200.h Part 9.  This file is compiled without FMA contraction, like
// lpips_ops.cu, so that the stated roundings hold.
#include "../../include/ga_b200.h"
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace {

__device__ __forceinline__ void unpack8(const uint4 &u, float *f)
{
    const __nv_bfloat162 *h = reinterpret_cast<const __nv_bfloat162 *>(&u);
#pragma unroll
    for (int e = 0; e < 4; e++) {
        const float2 x = __bfloat1622float2(h[e]);
        f[2 * e] = x.x;
        f[2 * e + 1] = x.y;
    }
}

// ---- tap backward.  A group of G = min(32, C / 8) lanes owns one pixel of the differentiated side, lane l holding
// channels 8 (l + G j) .. +7, j < C / (8 G), as in lpips_head_kernel; channel sums are each lane's channels in
// increasing order, then an xor butterfly over the group.  Every thread runs the body, so the full-warp shuffles never
// diverge; a group past the end computes on zeros and stores nothing.
constexpr int kTapThreads = 256;

template <int C>
__global__ void __launch_bounds__(kTapThreads) lpips_tap_backward_kernel(const uint4 *__restrict__ feat, int n, int H,
                                                                         int W, int side,
                                                                         const float *__restrict__ lin_w,
                                                                         const float *__restrict__ g,
                                                                         const float *__restrict__ dpool,
                                                                         uint4 *__restrict__ grad)
{
    constexpr int G = C / 8 < 32 ? C / 8 : 32;
    constexpr int V = C / (8 * G);
    constexpr int C8 = C / 8;
    constexpr int kGroups = kTapThreads / G;
    const int l = threadIdx.x % G;
    const int HW = H * W;
    const int64_t p = (int64_t)blockIdx.x * kGroups + threadIdx.x / G;   // pixel of [n, H, W]
    const bool active = p < (int64_t)n * HW;
    const int i = active ? (int)(p / HW) : 0, hw = active ? (int)(p - (int64_t)i * HW) : 0;
    const size_t self = (size_t)(side * n + i) * HW, other = (size_t)((1 - side) * n + i) * HW;
    float a[8 * V], c[8 * V], w[8 * V];
#pragma unroll
    for (int j = 0; j < V; j++) {
        const uint4 z = make_uint4(0u, 0u, 0u, 0u);
        unpack8(active ? __ldg(feat + (self + hw) * C8 + l + G * j) : z, a + 8 * j);
        unpack8(active ? __ldg(feat + (other + hw) * C8 + l + G * j) : z, c + 8 * j);
#pragma unroll
        for (int e = 0; e < 8; e++) w[8 * j + e] = __ldg(lin_w + 8 * (l + G * j) + e);
    }
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int k = 0; k < 8 * V; k++) { s0 += a[k] * a[k]; s1 += c[k] * c[k]; }
#pragma unroll
    for (int o = G / 2; o; o >>= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    }
    const float r0 = sqrtf(s0), n0 = r0 + 1e-10f, n1 = sqrtf(s1) + 1e-10f;
    float u[8 * V], S = 0.f;
#pragma unroll
    for (int k = 0; k < 8 * V; k++) {
        const float t = a[k] / n0 - c[k] / n1;
        u[k] = 2.f * (w[k] * t);
        S += u[k] * a[k];
    }
#pragma unroll
    for (int o = G / 2; o; o >>= 1) S += __shfl_xor_sync(0xffffffffu, S, o);
    if (!active) return;
    const float s = __ldg(g + i) / (float)HW;
    const float q = (S / n0) / n0;
    const int Ho = H / 2, Wo = W / 2;
    const int y = hw / W, x = hw - y * W;
    const bool pooled = dpool != nullptr && y < 2 * Ho && x < 2 * Wo;
    const int pos = 2 * (y & 1) + (x & 1);
    const size_t w00 = self + (size_t)(y & ~1) * W + (x & ~1);     // the window's top-left pixel
    const float *dp = pooled ? dpool + (((size_t)i * Ho + y / 2) * Wo + x / 2) * C : nullptr;
#pragma unroll
    for (int j = 0; j < V; j++) {
        const int ch = 8 * (l + G * j);
        float win[4][8], d[8];
        if (pooled) {
            unpack8(__ldg(feat + w00 * C8 + l + G * j), win[0]);
            unpack8(__ldg(feat + (w00 + 1) * C8 + l + G * j), win[1]);
            unpack8(__ldg(feat + (w00 + W) * C8 + l + G * j), win[2]);
            unpack8(__ldg(feat + (w00 + W + 1) * C8 + l + G * j), win[3]);
            const float4 d0 = __ldg(reinterpret_cast<const float4 *>(dp + ch));
            const float4 d1 = __ldg(reinterpret_cast<const float4 *>(dp + ch + 4));
            d[0] = d0.x; d[1] = d0.y; d[2] = d0.z; d[3] = d0.w; d[4] = d1.x; d[5] = d1.y; d[6] = d1.z; d[7] = d1.w;
        }
        float v[8];
#pragma unroll
        for (int e = 0; e < 8; e++) {
            const int k = 8 * j + e;
            const float head = r0 > 0.f ? s * (u[k] / n0 - (a[k] / r0) * q) : 0.f;
            float routed = 0.f;
            if (pooled) {
                int arg = 0;                                   // first maximum in row-major order
                float m = win[0][e];
#pragma unroll
                for (int t = 1; t < 4; t++)
                    if (win[t][e] > m) { m = win[t][e]; arg = t; }
                routed = arg == pos ? d[e] : 0.f;
            }
            const float sum = routed + head;
            v[k - 8 * j] = a[k] > 0.f ? sum : 0.f;
        }
        __nv_bfloat162 b0 = __floats2bfloat162_rn(v[0], v[1]), b1 = __floats2bfloat162_rn(v[2], v[3]);
        __nv_bfloat162 b2 = __floats2bfloat162_rn(v[4], v[5]), b3 = __floats2bfloat162_rn(v[6], v[7]);
        grad[((size_t)i * HW + hw) * C8 + l + G * j] =
            make_uint4(*reinterpret_cast<uint32_t *>(&b0), *reinterpret_cast<uint32_t *>(&b1),
                       *reinterpret_cast<uint32_t *>(&b2), *reinterpret_cast<uint32_t *>(&b3));
    }
}

// ---- features.0 dgrad + pack backward: one thread per input pixel, 32 x 8 pixels per block, the flipped weights in
// shared memory.  Sum over the taps in row-major order, and within a tap over the 64 channels in increasing order.
constexpr int kInTx = 32, kInTy = 8;
constexpr int kInC = 64;

__global__ void __launch_bounds__(kInTx * kInTy) lpips_input_backward_kernel(const uint4 *__restrict__ g0, int H, int W,
                                                                            const float *__restrict__ w_flip,
                                                                            const float *__restrict__ scale,
                                                                            int normalize, float *__restrict__ dx)
{
    __shared__ float ws[9 * kInC * 3];
    const int tid = threadIdx.y * kInTx + threadIdx.x;
    for (int t = tid; t < 9 * kInC * 3; t += kInTx * kInTy) ws[t] = __ldg(w_flip + t);
    __syncthreads();
    const int x = blockIdx.x * kInTx + threadIdx.x, y = blockIdx.y * kInTy + threadIdx.y;
    const size_t img = blockIdx.z;
    if (x >= W || y >= H) return;
    float acc[3] = {0.f, 0.f, 0.f};
    for (int tap = 0; tap < 9; tap++) {
        const int iy = y + tap / 3 - 1, ix = x + tap % 3 - 1;
        if (iy < 0 || iy >= H || ix < 0 || ix >= W) continue;
        const uint4 *src = g0 + ((img * H + iy) * W + ix) * (kInC / 8);
        const float *wt = ws + tap * kInC * 3;
#pragma unroll 2
        for (int q8 = 0; q8 < kInC / 8; q8++) {
            float gv[8];
            unpack8(__ldg(src + q8), gv);
#pragma unroll
            for (int e = 0; e < 8; e++) {
                const float *wc = wt + (8 * q8 + e) * 3;
                acc[0] += wc[0] * gv[e];
                acc[1] += wc[1] * gv[e];
                acc[2] += wc[2] * gv[e];
            }
        }
    }
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float v = acc[c] / __ldg(scale + c);
        if (normalize) v = 2.f * v;
        dx[((img * 3 + c) * H + y) * W + x] = v;
    }
}

}  // namespace

extern "C" int ga_lpips_tap_backward(const void *feat, int n, int H, int W, int C, int side, const float *lin_w,
                                     const float *g, const float *dpool, void *grad, void *stream)
{
    if (!feat || !lin_w || !g || !grad || n <= 0 || H <= 0 || W <= 0 || (side != 0 && side != 1)) return GA_ERR_BADARG;
    if (dpool && (H < 2 || W < 2)) return GA_ERR_BADARG;
    if ((reinterpret_cast<uintptr_t>(feat) & 15) || (reinterpret_cast<uintptr_t>(grad) & 15) ||
        (reinterpret_cast<uintptr_t>(dpool) & 15))
        return GA_ERR_BADARG;
    if ((int64_t)2 * n * H * W >= (int64_t)1 << 31 || (int64_t)H * W > (int64_t)1 << 24) return GA_ERR_SIZE;
    const uint4 *f = reinterpret_cast<const uint4 *>(feat);
    uint4 *o = reinterpret_cast<uint4 *>(grad);
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t px = (int64_t)n * H * W;
    auto blocks = [&](int groups) { return (unsigned)((px + groups - 1) / groups); };
    switch (C) {
    case 64: lpips_tap_backward_kernel<64><<<blocks(kTapThreads / 8), kTapThreads, 0, s>>>(f, n, H, W, side, lin_w, g, dpool, o); break;
    case 128: lpips_tap_backward_kernel<128><<<blocks(kTapThreads / 16), kTapThreads, 0, s>>>(f, n, H, W, side, lin_w, g, dpool, o); break;
    case 256: lpips_tap_backward_kernel<256><<<blocks(kTapThreads / 32), kTapThreads, 0, s>>>(f, n, H, W, side, lin_w, g, dpool, o); break;
    case 512: lpips_tap_backward_kernel<512><<<blocks(kTapThreads / 32), kTapThreads, 0, s>>>(f, n, H, W, side, lin_w, g, dpool, o); break;
    default: return GA_ERR_BADARG;
    }
    return (int)cudaGetLastError();
}

extern "C" int ga_lpips_input_backward(const void *g0, int n, int H, int W, const float *w_flip, const float *scale,
                                       int normalize, float *dx, void *stream)
{
    if (!g0 || !w_flip || !scale || !dx || n <= 0 || H <= 0 || W <= 0) return GA_ERR_BADARG;
    if (reinterpret_cast<uintptr_t>(g0) & 15) return GA_ERR_BADARG;
    if (n > 65535) return GA_ERR_SIZE;
    if ((int64_t)n * H * W >= (int64_t)1 << 31) return GA_ERR_SIZE;
    const dim3 grid((W + kInTx - 1) / kInTx, (H + kInTy - 1) / kInTy, n);
    lpips_input_backward_kernel<<<grid, dim3(kInTx, kInTy), 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const uint4 *>(g0), H, W, w_flip, scale, normalize, dx);
    return (int)cudaGetLastError();
}
