// Image-quality metrics: LPIPS (VGG) around the wgmma 3x3 convolution of vae_encoder.cu, and SSIM.
//   lpips_pack   : the two images of N pairs, fp32 NCHW -> one bf16 NHWC batch [2N, H, W, 8], scaled for VGG
//   maxpool2x2   : nn.MaxPool2d(2, 2) on NHWC bf16
//   lpips_head   : one VGG tap -> per-block partial sums of the weighted squared difference of the unit-normalised
//                  features of image i and image i + N
//   lpips_reduce : partials -> per-pair, per-tap spatial means and their sum
//   ssim         : 11x11 Gaussian-window SSIM map, per-block partial sums, then a per-image mean
// Formulas and roundings are stated in include/ga_b200.h Part 8 and restated by oracle/lpips_oracle.py.  This file is
// compiled without FMA contraction so that the stated roundings hold.
#include "../../include/ga_b200.h"
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace {

// ---- input pack: thread per pixel, one 16-byte store of 8 bf16 channels (3 used, 5 zero)
__global__ void lpips_pack_kernel(const float *__restrict__ in0, const float *__restrict__ in1, int n, int HW,
                                  int normalize, const float *__restrict__ shift, const float *__restrict__ scale,
                                  uint4 *__restrict__ out)
{
    const float sh[3] = {__ldg(shift), __ldg(shift + 1), __ldg(shift + 2)};
    const float sc[3] = {__ldg(scale), __ldg(scale + 1), __ldg(scale + 2)};
    const size_t total = (size_t)2 * n * HW;
    for (size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x; p < total; p += (size_t)gridDim.x * blockDim.x) {
        const size_t im = p / HW, hw = p - im * HW;
        const float *src = im < (size_t)n ? in0 + im * 3 * HW : in1 + (im - n) * 3 * HW;
        float v[3];
#pragma unroll
        for (int c = 0; c < 3; c++) {
            float x = __ldg(src + (size_t)c * HW + hw);
            if (normalize) x = 2.f * x - 1.f;
            v[c] = (x - sh[c]) / sc[c];
        }
        __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1]), b = __floats2bfloat162_rn(v[2], 0.f);
        out[p] = make_uint4(*reinterpret_cast<uint32_t *>(&a), *reinterpret_cast<uint32_t *>(&b), 0u, 0u);
    }
}

// ---- 2x2 / 2 max pool, floor: thread per (output pixel, 8 channels)
__global__ void maxpool2x2_kernel(const uint4 *__restrict__ x, int n, int H, int W, int C8, uint4 *__restrict__ out)
{
    const int Ho = H / 2, Wo = W / 2;
    const size_t total = (size_t)n * Ho * Wo * C8;
    for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(t % C8);
        const size_t q = t / C8;
        const int ox = (int)(q % Wo), oy = (int)((q / Wo) % Ho);
        const size_t im = q / ((size_t)Wo * Ho);
        const size_t i00 = ((im * H + 2 * oy) * W + 2 * ox) * C8 + c;
        uint4 v[4] = {__ldg(x + i00), __ldg(x + i00 + C8), __ldg(x + i00 + (size_t)W * C8),
                      __ldg(x + i00 + (size_t)W * C8 + C8)};
        uint32_t r[4];
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const uint32_t *a = reinterpret_cast<const uint32_t *>(&v[0]) + e, *b = reinterpret_cast<const uint32_t *>(&v[1]) + e;
            const uint32_t *cc = reinterpret_cast<const uint32_t *>(&v[2]) + e, *d = reinterpret_cast<const uint32_t *>(&v[3]) + e;
            const __nv_bfloat162 m = __hmax2(__hmax2(*reinterpret_cast<const __nv_bfloat162 *>(a), *reinterpret_cast<const __nv_bfloat162 *>(b)),
                                             __hmax2(*reinterpret_cast<const __nv_bfloat162 *>(cc), *reinterpret_cast<const __nv_bfloat162 *>(d)));
            r[e] = *reinterpret_cast<const uint32_t *>(&m);
        }
        out[t] = make_uint4(r[0], r[1], r[2], r[3]);
    }
}

// ---- LPIPS head.  A group of G = min(32, C / 8) lanes owns one pixel: lane l holds channels 8 (l + G j) .. +7,
// j < C / (8 G).  Sums over channels: each lane's channels in increasing order, then an xor butterfly over the group
// (every lane ends with the same bits).  Block b of pair i covers pixels [b * per, (b + 1) * per), per =
// ceil(HW / GA_LPIPS_HEAD_BLOCKS); the group's pixels p0 + g, p0 + g + groups, ... are added in that order, then the
// groups' sums in group order.  The partition depends on H and W only, so a pair's partials do not depend on n.
constexpr int kHeadThreads = 256;

template <int C>
__global__ void __launch_bounds__(kHeadThreads) lpips_head_kernel(const uint4 *__restrict__ feat, int n, int HW,
                                                                  const float *__restrict__ lin_w,
                                                                  float *__restrict__ partial)
{
    constexpr int G = C / 8 < 32 ? C / 8 : 32;
    constexpr int V = C / (8 * G);
    constexpr int C8 = C / 8;
    constexpr int kGroups = kHeadThreads / G;
    __shared__ float gsum[kGroups];
    const int pair = blockIdx.y, b = blockIdx.x;
    const int l = threadIdx.x % G, g = threadIdx.x / G;
    const int per = (HW + GA_LPIPS_HEAD_BLOCKS - 1) / GA_LPIPS_HEAD_BLOCKS;
    const int p0 = b * per, p1 = min(HW, p0 + per);
    float w[8 * V];
#pragma unroll
    for (int j = 0; j < V; j++)
#pragma unroll
        for (int e = 0; e < 8; e++) w[8 * j + e] = __ldg(lin_w + 8 * (l + G * j) + e);
    const uint4 *f0 = feat + (size_t)pair * HW * C8, *f1 = feat + (size_t)(pair + n) * HW * C8;
    float acc = 0.f;
    // every thread runs the same number of rounds, so the full-warp shuffles below never diverge; a group past p1
    // computes on zeros and adds nothing
    for (int pb = p0; pb < p1; pb += kGroups) {
        const int p = pb + g;
        const bool active = p < p1;
        float a[8 * V], c[8 * V];
#pragma unroll
        for (int j = 0; j < V; j++) {
            const uint4 z = make_uint4(0u, 0u, 0u, 0u);
            const uint4 u = active ? __ldg(f0 + (size_t)p * C8 + l + G * j) : z;
            const uint4 v = active ? __ldg(f1 + (size_t)p * C8 + l + G * j) : z;
            const __nv_bfloat162 *ua = reinterpret_cast<const __nv_bfloat162 *>(&u);
            const __nv_bfloat162 *va = reinterpret_cast<const __nv_bfloat162 *>(&v);
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const float2 x = __bfloat1622float2(ua[e]), y = __bfloat1622float2(va[e]);
                a[8 * j + 2 * e] = x.x; a[8 * j + 2 * e + 1] = x.y;
                c[8 * j + 2 * e] = y.x; c[8 * j + 2 * e + 1] = y.y;
            }
        }
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int k = 0; k < 8 * V; k++) { s0 += a[k] * a[k]; s1 += c[k] * c[k]; }
#pragma unroll
        for (int o = G / 2; o; o >>= 1) {
            s0 += __shfl_xor_sync(0xffffffffu, s0, o);
            s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        }
        const float n0 = sqrtf(s0) + 1e-10f, n1 = sqrtf(s1) + 1e-10f;
        float d = 0.f;
#pragma unroll
        for (int k = 0; k < 8 * V; k++) {
            const float t = a[k] / n0 - c[k] / n1;
            d += w[k] * (t * t);
        }
#pragma unroll
        for (int o = G / 2; o; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        if (active) acc += d;
    }
    if (l == 0) gsum[g] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int i = 0; i < kGroups; i++) s += gsum[i];
        partial[(size_t)pair * GA_LPIPS_HEAD_BLOCKS + b] = s;
    }
}

// ---- final LPIPS reduction: block per pair; thread k < 5 folds tap k's partials in block order in fp64
__global__ void lpips_reduce_kernel(const float *__restrict__ partial, int n, int H, int W, float *__restrict__ out)
{
    __shared__ float mean[GA_LPIPS_TAPS];
    const int pair = blockIdx.x, k = threadIdx.x;
    if (k < GA_LPIPS_TAPS) {
        const float *p = partial + ((size_t)k * n + pair) * GA_LPIPS_HEAD_BLOCKS;
        double s = 0.0;
        for (int b = 0; b < GA_LPIPS_HEAD_BLOCKS; b++) s += (double)p[b];
        mean[k] = (float)(s / ((double)(H >> k) * (double)(W >> k)));
        out[(size_t)pair * (GA_LPIPS_TAPS + 1) + k] = mean[k];
    }
    __syncthreads();
    if (k == 0) {
        float v = mean[0];
        for (int i = 1; i < GA_LPIPS_TAPS; i++) v += mean[i];
        out[(size_t)pair * (GA_LPIPS_TAPS + 1) + GA_LPIPS_TAPS] = v;
    }
}

// ---- SSIM: block of 16 x 16 output pixels of one (image, channel) plane; the 26 x 26 input tiles of both images
// in shared memory, zero outside the image.  Each window sum runs over the taps in row-major order, in fp64: in fp32,
// E[x^2] - mu^2 cancels to SSIM errors of ~2e-5.
constexpr int kSsimTile = 16, kSsimWin = GA_SSIM_WINDOW, kSsimHalo = kSsimTile + kSsimWin - 1;

__global__ void __launch_bounds__(kSsimTile * kSsimTile) ssim_kernel(const float *__restrict__ img1,
                                                                     const float *__restrict__ img2, int H, int W,
                                                                     const float *__restrict__ window,
                                                                     float *__restrict__ partial)
{
    __shared__ float sx[kSsimHalo][kSsimHalo], sy[kSsimHalo][kSsimHalo];
    __shared__ float win[kSsimWin * kSsimWin];
    __shared__ float wsum[kSsimTile * kSsimTile / 32];
    const int tid = threadIdx.y * kSsimTile + threadIdx.x;
    const size_t plane = blockIdx.z;
    const float *x = img1 + plane * H * W, *y = img2 + plane * H * W;
    const int ox0 = blockIdx.x * kSsimTile, oy0 = blockIdx.y * kSsimTile, r = kSsimWin / 2;
    for (int i = tid; i < kSsimWin * kSsimWin; i += kSsimTile * kSsimTile) win[i] = __ldg(window + i);
    for (int i = tid; i < kSsimHalo * kSsimHalo; i += kSsimTile * kSsimTile) {
        const int ty = i / kSsimHalo, tx = i - ty * kSsimHalo;
        const int iy = oy0 + ty - r, ix = ox0 + tx - r;
        const bool in = iy >= 0 && iy < H && ix >= 0 && ix < W;
        sx[ty][tx] = in ? __ldg(x + (size_t)iy * W + ix) : 0.f;
        sy[ty][tx] = in ? __ldg(y + (size_t)iy * W + ix) : 0.f;
    }
    __syncthreads();
    const int oy = oy0 + threadIdx.y, ox = ox0 + threadIdx.x;
    float v = 0.f;
    if (oy < H && ox < W) {
        double mu1 = 0.0, mu2 = 0.0, e11 = 0.0, e22 = 0.0, e12 = 0.0;
        for (int ky = 0; ky < kSsimWin; ky++) {
#pragma unroll
            for (int kx = 0; kx < kSsimWin; kx++) {
                const double w = win[ky * kSsimWin + kx];
                const double a = sx[threadIdx.y + ky][threadIdx.x + kx], b = sy[threadIdx.y + ky][threadIdx.x + kx];
                mu1 = fma(w, a, mu1);
                mu2 = fma(w, b, mu2);
                e11 = fma(w, a * a, e11);               // products of two fp32 values are exact in fp64
                e22 = fma(w, b * b, e22);
                e12 = fma(w, a * b, e12);
            }
        }
        const double C1 = 0.01 * 0.01, C2 = 0.03 * 0.03;
        const double mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu1_mu2 = mu1 * mu2;
        const double s1 = e11 - mu1_sq, s2 = e22 - mu2_sq, s12 = e12 - mu1_mu2;
        v = (float)(((2.0 * mu1_mu2 + C1) * (2.0 * s12 + C2)) / ((mu1_sq + mu2_sq + C1) * (s1 + s2 + C2)));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((tid & 31) == 0) wsum[tid >> 5] = v;
    __syncthreads();
    if (tid == 0) {
        float s = 0.f;
        for (int i = 0; i < kSsimTile * kSsimTile / 32; i++) s += wsum[i];
        partial[(plane * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = s;
    }
}

// ---- per-image SSIM mean: one warp per image folds its 3 planes' partials in fp64 (lane-strided, then a butterfly)
__global__ void ssim_reduce_kernel(const float *__restrict__ partial, int per_image, int H, int W, float *__restrict__ out)
{
    const float *p = partial + (size_t)blockIdx.x * per_image;
    double s = 0.0;
    for (int i = threadIdx.x; i < per_image; i += 32) s += (double)p[i];
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) out[blockIdx.x] = (float)(s / (3.0 * H * W));
}

unsigned grid_for(size_t work, int threads)
{
    const size_t b = (work + threads - 1) / threads;
    return (unsigned)(b < 8192 ? (b ? b : 1) : 8192);
}

}  // namespace

extern "C" int ga_lpips_pack(const float *in0, const float *in1, int n, int H, int W, int normalize, const float *shift,
                             const float *scale, void *out, void *stream)
{
    if (!in0 || !in1 || !shift || !scale || !out || n <= 0 || H <= 0 || W <= 0) return GA_ERR_BADARG;
    if (reinterpret_cast<uintptr_t>(out) & 15) return GA_ERR_BADARG;
    if ((int64_t)2 * n * H * W >= (int64_t)1 << 31) return GA_ERR_SIZE;
    const int HW = H * W;
    lpips_pack_kernel<<<grid_for((size_t)2 * n * HW, 256), 256, 0, (cudaStream_t)stream>>>(
        in0, in1, n, HW, normalize, shift, scale, reinterpret_cast<uint4 *>(out));
    return (int)cudaGetLastError();
}

extern "C" int ga_maxpool2x2_bf16(const void *x, int n, int H, int W, int C, void *out, void *stream)
{
    if (!x || !out || n <= 0 || H < 2 || W < 2 || C <= 0 || C % 8) return GA_ERR_BADARG;
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(out) & 15)) return GA_ERR_BADARG;
    if ((int64_t)n * H * W >= (int64_t)1 << 31) return GA_ERR_SIZE;
    const size_t work = (size_t)n * (H / 2) * (W / 2) * (C / 8);
    maxpool2x2_kernel<<<grid_for(work, 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const uint4 *>(x), n, H, W, C / 8, reinterpret_cast<uint4 *>(out));
    return (int)cudaGetLastError();
}

extern "C" int ga_lpips_head(const void *feat, int n, int H, int W, int C, const float *lin_w, float *partial,
                             void *stream)
{
    if (!feat || !lin_w || !partial || n <= 0 || n > 65535 || H <= 0 || W <= 0) return GA_ERR_BADARG;
    if (reinterpret_cast<uintptr_t>(feat) & 15) return GA_ERR_BADARG;
    if ((int64_t)2 * n * H * W >= (int64_t)1 << 31) return GA_ERR_SIZE;
    const dim3 grid(GA_LPIPS_HEAD_BLOCKS, n);
    const uint4 *f = reinterpret_cast<const uint4 *>(feat);
    cudaStream_t s = (cudaStream_t)stream;
    const int HW = H * W;
    switch (C) {
    case 64: lpips_head_kernel<64><<<grid, kHeadThreads, 0, s>>>(f, n, HW, lin_w, partial); break;
    case 128: lpips_head_kernel<128><<<grid, kHeadThreads, 0, s>>>(f, n, HW, lin_w, partial); break;
    case 256: lpips_head_kernel<256><<<grid, kHeadThreads, 0, s>>>(f, n, HW, lin_w, partial); break;
    case 512: lpips_head_kernel<512><<<grid, kHeadThreads, 0, s>>>(f, n, HW, lin_w, partial); break;
    default: return GA_ERR_BADARG;
    }
    return (int)cudaGetLastError();
}

extern "C" int ga_lpips_reduce(const float *partial, int n, int H, int W, float *out, void *stream)
{
    if (!partial || !out || n <= 0 || (H >> (GA_LPIPS_TAPS - 1)) < 1 || (W >> (GA_LPIPS_TAPS - 1)) < 1)
        return GA_ERR_BADARG;
    lpips_reduce_kernel<<<n, 32, 0, (cudaStream_t)stream>>>(partial, n, H, W, out);
    return (int)cudaGetLastError();
}

extern "C" size_t ga_ssim_scratch_bytes(int n, int H, int W)
{
    if (n <= 0 || H <= 0 || W <= 0) return 0;
    return (size_t)n * 3 * ((H + kSsimTile - 1) / kSsimTile) * ((W + kSsimTile - 1) / kSsimTile) * sizeof(float);
}

extern "C" int ga_ssim(const float *img1, const float *img2, int n, int H, int W, const float *window, void *scratch,
                       size_t scratch_bytes, float *out, void *stream)
{
    if (!img1 || !img2 || !window || !scratch || !out || n <= 0 || H <= 0 || W <= 0) return GA_ERR_BADARG;
    if (n > 65535 / 3) return GA_ERR_SIZE;
    if ((int64_t)H * W >= (int64_t)1 << 31) return GA_ERR_SIZE;
    if (scratch_bytes < ga_ssim_scratch_bytes(n, H, W)) return GA_ERR_WORKSPACE;
    const int gx = (W + kSsimTile - 1) / kSsimTile, gy = (H + kSsimTile - 1) / kSsimTile;
    cudaStream_t s = (cudaStream_t)stream;
    float *part = reinterpret_cast<float *>(scratch);
    ssim_kernel<<<dim3(gx, gy, 3 * n), dim3(kSsimTile, kSsimTile), 0, s>>>(img1, img2, H, W, window, part);
    ssim_reduce_kernel<<<n, 32, 0, s>>>(part, 3 * gx * gy, H, W, out);
    return (int)cudaGetLastError();
}
