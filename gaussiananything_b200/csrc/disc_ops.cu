// PatchGAN discriminator (the reference's nsr/losses/disc.py NLayerDiscriminator at input_nc 3, ndf 64, n_layers 3):
// forward with training-mode BatchNorm, and the input and weight gradients.  The 4x4 convolutions and their dgrad run
// on the implicit GEMM of conv_igemm.cuh; this file holds the entry points and the rest:
//   disc_conv5 / disc_conv5_backward : the 512 -> 1 convolution as a dot product, and its dgrad fused with the
//                                      LeakyReLU mask, BatchNorm partials and its weight gradient
//   bn_* kernels                     : BatchNorm finalize / apply, forward and backward
//   wgrad_kernel                     : weight gradients of the 4x4 convolutions, split over pixels (mma.sync)
//   input_backward_kernel            : conv 1's dgrad to the fp32 NCHW image
//   colsum kernels                   : fixed-order column sums (bias gradients, partial reductions)
// Formulas and roundings are stated in include/ga_b200.h Part 11.  Compiled without FMA contraction.
#include "conv_igemm.cuh"
#include <cuda_bf16.h>
#include <math.h>

namespace {

constexpr float kSlope = 0.2f;
constexpr int kC5 = 512;                    // conv 5's input channels

// ---- conv 5 forward: one warp per output pixel, lane l holding channels 8 l .. 8 l + 7 and 256 + 8 l .. + 7
__global__ void __launch_bounds__(256) disc_conv5_kernel(const __nv_bfloat16 *__restrict__ x, int n, int H, int W,
                                                         const float *__restrict__ w5, const float *__restrict__ bias,
                                                         float *__restrict__ out)
{
    __shared__ float ws[16 * kC5];
    for (int t = threadIdx.x; t < 16 * kC5; t += blockDim.x) ws[t] = __ldg(w5 + t);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int Ho = H - 1, Wo = W - 1;
    const int64_t total = (int64_t)n * Ho * Wo;
    for (int64_t o = (int64_t)blockIdx.x * 8 + warp; o < total; o += (int64_t)gridDim.x * 8) {
        const int img = (int)(o / (Ho * Wo)), r = (int)(o - (int64_t)img * Ho * Wo);
        const int oy = r / Wo, ox = r - oy * Wo;
        float acc = 0.f;
        for (int tap = 0; tap < 16; tap++) {
            const int iy = oy - 1 + tap / 4, ix = ox - 1 + (tap & 3);
            if (iy < 0 || iy >= H || ix < 0 || ix >= W) continue;
            const uint4 *src = reinterpret_cast<const uint4 *>(x + (((size_t)img * H + iy) * W + ix) * kC5);
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const uint4 u = __ldg(src + lane + 32 * j);
                const __nv_bfloat162 *h = reinterpret_cast<const __nv_bfloat162 *>(&u);
                const float *wt = ws + tap * kC5 + 8 * lane + 256 * j;
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const float2 f = __bfloat1622float2(h[e]);
                    acc = acc + f.x * wt[2 * e];
                    acc = acc + f.y * wt[2 * e + 1];
                }
            }
        }
#pragma unroll
        for (int s = 16; s; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
        if (lane == 0) out[o] = acc + __ldg(bias);
    }
}

// ---- conv 5 backward: block b owns input pixels [256 b, 256 b + 256) of [n, H, W], thread t channels 2t, 2t + 1
constexpr int kC5Pix = 256;

__global__ void __launch_bounds__(256) disc_conv5_backward_kernel(
    const float *__restrict__ g5, int n, int H, int W, const float *__restrict__ w5, const __nv_bfloat16 *__restrict__ a4,
    const float *__restrict__ z4, const float *__restrict__ mean4, const float *__restrict__ rstd4,
    float *__restrict__ gy4, float2 *__restrict__ bn_part, float *__restrict__ dw_part)
{
    const int c = 2 * threadIdx.x;
    const int Ho = H - 1, Wo = W - 1;
    const int64_t P = (int64_t)n * H * W;
    const int64_t p0 = (int64_t)blockIdx.x * kC5Pix, p1 = min(P, p0 + kC5Pix);
    float w[16][2], dw[16][2];
#pragma unroll
    for (int t = 0; t < 16; t++) {
        w[t][0] = __ldg(w5 + t * kC5 + c); w[t][1] = __ldg(w5 + t * kC5 + c + 1);
        dw[t][0] = dw[t][1] = 0.f;
    }
    const float mu0 = __ldg(mean4 + c), mu1 = __ldg(mean4 + c + 1), rs0 = __ldg(rstd4 + c), rs1 = __ldg(rstd4 + c + 1);
    float s0 = 0.f, s1 = 0.f, t0 = 0.f, t1 = 0.f;
    for (int64_t p = p0; p < p1; p++) {
        const int img = (int)(p / (H * W)), r = (int)(p - (int64_t)img * H * W);
        const int y = r / W, x = r - y * W;
        const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(a4 + p * kC5 + c));
        float ga0 = 0.f, ga1 = 0.f;
#pragma unroll
        for (int t = 0; t < 16; t++) {
            const int oy = y + 1 - t / 4, ox = x + 1 - (t & 3);
            if (oy < 0 || oy >= Ho || ox < 0 || ox >= Wo) continue;
            const float g = __ldg(g5 + ((size_t)img * Ho + oy) * Wo + ox);
            ga0 = ga0 + g * w[t][0];
            ga1 = ga1 + g * w[t][1];
            if (dw_part) {
                dw[t][0] = dw[t][0] + g * a.x;
                dw[t][1] = dw[t][1] + g * a.y;
            }
        }
        const float g0 = a.x > 0.f ? ga0 : kSlope * ga0, g1 = a.y > 0.f ? ga1 : kSlope * ga1;
        *reinterpret_cast<float2 *>(gy4 + p * kC5 + c) = make_float2(g0, g1);
        const float2 zz = *reinterpret_cast<const float2 *>(z4 + p * kC5 + c);
        s0 = s0 + g0; s1 = s1 + g1;
        t0 = t0 + g0 * ((zz.x - mu0) * rs0);
        t1 = t1 + g1 * ((zz.y - mu1) * rs1);
    }
    bn_part[(size_t)blockIdx.x * kC5 + c] = make_float2(s0, t0);
    bn_part[(size_t)blockIdx.x * kC5 + c + 1] = make_float2(s1, t1);
    if (!dw_part) return;
#pragma unroll
    for (int t = 0; t < 16; t++)
        *reinterpret_cast<float2 *>(dw_part + (size_t)blockIdx.x * 16 * kC5 + t * kC5 + c) = make_float2(dw[t][0], dw[t][1]);
}

// ---- fixed-order column sums.  Stage 1: block b owns rows [kColRows b, kColRows (b + 1)); its 256 threads are
// 256 / C row lanes x C columns, lane l adding rows l, l + 256 / C, ... in order (fp32), then the lanes in order.
// Stage 2: out[c] = fp32(sum over rows of part in order, fp64), one thread per column.
constexpr int kColRows = 1024;

template <typename T>
__global__ void __launch_bounds__(256) colsum_partial_kernel(const T *__restrict__ x, int64_t rows, int C,
                                                             float *__restrict__ part)
{
    __shared__ float red[256];
    const int lanes = 256 / C, c = threadIdx.x % C, l = threadIdx.x / C;
    const int64_t r0 = (int64_t)blockIdx.x * kColRows, r1 = min(rows, r0 + kColRows);
    float s = 0.f;
    if (l < lanes)
        for (int64_t r = r0 + l; r < r1; r += lanes) s = s + (float)x[r * C + c];
    red[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x < C) {
        float t = 0.f;
        for (int k = 0; k < lanes; k++) t = t + red[k * C + threadIdx.x];
        part[(size_t)blockIdx.x * C + threadIdx.x] = t;
    }
}

__global__ void reduce_rows_kernel(const float *__restrict__ part, int rows, int C, float *__restrict__ out)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double s = 0.0;
    for (int r = 0; r < rows; r++) s += (double)part[(size_t)r * C + c];
    out[c] = (float)s;
}

// ---- BatchNorm.  Forward finalize, one CTA of kFinThreads per channel: thread t merges the per-CTA (mean, M2)
// partials t, t + kFinThreads, ... in that order with Chan's rule in fp64, then the threads' states are merged by a
// fixed tree (t with t + s for s = kFinThreads / 2, ..., 1).
constexpr int kFinThreads = 128;

__device__ __forceinline__ void chan_merge(double &na, double &ma, double &m2a, double nb, double mb, double m2b)
{
    const double nn = na + nb;
    if (nn == 0.0) return;
    const double d = mb - ma;
    ma += d * (nb / nn);
    m2a += m2b + d * d * (na * nb / nn);
    na = nn;
}

__global__ void __launch_bounds__(kFinThreads) bn_finalize_kernel(const float2 *__restrict__ part, int nb, int64_t M,
                                                                  int C, int training, float momentum, float eps,
                                                                  float *__restrict__ running_mean,
                                                                  float *__restrict__ running_var,
                                                                  float *__restrict__ mean_out,
                                                                  float *__restrict__ rstd_out)
{
    __shared__ double sn[kFinThreads], sm[kFinThreads], s2[kFinThreads];
    const int c = blockIdx.x, t = threadIdx.x;
    if (!training) {
        if (t == 0) {
            mean_out[c] = running_mean[c];
            rstd_out[c] = (float)(1.0 / sqrt((double)running_var[c] + (double)eps));
        }
        return;
    }
    double na = 0.0, mean = 0.0, m2 = 0.0;
    for (int b = t; b < nb; b += kFinThreads) {
        const float2 q = part[(size_t)b * C + c];
        chan_merge(na, mean, m2, (double)min((int64_t)CBM, M - (int64_t)b * CBM), (double)q.x, (double)q.y);
    }
    sn[t] = na; sm[t] = mean; s2[t] = m2;
    __syncthreads();
    for (int h = kFinThreads / 2; h; h >>= 1) {
        if (t < h) {
            na = sn[t]; mean = sm[t]; m2 = s2[t];
            chan_merge(na, mean, m2, sn[t + h], sm[t + h], s2[t + h]);
            sn[t] = na; sm[t] = mean; s2[t] = m2;
        }
        __syncthreads();
    }
    if (t) return;
    mean = sm[0]; m2 = s2[0];
    const double var = m2 / (double)M;
    mean_out[c] = (float)mean;
    rstd_out[c] = (float)(1.0 / sqrt(var + (double)eps));
    running_mean[c] = (float)((1.0 - momentum) * (double)running_mean[c] + (double)momentum * mean);
    running_var[c] = (float)((1.0 - momentum) * (double)running_var[c] + (double)momentum * (m2 / (double)(M - 1)));
}

// a = bf16(lrelu(((z - mean) * rstd) * gamma + beta))
__global__ void bn_apply_kernel(const float *__restrict__ z, int64_t M, int C, const float *__restrict__ mean,
                                const float *__restrict__ rstd, const float *__restrict__ gamma,
                                const float *__restrict__ beta, __nv_bfloat16 *__restrict__ a)
{
    const int64_t total = M * C / 2;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)((2 * i) % C);
        const float2 v = reinterpret_cast<const float2 *>(z)[i];
        float y0 = ((v.x - __ldg(mean + c)) * __ldg(rstd + c)) * __ldg(gamma + c) + __ldg(beta + c);
        float y1 = ((v.y - __ldg(mean + c + 1)) * __ldg(rstd + c + 1)) * __ldg(gamma + c + 1) + __ldg(beta + c + 1);
        y0 = y0 > 0.f ? y0 : kSlope * y0;
        y1 = y1 > 0.f ? y1 : kSlope * y1;
        reinterpret_cast<__nv_bfloat162 *>(a)[i] = __floats2bfloat162_rn(y0, y1);
    }
}

// Backward finalize, one CTA per channel: S = sum g, T = sum g xhat over the partials, thread t adding partials
// t, t + kFinThreads, ... in order (fp64), then a fixed tree; dbeta = S, dgamma = T, k = (S / M, T / M)
__global__ void __launch_bounds__(kFinThreads) bn_grad_finalize_kernel(const float2 *__restrict__ part, int nb,
                                                                       int64_t M, int C, int training,
                                                                       float *__restrict__ dgamma,
                                                                       float *__restrict__ dbeta,
                                                                       float2 *__restrict__ k)
{
    __shared__ double ss[kFinThreads], st[kFinThreads];
    const int c = blockIdx.x, t = threadIdx.x;
    double s = 0.0, u = 0.0;
    for (int b = t; b < nb; b += kFinThreads) {
        const float2 q = part[(size_t)b * C + c];
        s += (double)q.x; u += (double)q.y;
    }
    ss[t] = s; st[t] = u;
    __syncthreads();
    for (int h = kFinThreads / 2; h; h >>= 1) {
        if (t < h) { ss[t] += ss[t + h]; st[t] += st[t + h]; }
        __syncthreads();
    }
    if (t) return;
    s = ss[0]; u = st[0];
    if (dbeta) dbeta[c] = (float)s;
    if (dgamma) dgamma[c] = (float)u;
    k[c] = training ? make_float2((float)(s / (double)M), (float)(u / (double)M)) : make_float2(0.f, 0.f);
}

// dz = bf16((gamma * rstd) * ((g - k.x) - xhat * k.y)), xhat = (z - mean) * rstd
__global__ void bn_grad_apply_kernel(const float *__restrict__ g, const float *__restrict__ z, int64_t M, int C,
                                     const float *__restrict__ mean, const float *__restrict__ rstd,
                                     const float *__restrict__ gamma, const float2 *__restrict__ k,
                                     __nv_bfloat16 *__restrict__ dz)
{
    const int64_t total = M * C / 2;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)((2 * i) % C);
        const float2 gv = reinterpret_cast<const float2 *>(g)[i], zv = reinterpret_cast<const float2 *>(z)[i];
        float out[2];
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const float rs = __ldg(rstd + c + e);
            const float xh = ((e ? zv.y : zv.x) - __ldg(mean + c + e)) * rs;
            const float2 kk = k[c + e];
            out[e] = (__ldg(gamma + c + e) * rs) * (((e ? gv.y : gv.x) - kk.x) - xh * kk.y);
        }
        reinterpret_cast<__nv_bfloat162 *>(dz)[i] = __floats2bfloat162_rn(out[0], out[1]);
    }
}

// ---- conv 1's dgrad to the image: one thread per input pixel; w1s[tap][co][c] fp32 in shared memory
__global__ void __launch_bounds__(256) disc_input_backward_kernel(const __nv_bfloat16 *__restrict__ g1, int n, int H,
                                                                  int W, const float *__restrict__ w1,
                                                                  float *__restrict__ dx)
{
    __shared__ float ws[16 * 64 * 3];
    for (int t = threadIdx.x; t < 16 * 64 * 3; t += blockDim.x) ws[t] = __ldg(w1 + t);
    __syncthreads();
    const int Ho = (H - 2) / 2 + 1, Wo = (W - 2) / 2 + 1;
    const int64_t total = (int64_t)n * H * W;
    for (int64_t p = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
        const int img = (int)(p / (H * W)), r = (int)(p - (int64_t)img * H * W);
        const int y = r / W, x = r - y * W;
        float acc[3] = {0.f, 0.f, 0.f};
        for (int tap = 0; tap < 16; tap++) {
            const int ky = tap / 4, kx = tap & 3;
            const int ty = y + 1 - ky, tx = x + 1 - kx;
            if (ty < 0 || tx < 0 || (ty & 1) || (tx & 1)) continue;
            const int oy = ty / 2, ox = tx / 2;
            if (oy >= Ho || ox >= Wo) continue;
            const uint4 *src = reinterpret_cast<const uint4 *>(g1 + (((size_t)img * Ho + oy) * Wo + ox) * 64);
            const float *wt = ws + tap * 64 * 3;
            for (int q8 = 0; q8 < 8; q8++) {
                const uint4 u = __ldg(src + q8);
                const __nv_bfloat162 *h = reinterpret_cast<const __nv_bfloat162 *>(&u);
#pragma unroll
                for (int e = 0; e < 8; e++) {
                    const float2 f2 = __bfloat1622float2(h[e / 2]);
                    const float gv = (e & 1) ? f2.y : f2.x;
                    const float *wc = wt + (8 * q8 + e) * 3;
                    acc[0] = acc[0] + wc[0] * gv;
                    acc[1] = acc[1] + wc[1] * gv;
                    acc[2] = acc[2] + wc[2] * gv;
                }
            }
        }
#pragma unroll
        for (int c = 0; c < 3; c++) dx[(((size_t)img * 3 + c) * H + y) * W + x] = acc[c];
    }
}

// ---- weight gradient of a 4x4 pad-1 convolution: D[co, (ky * 4 + kx) * Cin + ci] = sum_p dy[p, co] x[p + tap, ci]
// over the output pixels p.  CTA tile 128 co x 128 columns, K-blocks of 32 pixels; both operands are staged with
// cp.async in their natural (MN-contiguous) layout, rows padded to 136 elements, and read transposed by
// ldmatrix.trans into mma.sync m16n8k16 fragments.  Warp w: co rows 64 (w / 4), columns 32 (w % 4).  Split over
// pixels: blockIdx.z owns pixels [z chunk, (z + 1) chunk) and writes its fp32 tile to part[z].
constexpr int kWgBM = 128, kWgBN = 128, kWgBK = 32, kWgStages = 4, kWgPitch = 136;
constexpr int kWgStageElems = 2 * kWgBK * kWgPitch;
constexpr int kWgSmem = kWgStages * kWgStageElems * 2;

struct WgradArgs {
    const __nv_bfloat16 *dy, *x;
    int n, H, W, Cin, Ho, Wo, Co, stride, P, chunk, ncols;
    float *part;
};

__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t &r0, uint32_t &r1, uint32_t &r2, uint32_t &r3)
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];\n"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}

__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(256) wgrad_kernel(const WgradArgs a)
{
    extern __shared__ __align__(16) __nv_bfloat16 wsm[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp >> 2, wn = warp & 3;
    const int co0 = blockIdx.y * kWgBM, col0 = blockIdx.x * kWgBN;
    const int pz0 = blockIdx.z * a.chunk, pz1 = min(a.P, pz0 + a.chunk);
    const int nk = (pz1 - pz0 + kWgBK - 1) / kWgBK;
    const int hw = a.Ho * a.Wo;

    auto load = [&](int kb) {
        if (kb < nk) {
            __nv_bfloat16 *As = wsm + (kb % kWgStages) * kWgStageElems, *Bs = As + kWgBK * kWgPitch;
#pragma unroll
            for (int i = 0; i < 2; i++) {
                const int idx = tid + 256 * i, row = idx >> 4, ch = idx & 15;
                const int p = pz0 + kb * kWgBK + row;
                const bool pin = p < pz1;
                // A: dy[p, co0 + 8 ch ..]
                const int co = co0 + 8 * ch;
                const bool va = pin && co < a.Co;
                cp_async16(smem_u32(As + row * kWgPitch + 8 * ch), va ? a.dy + (size_t)p * a.Co + co : a.dy, va);
                // B: x at pixel p's tap, channels ci .. ci + 7 of column col0 + 8 ch
                const int col = col0 + 8 * ch, tap = col / a.Cin, ci = col - tap * a.Cin;
                bool vb = false;
                const __nv_bfloat16 *src = a.x;
                if (pin) {
                    const int img = p / hw, r = p - img * hw, oy = r / a.Wo, ox = r - oy * a.Wo;
                    const int iy = a.stride * oy - 1 + (tap >> 2), ix = a.stride * ox - 1 + (tap & 3);
                    vb = iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
                    if (vb) src = a.x + (((size_t)img * a.H + iy) * a.W + ix) * a.Cin + ci;
                }
                cp_async16(smem_u32(Bs + row * kWgPitch + 8 * ch), src, vb);
            }
        }
        cp_async_commit();
    };

    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int e = 0; e < 4; e++) acc[i][j][e] = 0.f;

    for (int s = 0; s < kWgStages - 1; s++) load(s);
    const int mat = lane >> 3, rr = lane & 7;
    for (int kb = 0; kb < nk; kb++) {
        cp_async_wait<kWgStages - 2>();
        __syncthreads();
        load(kb + kWgStages - 1);
        const __nv_bfloat16 *As = wsm + (kb % kWgStages) * kWgStageElems, *Bs = As + kWgBK * kWgPitch;
#pragma unroll
        for (int ks = 0; ks < kWgBK / 16; ks++) {
            uint32_t af[4][4], bf[4][2];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int k = ks * 16 + (mat >> 1) * 8 + rr, m = wm * 64 + i * 16 + (mat & 1) * 8;
                ldsm_x4_t(smem_u32(As + k * kWgPitch + m), af[i][0], af[i][1], af[i][2], af[i][3]);
            }
#pragma unroll
            for (int j = 0; j < 4; j += 2) {
                const int k = ks * 16 + (mat & 1) * 8 + rr, c = wn * 32 + j * 8 + (mat >> 1) * 8;
                ldsm_x4_t(smem_u32(Bs + k * kWgPitch + c), bf[j][0], bf[j][1], bf[j + 1][0], bf[j + 1][1]);
            }
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) mma_bf16_16816(acc[i][j], af[i], bf[j][0], bf[j][1]);
        }
    }
    cp_async_wait<0>();

    const int g = lane >> 2, cq = lane & 3;
    float *out = a.part + (size_t)blockIdx.z * a.Co * a.ncols;
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
            const int co = co0 + wm * 64 + i * 16 + g + 8 * hf;
            if (co >= a.Co) continue;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int col = col0 + wn * 32 + j * 8 + 2 * cq;
                *reinterpret_cast<float2 *>(out + (size_t)co * a.ncols + col) =
                    make_float2(acc[i][j][2 * hf], acc[i][j][2 * hf + 1]);
            }
        }
}

// dw[co, ci, ky, kx] = fp32(sum over splits in order, fp64) of part[s, co, (ky * 4 + kx) * Cin + ci], ci < cin_out
__global__ void wgrad_reduce_kernel(const float *__restrict__ part, int splits, int Co, int Cin, int cin_out,
                                    float *__restrict__ dw)
{
    const int64_t total = (int64_t)Co * cin_out * 16;
    const int64_t plane = (int64_t)Co * 16 * Cin;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int tap = (int)(i % 16), ci = (int)((i / 16) % cin_out), co = (int)(i / (16 * cin_out));
        const size_t col = (size_t)co * 16 * Cin + (size_t)tap * Cin + ci;
        double s = 0.0;
        for (int z = 0; z < splits; z++) s += (double)part[z * plane + col];
        dw[i] = (float)s;
    }
}

int wgrad_splits(int P, int Co, int Cin)
{
    const int tiles = ((Co + kWgBM - 1) / kWgBM) * (16 * Cin / kWgBN);
    int s = (2 * 132 + tiles - 1) / tiles;
    const int most = (P + 255) / 256;
    if (s > most) s = most;
    return s < 1 ? 1 : s;
}

inline unsigned grid_for(int64_t work, int per_block)
{
    int64_t b = (work + per_block - 1) / per_block;
    return (unsigned)(b < 1 ? 1 : (b > 65535 * 4 ? 65535 * 4 : b));
}

}  // namespace

// ---- entry points --------------------------------------------------------------------------------------------------
extern "C" int ga_conv4x4_out_size(int H, int stride)
{
    if (H <= 0 || (stride != 1 && stride != 2)) return GA_ERR_BADARG;
    const int o = (H - 2) / stride + 1;
    return H >= 2 && o > 0 ? o : GA_ERR_BADARG;
}

// the kernels read and write float2 and __nv_bfloat162 through these pointers
static inline bool misaligned(const void *p, uintptr_t bytes)
{
    return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) != 0;
}

static int conv4x4_args(ConvArgs &a, const void *x, int n, int H, int W, int Cin, const void *w_packed, int k_pitch,
                        const float *bias, int Cout, int stride, float *out_f32, void *out_bf16)
{
    const int Ho = ga_conv4x4_out_size(H, stride), Wo = ga_conv4x4_out_size(W, stride);
    if (Ho <= 0 || Wo <= 0) return GA_ERR_BADARG;
    return conv_args_common(a, 4, x, n, H, W, Cin, Ho, Wo, w_packed, k_pitch, bias, Cout, stride, 1, 1, nullptr,
                            out_f32, out_bf16);
}

extern "C" int ga_conv4x4_lrelu_bf16(const void *x, int n, int H, int W, int Cin, const void *w_packed, int k_pitch,
                                     const float *bias, int Cout, int stride, void *out_bf16, void *stream)
{
    ConvArgs a;
    const int rc = conv4x4_args(a, x, n, H, W, Cin, w_packed, k_pitch, bias, Cout, stride, nullptr, out_bf16);
    if (rc) return rc;
    if (!out_bf16 || misaligned(out_bf16, 4)) return GA_ERR_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    return Cout % 128 == 0 ? launch_conv<4, 128, kEpiLrelu>(a, s) : launch_conv<4, 64, kEpiLrelu>(a, s);
}

extern "C" int ga_conv4x4_stats(const void *x, int n, int H, int W, int Cin, const void *w_packed, int k_pitch,
                                int Cout, int stride, float *z, void *partial, void *stream)
{
    ConvArgs a;
    if (!z || misaligned(z, 8) || misaligned(partial, 8)) return GA_ERR_BADARG;
    const int rc = conv4x4_args(a, x, n, H, W, Cin, w_packed, k_pitch, nullptr, Cout, stride, z, nullptr);
    if (rc) return rc;
    a.partial = reinterpret_cast<float2 *>(partial);
    cudaStream_t s = (cudaStream_t)stream;
    if (!partial)                           // eval mode: the running statistics need no partials
        return Cout % 128 == 0 ? launch_conv<4, 128, kEpiNone>(a, s) : launch_conv<4, 64, kEpiNone>(a, s);
    return Cout % 128 == 0 ? launch_conv<4, 128, kEpiStats>(a, s) : launch_conv<4, 64, kEpiStats>(a, s);
}

extern "C" int ga_disc_bn_forward(const float *z, const void *partial, int64_t M, int C, const float *gamma,
                                  const float *beta, int training, float momentum, float eps, float *running_mean,
                                  float *running_var, float *mean_out, float *rstd_out, void *a_out, void *stream)
{
    if (!z || !gamma || !beta || !running_mean || !running_var || !mean_out || !rstd_out || !a_out) return GA_ERR_BADARG;
    if (M <= 0 || C <= 0 || C % 2 || (training && (!partial || M < 2))) return GA_ERR_BADARG;
    if (misaligned(z, 8) || misaligned(partial, 8) || misaligned(a_out, 4)) return GA_ERR_BADARG;
    if (M > ((int64_t)1 << 31) / CBM * CBM) return GA_ERR_SIZE;
    cudaStream_t s = (cudaStream_t)stream;
    const int nb = (int)((M + CBM - 1) / CBM);
    bn_finalize_kernel<<<C, kFinThreads, 0, s>>>(reinterpret_cast<const float2 *>(partial), nb, M, C, training,
                                                       momentum, eps, running_mean, running_var, mean_out, rstd_out);
    bn_apply_kernel<<<grid_for(M * C / 2, 256 * 8), 256, 0, s>>>(z, M, C, mean_out, rstd_out, gamma, beta,
                                                                  reinterpret_cast<__nv_bfloat16 *>(a_out));
    return (int)cudaGetLastError();
}

extern "C" int ga_disc_conv5(const void *x, int n, int H, int W, const float *w5, const float *bias, float *out,
                             void *stream)
{
    if (!x || !w5 || !bias || !out || n <= 0 || H < 2 || W < 2) return GA_ERR_BADARG;
    if (reinterpret_cast<uintptr_t>(x) & 15) return GA_ERR_BADARG;
    const int64_t total = (int64_t)n * (H - 1) * (W - 1);
    disc_conv5_kernel<<<grid_for(total, 8 * 4), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __nv_bfloat16 *>(x), n, H, W, w5, bias, out);
    return (int)cudaGetLastError();
}

extern "C" int ga_disc_conv5_partials(int n, int H, int W)
{
    if (n <= 0 || H <= 0 || W <= 0) return GA_ERR_BADARG;
    return (int)(((int64_t)n * H * W + kC5Pix - 1) / kC5Pix);
}

extern "C" int ga_disc_conv5_backward(const float *g5, int n, int H, int W, const float *w5, const void *a4,
                                      const float *z4, const float *mean4, const float *rstd4, float *gy4,
                                      void *bn_partial, float *dw_partial, float *dw5, void *stream)
{
    if (!g5 || !w5 || !a4 || !z4 || !mean4 || !rstd4 || !gy4 || !bn_partial || (!dw_partial) != (!dw5))
        return GA_ERR_BADARG;
    if (n <= 0 || H < 2 || W < 2) return GA_ERR_BADARG;
    if (misaligned(a4, 4) || misaligned(z4, 8) || misaligned(gy4, 8) || misaligned(bn_partial, 8) ||
        misaligned(dw_partial, 8))
        return GA_ERR_BADARG;
    const int nb = ga_disc_conv5_partials(n, H, W);
    cudaStream_t s = (cudaStream_t)stream;
    disc_conv5_backward_kernel<<<nb, kC5 / 2, 0, s>>>(g5, n, H, W, w5, reinterpret_cast<const __nv_bfloat16 *>(a4), z4,
                                                      mean4, rstd4, gy4, reinterpret_cast<float2 *>(bn_partial),
                                                      dw_partial);
    if (dw5) reduce_rows_kernel<<<16 * kC5 / 256, 256, 0, s>>>(dw_partial, nb, 16 * kC5, dw5);
    return (int)cudaGetLastError();
}

extern "C" int ga_disc_dgrad_partials(int n, int H, int W, int stride)
{
    if (n <= 0 || H <= 0 || W <= 0) return GA_ERR_BADARG;
    if (stride == 1) return (int)(((int64_t)n * H * W + CBM - 1) / CBM);
    if (stride != 2) return GA_ERR_BADARG;
    int64_t t = 0;
    for (int cls = 0; cls < 4; cls++) {
        const int64_t ha = (H - (cls >> 1) + 1) / 2, wa = (W - (cls & 1) + 1) / 2;
        t += (n * ha * wa + CBM - 1) / CBM;
    }
    return (int)t;
}

extern "C" int ga_disc_dgrad(const void *g, int n, int H, int W, int Cg, const void *w_packed, int k_pitch, int Cout,
                             int stride, const void *act, const float *z, const float *mean, const float *rstd,
                             float *gy_out, void *partial, void *out_bf16, void *stream)
{
    const int Hg = ga_conv4x4_out_size(H, stride), Wg = ga_conv4x4_out_size(W, stride);
    if (Hg <= 0 || Wg <= 0 || !act || (reinterpret_cast<uintptr_t>(act) & 3)) return GA_ERR_BADARG;
    const bool bn = z != nullptr;
    if (bn ? (!mean || !rstd || !gy_out || !partial || out_bf16) : (!out_bf16 || gy_out)) return GA_ERR_BADARG;
    if (misaligned(z, 8) || misaligned(gy_out, 8) || misaligned(partial, 8) || misaligned(out_bf16, 4))
        return GA_ERR_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    const int ncls = stride == 1 ? 1 : 4;
    int part_off = 0;
    for (int cls = 0; cls < ncls; cls++) {
        ConvArgs a;
        int rc;
        const __nv_bfloat16 *wc = reinterpret_cast<const __nv_bfloat16 *>(w_packed) + (size_t)cls * Cout * k_pitch;
        if (stride == 1) {
            // the 4x4 convolution of the gradient padded by 2, flipped weights: output H x W
            rc = conv_args_common(a, 4, g, n, Hg, Wg, Cg, H, W, wc, k_pitch, nullptr, Cout, 1, 2, 2, nullptr, gy_out,
                                  out_bf16);
        } else {
            const int py = cls >> 1, px = cls & 1;
            const int Ha = (H - py + 1) / 2, Wa = (W - px + 1) / 2;
            rc = conv_args_common(a, 2, g, n, Hg, Wg, Cg, Ha, Wa, wc, k_pitch, nullptr, Cout, 1, 1 - py, 1 - px, nullptr,
                                  gy_out, out_bf16);
            a.scatter = 1; a.o_H = H; a.o_W = W; a.o_s = 2; a.o_py = py; a.o_px = px;
        }
        if (rc) return rc;
        a.mask = reinterpret_cast<const __nv_bfloat16 *>(act);
        a.z = z; a.bn_mean = mean; a.bn_rstd = rstd;
        a.partial = reinterpret_cast<float2 *>(partial);
        a.part_off = part_off;
        part_off += (a.M + CBM - 1) / CBM;
        if (stride == 1)
            rc = bn ? (Cout % 128 == 0 ? launch_conv<4, 128, kEpiBnGrad>(a, s) : launch_conv<4, 64, kEpiBnGrad>(a, s))
                    : (Cout % 128 == 0 ? launch_conv<4, 128, kEpiLreluGrad>(a, s) : launch_conv<4, 64, kEpiLreluGrad>(a, s));
        else
            rc = bn ? (Cout % 128 == 0 ? launch_conv<2, 128, kEpiBnGrad>(a, s) : launch_conv<2, 64, kEpiBnGrad>(a, s))
                    : (Cout % 128 == 0 ? launch_conv<2, 128, kEpiLreluGrad>(a, s) : launch_conv<2, 64, kEpiLreluGrad>(a, s));
        if (rc) return rc;
    }
    return 0;
}

extern "C" int ga_disc_bn_backward(const float *gy, const float *z, int64_t M, int C, const float *mean,
                                   const float *rstd, const float *gamma, const void *partial, int n_partial,
                                   int training, float *dgamma, float *dbeta, void *k_scratch, void *dz_bf16,
                                   void *stream)
{
    if (!gy || !z || !mean || !rstd || !gamma || !partial || !k_scratch || !dz_bf16) return GA_ERR_BADARG;
    if (M <= 0 || C <= 0 || C % 2 || n_partial <= 0) return GA_ERR_BADARG;
    if (misaligned(gy, 8) || misaligned(z, 8) || misaligned(partial, 8) || misaligned(k_scratch, 8) ||
        misaligned(dz_bf16, 4))
        return GA_ERR_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    float2 *k = reinterpret_cast<float2 *>(k_scratch);
    bn_grad_finalize_kernel<<<C, kFinThreads, 0, s>>>(reinterpret_cast<const float2 *>(partial), n_partial, M, C,
                                                            training, dgamma, dbeta, k);
    bn_grad_apply_kernel<<<grid_for(M * C / 2, 256 * 8), 256, 0, s>>>(gy, z, M, C, mean, rstd, gamma, k,
                                                                       reinterpret_cast<__nv_bfloat16 *>(dz_bf16));
    return (int)cudaGetLastError();
}

extern "C" size_t ga_disc_wgrad_workspace_bytes(int n, int Ho, int Wo, int Co, int Cin)
{
    if (n <= 0 || Ho <= 0 || Wo <= 0 || Co <= 0 || Cin <= 0) return 0;
    const int64_t P = (int64_t)n * Ho * Wo;
    if (P >= (int64_t)1 << 31) return 0;
    return (size_t)wgrad_splits((int)P, Co, Cin) * Co * 16 * Cin * sizeof(float);
}

extern "C" int ga_disc_wgrad(const void *dy, const void *x, int n, int H, int W, int Cin, int Co, int stride,
                             int cin_out, void *workspace, size_t workspace_bytes, float *dw, void *stream)
{
    const int Ho = ga_conv4x4_out_size(H, stride), Wo = ga_conv4x4_out_size(W, stride);
    if (!dy || !x || !dw || n <= 0 || Ho <= 0 || Wo <= 0 || Cin <= 0 || Cin % 8 || Co <= 0 || Co % 64) return GA_ERR_BADARG;
    if (cin_out <= 0 || cin_out > Cin) return GA_ERR_BADARG;
    if ((reinterpret_cast<uintptr_t>(dy) & 15) || (reinterpret_cast<uintptr_t>(x) & 15)) return GA_ERR_BADARG;
    const int64_t P = (int64_t)n * Ho * Wo;
    if (P >= (int64_t)1 << 31 || (int64_t)n * H * W >= (int64_t)1 << 31) return GA_ERR_SIZE;
    if (!workspace || workspace_bytes < ga_disc_wgrad_workspace_bytes(n, Ho, Wo, Co, Cin)) return GA_ERR_WORKSPACE;
    if (misaligned(workspace, 8)) return GA_ERR_BADARG;
    static GaPerDevice attr_set;
    if (ga_first_use_on_device(attr_set)) {
        cudaError_t e = cudaFuncSetAttribute(wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmem);
        if (e != cudaSuccess) return (int)e;
    }
    WgradArgs a;
    a.dy = reinterpret_cast<const __nv_bfloat16 *>(dy);
    a.x = reinterpret_cast<const __nv_bfloat16 *>(x);
    a.n = n; a.H = H; a.W = W; a.Cin = Cin; a.Ho = Ho; a.Wo = Wo; a.Co = Co; a.stride = stride; a.P = (int)P;
    const int splits = wgrad_splits((int)P, Co, Cin);
    a.chunk = (int)((P + splits - 1) / splits);
    a.chunk = (a.chunk + kWgBK - 1) / kWgBK * kWgBK;
    a.ncols = 16 * Cin;
    a.part = reinterpret_cast<float *>(workspace);
    cudaStream_t s = (cudaStream_t)stream;
    const dim3 grid(a.ncols / kWgBN, (Co + kWgBM - 1) / kWgBM, splits);
    wgrad_kernel<<<grid, 256, kWgSmem, s>>>(a);
    wgrad_reduce_kernel<<<grid_for((int64_t)Co * cin_out * 16, 256), 256, 0, s>>>(a.part, splits, Co, Cin, cin_out, dw);
    return (int)cudaGetLastError();
}

extern "C" size_t ga_disc_colsum_scratch_bytes(int64_t rows, int C)
{
    if (rows <= 0 || C <= 0) return 0;
    return (size_t)((rows + kColRows - 1) / kColRows) * C * sizeof(float);
}

extern "C" int ga_disc_colsum(const void *x, int is_bf16, int64_t rows, int C, void *scratch, size_t scratch_bytes,
                              float *out, void *stream)
{
    if (!x || !out || rows <= 0 || C <= 0 || 256 % C) return GA_ERR_BADARG;
    if (!scratch || scratch_bytes < ga_disc_colsum_scratch_bytes(rows, C)) return GA_ERR_WORKSPACE;
    const int nb = (int)((rows + kColRows - 1) / kColRows);
    cudaStream_t s = (cudaStream_t)stream;
    float *part = reinterpret_cast<float *>(scratch);
    if (is_bf16)
        colsum_partial_kernel<__nv_bfloat16><<<nb, 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16 *>(x), rows, C, part);
    else
        colsum_partial_kernel<float><<<nb, 256, 0, s>>>(reinterpret_cast<const float *>(x), rows, C, part);
    reduce_rows_kernel<<<(C + 255) / 256, 256, 0, s>>>(part, nb, C, out);
    return (int)cudaGetLastError();
}

extern "C" int ga_disc_input_backward(const void *g1, int n, int H, int W, const float *w1, float *dx, void *stream)
{
    if (!g1 || !w1 || !dx || n <= 0 || H < 2 || W < 2) return GA_ERR_BADARG;
    if (reinterpret_cast<uintptr_t>(g1) & 15) return GA_ERR_BADARG;
    if ((int64_t)n * H * W >= (int64_t)1 << 31) return GA_ERR_SIZE;
    disc_input_backward_kernel<<<grid_for((int64_t)n * H * W, 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __nv_bfloat16 *>(g1), n, H, W, w1, dx);
    return (int)cudaGetLastError();
}
