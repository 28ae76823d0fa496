// 3D VAE encoder kernels (HybridEncoderPCDStructuredLatentSNoPCD, /root/reference/nsr/srt/encoder.py:454-652):
// the SD conv encoder's 3x3 convolutions as an implicit GEMM on wgmma, GroupNorm(32) [+ SiLU] in NHWC,
// farthest-point sampling, the input / token-xyz packing, the head-32 split of the SRT blocks and the readout head
// with the posterior.  The 1x1 convolutions, linears and attentions run on the Part 2 GEMM / attention entry points.
#include "../../include/ga_b200.h"
#include "conv_igemm.cuh"
#include "row_common.cuh"

using namespace ga_row;

namespace {

// ---------------------------------------------------------------------------------------------------------------
// GroupNorm(32) over NHWC fp32, deterministic split reduction.  Pass 1: one CTA per (pixel chunk, image) sums each
// channel's values shifted by the chunk's first pixel (the pivot), so a group whose |mean| is large against its std
// loses nothing to cancellation, and writes the chunk's per-group Chan terms (mean, M2 = sum of squared deviations)
// formed in fp64.  Pass 2: every CTA merges its image's terms in fp64 into mean and 1/sqrt(var + eps), then
// normalises its chunk, applies the affine and optional SiLU and writes bf16 or fp32.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kGnThreads = 256;
constexpr int kGroups = 32;
constexpr int kGnMergeLanes = kGnThreads / kGroups;     // pass 2: lanes that merge one group's chunk terms

__host__ __device__ inline int gn_chunk_px(int HW) { return HW >= 65536 ? 1024 : (HW >= 4096 ? 256 : 64); }

__global__ void __launch_bounds__(kGnThreads) gn_stats_kernel(const float *__restrict__ x, float2 *__restrict__ part,
                                                              int HW, int C, int chunk_px, int nchunk)
{
    __shared__ float2 red[kGnThreads * 4];
    __shared__ float2 ch_sum[1024];
    __shared__ float piv[1024];
    const int img = blockIdx.y, ck = blockIdx.x;
    const int quads = C / 4, slots = kGnThreads / quads;
    const int q = threadIdx.x % quads, s = threadIdx.x / quads;
    const int p0 = ck * chunk_px, p1 = min(HW, p0 + chunk_px);
    const float *xi = x + (size_t)img * HW * C;
    float sm[4] = {0.f, 0.f, 0.f, 0.f}, sq[4] = {0.f, 0.f, 0.f, 0.f};
    if (s < slots) {
        const float4 pv = __ldg(reinterpret_cast<const float4 *>(xi + (size_t)p0 * C) + q);
        if (s == 0) { piv[4 * q] = pv.x; piv[4 * q + 1] = pv.y; piv[4 * q + 2] = pv.z; piv[4 * q + 3] = pv.w; }
        for (int p = p0 + s; p < p1; p += slots) {
            const float4 v = __ldg(reinterpret_cast<const float4 *>(xi + (size_t)p * C) + q);
            const float d[4] = {v.x - pv.x, v.y - pv.y, v.z - pv.z, v.w - pv.w};
#pragma unroll
            for (int e = 0; e < 4; e++) { sm[e] += d[e]; sq[e] += d[e] * d[e]; }
        }
    }
#pragma unroll
    for (int e = 0; e < 4; e++) red[threadIdx.x * 4 + e] = make_float2(sm[e], sq[e]);
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += kGnThreads) {
        float a = 0.f, b = 0.f;
        for (int t = 0; t < slots; t++) {
            const float2 v = red[(t * quads + c / 4) * 4 + (c & 3)];
            a += v.x; b += v.y;
        }
        ch_sum[c] = make_float2(a, b);
    }
    __syncthreads();
    if (threadIdx.x < kGroups) {
        // channel c: mean_c = pivot_c + sum d / n, M2_c = sum d^2 - (sum d)^2 / n; the group's equal-count merge:
        // mean = average of mean_c, M2 = sum M2_c + n sum (mean_c - mean)^2
        const int cpg = C / kGroups, c0 = threadIdx.x * cpg;
        const double n = (double)(p1 - p0), rn = 1.0 / n;
        double mean = 0.0;
        for (int c = c0; c < c0 + cpg; c++) mean += (double)piv[c] + (double)ch_sum[c].x * rn;
        mean /= cpg;
        double m2 = 0.0;
        for (int c = c0; c < c0 + cpg; c++) {
            const double a = ch_sum[c].x, dm = (double)piv[c] + a * rn - mean;
            m2 += fmax((double)ch_sum[c].y - a * a * rn, 0.0) + n * dm * dm;
        }
        part[((size_t)img * nchunk + ck) * kGroups + threadIdx.x] = make_float2((float)mean, (float)m2);
    }
}

__global__ void __launch_bounds__(kGnThreads) gn_apply_kernel(const float *__restrict__ x, const float2 *__restrict__ part,
                                                              const float *__restrict__ gamma, const float *__restrict__ beta,
                                                              void *__restrict__ out, int out_bf16, int silu, int HW, int C,
                                                              int chunk_px, int nchunk, float eps)
{
    __shared__ float2 stat[kGroups];          // mean, rstd
    const int img = blockIdx.y, ck = blockIdx.x;
    {
        // Chan's merge of the chunks' (mean, M2), chunk i holding n_i pixels of the group's cpg channels: lane j of
        // the group's kGnMergeLanes takes chunks j, j + kGnMergeLanes, ...; the lanes' sums meet by xor shuffles
        const int g = threadIdx.x / kGnMergeLanes, j = threadIdx.x % kGnMergeLanes;
        const float2 *pg = part + (size_t)img * nchunk * kGroups + g;
        double a = 0.0;
        for (int i = j; i < nchunk; i += kGnMergeLanes) a += (double)min(chunk_px, HW - i * chunk_px) * pg[(size_t)i * kGroups].x;
#pragma unroll
        for (int o = 1; o < kGnMergeLanes; o <<= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        const double mean = a / HW;
        double b = 0.0;
        for (int i = j; i < nchunk; i += kGnMergeLanes) {
            const float2 v = pg[(size_t)i * kGroups];
            const double d = v.x - mean;
            b += v.y + (double)min(chunk_px, HW - i * chunk_px) * (C / kGroups) * d * d;
        }
#pragma unroll
        for (int o = 1; o < kGnMergeLanes; o <<= 1) b += __shfl_xor_sync(0xffffffffu, b, o);
        const double var = b / ((double)HW * (C / kGroups));
        if (j == 0) stat[g] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
    }
    __syncthreads();
    const int quads = C / 4, cpg = C / kGroups;
    const int p0 = ck * chunk_px, p1 = min(HW, p0 + chunk_px);
    const size_t base = ((size_t)img * HW + p0) * quads;
    const size_t total = (size_t)(p1 - p0) * quads;
    for (size_t i = threadIdx.x; i < total; i += kGnThreads) {
        const int q = (int)(i % quads);
        const float4 v = __ldg(reinterpret_cast<const float4 *>(x) + base + i);
        float y[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const int c = 4 * q + e;
            const float2 st = stat[c / cpg];
            float t = (y[e] - st.x) * st.y * __ldg(gamma + c) + __ldg(beta + c);
            if (silu) t = t / (1.f + __expf(-t));
            y[e] = t;
        }
        if (out_bf16) {
            __nv_bfloat162 lo = __floats2bfloat162_rn(y[0], y[1]), hi = __floats2bfloat162_rn(y[2], y[3]);
            uint2 u = make_uint2(*reinterpret_cast<uint32_t *>(&lo), *reinterpret_cast<uint32_t *>(&hi));
            reinterpret_cast<uint2 *>(out)[base + i] = u;
        } else {
            reinterpret_cast<float4 *>(out)[base + i] = make_float4(y[0], y[1], y[2], y[3]);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Farthest-point sampling, one 1024-thread CTA per sample; thread t owns points t, t + 1024, ... in registers.
// d(p, s) = (dx*dx + dy*dy) + dz*dz with every operation rounded on its own, so the order of selection is
// reproducible by any IEEE fp32 restatement; ties go to the lowest index.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kFpsThreads = 1024, kFpsPer = 16;

__device__ __forceinline__ bool fps_better(float d, int i, float d2, int i2) { return d > d2 || (d == d2 && i < i2); }

__global__ void __launch_bounds__(kFpsThreads, 1) fps_kernel(const float *__restrict__ pcd, int N, int K,
                                                             const int32_t *__restrict__ start, int32_t *__restrict__ idx_out,
                                                             float *__restrict__ xyz_out)
{
    __shared__ float wd[32];
    __shared__ int wix[32];
    __shared__ int sel;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float *P = pcd + (size_t)b * N * 3;
    float px[kFpsPer], py[kFpsPer], pz[kFpsPer], md[kFpsPer];
#pragma unroll
    for (int i = 0; i < kFpsPer; i++) {
        const int p = tid + i * kFpsThreads;
        if (p < N) { px[i] = P[3 * p]; py[i] = P[3 * p + 1]; pz[i] = P[3 * p + 2]; md[i] = INFINITY; }
        else { px[i] = py[i] = pz[i] = 0.f; md[i] = -1.f; }
    }
    int cur = start[b];
    for (int k = 0; k < K; k++) {
        const float sx = P[3 * cur], sy = P[3 * cur + 1], sz = P[3 * cur + 2];
        if (tid == 0) {
            idx_out[(size_t)b * K + k] = cur;
            float *o = xyz_out + ((size_t)b * K + k) * 3;
            o[0] = sx; o[1] = sy; o[2] = sz;
        }
        if (k + 1 == K) break;
        float best = -2.f;
        int bi = 0x7fffffff;
#pragma unroll
        for (int i = 0; i < kFpsPer; i++) {
            const int p = tid + i * kFpsThreads;
            if (p < N) {
                const float dx = __fsub_rn(px[i], sx), dy = __fsub_rn(py[i], sy), dz = __fsub_rn(pz[i], sz);
                const float d = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
                md[i] = fminf(md[i], d);
                if (md[i] > best) { best = md[i]; bi = p; }          // increasing p: strict > keeps the lowest index
            }
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const float d2 = __shfl_xor_sync(0xffffffffu, best, o);
            const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
            if (fps_better(d2, i2, best, bi)) { best = d2; bi = i2; }
        }
        if (lane == 0) { wd[warp] = best; wix[warp] = bi; }
        __syncthreads();
        if (warp == 0) {
            best = wd[lane]; bi = wix[lane];
#pragma unroll
            for (int o = 16; o; o >>= 1) {
                const float d2 = __shfl_xor_sync(0xffffffffu, best, o);
                const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
                if (fps_better(d2, i2, best, bi)) { best = d2; bi = i2; }
            }
            if (lane == 0) sel = bi;
        }
        __syncthreads();
        cur = sel;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Input packing: NCHW fp32 -> NHWC bf16 with the channels zero-padded to c_pad, and the token xyz
// x[:, xyz_c:xyz_c+3, off::step, off::step] in "(n h w) 3" order.
// ---------------------------------------------------------------------------------------------------------------
__global__ void pack_input_kernel(const float *__restrict__ img, int n, int C, int H, int W, int c_pad,
                                  __nv_bfloat16 *__restrict__ out)
{
    const size_t total = (size_t)n * H * W;
    for (size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x; p < total; p += (size_t)gridDim.x * blockDim.x) {
        const size_t im = p / ((size_t)H * W), hw = p - im * H * W;
        for (int c = 0; c < c_pad; c += 2) {
            const float a = c < C ? __ldg(img + (im * C + c) * H * W + hw) : 0.f;
            const float b = c + 1 < C ? __ldg(img + (im * C + c + 1) * H * W + hw) : 0.f;
            *reinterpret_cast<__nv_bfloat162 *>(out + p * c_pad + c) = __floats2bfloat162_rn(a, b);
        }
    }
}

__global__ void token_xyz_kernel(const float *__restrict__ img, int n, int C, int H, int W, int xyz_c, int step, int off,
                                 int Ht, int Wt, float *__restrict__ out)
{
    const int total = n * Ht * Wt;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
        const int im = t / (Ht * Wt), r = t - im * Ht * Wt;
        const int ty = r / Wt, tx = r - ty * Wt;
        const size_t pix = (size_t)(off + ty * step) * W + off + tx * step;
#pragma unroll
        for (int d = 0; d < 3; d++) out[(size_t)t * 3 + d] = __ldg(img + ((size_t)im * C + xyz_c + d) * H * W + pix);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// SRT attention with head_dim 32: qkv bf16 [R, 3 * H * 32] ("(K H D)" columns, bias already added) -> per-head
// RMSNorm(32) on q and k (fp32, then * weight), written zero-padded to head_dim 64 in the layout ga_attention_bf16
// reads: Q, K [B, H, tok_pitch, 64], Vt [B, H, 64, tok_pitch].  The padding contributes nothing to q.k or to P V.
// One warp per (token, head): lane = dimension.
// ---------------------------------------------------------------------------------------------------------------
__global__ void heads32_kernel(const __nv_bfloat16 *__restrict__ qkv, const float *__restrict__ qn_w,
                               const float *__restrict__ kn_w, int R, int H, int rows_per_batch, int tok_pitch, float eps,
                               __nv_bfloat16 *__restrict__ q, __nv_bfloat16 *__restrict__ k, __nv_bfloat16 *__restrict__ vt)
{
    const int lane = threadIdx.x & 31;
    const long wid = (blockIdx.x * (long)blockDim.x + threadIdx.x) >> 5;
    if (wid >= (long)R * H) return;
    const int m = (int)(wid / H), h = (int)(wid % H);
    const int b = m / rows_per_batch, t = m - b * rows_per_batch;
    const __nv_bfloat16 *row = qkv + (size_t)m * 3 * H * 32;
    const size_t qk_off = (((size_t)b * H + h) * tok_pitch + t) * 64;
#pragma unroll
    for (int which = 0; which < 2; which++) {
        const float v = __bfloat162float(row[(which * H + h) * 32 + lane]);
        float ss = v * v;
#pragma unroll
        for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        const float *w = which == 0 ? qn_w : kn_w;
        const float y = w ? v * rsqrtf(ss * (1.0f / 32.0f) + eps) * __ldg(w + lane) : v;
        __nv_bfloat16 *dst = (which == 0 ? q : k) + qk_off;
        dst[lane] = __float2bfloat16(y);
        dst[32 + lane] = __float2bfloat16(0.f);
    }
    __nv_bfloat16 *vd = vt + ((size_t)b * H + h) * 64 * tok_pitch + t;
    vd[(size_t)lane * tok_pitch] = row[(2 * H + h) * 32 + lane];
    vd[(size_t)(32 + lane) * tok_pitch] = __float2bfloat16(0.f);
}

// ---------------------------------------------------------------------------------------------------------------
// Readout head, one CTA per token, all fp32: Mlp_out = LayerNorm -> fc1 -> tanh-GELU -> fc2 (2 zc), then the
// decoder's quant_conv (fc1 -> tanh-GELU -> fc2), then DiagonalGaussianDistribution(soft_clamp=True):
// logvar = 20 tanh(logvar / 20), std = exp(logvar / 2), latent = mean + std * eps.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kHeadThreads = 256;
constexpr int kHeadRed = kHeadThreads / 32;        // block_sum's static shared floats

__device__ __forceinline__ float block_sum(float v, float *red)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = 0.f;
    for (int i = 0; i < kHeadThreads / 32; i++) s += red[i];
    return s;
}

// y[o] = b[o] + sum_i W[o, i] x[i] for o < n_out, one output per thread (strided)
__device__ __forceinline__ void row_linear(const float *__restrict__ W, const float *__restrict__ b, const float *x, int n_in,
                                           int n_out, float *y, int act)
{
    for (int o = threadIdx.x; o < n_out; o += kHeadThreads) {
        const float *w = W + (size_t)o * n_in;
        float s = b ? __ldg(b + o) : 0.f;
        for (int i = 0; i < n_in; i++) s = fmaf(__ldg(w + i), x[i], s);
        y[o] = act ? gelu_tanh(s) : s;
    }
}

__global__ void __launch_bounds__(kHeadThreads) readout_head_kernel(const GaVaeEncHead p, const float *__restrict__ x,
                                                                    const float *__restrict__ noise, int D, int hid, int zc,
                                                                    float *__restrict__ h_out, float *__restrict__ mean,
                                                                    float *__restrict__ logvar, float *__restrict__ stdv,
                                                                    float *__restrict__ latent)
{
    extern __shared__ float sh[];
    float *xn = sh, *hv = sh + D, *m = hv + hid, *q1 = m + 2 * zc, *q2 = q1 + 2 * zc;
    __shared__ float red[kHeadRed];
    const size_t r = blockIdx.x;
    const float *xr = x + r * D;
    float s = 0.f;
    for (int i = threadIdx.x; i < D; i += kHeadThreads) s += xr[i];
    const float mu = block_sum(s, red) / D;
    s = 0.f;
    for (int i = threadIdx.x; i < D; i += kHeadThreads) { const float d = xr[i] - mu; s += d * d; }
    const float rstd = rsqrtf(block_sum(s, red) / D + p.ln_eps);
    for (int i = threadIdx.x; i < D; i += kHeadThreads) xn[i] = (xr[i] - mu) * rstd * __ldg(p.ln_w + i) + __ldg(p.ln_b + i);
    __syncthreads();
    row_linear(p.fc1_w, p.fc1_b, xn, D, hid, hv, 1);
    __syncthreads();
    row_linear(p.fc2_w, p.fc2_b, hv, hid, 2 * zc, m, 0);
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * zc; i += kHeadThreads) h_out[r * 2 * zc + i] = m[i];
    row_linear(p.q1_w, p.q1_b, m, 2 * zc, 2 * zc, q1, 1);
    __syncthreads();
    row_linear(p.q2_w, p.q2_b, q1, 2 * zc, 2 * zc, q2, 0);
    __syncthreads();
    for (int i = threadIdx.x; i < zc; i += kHeadThreads) {
        const float mn = q2[i];
        const float lv = 20.f * tanhf(q2[zc + i] / 20.f);
        const float sd = expf(0.5f * lv);
        mean[r * zc + i] = mn;
        logvar[r * zc + i] = lv;
        if (stdv) stdv[r * zc + i] = sd;
        if (latent) latent[r * zc + i] = noise ? mn + sd * noise[r * zc + i] : mn;
    }
}

}  // namespace

// ---- host side ----------------------------------------------------------------------------------------------------
// the argument checks of the 3x3 entry points; fills `a` and returns 0, or the error code
static int conv_args(ConvArgs &a, const void *x, int n, int H, int W, int Cin, const void *w_packed, int k_pitch,
                     const float *bias, int Cout, int stride, const float *residual, float *out_f32, void *out_bf16)
{
    if (n <= 0 || Cin <= 0 || Cin % 8 || Cout <= 0 || Cout % 64) return GA_ERR_BADARG;
    if (!out_f32 && !out_bf16) return GA_ERR_BADARG;
    const int Ho = ga_conv3x3_out_size(H, stride), Wo = ga_conv3x3_out_size(W, stride);
    if (Ho <= 0 || Wo <= 0) return GA_ERR_BADARG;
    // the epilogue reads residual and writes out_f32 as float2, out_bf16 as __nv_bfloat162
    if (mis8(residual) || mis8(out_f32) || mis4(out_bf16)) return GA_ERR_BADARG;
    // stride 1: pad 1 on every side; stride 2: pad (0, 1, 0, 1), i.e. none on the top / left
    const int pad = stride == 1 ? 1 : 0;
    return conv_args_common(a, 3, x, n, H, W, Cin, Ho, Wo, w_packed, k_pitch, bias, Cout, stride, pad, pad, residual,
                            out_f32, out_bf16);
}

extern "C" int ga_conv3x3_out_size(int H, int stride)
{
    if (H <= 0) return GA_ERR_BADARG;
    if (stride == 1) return H;
    if (stride == 2) return H >= 2 ? (H - 2) / 2 + 1 : GA_ERR_BADARG;
    return GA_ERR_BADARG;
}

extern "C" int ga_conv3x3_bf16(const void *x, int n, int H, int W, int Cin, const void *w_packed, int k_pitch,
                               const float *bias, int Cout, int stride, const float *residual, float *out_f32,
                               void *out_bf16, void *stream)
{
    ConvArgs a;
    const int rc = conv_args(a, x, n, H, W, Cin, w_packed, k_pitch, bias, Cout, stride, residual, out_f32, out_bf16);
    if (rc) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    return Cout % 128 == 0 ? launch_conv<3, 128, kEpiNone>(a, s) : launch_conv<3, 64, kEpiNone>(a, s);
}

extern "C" int ga_conv3x3_relu_bf16(const void *x, int n, int H, int W, int Cin, const void *w_packed, int k_pitch,
                                    const float *bias, int Cout, void *out_bf16, void *stream)
{
    ConvArgs a;
    const int rc = conv_args(a, x, n, H, W, Cin, w_packed, k_pitch, bias, Cout, 1, nullptr, nullptr, out_bf16);
    if (rc) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    return Cout % 128 == 0 ? launch_conv<3, 128, kEpiRelu>(a, s) : launch_conv<3, 64, kEpiRelu>(a, s);
}

extern "C" int ga_conv3x3_mask_bf16(const void *x, int n, int H, int W, int Cin, const void *w_packed, int k_pitch,
                                    int Cout, const void *mask, void *out_bf16, void *stream)
{
    ConvArgs a;
    if (!mask || (reinterpret_cast<uintptr_t>(mask) & 3)) return GA_ERR_BADARG;
    const int rc = conv_args(a, x, n, H, W, Cin, w_packed, k_pitch, nullptr, Cout, 1, nullptr, nullptr, out_bf16);
    if (rc) return rc;
    a.mask = reinterpret_cast<const __nv_bfloat16 *>(mask);
    cudaStream_t s = (cudaStream_t)stream;
    return Cout % 128 == 0 ? launch_conv<3, 128, kEpiMask>(a, s) : launch_conv<3, 64, kEpiMask>(a, s);
}

extern "C" size_t ga_group_norm_scratch_bytes(int n, int HW)
{
    if (n <= 0 || HW <= 0) return 0;
    const int cp = gn_chunk_px(HW);
    return (size_t)n * ((HW + cp - 1) / cp) * kGroups * sizeof(float2);
}

extern "C" int ga_group_norm_nhwc(const float *x, const float *gamma, const float *beta, int n, int HW, int C, float eps,
                                  int silu, void *out, int out_bf16, void *scratch, size_t scratch_bytes, void *stream)
{
    if (!x || !gamma || !beta || !out || !scratch || n <= 0 || HW <= 0) return GA_ERR_BADARG;
    if (C <= 0 || C % kGroups || C % 4 || C > 1024) return GA_ERR_BADARG;
    if (C / 4 > kGnThreads) return GA_ERR_BADARG;
    if (mis16(x) || (out_bf16 ? mis8(out) : mis16(out))) return GA_ERR_BADARG;      // float4 loads, float4 / uint2 stores
    if (scratch_bytes < ga_group_norm_scratch_bytes(n, HW)) return GA_ERR_WORKSPACE;
    const int cp = gn_chunk_px(HW), nchunk = (HW + cp - 1) / cp;
    cudaStream_t s = (cudaStream_t)stream;
    float2 *part = reinterpret_cast<float2 *>(scratch);
    gn_stats_kernel<<<dim3(nchunk, n), kGnThreads, 0, s>>>(x, part, HW, C, cp, nchunk);
    gn_apply_kernel<<<dim3(nchunk, n), kGnThreads, 0, s>>>(x, part, gamma, beta, out, out_bf16, silu, HW, C, cp, nchunk, eps);
    return (int)cudaGetLastError();
}

extern "C" int ga_fps(const float *pcd, int batch, int N, int K, const int32_t *start_idx, int32_t *idx_out,
                      float *xyz_out, void *stream)
{
    if (!pcd || !start_idx || !idx_out || !xyz_out || batch <= 0 || N <= 0 || K <= 0) return GA_ERR_BADARG;
    if (N > kFpsThreads * kFpsPer || K > 1024 || K > N) return GA_ERR_SIZE;
    fps_kernel<<<batch, kFpsThreads, 0, (cudaStream_t)stream>>>(pcd, N, K, start_idx, idx_out, xyz_out);
    return (int)cudaGetLastError();
}

extern "C" int ga_vae_enc_input(const float *img, int n, int C, int H, int W, int c_pad, void *x_bf16, int xyz_c,
                                int step, int off, float *token_xyz, void *stream)
{
    if (!img || !x_bf16 || n <= 0 || C <= 0 || H <= 0 || W <= 0 || c_pad < C || c_pad % 8) return GA_ERR_BADARG;
    if (reinterpret_cast<uintptr_t>(x_bf16) & 3) return GA_ERR_BADARG;                  // __nv_bfloat162 stores
    if (token_xyz && (xyz_c < 0 || xyz_c + 3 > C || step <= 0 || off < 0 || off >= H || off >= W)) return GA_ERR_BADARG;
    cudaStream_t s = (cudaStream_t)stream;
    pack_input_kernel<<<1024, 256, 0, s>>>(img, n, C, H, W, c_pad, reinterpret_cast<__nv_bfloat16 *>(x_bf16));
    if (token_xyz) {
        const int Ht = (H - off + step - 1) / step, Wt = (W - off + step - 1) / step;
        token_xyz_kernel<<<256, 256, 0, s>>>(img, n, C, H, W, xyz_c, step, off, Ht, Wt, token_xyz);
    }
    return (int)cudaGetLastError();
}

extern "C" int ga_heads32_split(const void *qkv, const float *qn_w, const float *kn_w, int R, int heads,
                                int rows_per_batch, int tok_pitch, float eps, void *q, void *k, void *vt, void *stream)
{
    if (!qkv || !q || !k || !vt || R <= 0 || heads <= 0 || rows_per_batch <= 0 || tok_pitch < rows_per_batch)
        return GA_ERR_BADARG;
    const long threads = (long)R * heads * 32;
    heads32_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __nv_bfloat16 *>(qkv), qn_w, kn_w, R, heads, rows_per_batch, tok_pitch, eps,
        reinterpret_cast<__nv_bfloat16 *>(q), reinterpret_cast<__nv_bfloat16 *>(k), reinterpret_cast<__nv_bfloat16 *>(vt));
    return (int)cudaGetLastError();
}

extern "C" int ga_vae_enc_head(const GaVaeEncHead *p, const float *x, const float *noise, int R, int D, int hid, int zc,
                               float *h_out, float *mean, float *logvar, float *stdv, float *latent, void *stream)
{
    if (!p || !x || !h_out || !mean || !logvar || R <= 0 || D <= 0 || hid <= 0 || zc <= 0) return GA_ERR_BADARG;
    if (!p->ln_w || !p->ln_b || !p->fc1_w || !p->fc2_w || !p->q1_w || !p->q2_w) return GA_ERR_BADARG;
    // the launch fails unless static + dynamic shared memory fit the default 48 KiB per block
    const size_t smem = (size_t)(D + hid + 6 * zc) * sizeof(float);
    if (smem + kHeadRed * sizeof(float) > 48 * 1024) return GA_ERR_SIZE;
    readout_head_kernel<<<R, kHeadThreads, smem, (cudaStream_t)stream>>>(*p, x, noise, D, hid, zc, h_out, mean, logvar, stdv,
                                                                         latent);
    return (int)cudaGetLastError();
}
