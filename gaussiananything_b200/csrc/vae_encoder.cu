// 3D VAE encoder kernels (HybridEncoderPCDStructuredLatentSNoPCD, /root/reference/nsr/srt/encoder.py:454-652):
// the SD conv encoder's 3x3 convolutions as an implicit GEMM on wgmma, GroupNorm(32) [+ SiLU] in NHWC,
// farthest-point sampling, the input / token-xyz packing, the head-32 split of the SRT blocks and the readout head
// with the posterior.  The 1x1 convolutions, linears and attentions run on the Part 2 GEMM / attention entry points.
#include "../../include/ga_b200.h"
#include "device_once.cuh"
#include "sm90_ptx.cuh"

using namespace sm90;

namespace {

// ---------------------------------------------------------------------------------------------------------------
// 3x3 convolution, implicit GEMM: out[m, n] = bias[n] + sum_k A[m, k] W[n, k] (+ residual[m, n]),
// m = (image, oy, ox), k = (ky * 3 + kx) * Cin + c.  A is never materialised: every 16-byte piece (8 channels of one
// tap of one output pixel) is gathered with cp.async straight from the NHWC input, zero-filled where the tap falls
// into the padding or k runs past 9 * Cin.  The pieces land in the 128-byte-swizzled K-major layout that
// wgmma_desc_k_sw128 describes, the layout the TMA GEMM uses.  Two warpgroups, each 64 output pixels x BN channels;
// a kConvStages-deep cp.async ring keeps kConvStages - 2 K-blocks in flight ahead of the MMAs.
// ---------------------------------------------------------------------------------------------------------------
constexpr int CBM = 128, CBK = 64;
constexpr int kConvThreads = 256;
constexpr int kConvStages = 5;

template <int BN> struct ConvCfg {
    static constexpr int kABytes = CBM * CBK * 2;
    static constexpr int kBBytes = BN * CBK * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kSmem = kConvStages * kStageBytes + 1024;
};

struct ConvArgs {
    const __nv_bfloat16 *x;     // [n, H, W, Cin]
    const __nv_bfloat16 *w;     // [Cout, k_pitch]
    const float *bias;          // [Cout] or NULL
    const float *residual;      // [M, Cout] fp32 or NULL
    float *out_f32;             // [M, Cout] or NULL
    __nv_bfloat16 *out_bf16;    // [M, Cout] or NULL
    int H, W, Cin, Ho, Wo, Cout, k_pitch, stride, M, K;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, bool valid)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }
// cp.async writes through the generic proxy, wgmma reads through the async proxy
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

template <int BN>
__global__ void __launch_bounds__(kConvThreads, 1) conv3x3_kernel(const ConvArgs a)
{
    using Cfg = ConvCfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wg = warp >> 2, wi = warp & 3;
    const int m0 = blockIdx.x * CBM, n0 = blockIdx.y * BN;
    const int nk = (a.K + CBK - 1) / CBK;
    const int chunk = tid & 7;

    // the 4 output pixels this thread gathers for: rows r = tid / 8 + 32 i of the tile
    int img_base[4], oy0[4], ox0[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int m = m0 + (tid >> 3) + 32 * i;
        if (m < a.M) {
            const int hw = a.Ho * a.Wo;
            const int img = m / hw, p = m - img * hw;
            const int oy = p / a.Wo, ox = p - oy * a.Wo;
            img_base[i] = img;
            // stride 1: pad 1 on every side; stride 2: pad (0, 1, 0, 1), i.e. none on the top / left
            oy0[i] = a.stride == 1 ? oy - 1 : 2 * oy;
            ox0[i] = a.stride == 1 ? ox - 1 : 2 * ox;
        } else {
            img_base[i] = -1; oy0[i] = 0; ox0[i] = 0;
        }
    }

    pdl_wait();
    pdl_launch_dependents();

    auto load_stage = [&](int kb) {
        if (kb < nk) {
            const int s = kb % kConvStages;
            const uint32_t sa = smem_u32(smem + s * Cfg::kStageBytes);
            const uint32_t sb = sa + Cfg::kABytes;
            const int k = kb * CBK + chunk * 8;
            const bool kin = k < a.K;
            const int tap = kin ? k / a.Cin : 0;
            const int c = k - tap * a.Cin;
            const int ky = tap / 3, kx = tap - ky * 3;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int r = (tid >> 3) + 32 * i;
                const int iy = oy0[i] + ky, ix = ox0[i] + kx;
                const bool v = kin && img_base[i] >= 0 && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
                const __nv_bfloat16 *src = v ? a.x + (((size_t)img_base[i] * a.H + iy) * a.W + ix) * a.Cin + c : a.x;
                cp_async16(sa + r * 128 + ((chunk ^ (r & 7)) << 4), src, v);
            }
#pragma unroll
            for (int i = 0; i < BN / 32; i++) {
                const int r = (tid >> 3) + 32 * i;
                cp_async16(sb + r * 128 + ((chunk ^ (r & 7)) << 4), a.w + (size_t)(n0 + r) * a.k_pitch + kb * CBK + chunk * 8,
                           true);
            }
        }
        cp_async_commit();                  // an empty group past the end keeps the wait counts uniform
    };

    for (int kb = 0; kb < kConvStages - 2; kb++) load_stage(kb);

    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; i++) acc[i] = 0.f;
    for (int kb = 0; kb < nk; kb++) {
        cp_async_wait<kConvStages - 3>();   // this thread's pieces of K-block kb have landed
        fence_proxy_async();
        __syncthreads();                    // ... and everyone's; both warpgroups have retired the MMAs of kb - 2
        load_stage(kb + kConvStages - 2);   // into the slot of kb - 2
        const int s = kb % kConvStages;
        const uint64_t ad = wgmma_desc_k_sw128(smem_u32(smem + s * Cfg::kStageBytes + wg * 64 * 128));
        const uint64_t bd = wgmma_desc_k_sw128(smem_u32(smem + s * Cfg::kStageBytes + Cfg::kABytes));
        fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < CBK / 16; k++) wgmma_ss<BN>(acc, ad + (uint64_t)(k * 2), bd + (uint64_t)(k * 2), 1u);
        wgmma_commit();
        wgmma_wait<1>();
        fence_regs(acc);
    }
    wgmma_wait<0>();
    fence_regs(acc);
    cp_async_wait<0>();

    // epilogue straight from the fragment: row 16 wi + lane/4 (+8), columns 8 j + 2 (lane%4) (+1)
    const int r = lane >> 2, cq = lane & 3;
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
        const int n = n0 + 8 * j + 2 * cq;
        const float b0 = a.bias ? __ldg(a.bias + n) : 0.f, b1 = a.bias ? __ldg(a.bias + n + 1) : 0.f;
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
            const int m = m0 + wg * 64 + wi * 16 + r + 8 * hf;
            if (m >= a.M) continue;
            float v0 = acc[4 * j + 2 * hf] + b0, v1 = acc[4 * j + 2 * hf + 1] + b1;
            const size_t o = (size_t)m * a.Cout + n;
            if (a.residual) {
                const float2 rr = *reinterpret_cast<const float2 *>(a.residual + o);
                v0 += rr.x; v1 += rr.y;
            }
            if (a.out_f32) *reinterpret_cast<float2 *>(a.out_f32 + o) = make_float2(v0, v1);
            if (a.out_bf16) *reinterpret_cast<__nv_bfloat162 *>(a.out_bf16 + o) = __floats2bfloat162_rn(v0, v1);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// GroupNorm(32) over NHWC fp32, deterministic split reduction.  Pass 1: one CTA per (pixel chunk, image) writes the
// chunk's per-group fp32 sum and sum of squares.  Pass 2: every CTA folds its image's partials in fp64 into mean and
// 1/sqrt(var + eps), then normalises its chunk, applies the affine and optional SiLU and writes bf16 or fp32.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kGnThreads = 256;
constexpr int kGroups = 32;

__host__ __device__ inline int gn_chunk_px(int HW) { return HW >= 65536 ? 1024 : (HW >= 4096 ? 256 : 64); }

__global__ void __launch_bounds__(kGnThreads) gn_stats_kernel(const float *__restrict__ x, float2 *__restrict__ part,
                                                              int HW, int C, int chunk_px, int nchunk)
{
    __shared__ float2 red[kGnThreads * 4];
    __shared__ float2 ch_sum[1024];
    const int img = blockIdx.y, ck = blockIdx.x;
    const int quads = C / 4, slots = kGnThreads / quads;
    const int q = threadIdx.x % quads, s = threadIdx.x / quads;
    const int p0 = ck * chunk_px, p1 = min(HW, p0 + chunk_px);
    float sm[4] = {0.f, 0.f, 0.f, 0.f}, sq[4] = {0.f, 0.f, 0.f, 0.f};
    if (s < slots) {
        for (int p = p0 + s; p < p1; p += slots) {
            const float4 v = __ldg(reinterpret_cast<const float4 *>(x + ((size_t)img * HW + p) * C) + q);
            sm[0] += v.x; sm[1] += v.y; sm[2] += v.z; sm[3] += v.w;
            sq[0] += v.x * v.x; sq[1] += v.y * v.y; sq[2] += v.z * v.z; sq[3] += v.w * v.w;
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
        const int cpg = C / kGroups;
        float a = 0.f, b = 0.f;
        for (int c = threadIdx.x * cpg; c < (threadIdx.x + 1) * cpg; c++) { a += ch_sum[c].x; b += ch_sum[c].y; }
        part[((size_t)img * nchunk + ck) * kGroups + threadIdx.x] = make_float2(a, b);
    }
}

__global__ void __launch_bounds__(kGnThreads) gn_apply_kernel(const float *__restrict__ x, const float2 *__restrict__ part,
                                                              const float *__restrict__ gamma, const float *__restrict__ beta,
                                                              void *__restrict__ out, int out_bf16, int silu, int HW, int C,
                                                              int chunk_px, int nchunk, float eps)
{
    __shared__ float2 stat[kGroups];          // mean, rstd
    const int img = blockIdx.y, ck = blockIdx.x;
    if (threadIdx.x < kGroups) {
        double a = 0.0, b = 0.0;
        for (int i = 0; i < nchunk; i++) {
            const float2 v = part[((size_t)img * nchunk + i) * kGroups + threadIdx.x];
            a += v.x; b += v.y;
        }
        const double n = (double)HW * (C / kGroups);
        const double mean = a / n;
        double var = b / n - mean * mean;
        if (var < 0.0) var = 0.0;
        stat[threadIdx.x] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
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

__device__ __forceinline__ float gelu_tanh(float x)
{
    return 0.5f * x * (1.f + tanhf(0.7978845608028654f * (x + 0.044715f * x * x * x)));
}

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
    __shared__ float red[kHeadThreads / 32];
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
template <int BN>
static int launch_conv(const ConvArgs &a, cudaStream_t s)
{
    using Cfg = ConvCfg<BN>;
    static GaPerDevice attr_set;
    if (ga_first_use_on_device(attr_set)) {
        cudaError_t e = cudaFuncSetAttribute(conv3x3_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem);
        if (e != cudaSuccess) return (int)e;
    }
    dim3 grid((a.M + CBM - 1) / CBM, a.Cout / BN);
    return (int)ga_launch_pdl(conv3x3_kernel<BN>, grid, dim3(kConvThreads), (size_t)Cfg::kSmem, s, a);
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
    if (!x || !w_packed || n <= 0 || Cin <= 0 || Cin % 8 || Cout <= 0 || Cout % 64) return GA_ERR_BADARG;
    if (!out_f32 && !out_bf16) return GA_ERR_BADARG;
    const int Ho = ga_conv3x3_out_size(H, stride), Wo = ga_conv3x3_out_size(W, stride);
    if (Ho <= 0 || Wo <= 0) return GA_ERR_BADARG;
    if (k_pitch < ((9 * Cin + CBK - 1) / CBK) * CBK || (reinterpret_cast<uintptr_t>(w_packed) & 15) ||
        (reinterpret_cast<uintptr_t>(x) & 15))
        return GA_ERR_BADARG;
    if ((int64_t)n * Ho * Wo >= (int64_t)1 << 31) return GA_ERR_SIZE;
    ConvArgs a;
    a.x = reinterpret_cast<const __nv_bfloat16 *>(x);
    a.w = reinterpret_cast<const __nv_bfloat16 *>(w_packed);
    a.bias = bias; a.residual = residual; a.out_f32 = out_f32;
    a.out_bf16 = reinterpret_cast<__nv_bfloat16 *>(out_bf16);
    a.H = H; a.W = W; a.Cin = Cin; a.Ho = Ho; a.Wo = Wo; a.Cout = Cout; a.k_pitch = k_pitch; a.stride = stride;
    a.M = n * Ho * Wo; a.K = 9 * Cin;
    cudaStream_t s = (cudaStream_t)stream;
    return Cout % 128 == 0 ? launch_conv<128>(a, s) : launch_conv<64>(a, s);
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
    if (C % kGroups || C % 4 || C > 1024 || (C / kGroups) * kGroups != C) return GA_ERR_BADARG;
    if (C / 4 > kGnThreads) return GA_ERR_BADARG;
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
    cudaStream_t s = (cudaStream_t)stream;
    pack_input_kernel<<<1024, 256, 0, s>>>(img, n, C, H, W, c_pad, reinterpret_cast<__nv_bfloat16 *>(x_bf16));
    if (token_xyz) {
        if (xyz_c < 0 || xyz_c + 3 > C || step <= 0 || off < 0 || off >= H || off >= W) return GA_ERR_BADARG;
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
    const size_t smem = (size_t)(D + hid + 6 * zc) * sizeof(float);
    if (smem > 48 * 1024) return GA_ERR_SIZE;
    readout_head_kernel<<<R, kHeadThreads, smem, (cudaStream_t)stream>>>(*p, x, noise, D, hid, zc, h_out, mean, logvar, stdv,
                                                                         latent);
    return (int)cudaGetLastError();
}
