// Implicit-GEMM convolution on wgmma, shared by the VAE encoder and LPIPS (3x3, vae_encoder.cu) and the PatchGAN
// discriminator (4x4 and the 2x2 parity classes of its stride-2 dgrad, disc_ops.cu).  Formulas in include/ga_b200.h
// Parts 5 and 11.
#pragma once
#include "../../include/ga_b200.h"
#include "device_once.cuh"
#include "sm90_ptx.cuh"

namespace {

using namespace sm90;

// ---------------------------------------------------------------------------------------------------------------
// KS x KS convolution, implicit GEMM: out[m, n] = bias[n] + sum_k A[m, k] W[n, k] (+ residual[m, n]), then the
// epilogue EPI (below), m = (image, oy, ox) over [n, Ho, Wo], k = (ky * KS + kx) * Cin + c; the tap (ky, kx) of output
// pixel (oy, ox) reads input pixel (stride oy - pad_y + ky, stride ox - pad_x + kx).  A is never materialised: every
// 16-byte piece (8 channels of one tap of one output pixel) is gathered with cp.async straight from the NHWC input,
// zero-filled where the tap falls into the padding or k runs past KS * KS * Cin.  The pieces land in the
// 128-byte-swizzled K-major layout that wgmma_desc_k_sw128 describes, the layout the TMA GEMM uses.  Two warpgroups,
// each 64 output pixels x BN channels; a kConvStages-deep cp.async ring keeps kConvStages - 2 K-blocks in flight
// ahead of the MMAs.
// Output row: m itself, or with `scatter` the pixel (o_s oy + o_py, o_s ox + o_px) of an [n, o_H, o_W] map (the
// parity classes of a stride-2 dgrad write every other pixel of the full gradient).
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
    float *out_f32;             // [rows, Cout] or NULL
    __nv_bfloat16 *out_bf16;    // [rows, Cout] or NULL
    int H, W, Cin, Ho, Wo, Cout, k_pitch, stride, M, K;
    const __nv_bfloat16 *mask;  // [rows, Cout]: kEpiMask, kEpiLreluGrad, kEpiBnGrad (the activation whose sign selects)
    int pad_y, pad_x;
    int scatter, o_H, o_W, o_s, o_py, o_px;
    const float *z;             // kEpiBnGrad: [rows, Cout] the BatchNorm's input
    const float *bn_mean, *bn_rstd;   // kEpiBnGrad: [Cout]
    float2 *partial;            // kEpiStats / kEpiBnGrad: [part_off + gridDim.x, Cout]
    int part_off;
};

// kEpiNone as is; kEpiRelu max(., 0); kEpiMask mask > 0 ? . : 0 (a select: the ReLU backward, where mask is the
// forward's ReLU output, so a non-finite value never leaks through a masked zero); kEpiLrelu v > 0 ? v : 0.2 v;
// kEpiLreluGrad v * (mask > 0 ? 1 : 0.2) (the LeakyReLU backward, mask its output); kEpiStats fp32 out plus the
// CTA's per-channel (mean, M2) over its rows; kEpiBnGrad g = v * (mask > 0 ? 1 : 0.2) to out_f32 plus the CTA's
// per-channel (sum g, sum g xhat), xhat = (z - bn_mean) * bn_rstd.
constexpr int kEpiNone = 0, kEpiRelu = 1, kEpiMask = 2, kEpiLrelu = 3, kEpiLreluGrad = 4, kEpiStats = 5,
              kEpiBnGrad = 6;

// Per-channel sums over the CTA's 128 rows of two values per fragment element: lanes of equal l % 4 by an xor
// butterfly (16 rows per warp), then the eight warps in order.  red: 8 * BN float2 of shared memory.  Thread t < BN
// gets column t's sums.  Every thread of the CTA calls it.
template <int BN>
__device__ __forceinline__ float2 cta_column_sums(const float (&u)[BN / 2], const float (&v)[BN / 2], float2 *red)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
#pragma unroll
        for (int e = 0; e < 2; e++) {
            float s = u[4 * j + e] + u[4 * j + 2 + e], t = v[4 * j + e] + v[4 * j + 2 + e];
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
                s += __shfl_xor_sync(0xffffffffu, s, o);
                t += __shfl_xor_sync(0xffffffffu, t, o);
            }
            if (lane < 4) red[warp * BN + 8 * j + 2 * lane + e] = make_float2(s, t);
        }
    }
    __syncthreads();
    float2 r = make_float2(0.f, 0.f);
    if ((int)threadIdx.x < BN) {
#pragma unroll
        for (int w = 0; w < kConvThreads / 32; w++) {
            const float2 q = red[w * BN + threadIdx.x];
            r.x += q.x; r.y += q.y;
        }
    }
    __syncthreads();
    return r;
}

template <int KS, int BN, int EPI>
__global__ void __launch_bounds__(kConvThreads, 1) conv_igemm_kernel(const ConvArgs a)
{
    using Cfg = ConvCfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = align1024(smem_raw);
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
            oy0[i] = a.stride * oy - a.pad_y;
            ox0[i] = a.stride * ox - a.pad_x;
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
            const int ky = tap / KS, kx = tap - ky * KS;
            // sw128_off(r, chunk) written out so that sa + r * 128 is added first: calling it reorders the additions
            // and changes these kernels' register allocation
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
    constexpr bool kStat = EPI == kEpiStats || EPI == kEpiBnGrad;
    float su[kStat ? BN / 2 : 1], sv[kStat ? BN / 2 : 1];
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
        const int n = n0 + 8 * j + 2 * cq;
        const float b0 = a.bias ? __ldg(a.bias + n) : 0.f, b1 = a.bias ? __ldg(a.bias + n + 1) : 0.f;
        float mu0 = 0.f, mu1 = 0.f, rs0 = 0.f, rs1 = 0.f;
        if (EPI == kEpiBnGrad) {
            mu0 = __ldg(a.bn_mean + n); mu1 = __ldg(a.bn_mean + n + 1);
            rs0 = __ldg(a.bn_rstd + n); rs1 = __ldg(a.bn_rstd + n + 1);
        }
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
            const int m = m0 + wg * 64 + wi * 16 + r + 8 * hf;
            if constexpr (kStat) { su[4 * j + 2 * hf] = su[4 * j + 2 * hf + 1] = 0.f; sv[4 * j + 2 * hf] = sv[4 * j + 2 * hf + 1] = 0.f; }
            if (m >= a.M) continue;
            float v0 = acc[4 * j + 2 * hf] + b0, v1 = acc[4 * j + 2 * hf + 1] + b1;
            size_t row = m;
            if (a.scatter) {
                const int hw = a.Ho * a.Wo;
                const int img = m / hw, p = m - img * hw;
                const int oy = p / a.Wo, ox = p - oy * a.Wo;
                row = ((size_t)img * a.o_H + a.o_s * oy + a.o_py) * a.o_W + a.o_s * ox + a.o_px;
            }
            const size_t o = row * a.Cout + n;
            if (a.residual) {
                const float2 rr = *reinterpret_cast<const float2 *>(a.residual + o);
                v0 += rr.x; v1 += rr.y;
            }
            if (EPI == kEpiRelu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            if (EPI == kEpiMask) {
                const float2 mk = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(a.mask + o));
                v0 = mk.x > 0.f ? v0 : 0.f;
                v1 = mk.y > 0.f ? v1 : 0.f;
            }
            if (EPI == kEpiLrelu) {
                v0 = v0 > 0.f ? v0 : 0.2f * v0;
                v1 = v1 > 0.f ? v1 : 0.2f * v1;
            }
            if (EPI == kEpiLreluGrad || EPI == kEpiBnGrad) {
                const float2 mk = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(a.mask + o));
                v0 = mk.x > 0.f ? v0 : 0.2f * v0;
                v1 = mk.y > 0.f ? v1 : 0.2f * v1;
            }
            if constexpr (EPI == kEpiStats) { su[4 * j + 2 * hf] = v0; su[4 * j + 2 * hf + 1] = v1; }
            if constexpr (EPI == kEpiBnGrad) {
                const float2 zz = *reinterpret_cast<const float2 *>(a.z + o);
                su[4 * j + 2 * hf] = v0; su[4 * j + 2 * hf + 1] = v1;
                sv[4 * j + 2 * hf] = v0 * ((zz.x - mu0) * rs0);
                sv[4 * j + 2 * hf + 1] = v1 * ((zz.y - mu1) * rs1);
            }
            if (a.out_f32) *reinterpret_cast<float2 *>(a.out_f32 + o) = make_float2(v0, v1);
            if (a.out_bf16) *reinterpret_cast<__nv_bfloat162 *>(a.out_bf16 + o) = __floats2bfloat162_rn(v0, v1);
        }
    }
    if constexpr (kStat) {
        __syncthreads();                    // every warpgroup is past its MMAs: the ring is free
        float2 *red = reinterpret_cast<float2 *>(smem);
        float2 *part = a.partial + (size_t)(a.part_off + blockIdx.x) * a.Cout + n0;
        if constexpr (EPI == kEpiStats) {
            // Chan's per-CTA terms: mean over the CTA's valid rows, then M2 = sum (v - mean)^2 from the registers
            const int cnt = min(CBM, a.M - m0);
            float2 s = cta_column_sums<BN>(su, su, red);
            float *mean_s = reinterpret_cast<float *>(red + 8 * BN);
            if (tid < BN) mean_s[tid] = s.x / (float)cnt;
            __syncthreads();
#pragma unroll
            for (int j = 0; j < BN / 8; j++) {
#pragma unroll
                for (int hf = 0; hf < 2; hf++) {
                    const int m = m0 + wg * 64 + wi * 16 + r + 8 * hf;
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const float d = su[4 * j + 2 * hf + e] - mean_s[8 * j + 2 * cq + e];
                        sv[4 * j + 2 * hf + e] = m < a.M ? d * d : 0.f;
                    }
                }
            }
            const float2 q = cta_column_sums<BN>(sv, sv, red);
            if (tid < BN) part[tid] = make_float2(mean_s[tid], q.x);
        } else {
            const float2 s = cta_column_sums<BN>(su, sv, red);
            if (tid < BN) part[tid] = s;
        }
    }
}

// ---- host side ----------------------------------------------------------------------------------------------------
template <int KS, int BN, int EPI>
static int launch_conv(const ConvArgs &a, cudaStream_t s)
{
    using Cfg = ConvCfg<BN>;
    static GaPerDevice attr_set;
    if (ga_first_use_on_device(attr_set)) {
        cudaError_t e = cudaFuncSetAttribute(conv_igemm_kernel<KS, BN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             Cfg::kSmem);
        if (e != cudaSuccess) return (int)e;
    }
    dim3 grid((a.M + CBM - 1) / CBM, a.Cout / BN);
    return (int)ga_launch_pdl(conv_igemm_kernel<KS, BN, EPI>, grid, dim3(kConvThreads), (size_t)Cfg::kSmem, s, a);
}

// the common argument checks: fills `a` (no scatter, no epilogue extras) and returns 0, or the error code
static int conv_args_common(ConvArgs &a, int KS, const void *x, int n, int H, int W, int Cin, int Ho, int Wo,
                            const void *w_packed, int k_pitch, const float *bias, int Cout, int stride, int pad_y,
                            int pad_x, const float *residual, float *out_f32, void *out_bf16)
{
    if (!x || !w_packed || n <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cin % 8 || Cout <= 0 || Cout % 64)
        return GA_ERR_BADARG;
    if (!out_f32 && !out_bf16) return GA_ERR_BADARG;
    if (Ho <= 0 || Wo <= 0) return GA_ERR_BADARG;
    if (k_pitch < ((KS * KS * Cin + CBK - 1) / CBK) * CBK || (reinterpret_cast<uintptr_t>(w_packed) & 15) ||
        (reinterpret_cast<uintptr_t>(x) & 15))
        return GA_ERR_BADARG;
    if ((int64_t)n * Ho * Wo >= (int64_t)1 << 31) return GA_ERR_SIZE;
    a = ConvArgs{};
    a.x = reinterpret_cast<const __nv_bfloat16 *>(x);
    a.w = reinterpret_cast<const __nv_bfloat16 *>(w_packed);
    a.bias = bias; a.residual = residual; a.out_f32 = out_f32;
    a.out_bf16 = reinterpret_cast<__nv_bfloat16 *>(out_bf16);
    a.H = H; a.W = W; a.Cin = Cin; a.Ho = Ho; a.Wo = Wo; a.Cout = Cout; a.k_pitch = k_pitch; a.stride = stride;
    a.M = n * Ho * Wo; a.K = KS * KS * Cin;
    a.pad_y = pad_y; a.pad_x = pad_x;
    return 0;
}

}  // namespace
