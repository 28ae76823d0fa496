// wgmma GEMM for the DiT denoiser: C[M,N] = A[M,K] * W[N,K]^T, bf16 operands,
// fp32 accumulation in registers, fused epilogues.  Replaces the cuBLAS nn.Linear +
// separate bias / GELU / gate / residual / qk-RMSNorm / permute kernels of
// /root/reference/dit/dit_models_xformers.py:765-787,
// /root/reference/vit/vision_transformer.py:215-303 and
// /root/reference/ldm/modules/attention.py:484-561.
//
// The main loop is gemm_sm90.cuh's persistent kernel with both operands K-major; this file holds its epilogues.
#include "../../include/ga_b200.h"
#include "gemm_sm90.cuh"
#include "row_common.cuh"

using namespace ga_row;
using namespace gemm_sm90;

namespace {

// exact-erf GELU to ~3e-7 (Abramowitz-Stegun 7.1.28: erf x = 1 - (1 + a1 x + .. + a6 x^6)^-16), 1 MUFU + ~16 FP32
// ops per element; the library erff() costs about twice that and would make the GELU epilogue slower than the MMAs.
__device__ __forceinline__ float gelu_erf(float v)
{
    const float x = fabsf(v) * 0.70710678118654752f;
    float p = 0.0000430638f;
    p = fmaf(p, x, 0.0002765672f);
    p = fmaf(p, x, 0.0001520143f);
    p = fmaf(p, x, 0.0092705272f);
    p = fmaf(p, x, 0.0422820123f);
    p = fmaf(p, x, 0.0705230784f);
    p = fmaf(p, x, 1.0f);
    p = p * p; p = p * p; p = p * p; p = p * p;
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(p));
    const float erf_abs = 1.0f - r;
    return 0.5f * v * (1.0f + copysignf(erf_abs, v));
}

// ---- epilogue ---------------------------------------------------------------
// A warp's accumulator fragment covers 16 rows; a lane holds pairs of adjacent columns of two rows, so storing
// straight from registers would write 8-byte pieces of 8 rows per instruction.  Each consumer warp therefore owns a
// 2 KB staging buffer (16 rows x 128 B, 16-byte chunks XOR-swizzled by row&7 so both phases are bank-conflict free):
//   phase A (fragment layout)          : registers -> staging, 32 fp32 columns at a time
//   phase B (8 lanes = one 128 B row)  : staging -> bias / GELU / gate / residual -> coalesced global stores
// The epilogue mode is a template parameter, so the unrolled loops carry no run-time switch.
constexpr int kWarpRows = 16;              // accumulator rows per warp

// Epilogue of ga_linear_fc1_gelu_bf16 (include/ga_b200.h Part 13), outside the GA_EPI_* range so that
// ga_gemm_bf16_tn never reaches it: H = bf16(gelu_erf(v)) to out and Z = bf16(v) to q, v = acc + bias, both bf16
// [M, ld_out].  GaGemmEpilogue has no field for a second output; q is the one pointer this mode does not otherwise use.
constexpr int kEpiGeluKeepPre = 100;

// columns [32 ch, 32 ch + 32) of the warp's 16 rows -> staging (fp32, row-major, 128 B per row)
template <int R>
__device__ __forceinline__ void stage_chunk(uint32_t stg, int lane, const float (&acc)[R], int ch)
{
    const int r = lane >> 2, c = lane & 3;
#pragma unroll
    for (int jj = 0; jj < 4; jj++) {
        const int j = 4 * ch + jj;
        const int col = 8 * jj + 2 * c;                        // column inside the chunk
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
            const int row = r + 8 * hf;
            sts64(stg + row * 128 + (((col >> 2) ^ (row & 7)) << 4) + (col & 3) * 4, acc[4 * j + 2 * hf],
                  acc[4 * j + 2 * hf + 1]);
        }
    }
}

// per-lane column parameters of phase B (this lane's 4 columns nn .. nn+3)
struct ColParams { float bias[4]; float gate[4]; };

template <int MODE>
__device__ __forceinline__ void load_col_params(const GaGemmEpilogue &ep, int lane, int m0w, int n, int N, ColParams &cp)
{
    const int nn = n + (lane & 7) * 4;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        cp.bias[j] = (ep.bias && nn + j < N) ? __ldg(ep.bias + nn + j) : 0.f;
        cp.gate[j] = 1.f;
    }
    if (MODE == GA_EPI_RESID_GATE_F32 && ep.gate) {
        const int b = m0w / ep.rows_per_batch;           // used when the warp's rows sit in one batch element
#pragma unroll
        for (int j = 0; j < 4; j++) if (nn + j < N) cp.gate[j] = __ldg(ep.gate + (size_t)b * ep.gate_ld + nn + j);
    }
}

// 32 fp32 accumulator columns [n, n+32) of the warp's 16 rows [m0w, m0w+16), already staged by stage_chunk()
template <int MODE>
__device__ __forceinline__ void epilogue_chunk(const GaGemmEpilogue &ep, uint32_t stg, int lane, int m0w, int n, int M,
                                               int N, const ColParams &cp)
{
    constexpr int kIt = kWarpRows / 4;
    const int ch = lane & 7, rsub = lane >> 3;
    const int nn = n + ch * 4;                                 // this lane's 4 columns
    const bool vec = (nn + 4 <= N) && (ep.ld_out % 4) == 0;
    bool one_batch = true;
    if (MODE == GA_EPI_RESID_GATE_F32 && ep.gate)
        one_batch = (m0w + kWarpRows - 1) / ep.rows_per_batch == m0w / ep.rows_per_batch;
    uint4 acc[kIt];
#pragma unroll
    for (int it = 0; it < kIt; it++) {
        const int rr = it * 4 + rsub;
        acc[it] = lds128(stg + rr * 128 + ((ch ^ (rr & 7)) << 4));
    }
    // residual rows are read up front, all in flight at once: interleaved with the stores below the compiler
    // must assume they alias and the loop degenerates into serial L2 round trips per chunk
    float4 res[kIt];
    if (MODE == GA_EPI_RESID_GATE_F32 && vec) {
#pragma unroll
        for (int it = 0; it < kIt; it++) {
            const int m = m0w + it * 4 + rsub;
            res[it] = (m < M) ? *reinterpret_cast<const float4 *>(reinterpret_cast<const float *>(ep.out) +
                                                                   (size_t)m * ep.ld_out + nn)
                              : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    if (nn >= N) return;
#pragma unroll
    for (int it = 0; it < kIt; it++) {
        const int m = m0w + it * 4 + rsub;
        if (m >= M) continue;
        float v[4] = {__uint_as_float(acc[it].x) + cp.bias[0], __uint_as_float(acc[it].y) + cp.bias[1],
                      __uint_as_float(acc[it].z) + cp.bias[2], __uint_as_float(acc[it].w) + cp.bias[3]};
        if (MODE == GA_EPI_BF16 || MODE == GA_EPI_GELU_BF16) {
            if (MODE == GA_EPI_GELU_BF16) {
#pragma unroll
                for (int j = 0; j < 4; j++) v[j] = gelu_erf(v[j]);
            }
            __nv_bfloat16 *dst = reinterpret_cast<__nv_bfloat16 *>(ep.out) + (size_t)m * ep.ld_out + nn;
            if (vec) {
                *reinterpret_cast<uint2 *>(dst) = make_uint2(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]));
            } else {
#pragma unroll
                for (int j = 0; j < 4; j++) if (nn + j < N) dst[j] = __float2bfloat16(v[j]);
            }
        } else if (MODE == GA_EPI_F32) {
            float *dst = reinterpret_cast<float *>(ep.out) + (size_t)m * ep.ld_out + nn;
            if (vec) {
                *reinterpret_cast<float4 *>(dst) = make_float4(v[0], v[1], v[2], v[3]);
            } else {
#pragma unroll
                for (int j = 0; j < 4; j++) if (nn + j < N) dst[j] = v[j];
            }
        } else if (MODE == GA_EPI_GEGLU_BF16) {
            // columns interleaved at pack time as (x_j, gate_j) pairs: out[m, j] = x_j * gelu_erf(gate_j)
            __nv_bfloat16 *dst = reinterpret_cast<__nv_bfloat16 *>(ep.out) + (size_t)m * ep.ld_out + nn / 2;
            if (vec) {
                *reinterpret_cast<uint32_t *>(dst) = pack_bf16(v[0] * gelu_erf(v[1]), v[2] * gelu_erf(v[3]));
            } else {
#pragma unroll
                for (int j = 0; j < 4; j += 2) if (nn + j + 1 < N) dst[j / 2] = __float2bfloat16(v[j] * gelu_erf(v[j + 1]));
            }
        } else if (MODE == GA_EPI_RESID_GATE_F32) {
            // x[m, n] += gate[b, n] * (acc + bias)
            float *dst = reinterpret_cast<float *>(ep.out) + (size_t)m * ep.ld_out + nn;
            float g[4] = {cp.gate[0], cp.gate[1], cp.gate[2], cp.gate[3]};
            if (!one_batch) {
                const float *gp = ep.gate + (size_t)(m / ep.rows_per_batch) * ep.gate_ld + nn;
#pragma unroll
                for (int j = 0; j < 4; j++) if (nn + j < N) g[j] = __ldg(gp + j);
            }
            if (vec) {
                float4 x = res[it];
                x.x += g[0] * v[0]; x.y += g[1] * v[1]; x.z += g[2] * v[2]; x.w += g[3] * v[3];
                *reinterpret_cast<float4 *>(dst) = x;
            } else {
#pragma unroll
                for (int j = 0; j < 4; j++) if (nn + j < N) dst[j] += g[j] * v[j];
            }
        } else if (MODE == kEpiGeluKeepPre) {
            __nv_bfloat16 *dh = reinterpret_cast<__nv_bfloat16 *>(ep.out) + (size_t)m * ep.ld_out + nn;
            __nv_bfloat16 *dz = reinterpret_cast<__nv_bfloat16 *>(ep.q) + (size_t)m * ep.ld_out + nn;
            if (vec) {
                *reinterpret_cast<uint2 *>(dz) = make_uint2(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]));
                *reinterpret_cast<uint2 *>(dh) = make_uint2(pack_bf16(gelu_erf(v[0]), gelu_erf(v[1])),
                                                            pack_bf16(gelu_erf(v[2]), gelu_erf(v[3])));
            } else {
#pragma unroll
                for (int j = 0; j < 4; j++)
                    if (nn + j < N) {
                        dz[j] = __float2bfloat16(v[j]);
                        dh[j] = __float2bfloat16(gelu_erf(v[j]));
                    }
            }
        }
    }
}

// HEADS epilogue for one head (64 columns [n, n+64), accumulator groups 8h .. 8h+7) of the warp's 16 rows.
// which = n / inner (+ first_part): 0 q, 1 k, 2 v ; head = (n % inner) / 64   ("(K H D)" column layout,
// vit/vision_transformer.py:191,255).  q/k: per-head RMSNorm (dit/norm.py:27-40), fp32, then * weight; a row's 64
// columns sit in the 4 lanes of a quad, so its sum of squares is two shuffles.  A token's 64 bf16 are one 128 B line
// of the [B, H, tok_pitch, 64] layout.  v is stored transposed per head, [B, H, 64, tok_pitch], so that P*V is a
// K-major x K-major contraction: staged as [d][16 tokens].
template <int R>
__device__ __forceinline__ void epilogue_head(const GaGemmEpilogue &ep, uint32_t stg, const float (&acc)[R], int h,
                                              int lane, int m0w, int n, int M)
{
    const int inner = ep.heads * 64;
    const int which = n / inner + ep.first_part;
    const int head = (n % inner) / 64;
    const float *w = which == 0 ? ep.qn_w : (which == 1 ? ep.kn_w : nullptr);
    const int r = lane >> 2, c = lane & 3;
    float x[2][16];
#pragma unroll
    for (int jj = 0; jj < 8; jj++) {
        const int j = 8 * h + jj, col = 8 * jj + 2 * c;
        const float b0 = ep.bias ? __ldg(ep.bias + n + col) : 0.f;
        const float b1 = ep.bias ? __ldg(ep.bias + n + col + 1) : 0.f;
        x[0][2 * jj] = acc[4 * j] + b0;     x[0][2 * jj + 1] = acc[4 * j + 1] + b1;
        x[1][2 * jj] = acc[4 * j + 2] + b0; x[1][2 * jj + 1] = acc[4 * j + 3] + b1;
    }
    const int rpb = ep.rows_per_batch;
    const int b_first = m0w / rpb;
    const bool one_batch = (m0w + kWarpRows - 1) / rpb == b_first;
    if (which <= 1) {
        float rs[2] = {1.f, 1.f};
        if (w) {
#pragma unroll
            for (int hf = 0; hf < 2; hf++) {
                float ss = 0.f;
#pragma unroll
                for (int i = 0; i < 16; i++) ss += x[hf][i] * x[hf][i];
                ss += __shfl_xor_sync(0xffffffffu, ss, 1);
                ss += __shfl_xor_sync(0xffffffffu, ss, 2);
                rs[hf] = rsqrtf(ss * (1.0f / 64.0f) + ep.eps);
            }
        }
#pragma unroll
        for (int jj = 0; jj < 8; jj++) {
            const int col = 8 * jj + 2 * c;
            const float w0 = w ? __ldg(w + col) : 1.f, w1 = w ? __ldg(w + col + 1) : 1.f;
#pragma unroll
            for (int hf = 0; hf < 2; hf++) {
                const int row = r + 8 * hf;
                sts32(stg + row * 128 + ((jj ^ (row & 7)) << 4) + 4 * c,
                      pack_bf16(x[hf][2 * jj] * rs[hf] * w0, x[hf][2 * jj + 1] * rs[hf] * w1));
            }
        }
        warp_sync_smem();
        __nv_bfloat16 *base = reinterpret_cast<__nv_bfloat16 *>(which == 0 ? ep.q : ep.k);
        const int ch = lane & 7, rsub = lane >> 3;
        uint4 v[kWarpRows / 4];
#pragma unroll
        for (int it = 0; it < kWarpRows / 4; it++) {
            const int rr = it * 4 + rsub;
            v[it] = lds128(stg + rr * 128 + ((ch ^ (rr & 7)) << 4));
        }
#pragma unroll
        for (int it = 0; it < kWarpRows / 4; it++) {
            const int m = m0w + it * 4 + rsub;
            if (m >= M) continue;
            const int b = one_batch ? b_first : m / rpb;
            const int t = m - b * rpb;
            *reinterpret_cast<uint4 *>(base + (((size_t)b * ep.heads + head) * ep.tok_pitch + t) * 64 + ch * 8) = v[it];
        }
    } else {
        const int t0 = m0w - b_first * rpb;
        const bool fast = one_batch && (m0w + kWarpRows <= M) && (ep.tok_pitch % 8) == 0 && (t0 % 8) == 0;
        __nv_bfloat16 *vt = reinterpret_cast<__nv_bfloat16 *>(ep.vt);
        if (fast) {
            // staging [d][16 tokens]: 32 B per head dimension
#pragma unroll
            for (int jj = 0; jj < 8; jj++)
#pragma unroll
                for (int hf = 0; hf < 2; hf++)
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const __nv_bfloat16 hv = __float2bfloat16(x[hf][2 * jj + e]);
                        asm volatile("st.shared.b16 [%0], %1;\n" ::"r"(stg + (uint32_t)((8 * jj + 2 * c + e) * 32 + (r + 8 * hf) * 2)),
                                     "h"(*reinterpret_cast<const unsigned short *>(&hv)));
                    }
            warp_sync_smem();
            uint4 v[4];
#pragma unroll
            for (int it = 0; it < 4; it++) {
                const int idx = it * 32 + lane;
                v[it] = lds128(stg + (idx >> 1) * 32 + (idx & 1) * 16);
            }
#pragma unroll
            for (int it = 0; it < 4; it++) {
                const int idx = it * 32 + lane, dd = idx >> 1;
                *reinterpret_cast<uint4 *>(vt + (((size_t)b_first * ep.heads + head) * 64 + dd) * ep.tok_pitch + t0 +
                                           (idx & 1) * 8) = v[it];
            }
        } else {
#pragma unroll
            for (int hf = 0; hf < 2; hf++) {
                const int m = m0w + r + 8 * hf;
                if (m >= M) continue;
                const int b = m / rpb, t = m - b * rpb;
                __nv_bfloat16 *dst = vt + ((size_t)b * ep.heads + head) * 64 * ep.tok_pitch + t;
#pragma unroll
                for (int jj = 0; jj < 8; jj++)
#pragma unroll
                    for (int e = 0; e < 2; e++)
                        dst[(size_t)(8 * jj + 2 * c + e) * ep.tok_pitch] = __float2bfloat16(x[hf][2 * jj + e]);
            }
        }
    }
    warp_sync_smem();       // the staging buffer is rewritten by the next call
}

// One consumer warp drains its 16 rows x BN columns of the accumulator.
template <int BN, int MODE>
__device__ __forceinline__ void epilogue_tile(const GaGemmEpilogue &ep, uint32_t stg, const float (&acc)[BN / 2], int lane,
                                              int m0w, int n0, int M, int N)
{
    if (m0w >= M) return;                                          // warp-uniform: these rows are padding
    if constexpr (MODE == GA_EPI_HEADS) {
#pragma unroll
        for (int h = 0; h < BN / 64; h++)
            if (n0 + 64 * h < N) epilogue_head(ep, stg, acc, h, lane, m0w, n0 + 64 * h, M);
    } else {
#pragma unroll
        for (int ch = 0; ch < BN / 32; ch++) {
            if (n0 + 32 * ch >= N) break;                          // warp-uniform
            ColParams cp;
            load_col_params<MODE>(ep, lane, m0w, n0 + 32 * ch, N, cp);
            stage_chunk(stg, lane, acc, ch);
            warp_sync_smem();
            epilogue_chunk<MODE>(ep, stg, lane, m0w, n0 + 32 * ch, M, N, cp);
            warp_sync_smem();
        }
    }
}

// The epilogue type of gemm_sm90_kernel: the staged epilogue above.
template <int BN, int MODE> struct TnEpilogue {
    static constexpr bool kStaging = true;
    GaGemmEpilogue ep;
    __device__ __forceinline__ void operator()(const float (&acc)[BN / 2], uint32_t stg, int lane, int row0, int n0,
                                               int, int M, int N) const
    {
        epilogue_tile<BN, MODE>(ep, stg, acc, lane, row0, n0, M, N);
    }
};

// ---- host side -------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode()
{
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

}  // namespace

// 2-D bf16 row-major [rows, cols] tensor map with a {64 cols x box_rows} box, 128B swizzle.
int ga_make_tmap_bf16(CUtensorMap *map, const void *ptr, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                      uint32_t box_rows)
{
    EncodeTiledFn enc = get_encode();
    if (!enc) return GA_ERR_BADARG;
    if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (ld_elems * 2) % 16) return GA_ERR_BADARG;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {ld_elems * 2};
    cuuint32_t box[2] = {64, box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(ptr), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : 1000 + (int)r;
}

template <int BN>
static int launch_gemm(const void *A, int lda, const void *W, int ldw, const GaGemmEpilogue &ep, int M, int N, int K,
                       cudaStream_t s)
{
    CUtensorMap ta, tb;
    int rc = ga_make_tmap_bf16(&ta, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda, BM);
    if (rc) return rc;
    rc = ga_make_tmap_bf16(&tb, W, (uint64_t)N, (uint64_t)K, (uint64_t)ldw, (uint32_t)BN);
    if (rc) return rc;
    auto run = [&](auto epi) { return gemm_sm90_launch<BN, kMajorK, kMajorK, false>(ta, tb, epi, M, N, K, 1, s); };
    switch (ep.mode) {
    case GA_EPI_BF16: return run(TnEpilogue<BN, GA_EPI_BF16>{ep});
    case GA_EPI_GELU_BF16: return run(TnEpilogue<BN, GA_EPI_GELU_BF16>{ep});
    case GA_EPI_F32: return run(TnEpilogue<BN, GA_EPI_F32>{ep});
    case GA_EPI_RESID_GATE_F32: return run(TnEpilogue<BN, GA_EPI_RESID_GATE_F32>{ep});
    case GA_EPI_GEGLU_BF16: return run(TnEpilogue<BN, GA_EPI_GEGLU_BF16>{ep});
    case GA_EPI_HEADS:
        if constexpr (BN == 128 || BN == 256) return run(TnEpilogue<BN, GA_EPI_HEADS>{ep});
        else return GA_ERR_BADARG;
    case kEpiGeluKeepPre: return run(TnEpilogue<BN, kEpiGeluKeepPre>{ep});
    default: return GA_ERR_BADARG;
    }
}

// block_n = tile width {64, 128, 192, 256}
static int gemm_tn(const void *A, int lda, const void *W, int ldw, const GaGemmEpilogue &ep, int M, int N, int K,
                   int block_n, cudaStream_t s)
{
    if (block_n == 64) return launch_gemm<64>(A, lda, W, ldw, ep, M, N, K, s);
    if (block_n == 128) return launch_gemm<128>(A, lda, W, ldw, ep, M, N, K, s);
    if (block_n == 192) return launch_gemm<192>(A, lda, W, ldw, ep, M, N, K, s);
    return launch_gemm<256>(A, lda, W, ldw, ep, M, N, K, s);
}

static bool misaligned(const void *p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) != 0; }

// The rules of ga_b200.h, host only: every address and size the kernel derives from the arguments stays inside the
// buffers they describe and is aligned for the vector loads and stores it is used with.
extern "C" int ga_gemm_validate(const void *A, int lda, const void *W, int ldw, int M, int N, int K,
                                const GaGemmEpilogue *epi, int block_n)
{
    if (!A || !W || !epi || M <= 0 || N <= 0 || K <= 0) return GA_ERR_BADARG;
    // TMA operands: 16-byte base and row pitch; the pitch covers the K columns the tensor map describes
    if (misaligned(A, 16) || misaligned(W, 16) || lda % 8 || ldw % 8 || lda < K || ldw < K) return GA_ERR_BADARG;
    const int bn = block_n, mode = epi->mode;
    if (bn != 64 && bn != 128 && bn != 192 && bn != 256) return GA_ERR_BADARG;
    if (mode < GA_EPI_BF16 || mode > GA_EPI_GEGLU_BF16) return GA_ERR_BADARG;
    if (mode == GA_EPI_HEADS) {
        if (bn != 128 && bn != 256) return GA_ERR_BADARG;                   // the widths HEADS is instantiated for
        if (epi->heads <= 0 || epi->heads > N / 64 || N % (64 * epi->heads)) return GA_ERR_BADARG;
        if (epi->first_part != 0 && epi->first_part != 1) return GA_ERR_BADARG;
        const int parts = N / (64 * epi->heads);
        if (epi->first_part + parts > 3) return GA_ERR_BADARG;              // a fourth part would be written as V again
        void *const dst[3] = {epi->q, epi->k, epi->vt};
        for (int p = epi->first_part; p < epi->first_part + parts; p++)
            if (!dst[p] || misaligned(dst[p], 16)) return GA_ERR_BADARG;     // 16-byte token rows / Vt pieces
        if (epi->rows_per_batch < 1 || epi->tok_pitch < epi->rows_per_batch) return GA_ERR_BADARG;
        return 0;
    }
    if (!epi->out) return GA_ERR_BADARG;
    const bool f32 = mode == GA_EPI_F32 || mode == GA_EPI_RESID_GATE_F32;
    // float4 (fp32), 4 x bf16 (BF16, GELU) and 2 x bf16 (GEGLU) stores at row starts when ld_out % 4 == 0
    if (misaligned(epi->out, f32 ? 16 : (mode == GA_EPI_GEGLU_BF16 ? 4 : 8))) return GA_ERR_BADARG;
    if (mode == GA_EPI_GEGLU_BF16) {
        if (N % 2 || epi->ld_out < N / 2) return GA_ERR_BADARG;             // (x, gate) column pairs
    } else if (epi->ld_out < N) {
        return GA_ERR_BADARG;
    }
    if (mode == GA_EPI_RESID_GATE_F32 && epi->gate && (epi->rows_per_batch < 1 || epi->gate_ld < N))
        return GA_ERR_BADARG;
    return 0;
}

extern "C" int ga_gemm_bf16_tn(const void *A, int lda, const void *W, int ldw, int M, int N, int K,
                               const GaGemmEpilogue *epi, int block_n, void *stream)
{
    const int rc = ga_gemm_validate(A, lda, W, ldw, M, N, K, epi, block_n);
    if (rc) return rc;
    return gemm_tn(A, lda, W, ldw, *epi, M, N, K, block_n, (cudaStream_t)stream);
}

// fc1 of a FusedMLP for training (Part 13): the GEMM above with the kEpiGeluKeepPre epilogue.
extern "C" int ga_linear_fc1_gelu_bf16(const void *x, const void *w1, const float *b1, void *h, void *z, int M, int N,
                                       int K, int block_n, void *stream)
{
    const int rc = ga_linear_grad_validate(GA_LINEAR_FC1, x, w1, z, h, 0, M, N, K, block_n, nullptr, 0);
    if (rc) return rc;
    GaGemmEpilogue ep = {};
    ep.mode = kEpiGeluKeepPre;
    ep.bias = b1;
    ep.out = h;
    ep.ld_out = N;
    ep.q = z;
    return gemm_tn(x, K, w1, K, ep, M, N, K, block_n, (cudaStream_t)stream);
}
