// Linear-layer gradients on wgmma for training (include/ga_b200.h Part 13): for y = x W^T with x [M, K] and the
// nn.Linear weight W [N, K],
//   dgrad  out[M, K] = G[M, N] W[N, K]     (optionally fused with the GELU backward: dZ = bf16(v gelu'(Z)))
//   wgrad  dW[N, K]  = G^T x               (fp32, the parameter layout, split over M)
//   bias   db[N]     = column sums of G
// bf16 operands, fp32 accumulation in registers, no atomics.
//
// The GEMMs run the main loop of gemm_sm90.cuh at 128 x 128 tiles with this file's register-direct epilogue.  The
// operands that are contiguous along an output dimension ("MN-major": W in dgrad, both G and x in wgrad) are fed with
// wgmma's transposed operand mode on the TMA boxes as they land, so they reach the tensor cores with no shared-memory
// pass and the same pipeline as the forward.  attention_grad.cu builds transposed copies instead because it stages
// with cp.async through arbitrary strides and uses the same tiles as K-major operands of other products in the
// kernel; neither applies here.
//
// wgrad splits its contraction (the M rows) into S consecutive ranges of 64-row blocks so that small weights still
// fill the GPU (the SRT's 256 x 1024 weight has 16 output tiles); S depends on the shapes alone, so the bits do not
// depend on the card.  Each range writes an fp32 partial; a second kernel adds them in split order.
#include "../../include/ga_b200.h"
#include "gemm_sm90.cuh"
#include "row_common.cuh"

using namespace ga_row;
using namespace gemm_sm90;

namespace {

constexpr int BN = 128;                             // the one tile width of dgrad and wgrad
constexpr int kEpiBf16 = 0, kEpiF32 = 1, kEpiGeluBwd = 2;

constexpr int kColRows = 256;                       // bias gradient: rows per chunk
constexpr int kColWarps = 8;

struct GradArgs {
    void *out;                      // [M, N] (+ split * split_stride for wgrad partials)
    const __nv_bfloat16 *z;         // kEpiGeluBwd: fc1's pre-activation, bf16 [M, N]
    long long split_stride;         // elements between partials
};

// d/dz of z Phi(z): Phi(z) + z phi(z), fp32
__device__ __forceinline__ float gelu_grad(float z)
{
    const float cdf = 0.5f * (1.0f + erff(z * 0.70710678118654752f));
    const float pdf = 0.39894228040143268f * expf(-0.5f * z * z);
    return fmaf(z, pdf, cdf);
}

// Accumulator of wgmma m64n128 (warp w of the warpgroup, lane l): acc[4 j + e] is row 16 w + l / 4 + 8 (e >> 1),
// column 8 j + 2 (l % 4) + (e & 1).  Stored straight from registers as column pairs (N % 8 == 0, so a pair is
// either wholly inside or wholly outside).
template <int EPI>
__device__ __forceinline__ void epilogue(const GradArgs &a, const float (&acc)[64], int row0, int n0, long long split,
                                         int lane, int M, int N)
{
    const int r = lane >> 2, c = 2 * (lane & 3);
    // Z is read up front, all in flight at once: interleaved with the stores below the compiler must assume they
    // alias, and each element would wait for its own load
    uint32_t zr[2][BN / 8];
    if constexpr (EPI == kEpiGeluBwd) {
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
            const int row = row0 + r + 8 * hf;
#pragma unroll
            for (int j = 0; j < BN / 8; j++) {
                const int col = n0 + 8 * j + c;
                zr[hf][j] = (row < M && col < N)
                                ? __ldg(reinterpret_cast<const unsigned int *>(a.z + (size_t)row * N + col))
                                : 0u;
            }
        }
    }
#pragma unroll
    for (int hf = 0; hf < 2; hf++) {
        const int row = row0 + r + 8 * hf;
        if (row >= M) continue;
#pragma unroll
        for (int j = 0; j < BN / 8; j++) {
            const int col = n0 + 8 * j + c;
            if (col >= N) continue;
            const size_t idx = (size_t)row * N + col;
            const float v0 = acc[4 * j + 2 * hf], v1 = acc[4 * j + 2 * hf + 1];
            if constexpr (EPI == kEpiBf16) {
                *reinterpret_cast<uint32_t *>(reinterpret_cast<__nv_bfloat16 *>(a.out) + idx) = pack_bf16(v0, v1);
            } else if constexpr (EPI == kEpiF32) {
                *reinterpret_cast<float2 *>(reinterpret_cast<float *>(a.out) + split * a.split_stride + idx) =
                    make_float2(v0, v1);
            } else {
                const float2 zz = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&zr[hf][j]));
                *reinterpret_cast<uint32_t *>(reinterpret_cast<__nv_bfloat16 *>(a.out) + idx) =
                    pack_bf16(v0 * gelu_grad(zz.x), v1 * gelu_grad(zz.y));
            }
        }
    }
}

// The epilogue type of gemm_sm90_kernel: epilogue<EPI> straight from the registers, no staging.
template <int EPI> struct GradEpilogue : GradArgs {
    static constexpr bool kStaging = false;
    __device__ __forceinline__ void operator()(const float (&acc)[64], uint32_t, int lane, int row0, int n0, int split,
                                               int M, int N) const
    {
        epilogue<EPI>(*this, acc, row0, n0, split, lane, M, N);
    }
};

// Column sums of g bf16 [M, N], one block per (64 columns, chunk of kColRows rows): warp w adds rows w, w + 8, ...
// of the chunk in order, lane l columns 2 l, 2 l + 1; the warp sums are added in warp order into out[chunk, :].
__global__ void __launch_bounds__(32 * kColWarps)
colsum_chunk_kernel(const __nv_bfloat16 *__restrict__ g, float *__restrict__ out, int M, int N, int col_blocks)
{
    __shared__ float2 part[kColWarps][32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int chunk = blockIdx.x / col_blocks, cb = blockIdx.x - chunk * col_blocks;
    const int c = cb * 64 + 2 * lane;
    const long long r0 = (long long)chunk * kColRows, r1 = min((long long)M, r0 + kColRows);
    float2 s = make_float2(0.f, 0.f);
    if (c < N) {
#pragma unroll 4
        for (long long r = r0 + warp; r < r1; r += kColWarps) {
            const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(g + r * N + c));
            s.x += v.x;
            s.y += v.y;
        }
    }
    part[warp][lane] = s;
    __syncthreads();
    if (warp == 0 && c < N) {
        float2 t = part[0][lane];
#pragma unroll
        for (int w = 1; w < kColWarps; w++) { t.x += part[w][lane].x; t.y += part[w][lane].y; }
        *reinterpret_cast<float2 *>(out + (long long)chunk * N + c) = t;
    }
}

int wgrad_splits(int M, int N, int K)
{
    const long long tiles = (long long)((N + BM - 1) / BM) * ((K + BN - 1) / BN);
    const int nkb = (M + BK - 1) / BK;
    long long s = (256 + tiles - 1) / tiles;        // about 256 tiles in all
    if (s > nkb / 2) s = nkb / 2;                   // at least two 64-row blocks per split
    if (s > 32) s = 32;
    return s < 1 ? 1 : (int)s;
}

int col_chunks(int M) { return (M + kColRows - 1) / kColRows; }

}  // namespace

extern "C" int ga_linear_wgrad_splits(int M, int N, int K)
{
    if (M < 1 || N < 1 || K < 1) return 1;
    return wgrad_splits(M, N, K);
}

extern "C" size_t ga_linear_wgrad_workspace_bytes(int M, int N, int K)
{
    const int s = ga_linear_wgrad_splits(M, N, K);
    return s > 1 ? (size_t)s * (size_t)N * (size_t)K * sizeof(float) : 0;
}

extern "C" size_t ga_linear_bias_grad_workspace_bytes(int M, int N)
{
    if (M < 1 || N < 1) return 0;
    const int chunks = col_chunks(M);
    return chunks > 1 ? (size_t)chunks * (size_t)N * sizeof(float) : 0;
}

extern "C" int ga_linear_grad_validate(int op, const void *a, const void *b, const void *aux, const void *out,
                                       int out_f32, int M, int N, int K, int block_n, const void *workspace,
                                       size_t workspace_bytes)
{
    if (op < GA_LINEAR_FC1 || op > GA_LINEAR_BGRAD) return GA_ERR_BADARG;
    if (M < 1 || N < 8 || N % 8) return GA_ERR_BADARG;
    if (op != GA_LINEAR_BGRAD && (K < 8 || K % 8)) return GA_ERR_BADARG;
    const long long wide = (op == GA_LINEAR_BGRAD || N >= K) ? N : K;
    if ((long long)M * wide >= (1LL << 31)) return GA_ERR_BADARG;
    if (!a || mis16(a) || !out || mis16(out)) return GA_ERR_BADARG;
    size_t need = 0;
    switch (op) {
    case GA_LINEAR_FC1:
        if (!b || mis16(b) || !aux || mis16(aux) || out_f32 != 0) return GA_ERR_BADARG;
        if (block_n != 64 && block_n != 128 && block_n != 192 && block_n != 256) return GA_ERR_BADARG;
        return 0;
    case GA_LINEAR_DGRAD:
        if (!b || mis16(b) || (out_f32 != 0 && out_f32 != 1)) return GA_ERR_BADARG;
        if (aux && (mis16(aux) || out_f32)) return GA_ERR_BADARG;
        return 0;
    case GA_LINEAR_WGRAD:
        if (!b || mis16(b) || out_f32 != 1) return GA_ERR_BADARG;
        need = ga_linear_wgrad_workspace_bytes(M, N, K);
        break;
    default:
        if (out_f32 != 1) return GA_ERR_BADARG;
        need = ga_linear_bias_grad_workspace_bytes(M, N);
        break;
    }
    if (workspace_bytes < need || (need > 0 && (!workspace || mis16(workspace)))) return GA_ERR_BADARG;
    return 0;
}

extern "C" int ga_linear_dgrad_bf16(const void *g, const void *w, const void *z, void *out, int out_f32, int M, int N,
                                    int K, void *stream)
{
    int rc = ga_linear_grad_validate(GA_LINEAR_DGRAD, g, w, z, out, out_f32, M, N, K, 0, nullptr, 0);
    if (rc) return rc;
    CUtensorMap ta, tb;
    rc = ga_make_tmap_bf16(&ta, g, (uint64_t)M, (uint64_t)N, (uint64_t)N, BM);        // K-major: 128 rows
    if (rc) return rc;
    rc = ga_make_tmap_bf16(&tb, w, (uint64_t)N, (uint64_t)K, (uint64_t)K, BK);        // MN-major: 64 rows along N
    if (rc) return rc;
    const GradArgs a = {out, reinterpret_cast<const __nv_bfloat16 *>(z), 0};
    cudaStream_t s = (cudaStream_t)stream;
    auto run = [&](auto epi) { return gemm_sm90_launch<BN, kMajorK, kMajorMN, false>(ta, tb, epi, M, K, N, 1, s); };
    if (z) return run(GradEpilogue<kEpiGeluBwd>{a});
    if (out_f32) return run(GradEpilogue<kEpiF32>{a});
    return run(GradEpilogue<kEpiBf16>{a});
}

extern "C" int ga_linear_wgrad_bf16(const void *g, const void *x, float *dw, int M, int N, int K, void *workspace,
                                    size_t workspace_bytes, void *stream)
{
    int rc = ga_linear_grad_validate(GA_LINEAR_WGRAD, g, x, nullptr, dw, 1, M, N, K, 0, workspace, workspace_bytes);
    if (rc) return rc;
    CUtensorMap ta, tb;
    rc = ga_make_tmap_bf16(&ta, g, (uint64_t)M, (uint64_t)N, (uint64_t)N, BK);        // MN-major: 64 rows along M
    if (rc) return rc;
    rc = ga_make_tmap_bf16(&tb, x, (uint64_t)M, (uint64_t)K, (uint64_t)K, BK);
    if (rc) return rc;
    const int S = wgrad_splits(M, N, K);
    const GradEpilogue<kEpiF32> epi = {{S > 1 ? workspace : dw, nullptr, (long long)N * K}};
    cudaStream_t s = (cudaStream_t)stream;
    rc = gemm_sm90_launch<BN, kMajorMN, kMajorMN, true>(ta, tb, epi, N, K, M, S, s);
    if (rc || S == 1) return rc;
    return (int)ga_launch_partial_sum(reinterpret_cast<const float *>(workspace), dw, 1, S, (long long)N * K, s);
}

extern "C" int ga_linear_bias_grad_bf16(const void *g, float *db, int M, int N, void *workspace, size_t workspace_bytes,
                                        void *stream)
{
    const int rc = ga_linear_grad_validate(GA_LINEAR_BGRAD, g, nullptr, nullptr, db, 1, M, N, 0, 0, workspace,
                                           workspace_bytes);
    if (rc) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const int chunks = col_chunks(M), col_blocks = (N + 63) / 64;
    float *part = chunks > 1 ? reinterpret_cast<float *>(workspace) : db;
    colsum_chunk_kernel<<<(unsigned)((long long)chunks * col_blocks), 32 * kColWarps, 0, s>>>(
        reinterpret_cast<const __nv_bfloat16 *>(g), part, M, N, col_blocks);
    if (chunks == 1) return (int)cudaGetLastError();
    return (int)ga_launch_partial_sum(part, db, 1, chunks, N, s);
}
