// The library's TMA + wgmma GEMM main loop, shared by the forward GEMM of dit_gemm.cu (ga_gemm_bf16_tn and fc1 of
// the FusedMLP) and the linear-layer gradients of linear_grad.cu: out[M, N] = sum_k A[m, k] B[n, k], bf16 operands,
// fp32 accumulation in registers, and an epilogue type that drains the accumulator.
//
// Persistent kernel, one CTA per SM looping over 128 x BN output tiles (m fastest, then n), three warpgroups:
//   warpgroup 0   : TMA producer (one elected thread; cp.async.bulk.tensor into 128B-swizzled tiles)
//   warpgroups 1-2: consumers, 64 rows each: wgmma m64nBNk16 from shared memory into registers, then the epilogue
// smem ring of kStages {A 128x64, B BNx64} bf16 tiles with full/empty mbarriers.  The producer keeps filling the ring
// for the next tile while the consumers run the epilogue of this one.
//
// Each operand is K-major (rows of 64 along the contraction: one TMA box of 128 or BN rows) or MN-major (contiguous
// along M or N: two boxes {64 along M or N, 64 along K}).  An MN-major box is exactly the swizzle atom wgmma reads in
// its transposed operand mode (wgmma_desc_mn_sw128), so both majors go from global memory to the tensor cores with no
// shared-memory pass.
//
// With kSplit the contraction's 64-deep blocks are cut into `splits` consecutive ranges, and every (range, tile) is a
// work item of its own; the epilogue gets the range index.  Which CTA takes a work item does not change its result.
#pragma once
#include "../../include/ga_b200.h"
#include "device_once.cuh"
#include "sm90_ptx.cuh"

// 2-D bf16 row-major [rows, cols] tensor map with a {64 cols x box_rows} box, 128B swizzle (dit_gemm.cu).
int ga_make_tmap_bf16(CUtensorMap *map, const void *ptr, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                      uint32_t box_rows);

namespace gemm_sm90 {

using namespace sm90;

constexpr int BM = 128, BK = 64;
constexpr int kConsumerWarps = 8;
constexpr int kThreads = 128 + 32 * kConsumerWarps;      // producer warpgroup + 2 consumer warpgroups
constexpr int kHalf = 64 * BK * 2;                       // one 64-wide box of an MN-major operand: 8 KB
constexpr int kStageBytes = 2048;                        // epilogue staging per consumer warp: 16 rows x 128 B

enum Major { kMajorK = 0, kMajorMN = 1 };                // wgmma's imm-trans-a / imm-trans-b

template <int BN> struct GemmCfg {
    static constexpr int kABytes = BM * BK * 2;
    static constexpr int kBBytes = BN * BK * 2;
    static constexpr int kStages = (200 * 1024) / (kABytes + kBBytes) > 8 ? 8 : (200 * 1024) / (kABytes + kBBytes);
    static constexpr int kRing = kStages * (kABytes + kBBytes);
    // the ring, 1 KB to align it to 1024 B and, for an epilogue that stages, kStageBytes per consumer warp
    static constexpr int smem(bool staging) { return kRing + 1024 + (staging ? kConsumerWarps * kStageBytes : 0); }
};
static_assert(GemmCfg<128>::kStages == 6, "the gradients' 128 x 128 tiles run a 6-stage ring");

struct GemmTile { int m0, n0, kb0, kb1, split; };

template <int BN, bool kSplit>
__device__ __forceinline__ GemmTile gemm_tile(int tile, int num_m, int per_split, int nk, int splits)
{
    GemmTile t = {0, 0, 0, nk, 0};
    if constexpr (kSplit) {
        t.split = tile / per_split;
        tile -= t.split * per_split;
        t.kb0 = (int)((long long)t.split * nk / splits);
        t.kb1 = (int)((long long)(t.split + 1) * nk / splits);
    }
    t.m0 = (tile % num_m) * BM;
    t.n0 = (tile / num_m) * BN;
    return t;
}

// out is M x N and the contraction K long; splits: the number of contraction ranges with kSplit, else unused.
// Epi has kStaging, whether it uses a kStageBytes shared-memory buffer per consumer warp, and
//   epi(acc, staging, lane, row0, n0, split, M, N)
// called by every consumer warp once per tile for its 16 rows [row0, row0 + 16) and the columns [n0, n0 + BN), with
// acc the wgmma m64nBN accumulator fragment (acc[4 j + e]: row row0 + lane / 4 + 8 (e >> 1), column
// n0 + 8 j + 2 (lane % 4) + (e & 1)) and staging the warp's buffer (0 without kStaging).  Rows and columns of a tile
// past M and N hold zeros (TMA zero-fills out-of-bounds boxes); the epilogue must not write them.
template <int BN, Major kMajorA, Major kMajorB, bool kSplit, class Epi>
__global__ void __launch_bounds__(kThreads, 1)
gemm_sm90_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b, const Epi epi,
                 const int M, const int N, const int K, const int splits)
{
    static_assert(kMajorB == kMajorK || BN == 128, "an MN-major B tile is two 64-wide boxes");
    using Cfg = GemmCfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t full_bar[Cfg::kStages], empty_bar[Cfg::kStages];
    uint8_t *smem = align1024(smem_raw);
    uint8_t *smem_a = smem, *smem_b = smem + Cfg::kStages * Cfg::kABytes;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wg = threadIdx.x >> 7;
    const int nk = (K + BK - 1) / BK;
    const int num_m = (M + BM - 1) / BM, num_n = (N + BN - 1) / BN;
    const int per_split = num_m * num_n, tiles = kSplit ? per_split * splits : per_split;

    if (threadIdx.x == 0) {
        prefetch_tmap(&tma_a);
        prefetch_tmap(&tma_b);
        for (int s = 0; s < Cfg::kStages; s++) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerWarps); }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();                     // the operands and whatever the epilogue reads come from earlier kernels
    pdl_launch_dependents();        // let the next kernel run its own prologue under our main loop

    if (wg == 0) {
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one()) {
            int it = 0;
            for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
                const GemmTile t = gemm_tile<BN, kSplit>(tile, num_m, per_split, nk, splits);
                for (int kb = t.kb0; kb < t.kb1; kb++, it++) {
                    const int s = it % Cfg::kStages;
                    mbar_wait(&empty_bar[s], ((it / Cfg::kStages) & 1) ^ 1);     // every consumer warp released it
                    mbar_expect_tx(&full_bar[s], Cfg::kABytes + Cfg::kBBytes);
                    uint8_t *sa = smem_a + s * Cfg::kABytes, *sb = smem_b + s * Cfg::kBBytes;
                    if constexpr (kMajorA == kMajorK) {
                        tma_load_2d(sa, &tma_a, &full_bar[s], kb * BK, t.m0);
                    } else {
                        tma_load_2d(sa, &tma_a, &full_bar[s], t.m0, kb * BK);
                        tma_load_2d(sa + kHalf, &tma_a, &full_bar[s], t.m0 + 64, kb * BK);
                    }
                    if constexpr (kMajorB == kMajorK) {
                        tma_load_2d(sb, &tma_b, &full_bar[s], kb * BK, t.n0);
                    } else {
                        tma_load_2d(sb, &tma_b, &full_bar[s], t.n0, kb * BK);
                        tma_load_2d(sb + kHalf, &tma_b, &full_bar[s], t.n0 + 64, kb * BK);
                    }
                }
            }
        }
    } else {
        setmaxnreg_inc<232>();
        const int cw = wg - 1;                      // which 64-row half of the tile
        const int wi = warp & 3;                    // 16-row slice of that half
        const uint32_t stg = Epi::kStaging ? smem_u32(smem + Cfg::kRing + (cw * 4 + wi) * kStageBytes) : 0u;
        // k-steps of 16: 16 columns (32 B) of a K-major tile or 16 rows (2 KB) of an MN-major one
        constexpr uint64_t a_step = kMajorA == kMajorK ? 2 : 128, b_step = kMajorB == kMajorK ? 2 : 128;
        float acc[BN / 2];
        int it = 0;
        for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
            const GemmTile t = gemm_tile<BN, kSplit>(tile, num_m, per_split, nk, splits);
            for (int kb = t.kb0; kb < t.kb1; kb++, it++) {
                const int s = it % Cfg::kStages;
                mbar_wait(&full_bar[s], (it / Cfg::kStages) & 1);
                const uint32_t sa = smem_u32(smem_a + s * Cfg::kABytes + cw * kHalf);
                const uint32_t sb = smem_u32(smem_b + s * Cfg::kBBytes);
                const uint64_t ad = kMajorA == kMajorK ? wgmma_desc_k_sw128(sa) : wgmma_desc_mn_sw128(sa, kHalf);
                const uint64_t bd = kMajorB == kMajorK ? wgmma_desc_k_sw128(sb) : wgmma_desc_mn_sw128(sb, kHalf);
                fence_regs(acc);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / 16; k++)
                    wgmma_ss<BN, kMajorA, kMajorB>(acc, ad + a_step * k, bd + b_step * k, (uint32_t)((kb != t.kb0) | k));
                wgmma_commit();
                fence_regs(acc);
                wgmma_wait<1>();                    // the previous stage's MMAs have retired: release its slot
                fence_regs(acc);
                if (kb > t.kb0 && lane == 0) mbar_arrive(&empty_bar[(it - 1) % Cfg::kStages]);
            }
            wgmma_wait<0>();
            fence_regs(acc);
            if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % Cfg::kStages]);
            epi(acc, stg, lane, t.m0 + cw * 64 + wi * 16, t.n0, t.split, M, N);
        }
    }
}

// grid = min(#work items, #SMs); the tensor maps' boxes must match the majors: {64, 128} (A) or {64, BN} (B) when
// K-major, {64, 64} when MN-major.
template <int BN, Major kMajorA, Major kMajorB, bool kSplit, class Epi>
int gemm_sm90_launch(const CUtensorMap &ta, const CUtensorMap &tb, const Epi &epi, int M, int N, int K, int splits,
                     cudaStream_t s)
{
    constexpr int smem = GemmCfg<BN>::smem(Epi::kStaging);
    static GaPerDevice attr_set;
    if (ga_first_use_on_device(attr_set)) {
        cudaError_t e = cudaFuncSetAttribute(gemm_sm90_kernel<BN, kMajorA, kMajorB, kSplit, Epi>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return (int)e;
    }
    const long long tiles = (long long)((M + BM - 1) / BM) * ((N + BN - 1) / BN) * (kSplit ? splits : 1);
    const int sms = ga_sm_count();
    const int grid = tiles < sms ? (int)tiles : sms;
    return (int)ga_launch_pdl(gemm_sm90_kernel<BN, kMajorA, kMajorB, kSplit, Epi>, dim3(grid), dim3(kThreads),
                              (size_t)smem, s, ta, tb, epi, M, N, K, splits);
}

}  // namespace gemm_sm90
