// wgmma flash attention (head_dim 64, no mask, no dropout) for the DiT
// self- and cross-attention: softmax(q k^T / 8) v.  Replaces
// xformers.ops.memory_efficient_attention at
// /root/reference/vit/vision_transformer.py:297 and
// /root/reference/ldm/modules/attention.py:538-546.
//
// Inputs are the head-split tensors the QKV GEMM epilogue writes:
//   Q  [B*H, tok_pitch_q, 64]   K [B*H, tok_pitch_k, 64]   Vt [B*H, 64, tok_pitch_k]   (bf16)
// Output O [B, Nq, H*64] bf16 (token-major: the A operand of the out-projection GEMM).
//
// One CTA = 128 queries of one (batch, head); keys in blocks of 128:
//   warps 0-7 : two consumer warpgroups, 64 queries each.  S = Q K^T (wgmma m64n128k16, both operands from shared
//               memory) lands in registers; the softmax runs on that fragment (a query row lives in the 4 lanes of a
//               quad); P is re-packed to bf16 in registers and is the A operand of O += P V (wgmma m64n64k16 with A
//               from registers), so P never touches shared memory.  The next block's Q K^T is issued right behind
//               this block's P V and both run under one wait.
//   warp 8    : TMA producer (Q once, K and V double buffered).
#include "../../include/ga_b200.h"
#include "device_once.cuh"
#include "sm90_ptx.cuh"

using namespace sm90;

int ga_make_tmap_bf16(CUtensorMap *map, const void *ptr, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                      uint32_t box_rows);

namespace {

constexpr int AQ = 128, AK = 128, HD = 64;
constexpr int kQBytes = AQ * HD * 2;            // 16 KB
constexpr int kKBytes = AK * HD * 2;            // 16 KB per stage, 2 stages
constexpr int kVBytes = HD * AK * 2;            // 16 KB per stage (two 64-key sub-tiles of 8 KB), 2 stages
constexpr int kSmemAttn = kQBytes + 2 * kKBytes + 2 * kVBytes + 1024;
constexpr int kConsumerWarps = 8;
constexpr int kAttnThreads = 32 * kConsumerWarps + 32;

__device__ __forceinline__ uint32_t pack2(float a, float b)
{
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&h);
}
__device__ __forceinline__ float ex2_fast(float x)
{
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// kStatic: the caller supplies an upper bound of |q.k| * scale (available for free when q and k are
// RMS-normalised: |q.k| <= 64 max|w_q| max|w_k|).  exp2(s*scale - bound) then never overflows, so no running
// maximum and no rescaling of O are needed.  Mathematically identical to softmax (the constant cancels in O / l).
//
// Fragment layout (wgmma accumulator, thread = warp wi of its warpgroup, lane l, r = l/4, c = l%4):
//   s[4j + e]: query row 16 wi + r + 8 (e >> 1), key 8 j + 2 c + (e & 1)
// The bf16 A fragment of m64k16 for keys [16 kk, 16 kk + 16) is {s[8kk..8kk+1], s[8kk+2..3], s[8kk+4..5], s[8kk+6..7]}
// packed in pairs, i.e. the accumulator of Q K^T is already in the order P V needs.
template <bool kStatic>
__global__ void __launch_bounds__(kAttnThreads, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tma_q, const __grid_constant__ CUtensorMap tma_k,
                const __grid_constant__ CUtensorMap tma_vt, __nv_bfloat16 *__restrict__ out,
                const int Nq, const int Nk, const int pitch_q, const int pitch_k, const int heads,
                const float scale_log2, const float bound_log2)
{
    extern __shared__ uint8_t smem_raw[];
    __shared__ uint64_t q_full, k_full[2], k_empty[2], v_full[2], v_empty[2];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t *sQ = smem;
    uint8_t *sK = sQ + kQBytes;
    uint8_t *sV = sK + 2 * kKBytes;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int bh = blockIdx.y;
    const int q0 = blockIdx.x * AQ;
    const int nb = (Nk + AK - 1) / AK;

    if (threadIdx.x == 0) {
        prefetch_tmap(&tma_q); prefetch_tmap(&tma_k); prefetch_tmap(&tma_vt);
        mbar_init(&q_full, 1);
        for (int s = 0; s < 2; s++) {
            mbar_init(&k_full[s], 1); mbar_init(&k_empty[s], kConsumerWarps);
            mbar_init(&v_full[s], 1); mbar_init(&v_empty[s], kConsumerWarps);
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();
    pdl_launch_dependents();

    if (warp == kConsumerWarps) {
        if (elect_one()) {
            mbar_expect_tx(&q_full, kQBytes);
            tma_load_2d(sQ, &tma_q, &q_full, 0, bh * pitch_q + q0);
            for (int j = 0; j < nb; j++) {
                const int s = j & 1;
                const uint32_t ph = ((j >> 1) & 1) ^ 1;
                mbar_wait(&k_empty[s], ph);
                mbar_expect_tx(&k_full[s], kKBytes);
                tma_load_2d(sK + s * kKBytes, &tma_k, &k_full[s], 0, bh * pitch_k + j * AK);
                mbar_wait(&v_empty[s], ph);
                mbar_expect_tx(&v_full[s], kVBytes);
                tma_load_2d(sV + s * kVBytes, &tma_vt, &v_full[s], j * AK, bh * HD);
                tma_load_2d(sV + s * kVBytes + kVBytes / 2, &tma_vt, &v_full[s], j * AK + 64, bh * HD);
            }
        }
        return;
    }

    const int cw = warp >> 2, wi = warp & 3;
    const int r = lane >> 2, c = lane & 3;
    const uint64_t qd = wgmma_desc_k_sw128(smem_u32(sQ + cw * 64 * 128));
    float s_acc[AK / 2];
    float o_acc[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; i++) o_acc[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

    auto issue_s = [&](int j) {
        const int s = j & 1;
        mbar_wait(&k_full[s], (j >> 1) & 1);
        const uint64_t kd = wgmma_desc_k_sw128(smem_u32(sK + s * kKBytes));
        fence_regs(s_acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < HD / 16; k++) wgmma_ss<AK>(s_acc, qd + (uint64_t)(2 * k), kd + (uint64_t)(2 * k), (uint32_t)(k != 0));
        wgmma_commit();
    };

    mbar_wait(&q_full, 0);
    issue_s(0);
    wgmma_wait<0>();
    fence_regs(s_acc);
    if (lane == 0) mbar_arrive(&k_empty[0]);

    for (int j = 0; j < nb; j++) {
        const int kbase = j * AK;
        if (kbase + AK > Nk) {                                   // ragged last block only: mask the padding keys
#pragma unroll
            for (int i = 0; i < AK / 2; i++)
                if (kbase + 8 * (i >> 2) + 2 * c + (i & 1) >= Nk) s_acc[i] = -INFINITY;
        }
        float m_use[2];
        if constexpr (kStatic) {
            m_use[0] = m_use[1] = bound_log2;
        } else {
            float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int i = 0; i < AK / 2; i++) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s_acc[i]);
#pragma unroll
            for (int hf = 0; hf < 2; hf++) {
                mx[hf] = fmaxf(mx[hf], __shfl_xor_sync(0xffffffffu, mx[hf], 1));
                mx[hf] = fmaxf(mx[hf], __shfl_xor_sync(0xffffffffu, mx[hf], 2));
                const float m_new = fmaxf(m_run[hf], mx[hf] * scale_log2);
                const float corr = ex2_fast(m_run[hf] - m_new);
                m_run[hf] = m_new;
                m_use[hf] = m_new;
                l_run[hf] *= corr;
#pragma unroll
                for (int jj = 0; jj < HD / 8; jj++) {
                    o_acc[4 * jj + 2 * hf] *= corr;
                    o_acc[4 * jj + 2 * hf + 1] *= corr;
                }
            }
        }
        uint32_t pa[AK / 16][4];
#pragma unroll
        for (int i = 0; i < AK / 2; i += 2) {
            const int hf = (i >> 1) & 1;
            const float p0 = ex2_fast(fmaf(s_acc[i], scale_log2, -m_use[hf]));
            const float p1 = ex2_fast(fmaf(s_acc[i + 1], scale_log2, -m_use[hf]));
            l_run[hf] += p0 + p1;
            pa[i >> 3][(i >> 1) & 3] = pack2(p0, p1);
        }
        // O += P V_j, then (under the same wait) S = Q K_{j+1}^T
        const int sv = j & 1;
        mbar_wait(&v_full[sv], (j >> 1) & 1);
        const uint64_t vd = wgmma_desc_k_sw128(smem_u32(sV + sv * kVBytes));
        fence_regs(o_acc);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < AK / 16; kk++)
            wgmma_m64n64k16_rs(o_acc, pa[kk], vd + (uint64_t)((kk >> 2) * ((kVBytes / 2) >> 4) + 2 * (kk & 3)), 1u);
        wgmma_commit();
        if (j + 1 < nb) issue_s(j + 1);
        wgmma_wait<0>();
        fence_regs(o_acc);
        fence_regs(s_acc);
#pragma unroll
        for (int kk = 0; kk < AK / 16; kk++)
#pragma unroll
            for (int e = 0; e < 4; e++) asm volatile("" : "+r"(pa[kk][e])::"memory");    // live until P V retired
        if (lane == 0) {
            mbar_arrive(&v_empty[sv]);
            if (j + 1 < nb) mbar_arrive(&k_empty[(j + 1) & 1]);
        }
    }

    const int b = bh / heads, h = bh % heads;
#pragma unroll
    for (int hf = 0; hf < 2; hf++) {
        float l = l_run[hf];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        const float inv = 1.0f / l;
        const int q = q0 + cw * 64 + wi * 16 + r + 8 * hf;
        if (q < Nq) {
            __nv_bfloat16 *dst = out + ((size_t)b * Nq + q) * (size_t)(heads * HD) + h * HD + 2 * c;
#pragma unroll
            for (int jj = 0; jj < HD / 8; jj++)
                *reinterpret_cast<uint32_t *>(dst + 8 * jj) = pack2(o_acc[4 * jj + 2 * hf] * inv, o_acc[4 * jj + 2 * hf + 1] * inv);
        }
    }
}

}  // namespace

extern "C" int ga_attention_bf16(const void *Q, const void *K, const void *Vt, void *out, int batch, int heads,
                                 int Nq, int Nk, int pitch_q, int pitch_k, float softmax_scale, float score_bound,
                                 void *stream)
{
    if (!Q || !K || !Vt || !out || batch <= 0 || heads <= 0 || Nq <= 0 || Nk <= 0) return GA_ERR_BADARG;
    if (pitch_q < Nq || pitch_k < Nk || pitch_k % 128 != 0) return GA_ERR_BADARG;
    const uint64_t BH = (uint64_t)batch * heads;
    static GaPerDevice attr_set;
    if (ga_first_use_on_device(attr_set)) {
        cudaError_t e = cudaFuncSetAttribute(attn_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemAttn);
        if (e != cudaSuccess) return (int)e;
        e = cudaFuncSetAttribute(attn_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemAttn);
        if (e != cudaSuccess) return (int)e;
    }
    // static-bound softmax only while exp(-2*bound) stays far from the fp32/bf16 underflow range
    const bool use_static = score_bound > 0.f && score_bound <= 40.f;
    CUtensorMap tq, tk, tv;
    int rc = ga_make_tmap_bf16(&tq, Q, BH * pitch_q, HD, HD, AQ);
    if (rc) return rc;
    rc = ga_make_tmap_bf16(&tk, K, BH * pitch_k, HD, HD, AK);
    if (rc) return rc;
    rc = ga_make_tmap_bf16(&tv, Vt, BH * HD, (uint64_t)pitch_k, (uint64_t)pitch_k, HD);
    if (rc) return rc;
    dim3 grid((Nq + AQ - 1) / AQ, (unsigned)BH);
    const float log2e = 1.4426950408889634f;
    const float scale_log2 = softmax_scale * log2e;
    __nv_bfloat16 *o = reinterpret_cast<__nv_bfloat16 *>(out);
    cudaStream_t st = (cudaStream_t)stream;
    if (use_static)
        return (int)ga_launch_pdl(attn_fwd_kernel<true>, grid, dim3(kAttnThreads), (size_t)kSmemAttn, st, tq, tk, tv, o, Nq,
                                  Nk, pitch_q, pitch_k, heads, scale_log2, score_bound * log2e);
    return (int)ga_launch_pdl(attn_fwd_kernel<false>, grid, dim3(kAttnThreads), (size_t)kSmemAttn, st, tq, tk, tv, o, Nq, Nk,
                              pitch_q, pitch_k, heads, scale_log2, 0.0f);
}
