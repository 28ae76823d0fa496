// Differentiable attention for training: softmax(q k^T * scale) v with head dimension 64 (32 zero-padded, which is
// exact), its log-sum-exp, and the backward (include/ga_b200.h Part 12).  q, k, v, o, dO and the gradients are read
// and written where they lie: [batch, tokens, heads, d] with any 16-byte-multiple strides (views of a packed qkv
// tensor) or [batch, tokens, d]; nothing is packed.
//
// Tiled path (Nq > 16 or Nk > 16): one warpgroup per CTA, 64 rows per CTA, inner blocks of 64, wgmma m64n64k16
// (bf16 operands, fp32 accumulation).  Operands are staged with a two-stage cp.async ring into 128-byte-swizzled
// K-major tiles (rows zero-filled past the end of the sequence and past d); cp.async rather than TMA because the
// tensors arrive with arbitrary (batch, token, head) strides.  S-type products (both operands contracted along d) read
// both tiles from shared memory; the products that contract along tokens take P or dS from registers and the other
// operand from a K-major transposed copy built in shared memory (V^T, dO^T, Q^T, K^T):
//   attn_fwd_lse_kernel : one CTA per query block; running-max softmax; O and lse = ln sum_j exp(s_ij)
//   attn_delta_kernel   : Delta_i = sum_c dO_ic O_ic (fp32)
//   attn_dkdv_kernel    : one CTA per key block walks the query blocks: S^T = K Q^T, P^T = exp(S^T - lse),
//                         dV += P^T dO, dP^T = V dO^T, dS^T = P^T (dP^T - Delta), dK += dS^T Q (dV alone when dK is
//                         not wanted: no Delta, no dP, no dS)
//   attn_dq_kernel      : one CTA per query block walks the key blocks: S, P, dP = dO V^T, dS, dQ += dS K
// Each gradient element is owned by one CTA and summed in a fixed order: no atomics, the same inputs give the same
// bits.  The price is that S and P are formed twice in the backward (once per kernel) and dP twice.
//
// Short path (Nq <= 16 and Nk <= 16, the decoder up-samplers' 9-, 5- and 4-token sequences): one warp per
// (sequence, head) on CUDA cores, bf16 operands staged in shared memory, everything else fp32.
#include "../../include/ga_b200.h"
#include "device_once.cuh"
#include "row_common.cuh"
#include "sm90_ptx.cuh"

using namespace ga_row;
using namespace sm90;

namespace {

constexpr int BR = 64;                  // rows per CTA: queries (forward, dQ) or keys (dK/dV)
constexpr int BC = 64;                  // rows per inner block
constexpr int TB = 64 * 128;            // bytes of one 64 x 64 bf16 tile: 128-byte rows, 128-byte swizzle
constexpr int kThreads = 128;           // one warpgroup
constexpr int kSmemFwd = 6 * TB + 1024;                         // Q, 2 x (K, V), V^T
constexpr int kSmemDkdv = 8 * TB + 4 * BC * 4 + 1024;           // K, V, 2 x (Q, dO), Q^T, dO^T, 2 x (lse, Delta)
constexpr int kSmemDq = 7 * TB + 1024;                          // Q, dO, 2 x (K, V), K^T
constexpr int kShortMax = 16;
constexpr int kShortWarps = 4;
constexpr int SP = 66;                  // short path: bf16 row pitch (33 words, rows in distinct banks)
constexpr int kShortFwdWarpBytes = 3 * kShortMax * SP * 2 + kShortMax * (kShortMax + 1) * 4;
constexpr int kShortBwdWarpBytes = 5 * kShortMax * SP * 2 + 2 * kShortMax * (kShortMax + 1) * 4 + kShortMax * 4;
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

struct Tens {
    const __nv_bfloat16 *p;
    long long sb, sn, sh;               // element strides of batch, token, head; d is contiguous
};
struct OutTens {
    __nv_bfloat16 *p;
    long long sb, sn, sh;
};

struct AttnArgs {
    Tens q, k, v, o, dout;
    OutTens o_out, dq, dk, dv;
    const float *lse_in;
    float *lse_out, *delta;
    int heads, Nq, Nk, dqk, dvv, nqb, nkb;
    long long BH;
    float scale, scale_log2;
};

__device__ __forceinline__ long long head_off(long long bh, int heads, long long sb, long long sh)
{
    const long long b = bh / heads;
    return b * sb + (bh - b * heads) * sh;
}

// rows [n0, n0 + 64) x columns [0, 64) of one head into a swizzled tile; rows >= N and columns >= d are zeros
__device__ __forceinline__ void load_tile(uint8_t *s, const Tens &t, long long base, int n0, int N, int d)
{
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const int idx = threadIdx.x + kThreads * i, row = idx >> 3, ch = idx & 7;
        const bool ok = n0 + row < N && ch * 8 < d;
        cp_async16(smem_u32(s) + sw128_off(row, ch), ok ? t.p + base + (long long)(n0 + row) * t.sn + ch * 8 : t.p, ok);
    }
}

// dst[c][r] = src[r][c] for swizzled 64 x 64 tiles: the K-major copy of an operand whose contraction runs along its
// rows (V in P V, dO in P^T dO, q in dS^T q, k in dS k).  Thread: rows 2m, 2m + 1, one 16-byte piece; each store is
// one 32-bit word (columns 2m, 2m + 1 of a destination row), a warp's 32 words cover one 128-byte row.
__device__ __forceinline__ void transpose_tile(uint8_t *dst, const uint8_t *src)
{
#pragma unroll
    for (int i = 0; i < 2; i++) {
        const int idx = threadIdx.x + kThreads * i, r0 = 2 * (idx & 31), ch = idx >> 5;
        const uint4 va = *reinterpret_cast<const uint4 *>(src + sw128_off(r0, ch));
        const uint4 vb = *reinterpret_cast<const uint4 *>(src + sw128_off(r0 + 1, ch));
        const uint16_t *ea = reinterpret_cast<const uint16_t *>(&va), *eb = reinterpret_cast<const uint16_t *>(&vb);
#pragma unroll
        for (int e = 0; e < 8; e++)
            *reinterpret_cast<uint32_t *>(dst + sw128_off(8 * ch + e, r0 >> 3) + (r0 & 7) * 2) =
                (uint32_t)ea[e] | ((uint32_t)eb[e] << 16);
    }
}

// Accumulator layout of wgmma m64n64 (thread of warp w, lane l, r = l / 4, c = 2 (l % 4)): acc[4 j + e] is row
// 16 w + r + 8 (e >> 1), column 8 j + c + (e & 1).  Warp w owns rows [16 w, 16 w + 16) of the CTA's 64.
// acc (=, or += when accumulate) A B^T, A and B swizzled 64 x 64 tiles in shared memory (K = 64 along their rows)
__device__ __forceinline__ void wg_ss(float (&acc)[32], const uint8_t *A, const uint8_t *B, bool accumulate)
{
    const uint64_t ad = sm90::wgmma_desc_k_sw128(smem_u32(A)), bd = sm90::wgmma_desc_k_sw128(smem_u32(B));
#pragma unroll
    for (int kk = 0; kk < 4; kk++) sm90::wgmma_m64n64k16_ss(acc, ad + 2 * kk, bd + 2 * kk, (accumulate || kk) ? 1u : 0u);
}
// acc += A B^T, A the bf16 fragments of a 64 x 64 operand in registers (c_to_a), B a swizzled tile
__device__ __forceinline__ void wg_rs(float (&acc)[32], const uint32_t (&a)[4][4], const uint8_t *B)
{
    const uint64_t bd = sm90::wgmma_desc_k_sw128(smem_u32(B));
#pragma unroll
    for (int kk = 0; kk < 4; kk++) sm90::wgmma_m64n64k16_rs(acc, a[kk], bd + 2 * kk, 1u);
}
// the register A operands of wgmma are read asynchronously: keep them live until the wait that retires them
__device__ __forceinline__ void keep_live(uint32_t (&a)[4][4])
{
#pragma unroll
    for (int kk = 0; kk < 4; kk++)
#pragma unroll
        for (int e = 0; e < 4; e++) asm volatile("" : "+r"(a[kk][e])::"memory");
}
__device__ __forceinline__ void wg_begin() { sm90::wgmma_fence(); }
__device__ __forceinline__ void wg_end()
{
    sm90::wgmma_commit();
    sm90::wgmma_wait<0>();
}

// 64 x 64 fp32 accumulator as bf16 A fragments over its 64 columns (the wgmma m64k16 register operand order)
__device__ __forceinline__ void c_to_a(uint32_t (&a)[4][4], const float (&c)[32])
{
#pragma unroll
    for (int kk = 0; kk < 4; kk++) {
        a[kk][0] = pack_bf16(c[8 * kk + 0], c[8 * kk + 1]);
        a[kk][1] = pack_bf16(c[8 * kk + 2], c[8 * kk + 3]);
        a[kk][2] = pack_bf16(c[8 * kk + 4], c[8 * kk + 5]);
        a[kk][3] = pack_bf16(c[8 * kk + 6], c[8 * kk + 7]);
    }
}
__device__ __forceinline__ void zero(float (&c)[32])
{
#pragma unroll
    for (int i = 0; i < 32; i++) c[i] = 0.f;
}
// rows row0 + r and row0 + r + 8 of the warp's 16 rows times mul, columns < d, rows < N, as bf16
__device__ __forceinline__ void store_rows(const OutTens &t, long long base, int row0, int N, int d, const float (&c)[32],
                                           float mul)
{
    const int lane = threadIdx.x & 31, r = lane >> 2, cc = 2 * (lane & 3);
#pragma unroll
    for (int hf = 0; hf < 2; hf++) {
        const int row = row0 + r + 8 * hf;
        if (row >= N) continue;
        __nv_bfloat16 *dst = t.p + base + (long long)row * t.sn + cc;
#pragma unroll
        for (int j = 0; j < 8; j++)
            if (8 * j < d)
                *reinterpret_cast<uint32_t *>(dst + 8 * j) =
                    pack_bf16(c[4 * j + 2 * hf] * mul, c[4 * j + 2 * hf + 1] * mul);
    }
}
// cp.async groups up to the current block have landed (this thread's), made visible to wgmma (async proxy) and to
// every thread
__device__ __forceinline__ void tiles_ready()
{
    cp_async_wait<1>();
    fence_proxy_async();
    __syncthreads();
}
// shared-memory stores (the transposed tiles) made visible to wgmma and to every thread
__device__ __forceinline__ void stores_ready()
{
    fence_proxy_async();
    __syncthreads();
}

__global__ void __launch_bounds__(kThreads) attn_fwd_lse_kernel(const AttnArgs a)
{
    extern __shared__ uint8_t smem_raw[];
    uint8_t *sm = align1024(smem_raw);
    uint8_t *sQ = sm, *sK = sm + TB, *sV = sm + 3 * TB, *sVt = sm + 5 * TB;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = lane >> 2, cc = 2 * (lane & 3);
    const long long bh = blockIdx.x / a.nqb;
    const int q0 = (int)(blockIdx.x - bh * a.nqb) * BR;
    const long long bq = head_off(bh, a.heads, a.q.sb, a.q.sh), bk = head_off(bh, a.heads, a.k.sb, a.k.sh),
                    bv = head_off(bh, a.heads, a.v.sb, a.v.sh);

    load_tile(sQ, a.q, bq, q0, a.Nq, a.dqk);
    load_tile(sK, a.k, bk, 0, a.Nk, a.dqk);
    load_tile(sV, a.v, bv, 0, a.Nk, a.dvv);
    cp_async_commit();

    float o[32];
    zero(o);
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    for (int j = 0; j < a.nkb; j++) {
        if (j + 1 < a.nkb) {
            const int st = (j + 1) & 1;
            load_tile(sK + st * TB, a.k, bk, (j + 1) * BC, a.Nk, a.dqk);
            load_tile(sV + st * TB, a.v, bv, (j + 1) * BC, a.Nk, a.dvv);
        }
        cp_async_commit();
        tiles_ready();
        transpose_tile(sVt, sV + (j & 1) * TB);
        stores_ready();
        float s[32];
        zero(s);
        fence_regs(s);
        wg_begin();
        wg_ss(s, sQ, sK + (j & 1) * TB, false);                // S = Q K^T
        wg_end();
        fence_regs(s);
        const int kbase = j * BC;
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < 32; i++) {
            const float t = kbase + 8 * (i >> 2) + cc + (i & 1) < a.Nk ? s[i] * a.scale_log2 : -INFINITY;
            s[i] = t;
            mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], t);
        }
        float m_use[2];
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
            mx[hf] = fmaxf(mx[hf], __shfl_xor_sync(0xffffffffu, mx[hf], 1));
            mx[hf] = fmaxf(mx[hf], __shfl_xor_sync(0xffffffffu, mx[hf], 2));
            const float m_new = fmaxf(m_run[hf], mx[hf]);      // finite: every key block holds a real key
            const float corr = exp2f(m_run[hf] - m_new);
            m_run[hf] = m_use[hf] = m_new;
            l_run[hf] *= corr;
#pragma unroll
            for (int jt = 0; jt < 8; jt++) {
                o[4 * jt + 2 * hf] *= corr;
                o[4 * jt + 2 * hf + 1] *= corr;
            }
        }
#pragma unroll
        for (int i = 0; i < 32; i++) {
            const float p = exp2f(s[i] - m_use[(i >> 1) & 1]);
            s[i] = p;
            l_run[(i >> 1) & 1] += p;
        }
        uint32_t pa[4][4];
        c_to_a(pa, s);
        fence_regs(o);
        wg_begin();
        wg_rs(o, pa, sVt);                                     // O += P V
        wg_end();
        fence_regs(o);
        keep_live(pa);
        __syncthreads();
    }
    cp_async_wait<0>();

    float inv[2];
#pragma unroll
    for (int hf = 0; hf < 2; hf++) {
        float l = l_run[hf];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        inv[hf] = 1.f / l;
        const int q = q0 + 16 * warp + r + 8 * hf;
        if ((lane & 3) == 0 && q < a.Nq) a.lse_out[bh * a.Nq + q] = (m_run[hf] + log2f(l)) * kLn2;
    }
#pragma unroll
    for (int i = 0; i < 32; i++) o[i] *= inv[(i >> 1) & 1];
    store_rows(a.o_out, head_off(bh, a.heads, a.o_out.sb, a.o_out.sh), q0 + 16 * warp, a.Nq, a.dvv, o, 1.f);
}

// Delta[bh, q] = sum over c < dv of dO * O, in c order (fp32)
__global__ void __launch_bounds__(256) attn_delta_kernel(const AttnArgs a)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.BH * a.Nq) return;
    const long long bh = i / a.Nq;
    const int q = (int)(i - bh * a.Nq);
    const __nv_bfloat16 *o = a.o.p + head_off(bh, a.heads, a.o.sb, a.o.sh) + (long long)q * a.o.sn;
    const __nv_bfloat16 *g = a.dout.p + head_off(bh, a.heads, a.dout.sb, a.dout.sh) + (long long)q * a.dout.sn;
    float acc = 0.f;
    for (int c = 0; c < a.dvv; c += 8) {
        const uint4 ov = *reinterpret_cast<const uint4 *>(o + c), gv = *reinterpret_cast<const uint4 *>(g + c);
        const __nv_bfloat162 *o2 = reinterpret_cast<const __nv_bfloat162 *>(&ov);
        const __nv_bfloat162 *g2 = reinterpret_cast<const __nv_bfloat162 *>(&gv);
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const float2 of = __bfloat1622float2(o2[e]), gf = __bfloat1622float2(g2[e]);
            acc = fmaf(gf.x, of.x, acc);
            acc = fmaf(gf.y, of.y, acc);
        }
    }
    a.delta[i] = acc;
}

// lse (in log2 units) and, when with_delta, Delta of the query rows [q0, q0 + 64) into shared memory; 0 past Nq
__device__ __forceinline__ void load_rowstats(float *sl, float *sd, const AttnArgs &a, long long bh, int q0,
                                              bool with_delta)
{
    const int t = threadIdx.x;
    if (t < BC) {
        const int q = q0 + t;
        sl[t] = q < a.Nq ? a.lse_in[bh * a.Nq + q] * kLog2e : 0.f;
    } else if (with_delta) {
        const int q = q0 + t - BC;
        sd[t - BC] = q < a.Nq ? a.delta[bh * a.Nq + q] : 0.f;
    }
}

// kDK: form dS and dK as well as dV (false: a dV-only backward, P^T dO alone)
template <bool kDK>
__global__ void __launch_bounds__(kThreads) attn_dkdv_kernel(const AttnArgs a)
{
    extern __shared__ uint8_t smem_raw[];
    uint8_t *sm = align1024(smem_raw);
    uint8_t *sK = sm, *sV = sm + TB, *sQ = sm + 2 * TB, *sG = sm + 4 * TB, *sQt = sm + 6 * TB, *sGt = sm + 7 * TB;
    float *sL = reinterpret_cast<float *>(sm + 8 * TB), *sD = sL + 2 * BC;     // [2][64] each
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, cc = 2 * (lane & 3);
    const long long bh = blockIdx.x / a.nkb;
    const int k0 = (int)(blockIdx.x - bh * a.nkb) * BR;
    const long long bq = head_off(bh, a.heads, a.q.sb, a.q.sh), bk = head_off(bh, a.heads, a.k.sb, a.k.sh),
                    bv = head_off(bh, a.heads, a.v.sb, a.v.sh), bg = head_off(bh, a.heads, a.dout.sb, a.dout.sh);

    load_tile(sK, a.k, bk, k0, a.Nk, a.dqk);
    if (kDK) load_tile(sV, a.v, bv, k0, a.Nk, a.dvv);
    load_tile(sQ, a.q, bq, 0, a.Nq, a.dqk);
    load_tile(sG, a.dout, bg, 0, a.Nq, a.dvv);
    cp_async_commit();
    load_rowstats(sL, sD, a, bh, 0, kDK);

    float dk[32], dv[32];
    zero(dk);
    zero(dv);
    for (int i = 0; i < a.nqb; i++) {
        if (i + 1 < a.nqb) {
            const int st = (i + 1) & 1;
            load_tile(sQ + st * TB, a.q, bq, (i + 1) * BC, a.Nq, a.dqk);
            load_tile(sG + st * TB, a.dout, bg, (i + 1) * BC, a.Nq, a.dvv);
        }
        cp_async_commit();
        tiles_ready();
        if (i + 1 < a.nqb) load_rowstats(sL + ((i + 1) & 1) * BC, sD + ((i + 1) & 1) * BC, a, bh, (i + 1) * BC, kDK);
        const uint8_t *q_t = sQ + (i & 1) * TB, *g_t = sG + (i & 1) * TB;
        transpose_tile(sGt, g_t);
        if (kDK) transpose_tile(sQt, q_t);
        stores_ready();
        const float *lse = sL + (i & 1) * BC, *dlt = sD + (i & 1) * BC;
        const int qbase = i * BC;
        float p[32], ds[32];
        zero(p);
        zero(ds);
        fence_regs(p);
        fence_regs(ds);
        wg_begin();
        wg_ss(p, sK, q_t, false);                              // S^T = K Q^T
        if (kDK) wg_ss(ds, sV, g_t, false);                    // dP^T = V dO^T
        wg_end();
        fence_regs(p);
        fence_regs(ds);
        // P^T = exp(S^T scale - lse), zero for queries past Nq
#pragma unroll
        for (int e = 0; e < 32; e++) {
            const int qc = 8 * (e >> 2) + cc + (e & 1);
            p[e] = qbase + qc < a.Nq ? exp2f(fmaf(p[e], a.scale_log2, -lse[qc])) : 0.f;
        }
        uint32_t pa[4][4], da[4][4];
        c_to_a(pa, p);
        if (kDK) {
#pragma unroll
            for (int e = 0; e < 32; e++) ds[e] = p[e] * (ds[e] - dlt[8 * (e >> 2) + cc + (e & 1)]);
            c_to_a(da, ds);
        }
        fence_regs(dv);
        fence_regs(dk);
        wg_begin();
        wg_rs(dv, pa, sGt);                                    // dV += P^T dO
        if (kDK) wg_rs(dk, da, sQt);                           // dK += dS^T Q
        wg_end();
        fence_regs(dv);
        fence_regs(dk);
        keep_live(pa);
        if (kDK) keep_live(da);
        __syncthreads();
    }
    cp_async_wait<0>();
    if (kDK && a.dk.p)
        store_rows(a.dk, head_off(bh, a.heads, a.dk.sb, a.dk.sh), k0 + 16 * warp, a.Nk, a.dqk, dk, a.scale);
    if (a.dv.p) store_rows(a.dv, head_off(bh, a.heads, a.dv.sb, a.dv.sh), k0 + 16 * warp, a.Nk, a.dvv, dv, 1.f);
}

__global__ void __launch_bounds__(kThreads) attn_dq_kernel(const AttnArgs a)
{
    extern __shared__ uint8_t smem_raw[];
    uint8_t *sm = align1024(smem_raw);
    uint8_t *sQ = sm, *sG = sm + TB, *sK = sm + 2 * TB, *sV = sm + 4 * TB, *sKt = sm + 6 * TB;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = lane >> 2, cc = 2 * (lane & 3);
    const long long bh = blockIdx.x / a.nqb;
    const int q0 = (int)(blockIdx.x - bh * a.nqb) * BR;
    const long long bq = head_off(bh, a.heads, a.q.sb, a.q.sh), bk = head_off(bh, a.heads, a.k.sb, a.k.sh),
                    bv = head_off(bh, a.heads, a.v.sb, a.v.sh), bg = head_off(bh, a.heads, a.dout.sb, a.dout.sh);

    load_tile(sQ, a.q, bq, q0, a.Nq, a.dqk);
    load_tile(sG, a.dout, bg, q0, a.Nq, a.dvv);
    load_tile(sK, a.k, bk, 0, a.Nk, a.dqk);
    load_tile(sV, a.v, bv, 0, a.Nk, a.dvv);
    cp_async_commit();

    float lse[2], dlt[2];
#pragma unroll
    for (int hf = 0; hf < 2; hf++) {
        const int q = q0 + 16 * warp + r + 8 * hf;
        lse[hf] = q < a.Nq ? a.lse_in[bh * a.Nq + q] * kLog2e : 0.f;
        dlt[hf] = q < a.Nq ? a.delta[bh * a.Nq + q] : 0.f;
    }
    float dq[32];
    zero(dq);
    for (int j = 0; j < a.nkb; j++) {
        if (j + 1 < a.nkb) {
            const int st = (j + 1) & 1;
            load_tile(sK + st * TB, a.k, bk, (j + 1) * BC, a.Nk, a.dqk);
            load_tile(sV + st * TB, a.v, bv, (j + 1) * BC, a.Nk, a.dvv);
        }
        cp_async_commit();
        tiles_ready();
        const uint8_t *k_t = sK + (j & 1) * TB, *v_t = sV + (j & 1) * TB;
        transpose_tile(sKt, k_t);
        stores_ready();
        const int kbase = j * BC;
        float p[32], ds[32];
        zero(p);
        zero(ds);
        fence_regs(p);
        fence_regs(ds);
        wg_begin();
        wg_ss(p, sQ, k_t, false);                              // S = Q K^T
        wg_ss(ds, sG, v_t, false);                             // dP = dO V^T
        wg_end();
        fence_regs(p);
        fence_regs(ds);
#pragma unroll
        for (int e = 0; e < 32; e++) {
            const float pe = kbase + 8 * (e >> 2) + cc + (e & 1) < a.Nk
                                 ? exp2f(fmaf(p[e], a.scale_log2, -lse[(e >> 1) & 1])) : 0.f;
            ds[e] = pe * (ds[e] - dlt[(e >> 1) & 1]);
        }
        uint32_t da[4][4];
        c_to_a(da, ds);
        fence_regs(dq);
        wg_begin();
        wg_rs(dq, da, sKt);                                    // dQ += dS K
        wg_end();
        fence_regs(dq);
        keep_live(da);
        __syncthreads();
    }
    cp_async_wait<0>();
    store_rows(a.dq, head_off(bh, a.heads, a.dq.sb, a.dq.sh), q0 + 16 * warp, a.Nq, a.dqk, dq, a.scale);
}

// ---- short path: one warp per (sequence, head), Nq, Nk <= 16 ----
// rows [0, N) x columns [0, 64) of one head as bf16 pairs (zero past d) into a [16][SP] shared array
__device__ __forceinline__ void short_load(__nv_bfloat16 *s, const Tens &t, long long base, int N, int d, int lane)
{
    for (int idx = lane; idx < N * 32; idx += 32) {
        const int row = idx >> 5, c = 2 * (idx & 31);
        __nv_bfloat162 v = __floats2bfloat162_rn(0.f, 0.f);
        if (c < d) v = *reinterpret_cast<const __nv_bfloat162 *>(t.p + base + (long long)row * t.sn + c);
        *reinterpret_cast<__nv_bfloat162 *>(s + row * SP + c) = v;
    }
}
// sum over c < 64 of x[i][c] y[j][c], pairs in c order
__device__ __forceinline__ float short_dot(const __nv_bfloat16 *x, const __nv_bfloat16 *y)
{
    float acc = 0.f;
#pragma unroll 8
    for (int c = 0; c < 64; c += 2) {
        const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(x + c));
        const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(y + c));
        acc = fmaf(a.x, b.x, acc);
        acc = fmaf(a.y, b.y, acc);
    }
    return acc;
}
// out[row][c..c+1] = mul * sum over m < M of w[m][row] (w_row_major ? w[row][m]) * x[m][c..c+1], rows < N, c < d
__device__ __forceinline__ void short_combine(const OutTens &t, long long base, int N, int M, int d, const float *w,
                                              bool w_by_row, const __nv_bfloat16 *x, float mul, int lane)
{
    const int half = d >> 1;
    for (int idx = lane; idx < N * half; idx += 32) {
        const int row = idx / half, c = 2 * (idx - row * half);
        float a0 = 0.f, a1 = 0.f;
        for (int m = 0; m < M; m++) {
            const float wm = w_by_row ? w[row * (kShortMax + 1) + m] : w[m * (kShortMax + 1) + row];
            const float2 xv = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(x + m * SP + c));
            a0 = fmaf(wm, xv.x, a0);
            a1 = fmaf(wm, xv.y, a1);
        }
        *reinterpret_cast<__nv_bfloat162 *>(t.p + base + (long long)row * t.sn + c) = __floats2bfloat162_rn(a0 * mul, a1 * mul);
    }
}

__global__ void __launch_bounds__(32 * kShortWarps) attn_short_fwd_kernel(const AttnArgs a)
{
    extern __shared__ __align__(16) uint8_t short_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long bh = (long long)blockIdx.x * kShortWarps + warp;
    if (bh >= a.BH) return;
    uint8_t *base = short_smem + warp * kShortFwdWarpBytes;
    __nv_bfloat16 *sq = reinterpret_cast<__nv_bfloat16 *>(base), *sk = sq + kShortMax * SP, *sv = sk + kShortMax * SP;
    float *sp = reinterpret_cast<float *>(sv + kShortMax * SP);
    short_load(sq, a.q, head_off(bh, a.heads, a.q.sb, a.q.sh), a.Nq, a.dqk, lane);
    short_load(sk, a.k, head_off(bh, a.heads, a.k.sb, a.k.sh), a.Nk, a.dqk, lane);
    short_load(sv, a.v, head_off(bh, a.heads, a.v.sb, a.v.sh), a.Nk, a.dvv, lane);
    __syncwarp();
    for (int idx = lane; idx < a.Nq * a.Nk; idx += 32) {
        const int i = idx / a.Nk, j = idx - i * a.Nk;
        sp[i * (kShortMax + 1) + j] = short_dot(sq + i * SP, sk + j * SP) * a.scale;
    }
    __syncwarp();
    if (lane < a.Nq) {
        float *row = sp + lane * (kShortMax + 1);
        float m = -INFINITY;
        for (int j = 0; j < a.Nk; j++) m = fmaxf(m, row[j]);
        float l = 0.f;
        for (int j = 0; j < a.Nk; j++) {
            row[j] = expf(row[j] - m);
            l += row[j];
        }
        const float inv = 1.f / l;
        for (int j = 0; j < a.Nk; j++) row[j] *= inv;
        a.lse_out[bh * a.Nq + lane] = m + logf(l);
    }
    __syncwarp();
    short_combine(a.o_out, head_off(bh, a.heads, a.o_out.sb, a.o_out.sh), a.Nq, a.Nk, a.dvv, sp, true, sv, 1.f, lane);
}

__global__ void __launch_bounds__(32 * kShortWarps) attn_short_bwd_kernel(const AttnArgs a)
{
    extern __shared__ __align__(16) uint8_t short_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long bh = (long long)blockIdx.x * kShortWarps + warp;
    if (bh >= a.BH) return;
    uint8_t *base = short_smem + warp * kShortBwdWarpBytes;
    __nv_bfloat16 *sq = reinterpret_cast<__nv_bfloat16 *>(base), *sk = sq + kShortMax * SP, *sv = sk + kShortMax * SP,
                  *sg = sv + kShortMax * SP, *so = sg + kShortMax * SP;
    float *sp = reinterpret_cast<float *>(so + kShortMax * SP), *sds = sp + kShortMax * (kShortMax + 1),
          *sdl = sds + kShortMax * (kShortMax + 1);
    short_load(sq, a.q, head_off(bh, a.heads, a.q.sb, a.q.sh), a.Nq, a.dqk, lane);
    short_load(sk, a.k, head_off(bh, a.heads, a.k.sb, a.k.sh), a.Nk, a.dqk, lane);
    short_load(sv, a.v, head_off(bh, a.heads, a.v.sb, a.v.sh), a.Nk, a.dvv, lane);
    short_load(sg, a.dout, head_off(bh, a.heads, a.dout.sb, a.dout.sh), a.Nq, a.dvv, lane);
    short_load(so, a.o, head_off(bh, a.heads, a.o.sb, a.o.sh), a.Nq, a.dvv, lane);
    __syncwarp();
    if (lane < a.Nq) sdl[lane] = short_dot(sg + lane * SP, so + lane * SP);
    for (int idx = lane; idx < a.Nq * a.Nk; idx += 32) {
        const int i = idx / a.Nk, j = idx - i * a.Nk;
        sp[i * (kShortMax + 1) + j] = expf(short_dot(sq + i * SP, sk + j * SP) * a.scale - a.lse_in[bh * a.Nq + i]);
    }
    __syncwarp();
    for (int idx = lane; idx < a.Nq * a.Nk; idx += 32) {
        const int i = idx / a.Nk, j = idx - i * a.Nk;
        const float p = sp[i * (kShortMax + 1) + j];
        sds[i * (kShortMax + 1) + j] = p * (short_dot(sg + i * SP, sv + j * SP) - sdl[i]);
    }
    __syncwarp();
    if (a.dv.p)
        short_combine(a.dv, head_off(bh, a.heads, a.dv.sb, a.dv.sh), a.Nk, a.Nq, a.dvv, sp, false, sg, 1.f, lane);
    if (a.dk.p)
        short_combine(a.dk, head_off(bh, a.heads, a.dk.sb, a.dk.sh), a.Nk, a.Nq, a.dqk, sds, false, sq, a.scale, lane);
    if (a.dq.p)
        short_combine(a.dq, head_off(bh, a.heads, a.dq.sb, a.dq.sh), a.Nq, a.Nk, a.dqk, sds, true, sk, a.scale, lane);
}

Tens in_tens(const void *p, const int64_t *s) { return Tens{reinterpret_cast<const __nv_bfloat16 *>(p), s[0], s[1], s[2]}; }
OutTens out_tens(const void *p, const int64_t *s) { return OutTens{reinterpret_cast<__nv_bfloat16 *>(const_cast<void *>(p)), s[0], s[1], s[2]}; }

AttnArgs make_args(const void *q, const void *k, const void *v, const void *o, const void *dout, const int64_t *strides,
                   int batch, int heads, int Nq, int Nk, int d_qk, int d_v, float scale)
{
    AttnArgs a{};
    a.q = in_tens(q, strides);
    a.k = in_tens(k, strides + 3);
    a.v = in_tens(v, strides + 6);
    a.o = in_tens(o, strides + 9);
    a.o_out = out_tens(o, strides + 9);
    if (dout) a.dout = in_tens(dout, strides + 12);
    a.heads = heads;
    a.Nq = Nq;
    a.Nk = Nk;
    a.dqk = d_qk;
    a.dvv = d_v;
    a.nqb = (Nq + BR - 1) / BR;
    a.nkb = (Nk + BR - 1) / BR;
    a.BH = (long long)batch * heads;
    a.scale = scale;
    a.scale_log2 = scale * kLog2e;
    return a;
}

bool is_short(int Nq, int Nk) { return Nq <= kShortMax && Nk <= kShortMax; }

int set_smem_attrs()
{
    static GaPerDevice attr_set;
    if (!ga_first_use_on_device(attr_set)) return 0;
    const struct { const void *f; int bytes; } k[] = {
        {(const void *)attn_fwd_lse_kernel, kSmemFwd},
        {(const void *)attn_dkdv_kernel<true>, kSmemDkdv},
        {(const void *)attn_dkdv_kernel<false>, kSmemDkdv},
        {(const void *)attn_dq_kernel, kSmemDq},
        {(const void *)attn_short_fwd_kernel, kShortWarps * kShortFwdWarpBytes},
        {(const void *)attn_short_bwd_kernel, kShortWarps * kShortBwdWarpBytes},
    };
    for (const auto &e : k) {
        const cudaError_t err = cudaFuncSetAttribute(e.f, cudaFuncAttributeMaxDynamicSharedMemorySize, e.bytes);
        if (err != cudaSuccess) return (int)err;
    }
    return 0;
}

}  // namespace

extern "C" int ga_attention_grad_validate(const void *q, const void *k, const void *v, const void *o, const float *lse,
                                          const void *dout, const float *delta, const void *dq, const void *dk,
                                          const void *dv, int batch, int heads, int Nq, int Nk, int d_qk, int d_v,
                                          const int64_t *strides, int backward)
{
    if (!q || !k || !v || !o || !lse || !strides || batch <= 0 || heads <= 0 || Nq <= 0 || Nk <= 0) return GA_ERR_BADARG;
    if ((d_qk != 32 && d_qk != 64) || (d_v != 32 && d_v != 64)) return GA_ERR_BADARG;
    if (backward && (!dout || !delta)) return GA_ERR_BADARG;
    const auto misaligned = [](const void *p, uintptr_t b) { return (reinterpret_cast<uintptr_t>(p) & (b - 1)) != 0; };
    const void *t[8] = {q, k, v, o, backward ? dout : nullptr, backward ? dq : nullptr, backward ? dk : nullptr,
                        backward ? dv : nullptr};
    for (int i = 0; i < 8; i++) {
        if (!t[i]) continue;
        if (misaligned(t[i], 16)) return GA_ERR_BADARG;             // 16-byte row pieces (cp.async, vector loads)
        for (int j = 0; j < 3; j++)
            if (strides[3 * i + j] < 0 || strides[3 * i + j] % 8 != 0) return GA_ERR_BADARG;
        // outputs (o, dq, dk, dv): a zero stride on a dimension of size > 1 would make CTAs write the same elements
        const bool output = i == 3 || i >= 5;
        const int64_t extent[3] = {batch, (i == 1 || i == 2 || i == 6 || i == 7) ? Nk : Nq, heads};
        for (int j = 0; output && j < 3; j++)
            if (strides[3 * i + j] == 0 && extent[j] > 1) return GA_ERR_BADARG;
    }
    if (misaligned(lse, 4) || (backward && misaligned(delta, 4))) return GA_ERR_BADARG;
    const int64_t BH = (int64_t)batch * heads;
    const int64_t blocks = is_short(Nq, Nk) ? (BH + kShortWarps - 1) / kShortWarps
                                            : BH * (((Nq > Nk ? Nq : Nk) + BR - 1) / BR);
    if (blocks > 0x7fffffff) return GA_ERR_SIZE;                      // one-dimensional grid
    return 0;
}

extern "C" int ga_attention_fwd_lse_bf16(const void *q, const void *k, const void *v, void *o, float *lse, int batch,
                                         int heads, int Nq, int Nk, int d_qk, int d_v, const int64_t *strides,
                                         float scale, void *stream)
{
    int rc = ga_attention_grad_validate(q, k, v, o, lse, nullptr, nullptr, nullptr, nullptr, nullptr, batch, heads, Nq,
                                        Nk, d_qk, d_v, strides, 0);
    if (rc) return rc;
    if ((rc = set_smem_attrs())) return rc;
    AttnArgs a = make_args(q, k, v, o, nullptr, strides, batch, heads, Nq, Nk, d_qk, d_v, scale);
    a.lse_out = lse;
    cudaStream_t st = (cudaStream_t)stream;
    if (is_short(Nq, Nk))
        attn_short_fwd_kernel<<<(unsigned)((a.BH + kShortWarps - 1) / kShortWarps), 32 * kShortWarps,
                                kShortWarps * kShortFwdWarpBytes, st>>>(a);
    else
        attn_fwd_lse_kernel<<<(unsigned)(a.BH * a.nqb), kThreads, kSmemFwd, st>>>(a);
    return (int)cudaGetLastError();
}

extern "C" int ga_attention_bwd_bf16(const void *q, const void *k, const void *v, const void *o, const float *lse,
                                     const void *dout, float *delta, void *dq, void *dk, void *dv, int batch, int heads,
                                     int Nq, int Nk, int d_qk, int d_v, const int64_t *strides, float scale,
                                     void *stream)
{
    int rc = ga_attention_grad_validate(q, k, v, o, lse, dout, delta, dq, dk, dv, batch, heads, Nq, Nk, d_qk, d_v,
                                        strides, 1);
    if (rc) return rc;
    if ((rc = set_smem_attrs())) return rc;
    AttnArgs a = make_args(q, k, v, o, dout, strides, batch, heads, Nq, Nk, d_qk, d_v, scale);
    a.lse_in = lse;
    a.delta = delta;
    a.dq = out_tens(dq, strides + 15);
    a.dk = out_tens(dk, strides + 18);
    a.dv = out_tens(dv, strides + 21);
    cudaStream_t st = (cudaStream_t)stream;
    if (is_short(Nq, Nk)) {
        if (dq || dk || dv)
            attn_short_bwd_kernel<<<(unsigned)((a.BH + kShortWarps - 1) / kShortWarps), 32 * kShortWarps,
                                    kShortWarps * kShortBwdWarpBytes, st>>>(a);
        return (int)cudaGetLastError();
    }
    // Delta and dS serve dK and dQ only: a dV-only backward forms P^T dO and nothing else
    if (dk || dq) attn_delta_kernel<<<(unsigned)((a.BH * Nq + 255) / 256), 256, 0, st>>>(a);
    if (dk) attn_dkdv_kernel<true><<<(unsigned)(a.BH * a.nkb), kThreads, kSmemDkdv, st>>>(a);
    else if (dv) attn_dkdv_kernel<false><<<(unsigned)(a.BH * a.nkb), kThreads, kSmemDkdv, st>>>(a);
    if (dq) attn_dq_kernel<<<(unsigned)(a.BH * a.nqb), kThreads, kSmemDq, st>>>(a);
    return (int)cudaGetLastError();
}
