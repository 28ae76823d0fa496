// Row-wise kernels of the VAE decode path latent tokens -> surfels (SURVEY.md 8f row N1): everything
// around the wgmma GEMMs / attention that the DiT kernels do not already cover.
//   layernorm_modulate : LayerNorm [* w + b] [* (1 + scale[row]) + shift[row]] -> bf16      (DiTBlock2, PreNorm)
//   thin_linear        : [LayerNorm affine] [SiLU] x . W^T + b with <= 16 outputs              (conv_sr, residual heads)
//   micro_attention    : qk-normed attention over sequences of <= 16 tokens, one warp per (sequence, head)
//   micro_seq_build    : [parent token ; f learned queries] sequences of the cascaded up-samplers
//   surfel_cascade_pack: residual + parent pre-activation -> activations -> packed [R, 13] surfels
// Math follows /root/reference/vit/vit_triplane.py:287-345,991-1064,1289-1313,1388-1440,
// /root/reference/dit/dit_decoder.py:15-42, /root/reference/nsr/srt/layers.py:82-90,146-186 and
// /root/reference/vit/vision_transformer.py:215-303; the checker is oracle/vae_decoder_oracle.py.
#include "../../include/ga_b200.h"
#include "device_once.cuh"
#include "row_common.cuh"

using namespace ga_row;

namespace {

// Warp sums of N values at once (N a power of two <= 32): at every butterfly step a lane keeps one half of its values
// and hands the other half to its partner, so N totals cost N - 1 + log2(32 / N) shuffles instead of 5 N.  Lane l ends
// up with the total of value index (l >> log2(32 / N)) & (N - 1); the additions are the ones the plain butterfly makes,
// in the same order, so the totals are bit-identical to warp_sum().
template <int N>
__device__ __forceinline__ float packed_wsum(float (&v)[N], int lane)
{
    int n = N, o = 16;
#pragma unroll
    for (; n > 1; n >>= 1, o >>= 1) {
        const bool upper = (lane & o) != 0;
#pragma unroll
        for (int m = 0; m < n / 2; m++) {
            const float keep = upper ? v[m + n / 2] : v[m], send = upper ? v[m] : v[m + n / 2];
            v[m] = keep + __shfl_xor_sync(0xffffffffu, send, o);
        }
    }
#pragma unroll
    for (; o > 0; o >>= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
    return v[0];
}

// one warp per row, row cached in registers (D % 4 == 0, D <= 1024)
__global__ void __launch_bounds__(256)
layernorm_modulate_kernel(const float *__restrict__ x, const float *__restrict__ w, const float *__restrict__ bias,
                          const float *__restrict__ shift, const float *__restrict__ scale, int mod_ld,
                          int rows_per_batch, __nv_bfloat16 *__restrict__ out, int R, int D, float eps)
{
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= R) return;
    const float4 *x4 = reinterpret_cast<const float4 *>(x + (size_t)r * D);
    const int n4 = D >> 2;
    float4 c[8];
    float s = 0.f;
#pragma unroll
    for (int u = 0; u < 8; u++) {
        const int i = lane + 32 * u;
        c[u] = i < n4 ? x4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        s += (c[u].x + c[u].y) + (c[u].z + c[u].w);
    }
    const float mean = warp_sum(s) / (float)D;
    float v = 0.f;
#pragma unroll
    for (int u = 0; u < 8; u++) {
        if (lane + 32 * u < n4) {
            const float d0 = c[u].x - mean, d1 = c[u].y - mean, d2 = c[u].z - mean, d3 = c[u].w - mean;
            v += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
        }
    }
    const float rs = rsqrtf(warp_sum(v) / (float)D + eps);
    const int b = r / rows_per_batch;
    const float4 *w4 = reinterpret_cast<const float4 *>(w), *b4 = reinterpret_cast<const float4 *>(bias);
    const float4 *sh4 = shift ? reinterpret_cast<const float4 *>(shift + (size_t)b * mod_ld) : nullptr;
    const float4 *sc4 = scale ? reinterpret_cast<const float4 *>(scale + (size_t)b * mod_ld) : nullptr;
    uint2 *o = reinterpret_cast<uint2 *>(out + (size_t)r * D);
#pragma unroll
    for (int u = 0; u < 8; u++) {
        const int i = lane + 32 * u;
        if (i < n4) {
            float4 y = make_float4((c[u].x - mean) * rs, (c[u].y - mean) * rs, (c[u].z - mean) * rs, (c[u].w - mean) * rs);
            if (w) {
                const float4 ww = __ldg(w4 + i);
                y.x *= ww.x; y.y *= ww.y; y.z *= ww.z; y.w *= ww.w;
            }
            if (bias) {
                const float4 bb = __ldg(b4 + i);
                y.x += bb.x; y.y += bb.y; y.z += bb.z; y.w += bb.w;
            }
            if (sc4) {
                const float4 a = __ldg(sc4 + i), t = __ldg(sh4 + i);
                y.x = y.x * (1.f + a.x) + t.x; y.y = y.y * (1.f + a.y) + t.y;
                y.z = y.z * (1.f + a.z) + t.z; y.w = y.w * (1.f + a.w) + t.w;
            }
            __nv_bfloat162 p0 = __floats2bfloat162_rn(y.x, y.y), p1 = __floats2bfloat162_rn(y.z, y.w);
            o[i] = make_uint2(*reinterpret_cast<uint32_t *>(&p0), *reinterpret_cast<uint32_t *>(&p1));
        }
    }
}

// y[r, c] = b[c] + sum_d f(x[r])[d] W[c, d], f = [LayerNorm affine] then [SiLU]; C <= 16.  One warp per THIN_ROWS rows:
// the C x D weight (40 KB at 13 x 768) comes through L1 once per warp-iteration, so with one row per warp the kernel was
// bound by L1 bandwidth (13 weight loads per x load), not by the x stream; two rows share every weight load.  Per-row
// arithmetic (order of the partial sums, the butterfly reductions) does not depend on THIN_ROWS.
#ifndef GA_THIN_ROWS
#define GA_THIN_ROWS 2
#endif
constexpr int THIN_ROWS = GA_THIN_ROWS;

__global__ void __launch_bounds__(256)
thin_linear_kernel(const float *__restrict__ x, const float *__restrict__ ln_w, const float *__restrict__ ln_b,
                   int apply_silu, const float *__restrict__ W, const float *__restrict__ bias,
                   float *__restrict__ y, int R, int D, int C, float eps)
{
    const int r0 = (blockIdx.x * 8 + (threadIdx.x >> 5)) * THIN_ROWS;
    const int lane = threadIdx.x & 31;
    if (r0 >= R) return;
    const int n4 = D >> 2;
    float4 c[THIN_ROWS][8];
    float mean[THIN_ROWS], rs[THIN_ROWS];
#pragma unroll
    for (int q = 0; q < THIN_ROWS; q++) {
        const int r = min(r0 + q, R - 1);                   // a missing last row re-reads the previous one (not stored)
        const float4 *x4 = reinterpret_cast<const float4 *>(x + (size_t)r * D);
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int i = lane + 32 * u;
            c[q][u] = i < n4 ? x4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
#pragma unroll
    for (int q = 0; q < THIN_ROWS; q++) {
        mean[q] = 0.f; rs[q] = 1.f;
        if (ln_w) {
            float s = 0.f;
#pragma unroll
            for (int u = 0; u < 8; u++) s += (c[q][u].x + c[q][u].y) + (c[q][u].z + c[q][u].w);
            mean[q] = warp_sum(s) / (float)D;
            float v = 0.f;
#pragma unroll
            for (int u = 0; u < 8; u++) {
                if (lane + 32 * u < n4) {
                    const float d0 = c[q][u].x - mean[q], d1 = c[q][u].y - mean[q], d2 = c[q][u].z - mean[q], d3 = c[q][u].w - mean[q];
                    v += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
                }
            }
            rs[q] = rsqrtf(warp_sum(v) / (float)D + eps);
        }
    }
    float acc[THIN_ROWS][16];
#pragma unroll
    for (int q = 0; q < THIN_ROWS; q++)
#pragma unroll
        for (int k = 0; k < 16; k++) acc[q][k] = 0.f;
#pragma unroll
    for (int u = 0; u < 8; u++) {
        const int i = lane + 32 * u;
        if (i < n4) {
            float4 h[THIN_ROWS];
            float4 ww = make_float4(1.f, 1.f, 1.f, 1.f), bb = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ln_w) {
                ww = __ldg(reinterpret_cast<const float4 *>(ln_w) + i);
                if (ln_b) bb = __ldg(reinterpret_cast<const float4 *>(ln_b) + i);
            }
#pragma unroll
            for (int q = 0; q < THIN_ROWS; q++) {
                h[q] = c[q][u];
                if (ln_w) {
                    h[q].x = (h[q].x - mean[q]) * rs[q] * ww.x + bb.x; h[q].y = (h[q].y - mean[q]) * rs[q] * ww.y + bb.y;
                    h[q].z = (h[q].z - mean[q]) * rs[q] * ww.z + bb.z; h[q].w = (h[q].w - mean[q]) * rs[q] * ww.w + bb.w;
                }
                if (apply_silu) { h[q].x = silu(h[q].x); h[q].y = silu(h[q].y); h[q].z = silu(h[q].z); h[q].w = silu(h[q].w); }
            }
#pragma unroll
            for (int k = 0; k < 16; k++) {
                if (k < C) {
                    const float4 wk = __ldg(reinterpret_cast<const float4 *>(W + (size_t)k * D) + i);
#pragma unroll
                    for (int q = 0; q < THIN_ROWS; q++)
                        acc[q][k] += h[q].x * wk.x + h[q].y * wk.y + h[q].z * wk.z + h[q].w * wk.w;
                }
            }
        }
    }
#pragma unroll
    for (int q = 0; q < THIN_ROWS; q++) {
#pragma unroll
        for (int k = 0; k < 16; k++) {
            if (k < C) {
                const float t = warp_sum(acc[q][k]);
                if (lane == 0 && r0 + q < R) y[(size_t)(r0 + q) * C + k] = t + (bias ? bias[k] : 0.f);
            }
        }
    }
}

// Attention over micro-sequences: qkv bf16 [S*L, 3*H*64] in "(K H D)" column order (q | k | v), per-head RMSNorm of
// q and k (weights qn_w, kn_w [64]), softmax(q k^T / 8) v, out bf16 [S*L, H*64].  One warp per (sequence, head); the
// L x 64 tiles live in shared memory as fp32 (rows padded to 65 floats: conflict-free column walks).  The footprint is
// sized by the actual L (5, 9, 4 rows in the deployed cascade, not the maximum 16): 3.2-7.4 KB per warp, so 28-64 warps
// stay resident per SM -- the kernel is a 1.5 KB-in / 0.5 KB-out stream per item and lives on loads in flight (round 2:
// with the fixed 13.5 KB footprint only 16 warps were resident and the kernel ran at 1/7 of the HBM rate).
constexpr int kMicroL = 16, kMicroPitch = 65, kMicroWarps = 4;
__host__ __device__ constexpr int micro_floats_per_warp(int L) { return 3 * L * kMicroPitch + L * (L + 1); }

#ifndef GA_MICRO_SMALL
#define GA_MICRO_SMALL 1          // 0: every length goes through the generic kernel below
#endif
__global__ void __launch_bounds__(32 * kMicroWarps)
micro_attention_kernel(const __nv_bfloat16 *__restrict__ qkv, const float *__restrict__ qn_w,
                       const float *__restrict__ kn_w, __nv_bfloat16 *__restrict__ out, int S, int L, int H, float eps)
{
    extern __shared__ float micro_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long item = (long long)blockIdx.x * kMicroWarps + warp;
    if (item >= (long long)S * H) return;
    const int s = (int)(item / H), h = (int)(item % H);
    const int LP = L + 1;
    float *sq = micro_smem + (size_t)warp * micro_floats_per_warp(L);
    float *sk = sq + L * kMicroPitch, *sv = sk + L * kMicroPitch, *sp = sv + L * kMicroPitch;
    const int C = H * 64;
    const float wq0 = qn_w[2 * lane], wq1 = qn_w[2 * lane + 1], wk0 = kn_w[2 * lane], wk1 = kn_w[2 * lane + 1];
    const __nv_bfloat16 *base = qkv + (size_t)s * L * (3 * C) + h * 64 + 2 * lane;
    for (int i0 = 0; i0 < L; i0 += 4) {
        // up to 12 independent 128-byte row segments per warp are requested before the first reduction needs one
        __nv_bfloat162 rq[4], rk[4], rv[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            if (i0 + u < L) {
                const __nv_bfloat16 *row = base + (size_t)(i0 + u) * (3 * C);
                rq[u] = *reinterpret_cast<const __nv_bfloat162 *>(row);
                rk[u] = *reinterpret_cast<const __nv_bfloat162 *>(row + C);
                rv[u] = *reinterpret_cast<const __nv_bfloat162 *>(row + 2 * C);
            }
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            if (i0 + u < L) {
                const int i = i0 + u;
                const float2 q = __bfloat1622float2(rq[u]), k = __bfloat1622float2(rk[u]), v = __bfloat1622float2(rv[u]);
                const float nq = rsqrtf(warp_sum(q.x * q.x + q.y * q.y) * (1.0f / 64.0f) + eps);
                const float nk = rsqrtf(warp_sum(k.x * k.x + k.y * k.y) * (1.0f / 64.0f) + eps);
                sq[i * kMicroPitch + 2 * lane] = q.x * nq * wq0; sq[i * kMicroPitch + 2 * lane + 1] = q.y * nq * wq1;
                sk[i * kMicroPitch + 2 * lane] = k.x * nk * wk0; sk[i * kMicroPitch + 2 * lane + 1] = k.y * nk * wk1;
                sv[i * kMicroPitch + 2 * lane] = v.x; sv[i * kMicroPitch + 2 * lane + 1] = v.y;
            }
        }
    }
    __syncwarp();
    for (int e = lane; e < L * L; e += 32) {                  // scores, scaled by 1/sqrt(64)
        const int i = e / L, j = e % L;
        float a = 0.f;
#pragma unroll 16
        for (int d = 0; d < 64; d++) a += sq[i * kMicroPitch + d] * sk[j * kMicroPitch + d];
        sp[i * LP + j] = a * 0.125f;
    }
    __syncwarp();
    if (lane < L) {                                           // one lane per query row
        float m = -INFINITY;
        for (int j = 0; j < L; j++) m = fmaxf(m, sp[lane * LP + j]);
        float l = 0.f;
        for (int j = 0; j < L; j++) {
            const float p = __expf(sp[lane * LP + j] - m);
            sp[lane * LP + j] = p;
            l += p;
        }
        const float inv = 1.0f / l;
        for (int j = 0; j < L; j++) sp[lane * LP + j] *= inv;
    }
    __syncwarp();
    for (int i = 0; i < L; i++) {
        float o0 = 0.f, o1 = 0.f;
        for (int j = 0; j < L; j++) {
            const float p = sp[i * LP + j];
            o0 += p * sv[j * kMicroPitch + 2 * lane];
            o1 += p * sv[j * kMicroPitch + 2 * lane + 1];
        }
        *reinterpret_cast<__nv_bfloat162 *>(out + ((size_t)s * L + i) * C + h * 64 + 2 * lane) = __floats2bfloat162_rn(o0, o1);
    }
}

// The deployed cascade's sequence lengths (1 + f = 9, 5, 4) get a compile-time-L version of the same algorithm: q and k
// rows at a 68-float pitch (16-byte aligned: the 64-long dot products run on LDS.128, and consecutive rows start 4 banks
// apart, so the <= 8 distinct rows one quarter-warp touches never collide), v stays in the loading lane's registers (each
// lane owns two head dims of every row), every loop is unrolled and e / L, e % L are constants.  ~380 warp instructions
// per (sequence, head) item at L = 4 against ~1 090 for the generic kernel, which ncu showed issue-bound (77 % issue-active,
// 19 % of the DRAM rate) once its occupancy was fixed.
template <int L>
__global__ void __launch_bounds__(32 * kMicroWarps)
micro_attention_small_kernel(const __nv_bfloat16 *__restrict__ qkv, const float *__restrict__ qn_w,
                             const float *__restrict__ kn_w, __nv_bfloat16 *__restrict__ out, int S, int H, float eps)
{
    constexpr bool SPLIT = L == 4;                                // 2 L^2 = 32: two lanes share one dot product
    constexpr int PITCH = SPLIT ? 72 : 68, LP = L + 1;            // split: rows 8 banks apart, the two halves 4 apart
    constexpr int PER_WARP = (2 * L * PITCH + L * LP + 3) & ~3;
    __shared__ __align__(16) float smem[kMicroWarps * PER_WARP];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const unsigned item = blockIdx.x * kMicroWarps + warp;        // the launcher keeps S * H below 2^31
    if (item >= (unsigned)S * (unsigned)H) return;                // warps are independent: no block-wide barrier below
    const unsigned s = item / (unsigned)H, h = item - s * (unsigned)H;
    float *sq = smem + warp * PER_WARP, *sk = sq + L * PITCH, *sp = sk + L * PITCH;
    const int C = H * 64;
    const float2 wq = *reinterpret_cast<const float2 *>(qn_w + 2 * lane), wk = *reinterpret_cast<const float2 *>(kn_w + 2 * lane);
    const __nv_bfloat16 *base = qkv + (size_t)s * L * (3 * C) + h * 64 + 2 * lane;
    __nv_bfloat162 rq[L], rk[L], rv[L];
#pragma unroll
    for (int i = 0; i < L; i++) {                                 // 3 L independent 128-byte row segments per warp
        const __nv_bfloat16 *row = base + (size_t)i * (3 * C);
        rq[i] = *reinterpret_cast<const __nv_bfloat162 *>(row);
        rk[i] = *reinterpret_cast<const __nv_bfloat162 *>(row + C);
        rv[i] = *reinterpret_cast<const __nv_bfloat162 *>(row + 2 * C);
    }
    float2 q[L], k[L], v[L];
    constexpr int NP = L <= 4 ? 8 : (L <= 8 ? 16 : 32);           // 2 L sums of squares, padded to a power of two
    constexpr int SH = NP == 8 ? 2 : (NP == 16 ? 1 : 0);
    float ssq[NP];
#pragma unroll
    for (int i = 0; i < NP; i++) ssq[i] = 0.f;
#pragma unroll
    for (int i = 0; i < L; i++) {
        q[i] = __bfloat1622float2(rq[i]); k[i] = __bfloat1622float2(rk[i]); v[i] = __bfloat1622float2(rv[i]);
        ssq[2 * i] = q[i].x * q[i].x + q[i].y * q[i].y;
        ssq[2 * i + 1] = k[i].x * k[i].x + k[i].y * k[i].y;
    }
    const float rn = rsqrtf(packed_wsum<NP>(ssq, lane) * (1.0f / 64.0f) + eps);     // this lane's one RMS factor
#pragma unroll
    for (int i = 0; i < L; i++) {
        const float nq = __shfl_sync(0xffffffffu, rn, (2 * i) << SH), nk = __shfl_sync(0xffffffffu, rn, (2 * i + 1) << SH);
        *reinterpret_cast<float2 *>(sq + i * PITCH + 2 * lane) = make_float2(q[i].x * nq * wq.x, q[i].y * nq * wq.y);
        *reinterpret_cast<float2 *>(sk + i * PITCH + 2 * lane) = make_float2(k[i].x * nk * wk.x, k[i].y * nk * wk.y);
    }
    __syncwarp();
    if constexpr (SPLIT) {                                        // scores: lane pair per (i, j), alternate 16-byte chunks
        const int e = lane >> 1, half = lane & 1;
        const int i = e / L, j = e % L;
        const float4 *q4 = reinterpret_cast<const float4 *>(sq + (e < L * L ? i : 0) * PITCH) + half;
        const float4 *k4 = reinterpret_cast<const float4 *>(sk + (e < L * L ? j : 0) * PITCH) + half;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
        for (int d = 0; d < 8; d++) {
            const float4 a = q4[2 * d], b = k4[2 * d];
            a0 += a.x * b.x; a1 += a.y * b.y; a2 += a.z * b.z; a3 += a.w * b.w;
        }
        float a = (a0 + a1) + (a2 + a3);
        a += __shfl_xor_sync(0xffffffffu, a, 1);
        // every lane now holds one score; the four (i, .) scores sit in the lanes l, l^2, l^4, l^6: softmax by shuffles
        const float sc = a * 0.125f;
        float m = fmaxf(sc, __shfl_xor_sync(0xffffffffu, sc, 2));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
        const float pe = __expf(sc - m);
        float l = pe + __shfl_xor_sync(0xffffffffu, pe, 2);
        l += __shfl_xor_sync(0xffffffffu, l, 4);
        if (half == 0) sp[i * LP + j] = pe * (1.0f / l);
    } else
#pragma unroll
    for (int e0 = 0; e0 < L * L; e0 += 32) {                      // scores, scaled by 1/sqrt(64): one lane per (i, j)
        const int e = e0 + lane;
        if (e < L * L) {
            const int i = e / L, j = e % L;
            const float4 *q4 = reinterpret_cast<const float4 *>(sq + i * PITCH);
            const float4 *k4 = reinterpret_cast<const float4 *>(sk + j * PITCH);
            float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
            for (int d = 0; d < 16; d++) {
                const float4 a = q4[d], b = k4[d];
                a0 += a.x * b.x; a1 += a.y * b.y; a2 += a.z * b.z; a3 += a.w * b.w;
            }
            sp[i * LP + j] = ((a0 + a1) + (a2 + a3)) * 0.125f;
        }
    }
    __syncwarp();
    if (!SPLIT && lane < L) {                                     // one lane per query row
        float pr[L];
        float m = -INFINITY;
#pragma unroll
        for (int j = 0; j < L; j++) { pr[j] = sp[lane * LP + j]; m = fmaxf(m, pr[j]); }
        float l = 0.f;
#pragma unroll
        for (int j = 0; j < L; j++) { pr[j] = __expf(pr[j] - m); l += pr[j]; }
        const float inv = 1.0f / l;
#pragma unroll
        for (int j = 0; j < L; j++) sp[lane * LP + j] = pr[j] * inv;
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < L; i++) {
        float o0 = 0.f, o1 = 0.f;
#pragma unroll
        for (int j = 0; j < L; j++) {
            const float pij = sp[i * LP + j];                     // same address in every lane: a broadcast
            o0 += pij * v[j].x;
            o1 += pij * v[j].y;
        }
        *reinterpret_cast<__nv_bfloat162 *>(out + ((size_t)s * L + i) * C + h * 64 + 2 * lane) = __floats2bfloat162_rn(o0, o1);
    }
}

// seq[s, 0, :] = parent token of sequence s, seq[s, 1 + j, :] = queries[j, :]   (fp32 residual stream)
// parent token: prev_f == 0 -> parents[s, :]; else the j-th child of the previous stage's sequence buffer
// [S / prev_f, 1 + prev_f, D]:  parents[(s / prev_f) * (1 + prev_f) + 1 + s % prev_f, :]
__global__ void micro_seq_build_kernel(const float *__restrict__ parents, int prev_f, const float *__restrict__ queries,
                                       float *__restrict__ seq, long long S, int f, int D)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int n4 = D >> 2;
    const long long total = S * (1 + f) * n4;
    if (i >= total) return;
    const int d4 = (int)(i % n4);
    const long long row = i / n4;
    const long long s = row / (1 + f);
    const int t = (int)(row % (1 + f));
    float4 v;
    if (t == 0) {
        const long long prow = prev_f == 0 ? s : (s / prev_f) * (1 + prev_f) + 1 + (s % prev_f);
        v = reinterpret_cast<const float4 *>(parents + prow * D)[d4];
    } else {
        v = __ldg(reinterpret_cast<const float4 *>(queries + (size_t)(t - 1) * D) + d4);
    }
    reinterpret_cast<float4 *>(seq)[i] = v;
}

// res [R, 13]: raw 13-channel prediction of child r (for the base level: of token r).
// pre = res + parent_pre[r / f] (parent_pre may be NULL: base level); position = tanh(res[0:3]) * offset_scale +
// parent_pos[r / f]; channels 3.. from pre: sigmoid | softplus * scale_factor (2) | normalise (4) | 0.5 tanh + 0.5 (3).
__global__ void surfel_cascade_pack_kernel(const float *__restrict__ res, int res_in_sequences,
                                           const float *__restrict__ parent_pre,
                                           const float *__restrict__ parent_pos, int parent_pos_stride, int f,
                                           float offset_scale, float scale_factor, float *__restrict__ out_gauss,
                                           float *__restrict__ out_pre, long long R)
{
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    const long long pr = r / f;
    // res_in_sequences: res holds one row per token of the [R/f, 1+f] micro-sequences (row 0 = the parent token)
    const long long rr = res_in_sequences ? pr * (1 + f) + 1 + (r % f) : r;
    float p[13];
#pragma unroll
    for (int k = 0; k < 13; k++) p[k] = res[rr * 13 + k];
    float g[13];
#pragma unroll
    for (int k = 0; k < 3; k++) g[k] = tanhf(p[k]) * offset_scale + parent_pos[pr * parent_pos_stride + k];
    if (parent_pre) {
#pragma unroll
        for (int k = 0; k < 13; k++) p[k] += parent_pre[pr * 13 + k];
    }
    g[3] = 1.0f / (1.0f + expf(-p[3]));
#pragma unroll
    for (int k = 4; k < 6; k++) g[k] = (p[k] > 20.f ? p[k] : log1pf(expf(p[k]))) * scale_factor;      // F.softplus
    const float n = fmaxf(sqrtf(p[6] * p[6] + p[7] * p[7] + p[8] * p[8] + p[9] * p[9]), 1e-12f);        // F.normalize
#pragma unroll
    for (int k = 6; k < 10; k++) g[k] = p[k] / n;
#pragma unroll
    for (int k = 10; k < 13; k++) g[k] = 0.5f * tanhf(p[k]) + 0.5f;
#pragma unroll
    for (int k = 0; k < 13; k++) out_gauss[r * 13 + k] = g[k];
    if (out_pre) {
#pragma unroll
        for (int k = 0; k < 13; k++) out_pre[r * 13 + k] = p[k];
    }
}

__global__ void silu_to_bf16_kernel(const float *__restrict__ x, __nv_bfloat16 *__restrict__ y, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = __float2bfloat16(silu(x[i]));
}

inline int last_err() { return (int)cudaGetLastError(); }
inline bool row_ok(int D) { return D > 0 && (D & 3) == 0 && D <= 1024; }

}  // namespace

extern "C" int ga_layernorm_modulate(const float *x, const float *w, const float *bias, const float *shift,
                                     const float *scale, int mod_ld, int rows_per_batch, void *out_bf16, int R, int D,
                                     float eps, void *stream)
{
    if (!x || !out_bf16 || R <= 0 || !row_ok(D) || (bias && !w) || ((shift == nullptr) != (scale == nullptr))) return GA_ERR_BADARG;
    if (shift && (rows_per_batch <= 0 || (mod_ld & 3))) return GA_ERR_BADARG;
    if (mis16(x) || mis16(w) || mis16(bias) || mis16(shift) || mis16(scale) || mis8(out_bf16)) return GA_ERR_BADARG;
    layernorm_modulate_kernel<<<(R + 7) / 8, 256, 0, (cudaStream_t)stream>>>(
        x, w, bias, shift, scale, mod_ld, rows_per_batch > 0 ? rows_per_batch : 1, reinterpret_cast<__nv_bfloat16 *>(out_bf16), R,
        D, eps);
    return last_err();
}

extern "C" int ga_thin_linear(const float *x, const float *ln_w, const float *ln_b, int apply_silu, const float *W,
                              const float *bias, float *y, int R, int D, int C, float eps, void *stream)
{
    if (!x || !W || !y || R <= 0 || !row_ok(D) || C <= 0 || C > 16 || (ln_b && !ln_w)) return GA_ERR_BADARG;
    if (mis16(x) || mis16(ln_w) || mis16(ln_b) || mis16(W)) return GA_ERR_BADARG;
    thin_linear_kernel<<<(R + 8 * THIN_ROWS - 1) / (8 * THIN_ROWS), 256, 0, (cudaStream_t)stream>>>(x, ln_w, ln_b, apply_silu, W, bias, y, R, D, C, eps);
    return last_err();
}

extern "C" int ga_micro_attention_bf16(const void *qkv, const float *qn_w, const float *kn_w, void *out, int S, int L,
                                       int H, float eps, void *stream)
{
    if (!qkv || !qn_w || !kn_w || !out || S <= 0 || L <= 0 || L > kMicroL || H <= 0) return GA_ERR_BADARG;
    // __nv_bfloat162 loads and stores; the small kernel reads the norm weights as float2
    if (mis4(qkv) || mis4(out) || mis8(qn_w) || mis8(kn_w)) return GA_ERR_BADARG;
    static GaPerDevice attr_set;
    if (ga_first_use_on_device(attr_set)) {
        cudaError_t e = cudaFuncSetAttribute(micro_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             kMicroWarps * micro_floats_per_warp(kMicroL) * (int)sizeof(float));
        if (e != cudaSuccess) return (int)e;
    }
    const long long items = (long long)S * H;
    const unsigned grid = (unsigned)((items + kMicroWarps - 1) / kMicroWarps);
    const __nv_bfloat16 *qp = reinterpret_cast<const __nv_bfloat16 *>(qkv);
    __nv_bfloat16 *op = reinterpret_cast<__nv_bfloat16 *>(out);
#if GA_MICRO_SMALL
    if ((L == 4 || L == 5 || L == 9) && items < (1ll << 31)) {
        if (L == 4) micro_attention_small_kernel<4><<<grid, 32 * kMicroWarps, 0, (cudaStream_t)stream>>>(qp, qn_w, kn_w, op, S, H, eps);
        else if (L == 5) micro_attention_small_kernel<5><<<grid, 32 * kMicroWarps, 0, (cudaStream_t)stream>>>(qp, qn_w, kn_w, op, S, H, eps);
        else micro_attention_small_kernel<9><<<grid, 32 * kMicroWarps, 0, (cudaStream_t)stream>>>(qp, qn_w, kn_w, op, S, H, eps);
        return last_err();
    }
#endif
    micro_attention_kernel<<<(unsigned)((items + kMicroWarps - 1) / kMicroWarps), 32 * kMicroWarps,
                             kMicroWarps * micro_floats_per_warp(L) * sizeof(float), (cudaStream_t)stream>>>(
        reinterpret_cast<const __nv_bfloat16 *>(qkv), qn_w, kn_w, reinterpret_cast<__nv_bfloat16 *>(out), S, L, H, eps);
    return last_err();
}

extern "C" int ga_micro_seq_build(const float *parents, int prev_f, const float *queries, float *seq, int64_t S, int f,
                                  int D, void *stream)
{
    if (!parents || !queries || !seq || S <= 0 || f <= 0 || prev_f < 0 || !row_ok(D)) return GA_ERR_BADARG;
    if (prev_f > 0 && S % prev_f) return GA_ERR_BADARG;
    if (mis16(parents) || mis16(queries) || mis16(seq)) return GA_ERR_BADARG;
    const long long total = S * (1 + f) * (D >> 2);
    micro_seq_build_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(parents, prev_f, queries, seq, S,
                                                                                            f, D);
    return last_err();
}

extern "C" int ga_surfel_cascade_pack(const float *res, int res_in_sequences, const float *parent_pre, const float *parent_pos,
                                      int parent_pos_stride, int f, float offset_scale, float scale_factor,
                                      float *out_gauss13, float *out_pre, int64_t R, void *stream)
{
    if (!res || !parent_pos || !out_gauss13 || R <= 0 || f <= 0 || parent_pos_stride < 3) return GA_ERR_BADARG;
    surfel_cascade_pack_kernel<<<(unsigned)((R + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        res, res_in_sequences, parent_pre, parent_pos, parent_pos_stride, f, offset_scale, scale_factor, out_gauss13, out_pre, R);
    return last_err();
}

extern "C" int ga_silu_to_bf16(const float *x, void *y, int64_t n, void *stream)
{
    if (!x || !y || n <= 0) return GA_ERR_BADARG;
    silu_to_bf16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        x, reinterpret_cast<__nv_bfloat16 *>(y), (size_t)n);
    return last_err();
}
