// Backwards of the image-to-3D DiT outside its blocks (include/ga_b200.h Part 15): the final layer (T2IFinalLayer),
// the token embedder's fc1 (tanh-GELU), the fp32 B-row linears of the timestep / pooled-vector / adaLN stem and the
// pooled vector's LayerNorm.  The GEMMs around them (fc2, the xyz projection) are Part 13's.
//
// No atomics: sums over the token rows are written as one fp32 partial per chunk of kChunkRows rows (chunks never
// cross a batch item, ga_dit_grad_partials counts them), added within a chunk in a fixed order, and reduced by
// ga_dit_grad_reduce in index order.  Sums over the B rows of the stem are taken in row order.
#include "../../include/ga_b200.h"
#include "row_common.cuh"

using namespace ga_row;

namespace {

constexpr int kMaxCout = 16;            // ga_final_layer's output width limit
constexpr int kMaxK = 16;               // fc1's input width limit (x channels + xyz)

// ---- final layer ----------------------------------------------------------------------------------------------------
// One CTA per chunk (b, c) of rows b N + 32 c + i.  Phase 1, warp w taking rows i = w, w + 8, ...: n = LN(x), dh =
// dy W, dshift += dh, dscale += dh n, dx = rstd (dn - mean(dn) - n mean(dn n)), dn = dh (1 + scale[b]).  Phase 2,
// thread q owning columns 4q .. 4q + 3: dW[c] += dy[i, c] h[i] over the chunk's rows in increasing order, h =
// n (1 + scale[b]) + shift[b] recomputed from the row's mean and rstd.
__global__ void __launch_bounds__(32 * kWarps)
final_layer_bwd_kernel(const float *__restrict__ x, const float *__restrict__ mod, const float *__restrict__ W,
                       const float *__restrict__ dy, float *__restrict__ dx, float *__restrict__ part_dmod,
                       float *__restrict__ part_dw, float *__restrict__ part_db, int rows_per_batch, int D, int Cout,
                       float eps)
{
    __shared__ float4 red[kWarps][kMaxD / 4];
    __shared__ float s_dy[kChunkRows][kMaxCout];
    __shared__ float s_mu[kChunkRows], s_rs[kChunkRows];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int chunks = (rows_per_batch + kChunkRows - 1) / kChunkRows;
    const int p = blockIdx.x, b = p / chunks, c = p - b * chunks;
    const int i0 = c * kChunkRows, rows = min(kChunkRows, rows_per_batch - i0);
    const size_t r0 = (size_t)b * rows_per_batch + i0;
    const int n4 = D >> 2;
    const float *sh = mod + (size_t)b * 2 * D, *sc = sh + D;
    float4 a_sh[8], a_sc[8];
#pragma unroll
    for (int u = 0; u < 8; u++) a_sh[u] = a_sc[u] = zero4();
    for (int i = warp; i < rows; i += kWarps) {
        const size_t r = r0 + i;
        const float dyl = lane < Cout ? dy[r * Cout + lane] : 0.f;
        if (lane < kMaxCout) s_dy[i][lane] = dyl;
        float dyv[kMaxCout];
#pragma unroll
        for (int k = 0; k < kMaxCout; k++) dyv[k] = __shfl_sync(0xffffffffu, dyl, k);
        float4 xv[8], dh[8];
        float s = 0.f;
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int j = lane + 32 * u;
            xv[u] = j < n4 ? reinterpret_cast<const float4 *>(x + r * D)[j] : zero4();
            s += sum4(xv[u]);
        }
        const float mean = warp_sum(s) / (float)D;
        float v = 0.f;
#pragma unroll
        for (int u = 0; u < 8; u++) {
            if (lane + 32 * u < n4) {
                const float4 d = make_float4(xv[u].x - mean, xv[u].y - mean, xv[u].z - mean, xv[u].w - mean);
                v += dot4(d, d);
            }
        }
        const float rs = rsqrtf(warp_sum(v) / (float)D + eps);
        if (lane == 0) { s_mu[i] = mean; s_rs[i] = rs; }
        float sdn = 0.f, sdnn = 0.f;
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int j = lane + 32 * u;
            if (j < n4) {
                float4 g = zero4();
#pragma unroll
                for (int k = 0; k < kMaxCout; k++)
                    if (k < Cout) fma4(g, dyv[k], ld4(W + (size_t)k * D, j));
                const float4 n = make_float4((xv[u].x - mean) * rs, (xv[u].y - mean) * rs, (xv[u].z - mean) * rs,
                                             (xv[u].w - mean) * rs);
                add4(a_sh[u], g);
                add4(a_sc[u], mul4(g, n));
                const float4 a = ld4(sc, j);
                const float4 dn = make_float4(g.x * (1.f + a.x), g.y * (1.f + a.y), g.z * (1.f + a.z), g.w * (1.f + a.w));
                sdn += sum4(dn);
                sdnn += dot4(dn, n);
                xv[u] = n;
                dh[u] = dn;
            }
        }
        if (dx) {
            const float m1 = warp_sum(sdn) / (float)D, m2 = warp_sum(sdnn) / (float)D;
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int j = lane + 32 * u;
                if (j < n4)
                    reinterpret_cast<float4 *>(dx + r * D)[j] =
                        make_float4(rs * (dh[u].x - m1 - xv[u].x * m2), rs * (dh[u].y - m1 - xv[u].y * m2),
                                    rs * (dh[u].z - m1 - xv[u].z * m2), rs * (dh[u].w - m1 - xv[u].w * m2));
            }
        }
    }
    if (part_dmod) {
        cta_colsum(red, a_sh, part_dmod + (size_t)p * 2 * D, n4);
        cta_colsum(red, a_sc, part_dmod + (size_t)p * 2 * D + D, n4);
    } else {
        __syncthreads();
    }
    if (part_db && threadIdx.x < Cout) {
        float s = 0.f;
        for (int i = 0; i < rows; i++) s += s_dy[i][threadIdx.x];
        part_db[(size_t)p * Cout + threadIdx.x] = s;
    }
    if (!part_dw) return;
    for (int q = threadIdx.x; q < n4; q += blockDim.x) {
        const float4 a = ld4(sc, q), t = ld4(sh, q);
        float4 acc[kMaxCout];
#pragma unroll
        for (int k = 0; k < kMaxCout; k++) acc[k] = zero4();
        for (int i = 0; i < rows; i++) {
            const float4 xq = reinterpret_cast<const float4 *>(x + (r0 + i) * D)[q];
            const float mu = s_mu[i], rs = s_rs[i];
            const float4 h = make_float4((xq.x - mu) * rs * (1.f + a.x) + t.x, (xq.y - mu) * rs * (1.f + a.y) + t.y,
                                         (xq.z - mu) * rs * (1.f + a.z) + t.z, (xq.w - mu) * rs * (1.f + a.w) + t.w);
#pragma unroll
            for (int k = 0; k < kMaxCout; k++)
                if (k < Cout) fma4(acc[k], s_dy[i][k], h);
        }
#pragma unroll
        for (int k = 0; k < kMaxCout; k++)
            if (k < Cout) reinterpret_cast<float4 *>(part_dw + ((size_t)p * Cout + k) * D)[q] = acc[k];
    }
}

// ---- token embedder fc1 ---------------------------------------------------------------------------------------------
// One CTA per chunk of 32 rows; thread t owns columns n = t, t + 256, ... (D <= 1024: at most 4).  Over the chunk's
// rows in increasing order: v = b1[n] + sum_c in[c] W1[n, c] (ga_embed_fc1's order), dv = de1 gelu_tanh'(v),
// dW1[n] += dv in, db1[n] += dv.  dxin[r, c] = sum_n dv W1[n, C2 + c]: each thread's columns in increasing order,
// then the lanes by warp_sum, then the warps in warp order.
__global__ void __launch_bounds__(32 * kWarps)
embed_fc1_bwd_kernel(const float *__restrict__ xin, int Cx, const float *__restrict__ xin2, int C2,
                     const float *__restrict__ W1, const float *__restrict__ b1, const float *__restrict__ de1,
                     float *__restrict__ part_dw1, float *__restrict__ part_db1, float *__restrict__ dxin, int R, int D)
{
    __shared__ float s_in[kChunkRows][kMaxK];
    __shared__ float red[kWarps][kChunkRows][kMaxK];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int K = Cx + C2, p = blockIdx.x;
    const int r0 = p * kChunkRows, rows = min(kChunkRows, R - r0);
    for (int e = threadIdx.x; e < rows * K; e += blockDim.x) {
        const int i = e / K, k = e - i * K;
        s_in[i][k] = k < C2 ? xin2[(size_t)(r0 + i) * C2 + k] : xin[(size_t)(r0 + i) * Cx + k - C2];
    }
    __syncthreads();
    float w[4][kMaxK], bias[4], aw[4][kMaxK], ab[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int n = threadIdx.x + 256 * j;
        bias[j] = n < D ? b1[n] : 0.f;
        ab[j] = 0.f;
#pragma unroll
        for (int k = 0; k < kMaxK; k++) {
            w[j][k] = (n < D && k < K) ? W1[(size_t)n * K + k] : 0.f;
            aw[j][k] = 0.f;
        }
    }
    for (int i = 0; i < rows; i++) {
        float px[kMaxK];
#pragma unroll
        for (int k = 0; k < kMaxK; k++) px[k] = 0.f;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int n = threadIdx.x + 256 * j;
            if (n < D) {
                float v = bias[j];
#pragma unroll
                for (int k = 0; k < kMaxK; k++)
                    if (k < K) v += s_in[i][k] * w[j][k];
                const float dv = de1[(size_t)(r0 + i) * D + n] * gelu_tanh_grad(v);
                ab[j] += dv;
#pragma unroll
                for (int k = 0; k < kMaxK; k++)
                    if (k < K) aw[j][k] = fmaf(dv, s_in[i][k], aw[j][k]);
#pragma unroll
                for (int k = 0; k < kMaxK; k++)
                    if (k < K) px[k] = fmaf(dv, w[j][k], px[k]);
            }
        }
        if (dxin) {
#pragma unroll
            for (int k = 0; k < kMaxK; k++) {
                if (k >= C2 && k < K) {                  // the x columns only: the xyz input is a constant
                    const float s = warp_sum(px[k]);
                    if (lane == 0) red[warp][i][k - C2] = s;
                }
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int n = threadIdx.x + 256 * j;
        if (n < D) {
            part_db1[(size_t)p * D + n] = ab[j];
#pragma unroll
            for (int k = 0; k < kMaxK; k++)
                if (k < K) part_dw1[((size_t)p * D + n) * K + k] = aw[j][k];
        }
    }
    if (!dxin) return;
    __syncthreads();
    for (int e = threadIdx.x; e < rows * Cx; e += blockDim.x) {
        const int i = e / Cx, k = e - i * Cx;
        float s = red[0][i][k];
#pragma unroll
        for (int q = 1; q < kWarps; q++) s += red[q][i][k];
        dxin[(size_t)(r0 + i) * Cx + k] = s;
    }
}

// ---- small fp32 linear ----------------------------------------------------------------------------------------------
// One CTA per chunk of 32 output rows n (ga_dit_grad_partials(N, N) chunks); thread q owns input columns 4q .. 4q + 3.
// dW[n] = sum over b = 0, 1, ... of dy[b, n] act(x[b]); db[n] likewise; part[p, b] = sum over the chunk's n in
// increasing order of dy[b, n] W[n] (the chunk's W rows are read from memory once, then from cache for each further
// group of 8 b).
__global__ void __launch_bounds__(256)
linear_small_bwd_kernel(const float *__restrict__ x, int act_in, const float *__restrict__ W,
                        const float *__restrict__ dy, float *__restrict__ dW, float *__restrict__ db,
                        float *__restrict__ part, int B, int N, int K)
{
    const int p = blockIdx.x, n0 = p * kChunkRows, nn = min(kChunkRows, N - n0), K4 = K >> 2;
    const float4 *x4 = reinterpret_cast<const float4 *>(x), *W4 = reinterpret_cast<const float4 *>(W);
    if (db && (int)threadIdx.x < nn) {
        float s = 0.f;
        for (int b = 0; b < B; b++) s += dy[(size_t)b * N + n0 + threadIdx.x];
        db[n0 + threadIdx.x] = s;
    }
    for (int q = threadIdx.x; q < K4; q += blockDim.x) {
        if (dW) {
            for (int s0 = 0; s0 < nn; s0 += 8) {
                float4 acc[8];
#pragma unroll
                for (int j = 0; j < 8; j++) acc[j] = zero4();
                for (int b = 0; b < B; b++) {
                    float4 a = __ldg(x4 + (size_t)b * K4 + q);
                    if (act_in) a = silu4(a);
                    const float *d = dy + (size_t)b * N + n0 + s0;
#pragma unroll
                    for (int j = 0; j < 8; j++)
                        if (s0 + j < nn) fma4(acc[j], __ldg(d + j), a);
                }
#pragma unroll
                for (int j = 0; j < 8; j++)
                    if (s0 + j < nn) reinterpret_cast<float4 *>(dW)[(size_t)(n0 + s0 + j) * K4 + q] = acc[j];
            }
        }
        if (part) {
            for (int b0 = 0; b0 < B; b0 += 8) {
                float4 acc[8];
#pragma unroll
                for (int j = 0; j < 8; j++) acc[j] = zero4();
                for (int i = 0; i < nn; i++) {
                    const float4 w = __ldg(W4 + (size_t)(n0 + i) * K4 + q);
#pragma unroll
                    for (int j = 0; j < 8; j++)
                        if (b0 + j < B) fma4(acc[j], __ldg(dy + (size_t)(b0 + j) * N + n0 + i), w);
                }
#pragma unroll
                for (int j = 0; j < 8; j++)
                    if (b0 + j < B) reinterpret_cast<float4 *>(part)[((size_t)p * B + b0 + j) * K4 + q] = acc[j];
            }
        }
    }
}

// dx[i] = dx_in[i] + act'(x[i]) sum over p in increasing order of part[p, i], i over the B K inputs
__global__ void linear_small_dx_kernel(const float *__restrict__ x, int act_in, const float *__restrict__ part,
                                       int parts, const float *dx_in, float *dx, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float s = part[i];
    for (int p = 1; p < parts; p++) s += part[(size_t)p * n + i];
    float d = act_in ? silu_grad(x[i]) * s : s;
    if (dx_in) d += dx_in[i];
    dx[i] = d;
}

// ---- LayerNorm over the B rows ------------------------------------------------------------------------------------
// One CTA; thread t owns columns 4t .. 4t + 3; rows in increasing order.  n = (x - mean) rstd, dn = dy w,
// dx = rstd (dn - mean(dn) - n mean(dn n)), dw += dy n, db += dy.
__device__ __forceinline__ void cta_sum2(float &a, float &b, float *red)      // red: 2 kWarps shared floats
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    a = warp_sum(a);
    b = warp_sum(b);
    if (lane == 0) { red[warp] = a; red[kWarps + warp] = b; }
    __syncthreads();
    a = red[0];
    b = red[kWarps];
#pragma unroll
    for (int w = 1; w < kWarps; w++) { a += red[w]; b += red[kWarps + w]; }
    __syncthreads();
}

__global__ void __launch_bounds__(256)
layernorm_rows_bwd_kernel(const float *__restrict__ x, const float *__restrict__ w, const float *__restrict__ dy,
                          float *__restrict__ dx, float *__restrict__ dw, float *__restrict__ db, int R, int D,
                          float eps)
{
    __shared__ float red[2 * kWarps];
    const int q = threadIdx.x, n4 = D >> 2;
    const bool live = q < n4;
    const float4 wv = live ? ld4(w, q) : zero4();
    float4 aw = zero4(), ab = zero4();
    for (int r = 0; r < R; r++) {
        const float4 xv = live ? reinterpret_cast<const float4 *>(x + (size_t)r * D)[q] : zero4();
        const float4 g = live ? reinterpret_cast<const float4 *>(dy + (size_t)r * D)[q] : zero4();
        float s1 = sum4(xv), s2 = 0.f;
        cta_sum2(s1, s2, red);
        const float mean = s1 / (float)D;
        const float4 d = live ? make_float4(xv.x - mean, xv.y - mean, xv.z - mean, xv.w - mean) : zero4();
        s1 = dot4(d, d);
        cta_sum2(s1, s2, red);
        const float rs = rsqrtf(s1 / (float)D + eps);
        const float4 n = scale4(d, rs), dn = mul4(g, wv);
        add4(aw, mul4(g, n));
        add4(ab, g);
        if (dx) {
            float m1 = sum4(dn), m2 = dot4(dn, n);
            cta_sum2(m1, m2, red);
            m1 /= (float)D;
            m2 /= (float)D;
            if (live)
                reinterpret_cast<float4 *>(dx + (size_t)r * D)[q] =
                    make_float4(rs * (dn.x - m1 - n.x * m2), rs * (dn.y - m1 - n.y * m2), rs * (dn.z - m1 - n.z * m2),
                                rs * (dn.w - m1 - n.w * m2));
        }
    }
    if (!live) return;
    if (dw) reinterpret_cast<float4 *>(dw)[q] = aw;
    if (db) reinterpret_cast<float4 *>(db)[q] = ab;
}

}  // namespace

extern "C" int ga_dit_final_layer_bwd_validate(const float *x, const float *mod, const float *W, const float *dy,
                                               const float *dx, const float *part_dmod, const float *part_dw,
                                               const float *part_db, int rows_per_batch, int R, int D, int Cout)
{
    if (R < 1 || rows_per_batch < 1 || R % rows_per_batch || D < 4 || D % 4 || D > kMaxD) return GA_ERR_BADARG;
    if (Cout < 1 || Cout > kMaxCout || (long long)R * D >= (1LL << 31)) return GA_ERR_BADARG;
    for (const void *p : {(const void *)x, (const void *)mod, (const void *)W})
        if (!p || mis16(p)) return GA_ERR_BADARG;
    if (!dy || mis4(dy) || !part_db != !part_dw) return GA_ERR_BADARG;
    for (const void *p : {(const void *)dx, (const void *)part_dmod, (const void *)part_dw})
        if (p && mis16(p)) return GA_ERR_BADARG;
    if (part_db && mis4(part_db)) return GA_ERR_BADARG;
    return 0;
}

extern "C" int ga_dit_final_layer_bwd(const float *x, const float *mod, const float *W, const float *dy, float *dx,
                                      float *part_dmod, float *part_dw, float *part_db, int rows_per_batch, int R,
                                      int D, int Cout, float eps, void *stream)
{
    const int rc = ga_dit_final_layer_bwd_validate(x, mod, W, dy, dx, part_dmod, part_dw, part_db, rows_per_batch, R,
                                                   D, Cout);
    if (rc) return rc;
    final_layer_bwd_kernel<<<ga_dit_grad_partials(R, rows_per_batch), 32 * kWarps, 0, (cudaStream_t)stream>>>(
        x, mod, W, dy, dx, part_dmod, part_dw, part_db, rows_per_batch, D, Cout, eps);
    return (int)cudaGetLastError();
}

extern "C" int ga_dit_embed_fc1_bwd_validate(const float *xin, int Cx, const float *xin2, int C2, const float *W1,
                                             const float *b1, const float *de1, const float *part_dw1,
                                             const float *part_db1, const float *dxin, int R, int D)
{
    if (R < 1 || D < 1 || D > kMaxD || Cx < 1 || C2 < 0 || Cx + C2 > kMaxK) return GA_ERR_BADARG;
    if ((long long)R * D >= (1LL << 31)) return GA_ERR_BADARG;
    if (C2 > 0 ? (!xin2 || mis4(xin2)) : xin2 != nullptr) return GA_ERR_BADARG;
    for (const void *p : {(const void *)xin, (const void *)W1, (const void *)b1, (const void *)de1,
                          (const void *)part_dw1, (const void *)part_db1})
        if (!p || mis4(p)) return GA_ERR_BADARG;
    if (dxin && mis4(dxin)) return GA_ERR_BADARG;
    return 0;
}

extern "C" int ga_dit_embed_fc1_bwd(const float *xin, int Cx, const float *xin2, int C2, const float *W1,
                                    const float *b1, const float *de1, float *part_dw1, float *part_db1, float *dxin,
                                    int R, int D, void *stream)
{
    const int rc = ga_dit_embed_fc1_bwd_validate(xin, Cx, xin2, C2, W1, b1, de1, part_dw1, part_db1, dxin, R, D);
    if (rc) return rc;
    embed_fc1_bwd_kernel<<<ga_dit_grad_partials(R, R), 32 * kWarps, 0, (cudaStream_t)stream>>>(
        xin, Cx, xin2, C2, W1, b1, de1, part_dw1, part_db1, dxin, R, D);
    return (int)cudaGetLastError();
}

extern "C" int ga_dit_linear_small_bwd_validate(const float *x, int act_in, const float *W, const float *dy,
                                                const float *dW, const float *db, const float *part,
                                                const float *dx_in, const float *dx, int rows, int N, int K)
{
    if (rows < 1 || N < 1 || K < 4 || K % 4 || (act_in != 0 && act_in != 1)) return GA_ERR_BADARG;
    if ((long long)N * K >= (1LL << 31) || (long long)ga_dit_grad_partials(N, N) * rows * K >= (1LL << 31))
        return GA_ERR_BADARG;
    for (const void *p : {(const void *)x, (const void *)W})
        if (!p || mis16(p)) return GA_ERR_BADARG;
    if (!dy || mis4(dy)) return GA_ERR_BADARG;
    if ((dW && mis16(dW)) || (db && mis4(db))) return GA_ERR_BADARG;
    if (dx ? (!part || mis16(part) || mis4(dx)) : (part || dx_in)) return GA_ERR_BADARG;
    if (dx_in && mis4(dx_in)) return GA_ERR_BADARG;
    return 0;
}

extern "C" int ga_dit_linear_small_bwd(const float *x, int act_in, const float *W, const float *dy, float *dW,
                                       float *db, float *part, const float *dx_in, float *dx, int rows, int N, int K,
                                       void *stream)
{
    const int rc = ga_dit_linear_small_bwd_validate(x, act_in, W, dy, dW, db, part, dx_in, dx, rows, N, K);
    if (rc) return rc;
    if (!dW && !db && !dx) return 0;
    const int P = ga_dit_grad_partials(N, N);
    linear_small_bwd_kernel<<<P, 256, 0, (cudaStream_t)stream>>>(x, act_in, W, dy, dW, db, dx ? part : nullptr, rows,
                                                                 N, K);
    if (dx) {
        const int n = rows * K;
        linear_small_dx_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(x, act_in, part, P, dx_in, dx, n);
    }
    return (int)cudaGetLastError();
}

extern "C" int ga_dit_layernorm_rows_bwd_validate(const float *x, const float *w, const float *dy, const float *dx,
                                                  const float *dw, const float *db, int R, int D)
{
    if (R < 1 || D < 4 || D % 4 || D > kMaxD || (long long)R * D >= (1LL << 31)) return GA_ERR_BADARG;
    for (const void *p : {(const void *)x, (const void *)w, (const void *)dy})
        if (!p || mis16(p)) return GA_ERR_BADARG;
    for (const void *p : {(const void *)dx, (const void *)dw, (const void *)db})
        if (p && mis16(p)) return GA_ERR_BADARG;
    return 0;
}

extern "C" int ga_dit_layernorm_rows_bwd(const float *x, const float *w, const float *dy, float *dx, float *dw,
                                         float *db, int R, int D, float eps, void *stream)
{
    const int rc = ga_dit_layernorm_rows_bwd_validate(x, w, dy, dx, dw, db, R, D);
    if (rc) return rc;
    layernorm_rows_bwd_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(x, w, dy, dx, dw, db, R, D, eps);
    return (int)cudaGetLastError();
}
