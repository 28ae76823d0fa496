// Row kernels of the DiT block's training forward and backward (include/ga_b200.h Part 14): the RMSNorm(+modulate)
// backward, the per-head q/k RMSNorm forward and backward, the gate backward, the gated residual forward (fused with
// the next RMSNorm-modulate) and the deterministic reduction of their partials.  The GEMMs and attentions of the
// block are Parts 2, 12 and 13.
//
// No atomics: every kernel that sums over rows writes one fp32 partial per chunk of kChunkRows rows (chunks never
// cross a batch item), adding within a chunk in a fixed order, and ga_dit_grad_reduce adds the partials in index
// order.  The number of partials depends on the shapes alone.
#include "../../include/ga_b200.h"
#include "row_common.cuh"

using namespace ga_row;

namespace {

__device__ __forceinline__ float sum8(float v)       // over the 8 lanes of an aligned lane group
{
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    return v;
}

// One CTA per chunk (b, c): rows b N + 32 c + i, i < 32, warp w taking i = w, w + 8, ... in increasing order.
// n = x rstd, dy0 = dh (1 + scale[b]), dw += dy0 n, dscale += dh n w, dshift += dh,
// dx = rstd (dy0 w - n mean(dy0 w n)).
__global__ void __launch_bounds__(32 * kWarps)
rmsnorm_bwd_kernel(const float *__restrict__ dh, const float *__restrict__ x, const float *__restrict__ w,
                   const float *__restrict__ scale, int mod_ld, const float *dx_in, float *dx_out,
                   float *__restrict__ part_dw, float *__restrict__ part_dshift, float *__restrict__ part_dscale,
                   int part_ld, int rows_per_batch, int D, float eps)
{
    __shared__ float4 red[kWarps][kMaxD / 4];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int chunks = (rows_per_batch + kChunkRows - 1) / kChunkRows;
    const int p = blockIdx.x, b = p / chunks, c = p - b * chunks;
    const int n4 = D >> 2;
    const float *sc = scale ? scale + (size_t)b * mod_ld : nullptr;
    float4 a_dw[8], a_sc[8], a_sh[8];
#pragma unroll
    for (int u = 0; u < 8; u++) a_dw[u] = a_sc[u] = a_sh[u] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = c * kChunkRows + warp; i < min(rows_per_batch, (c + 1) * kChunkRows); i += kWarps) {
        const size_t r = (size_t)b * rows_per_batch + i;
        float4 xv[8], gv[8];
        float ss = 0.f;
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int j = lane + 32 * u;
            if (j < n4) {
                xv[u] = reinterpret_cast<const float4 *>(x + r * D)[j];
                gv[u] = reinterpret_cast<const float4 *>(dh + r * D)[j];
                ss += dot4(xv[u], xv[u]);
            }
        }
        const float rs = rsqrtf(warp_sum(ss) / (float)D + eps);
        float dot = 0.f;
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int j = lane + 32 * u;
            if (j < n4) {
                const float4 n = make_float4(xv[u].x * rs, xv[u].y * rs, xv[u].z * rs, xv[u].w * rs);
                const float4 ww = ld4(w, j);
                float4 dy0 = gv[u];
                if (sc) {
                    const float4 s = ld4(sc, j);
                    dy0 = make_float4(gv[u].x * (1.f + s.x), gv[u].y * (1.f + s.y), gv[u].z * (1.f + s.z),
                                      gv[u].w * (1.f + s.w));
                    add4(a_sc[u], mul4(gv[u], mul4(n, ww)));
                    add4(a_sh[u], gv[u]);
                }
                add4(a_dw[u], mul4(dy0, n));
                const float4 dn = mul4(dy0, ww);
                dot += dot4(dn, n);
                xv[u] = n;                  // keep n and dn for the second pass
                gv[u] = dn;
            }
        }
        const float mean = warp_sum(dot) / (float)D;
        if (dx_out) {
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int j = lane + 32 * u;
                if (j < n4) {
                    float4 d = make_float4(rs * (gv[u].x - xv[u].x * mean), rs * (gv[u].y - xv[u].y * mean),
                                           rs * (gv[u].z - xv[u].z * mean), rs * (gv[u].w - xv[u].w * mean));
                    if (dx_in) add4(d, reinterpret_cast<const float4 *>(dx_in + r * D)[j]);
                    reinterpret_cast<float4 *>(dx_out + r * D)[j] = d;
                }
            }
        }
    }
    cta_colsum(red, a_dw, part_dw + (size_t)p * D, n4);
    if (sc) {
        cta_colsum(red, a_sh, part_dshift + (size_t)p * part_ld, n4);
        cta_colsum(red, a_sc, part_dscale + (size_t)p * part_ld, n4);
    }
}

// da = bf16(gate[b] dy), dgate partial = sum over the chunk's rows of dy a (same chunks and order as above)
__global__ void __launch_bounds__(32 * kWarps)
gate_bwd_kernel(const float *__restrict__ dy, const float *__restrict__ a, const float *__restrict__ gate,
                int gate_ld, __nv_bfloat16 *__restrict__ da, float *__restrict__ part, int part_ld,
                int rows_per_batch, int D)
{
    __shared__ float4 red[kWarps][kMaxD / 4];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int chunks = (rows_per_batch + kChunkRows - 1) / kChunkRows;
    const int p = blockIdx.x, b = p / chunks, c = p - b * chunks;
    const int n4 = D >> 2;
    const float *g = gate + (size_t)b * gate_ld;
    float4 acc[8];
#pragma unroll
    for (int u = 0; u < 8; u++) acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int i = c * kChunkRows + warp; i < min(rows_per_batch, (c + 1) * kChunkRows); i += kWarps) {
        const size_t r = (size_t)b * rows_per_batch + i;
        float4 dv[8], av[8];
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int j = lane + 32 * u;
            if (j < n4) {
                dv[u] = reinterpret_cast<const float4 *>(dy + r * D)[j];
                av[u] = reinterpret_cast<const float4 *>(a + r * D)[j];
            }
        }
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int j = lane + 32 * u;
            if (j < n4) {
                add4(acc[u], mul4(dv[u], av[u]));
                reinterpret_cast<uint2 *>(da + r * D)[j] = pack4(mul4(ld4(g, j), dv[u]));
            }
        }
    }
    cta_colsum(red, acc, part + (size_t)p * part_ld, n4);
}

// x_out = x + gate[b] a (gate NULL: x + a); with w: h = bf16(RMSNorm(x_out) w [(1 + scale[b]) + shift[b]]).
// One warp per row.
__global__ void __launch_bounds__(256)
gate_residual_kernel(const float *__restrict__ x, const float *__restrict__ a, const float *__restrict__ gate,
                     int gate_ld, float *__restrict__ x_out, const float *__restrict__ w,
                     const float *__restrict__ shift, const float *__restrict__ scale, int mod_ld,
                     __nv_bfloat16 *__restrict__ h, int rows_per_batch, int R, int D, float eps)
{
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= R) return;
    const int b = r / rows_per_batch, n4 = D >> 2;
    const float4 *x4 = reinterpret_cast<const float4 *>(x + (size_t)r * D);
    const float4 *a4 = reinterpret_cast<const float4 *>(a + (size_t)r * D);
    float4 *o4 = reinterpret_cast<float4 *>(x_out + (size_t)r * D);
    float4 v[8];
    float ss = 0.f;
#pragma unroll
    for (int u = 0; u < 8; u++) {
        const int j = lane + 32 * u;
        if (j < n4) {
            const float4 xv = x4[j], av = a4[j];
            const float4 g = gate ? ld4(gate + (size_t)b * gate_ld, j) : make_float4(1.f, 1.f, 1.f, 1.f);
            v[u] = make_float4(fmaf(g.x, av.x, xv.x), fmaf(g.y, av.y, xv.y), fmaf(g.z, av.z, xv.z),
                               fmaf(g.w, av.w, xv.w));
            o4[j] = v[u];
            ss += dot4(v[u], v[u]);
        }
    }
    if (!w) return;
    const float rs = rsqrtf(warp_sum(ss) / (float)D + eps);
    uint2 *h2 = reinterpret_cast<uint2 *>(h + (size_t)r * D);
#pragma unroll
    for (int u = 0; u < 8; u++) {
        const int j = lane + 32 * u;
        if (j < n4) {
            const float4 ww = ld4(w, j);
            float4 y = make_float4(v[u].x * rs * ww.x, v[u].y * rs * ww.y, v[u].z * rs * ww.z, v[u].w * rs * ww.w);
            if (scale) {
                const float4 s = ld4(scale + (size_t)b * mod_ld, j), t = ld4(shift + (size_t)b * mod_ld, j);
                y = make_float4(y.x * (1.f + s.x) + t.x, y.y * (1.f + s.y) + t.y, y.z * (1.f + s.z) + t.z,
                                y.w * (1.f + s.w) + t.w);
            }
            h2[j] = pack4(y);
        }
    }
}

// Per-head RMSNorm over 64 columns: 8 consecutive lanes own one (row, group), 8 columns each.  Group g of a row
// (g < parts * heads) is columns 64 g .. 64 g + 63; its weight is w0 for g < heads, else w1.
__global__ void __launch_bounds__(256)
qk_norm_fwd_kernel(const __nv_bfloat16 *__restrict__ in, int ld_in, __nv_bfloat16 *__restrict__ out, int ld_out,
                   const float *__restrict__ w0, const float *__restrict__ w1, long long items, int groups,
                   int heads, float eps)
{
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const long long item = t >> 3;
    const int sub = (int)(t & 7);
    const bool live = item < items;
    const long long row = live ? item / groups : 0;
    const int g = live ? (int)(item - row * groups) : 0;
    float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (live) unpack8(*reinterpret_cast<const uint4 *>(in + row * ld_in + 64 * g + 8 * sub), f);
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < 8; i++) ss += f[i] * f[i];
    const float rs = rsqrtf(sum8(ss) * (1.f / 64.f) + eps);
    if (!live) return;
    const float *w = (g < heads ? w0 : w1) + 8 * sub;
#pragma unroll
    for (int i = 0; i < 8; i++) f[i] = f[i] * rs * __ldg(w + i);
    *reinterpret_cast<uint4 *>(out + row * ld_out + 64 * g + 8 * sub) = pack8(f);
}

// Backward of the above over a chunk of 32 rows per CTA: din = bf16(rstd (dn - n mean(dn n))), dn = dout w,
// dw partial += dout n.  The CTA's 32 lane groups ("slots") take the chunk's (row, group) items s, s + 32, ... in
// increasing order (item = row * groups + g); the slot sums are added in slot order.  din may be dout.
__global__ void __launch_bounds__(256)
qk_norm_bwd_kernel(const __nv_bfloat16 *__restrict__ in, int ld_in, const __nv_bfloat16 *dout, int ld_dout,
                   __nv_bfloat16 *din, int ld_din, const float *__restrict__ w0, const float *__restrict__ w1,
                   float *__restrict__ part, int rows, int groups, int heads, float eps)
{
    __shared__ float red[32][2][64];
    const int slot = threadIdx.x >> 3, sub = threadIdx.x & 7;
    const int r0 = blockIdx.x * kChunkRows, r1 = min(rows, r0 + kChunkRows);
    const int items = (r1 - r0) * groups;
    float acc[2][8];
#pragma unroll
    for (int i = 0; i < 8; i++) acc[0][i] = acc[1][i] = 0.f;
    // every lane of a warp runs the same number of iterations (the shuffles need them all): the bound is rounded up
    // to the warp's four slots
    const int iters = (items + 31) / 32;
    for (int k = 0; k < iters; k++) {
        const int it = slot + 32 * k;
        const bool live = it < items;
        const int row = r0 + (live ? it / groups : 0), g = live ? it % groups : 0;
        float u[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, d[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (live) {
            unpack8(*reinterpret_cast<const uint4 *>(in + (size_t)row * ld_in + 64 * g + 8 * sub), u);
            unpack8(*reinterpret_cast<const uint4 *>(dout + (size_t)row * ld_dout + 64 * g + 8 * sub), d);
        }
        float ss = 0.f;
#pragma unroll
        for (int i = 0; i < 8; i++) ss += u[i] * u[i];
        const float rs = rsqrtf(sum8(ss) * (1.f / 64.f) + eps);
        const int part_i = g < heads ? 0 : 1;
        const float *w = (part_i ? w1 : w0) + 8 * sub;
        float dot = 0.f, dn[8];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            u[i] *= rs;                                      // n
            dn[i] = live ? d[i] * __ldg(w + i) : 0.f;
            dot += dn[i] * u[i];
        }
        const float mean = sum8(dot) * (1.f / 64.f);
        if (!live) continue;
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const float v = d[i] * u[i];
            acc[0][i] += part_i ? 0.f : v;           // selects, not a dynamic index: acc stays in registers
            acc[1][i] += part_i ? v : 0.f;
            dn[i] = rs * (dn[i] - u[i] * mean);
        }
        *reinterpret_cast<uint4 *>(din + (size_t)row * ld_din + 64 * g + 8 * sub) = pack8(dn);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) {
        red[slot][0][8 * sub + i] = acc[0][i];
        red[slot][1][8 * sub + i] = acc[1][i];
    }
    __syncthreads();
    const int parts = groups / heads;
    if (threadIdx.x < 64 * parts) {
        const int pi = threadIdx.x >> 6, col = threadIdx.x & 63;
        float s = red[0][pi][col];
        for (int k = 1; k < 32; k++) s += red[k][pi][col];
        part[((size_t)pi * gridDim.x + blockIdx.x) * 64 + col] = s;
    }
}

// out[g, c] = part[g parts, c] + part[g parts + 1, c] + ... in increasing order (ga_launch_partial_sum), one thread
// per output element; T is float or float4, four columns added one by one
template <typename T>
__global__ void partial_sum_kernel(const T *__restrict__ part, T *__restrict__ out, long long n, int parts,
                                   long long cols)
{
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const long long g = i / cols, c = i - g * cols;
    const T *src = part + g * parts * cols + c;
    const auto add = [](T &a, const T &b) {
        if constexpr (sizeof(T) == sizeof(float4)) add4(a, b);
        else a += b;
    };
    T s = src[0];
    int p = 1;
    // sixteen loads in flight before their additions (which stay in order): with a few thousand columns the sum is
    // bound by load latency
    for (; p + 16 <= parts; p += 16) {
        T v[16];
#pragma unroll
        for (int u = 0; u < 16; u++) v[u] = src[(p + u) * cols];
#pragma unroll
        for (int u = 0; u < 16; u++) add(s, v[u]);
    }
    for (; p < parts; p++) add(s, src[p * cols]);
    out[i] = s;
}

bool bad_rows(int R, int rows_per_batch, int D)
{
    return R < 1 || rows_per_batch < 1 || R % rows_per_batch || D < 4 || D % 4 || D > kMaxD;
}

}  // namespace

cudaError_t ga_launch_partial_sum(const float *part, float *out, long long groups, int parts, long long cols,
                                  cudaStream_t s)
{
    // float4 only when a quarter of the columns still gives each of the H100's 132 SMs a CTA: narrower sums (the
    // DiT partials, bias chunks) are latency-bound and run faster with one thread per column
    const bool vec = cols % 4 == 0 && cols / 4 >= 132 * 256 && !mis16(part) && !mis16(out);
    const long long w = vec ? cols / 4 : cols, n = groups * w;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    if (vec)
        partial_sum_kernel<<<blocks, 256, 0, s>>>(reinterpret_cast<const float4 *>(part), reinterpret_cast<float4 *>(out),
                                                  n, parts, w);
    else
        partial_sum_kernel<<<blocks, 256, 0, s>>>(part, out, n, parts, w);
    return cudaGetLastError();
}

extern "C" int ga_dit_grad_partials(int rows, int rows_per_batch)
{
    if (rows < 1 || rows_per_batch < 1 || rows % rows_per_batch) return 0;
    return (rows / rows_per_batch) * ((rows_per_batch + kChunkRows - 1) / kChunkRows);
}

extern "C" int ga_dit_rmsnorm_bwd_validate(const float *dh, const float *x, const float *w, const float *scale,
                                           int mod_ld, const float *dx_in, const float *dx_out, const float *part_dw,
                                           const float *part_dshift, const float *part_dscale, int part_ld,
                                           int rows_per_batch, int R, int D)
{
    if (bad_rows(R, rows_per_batch, D)) return GA_ERR_BADARG;
    if ((long long)R * D >= (1LL << 31)) return GA_ERR_BADARG;
    for (const void *p : {(const void *)dh, (const void *)x, (const void *)w, (const void *)part_dw})
        if (!p || mis16(p)) return GA_ERR_BADARG;
    if (dx_in && (!dx_out || mis16(dx_in))) return GA_ERR_BADARG;
    if (dx_out && mis16(dx_out)) return GA_ERR_BADARG;
    if (scale) {
        if (mis16(scale) || mod_ld < D || mod_ld % 4) return GA_ERR_BADARG;
        if (!part_dshift || !part_dscale || mis16(part_dshift) || mis16(part_dscale) || part_ld < D || part_ld % 4)
            return GA_ERR_BADARG;
    } else if (part_dshift || part_dscale) {
        return GA_ERR_BADARG;
    }
    return 0;
}

extern "C" int ga_dit_rmsnorm_bwd(const float *dh, const float *x, const float *w, const float *scale, int mod_ld,
                                  const float *dx_in, float *dx_out, float *part_dw, float *part_dshift,
                                  float *part_dscale, int part_ld, int rows_per_batch, int R, int D, float eps,
                                  void *stream)
{
    const int rc = ga_dit_rmsnorm_bwd_validate(dh, x, w, scale, mod_ld, dx_in, dx_out, part_dw, part_dshift,
                                               part_dscale, part_ld, rows_per_batch, R, D);
    if (rc) return rc;
    rmsnorm_bwd_kernel<<<ga_dit_grad_partials(R, rows_per_batch), 32 * kWarps, 0, (cudaStream_t)stream>>>(
        dh, x, w, scale, mod_ld, dx_in, dx_out, part_dw, part_dshift, part_dscale, part_ld, rows_per_batch, D, eps);
    return (int)cudaGetLastError();
}

extern "C" int ga_dit_gate_bwd_validate(const float *dy, const float *a, const float *gate, int gate_ld,
                                        const void *da_bf16, const float *part_dgate, int part_ld,
                                        int rows_per_batch, int R, int D)
{
    if (bad_rows(R, rows_per_batch, D)) return GA_ERR_BADARG;
    if ((long long)R * D >= (1LL << 31)) return GA_ERR_BADARG;
    for (const void *p : {(const void *)dy, (const void *)a, (const void *)gate, (const void *)part_dgate})
        if (!p || mis16(p)) return GA_ERR_BADARG;
    if (!da_bf16 || mis8(da_bf16)) return GA_ERR_BADARG;
    if (gate_ld < D || gate_ld % 4 || part_ld < D || part_ld % 4) return GA_ERR_BADARG;
    return 0;
}

extern "C" int ga_dit_gate_bwd(const float *dy, const float *a, const float *gate, int gate_ld, void *da_bf16,
                               float *part_dgate, int part_ld, int rows_per_batch, int R, int D, void *stream)
{
    const int rc = ga_dit_gate_bwd_validate(dy, a, gate, gate_ld, da_bf16, part_dgate, part_ld, rows_per_batch, R, D);
    if (rc) return rc;
    gate_bwd_kernel<<<ga_dit_grad_partials(R, rows_per_batch), 32 * kWarps, 0, (cudaStream_t)stream>>>(
        dy, a, gate, gate_ld, reinterpret_cast<__nv_bfloat16 *>(da_bf16), part_dgate, part_ld, rows_per_batch, D);
    return (int)cudaGetLastError();
}

extern "C" int ga_dit_gate_residual_validate(const float *x, const float *a, const float *gate, int gate_ld,
                                             const float *x_out, const float *w, const float *shift,
                                             const float *scale, int mod_ld, const void *h_bf16,
                                             int rows_per_batch, int R, int D)
{
    if (bad_rows(R, rows_per_batch, D)) return GA_ERR_BADARG;
    if ((long long)R * D >= (1LL << 31)) return GA_ERR_BADARG;
    for (const void *p : {(const void *)x, (const void *)a, (const void *)x_out})
        if (!p || mis16(p)) return GA_ERR_BADARG;
    if (gate && (mis16(gate) || gate_ld < D || gate_ld % 4)) return GA_ERR_BADARG;
    if (!w) return (shift || scale || h_bf16) ? GA_ERR_BADARG : 0;
    if (mis16(w) || !h_bf16 || mis8(h_bf16)) return GA_ERR_BADARG;
    if ((shift == nullptr) != (scale == nullptr)) return GA_ERR_BADARG;
    if (scale && (mis16(shift) || mis16(scale) || mod_ld < D || mod_ld % 4)) return GA_ERR_BADARG;
    return 0;
}

extern "C" int ga_dit_gate_residual(const float *x, const float *a, const float *gate, int gate_ld, float *x_out,
                                    const float *w, const float *shift, const float *scale, int mod_ld, void *h_bf16,
                                    int rows_per_batch, int R, int D, float eps, void *stream)
{
    const int rc = ga_dit_gate_residual_validate(x, a, gate, gate_ld, x_out, w, shift, scale, mod_ld, h_bf16,
                                                 rows_per_batch, R, D);
    if (rc) return rc;
    gate_residual_kernel<<<(R + 7) / 8, 256, 0, (cudaStream_t)stream>>>(
        x, a, gate, gate_ld, x_out, w, shift, scale, mod_ld, reinterpret_cast<__nv_bfloat16 *>(h_bf16),
        rows_per_batch, R, D, eps);
    return (int)cudaGetLastError();
}

extern "C" int ga_dit_qk_norm_validate(int backward, const void *in, int ld_in, const void *dout, int ld_dout,
                                       const void *out, int ld_out, const float *w0, const float *w1,
                                       const float *part_dw, int rows, int heads, int parts)
{
    if (backward != 0 && backward != 1) return GA_ERR_BADARG;
    if (rows < 1 || heads < 1 || (parts != 1 && parts != 2)) return GA_ERR_BADARG;
    const long long width = 64LL * heads * parts;
    if (width > (1LL << 30)) return GA_ERR_BADARG;
    if (!in || mis16(in) || !out || mis16(out) || !w0 || mis16(w0)) return GA_ERR_BADARG;
    if (parts == 2 ? (!w1 || mis16(w1)) : w1 != nullptr) return GA_ERR_BADARG;
    if (ld_in < width || ld_in % 8 || ld_out < width || ld_out % 8) return GA_ERR_BADARG;
    if (!backward) return (dout || part_dw) ? GA_ERR_BADARG : 0;
    if (!dout || mis16(dout) || ld_dout < width || ld_dout % 8 || !part_dw || mis16(part_dw)) return GA_ERR_BADARG;
    return 0;
}

extern "C" int ga_dit_qk_norm_fwd_bf16(const void *in, int ld_in, void *out, int ld_out, const float *w0,
                                       const float *w1, int rows, int heads, int parts, float eps, void *stream)
{
    const int rc = ga_dit_qk_norm_validate(0, in, ld_in, nullptr, 0, out, ld_out, w0, w1, nullptr, rows, heads,
                                           parts);
    if (rc) return rc;
    const long long items = (long long)rows * heads * parts;
    qk_norm_fwd_kernel<<<(unsigned)((items * 8 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __nv_bfloat16 *>(in), ld_in, reinterpret_cast<__nv_bfloat16 *>(out), ld_out, w0,
        w1 ? w1 : w0, items, heads * parts, heads, eps);
    return (int)cudaGetLastError();
}

extern "C" int ga_dit_qk_norm_bwd_bf16(const void *in, int ld_in, const void *dout, int ld_dout, void *din,
                                       int ld_din, const float *w0, const float *w1, float *part_dw, int rows,
                                       int heads, int parts, float eps, void *stream)
{
    const int rc = ga_dit_qk_norm_validate(1, in, ld_in, dout, ld_dout, din, ld_din, w0, w1, part_dw, rows, heads,
                                           parts);
    if (rc) return rc;
    qk_norm_bwd_kernel<<<ga_dit_grad_partials(rows, rows), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const __nv_bfloat16 *>(in), ld_in, reinterpret_cast<const __nv_bfloat16 *>(dout), ld_dout,
        reinterpret_cast<__nv_bfloat16 *>(din), ld_din, w0, w1 ? w1 : w0, part_dw, rows, heads * parts, heads, eps);
    return (int)cudaGetLastError();
}

extern "C" int ga_dit_grad_reduce_validate(const float *part, const float *out, int groups, int parts, int cols)
{
    return (!part || !out || groups < 1 || parts < 1 || cols < 1) ? GA_ERR_BADARG : 0;
}

extern "C" int ga_dit_grad_reduce(const float *part, float *out, int groups, int parts, int cols, void *stream)
{
    const int rc = ga_dit_grad_reduce_validate(part, out, groups, parts, cols);
    if (rc) return rc;
    return (int)ga_launch_partial_sum(part, out, groups, parts, cols, (cudaStream_t)stream);
}
