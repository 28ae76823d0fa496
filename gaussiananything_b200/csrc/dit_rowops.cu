// Row-wise / small kernels of the DiT denoiser (everything that is not a
// wgmma contraction): fused RMSNorm + adaLN modulate, the timestep /
// pooled-vector / adaLN prologue, the token embedder, the final layer with the
// classifier-free-guidance combine, and the ODE state update.
// Math follows /root/reference/dit/dit_i23d.py:511-567,707-750,
// /root/reference/dit/dit_models_xformers.py:62-128 and /root/reference/dit/norm.py.
#include "../../include/ga_b200.h"
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <cstdlib>

namespace {

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float silu(float x) { return x / (1.0f + __expf(-x)); }
__device__ __forceinline__ float gelu_tanh(float x)
{
    const float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
    return 0.5f * x * (1.0f + tanhf(u));
}

// out_bf16[r, :] = RMSNorm(x[r, :]) * w  [* (1 + scale[b]) + shift[b]]      one warp per row; the row is kept in
// registers (D <= 1024: 8 float4 per lane) so x is read once.
__global__ void __launch_bounds__(256)
rmsnorm_modulate_kernel(const float *__restrict__ x, const float *__restrict__ w,
                        const float *__restrict__ shift, const float *__restrict__ scale, int mod_ld,
                        int rows_per_batch, __nv_bfloat16 *__restrict__ out, int R, int D, float eps)
{
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    asm volatile("griddepcontrol.wait;\n" ::: "memory");            // x comes from the previous GEMM's epilogue
    asm volatile("griddepcontrol.launch_dependents;\n" ::: "memory");
    if (r >= R) return;
    const float4 *xr = reinterpret_cast<const float4 *>(x + (size_t)r * D);
    const int n4 = D >> 2;
    float4 cache[8];
    float ss = 0.f;
#pragma unroll
    for (int u = 0; u < 8; u++) {
        const int i = lane + 32 * u;
        if (i < n4) {
            const float4 v = xr[i];
            cache[u] = v;
            ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
        }
    }
    for (int i = lane + 256; i < n4; i += 32) {          // D > 1024: tail re-read below
        const float4 v = xr[i];
        ss += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    }
    ss = warp_sum(ss);
    const float rs = rsqrtf(ss / (float)D + eps);
    const int b = r / rows_per_batch;
    const float4 *w4 = reinterpret_cast<const float4 *>(w);
    const float4 *sh4 = shift ? reinterpret_cast<const float4 *>(shift + (size_t)b * mod_ld) : nullptr;
    const float4 *sc4 = scale ? reinterpret_cast<const float4 *>(scale + (size_t)b * mod_ld) : nullptr;
    uint2 *o = reinterpret_cast<uint2 *>(out + (size_t)r * D);
    auto emit = [&](int i, const float4 v) {
        const float4 ww = __ldg(w4 + i);
        float4 y = make_float4(v.x * rs * ww.x, v.y * rs * ww.y, v.z * rs * ww.z, v.w * rs * ww.w);
        if (sc4) {
            const float4 s = __ldg(sc4 + i), t = __ldg(sh4 + i);
            y.x = y.x * (1.f + s.x) + t.x; y.y = y.y * (1.f + s.y) + t.y;
            y.z = y.z * (1.f + s.z) + t.z; y.w = y.w * (1.f + s.w) + t.w;
        }
        __nv_bfloat162 a = __floats2bfloat162_rn(y.x, y.y), c = __floats2bfloat162_rn(y.z, y.w);
        o[i] = make_uint2(*reinterpret_cast<uint32_t *>(&a), *reinterpret_cast<uint32_t *>(&c));
    };
#pragma unroll
    for (int u = 0; u < 8; u++) {
        const int i = lane + 32 * u;
        if (i < n4) emit(i, cache[u]);
    }
    for (int i = lane + 256; i < n4; i += 32) emit(i, xr[i]);
}

// y[b, n] = act_out( bias[n] + sum_k act_in(x[b, k]) * W[n, k] )   small batch (<= 16 rows), fp32
// one warp per output column n, all batch rows at once.
__global__ void __launch_bounds__(256)
linear_small_kernel(const float *__restrict__ x, const float *__restrict__ W, const float *__restrict__ bias,
                    float *__restrict__ y, int Bn, int N, int K, int act_in, int act_out, int accumulate)
{
    const int n = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= N) return;
    float acc[16];
#pragma unroll
    for (int b = 0; b < 16; b++) acc[b] = 0.f;
    const float *wr = W + (size_t)n * K;
    if ((K & 127) == 0 && K <= 1024) {
        // the whole weight row is fetched up front (<= 8 independent 16-byte loads per lane): with the scalar loop
        // below the 24 dependent-latency iterations made this a 25 us kernel for 14 MB of weights
        const float4 *w4 = reinterpret_cast<const float4 *>(wr);
        float4 wv[8];
#pragma unroll
        for (int u = 0; u < 8; u++)
            wv[u] = (lane + 32 * u) * 4 < K ? __ldg(w4 + lane + 32 * u) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int b = 0; b < 16; b++) {
            if (b < Bn) {
                const float4 *x4 = reinterpret_cast<const float4 *>(x + (size_t)b * K);
#pragma unroll
                for (int u = 0; u < 8; u++) {
                    if ((lane + 32 * u) * 4 < K) {
                        float4 xv = x4[lane + 32 * u];
                        if (act_in == 1) { xv.x = silu(xv.x); xv.y = silu(xv.y); xv.z = silu(xv.z); xv.w = silu(xv.w); }
                        acc[b] += xv.x * wv[u].x + xv.y * wv[u].y + xv.z * wv[u].z + xv.w * wv[u].w;
                    }
                }
            }
        }
    } else {
        for (int k = lane; k < K; k += 32) {
            const float wv = wr[k];
#pragma unroll
            for (int b = 0; b < 16; b++) {
                if (b < Bn) {
                    float xv = x[(size_t)b * K + k];
                    if (act_in == 1) xv = silu(xv);
                    acc[b] += xv * wv;
                }
            }
        }
    }
#pragma unroll
    for (int b = 0; b < 16; b++) {
        if (b < Bn) {
            float v = warp_sum(acc[b]);
            if (lane == 0) {
                v += bias ? bias[n] : 0.f;
                if (act_out == 1) v = silu(v);
                if (accumulate) v += y[(size_t)b * N + n];
                y[(size_t)b * N + n] = v;
            }
        }
    }
}

// timestep_embedding(t, 256): [cos(t f_i) | sin(t f_i)], f_i = exp(-ln(1e4) i / 128)
__global__ void timestep_sinusoid_kernel(const float *__restrict__ t, float *__restrict__ out, int Bn, int dim)
{
    const int b = blockIdx.x, i = threadIdx.x, half = dim / 2;
    if (b >= Bn || i >= half) return;
    const float freq = expf(-logf(10000.0f) * (float)i / (float)half);
    const float a = t[b] * freq;
    out[(size_t)b * dim + i] = cosf(a);
    out[(size_t)b * dim + half + i] = sinf(a);
}

// LayerNorm over the last dim (affine optional), fp32 in/out, one warp per row
__global__ void __launch_bounds__(256)
layernorm_rows_kernel(const float *__restrict__ x, const float *__restrict__ w, const float *__restrict__ bvec,
                      float *__restrict__ y, int R, int D, float eps)
{
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= R) return;
    const float *xr = x + (size_t)r * D;
    if ((D & 3) == 0 && D <= 1024) {
        // row in registers: one round of independent 16-byte loads instead of three dependent passes
        const float4 *x4 = reinterpret_cast<const float4 *>(xr);
        const int n4 = D >> 2;
        float4 cache[8];
        float s = 0.f;
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int i = lane + 32 * u;
            cache[u] = i < n4 ? x4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
            s += cache[u].x + cache[u].y + cache[u].z + cache[u].w;
        }
        const float mean = warp_sum(s) / (float)D;
        float v = 0.f;
#pragma unroll
        for (int u = 0; u < 8; u++) {
            if (lane + 32 * u < n4) {
                const float d0 = cache[u].x - mean, d1 = cache[u].y - mean, d2 = cache[u].z - mean, d3 = cache[u].w - mean;
                v += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
            }
        }
        const float rs = rsqrtf(warp_sum(v) / (float)D + eps);
        float4 *y4 = reinterpret_cast<float4 *>(y + (size_t)r * D);
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int i = lane + 32 * u;
            if (i < n4) {
                float4 o = make_float4((cache[u].x - mean) * rs, (cache[u].y - mean) * rs, (cache[u].z - mean) * rs,
                                       (cache[u].w - mean) * rs);
                if (w) {
                    const float4 ww = __ldg(reinterpret_cast<const float4 *>(w) + i);
                    const float4 bb = bvec ? __ldg(reinterpret_cast<const float4 *>(bvec) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
                    o.x = o.x * ww.x + bb.x; o.y = o.y * ww.y + bb.y; o.z = o.z * ww.z + bb.z; o.w = o.w * ww.w + bb.w;
                }
                y4[i] = o;
            }
        }
        return;
    }
    float s = 0.f;
    for (int i = lane; i < D; i += 32) s += xr[i];
    const float mean = warp_sum(s) / (float)D;
    float v = 0.f;
    for (int i = lane; i < D; i += 32) { const float d = xr[i] - mean; v += d * d; }
    const float rs = rsqrtf(warp_sum(v) / (float)D + eps);
    for (int i = lane; i < D; i += 32) {
        float o = (xr[i] - mean) * rs;
        if (w) o = o * w[i] + (bvec ? bvec[i] : 0.f);
        y[(size_t)r * D + i] = o;
    }
}

// mod[l, b, j, :] = table[l, j, :] + t0[b, j, :]        (j = 0..J-1)
__global__ void add_tables_kernel(const float *__restrict__ tables, const float *__restrict__ t0,
                                  float *__restrict__ mod, int L, int Bn, int JD, int t0_ld)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t total = (size_t)L * Bn * JD;
    if (i >= total) return;
    const int e = (int)(i % JD);
    const int b = (int)((i / JD) % Bn);
    const int l = (int)(i / ((size_t)JD * Bn));
    mod[i] = tables[(size_t)l * JD + e] + t0[(size_t)b * t0_ld + (e % t0_ld)];
}

// token embedder first layer: h[r, n] = gelu_tanh(b1[n] + sum_c in[r, c] W1[n, c]) -> bf16   (tiny K)
__global__ void __launch_bounds__(256)
embed_fc1_kernel(const float *__restrict__ xin, int Cx, const float *__restrict__ xin2, int C2,
                 const float *__restrict__ W1, const float *__restrict__ b1, __nv_bfloat16 *__restrict__ h,
                 int R, int D)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)R * D) return;
    const int r = (int)(i / D), n = (int)(i % D);
    const int K = Cx + C2;
    float acc = b1[n];
    // optional second input is concatenated FIRST (stage-2 concat mode: cat([fps_xyz, x]), dit_i23d.py:739)
    for (int c = 0; c < C2; c++) acc += xin2[(size_t)r * C2 + c] * W1[(size_t)n * K + c];
    for (int c = 0; c < Cx; c++) acc += xin[(size_t)r * Cx + c] * W1[(size_t)n * K + C2 + c];
    h[i] = __float2bfloat16(gelu_tanh(acc));
}

// NeRF positional encoding of xyz (utils/nerf_utils.py:50-65, multires 10): [x, sin(2^k x), cos(2^k x)]_k,
// 63 features padded to 64 (bf16) so the projection is one wgmma GEMM with K = 64.
__global__ void xyz_pe_kernel(const float *__restrict__ xyz, __nv_bfloat16 *__restrict__ out, int R)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    const float p[3] = {xyz[(size_t)r * 3], xyz[(size_t)r * 3 + 1], xyz[(size_t)r * 3 + 2]};
    __nv_bfloat16 *o = out + (size_t)r * 64;
    for (int c = 0; c < 3; c++) o[c] = __float2bfloat16(p[c]);
    float f = 1.0f;
    for (int k = 0; k < 10; k++) {
        for (int c = 0; c < 3; c++) {
            o[3 + 6 * k + c] = __float2bfloat16(sinf(p[c] * f));
            o[3 + 6 * k + 3 + c] = __float2bfloat16(cosf(p[c] * f));
        }
        f *= 2.0f;
    }
    o[63] = __float2bfloat16(0.f);
}

// final layer (T2IFinalLayer): y[r, c] = bias[c] + sum_d (LN(x[r])[d] * (1 + scale[b, d]) + shift[b, d]) * W[c, d]
// one warp per row; Cout <= 16.  mod = [B, 2, D] (shift, scale).
__global__ void __launch_bounds__(256)
final_layer_kernel(const float *__restrict__ x, const float *__restrict__ mod, const float *__restrict__ W,
                   const float *__restrict__ bias, float *__restrict__ y, int R, int D, int Cout,
                   int rows_per_batch, float eps)
{
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= R) return;
    const float *xr = x + (size_t)r * D;
    const int b = r / rows_per_batch;
    const float *sh = mod + (size_t)b * 2 * D, *sc = sh + D;
    float acc[16];
#pragma unroll
    for (int c = 0; c < 16; c++) acc[c] = 0.f;
    if ((D & 3) == 0 && D <= 1024) {
        // the row lives in registers (8 float4 per lane): x is read once, all loads in flight together
        const float4 *x4 = reinterpret_cast<const float4 *>(xr);
        const int n4 = D >> 2;
        float4 cache[8];
        float s = 0.f;
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int i = lane + 32 * u;
            cache[u] = i < n4 ? x4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
            s += cache[u].x + cache[u].y + cache[u].z + cache[u].w;
        }
        const float mean = warp_sum(s) / (float)D;
        float v = 0.f;
#pragma unroll
        for (int u = 0; u < 8; u++) {
            if (lane + 32 * u < n4) {
                const float d0 = cache[u].x - mean, d1 = cache[u].y - mean, d2 = cache[u].z - mean, d3 = cache[u].w - mean;
                v += d0 * d0 + d1 * d1 + d2 * d2 + d3 * d3;
            }
        }
        const float rs = rsqrtf(warp_sum(v) / (float)D + eps);
        const float4 *sh4 = reinterpret_cast<const float4 *>(sh), *sc4 = reinterpret_cast<const float4 *>(sc);
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int i = lane + 32 * u;
            if (i < n4) {
                const float4 a = __ldg(sc4 + i), t = __ldg(sh4 + i);
                const float h0 = (cache[u].x - mean) * rs * (1.f + a.x) + t.x, h1 = (cache[u].y - mean) * rs * (1.f + a.y) + t.y;
                const float h2 = (cache[u].z - mean) * rs * (1.f + a.z) + t.z, h3 = (cache[u].w - mean) * rs * (1.f + a.w) + t.w;
#pragma unroll
                for (int c = 0; c < 16; c++) {
                    if (c < Cout) {
                        const float4 w = __ldg(reinterpret_cast<const float4 *>(W + (size_t)c * D) + i);
                        acc[c] += h0 * w.x + h1 * w.y + h2 * w.z + h3 * w.w;
                    }
                }
            }
        }
    } else {
        float s = 0.f;
        for (int i = lane; i < D; i += 32) s += xr[i];
        const float mean = warp_sum(s) / (float)D;
        float v = 0.f;
        for (int i = lane; i < D; i += 32) { const float d = xr[i] - mean; v += d * d; }
        const float rs = rsqrtf(warp_sum(v) / (float)D + eps);
        for (int i = lane; i < D; i += 32) {
            const float h = (xr[i] - mean) * rs * (1.f + sc[i]) + sh[i];
#pragma unroll
            for (int c = 0; c < 16; c++)
                if (c < Cout) acc[c] += h * W[(size_t)c * D + i];
        }
    }
#pragma unroll
    for (int c = 0; c < 16; c++) {
        if (c < Cout) {
            const float t = warp_sum(acc[c]);
            if (lane == 0) y[(size_t)r * Cout + c] = t + bias[c];
        }
    }
}

// classifier-free guidance (dit_i23d.py:159-172): eps [2B, n] -> h = u + s (c - u), written to both halves
__global__ void cfg_combine_kernel(const float *__restrict__ eps, float *__restrict__ out, size_t half, float s)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= half) return;
    const float c = eps[i], u = eps[half + i];
    const float h = u + s * (c - u);
    out[i] = h;
    out[half + i] = h;
}

__global__ void axpy_kernel(float *__restrict__ x, const float *__restrict__ v, float a, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) x[i] += a * v[i];
}

__global__ void f32_to_bf16_kernel(const float *__restrict__ x, __nv_bfloat16 *__restrict__ y, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = __float2bfloat16(x[i]);
}

inline int last_err() { return (int)cudaGetLastError(); }

}  // namespace

extern "C" int ga_rmsnorm_modulate(const float *x, const float *w, const float *shift, const float *scale,
                                   int mod_ld, int rows_per_batch, void *out_bf16, int R, int D, float eps,
                                   void *stream)
{
    if (!x || !w || !out_bf16 || R <= 0 || D <= 0 || D % 4 || rows_per_batch <= 0) return GA_ERR_BADARG;
    if ((shift == nullptr) != (scale == nullptr)) return GA_ERR_BADARG;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((R + 7) / 8); cfg.blockDim = dim3(256); cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    static int use_pdl = -1;
    if (use_pdl < 0) { const char *e = getenv("GA_B200_PDL"); use_pdl = (e && e[0] == '0') ? 0 : 1; }
    cfg.attrs = attr; cfg.numAttrs = use_pdl ? 1 : 0;
    return (int)cudaLaunchKernelEx(&cfg, rmsnorm_modulate_kernel, x, w, shift, scale, mod_ld, rows_per_batch,
                                   reinterpret_cast<__nv_bfloat16 *>(out_bf16), R, D, eps);
}

extern "C" int ga_linear_small(const float *x, const float *W, const float *bias, float *y, int rows, int N, int K,
                               int act_in, int act_out, int accumulate, void *stream)
{
    if (!x || !W || !y || rows <= 0 || rows > 16 || N <= 0 || K <= 0) return GA_ERR_BADARG;
    linear_small_kernel<<<(N + 7) / 8, 256, 0, (cudaStream_t)stream>>>(x, W, bias, y, rows, N, K, act_in, act_out,
                                                                       accumulate);
    return last_err();
}

extern "C" int ga_timestep_sinusoid(const float *t, float *out, int rows, int dim, void *stream)
{
    if (!t || !out || rows <= 0 || dim <= 0 || dim % 2 || dim / 2 > 1024) return GA_ERR_BADARG;
    timestep_sinusoid_kernel<<<rows, dim / 2, 0, (cudaStream_t)stream>>>(t, out, rows, dim);
    return last_err();
}

extern "C" int ga_layernorm_rows(const float *x, const float *w, const float *b, float *y, int R, int D, float eps,
                                 void *stream)
{
    if (!x || !y || R <= 0 || D <= 0) return GA_ERR_BADARG;
    layernorm_rows_kernel<<<(R + 7) / 8, 256, 0, (cudaStream_t)stream>>>(x, w, b, y, R, D, eps);
    return last_err();
}

extern "C" int ga_add_tables(const float *tables, const float *t0, float *mod, int L, int rows, int JD, int t0_ld,
                             void *stream)
{
    if (!tables || !t0 || !mod || L <= 0 || rows <= 0 || JD <= 0 || t0_ld <= 0) return GA_ERR_BADARG;
    const size_t total = (size_t)L * rows * JD;
    add_tables_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(tables, t0, mod, L, rows, JD,
                                                                                        t0_ld);
    return last_err();
}

extern "C" int ga_embed_fc1(const float *xin, int Cx, const float *xin2, int C2, const float *W1, const float *b1,
                            void *h_bf16, int R, int D, void *stream)
{
    if (!xin || !W1 || !b1 || !h_bf16 || R <= 0 || D <= 0 || Cx <= 0 || (C2 > 0 && !xin2)) return GA_ERR_BADARG;
    const size_t total = (size_t)R * D;
    embed_fc1_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        xin, Cx, xin2, C2, W1, b1, reinterpret_cast<__nv_bfloat16 *>(h_bf16), R, D);
    return last_err();
}

extern "C" int ga_xyz_posenc(const float *xyz, void *out_bf16, int R, void *stream)
{
    if (!xyz || !out_bf16 || R <= 0) return GA_ERR_BADARG;
    xyz_pe_kernel<<<(R + 127) / 128, 128, 0, (cudaStream_t)stream>>>(xyz, reinterpret_cast<__nv_bfloat16 *>(out_bf16), R);
    return last_err();
}

extern "C" int ga_final_layer(const float *x, const float *mod, const float *W, const float *bias, float *y, int R,
                              int D, int Cout, int rows_per_batch, float eps, void *stream)
{
    if (!x || !mod || !W || !bias || !y || R <= 0 || D <= 0 || Cout <= 0 || Cout > 16) return GA_ERR_BADARG;
    final_layer_kernel<<<(R + 7) / 8, 256, 0, (cudaStream_t)stream>>>(x, mod, W, bias, y, R, D, Cout, rows_per_batch,
                                                                      eps);
    return last_err();
}

extern "C" int ga_cfg_combine(const float *eps, float *out, int64_t half_elems, float cfg_scale, void *stream)
{
    if (!eps || !out || half_elems <= 0) return GA_ERR_BADARG;
    cfg_combine_kernel<<<(unsigned)((half_elems + 255) / 256), 256, 0, (cudaStream_t)stream>>>(eps, out,
                                                                                               (size_t)half_elems,
                                                                                               cfg_scale);
    return last_err();
}

extern "C" int ga_axpy(float *x, const float *v, float a, int64_t n, void *stream)
{
    if (!x || !v || n <= 0) return GA_ERR_BADARG;
    axpy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, v, a, (size_t)n);
    return last_err();
}

extern "C" int ga_f32_to_bf16(const float *x, void *y, int64_t n, void *stream)
{
    if (!x || !y || n <= 0) return GA_ERR_BADARG;
    f32_to_bf16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        x, reinterpret_cast<__nv_bfloat16 *>(y), (size_t)n);
    return last_err();
}
