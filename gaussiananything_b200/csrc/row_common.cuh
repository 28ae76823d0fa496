// Shared pieces of the row-wise and training kernels (DiT, VAE, attention, linear gradients): warp sums, float4
// arithmetic, SiLU and tanh-GELU with their gradients, bf16 packing, the chunked partials of the DiT gradients
// (include/ga_b200.h Parts 14-15) and the host-side alignment tests.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ga_row {

// ---- partials of the DiT gradients: one fp32 partial per chunk of kChunkRows rows (ga_dit_grad_partials)
constexpr int kChunkRows = 32;          // rows per partial
constexpr int kWarps = 8;               // warps per CTA of the row kernels
constexpr int kMaxD = 1024;             // widest row kept in registers (8 float4 per lane)

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---- float4
__device__ __forceinline__ float4 ld4(const float *p, int i) { return __ldg(reinterpret_cast<const float4 *>(p) + i); }
__device__ __forceinline__ float dot4(float4 a, float4 b) { return a.x * b.x + a.y * b.y + a.z * b.z + a.w * b.w; }
__device__ __forceinline__ float sum4(float4 a) { return a.x + a.y + a.z + a.w; }
__device__ __forceinline__ float4 mul4(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float4 scale4(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ void add4(float4 &a, float4 b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
__device__ __forceinline__ void fma4(float4 &a, float s, float4 b)
{
    a.x = fmaf(s, b.x, a.x); a.y = fmaf(s, b.y, a.y); a.z = fmaf(s, b.z, a.z); a.w = fmaf(s, b.w, a.w);
}
__device__ __forceinline__ float4 zero4() { return make_float4(0.f, 0.f, 0.f, 0.f); }

// ---- activations
__device__ __forceinline__ float silu(float x) { return x / (1.0f + __expf(-x)); }
__device__ __forceinline__ float silu_grad(float x)
{
    const float s = 1.0f / (1.0f + __expf(-x));
    return s * (1.0f + x * (1.0f - s));
}
__device__ __forceinline__ float4 silu4(float4 v) { return make_float4(silu(v.x), silu(v.y), silu(v.z), silu(v.w)); }

// 0.5 x (1 + tanh(k0 (x + k1 x^3)))
__device__ __forceinline__ float gelu_tanh(float x)
{
    const float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
    return 0.5f * x * (1.0f + tanhf(u));
}
__device__ __forceinline__ float gelu_tanh_grad(float v)
{
    const float k0 = 0.7978845608028654f, k1 = 0.044715f;
    const float th = tanhf(k0 * (v + k1 * v * v * v));
    return 0.5f * (1.0f + th) + 0.5f * v * (1.0f - th * th) * k0 * (1.0f + 3.0f * k1 * v * v);
}

// ---- bf16 packing (round to nearest even)
__device__ __forceinline__ uint32_t pack_bf16(float a, float b)
{
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&h);
}
__device__ __forceinline__ uint2 pack4(float4 v) { return make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w)); }
__device__ __forceinline__ uint4 pack8(const float (&f)[8])
{
    return make_uint4(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]), pack_bf16(f[4], f[5]), pack_bf16(f[6], f[7]));
}
__device__ __forceinline__ void unpack8(uint4 u, float (&f)[8])
{
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const float2 p = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&w[i]));
        f[2 * i] = p.x;
        f[2 * i + 1] = p.y;
    }
}

// The CTA's sum of acc (float4 index lane + 32 u of each warp), warps added in warp order, written to out[0, D).
__device__ __forceinline__ void cta_colsum(float4 (*red)[kMaxD / 4], const float4 (&acc)[8], float *out, int n4)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int u = 0; u < 8; u++)
        if (lane + 32 * u < n4) red[warp][lane + 32 * u] = acc[u];
    __syncthreads();
    for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        float4 s = red[0][i];
#pragma unroll
        for (int w = 1; w < kWarps; w++) add4(s, red[w][i]);
        reinterpret_cast<float4 *>(out)[i] = s;
    }
    __syncthreads();
}

// ---- host
static inline bool mis16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }
static inline bool mis8(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 7) != 0; }
static inline bool mis4(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 3) != 0; }

}  // namespace ga_row

// out[g, c] = part[g parts, c] + part[g parts + 1, c] + ... + part[g parts + parts - 1, c] in fp32, in that order, for
// g < groups, c < cols; part is [groups * parts, cols], out [groups, cols].  Reads four columns at a time when cols is a
// large multiple of 4 (the wgrad split sums) and both pointers are 16-byte aligned.  Defined in dit_grad.cu.
cudaError_t ga_launch_partial_sum(const float *part, float *out, long long groups, int parts, long long cols,
                                  cudaStream_t s);
