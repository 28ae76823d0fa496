// DINOv2 image conditioner (SURVEY.md 8f row N3): the two steps around the ViT-L blocks that the DiT kernels do not
// already cover.
//   frontend : image [B,3,H,W] fp32 in [-1,1] -> optional separable Gaussian blur (kornia's antialias for
//              downscaling) -> bicubic align_corners=True resize -> (x+1)/2 -> ImageNet normalisation -> the bf16
//              im2col matrix [B*np*np, k_pitch] of the patch-embed GEMM (column c*p*p + ky*p + kx, i.e.
//              proj.weight.reshape(D, 3*p*p); columns >= 3*p*p are zero)
//   tokens   : patch-embed output + cls / register tokens + pos_embed -> the fp32 residual stream
//              [B, 1 + n_reg + n_patch, D] in the order cls | registers | patches (registers get no pos_embed)
// Math follows /root/reference/sgm/modules/encoders/modules.py:862-875 and the DINOv2 token preparation; the checker
// is oracle/dino_oracle.py.  The front end runs in fp32 whatever the caller's image dtype.
#include "../../include/ga_b200.h"
#include "row_common.cuh"
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>

namespace {

constexpr int kMaxSide = 4096;
constexpr int kMaxTaps = 1024;              // Gaussian taps held in shared memory by the blur pass

// torch's 'reflect' padding: the edge sample is not repeated
__device__ __forceinline__ int reflect_index(int i, int n)
{
    if (n == 1) return 0;
    while (i < 0 || i >= n) i = i < 0 ? -i : 2 * (n - 1) - i;
    return i;
}

// One pass of a separable, normalised Gaussian exp(-x^2 / 2 sigma^2), x = i - ks/2, over planes [planes, H, W]:
// axis 0 filters along x, axis 1 along y.  Every block builds the normalised taps in shared memory.
__global__ void __launch_bounds__(256)
blur_pass_kernel(const float *__restrict__ in, float *__restrict__ out, long long planes, int H, int W, int axis, int ks,
                 float sigma)
{
    __shared__ float w[kMaxTaps];
    __shared__ float wsum;
    const int r = ks / 2;
    const float den = 2.0f * (sigma * sigma);
    for (int i = threadIdx.x; i < ks; i += blockDim.x) {
        const float x = (float)(i - r);
        w[i] = expf(-(x * x) / den);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int i = 0; i < ks; i++) s += w[i];
        wsum = s;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < ks; i += blockDim.x) w[i] = w[i] / wsum;
    __syncthreads();
    const long long total = planes * H * W;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(e % W);
        const long long py = e / W;
        const int y = (int)(py % H);
        const float *pl = in + (py / H) * H * (long long)W;
        float acc = 0.f;
        if (axis == 0) {
            const float *row = pl + (size_t)y * W;
            for (int i = 0; i < ks; i++) acc += w[i] * row[reflect_index(x + i - r, W)];
        } else {
            for (int i = 0; i < ks; i++) acc += w[i] * pl[(size_t)reflect_index(y + i - r, H) * W + x];
        }
        out[e] = acc;
    }
}

// PyTorch's bicubic convolution (A = -0.75) and its align_corners=True source index with clamped border taps
__device__ __forceinline__ float cubic_near(float x) { return ((1.25f * x - 2.25f) * x) * x + 1.f; }           // |x| <= 1
__device__ __forceinline__ float cubic_far(float x) { return ((-0.75f * x + 3.75f) * x - 6.f) * x + 3.f; }     // 1 < |x| < 2

__device__ __forceinline__ void cubic_taps(int o, int n_in, float scale, int (&idx)[4], float (&w)[4])
{
    const float real = scale * (float)o;
    const int i0 = min((int)floorf(real), n_in - 1);
    const float t = fminf(fmaxf(real - (float)i0, 0.f), 1.f);
    w[0] = cubic_far(t + 1.f);
    w[1] = cubic_near(t);
    w[2] = cubic_near(1.f - t);
    w[3] = cubic_far(2.f - t);
#pragma unroll
    for (int j = 0; j < 4; j++) idx[j] = min(max(i0 - 1 + j, 0), n_in - 1);
}

struct Norm { float mean[3], std[3]; };

// one thread per element of the patch matrix [B * np * np, k_pitch]
__global__ void __launch_bounds__(256)
patch_matrix_kernel(const float *__restrict__ src, int H, int W, int p, int np, int k_pitch, int resize,
                    float scale_y, float scale_x, Norm nrm, __nv_bfloat16 *__restrict__ out, long long total)
{
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int col = (int)(e % k_pitch);
    const long long row = e / k_pitch;
    const int pp = p * p;
    if (col >= 3 * pp) {
        out[e] = __float2bfloat16(0.f);
        return;
    }
    const int npp = np * np;
    const long long b = row / npp;
    const int t = (int)(row % npp);
    const int c = col / pp, ky = (col % pp) / p, kx = col % p;
    const int oy = (t / np) * p + ky, ox = (t % np) * p + kx;
    const float *pl = src + (b * 3 + c) * H * (long long)W;
    float v;
    if (!resize) {
        v = pl[(size_t)oy * W + ox];                        // S == H == W: kornia returns the input unchanged
    } else {
        int iy[4], ix[4];
        float wy[4], wx[4];
        cubic_taps(oy, H, scale_y, iy, wy);
        cubic_taps(ox, W, scale_x, ix, wx);
        v = 0.f;
#pragma unroll
        for (int k = 0; k < 4; k++) {                       // along x first, then the four rows along y
            const float *rw = pl + (size_t)iy[k] * W;
            float h = 0.f;
#pragma unroll
            for (int j = 0; j < 4; j++) h += rw[ix[j]] * wx[j];
            v += h * wy[k];
        }
    }
    // (x + 1) / 2, then (x - mean) / std: explicitly rounded, so no contraction changes the fp32 result
    const float u = __fdiv_rn(__fadd_rn(v, 1.0f), 2.0f);
    const float mean = c == 0 ? nrm.mean[0] : (c == 1 ? nrm.mean[1] : nrm.mean[2]);
    const float sd = c == 0 ? nrm.std[0] : (c == 1 ? nrm.std[1] : nrm.std[2]);
    out[e] = __float2bfloat16(__fdiv_rn(__fsub_rn(u, mean), sd));
}

// x[b, t, :]: t = 0 cls + pos[0]; 1 .. n_reg registers; then patch j = t - 1 - n_reg: patch_out[b, j] + pos[1 + j]
__global__ void __launch_bounds__(256)
tokens_kernel(const float4 *__restrict__ patch_out, const float4 *__restrict__ cls, const float4 *__restrict__ reg,
              int n_reg, const float4 *__restrict__ pos, float4 *__restrict__ x, int n_patch, int D4, long long total)
{
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int d = (int)(e % D4);
    const long long r = e / D4;
    const int nt = 1 + n_reg + n_patch;
    const long long b = r / nt;
    const int t = (int)(r % nt);
    float4 v;
    if (t == 0) {
        const float4 a = cls[d], q = pos[d];
        v = make_float4(a.x + q.x, a.y + q.y, a.z + q.z, a.w + q.w);
    } else if (t <= n_reg) {
        v = reg[(size_t)(t - 1) * D4 + d];
    } else {
        const int j = t - 1 - n_reg;
        const float4 a = patch_out[((size_t)b * n_patch + j) * D4 + d], q = pos[(size_t)(1 + j) * D4 + d];
        v = make_float4(a.x + q.x, a.y + q.y, a.z + q.z, a.w + q.w);
    }
    x[e] = v;
}

inline int last_err() { return (int)cudaGetLastError(); }

// kornia.geometry.resize(antialias=True): blur only when downscaling; sigma = max((H/S - 1) / 2, 0.001),
// ks = int(max(4 sigma, 3)) made odd
bool needs_blur(int H, int W, int S) { return H > S || W > S; }
void blur_params(int n, int S, float *sigma, int *ks)
{
    const double s = fmax(((double)n / (double)S - 1.0) / 2.0, 0.001);
    int k = (int)fmax(4.0 * s, 3.0);
    if (k % 2 == 0) k += 1;
    *sigma = (float)s;
    *ks = k;
}

}  // namespace

extern "C" size_t ga_dino_frontend_scratch_bytes(int batch, int H, int W, int out_size)
{
    if (batch <= 0 || H <= 0 || W <= 0 || out_size <= 0 || !needs_blur(H, W, out_size)) return 0;
    return 2 * (size_t)batch * 3 * (size_t)H * (size_t)W * sizeof(float);
}

extern "C" int ga_dino_frontend(const float *img, int batch, int H, int W, int out_size, int patch, void *patches_bf16,
                                int k_pitch, void *scratch, size_t scratch_bytes, void *stream)
{
    if (!img || !patches_bf16 || batch <= 0 || H <= 0 || W <= 0 || patch <= 0 || out_size <= 0) return GA_ERR_BADARG;
    if (out_size % patch || k_pitch < 3 * patch * patch || k_pitch % 8) return GA_ERR_BADARG;
    if (H > kMaxSide || W > kMaxSide || out_size > kMaxSide) return GA_ERR_SIZE;
    cudaStream_t s = (cudaStream_t)stream;
    const float *src = img;
    const bool resize = !(H == out_size && W == out_size);
    if (needs_blur(H, W, out_size)) {
        const size_t plane = (size_t)batch * 3 * (size_t)H * (size_t)W;
        if (!scratch || scratch_bytes < ga_dino_frontend_scratch_bytes(batch, H, W, out_size)) return GA_ERR_WORKSPACE;
        float sy, sx;
        int ky, kx;
        blur_params(H, out_size, &sy, &ky);
        blur_params(W, out_size, &sx, &kx);
        if (ky > kMaxTaps || kx > kMaxTaps) return GA_ERR_SIZE;
        float *t0 = reinterpret_cast<float *>(scratch), *t1 = t0 + plane;
        const unsigned grid = (unsigned)((plane + 255) / 256 < 132 * 16 ? (plane + 255) / 256 : 132 * 16);
        blur_pass_kernel<<<grid, 256, 0, s>>>(img, t0, (long long)batch * 3, H, W, 0, kx, sx);       // along x first
        blur_pass_kernel<<<grid, 256, 0, s>>>(t0, t1, (long long)batch * 3, H, W, 1, ky, sy);
        src = t1;
    }
    const float scale_y = out_size > 1 ? (float)(H - 1) / (float)(out_size - 1) : 0.f;
    const float scale_x = out_size > 1 ? (float)(W - 1) / (float)(out_size - 1) : 0.f;
    const Norm nrm = {{0.485f, 0.456f, 0.406f}, {0.229f, 0.224f, 0.225f}};
    const int np = out_size / patch;
    const long long total = (long long)batch * np * np * k_pitch;
    patch_matrix_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(
        src, H, W, patch, np, k_pitch, resize ? 1 : 0, scale_y, scale_x, nrm,
        reinterpret_cast<__nv_bfloat16 *>(patches_bf16), total);
    return last_err();
}

extern "C" int ga_dino_tokens(const float *patch_out, const float *cls_token, const float *reg_tokens, int n_reg,
                              const float *pos_embed, float *x, int batch, int n_patch, int D, void *stream)
{
    if (!patch_out || !cls_token || !pos_embed || !x || batch <= 0 || n_patch <= 0 || n_reg < 0 || D <= 0 || D % 4)
        return GA_ERR_BADARG;
    if (n_reg > 0 && !reg_tokens) return GA_ERR_BADARG;
    using ga_row::mis16;
    if (mis16(patch_out) || mis16(cls_token) || mis16(reg_tokens) || mis16(pos_embed) || mis16(x)) return GA_ERR_BADARG;
    const int D4 = D / 4;
    const long long total = (long long)batch * (1 + n_reg + n_patch) * D4;
    tokens_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const float4 *>(patch_out), reinterpret_cast<const float4 *>(cls_token),
        reinterpret_cast<const float4 *>(reg_tokens), n_reg, reinterpret_cast<const float4 *>(pos_embed),
        reinterpret_cast<float4 *>(x), n_patch, D4, total);
    return last_err();
}
