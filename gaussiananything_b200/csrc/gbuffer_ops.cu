// 3D VAE reconstruction from G-buffer chunk folders: the step before the encoder and the step after the renderer.
//   gbuffer_pack  : the chunk's decoded files (tiled uint8 RGB / normal / alpha, fp32 depth, 25-float cameras) ->
//                   img_to_encoder [V, 15, H, W] and, optionally, the render targets of the same views, in one launch
//   recon_metrics : rendered maps against those targets -> a [V, 8] table of per-view sums, two fixed-order stages
// Math follows the reference's PostProcess._post_process_sample_batch (datasets/g_buffer_objaverse.py:481-702) at the
// deployed configuration; the rounding of every step is stated in include/ga_b200.h and restated by
// oracle/gbuffer_oracle.py.  This file is compiled without FMA contraction so that the stated roundings hold.
#include "../../include/ga_b200.h"
#include "gbuffer_common.cuh"
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

namespace {

// torchvision Normalize with the ImageNet statistics (PostProcess.__init__ with imgnet_normalize=True, which is what
// load_eval_data's chunk branch passes)
__constant__ float RGB_MEAN[3] = {0.485f, 0.456f, 0.406f};
__constant__ float RGB_STD[3] = {0.229f, 0.224f, 0.225f};

struct PackArgs {
    const uint8_t *raw, *normal, *alpha;
    const float *depth, *cams;
    const int32_t *views;
    int n_chunk, H, W;
    float *enc, *t_img, *t_alpha, *t_depth, *t_mask;
};

__device__ __forceinline__ void store4(float *p, float a, float b, float c, float d)
{
    *reinterpret_cast<float4 *>(p) = make_float4(a, b, c, d);
}

// 3 bytes x 4 pixels = three aligned 32-bit words -> ch[channel][pixel]
__device__ __forceinline__ void load_rgb4(const uint8_t *p, float ch[3][4])
{
    const uint32_t *q = reinterpret_cast<const uint32_t *>(p);
    const uint32_t w[3] = {__ldg(q), __ldg(q + 1), __ldg(q + 2)};
#pragma unroll
    for (int i = 0; i < 12; i++) ch[i % 3][i / 3] = (float)((w[i >> 2] >> (8 * (i & 3))) & 0xffu);
}

// grid (H, V), W / 4 threads: one thread per four pixels of a row of one selected view, so every store is 16 bytes.
__global__ void __launch_bounds__(256)
gbuffer_pack_kernel(PackArgs a)
{
    __shared__ float cam[25];
    const int slot = blockIdx.y, y = blockIdx.x, x0 = threadIdx.x * 4;
    const int view = a.views[slot];
    for (int i = threadIdx.x; i < 25; i += blockDim.x) cam[i] = a.cams[view * 25 + i];
    __syncthreads();
    const int H = a.H, W = a.W;
    const size_t HW = (size_t)H * W, pix = (size_t)y * W + x0;
    const size_t tiled = ((size_t)y * a.n_chunk + view) * W + x0;            // pixel index in the side-by-side files
    float *enc = a.enc + (size_t)slot * 15 * HW + pix;

    float rgb[3][4], nrm[3][4];
    load_rgb4(a.raw + tiled * 3, rgb);
    load_rgb4(a.normal + tiled * 3, nrm);
    const float4 dep = __ldg(reinterpret_cast<const float4 *>(a.depth + (size_t)view * HW + pix));
    const float d4[4] = {dep.x, dep.y, dep.z, dep.w};

#pragma unroll
    for (int c = 0; c < 3; c++) {
        float v[4], n[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            rgb[c][i] = rgb[c][i] / 255.0f;
            v[i] = (rgb[c][i] - RGB_MEAN[c]) / RGB_STD[c];
            n[i] = (nrm[c][i] / 255.0f) * 2.0f - 1.0f;
        }
        store4(enc + c * HW, v[0], v[1], v[2], v[3]);
        // unity2blender_fix: (x, y, z) -> (-x, -z, y)
        if (c == 0) store4(enc + 3 * HW, -n[0], -n[1], -n[2], -n[3]);
        if (c == 1) store4(enc + 5 * HW, n[0], n[1], n[2], n[3]);
        if (c == 2) store4(enc + 4 * HW, -n[0], -n[1], -n[2], -n[3]);
    }

    const float ox = cam[3], oy = cam[7], oz = cam[11];
    const float fx = cam[16], cx = cam[18], fy = cam[20], cy = cam[21];
    const float v_cam = ((float)y + 0.5f) / (float)H;
    float pl[6][4], xyz[3][4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const float u_cam = ((float)(x0 + i) + 0.5f) / (float)W;
        // gen_rays: normalise the camera-space direction, then rotate
        float gx = (u_cam - cx) / fx, gy = (v_cam - cy) / fy;
        const float gn = sqrtf(gx * gx + gy * gy + 1.0f);
        gx = gx / gn;
        gy = gy / gn;
        const float gz = 1.0f / gn;
        const float dx = cam[0] * gx + cam[1] * gy + cam[2] * gz;
        const float dy = cam[4] * gx + cam[5] * gy + cam[6] * gz;
        const float dz = cam[8] * gx + cam[9] * gy + cam[10] * gz;
        pl[0][i] = oy * dz - oz * dy;
        pl[1][i] = oz * dx - ox * dz;
        pl[2][i] = ox * dy - oy * dx;
        pl[3][i] = dx;
        pl[4][i] = dy;
        pl[5][i] = dz;
        float p[3];
        gbuf::unproject(cam, u_cam, v_cam, d4[i], p);
#pragma unroll
        for (int c = 0; c < 3; c++) xyz[c][i] = p[c];
    }
#pragma unroll
    for (int c = 0; c < 6; c++) store4(enc + (6 + c) * HW, pl[c][0], pl[c][1], pl[c][2], pl[c][3]);
#pragma unroll
    for (int c = 0; c < 3; c++) store4(enc + (12 + c) * HW, xyz[c][0], xyz[c][1], xyz[c][2], xyz[c][3]);

    if (a.t_img) {
#pragma unroll
        for (int c = 0; c < 3; c++)
            store4(a.t_img + ((size_t)slot * 3 + c) * HW + pix, rgb[c][0] * 2.0f - 1.0f, rgb[c][1] * 2.0f - 1.0f,
                   rgb[c][2] * 2.0f - 1.0f, rgb[c][3] * 2.0f - 1.0f);
        const uint32_t aw = __ldg(reinterpret_cast<const uint32_t *>(a.alpha + tiled));
        store4(a.t_alpha + (size_t)slot * HW + pix, (float)(aw & 0xffu) / 255.0f, (float)((aw >> 8) & 0xffu) / 255.0f,
               (float)((aw >> 16) & 0xffu) / 255.0f, (float)(aw >> 24) / 255.0f);
        store4(a.t_depth + (size_t)slot * HW + pix, d4[0], d4[1], d4[2], d4[3]);
        store4(a.t_mask + (size_t)slot * HW + pix, d4[0] > 0.0f ? 1.0f : 0.0f, d4[1] > 0.0f ? 1.0f : 0.0f,
               d4[2] > 0.0f ? 1.0f : 0.0f, d4[3] > 0.0f ? 1.0f : 0.0f);
    }
}

constexpr int MB = GA_RECON_METRICS_BLOCKS, MT = 256, NM = 8;

struct MetricArgs {
    const float *image, *depth, *alpha, *normal;             // rendered
    const float *t_img, *t_depth, *t_alpha, *t_mask, *t_normal;
    int64_t t_normal_stride;
    int HW;
    float *partial, *out;
};

// grid (MB, V): block b of view v takes pixels [b * per, (b + 1) * per); thread t takes every MT-th of them.  The
// block's eight sums are folded lane by lane with shuffles, then warp by warp in warp order: a fixed tree.
__global__ void __launch_bounds__(MT)
recon_metrics_partial_kernel(MetricArgs a)
{
    __shared__ float s[MT / 32][NM];
    const int v = blockIdx.y, HW = a.HW;
    const int per = (HW + MB - 1) / MB, lo = blockIdx.x * per, hi = min(HW, lo + per);
    const float *img = a.image + (size_t)v * 3 * HW, *nr = a.normal + (size_t)v * 3 * HW;
    const float *ti = a.t_img + (size_t)v * 3 * HW, *tn = a.t_normal + (size_t)v * a.t_normal_stride;
    const size_t o1 = (size_t)v * HW;
    float m[NM] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int p = lo + threadIdx.x; p < hi; p += MT) {
        float se = 0.0f, dot = 0.0f;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const float e = img[c * HW + p] - (ti[c * HW + p] + 1.0f) * 0.5f;
            se += e * e;
            dot += nr[c * HW + p] * tn[c * HW + p];
        }
        const float mk = a.t_mask[o1 + p], pa = a.alpha[o1 + p], ta = a.t_alpha[o1 + p];
        const bool pi = pa > 0.5f, gi = ta > 0.5f;
        m[0] += se;
        m[1] += mk * fabsf(a.depth[o1 + p] - a.t_depth[o1 + p]);
        m[2] += mk;
        m[3] += mk * (1.0f - dot);
        m[4] += fabsf(pa - ta);
        m[5] += (pi && gi) ? 1.0f : 0.0f;
        m[6] += (pi || gi) ? 1.0f : 0.0f;
        m[7] += 1.0f;
    }
#pragma unroll
    for (int k = 0; k < NM; k++)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m[k] += __shfl_down_sync(0xffffffffu, m[k], o);
    if ((threadIdx.x & 31) == 0)
#pragma unroll
        for (int k = 0; k < NM; k++) s[threadIdx.x >> 5][k] = m[k];
    __syncthreads();
    if (threadIdx.x < NM) {
        float t = 0.0f;
        for (int w = 0; w < MT / 32; w++) t += s[w][threadIdx.x];
        a.partial[((size_t)v * MB + blockIdx.x) * NM + threadIdx.x] = t;
    }
}

// one block per view: column k of the view's MB partial rows, added in block order
__global__ void __launch_bounds__(32)
recon_metrics_final_kernel(const float *__restrict__ partial, float *__restrict__ out)
{
    if (threadIdx.x >= NM) return;
    const float *p = partial + (size_t)blockIdx.x * MB * NM + threadIdx.x;
    float t = 0.0f;
    for (int b = 0; b < MB; b++) t += p[b * NM];
    out[blockIdx.x * NM + threadIdx.x] = t;
}

}  // namespace

extern "C" int ga_gbuffer_pack(const uint8_t *raw_img, const uint8_t *normal, const uint8_t *alpha, const float *depth,
                               const float *cams, int n_chunk, int H, int W, const int32_t *views, int n_views,
                               float *img_to_encoder, float *t_img, float *t_alpha, float *t_depth, float *t_mask,
                               void *stream)
{
    if (!raw_img || !normal || !depth || !cams || !views || !img_to_encoder || n_chunk <= 0 || n_views <= 0 || H <= 0 ||
        W <= 0 || W % 4 != 0 || W > 1024 || n_views > 65535)
        return GA_ERR_BADARG;
    const int targets = (t_img != nullptr) + (t_alpha != nullptr) + (t_depth != nullptr) + (t_mask != nullptr);
    if ((targets != 0 && targets != 4) || (targets == 4 && !alpha)) return GA_ERR_BADARG;
    PackArgs a{raw_img, normal, alpha, depth, cams, views, n_chunk, H, W, img_to_encoder, t_img, t_alpha, t_depth, t_mask};
    gbuffer_pack_kernel<<<dim3(H, n_views), W / 4, 0, (cudaStream_t)stream>>>(a);
    return (int)cudaGetLastError();
}

extern "C" int ga_recon_metrics(const float *image, const float *depth, const float *alpha, const float *rend_normal,
                                const float *t_img, const float *t_depth, const float *t_alpha, const float *t_mask,
                                const float *t_normal, int64_t t_normal_stride, int n_views, int H, int W,
                                float *partial, float *table, void *stream)
{
    if (!image || !depth || !alpha || !rend_normal || !t_img || !t_depth || !t_alpha || !t_mask || !t_normal ||
        !partial || !table || n_views <= 0 || n_views > 65535 || H <= 0 || W <= 0 || (int64_t)H * W > (1 << 24) ||
        t_normal_stride < (int64_t)3 * H * W)
        return GA_ERR_BADARG;
    MetricArgs a{image, depth, alpha, rend_normal, t_img, t_depth, t_alpha, t_mask, t_normal, t_normal_stride, H * W,
                 partial, table};
    recon_metrics_partial_kernel<<<dim3(MB, n_views), MT, 0, (cudaStream_t)stream>>>(a);
    recon_metrics_final_kernel<<<n_views, 32, 0, (cudaStream_t)stream>>>(partial, table);
    return (int)cudaGetLastError();
}
