// TSDF fusion of V rendered RGB-D views (include/ga_b200.h Part 4): image preparation, touched-unit marking and
// per-unit integration.  Restates Open3D's ScalableTSDFVolume::Integrate and
// UniformTSDFVolume::IntegrateWithDepthToCameraDistanceMultiplier as FlowMatchingEngine.extract_mesh_bounded uses
// them (nsr/lsgm/flow_matching_trainer.py:1364-1394).  Built with --fmad=false (build.py): every product and sum is
// rounded on its own, in the order written, so weights, tsdf and colours match oracle/tsdf_oracle.py bit for bit.
#include "mesh_common.cuh"

namespace {

using namespace ga_mesh;

__global__ void __launch_bounds__(256)
prepare_kernel(const float *__restrict__ rgb, const float *__restrict__ depth, const float *__restrict__ alpha,
               int HW, const double *__restrict__ depth_trunc, float alpha_thres, uint2 *__restrict__ texels)
{
    const int v = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= HW) return;
    const size_t p = (size_t)v * HW + i;
    float d = depth[p];
    if (alpha[p] < alpha_thres) d = 0.f;
    if ((double)d >= depth_trunc[v]) d = 0.f;
    unsigned c = 0;
#pragma unroll
    for (int k = 0; k < 3; k++) {
        const float x = fminf(fmaxf(rgb[((size_t)v * 3 + k) * HW + i], 0.f), 1.f) * 255.f;
        c |= (unsigned)x << (8 * k);
    }
    texels[p] = make_uint2(__float_as_uint(d), c);
}

// one thread per sampled pixel (every 4th row and column) of view blockIdx.y
__global__ void __launch_bounds__(256)
touch_kernel(const uint2 *__restrict__ texels, int H, int W, const double *__restrict__ cams_d,
             const double *__restrict__ volume, const int32_t *__restrict__ box, int words,
             unsigned *__restrict__ unit_table, int32_t *__restrict__ status)
{
    const int v = blockIdx.y;
    const int sw = (W + 3) / 4, sh = (H + 3) / 4;
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= sw * sh) return;
    const int i = (s / sw) * 4, j = (s % sw) * 4;
    const float d = __uint_as_float(texels[((size_t)v * H + i) * W + j].x);
    if (!(d > 0.f)) return;
    const double *M = cams_d + (size_t)v * GA_MESH_CAM_FLOATS;
    const double z = (double)d;
    const double x = ((double)j - M[18]) * z / M[16];
    const double y = ((double)i - M[19]) * z / M[17];
    const double st = volume[1], ul = volume[0] * GA_MESH_UNIT;
    int lo[3], n[3];
#pragma unroll
    for (int r = 0; r < 3; r++) {
        const double p = M[4 * r] * x + M[4 * r + 1] * y + M[4 * r + 2] * z + M[4 * r + 3];
        const double a = floor((p - st) / ul), b = floor((p + st) / ul);
        if (!(a >= (double)box[r] && b < (double)box[r] + box[3 + r])) {    // also false for NaN
            atomicOr(&status[1], 1);
            return;
        }
        lo[r] = (int)a - box[r];
        n[r] = (int)b - (int)a + 1;
    }
    const unsigned bit = 1u << (v & 31);
    for (int a = 0; a < n[0]; a++)
        for (int b = 0; b < n[1]; b++)
            for (int c = 0; c < n[2]; c++) {
                const size_t u = ((size_t)(lo[0] + a) * box[4] + lo[1] + b) * box[5] + lo[2] + c;
                unsigned *w = unit_table + u * words + (v >> 5);
                if (!(*w & bit)) atomicOr(w, bit);
            }
}

__global__ void __launch_bounds__(256)
unit_flag_kernel(const unsigned *__restrict__ unit_table, int words, int n, int *__restrict__ flag)
{
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n) return;
    unsigned any = 0;
    for (int k = 0; k < words; k++) any |= unit_table[(size_t)u * words + k];
    flag[u] = any != 0;
}

__global__ void __launch_bounds__(256)
unit_pool_kernel(const unsigned *__restrict__ unit_table, int words, int n, const int *__restrict__ off,
                 int32_t *__restrict__ pool, int32_t *__restrict__ unit_slot)
{
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n) return;
    unsigned any = 0;
    for (int k = 0; k < words; k++) any |= unit_table[(size_t)u * words + k];
    unit_slot[u] = any ? off[u] : -1;
    if (any) pool[off[u]] = u;
}

constexpr int INT_THREADS = 256;
constexpr int VOX_PER_THREAD = 4096 / INT_THREADS;

// one CTA per pooled unit; the 4096 voxels' state stays in registers across the view loop and is written once
__global__ void __launch_bounds__(INT_THREADS)
integrate_kernel(const uint2 *__restrict__ texels, int views, int H, int W, const float *__restrict__ cams_f,
                 const double *__restrict__ volume, const int32_t *__restrict__ box,
                 const unsigned *__restrict__ unit_table, int words, const int32_t *__restrict__ pool, int n_units,
                 float *__restrict__ voxels)
{
    extern __shared__ float cam[];
    for (int k = threadIdx.x; k < views * GA_MESH_CAM_FLOATS; k += blockDim.x) cam[k] = cams_f[k];
    __syncthreads();
    const int slot = blockIdx.x;
    const int u = pool[slot];
    const int ny = box[4], nz = box[5];
    const int gu[3] = {box[0] + u / (ny * nz), box[1] + (u / nz) % ny, box[2] + u % nz};
    const double vl = volume[0];
    const float vl_f = (float)vl, half_f = vl_f * 0.5f, st_f = (float)volume[1];
    const float inv_st = 1.0f / st_f;
    float org[3];
#pragma unroll
    for (int a = 0; a < 3; a++) org[a] = (float)((double)gu[a] * (vl * GA_MESH_UNIT));
    // voxel k of this thread: index threadIdx.x + 256 k = (x * 16 + y) * 16 + z  ->  x = k, y = tid >> 4, z = tid & 15
    const float Y = half_f + vl_f * (float)(threadIdx.x >> 4) + org[1];
    const float Z = half_f + vl_f * (float)(threadIdx.x & 15) + org[2];
    float T[VOX_PER_THREAD], Wt[VOX_PER_THREAD], R[VOX_PER_THREAD], G[VOX_PER_THREAD], B[VOX_PER_THREAD];
#pragma unroll
    for (int k = 0; k < VOX_PER_THREAD; k++) T[k] = Wt[k] = R[k] = G[k] = B[k] = 0.f;
    const float Wf = (float)W - 0.0001f, Hf = (float)H - 0.0001f;
    for (int v = 0; v < views; v++) {
        if (!((unit_table[(size_t)u * words + (v >> 5)] >> (v & 31)) & 1u)) continue;
        const float *E = cam + v * GA_MESH_CAM_FLOATS;
        const float fx = E[16], fy = E[17], cx = E[18], cy = E[19];
        const float ifx = 1.0f / fx, ify = 1.0f / fy;
        const uint2 *tex = texels + (size_t)v * H * W;
#pragma unroll
        for (int k = 0; k < VOX_PER_THREAD; k++) {
            const float X = half_f + vl_f * (float)k + org[0];
            const float pz = E[8] * X + E[9] * Y + E[10] * Z + E[11];
            if (!(pz > 0.f)) continue;
            const float px = E[0] * X + E[1] * Y + E[2] * Z + E[3];
            const float py = E[4] * X + E[5] * Y + E[6] * Z + E[7];
            const float uf = px * fx / pz + cx + 0.5f;
            const float vf = py * fy / pz + cy + 0.5f;
            if (!(uf >= 0.0001f && uf < Wf && vf >= 0.0001f && vf < Hf)) continue;
            const int iu = (int)uf, iv = (int)vf;
            const uint2 t = tex[(size_t)iv * W + iu];
            const float d = __uint_as_float(t.x);
            if (!(d > 0.f)) continue;
            const float xx = ((float)iu - cx) * ifx, yy = ((float)iv - cy) * ify;
            const float sdf = (d - pz) * sqrtf(xx * xx + yy * yy + 1.0f);
            if (!(sdf > -st_f)) continue;
            const float tsdf = fminf(1.0f, sdf * inv_st);
            const float w = Wt[k], w1 = w + 1.0f;
            T[k] = (T[k] * w + tsdf) / w1;
            R[k] = (R[k] * w + (float)(t.y & 255u)) / w1;
            G[k] = (G[k] * w + (float)((t.y >> 8) & 255u)) / w1;
            B[k] = (B[k] * w + (float)((t.y >> 16) & 255u)) / w1;
            Wt[k] = w1;
        }
    }
    const size_t nv = (size_t)n_units * 4096;
#pragma unroll
    for (int k = 0; k < VOX_PER_THREAD; k++) {
        const size_t i = (size_t)slot * 4096 + threadIdx.x + INT_THREADS * k;
        voxels[i] = T[k];
        voxels[nv + i] = Wt[k];
        voxels[2 * nv + i] = R[k];
        voxels[3 * nv + i] = G[k];
        voxels[4 * nv + i] = B[k];
    }
}

}  // namespace

extern "C" size_t ga_mesh_work_bytes(int64_t n)
{
    if (n < 0) return 0;
    return (size_t)(3 * n + scan_partials(n) + 2) * sizeof(int32_t);
}

extern "C" int ga_mesh_prepare(const float *rgb, const float *depth, const float *alpha, int views, int H, int W,
                               const double *depth_trunc, float alpha_thres, void *texels, void *stream)
{
    if (!rgb || !depth || !alpha || !depth_trunc || !texels || views <= 0 || H <= 0 || W <= 0) return GA_ERR_BADARG;
    if ((int64_t)H * W > (1 << 26) || views > 65535) return GA_ERR_SIZE;
    const int HW = H * W;
    prepare_kernel<<<dim3((HW + 255) / 256, views), 256, 0, (cudaStream_t)stream>>>(
        rgb, depth, alpha, HW, depth_trunc, alpha_thres, (uint2 *)texels);
    return (int)cudaGetLastError();
}

extern "C" int ga_mesh_touch(const void *texels, int views, int H, int W, const double *cams_d, const double *volume,
                             const int32_t *box, int box_units, int32_t *unit_table, int32_t *pool, int32_t *unit_slot,
                             void *work, int32_t *status, int32_t *status_host, void *status_event, void *stream)
{
    if (!texels || !cams_d || !volume || !box || !unit_table || !pool || !unit_slot || !work || !status
        || views <= 0 || H <= 0 || W <= 0 || box_units <= 0) return GA_ERR_BADARG;
    if ((status_host == nullptr) != (status_event == nullptr)) return GA_ERR_BADARG;
    if ((int64_t)H * W > (1 << 26) || views > 65535) return GA_ERR_SIZE;
    cudaStream_t s = (cudaStream_t)stream;
    const int words = (views + 31) / 32;
    cudaError_t e;
    if ((e = cudaMemsetAsync(unit_table, 0, (size_t)box_units * words * sizeof(int32_t), s)) != cudaSuccess) return (int)e;
    if ((e = cudaMemsetAsync(status, 0, 2 * sizeof(int32_t), s)) != cudaSuccess) return (int)e;
    const int samples = ((W + 3) / 4) * ((H + 3) / 4);
    touch_kernel<<<dim3((samples + 255) / 256, views), 256, 0, s>>>((const uint2 *)texels, H, W, cams_d, volume, box,
                                                                    words, (unsigned *)unit_table, status);
    int *flag = (int *)work, *partials = flag + box_units;
    const unsigned nb = (box_units + 255) / 256;
    unit_flag_kernel<<<nb, 256, 0, s>>>((const unsigned *)unit_table, words, box_units, flag);
    if ((e = scan_exclusive(flag, box_units, partials, &status[0], s)) != cudaSuccess) return (int)e;
    unit_pool_kernel<<<nb, 256, 0, s>>>((const unsigned *)unit_table, words, box_units, flag, pool, unit_slot);
    if ((e = cudaGetLastError()) != cudaSuccess) return (int)e;
    return (int)publish_status(status, status_host, status_event, s);
}

extern "C" int ga_mesh_integrate(const void *texels, int views, int H, int W, const float *cams_f,
                                 const double *volume, const int32_t *box, const int32_t *unit_table,
                                 const int32_t *pool, int n_units, float *voxels, void *stream)
{
    if (!texels || !cams_f || !volume || !box || !unit_table || !pool || n_units < 0 || views <= 0 || H <= 0 || W <= 0)
        return GA_ERR_BADARG;
    if (views > 256 || (int64_t)H * W > (1 << 26)) return GA_ERR_SIZE;
    if (n_units == 0) return 0;
    if (!voxels) return GA_ERR_BADARG;
    integrate_kernel<<<n_units, INT_THREADS, views * GA_MESH_CAM_FLOATS * sizeof(float), (cudaStream_t)stream>>>(
        (const uint2 *)texels, views, H, W, cams_f, volume, box, (const unsigned *)unit_table, (views + 31) / 32, pool,
        n_units, voxels);
    return (int)cudaGetLastError();
}
