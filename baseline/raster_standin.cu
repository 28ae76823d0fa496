// GPU comparison baseline ("stand-in") for the surfel rasteriser -- NOT the product path, nothing under
// gaussiananything_b200/ includes or links this file.
//
// The reference's GPU build drives github.com/hbb1/diff-surfel-rasterization, which is neither vendored nor
// installable here (BASELINE.md section 4).  This file restates THAT package's flow as literally as its published
// structure allows, so bench.py can time "what the reference GPU build does" on the same GPU:
//   per VIEW (the reference loops views in Python, /root/reference/nsr/gs_surfel.py:65-114):
//     preprocessCUDA (one thread per surfel) -> cub::DeviceScan::InclusiveSum of tiles_touched -> cudaMemcpy of
//     num_rendered to the host (a device sync per view) -> duplicateWithKeys ((tile << 32) | depth keys) ->
//     cub::DeviceRadixSort::SortPairs over the whole instance list -> identifyTileRanges -> renderCUDA
//     (one 16x16 tile per block, 256 records staged per round, EVERY pixel evaluates EVERY staged surfel);
//   backward: renderCUDA back to front with one atomicAdd per (pixel, surfel, gradient component), then the
//     per-surfel preprocess backward.
// Same constants and arithmetic as oracle/surfel_oracle.c (SURVEY.md App. A); tests/test_standin_gpu.py checks it
// against the oracle so that the timing compares like with like.
#include <cub/cub.cuh>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define BX 16
#define BY 16
#define NEAR_N 0.2f
#define FAR_N 100.0f
#define FILTER_SIZE 0.707106f
#define FILTER_INV_SQUARE 2.0f

struct StCtx {
    int P = 0, H = 0, W = 0, gx = 0, gy = 0;
    // geometry state (P)
    float *transmat = nullptr, *normal_opacity = nullptr, *xy = nullptr, *depth = nullptr;
    int *radii = nullptr;
    uint32_t *tiles_touched = nullptr, *offsets = nullptr;
    int *rect = nullptr;
    // binning state (num_rendered)
    size_t cap = 0;
    uint64_t *keys = nullptr, *keys_sorted = nullptr;
    uint32_t *vals = nullptr, *vals_sorted = nullptr;
    int2 *ranges = nullptr;
    void *scan_tmp = nullptr, *sort_tmp = nullptr;
    size_t scan_bytes = 0, sort_bytes = 0;
    // image state
    float *final_T = nullptr;
    int *n_contrib = nullptr;
    // backward accumulators
    float *dL_dtransmat = nullptr, *dL_dmean2D = nullptr, *dL_dnormal = nullptr, *dL_dopacity = nullptr, *dL_dcolor = nullptr;
    int num_rendered = 0;
};

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return (int)e_; } while (0)

__device__ __forceinline__ void quat_to_rotmat(const float *q, float R[3][3])
{
    const float s = rsqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    const float w = q[0] * s, x = q[1] * s, y = q[2] * s, z = q[3] * s;
    R[0][0] = 1.f - 2.f * (y * y + z * z); R[1][0] = 2.f * (x * y + w * z); R[2][0] = 2.f * (x * z - w * y);
    R[0][1] = 2.f * (x * y - w * z); R[1][1] = 1.f - 2.f * (x * x + z * z); R[2][1] = 2.f * (y * z + w * x);
    R[0][2] = 2.f * (x * z + w * y); R[1][2] = 2.f * (y * z - w * x); R[2][2] = 1.f - 2.f * (x * x + y * y);
}

__global__ void st_preprocess(int P, const float *__restrict__ g13, const float *__restrict__ vm, const float *__restrict__ pm,
                              int H, int W, int gx, int gy, float mod, float *transmat, float *normal_opacity, float *xy,
                              float *depth, int *radii, uint32_t *tiles_touched, int *rect)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    radii[i] = 0; tiles_touched[i] = 0;
    const float *g = g13 + (size_t)i * 13;
    const float px = g[0], py = g[1], pz = g[2];
    const float vx = vm[0] * px + vm[4] * py + vm[8] * pz + vm[12];
    const float vy = vm[1] * px + vm[5] * py + vm[9] * pz + vm[13];
    const float vz = vm[2] * px + vm[6] * py + vm[10] * pz + vm[14];
    if (vz <= NEAR_N) return;
    float R[3][3];
    quat_to_rotmat(g + 6, R);
    const float sx = mod * g[4], sy = mod * g[5];
    const float L0[3] = {R[0][0] * sx, R[1][0] * sx, R[2][0] * sx}, L1[3] = {R[0][1] * sy, R[1][1] * sy, R[2][1] * sy};
    const float L2[3] = {R[0][2], R[1][2], R[2][2]};
    const float hw = 0.5f * W, hh = 0.5f * H, cw = 0.5f * (W - 1), ch = 0.5f * (H - 1);
    float B0[3], B1[3], B3[3];
    B0[0] = L0[0] * pm[0] + L0[1] * pm[4] + L0[2] * pm[8]; B0[1] = L1[0] * pm[0] + L1[1] * pm[4] + L1[2] * pm[8];
    B0[2] = px * pm[0] + py * pm[4] + pz * pm[8] + pm[12];
    B1[0] = L0[0] * pm[1] + L0[1] * pm[5] + L0[2] * pm[9]; B1[1] = L1[0] * pm[1] + L1[1] * pm[5] + L1[2] * pm[9];
    B1[2] = px * pm[1] + py * pm[5] + pz * pm[9] + pm[13];
    B3[0] = L0[0] * pm[3] + L0[1] * pm[7] + L0[2] * pm[11]; B3[1] = L1[0] * pm[3] + L1[1] * pm[7] + L1[2] * pm[11];
    B3[2] = px * pm[3] + py * pm[7] + pz * pm[11] + pm[15];
    float Tu[3], Tv[3], Tw[3];
    for (int r = 0; r < 3; r++) { Tu[r] = B0[r] * hw + B3[r] * cw; Tv[r] = B1[r] * hh + B3[r] * ch; Tw[r] = B3[r]; }
    float *tm = transmat + (size_t)i * 9;
    for (int r = 0; r < 3; r++) { tm[r] = Tu[r]; tm[3 + r] = Tv[r]; tm[6 + r] = Tw[r]; }
    float nx = vm[0] * L2[0] + vm[4] * L2[1] + vm[8] * L2[2];
    float ny = vm[1] * L2[0] + vm[5] * L2[1] + vm[9] * L2[2];
    float nz = vm[2] * L2[0] + vm[6] * L2[1] + vm[10] * L2[2];
    const float cosv = -(vx * nx + vy * ny + vz * nz);
    if (cosv == 0.f) return;
    const float mult = cosv > 0.f ? 1.f : -1.f;
    nx *= mult; ny *= mult; nz *= mult;
    const float t0 = 9.f, t1 = 9.f, t2 = -1.f;
    const float d = t0 * Tw[0] * Tw[0] + t1 * Tw[1] * Tw[1] + t2 * Tw[2] * Tw[2];
    if (d == 0.f) return;
    const float f0 = t0 / d, f1 = t1 / d, f2 = t2 / d;
    const float cx = f0 * Tu[0] * Tw[0] + f1 * Tu[1] * Tw[1] + f2 * Tu[2] * Tw[2];
    const float cy = f0 * Tv[0] * Tw[0] + f1 * Tv[1] * Tw[1] + f2 * Tv[2] * Tw[2];
    const float hx0 = cx * cx - (f0 * Tu[0] * Tu[0] + f1 * Tu[1] * Tu[1] + f2 * Tu[2] * Tu[2]);
    const float hy0 = cy * cy - (f0 * Tv[0] * Tv[0] + f1 * Tv[1] * Tv[1] + f2 * Tv[2] * Tv[2]);
    const float ex = sqrtf(fmaxf(1e-4f, hx0)), ey = sqrtf(fmaxf(1e-4f, hy0));
    const int mr = (int)ceilf(fmaxf(fmaxf(ex, ey), 3.f * FILTER_SIZE));
    const int x0 = min(gx, max(0, (int)((cx - mr) / BX))), y0 = min(gy, max(0, (int)((cy - mr) / BY)));
    const int x1 = min(gx, max(0, (int)((cx + mr + BX - 1) / BX))), y1 = min(gy, max(0, (int)((cy + mr + BY - 1) / BY)));
    if ((x1 - x0) * (y1 - y0) == 0) return;
    depth[i] = vz; radii[i] = mr; xy[2 * i] = cx; xy[2 * i + 1] = cy;
    normal_opacity[4 * i] = nx; normal_opacity[4 * i + 1] = ny; normal_opacity[4 * i + 2] = nz; normal_opacity[4 * i + 3] = g[3];
    tiles_touched[i] = (uint32_t)((y1 - y0) * (x1 - x0));
    rect[4 * i] = x0; rect[4 * i + 1] = y0; rect[4 * i + 2] = x1; rect[4 * i + 3] = y1;
}

__global__ void st_duplicate(int P, const float *depth, const uint32_t *offsets, const int *radii, const int *rect, int gx,
                             uint64_t *keys, uint32_t *vals)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P || radii[i] <= 0) return;
    uint32_t off = i == 0 ? 0 : offsets[i - 1];
    for (int y = rect[4 * i + 1]; y < rect[4 * i + 3]; y++)
        for (int x = rect[4 * i]; x < rect[4 * i + 2]; x++) {
            keys[off] = ((uint64_t)(y * gx + x) << 32) | (uint64_t)__float_as_uint(depth[i]);
            vals[off] = (uint32_t)i;
            off++;
        }
}

__global__ void st_ranges(int L, const uint64_t *keys, int2 *ranges)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L) return;
    const uint32_t t = (uint32_t)(keys[i] >> 32);
    if (i == 0) ranges[t].x = 0;
    else {
        const uint32_t p = (uint32_t)(keys[i - 1] >> 32);
        if (t != p) { ranges[p].y = i; ranges[t].x = i; }
    }
    if (i == L - 1) ranges[t].y = L;
}

__global__ void __launch_bounds__(BX *BY)
st_render_fwd(const int2 *__restrict__ ranges, const uint32_t *__restrict__ ids, int W, int H, const float *__restrict__ xy,
              const float *__restrict__ transmat, const float *__restrict__ normal_opacity, const float *__restrict__ g13,
              const float *__restrict__ bg, float *final_T, int *n_contrib, float *out_color, float *out_allmap)
{
    __shared__ int s_id[256];
    __shared__ float2 s_xy[256];
    __shared__ float4 s_no[256];
    __shared__ float s_T[256][9];
    const int gx = (W + BX - 1) / BX;
    const int pxi = blockIdx.x * BX + threadIdx.x, pyi = blockIdx.y * BY + threadIdx.y;
    const int tid = threadIdx.y * BX + threadIdx.x;
    const bool inside = pxi < W && pyi < H;
    const float pfx = (float)pxi, pfy = (float)pyi;
    const int2 range = ranges[blockIdx.y * gx + blockIdx.x];
    const int rounds = (range.y - range.x + 255) / 256;
    int todo = range.y - range.x;
    bool done = !inside;
    float T = 1.f, C[3] = {0, 0, 0}, N[3] = {0, 0, 0}, Dacc = 0, M1 = 0, M2 = 0, dist = 0, median_depth = 0;
    int contributor = 0, last_contributor = 0, median_contributor = -1;
    for (int i = 0; i < rounds; i++, todo -= 256) {
        if (__syncthreads_count(done) == 256) break;
        const int progress = i * 256 + tid;
        if (range.x + progress < range.y) {
            const int id = (int)ids[range.x + progress];
            s_id[tid] = id;
            s_xy[tid] = make_float2(xy[2 * id], xy[2 * id + 1]);
            s_no[tid] = *reinterpret_cast<const float4 *>(normal_opacity + 4 * (size_t)id);
            for (int r = 0; r < 9; r++) s_T[tid][r] = transmat[9 * (size_t)id + r];
        }
        __syncthreads();
        for (int j = 0; !done && j < min(256, todo); j++) {
            contributor++;
            const float *Tu = s_T[j], *Tv = Tu + 3, *Tw = Tu + 6;
            const float k0 = pfx * Tw[0] - Tu[0], k1 = pfx * Tw[1] - Tu[1], k2 = pfx * Tw[2] - Tu[2];
            const float l0 = pfy * Tw[0] - Tv[0], l1 = pfy * Tw[1] - Tv[1], l2 = pfy * Tw[2] - Tv[2];
            const float p0 = k1 * l2 - k2 * l1, p1 = k2 * l0 - k0 * l2, p2 = k0 * l1 - k1 * l0;
            if (p2 == 0.f) continue;
            const float s0 = p0 / p2, s1 = p1 / p2;
            const float rho3d = s0 * s0 + s1 * s1;
            const float dx = s_xy[j].x - pfx, dy = s_xy[j].y - pfy;
            const float rho2d = FILTER_INV_SQUARE * (dx * dx + dy * dy);
            const float rho = fminf(rho3d, rho2d);
            const float depth = (rho3d <= rho2d) ? (s0 * Tw[0] + s1 * Tw[1]) + Tw[2] : Tw[2];
            if (depth < NEAR_N) continue;
            const float4 no = s_no[j];
            const float power = -0.5f * rho;
            if (power > 0.f) continue;
            const float alpha = fminf(0.99f, no.w * __expf(power));
            if (alpha < 1.f / 255.f) continue;
            const float test_T = T * (1 - alpha);
            if (test_T < 0.0001f) { done = true; continue; }
            const float w = alpha * T, A = 1 - T;
            const float m = FAR_N / (FAR_N - NEAR_N) * (1 - NEAR_N / depth);
            dist += (m * m * A + M2 - 2 * m * M1) * w;
            Dacc += depth * w; M1 += m * w; M2 += m * m * w;
            if (T > 0.5f) { median_depth = depth; median_contributor = contributor; }
            N[0] += no.x * w; N[1] += no.y * w; N[2] += no.z * w;
            const float *col = g13 + (size_t)s_id[j] * 13 + 10;
            C[0] += col[0] * w; C[1] += col[1] * w; C[2] += col[2] * w;
            T = test_T;
            last_contributor = contributor;
        }
    }
    if (inside) {
        const size_t HW = (size_t)H * W, pix = (size_t)pyi * W + pxi;
        final_T[pix] = T; final_T[pix + HW] = M1; final_T[pix + 2 * HW] = M2;
        n_contrib[pix] = last_contributor; n_contrib[pix + HW] = median_contributor;
        for (int c = 0; c < 3; c++) out_color[c * HW + pix] = C[c] + T * bg[c];
        out_allmap[pix] = Dacc; out_allmap[HW + pix] = 1 - T;
        for (int c = 0; c < 3; c++) out_allmap[(2 + c) * HW + pix] = N[c];
        out_allmap[5 * HW + pix] = median_depth; out_allmap[6 * HW + pix] = dist;
    }
}

__global__ void __launch_bounds__(BX *BY)
st_render_bwd(const int2 *__restrict__ ranges, const uint32_t *__restrict__ ids, int W, int H, const float *__restrict__ xy,
              const float *__restrict__ transmat, const float *__restrict__ normal_opacity, const float *__restrict__ g13,
              const float *__restrict__ bg, const float *__restrict__ final_T, const int *__restrict__ n_contrib,
              const float *__restrict__ dL_dpix, const float *__restrict__ dL_dallmap, float *dL_dtransmat, float *dL_dmean2D,
              float *dL_dnormal, float *dL_dopacity, float *dL_dcolor)
{
    __shared__ int s_id[256];
    __shared__ float2 s_xy[256];
    __shared__ float4 s_no[256];
    __shared__ float s_T[256][9];
    __shared__ float s_col[256][3];
    const int gx = (W + BX - 1) / BX;
    const int pxi = blockIdx.x * BX + threadIdx.x, pyi = blockIdx.y * BY + threadIdx.y;
    const int tid = threadIdx.y * BX + threadIdx.x;
    const bool inside = pxi < W && pyi < H;
    const float pfx = (float)pxi, pfy = (float)pyi;
    const size_t HW = (size_t)H * W, pix = inside ? (size_t)pyi * W + pxi : 0;
    const int2 range = ranges[blockIdx.y * gx + blockIdx.x];
    const int rounds = (range.y - range.x + 255) / 256;
    int todo = range.y - range.x;
    bool done = !inside;
    const float T_final = inside ? final_T[pix] : 0;
    float T = T_final;
    int contributor = todo;
    const int last_contributor = inside ? n_contrib[pix] : 0, median_contributor = inside ? n_contrib[pix + HW] : 0;
    float accum_rec[3] = {0, 0, 0}, dL_dpixel[3] = {0, 0, 0}, dn[3] = {0, 0, 0};
    float dL_ddepth = 0, dL_daccum = 0, dL_dmedian = 0, dL_dreg = 0;
    if (inside) {
        for (int c = 0; c < 3; c++) dL_dpixel[c] = dL_dpix[c * HW + pix];
        dL_ddepth = dL_dallmap[pix]; dL_daccum = dL_dallmap[HW + pix];
        for (int c = 0; c < 3; c++) dn[c] = dL_dallmap[(2 + c) * HW + pix];
        dL_dmedian = dL_dallmap[5 * HW + pix]; dL_dreg = dL_dallmap[6 * HW + pix];
    }
    float last_depth = 0, last_normal[3] = {0, 0, 0}, accum_depth_rec = 0, accum_alpha_rec = 0, accum_normal_rec[3] = {0, 0, 0};
    const float final_D = inside ? final_T[pix + HW] : 0, final_D2 = inside ? final_T[pix + 2 * HW] : 0, final_A = 1 - T_final;
    float last_dL_dT = 0, last_alpha = 0, last_color[3] = {0, 0, 0};
    const float bg_dot = bg[0] * dL_dpixel[0] + bg[1] * dL_dpixel[1] + bg[2] * dL_dpixel[2];
    for (int i = 0; i < rounds; i++, todo -= 256) {
        __syncthreads();
        const int progress = i * 256 + tid;
        if (range.x + progress < range.y) {
            const int id = (int)ids[range.y - progress - 1];
            s_id[tid] = id;
            s_xy[tid] = make_float2(xy[2 * id], xy[2 * id + 1]);
            s_no[tid] = *reinterpret_cast<const float4 *>(normal_opacity + 4 * (size_t)id);
            for (int r = 0; r < 9; r++) s_T[tid][r] = transmat[9 * (size_t)id + r];
            for (int c = 0; c < 3; c++) s_col[tid][c] = g13[(size_t)id * 13 + 10 + c];
        }
        __syncthreads();
        for (int j = 0; !done && j < min(256, todo); j++) {
            contributor--;
            if (contributor >= last_contributor) continue;
            const float *Tu = s_T[j], *Tv = Tu + 3, *Tw = Tu + 6;
            const float k0 = pfx * Tw[0] - Tu[0], k1 = pfx * Tw[1] - Tu[1], k2 = pfx * Tw[2] - Tu[2];
            const float l0 = pfy * Tw[0] - Tv[0], l1 = pfy * Tw[1] - Tv[1], l2 = pfy * Tw[2] - Tv[2];
            const float p0 = k1 * l2 - k2 * l1, p1 = k2 * l0 - k0 * l2, p2 = k0 * l1 - k1 * l0;
            if (p2 == 0.f) continue;
            const float s0 = p0 / p2, s1 = p1 / p2;
            const float rho3d = s0 * s0 + s1 * s1;
            const float dx = s_xy[j].x - pfx, dy = s_xy[j].y - pfy;
            const float rho2d = FILTER_INV_SQUARE * (dx * dx + dy * dy);
            const float rho = fminf(rho3d, rho2d);
            const float c_d = (rho3d <= rho2d) ? (s0 * Tw[0] + s1 * Tw[1]) + Tw[2] : Tw[2];
            if (c_d < NEAR_N) continue;
            const float4 no = s_no[j];
            const float opa = no.w, power = -0.5f * rho;
            if (power > 0.f) continue;
            const float G = __expf(power), alpha = fminf(0.99f, opa * G);
            if (alpha < 1.f / 255.f) continue;
            const int g = s_id[j];
            T = T / (1.f - alpha);
            const float w = alpha * T;
            float dL_dalpha = 0.f;
            for (int c = 0; c < 3; c++) {
                const float col = s_col[j][c];
                accum_rec[c] = last_alpha * last_color[c] + (1.f - last_alpha) * accum_rec[c];
                last_color[c] = col;
                dL_dalpha += (col - accum_rec[c]) * dL_dpixel[c];
                atomicAdd(&dL_dcolor[3 * (size_t)g + c], w * dL_dpixel[c]);
            }
            float dL_dz = 0.f;
            const float m_d = FAR_N / (FAR_N - NEAR_N) * (1 - NEAR_N / c_d);
            const float dmd_dd = (FAR_N * NEAR_N) / ((FAR_N - NEAR_N) * c_d * c_d);
            if (contributor == median_contributor - 1) dL_dz += dL_dmedian;
            const float dL_dweight = (final_D2 + m_d * m_d * final_A - 2 * m_d * final_D) * dL_dreg;
            dL_dalpha += dL_dweight - last_dL_dT;
            last_dL_dT = dL_dweight * alpha + (1 - alpha) * last_dL_dT;
            dL_dz += 2.0f * (T * alpha) * (m_d * final_A - final_D) * dL_dreg * dmd_dd;
            accum_depth_rec = last_alpha * last_depth + (1.f - last_alpha) * accum_depth_rec;
            last_depth = c_d;
            dL_dalpha += (c_d - accum_depth_rec) * dL_ddepth;
            accum_alpha_rec = last_alpha + (1.f - last_alpha) * accum_alpha_rec;
            dL_dalpha += (1 - accum_alpha_rec) * dL_daccum;
            const float nn[3] = {no.x, no.y, no.z};
            for (int c = 0; c < 3; c++) {
                accum_normal_rec[c] = last_alpha * last_normal[c] + (1.f - last_alpha) * accum_normal_rec[c];
                last_normal[c] = nn[c];
                dL_dalpha += (nn[c] - accum_normal_rec[c]) * dn[c];
                atomicAdd(&dL_dnormal[3 * (size_t)g + c], w * dn[c]);
            }
            dL_dalpha *= T;
            last_alpha = alpha;
            dL_dalpha += (-T_final / (1.f - alpha)) * bg_dot;
            const float dL_dG = opa * dL_dalpha;
            dL_dz += w * dL_ddepth;
            if (rho3d <= rho2d) {
                const float dL_ds0 = dL_dG * -G * s0 + dL_dz * Tw[0], dL_ds1 = dL_dG * -G * s1 + dL_dz * Tw[1];
                const float q0 = dL_ds0 / p2, q1 = dL_ds1 / p2, q2 = -(q0 * s0 + q1 * s1);
                const float dk0 = l1 * q2 - l2 * q1, dk1 = l2 * q0 - l0 * q2, dk2 = l0 * q1 - l1 * q0;
                const float dl0 = q1 * k2 - q2 * k1, dl1 = q2 * k0 - q0 * k2, dl2 = q0 * k1 - q1 * k0;
                float *gt = dL_dtransmat + 9 * (size_t)g;
                atomicAdd(gt + 0, -dk0); atomicAdd(gt + 1, -dk1); atomicAdd(gt + 2, -dk2);
                atomicAdd(gt + 3, -dl0); atomicAdd(gt + 4, -dl1); atomicAdd(gt + 5, -dl2);
                atomicAdd(gt + 6, pfx * dk0 + pfy * dl0 + dL_dz * s0);
                atomicAdd(gt + 7, pfx * dk1 + pfy * dl1 + dL_dz * s1);
                atomicAdd(gt + 8, pfx * dk2 + pfy * dl2 + dL_dz);
            } else {
                atomicAdd(&dL_dmean2D[2 * (size_t)g], dL_dG * (-G * FILTER_INV_SQUARE * dx));
                atomicAdd(&dL_dmean2D[2 * (size_t)g + 1], dL_dG * (-G * FILTER_INV_SQUARE * dy));
                atomicAdd(&dL_dtransmat[9 * (size_t)g + 8], dL_dz);
            }
            atomicAdd(&dL_dopacity[g], G * dL_dalpha);
        }
    }
}

// per-surfel backward of one view; ACCUMULATES into grad13 [P][13]
__global__ void st_preprocess_bwd(int P, const float *__restrict__ g13, const float *__restrict__ vm, const float *__restrict__ pm,
                                  int H, int W, float mod, const int *__restrict__ radii, const float *__restrict__ transmat,
                                  const float *__restrict__ dL_dtransmat, const float *__restrict__ dL_dmean2D,
                                  const float *__restrict__ dL_dnormal, const float *__restrict__ dL_dopacity,
                                  const float *__restrict__ dL_dcolor, float *grad13)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P || radii[i] <= 0) return;
    const float *g = g13 + (size_t)i * 13;
    float G[3][3];
    for (int c = 0; c < 3; c++) for (int r = 0; r < 3; r++) G[c][r] = dL_dtransmat[9 * (size_t)i + 3 * c + r];
    const float *Tm = transmat + 9 * (size_t)i;
    const float gmx = dL_dmean2D[2 * (size_t)i], gmy = dL_dmean2D[2 * (size_t)i + 1];
    if (gmx != 0.f || gmy != 0.f) {
        const float t[3] = {9.f, 9.f, -1.f};
        const float Tu[3] = {Tm[0], Tm[1], Tm[2]}, Tv[3] = {Tm[3], Tm[4], Tm[5]}, Tw[3] = {Tm[6], Tm[7], Tm[8]};
        float d = 0.f;
        for (int r = 0; r < 3; r++) d += t[r] * Tw[r] * Tw[r];
        float f[3], dL_dd = 0.f;
        for (int r = 0; r < 3; r++) f[r] = t[r] / d;
        for (int r = 0; r < 3; r++) {
            G[0][r] += gmx * f[r] * Tw[r]; G[1][r] += gmy * f[r] * Tw[r];
            G[2][r] += gmx * f[r] * Tu[r] + gmy * f[r] * Tv[r];
            dL_dd += (gmx * Tu[r] * Tw[r] + gmy * Tv[r] * Tw[r]) * f[r];
        }
        dL_dd *= (-1.0f / d);
        for (int r = 0; r < 3; r++) G[2][r] += dL_dd * t[r] * Tw[r] * 2.0f;
    }
    const float hw = 0.5f * W, hh = 0.5f * H, cw = 0.5f * (W - 1), ch = 0.5f * (H - 1);
    float dM[3][3];
    for (int k = 0; k < 3; k++) {
        const float an0 = pm[4 * k] * hw + pm[4 * k + 3] * cw, an1 = pm[4 * k + 1] * hh + pm[4 * k + 3] * ch, an2 = pm[4 * k + 3];
        for (int r = 0; r < 3; r++) dM[r][k] = an0 * G[0][r] + an1 * G[1][r] + an2 * G[2][r];
    }
    float R[3][3];
    quat_to_rotmat(g + 6, R);
    const float sx = mod * g[4], sy = mod * g[5], px = g[0], py = g[1], pz = g[2];
    const float vx = vm[0] * px + vm[4] * py + vm[8] * pz + vm[12], vy = vm[1] * px + vm[5] * py + vm[9] * pz + vm[13];
    const float vz = vm[2] * px + vm[6] * py + vm[10] * pz + vm[14];
    const float nx = vm[0] * R[0][2] + vm[4] * R[1][2] + vm[8] * R[2][2], ny = vm[1] * R[0][2] + vm[5] * R[1][2] + vm[9] * R[2][2];
    const float nz = vm[2] * R[0][2] + vm[6] * R[1][2] + vm[10] * R[2][2];
    const float mult = -(vx * nx + vy * ny + vz * nz) > 0.f ? 1.f : -1.f;
    const float gn0 = dL_dnormal[3 * (size_t)i], gn1 = dL_dnormal[3 * (size_t)i + 1], gn2 = dL_dnormal[3 * (size_t)i + 2];
    const float dtn[3] = {mult * (vm[0] * gn0 + vm[1] * gn1 + vm[2] * gn2), mult * (vm[4] * gn0 + vm[5] * gn1 + vm[6] * gn2),
                          mult * (vm[8] * gn0 + vm[9] * gn1 + vm[10] * gn2)};
    float dR[3][3], gs0 = 0, gs1 = 0;
    for (int k = 0; k < 3; k++) {
        dR[k][0] = dM[0][k] * sx; dR[k][1] = dM[1][k] * sy; dR[k][2] = dtn[k];
        gs0 += dM[0][k] * R[k][0]; gs1 += dM[1][k] * R[k][1];
    }
    const float s = rsqrtf(g[6] * g[6] + g[7] * g[7] + g[8] * g[8] + g[9] * g[9]);
    const float w = g[6] * s, x = g[7] * s, y = g[8] * s, z = g[9] * s;
    float *o = grad13 + (size_t)i * 13;
    o[0] += dM[2][0]; o[1] += dM[2][1]; o[2] += dM[2][2];
    o[3] += dL_dopacity[i];
    o[4] += mod * gs0; o[5] += mod * gs1;
    o[6] += 2 * (z * (dR[1][0] - dR[0][1]) + y * (dR[0][2] - dR[2][0]) + x * (dR[2][1] - dR[1][2]));
    o[7] += 2 * (-2 * x * (dR[1][1] + dR[2][2]) + y * (dR[1][0] + dR[0][1]) + z * (dR[2][0] + dR[0][2]) + w * (dR[2][1] - dR[1][2]));
    o[8] += 2 * (x * (dR[1][0] + dR[0][1]) - 2 * y * (dR[0][0] + dR[2][2]) + z * (dR[2][1] + dR[1][2]) + w * (dR[0][2] - dR[2][0]));
    o[9] += 2 * (x * (dR[2][0] + dR[0][2]) + y * (dR[2][1] + dR[1][2]) - 2 * z * (dR[0][0] + dR[1][1]) + w * (dR[1][0] - dR[0][1]));
    o[10] += dL_dcolor[3 * (size_t)i]; o[11] += dL_dcolor[3 * (size_t)i + 1]; o[12] += dL_dcolor[3 * (size_t)i + 2];
}

extern "C" void *st_create(int P, int H, int W)
{
    StCtx *c = new StCtx();
    c->P = P; c->H = H; c->W = W; c->gx = (W + BX - 1) / BX; c->gy = (H + BY - 1) / BY;
    const size_t HW = (size_t)H * W;
    bool ok = cudaMalloc(&c->transmat, sizeof(float) * 9 * P) == cudaSuccess && cudaMalloc(&c->normal_opacity, sizeof(float) * 4 * P) == cudaSuccess &&
              cudaMalloc(&c->xy, sizeof(float) * 2 * P) == cudaSuccess && cudaMalloc(&c->depth, sizeof(float) * P) == cudaSuccess &&
              cudaMalloc(&c->radii, sizeof(int) * P) == cudaSuccess && cudaMalloc(&c->tiles_touched, sizeof(uint32_t) * P) == cudaSuccess &&
              cudaMalloc(&c->offsets, sizeof(uint32_t) * P) == cudaSuccess && cudaMalloc(&c->rect, sizeof(int) * 4 * P) == cudaSuccess &&
              cudaMalloc(&c->ranges, sizeof(int2) * c->gx * c->gy) == cudaSuccess && cudaMalloc(&c->final_T, sizeof(float) * 3 * HW) == cudaSuccess &&
              cudaMalloc(&c->n_contrib, sizeof(int) * 2 * HW) == cudaSuccess && cudaMalloc(&c->dL_dtransmat, sizeof(float) * 18 * P) == cudaSuccess;
    if (!ok) { delete c; return nullptr; }
    c->dL_dmean2D = c->dL_dtransmat + 9 * (size_t)P; c->dL_dnormal = c->dL_dmean2D + 2 * (size_t)P;
    c->dL_dopacity = c->dL_dnormal + 3 * (size_t)P; c->dL_dcolor = c->dL_dopacity + P;
    cub::DeviceScan::InclusiveSum(nullptr, c->scan_bytes, c->tiles_touched, c->offsets, P);
    cudaMalloc(&c->scan_tmp, c->scan_bytes);
    return c;
}

extern "C" void st_destroy(void *h)
{
    StCtx *c = (StCtx *)h;
    if (!c) return;
    void *ptrs[] = {c->transmat, c->normal_opacity, c->xy, c->depth, c->radii, c->tiles_touched, c->offsets, c->rect, c->ranges,
                    c->final_T, c->n_contrib, c->dL_dtransmat, c->scan_tmp, c->sort_tmp, c->keys, c->keys_sorted, c->vals, c->vals_sorted};
    for (void *p : ptrs) if (p) cudaFree(p);
    delete c;
}

// one view forward; returns num_rendered (>= 0) or a negative CUDA error
extern "C" int st_forward(void *h, const float *g13, const float *vm, const float *pm, const float *bg, float mod, float *out_color,
                          float *out_allmap, int *out_radii, void *stream)
{
    StCtx *c = (StCtx *)h;
    cudaStream_t s = (cudaStream_t)stream;
    const int P = c->P;
    st_preprocess<<<(P + 255) / 256, 256, 0, s>>>(P, g13, vm, pm, c->H, c->W, c->gx, c->gy, mod, c->transmat, c->normal_opacity, c->xy,
                                                  c->depth, c->radii, c->tiles_touched, c->rect);
    cub::DeviceScan::InclusiveSum(c->scan_tmp, c->scan_bytes, c->tiles_touched, c->offsets, P, s);
    uint32_t n = 0;
    if (cudaMemcpyAsync(&n, c->offsets + P - 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, s) != cudaSuccess) return -1;
    if (cudaStreamSynchronize(s) != cudaSuccess) return -2;            // upstream reads num_rendered back here
    c->num_rendered = (int)n;
    if ((size_t)n > c->cap) {
        for (void *p : {(void *)c->keys, (void *)c->keys_sorted, (void *)c->vals, (void *)c->vals_sorted, c->sort_tmp}) if (p) cudaFree(p);
        c->cap = (size_t)n + n / 4 + 1024;
        cudaMalloc(&c->keys, 8 * c->cap); cudaMalloc(&c->keys_sorted, 8 * c->cap);
        cudaMalloc(&c->vals, 4 * c->cap); cudaMalloc(&c->vals_sorted, 4 * c->cap);
        cub::DeviceRadixSort::SortPairs(nullptr, c->sort_bytes, c->keys, c->keys_sorted, c->vals, c->vals_sorted, (int)c->cap);
        cudaMalloc(&c->sort_tmp, c->sort_bytes);
    }
    cudaMemsetAsync(c->ranges, 0, sizeof(int2) * c->gx * c->gy, s);
    if (n > 0) {
        st_duplicate<<<(P + 255) / 256, 256, 0, s>>>(P, c->depth, c->offsets, c->radii, c->rect, c->gx, c->keys, c->vals);
        int bit = 0;
        for (uint32_t t = (uint32_t)(c->gx * c->gy); t > 0; t >>= 1) bit++;
        cub::DeviceRadixSort::SortPairs(c->sort_tmp, c->sort_bytes, c->keys, c->keys_sorted, c->vals, c->vals_sorted, (int)n, 0, 32 + bit, s);
        st_ranges<<<(n + 255) / 256, 256, 0, s>>>((int)n, c->keys_sorted, c->ranges);
    }
    dim3 grid(c->gx, c->gy), block(BX, BY);
    st_render_fwd<<<grid, block, 0, s>>>(c->ranges, c->vals_sorted, c->W, c->H, c->xy, c->transmat, c->normal_opacity, g13, bg,
                                         c->final_T, c->n_contrib, out_color, out_allmap);
    if (out_radii) cudaMemcpyAsync(out_radii, c->radii, sizeof(int) * P, cudaMemcpyDeviceToDevice, s);
    return cudaGetLastError() == cudaSuccess ? (int)n : -3;
}

// one view backward; grad13 [P][13] is accumulated into (zero it before the first view)
extern "C" int st_backward(void *h, const float *g13, const float *vm, const float *pm, const float *bg, float mod,
                           const float *dL_dcolor_px, const float *dL_dallmap_px, float *grad13, void *stream)
{
    StCtx *c = (StCtx *)h;
    cudaStream_t s = (cudaStream_t)stream;
    const int P = c->P;
    cudaMemsetAsync(c->dL_dtransmat, 0, sizeof(float) * 18 * P, s);
    dim3 grid(c->gx, c->gy), block(BX, BY);
    if (c->num_rendered > 0)
        st_render_bwd<<<grid, block, 0, s>>>(c->ranges, c->vals_sorted, c->W, c->H, c->xy, c->transmat, c->normal_opacity, g13, bg,
                                             c->final_T, c->n_contrib, dL_dcolor_px, dL_dallmap_px, c->dL_dtransmat, c->dL_dmean2D,
                                             c->dL_dnormal, c->dL_dopacity, c->dL_dcolor);
    st_preprocess_bwd<<<(P + 255) / 256, 256, 0, s>>>(P, g13, vm, pm, c->H, c->W, mod, c->radii, c->transmat, c->dL_dtransmat,
                                                      c->dL_dmean2D, c->dL_dnormal, c->dL_dopacity, c->dL_dcolor, grad13);
    return (int)cudaGetLastError();
}
