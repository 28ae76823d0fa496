// K1: per-(view,surfel) stage of the surfel rasteriser, and K5: its backward.
//
// Restates upstream forward.cu preprocessCUDA / compute_transmat / compute_aabb
// and backward.cu compute_transmat_aabb (github.com/hbb1/diff-surfel-rasterization,
// called from /root/reference/nsr/gs_surfel.py:100-114), batched over every
// (batch item, view) of the loop at /root/reference/nsr/gs_surfel.py:65,74.
//
// THIS FILE IS COMPILED WITH --fmad=false: every float operation of K1 is a
// single IEEE binary32 op in the same order as oracle/surfel_oracle.c, which
// makes radii, tile rectangles, depth bits (sort keys) bit-exact.
#include "raster_common.cuh"

__device__ __forceinline__ void quat_to_rotmat(const float *q, float R[3][3])
{
    float n2 = ((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3];
    float s = 1.0f / sqrtf(n2);
    float w = q[0] * s, x = q[1] * s, y = q[2] * s, z = q[3] * s;
    R[0][0] = 1.f - 2.f * (y * y + z * z);
    R[1][0] = 2.f * (x * y + w * z);
    R[2][0] = 2.f * (x * z - w * y);
    R[0][1] = 2.f * (x * y - w * z);
    R[1][1] = 1.f - 2.f * (x * x + z * z);
    R[2][1] = 2.f * (y * z + w * x);
    R[0][2] = 2.f * (x * z + w * y);
    R[1][2] = 2.f * (y * z - w * x);
    R[2][2] = 1.f - 2.f * (x * x + y * y);
}

// T = (Tu, Tv, Tw): the surfel's ray-splat transform for one view, stored in the record.
__device__ __forceinline__ void surfel_transmat(const float R[3][3], float sx, float sy, float px, float py, float pz,
                                                const float *pm, int W, int H, float Tu[3], float Tv[3], float Tw[3])
{
    float L0[3] = {R[0][0] * sx, R[1][0] * sx, R[2][0] * sx};
    float L1[3] = {R[0][1] * sy, R[1][1] * sy, R[2][1] * sy};
    const float hw = 0.5f * (float)W, hh = 0.5f * (float)H;
    const float cw = 0.5f * (float)(W - 1), ch = 0.5f * (float)(H - 1);
    {
        float B0[3], B1[3], B3[3];   // columns j = 0,1,3 of B = M^T A
        B0[0] = (L0[0] * pm[0] + L0[1] * pm[4]) + L0[2] * pm[8];
        B0[1] = (L1[0] * pm[0] + L1[1] * pm[4]) + L1[2] * pm[8];
        B0[2] = ((px * pm[0] + py * pm[4]) + pz * pm[8]) + pm[12];
        B1[0] = (L0[0] * pm[1] + L0[1] * pm[5]) + L0[2] * pm[9];
        B1[1] = (L1[0] * pm[1] + L1[1] * pm[5]) + L1[2] * pm[9];
        B1[2] = ((px * pm[1] + py * pm[5]) + pz * pm[9]) + pm[13];
        B3[0] = (L0[0] * pm[3] + L0[1] * pm[7]) + L0[2] * pm[11];
        B3[1] = (L1[0] * pm[3] + L1[1] * pm[7]) + L1[2] * pm[11];
        B3[2] = ((px * pm[3] + py * pm[7]) + pz * pm[11]) + pm[15];
#pragma unroll
        for (int r = 0; r < 3; r++) {
            Tu[r] = B0[r] * hw + B3[r] * cw;
            Tv[r] = B1[r] * hh + B3[r] * ch;
            Tw[r] = B3[r];
        }
    }
}

__device__ __forceinline__ void preprocess_one(const RasterDims &d, const RasterWs &ws, const float *g,
                                               const float *s_cam, int view, int i, float4 *rec_out,
                                               int32_t *__restrict__ out_radii)
{
    const size_t vi = (size_t)view * d.P + i;
    const float *vm = s_cam, *pm = s_cam + 16;
    const int H = d.H, W = d.W;

    int radius_i = 0;
    uint32_t rect_packed = 0;
    float depth_out = 0.f;
    float rec[GA_REC_F];
#pragma unroll
    for (int k = 0; k < GA_REC_F; k++) rec[k] = 0.f;
    // empty cull box by default
    rec[16] = 1e30f; rec[17] = -1e30f; rec[18] = 1e30f; rec[19] = -1e30f;

    const float px = g[0], py = g[1], pz = g[2];
    float vx = ((vm[0] * px + vm[4] * py) + vm[8] * pz) + vm[12];
    float vy = ((vm[1] * px + vm[5] * py) + vm[9] * pz) + vm[13];
    float vz = ((vm[2] * px + vm[6] * py) + vm[10] * pz) + vm[14];
    if (vz > GA_NEAR_N) {
        float R[3][3];
        quat_to_rotmat(g + 6, R);
        const float sx = d.scale_modifier * g[4], sy = d.scale_modifier * g[5];
        float L2[3] = {R[0][2], R[1][2], R[2][2]};
        float Tu[3], Tv[3], Tw[3];
        surfel_transmat(R, sx, sy, px, py, pz, pm, W, H, Tu, Tv, Tw);
        float nx = (vm[0] * L2[0] + vm[4] * L2[1]) + vm[8] * L2[2];
        float ny = (vm[1] * L2[0] + vm[5] * L2[1]) + vm[9] * L2[2];
        float nz = (vm[2] * L2[0] + vm[6] * L2[1]) + vm[10] * L2[2];
        rec[0] = Tu[0]; rec[1] = Tu[1]; rec[2] = Tu[2];
        rec[3] = Tv[0]; rec[4] = Tv[1]; rec[5] = Tv[2];
        rec[6] = Tw[0]; rec[7] = Tw[1]; rec[8] = Tw[2];
        float cosv = -((vx * nx + vy * ny) + vz * nz);
        if (cosv != 0.f) {
            float mult = cosv > 0.f ? 1.f : -1.f;
            nx = mult * nx; ny = mult * ny; nz = mult * nz;
            const float t0 = GA_CUTOFF * GA_CUTOFF, t1 = GA_CUTOFF * GA_CUTOFF, t2 = -1.0f;
            float dd = (t0 * (Tw[0] * Tw[0]) + t1 * (Tw[1] * Tw[1])) + t2 * (Tw[2] * Tw[2]);
            if (dd != 0.0f) {
                float inv = 1.0f / dd;
                float f0 = inv * t0, f1 = inv * t1, f2 = inv * t2;
                float cx = (f0 * (Tu[0] * Tw[0]) + f1 * (Tu[1] * Tw[1])) + f2 * (Tu[2] * Tw[2]);
                float cy = (f0 * (Tv[0] * Tw[0]) + f1 * (Tv[1] * Tw[1])) + f2 * (Tv[2] * Tw[2]);
                float hx0 = cx * cx - ((f0 * (Tu[0] * Tu[0]) + f1 * (Tu[1] * Tu[1])) + f2 * (Tu[2] * Tu[2]));
                float hy0 = cy * cy - ((f0 * (Tv[0] * Tv[0]) + f1 * (Tv[1] * Tv[1])) + f2 * (Tv[2] * Tv[2]));
                float ex = sqrtf(fmaxf(1e-4f, hx0)), ey = sqrtf(fmaxf(1e-4f, hy0));
                float radius = d.radius_formula == 0 ? ceilf(fmaxf(fmaxf(ex, ey), GA_CUTOFF * GA_FILTER_SIZE))
                                                     : ceilf(GA_CUTOFF * fmaxf(fmaxf(ex, ey), GA_FILTER_SIZE));
                int mr = (int)radius;
                int x0 = min(d.gx, max(0, (int)((cx - (float)mr) / (float)GA_BLOCK_X)));
                int y0 = min(d.gy, max(0, (int)((cy - (float)mr) / (float)GA_BLOCK_Y)));
                int x1 = min(d.gx, max(0, (int)((cx + (float)mr + (float)(GA_BLOCK_X - 1)) / (float)GA_BLOCK_X)));
                int y1 = min(d.gy, max(0, (int)((cy + (float)mr + (float)(GA_BLOCK_Y - 1)) / (float)GA_BLOCK_Y)));
                if ((x1 - x0) * (y1 - y0) != 0) {
                    radius_i = mr;
                    depth_out = vz;
                    rect_packed = (uint32_t)x0 | ((uint32_t)y0 << 8) | ((uint32_t)x1 << 16) | ((uint32_t)y1 << 24);
                    const float opa = g[3];
                    rec[9] = cx; rec[10] = cy; rec[11] = opa;
                    rec[12] = nx; rec[13] = ny; rec[14] = nz; rec[15] = g[10];
                    rec[20] = g[11]; rec[21] = g[12];
                    // the backward's normal sign, cosv > 0 ? 1 : -1; a surfel with cosv == 0 gets no tiles, so the
                    // sign of every instance the backward reads is this one
                    rec[22] = mult;
                    // ---- conservative cull box: a pixel outside can never reach
                    // alpha >= 1/255, i.e. needs min(rho3d, rho2d) <= tau = 2 ln(255 o).
                    float bx0 = 1e30f, bx1 = -1e30f, by0 = 1e30f, by1 = -1e30f;
                    float a255 = 255.0f * opa;
                    if (a255 >= 1.0f) {
                        float tau = 2.0f * logf(a255) * 1.001f + 1e-3f;
                        float r2 = sqrtf(0.5f * tau) + 0.51f;       // low-pass disc
                        bx0 = cx - r2; bx1 = cx + r2; by0 = cy - r2; by1 = cy + r2;
                        float dt = tau * (Tw[0] * Tw[0] + Tw[1] * Tw[1]) - Tw[2] * Tw[2];
                        if (Tw[2] > 0.f && dt < -1e-3f * (Tw[2] * Tw[2])) {
                            float iv = 1.0f / dt;
                            float g0 = iv * tau, g2 = -iv;
                            float ccx = g0 * (Tu[0] * Tw[0] + Tu[1] * Tw[1]) + g2 * (Tu[2] * Tw[2]);
                            float ccy = g0 * (Tv[0] * Tw[0] + Tv[1] * Tw[1]) + g2 * (Tv[2] * Tw[2]);
                            float qx = ccx * ccx - (g0 * (Tu[0] * Tu[0] + Tu[1] * Tu[1]) + g2 * (Tu[2] * Tu[2]));
                            float qy = ccy * ccy - (g0 * (Tv[0] * Tv[0] + Tv[1] * Tv[1]) + g2 * (Tv[2] * Tv[2]));
                            float hx = sqrtf(fmaxf(0.f, qx)) * 1.01f + 0.51f;
                            float hy = sqrtf(fmaxf(0.f, qy)) * 1.01f + 0.51f;
                            bx0 = fminf(bx0, ccx - hx); bx1 = fmaxf(bx1, ccx + hx);
                            by0 = fminf(by0, ccy - hy); by1 = fmaxf(by1, ccy + hy);
                        } else {
                            bx0 = -1e30f; bx1 = 1e30f; by0 = -1e30f; by1 = 1e30f;
                        }
                    }
                    rec[16] = bx0; rec[17] = bx1; rec[18] = by0; rec[19] = by1;
                }
            }
        }
    }
    out_radii[vi] = radius_i;
    ws.depth[vi] = depth_out;
    ws.rect[vi] = rect_packed;
#pragma unroll
    for (int q = 0; q < GA_REC_F / 4; q++)
        rec_out[q] = make_float4(rec[4 * q], rec[4 * q + 1], rec[4 * q + 2], rec[4 * q + 3]);
    if (radius_i > 0) {
        const int x0 = rect_packed & 255, y0 = (rect_packed >> 8) & 255;
        const int x1 = (rect_packed >> 16) & 255, y1 = rect_packed >> 24;
        uint32_t *tc = ws.tile_count + (size_t)view * d.T * GA_TILE_REPLICAS + ((threadIdx.x >> 5) & (GA_TILE_REPLICAS - 1));
        for (int y = y0; y < y1; y++)
            for (int x = x0; x < x1; x++) atomicAdd(&tc[(y * d.gx + x) * GA_TILE_REPLICAS], 1u);
    }
}

// The CTA's 256 records are staged in shared memory and written out as whole lines (a thread's own record is
// 96 bytes, so per-thread float4 stores would leave every store instruction touching 32 different lines).
__global__ void __launch_bounds__(256, 4)
preprocess_kernel(RasterDims d, RasterWs ws, const float *__restrict__ gauss13,
                  const float *__restrict__ viewmats, const float *__restrict__ projmats,
                  int32_t *__restrict__ out_radii)
{
    __shared__ float s_g[256 * 13];
    __shared__ float s_cam[32];
    __shared__ float4 s_rec[256 * GA_REC_F / 4];
    const int view = blockIdx.y;
    const int b = view / d.views;
    const int i0 = blockIdx.x * 256;
    const int n = min(256, d.P - i0);
    const float *src = gauss13 + ((size_t)b * d.P + i0) * 13;
    for (int t = threadIdx.x; t < n * 13; t += 256) s_g[t] = src[t];
    if (threadIdx.x < 16) s_cam[threadIdx.x] = viewmats[view * 16 + threadIdx.x];
    else if (threadIdx.x < 32) s_cam[threadIdx.x] = projmats[view * 16 + threadIdx.x - 16];
    __syncthreads();
    if ((int)threadIdx.x < n) preprocess_one(d, ws, s_g + threadIdx.x * 13, s_cam, view, i0 + threadIdx.x,
                                             s_rec + threadIdx.x * (GA_REC_F / 4), out_radii);
    __syncthreads();
    float4 *dst = reinterpret_cast<float4 *>(ws.rec + ((size_t)view * d.P + i0) * GA_REC_F);
    for (int t = threadIdx.x; t < n * (GA_REC_F / 4); t += 256) dst[t] = s_rec[t];
}

cudaError_t ga_launch_preprocess(const RasterDims &d, const RasterWs &w, const float *gauss13,
                                 const float *viewmats, const float *projmats,
                                 int32_t *out_radii, cudaStream_t s)
{
    dim3 grid((d.P + 255) / 256, d.NV);
    preprocess_kernel<<<grid, 256, 0, s>>>(d, w, gauss13, viewmats, projmats, out_radii);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------
// K5: per-surfel backward from the surfel's gradient row.
// grad_rows: [batch][P][16], already summed over the views of the batch item by render_bwd, which also applied each
// view's chain rule through T = (Tu, Tv, Tw) and the normal (layout in raster_common.cuh).  What is left depends on
// the surfel alone.  A surfel with radii <= 0 in a view got no tiles there from K1 (its rectangle is empty), so that
// view added nothing to its row.  grad_gauss13 [batch][P][13].
// ---------------------------------------------------------------------------
// One surfel: its 13 inputs at g (shared memory) are replaced by its 13 gradient columns; row = its gradient row.
__device__ __forceinline__ void preprocess_bwd_one(const RasterDims &d, float *g, const float4 *row)
{
    float q[4] = {g[6], g[7], g[8], g[9]};
    float R[3][3];
    quat_to_rotmat(q, R);
    const float sx = d.scale_modifier * g[4], sy = d.scale_modifier * g[5];
    const float4 r0 = row[0], r1 = row[1], r2 = row[2], r3 = row[3];
    const float dM[3][3] = {{r0.x, r0.y, r0.z}, {r0.w, r1.x, r1.y}, {r1.z, r1.w, r2.x}};
    const float dtn[3] = {r2.y, r2.z, r2.w};
    float gm[3], gs[2] = {0, 0}, dR[3][3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        dR[k][0] = dM[0][k] * sx;
        dR[k][1] = dM[1][k] * sy;
        dR[k][2] = dtn[k];
        gs[0] += dM[0][k] * R[k][0];
        gs[1] += dM[1][k] * R[k][1];
        gm[k] = dM[2][k];
    }
    const float gop = r3.x, gcol[3] = {r3.y, r3.z, r3.w};
    float n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    float s = rsqrtf(n2);
    float w = q[0] * s, x = q[1] * s, y = q[2] * s, z = q[3] * s;
    float gw = 2 * (z * (dR[1][0] - dR[0][1]) + y * (dR[0][2] - dR[2][0]) + x * (dR[2][1] - dR[1][2]));
    float gxq = 2 * (-2 * x * (dR[1][1] + dR[2][2]) + y * (dR[1][0] + dR[0][1]) + z * (dR[2][0] + dR[0][2]) + w * (dR[2][1] - dR[1][2]));
    float gyq = 2 * (x * (dR[1][0] + dR[0][1]) - 2 * y * (dR[0][0] + dR[2][2]) + z * (dR[2][1] + dR[1][2]) + w * (dR[0][2] - dR[2][0]));
    float gzq = 2 * (x * (dR[2][0] + dR[0][2]) + y * (dR[2][1] + dR[1][2]) - 2 * z * (dR[0][0] + dR[1][1]) + w * (dR[1][0] - dR[0][1]));
    if (d.quat_norm_grad) {          // chain through q_hat = q / |q|: g_raw = (g - q_hat (q_hat . g)) / |q|
        const float dot = w * gw + x * gxq + y * gyq + z * gzq;
        gw = (gw - w * dot) * s; gxq = (gxq - x * dot) * s; gyq = (gyq - y * dot) * s; gzq = (gzq - z * dot) * s;
    }
    float *o = g;                    // the inputs are all read above; the outputs take their place
    o[0] = gm[0]; o[1] = gm[1]; o[2] = gm[2];
    o[3] = gop;
    o[4] = d.scale_modifier * gs[0]; o[5] = d.scale_modifier * gs[1];
    o[6] = gw; o[7] = gxq; o[8] = gyq; o[9] = gzq;
    o[10] = gcol[0]; o[11] = gcol[1]; o[12] = gcol[2];
}

// The CTA's 256 surfels and their 13 output columns are staged in shared memory and moved as whole lines, as in K1:
// a thread's own 52 bytes would make every load and store instruction touch 32 different lines.
__global__ void __launch_bounds__(256)
preprocess_bwd_kernel(RasterDims d, const float *__restrict__ gauss13, const float *__restrict__ grad_rows,
                      float *__restrict__ grad_gauss13)
{
    __shared__ float s_g[256 * 13];
    const int b = blockIdx.y;
    const int i0 = blockIdx.x * 256;
    const int n = min(256, d.P - i0);
    const size_t base = ((size_t)b * d.P + i0) * 13;
    for (int t = threadIdx.x; t < n * 13; t += 256) s_g[t] = gauss13[base + t];
    __syncthreads();
    if ((int)threadIdx.x < n)
        preprocess_bwd_one(d, s_g + threadIdx.x * 13,
                           reinterpret_cast<const float4 *>(grad_rows + ((size_t)b * d.P + i0 + threadIdx.x) * GA_ROW_F));
    __syncthreads();
    for (int t = threadIdx.x; t < n * 13; t += 256) grad_gauss13[base + t] = s_g[t];
}

cudaError_t ga_launch_preprocess_bwd(const RasterDims &d, const float *gauss13, const float *grad_rows,
                                     float *grad_gauss13, cudaStream_t s)
{
    dim3 grid((d.P + 255) / 256, d.batch);
    preprocess_bwd_kernel<<<grid, 256, 0, s>>>(d, gauss13, grad_rows, grad_gauss13);
    return cudaGetLastError();
}
