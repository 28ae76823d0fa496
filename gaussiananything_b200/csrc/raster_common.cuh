// Shared definitions of the surfel rasteriser kernels (sm_90a).
// Algorithm: github.com/hbb1/diff-surfel-rasterization as called by
// /root/reference/nsr/gs_surfel.py:85-114; constants per SURVEY.md App. A.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define GA_BLOCK_X 16
#define GA_BLOCK_Y 16
#define GA_NEAR_N 0.2f
#define GA_FAR_N 100.0f
#define GA_FILTER_SIZE 0.707106f
#define GA_FILTER_INV_SQUARE 2.0f
#define GA_CUTOFF 3.0f
#define GA_REC_F 24
#define GA_GRAD_F 18
#define GA_ROW_F 16

// record float offsets (6 x float4):
//  q0 = Tu.x Tu.y Tu.z Tv.x | q1 = Tv.y Tv.z Tw.x Tw.y | q2 = Tw.z xy.x xy.y opacity
//  q3 = n.x n.y n.z r        | q4 = bbox x0 x1 y0 y1    | q5 = g b sign -
// sign: +1 or -1, the factor K1 applied to the view-space normal so that it faces the camera.
// Per-(tile, instance) gradient components that the backward's phase B sums over a surfel's records (GA_GRAD_F):
//  0-8 dL/dT (Tu,Tv,Tw) | 9-10 dL/dmean2D | 11-13 dL/dnormal | 14 dL/dopacity | 15-17 dL/drgb
// Per-surfel gradient row, summed over the views of the batch item (GA_ROW_F), [batch][P][16]:
//  0-8 dL/dM, entry 3r+k = row r (0: scale-x axis, 1: scale-y axis, 2: position) and world axis k | 9-11 dL/dR column
//  2 (the normal) | 12 dL/dopacity | 13-15 dL/drgb
// The map from the 18 components to the row is linear and depends only on the view and on the record, so the
// backward applies it to each (tile, instance) partial sum before it adds the partial to the row.

struct RasterDims {
    int batch, P, views, NV;   // NV = batch*views images
    int H, W, gx, gy, T;       // T = gx*gy tiles per image
    float scale_modifier;
    int64_t max_instances;
    int list_k;                // > 0: the forward records every pixel's contributions (<= list_k per pixel), see RasterWs.lists
    // the two unpinned judgement calls of the restatement (oracle/surfel_oracle.c), switchable so that pinning against
    // upstream is a flip of the defaults below; ga_raster_set_variant() overrides them at run time (tests)
    int radius_formula;        // 0: ceil(max(ex, ey, 3*FilterSize))   1: ceil(3*max(ex, ey, FilterSize))
    int quat_norm_grad;        // 0: quaternion vjp not chained through q/|q| (upstream)   1: chained
};
#ifndef GA_RADIUS_FORMULA
#define GA_RADIUS_FORMULA 0
#endif
#ifndef GA_QUAT_NORM_GRAD
#define GA_QUAT_NORM_GRAD 0
#endif

struct RasterWs {
    int32_t *status;
    float *rec;
    float *depth;
    uint32_t *rect;
    uint32_t *tile_count;
    uint32_t *big_tiles;       // tiles above 512 instances, listed by the tile scan as a diagnostic (status[3]
                               // entries); kept in the tile_count region of the layout, after the counters
    uint32_t *tile_start;
    unsigned long long *keys;
    uint32_t *ids;
    float *final_T;
    int32_t *n_contrib;
    // per-pixel contribution lists written by the forward when list_k > 0 (the backward then neither culls nor
    // re-evaluates pairs): entry k of pixel p of tile t at lists[(t * list_k + k) * 256 + p] = {list position, alpha
    // bits, depth bits, 0}; n_list[pixel] = contributions of the pixel; tile_flag[t] = 1 when a pixel of the tile had
    // more than list_k (that tile's backward recomputes instead)
    uint4 *lists;
    int32_t *n_list;
    uint32_t *tile_flag;
    uint32_t *inst_cnt;        // (list_k > 0) contributions of every instance, counted by the forward
};

// kernel launchers (defined in the .cu files, called from raster_api.cu)
cudaError_t ga_launch_preprocess(const RasterDims &d, const RasterWs &w, const float *gauss13,
                                 const float *viewmats, const float *projmats,
                                 int32_t *out_radii, cudaStream_t s);
// status_host / status_event (both NULL, or both set): after the tile scan -- the first point where the instance
// count and the overflow flag are known -- status[0..3] is copied to pinned host memory and the event recorded, so
// the host can look at them while the scatter and composite kernels are still running.
// Tile counters / scatter cursors are kept in GA_TILE_REPLICAS copies per tile (replica = warp index mod R): the
// 1.05M atomics of the C2 scene otherwise queue up on 6144 addresses, ~170 deep, and L2 serialises same-address
// atomics (scatter: 48 us for 1M atomics).  The scan sums the replicas of a tile and hands every replica its own
// sub-range of the tile's slots; the forward sorts each tile before it composites, so results do not change.
#ifndef GA_TILE_REPLICAS
#define GA_TILE_REPLICAS 8
#endif

cudaError_t ga_launch_binning(const RasterDims &d, const RasterWs &w, cudaStream_t s, int32_t *status_host,
                              cudaEvent_t status_event);
cudaError_t ga_launch_render_fwd(const RasterDims &d, const RasterWs &w, const float *bg,
                                 float *out_color, float *out_allmap, cudaStream_t s);
// grad_rows: [batch][P][GA_ROW_F], zeroed by the caller; render_bwd adds into it and preprocess_bwd reads it
cudaError_t ga_launch_render_bwd(const RasterDims &d, const RasterWs &w, const float *bg,
                                 const float *viewmats, const float *projmats,
                                 const float *dL_dcolor, const float *dL_dallmap,
                                 float *grad_rows, cudaStream_t s);
cudaError_t ga_launch_preprocess_bwd(const RasterDims &d, const float *gauss13, const float *grad_rows,
                                     float *grad_gauss13, cudaStream_t s);
