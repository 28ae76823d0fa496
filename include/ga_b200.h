/*
 * ga_b200.h -- C ABI of libga_b200.so: H100 (sm_90a) kernels for the two hot
 * paths of GaussianAnything.  Plain pointers and sizes only; no torch types.
 *
 * All pointers are DEVICE pointers unless stated otherwise.  No entry point
 * allocates, frees or synchronises; everything is enqueued on `stream`
 * (a cudaStream_t passed as void*).  Return value: 0 on success, a negative
 * GA_ERR_* code on a bad argument, or a positive cudaError_t from the launch.
 *
 * ---------------------------------------------------------------------------
 * Part 1: surfel (2D Gaussian) rasteriser.
 * Replaces the native module `diff_surfel_rasterization._C` that the reference
 * binds at /root/reference/nsr/gs_surfel.py:15 and calls at
 * /root/reference/nsr/gs_surfel.py:100-114 (`_C.rasterize_gaussians`,
 * `_C.rasterize_gaussians_backward`), batched over every (batch item, view)
 * of the Python loop at /root/reference/nsr/gs_surfel.py:65,74.
 * ---------------------------------------------------------------------------
 */
#ifndef GA_B200_H
#define GA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GA_ERR_BADARG   (-1)
#define GA_ERR_WORKSPACE (-2)   /* workspace too small for the stated sizes */
#define GA_ERR_SIZE     (-3)    /* image larger than 4080 px or P*views overflow */

#define GA_RASTER_REC_FLOATS 24   /* packed per-(view,surfel) record, 96 bytes */
#define GA_RASTER_GRAD_FLOATS 18  /* per-(view,surfel) gradient accumulator */

/* Byte offsets of the sections inside the forward workspace.  The forward
 * pass fills them; the backward pass reads them (the workspace is the
 * equivalent of upstream's geomBuffer/binningBuffer/imgBuffer). */
typedef struct GaRasterLayout {
    size_t total_bytes;
    size_t status;      /* int32[16]: [0]=instances D, [1]=overflow flag, [2]=tiles above 4096 instances (sorted in global memory), [3]=tiles above 512 */
    size_t rec;         /* float[NV*P][24]  Tu3 Tv3 Tw3 | xy2 opacity | normal3 | r | bbox x0 x1 y0 y1 | g b - - */
    size_t depth;       /* float[NV*P]      view-space z (0 when culled) */
    size_t rect;        /* uint32[NV*P]     x0 | y0<<8 | x1<<16 | y1<<24 (tile units) */
    size_t tile_count;  /* uint32[NV*T*9]   scratch: per-tile counters, then fill cursors (8 replicas per tile); then the list of tiles above 512 instances */
    size_t tile_start;  /* uint32[NV*T+1]   exclusive scan == tile ranges [start,end) */
    size_t keys;        /* uint64[max_instances]  (depth bits<<32 | surfel), sorted per tile */
    size_t ids;         /* uint32[max_instances]  sorted surfel index per instance */
    size_t final_T;     /* float[NV][3][H*W]  T, M1, M2 */
    size_t n_contrib;   /* int32[NV][2][H*W]  last contributor, median contributor */
    size_t inst_cnt;    /* uint32[max_instances]  (list_k > 0) contributions of every instance, counted by the forward */
    size_t n_list;      /* int32[NV][H*W]         (list_k > 0) contributions recorded per pixel */
    size_t tile_flag;   /* uint32[NV*T]           (list_k > 0) 1: a pixel of the tile had more than list_k */
    size_t lists;       /* uint4[NV*T][list_k][256] (list_k > 0) {list position, alpha bits, depth bits, 0} */
} GaRasterLayout;

/* Fills *layout for NV = batch*views images of H x W, P surfels per batch item
 * and room for max_instances (surfel,tile) pairs over all images, plus room for
 * the per-pixel contribution lists the forward records when list_k > 0
 * (list_k * 4 KB per tile; 32 is the default the Python mirror uses for calls
 * that need gradients, 0 records none).  Host-only, no CUDA call. */
int ga_raster_layout_ex(int batch, int P, int views, int H, int W,
                        int64_t max_instances, int list_k, GaRasterLayout *layout);

/*
 * Forward.  gauss13: [batch][P][13] = xyz3 opacity1 scale2 quat4(wxyz) rgb3, the
 * layout of /root/reference/nsr/gs_surfel.py:68-72.  viewmats / projmats:
 * [batch*views][16] exactly as the reference passes `viewmatrix` /
 * `projmatrix` (row-vector convention).  bg: [3].
 * Outputs: out_color [NV][3][H][W], out_allmap [NV][7][H][W] (channel order of
 * /root/reference/nsr/gs_surfel.py:121-142), out_radii int32 [NV][P].
 * If the instance count exceeds max_instances, status[1] is set and the
 * images are undefined (no out-of-bounds access happens); the caller re-runs
 * with a larger workspace.
 *
 * list_k > 0 makes the composite record, for every pixel, the (list position, alpha, depth) of each surfel that
 * contributed (up to list_k per pixel; a tile with a longer pixel is flagged and its backward recomputes).
 * ga_raster_backward_ex with the same list_k then walks those lists instead of re-culling and re-evaluating every
 * (pixel, surfel) pair -- what upstream's backward.cu renderCUDA does.  The workspace must be laid out with the
 * same list_k.
 *
 * Status read-back: status_host and status_event are both NULL, or both set.  When set, right after the tile scan
 * (before the scatter and the composite, which sorts each tile) status[0..3] = {instance count, overflow flag, 0,
 * tiles above 512 instances} is copied to `status_host` (pinned host memory, 4 ints) and `status_event` (a cudaEvent_t) is
 * recorded.  The caller synchronises on the event -- the GPU is still busy with the rest of the forward -- and, if
 * the overflow flag is set, re-runs with a larger workspace (the kernels after the scan exit early in that case).
 */
int ga_raster_forward_ex(const float *gauss13, int batch, int P, int views,
                         const float *viewmats, const float *projmats, const float *bg,
                         int H, int W, float scale_modifier,
                         float *out_color, float *out_allmap, int32_t *out_radii,
                         void *workspace, size_t workspace_bytes, int64_t max_instances, int list_k,
                         int32_t *status_host, void *status_event, void *stream);

/* Bytes of scratch the backward wants: the gradient accumulators [NV*P][18].  A larger buffer is accepted; the
 * rest of it is not used. */
size_t ga_raster_backward_scratch_bytes(int batch, int P, int views);

/*
 * Backward.  dL_dcolor [NV][3][H][W], dL_dallmap [NV][7][H][W]; grad_gauss13
 * [batch][P][13] is OVERWRITTEN with the gradient summed over the views of
 * each batch item (same column order as gauss13).  workspace and list_k must
 * be the ones the matching ga_raster_forward_ex filled and used.
 */
int ga_raster_backward_ex(const float *gauss13, int batch, int P, int views,
                          const float *viewmats, const float *projmats, const float *bg,
                          int H, int W, float scale_modifier,
                          const int32_t *radii,
                          const float *dL_dcolor, const float *dL_dallmap,
                          const void *workspace, size_t workspace_bytes, int64_t max_instances, int list_k,
                          void *scratch, size_t scratch_bytes,
                          float *grad_gauss13, void *stream);

/* Post-processing of /root/reference/nsr/gs_surfel.py:121-163 for all views at once: image = clamp(color,0,1),
 * alpha = allmap[1], depth = nan_to_num(allmap[5], 0, 0), normal[d] = sum_c allmap[2+c] * view[d][c], dist = allmap[6].
 * color [NV,3,H,W], allmap [NV,7,H,W], viewmats [NV,16] (as passed to the rasteriser); outputs contiguous. */
int ga_render_post_forward(const float *color, const float *allmap, const float *viewmats, int num_views,
                           int H, int W, float *image, float *alpha, float *depth, float *normal, float *dist,
                           void *stream);
/* Its backward: any g_* may be NULL (= zero); writes g_color [NV,3,H,W] and g_allmap [NV,7,H,W]. */
int ga_render_post_backward(const float *color, const float *allmap, const float *viewmats, int num_views,
                            int H, int W, const float *g_image, const float *g_alpha, const float *g_depth,
                            const float *g_normal, const float *g_dist, float *g_color, float *g_allmap, void *stream);

/*
 * The two judgement calls of the (parity-unpinned) restatement of upstream's preprocess stage, switchable at run
 * time; the process-wide defaults are the compile-time macros GA_RADIUS_FORMULA / GA_QUAT_NORM_GRAD (both 0):
 *   radius_formula 0: radius = ceil(max(extent.x, extent.y, 3*FilterSize))   1: ceil(3*max(extent.x, extent.y, FilterSize))
 *   quat_norm_grad 0: dL/dquat is the vjp at q/|q|, not chained through the normalisation   1: chained
 * Replaces nothing in the reference (upstream hard-codes its choice); exists so that pinning against
 * github.com/hbb1/diff-surfel-rasterization forward.cu / backward.cu is a one-line flip.  oracle/surfel_oracle.c
 * has the same switch (so_set_variant).  Affects calls made after it returns.
 */
int ga_raster_set_variant(int radius_formula, int quat_norm_grad);

/*
 * ---------------------------------------------------------------------------
 * Part 2: DiT denoiser forward (bf16 tensor-core path, fp32 residual stream).
 * Replaces, for DiT_I23D_PCD_PixelArt_noclip[_clay_stage2].forward
 * (/root/reference/dit/dit_i23d.py:511-567,707-750) and its block
 * ImageCondDiTBlockPixelArtRMSNormClayLRM.forward
 * (/root/reference/dit/dit_models_xformers.py:765-787), the cuBLAS nn.Linear
 * calls, xformers.ops.memory_efficient_attention
 * (/root/reference/vit/vision_transformer.py:297,
 * /root/reference/ldm/modules/attention.py:538-546), xformers FusedMLP
 * (/root/reference/dit/dit_models_xformers.py:281-286) and the RMSNorm /
 * modulate / gate / residual elementwise launches around them.
 * ---------------------------------------------------------------------------
 */

/* Epilogues fused into the wgmma GEMM  C[M,N] = A[M,K] * W[N,K]^T (+ bias). */
#define GA_EPI_BF16            0   /* out bf16 [M, ld_out]                                   */
#define GA_EPI_GELU_BF16       1   /* out bf16 = gelu_erf(acc + bias)   (FusedMLP first half) */
#define GA_EPI_F32             2   /* out fp32 [M, ld_out]                                   */
#define GA_EPI_RESID_GATE_F32  3   /* out fp32 [M, ld_out] += gate[m / rows_per_batch, n] * (acc + bias)   */
#define GA_EPI_HEADS           4   /* split columns "(K H 64)" into heads: per-head RMSNorm on q/k, write
                                      Q,K [B,H,tok_pitch,64] and V transposed [B,H,64,tok_pitch] (bf16) */
#define GA_EPI_GEGLU_BF16      5   /* W rows interleaved as (x_j, gate_j) pairs: out bf16 [M, ld_out] column j =
                                      (acc + bias)[2j] * gelu_erf((acc + bias)[2j+1])  (GEGLU, N/2 columns) */

typedef struct GaGemmEpilogue {
    int mode;
    const float *bias;        /* [N] or NULL */
    void *out;                /* modes 0-3 */
    int ld_out;
    const float *gate;        /* mode 3: [batch, gate_ld] (already offset to the gate chunk) or NULL (= 1) */
    int gate_ld;
    int rows_per_batch;       /* tokens per batch item (modes 3, 4) */
    void *q, *k, *vt;         /* mode 4 outputs (any may be NULL when that part is absent) */
    const float *qn_w, *kn_w; /* per-head RMSNorm weights [64] (NULL = no norm) */
    int heads;
    int first_part;           /* mode 4: 0 when columns start with q, 1 when they start with k (cross-attn k|v) */
    int tok_pitch;            /* padded token count of the Q/K rows and Vt columns (multiple of 128) */
    float eps;
} GaGemmEpilogue;

/* A [M, lda] bf16 row-major, W [N, ldw] bf16 row-major (nn.Linear weight), K contiguous in both.
 * block_n = tile width {64, 128, 192, 256} of the 128 x width output tile (192: not for GA_EPI_HEADS).
 * lda, ldw multiples of 8. */
int ga_gemm_bf16_tn(const void *A, int lda, const void *W, int ldw, int M, int N, int K,
                    const GaGemmEpilogue *epi, int block_n, void *stream);

/* softmax(Q K^T * softmax_scale) V, head_dim 64.  Q [B*H, pitch_q, 64], K [B*H, pitch_k, 64],
 * Vt [B*H, 64, pitch_k] (bf16, padding beyond Nk must be finite); out [B, Nq, H*64] bf16.
 * pitch_k must be a multiple of 128. */
int ga_attention_bf16(const void *Q, const void *K, const void *Vt, void *out, int batch, int heads,
                      int Nq, int Nk, int pitch_q, int pitch_k, float softmax_scale, float score_bound,
                      void *stream);
/* score_bound: an upper bound of |q.k| * softmax_scale over all (q, k) pairs, or <= 0 if unknown.  With
 * RMS-normalised q and k (the DiT's qk-norm) it is 64 * max|w_q| * max|w_k| * softmax_scale; when given
 * (and <= 40) the kernel uses it instead of a running row maximum (same result, one pass over the scores). */

/* out_bf16[r,:] = RMSNorm(x[r,:]; eps) * w [* (1 + scale[b,:]) + shift[b,:]], b = r / rows_per_batch;
 * shift/scale both NULL or both set, rows mod_ld apart. */
int ga_rmsnorm_modulate(const float *x, const float *w, const float *shift, const float *scale,
                        int mod_ld, int rows_per_batch, void *out_bf16, int R, int D, float eps, void *stream);

/* y[b,n] (+)= act_out(bias[n] + sum_k act_in(x[b,k]) W[n,k]);  rows <= 16; act: 0 none, 1 SiLU. */
int ga_linear_small(const float *x, const float *W, const float *bias, float *y, int rows, int N, int K,
                    int act_in, int act_out, int accumulate, void *stream);
int ga_timestep_sinusoid(const float *t, float *out, int rows, int dim, void *stream);
int ga_layernorm_rows(const float *x, const float *w, const float *b, float *y, int R, int D, float eps, void *stream);
/* mod[l,b,e] = tables[l,e] + t0[b, e % t0_ld], e in [0, JD) */
int ga_add_tables(const float *tables, const float *t0, float *mod, int L, int rows, int JD, int t0_ld, void *stream);
/* h = gelu_tanh(W1 [xin2 | xin] + b1) -> bf16 [R, D] (token embedder, first layer) */
int ga_embed_fc1(const float *xin, int Cx, const float *xin2, int C2, const float *W1, const float *b1,
                 void *h_bf16, int R, int D, void *stream);
/* NeRF positional encoding of xyz (63 features, padded to 64) -> bf16 [R, 64] */
int ga_xyz_posenc(const float *xyz, void *out_bf16, int R, void *stream);
/* y[r,c] = bias[c] + sum_d (LayerNorm(x[r])[d] (1 + scale[b,d]) + shift[b,d]) W[c,d]; mod [B,2,D]; Cout <= 16 */
int ga_final_layer(const float *x, const float *mod, const float *W, const float *bias, float *y, int R,
                   int D, int Cout, int rows_per_batch, float eps, void *stream);
/* eps [2*half] = (cond | uncond) -> h = u + s (c - u) written to both halves of out */
int ga_cfg_combine(const float *eps, float *out, int64_t half_elems, float cfg_scale, void *stream);
int ga_axpy(float *x, const float *v, float a, int64_t n, void *stream);          /* x += a v */
int ga_f32_to_bf16(const float *x, void *y, int64_t n, void *stream);

/* ---- VAE decode path latent tokens -> surfels (SURVEY 8f row N1; building blocks) -------------
 * Replaces the elementwise / small-matrix torch ops of /root/reference/vit/vit_triplane.py:287-345,991-1064,1289-1313,
 * 1388-1440, /root/reference/dit/dit_decoder.py:15-42 and /root/reference/nsr/srt/layers.py:82-90,146-186. */
/* out_bf16[r] = LayerNorm(x[r]) [* w + bias] [* (1 + scale[b]) + shift[b]], b = r / rows_per_batch (1 = per token);
 * D % 4 == 0, D <= 1024 */
int ga_layernorm_modulate(const float *x, const float *w, const float *bias, const float *shift, const float *scale,
                          int mod_ld, int rows_per_batch, void *out_bf16, int R, int D, float eps, void *stream);
/* y[r, c] = bias[c] + sum_d f(x[r])[d] W[c, d], f = optional LayerNorm (ln_w, ln_b) then optional SiLU; C <= 16 */
int ga_thin_linear(const float *x, const float *ln_w, const float *ln_b, int apply_silu, const float *W,
                   const float *bias, float *y, int R, int D, int C, float eps, void *stream);
/* attention over S sequences of L <= 16 tokens: qkv bf16 [S*L, 3*H*64] ("(K H D)" columns), q/k RMS-normalised per
 * head with weights qn_w / kn_w [64], softmax(q k^T / 8) v -> out bf16 [S*L, H*64] */
int ga_micro_attention_bf16(const void *qkv, const float *qn_w, const float *kn_w, void *out, int S, int L, int H,
                            float eps, void *stream);
/* seq [S, 1+f, D] fp32: row 0 = the parent token (prev_f == 0: parents[s]; else child s % prev_f of sequence
 * s / prev_f of the previous stage's [S/prev_f, 1+prev_f, D] buffer), rows 1..f = queries [f, D] */
int ga_micro_seq_build(const float *parents, int prev_f, const float *queries, float *seq, int64_t S, int f, int D,
                       void *stream);
/* child r of parent r / f: res row = r, or (res_in_sequences) row (r/f)(1+f) + 1 + r%f of the [R/f, 1+f] sequence
 * layout; pre = res[row] + parent_pre[r/f] (parent_pre NULL at the base level); xyz = tanh(res[row][0:3])
 * * offset_scale + parent_pos[(r/f) * parent_pos_stride + 0..2]; other channels from pre: sigmoid | softplus *
 * scale_factor | normalise | 0.5 tanh + 0.5.  out_gauss13 [R,13] is rasteriser input; out_pre [R,13] feeds the next level */
int ga_surfel_cascade_pack(const float *res, int res_in_sequences, const float *parent_pre, const float *parent_pos,
                           int parent_pos_stride,
                           int f, float offset_scale, float scale_factor, float *out_gauss13, float *out_pre,
                           int64_t R, void *stream);
int ga_silu_to_bf16(const float *x, void *y, int64_t n, void *stream);            /* y = bf16(silu(x)) */

/*
 * ---------------------------------------------------------------------------
 * Part 3: image conditioner (DINOv2 ViT-L/14 with 4 registers, SURVEY 8f row N3).
 * Replaces FrozenDinov2ImageEmbedder.preprocess (kornia resize + normalise,
 * /root/reference/sgm/modules/encoders/modules.py:862-875) and the token
 * preparation in front of the ViT blocks.  The blocks themselves run on the
 * Part 2 entry points (ga_layernorm_modulate, ga_gemm_bf16_tn,
 * ga_attention_bf16) and the final norm on ga_layernorm_rows.
 * ---------------------------------------------------------------------------
 */
/* Bytes of fp32 scratch ga_dino_frontend needs: 0 unless the image is downscaled (H or W > out_size), when the
 * antialias blur writes two [batch, 3, H, W] planes. */
size_t ga_dino_frontend_scratch_bytes(int batch, int H, int W, int out_size);
/* img fp32 [batch, 3, H, W] in [-1, 1] -> (blur if downscaling) -> bicubic align_corners=True resize to
 * out_size^2 (skipped when H == W == out_size) -> (x + 1) / 2 -> (x - ImageNet mean) / std -> patches_bf16
 * [batch * np * np, k_pitch], np = out_size / patch, column c*patch^2 + ky*patch + kx (conv weight
 * reshape(D, 3*patch^2)), columns from 3*patch^2 on zero.  out_size % patch == 0, k_pitch >= 3*patch^2 and a
 * multiple of 8; H, W, out_size <= 4096 (GA_ERR_SIZE above). */
int ga_dino_frontend(const float *img, int batch, int H, int W, int out_size, int patch, void *patches_bf16,
                     int k_pitch, void *scratch, size_t scratch_bytes, void *stream);
/* x fp32 [batch, 1 + n_reg + n_patch, D] = cls_token + pos_embed[0] | reg_tokens [n_reg, D] (no pos_embed) |
 * patch_out [batch * n_patch, D] + pos_embed[1 ..] ; pos_embed [1 + n_patch, D], D % 4 == 0 */
int ga_dino_tokens(const float *patch_out, const float *cls_token, const float *reg_tokens, int n_reg,
                   const float *pos_embed, float *x, int batch, int n_patch, int D, void *stream);

/*
 * ---------------------------------------------------------------------------
 * Part 4: mesh extraction (TSDF fusion of rendered RGB-D views, marching cubes, cluster filtering; SURVEY 8f row
 * N4).  Replaces Open3D's ScalableTSDFVolume integrate / extract_triangle_mesh and TriangleMesh
 * cluster_connected_triangles / remove_* as FlowMatchingEngine.extract_mesh_bounded and utils/mesh_util.post_process_mesh
 * call them (nsr/lsgm/flow_matching_trainer.py:1244-1395, utils/mesh_util.py:22-44).
 *
 * The volume is made of units of 16^3 voxels.  Units are addressed inside a box of nx*ny*nz units whose first unit
 * is (x0, y0, z0): box is int32[6] = {x0, y0, z0, nx, ny, nz} (device).  A unit's box index is
 * (ux * ny + uy) * nz + uz; a voxel's index inside its unit is (x * 16 + y) * 16 + z.
 * volume is double[2] = {voxel_length, sdf_trunc} (device).
 * Counts come back in status int32[GA_MESH_STATUS_INTS] (device); each entry point below writes only its own
 * words.  status_host (pinned, GA_MESH_STATUS_INTS ints) and status_event (a cudaEvent_t) are both NULL or both
 * set; when set, the entry point copies all the status words there after its counts are final and records the
 * event.  work: scratch of ga_mesh_work_bytes(n) bytes, n as stated at each entry point.
 * ---------------------------------------------------------------------------
 */
#define GA_MESH_UNIT 16
#define GA_MESH_CAM_FLOATS 20     /* per view, float and double: row-major 4x4 | fx fy cx cy */
#define GA_MESH_STATUS_INTS 8     /* [0] units [1] point outside the box [2] vertices [3] triangles [4] clusters
                                     [5] kept vertices [6] kept triangles */
#define GA_MESH_TRI_ROW 16        /* int8 per marching-cubes case: edge triples, then -1 */

/* Bytes of the `work` scratch for n items. Host-only. */
size_t ga_mesh_work_bytes(int64_t n);
/* rgb [V,3,H,W], depth [V,H,W], alpha [V,H,W] fp32 -> texels uint2 [V,H,W] = {depth bits, r | g << 8 | b << 16}:
 * depth = 0 where alpha < alpha_thres or (double)depth >= depth_trunc[v] (double [V]); channel = uint8(clip(c,0,1)*255),
 * truncated. */
int ga_mesh_prepare(const float *rgb, const float *depth, const float *alpha, int views, int H, int W,
                    const double *depth_trunc, float alpha_thres, void *texels, void *stream);
/* Marks the units within sdf_trunc of every 4th pixel (rows and columns) with depth > 0, unprojected with
 * cams_d[v] = {camera-to-world 4x4, fx fy cx cy} (double [V][20]): unit_table int32 [nx*ny*nz][(V+31)/32] gets bit v.
 * A point whose units leave the box sets status[1] and marks nothing.  Then pool int32 [nx*ny*nz] lists the marked
 * box indices in increasing order, unit_slot int32 [nx*ny*nz] maps a box index to its pool position or -1, and
 * status[0] = number of marked units.  work: n = nx*ny*nz. */
int ga_mesh_touch(const void *texels, int views, int H, int W, const double *cams_d, const double *volume,
                  const int32_t *box, int box_units, int32_t *unit_table, int32_t *pool, int32_t *unit_slot,
                  void *work, int32_t *status, int32_t *status_host, void *status_event, void *stream);
/* TSDF integration of views 0..V-1, in order, into the n_units pooled units, each view only into the units it marked.
 * cams_f[v] = {world-to-camera 4x4, fx fy cx cy} (float [V][20]); V <= 256.  voxels float [5][n_units * 4096]
 * = tsdf | weight | r | g | b (r, g, b in 0..255) is overwritten. */
int ga_mesh_integrate(const void *texels, int views, int H, int W, const float *cams_f, const double *volume,
                      const int32_t *box, const int32_t *unit_table, const int32_t *pool, int n_units,
                      float *voxels, void *stream);
/* Marching cubes, counting pass.  cube uint8 [2][n_units * 4096]: case index of the cube at each voxel (0 when a
 * corner's unit is missing or its weight is 0) | which of the voxel's +x, +y, +z edges carry a vertex (bits 0-2).
 * vert_off / tri_off int32 [n_units * 4096]: exclusive offsets of each voxel's vertices / triangles; status[2],
 * status[3] = totals.  tri_table int8 [256][GA_MESH_TRI_ROW].  work: n = n_units * 4096. */
int ga_mesh_cubes_count(const float *voxels, int n_units, const int32_t *pool, const int32_t *unit_slot,
                        const int32_t *box, const int8_t *tri_table, uint8_t *cube, int32_t *vert_off,
                        int32_t *tri_off, void *work, int32_t *status, int32_t *status_host, void *status_event,
                        void *stream);
/* Marching cubes, emitting pass: vertices / colors double [status[2]][3] (colour in [0,1]), triangles int32
 * [status[3]][3], in pool order, then voxel order, then x, y, z edge / table order. */
int ga_mesh_cubes_emit(const float *voxels, int n_units, const int32_t *pool, const int32_t *unit_slot,
                       const int32_t *box, const double *volume, const int8_t *tri_table, const uint8_t *cube,
                       const int32_t *vert_off, const int32_t *tri_off, double *vertices, double *colors,
                       int32_t *triangles, void *stream);
/* Connected components of triangles that share an edge (vertex pair).  hash: hash_slots * 12 bytes, hash_slots a
 * power of two >= 6 * n_tri.  label int32 [n_tri] = cluster of each triangle, clusters numbered by their smallest
 * triangle; cluster_size int32 [n_tri], first status[4] entries valid.  work: n = n_tri. */
int ga_mesh_clusters(const int32_t *triangles, int n_tri, void *hash, int64_t hash_slots, int32_t *label,
                     int32_t *cluster_size, void *work, int32_t *status, int32_t *status_host, void *status_event,
                     void *stream);
/* Keeps the triangles whose cluster has >= min_size triangles, then the vertices they reference (in order), then
 * drops the kept triangles with a repeated vertex.  out_* sized like the inputs; status[5], status[6] = kept
 * vertices, kept triangles.  work: n = n_vert + n_tri. */
int ga_mesh_filter(const double *vertices, const double *colors, int n_vert, const int32_t *triangles, int n_tri,
                   const int32_t *label, const int32_t *cluster_size, int min_size, double *out_vertices,
                   double *out_colors, int32_t *out_triangles, void *work, int32_t *status, int32_t *status_host,
                   void *status_event, void *stream);

/*
 * ---------------------------------------------------------------------------
 * Part 5: 3D VAE encoder (HybridEncoderPCDStructuredLatentSNoPCD, /root/reference/nsr/srt/encoder.py:454-652, and the
 * posterior of /root/reference/vit/vit_triplane.py:1347-1385).  Replaces the cuDNN 3x3 convolutions and GroupNorm
 * of the SD conv encoder (ldm/modules/diffusionmodules/model.py:81-162,469-572), pytorch3d's
 * sample_farthest_points + masked_gather, the per-head RMSNorm(32) of the SRT blocks and the readout MLPs.  The 1x1
 * convolutions, linears and attentions of the encoder run on the Part 2 entry points (GEGLU via GA_EPI_GEGLU_BF16,
 * the SRT's head_dim 32 zero-padded to 64 by ga_heads32_split).  Activations are NHWC.
 * ---------------------------------------------------------------------------
 */
/* Output height (or width) of ga_conv3x3_bf16 for an input of H: H for stride 1, (H - 2) / 2 + 1 for stride 2.
 * Host-only. */
int ga_conv3x3_out_size(int H, int stride);
/* 3x3 convolution as an implicit GEMM (wgmma, bf16 operands, fp32 accumulation).  x bf16 NHWC [n, H, W, Cin],
 * Cin % 8 == 0; w_packed bf16 [Cout, k_pitch], column (ky * 3 + kx) * Cin + c, zero beyond 9 * Cin, k_pitch >=
 * 9 * Cin rounded up to 64; Cout % 64 == 0.  stride 1: pad 1 on every side; stride 2: pad (0, 1, 0, 1) (the SD
 * Downsample).  out[m, :] = bias + conv (+ residual[m, :], fp32), m = (image, oy, ox) over [n, Ho, Wo]; written to
 * out_f32 and / or out_bf16 (either may be NULL, not both). */
int ga_conv3x3_bf16(const void *x, int n, int H, int W, int Cin, const void *w_packed, int k_pitch,
                    const float *bias, int Cout, int stride, const float *residual, float *out_f32,
                    void *out_bf16, void *stream);
/* Bytes of scratch ga_group_norm_nhwc needs for n images of HW pixels.  Host-only. */
size_t ga_group_norm_scratch_bytes(int n, int HW);
/* GroupNorm(32 groups) over x fp32 NHWC [n, HW, C] (statistics per image and group, fp32 partial sums folded in
 * fp64), * gamma + beta, then SiLU if silu != 0; out bf16 (out_bf16 != 0) or fp32, same layout.  C % 32 == 0,
 * C <= 1024.  Deterministic. */
int ga_group_norm_nhwc(const float *x, const float *gamma, const float *beta, int n, int HW, int C, float eps,
                       int silu, void *out, int out_bf16, void *scratch, size_t scratch_bytes, void *stream);
/* Farthest-point sampling, one CTA per sample: pcd fp32 [batch, N, 3], N <= 16384, K <= min(N, 1024).  Point 0 is
 * start_idx[b]; point k is the one with the largest distance to the points already chosen, distances fp32
 * (dx*dx + dy*dy) + dz*dz with each operation rounded on its own, ties to the lowest index.  idx_out int32
 * [batch, K], xyz_out fp32 [batch, K, 3] (the gathered points). */
int ga_fps(const float *pcd, int batch, int N, int K, const int32_t *start_idx, int32_t *idx_out,
           float *xyz_out, void *stream);
/* img fp32 NCHW [n, C, H, W] -> x_bf16 NHWC [n, H, W, c_pad] (channels from C on zero; c_pad % 8 == 0), and, when
 * token_xyz is not NULL, token_xyz fp32 ["(n ty tx)", 3] = img[:, xyz_c:xyz_c+3, off::step, off::step]. */
int ga_vae_enc_input(const float *img, int n, int C, int H, int W, int c_pad, void *x_bf16, int xyz_c,
                     int step, int off, float *token_xyz, void *stream);
/* Head split for head_dim 32: qkv bf16 [R, 3 * heads * 32] ("(K H D)" columns, bias included) -> q, k per-head
 * RMSNorm(32) (fp32, * qn_w / kn_w [32]; NULL = no norm), written zero-padded to 64 as Q, K [B, heads, tok_pitch, 64]
 * and Vt [B, heads, 64, tok_pitch] (rows 32..63 zero), B = R / rows_per_batch: the ga_attention_bf16 layout. */
int ga_heads32_split(const void *qkv, const float *qn_w, const float *kn_w, int R, int heads,
                     int rows_per_batch, int tok_pitch, float eps, void *q, void *k, void *vt, void *stream);
/* Weights of the readout head (all fp32, nn.Linear layout [out, in]). */
typedef struct GaVaeEncHead {
    const float *ln_w, *ln_b;       /* Mlp_out PreNorm LayerNorm [D] */
    const float *fc1_w, *fc1_b;     /* [hid, D], [hid] */
    const float *fc2_w, *fc2_b;     /* [2 zc, hid], [2 zc] */
    const float *q1_w, *q1_b;       /* quant_conv fc1 [2 zc, 2 zc], [2 zc] */
    const float *q2_w, *q2_b;       /* quant_conv fc2 [2 zc, 2 zc], [2 zc] */
    float ln_eps;
} GaVaeEncHead;
/* Per token r of x fp32 [R, D]: h = fc2(gelu_tanh(fc1(LayerNorm(x)))) -> h_out [R, 2 zc]; moments =
 * q2(gelu_tanh(q1(h))); mean = moments[:zc], logvar = 20 tanh(moments[zc:] / 20), std = exp(logvar / 2) (stdv may
 * be NULL), latent = mean + std * noise (noise fp32 [R, zc]; NULL gives latent = mean; latent may be NULL). */
int ga_vae_enc_head(const GaVaeEncHead *p, const float *x, const float *noise, int R, int D, int hid, int zc,
                    float *h_out, float *mean, float *logvar, float *stdv, float *latent, void *stream);

/* Measurement aid: when enabled, cudaEvents are recorded around every kernel
 * stage of the next forward/backward; ga_profile_read synchronises on them and
 * returns per-stage milliseconds: [0] preprocess, [1] binning, [2] render fwd,
 * [3] render bwd (+accumulator memset), [4] per-surfel bwd.  Returns the number
 * of stages written (0 if profiling never ran). */
int ga_profile_enable(int on);
int ga_profile_read(float *ms, int n);

/* Library self-description (host only). */
const char *ga_b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* GA_B200_H */
