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
#define GA_RASTER_GRAD_FLOATS 18  /* per (view, surfel): sizes the backward's scratch, see ga_raster_backward_scratch_bytes */
#define GA_RASTER_ROW_FLOATS 16   /* per (batch item, surfel): the backward's gradient row, summed over the views */

/* Byte offsets of the sections inside the forward workspace.  The forward
 * pass fills them; the backward pass reads them (the workspace is the
 * equivalent of upstream's geomBuffer/binningBuffer/imgBuffer). */
typedef struct GaRasterLayout {
    size_t total_bytes;
    size_t status;      /* int32[16]: [0]=instances D, [1]=overflow flag, [2]=tiles above 4096 instances (sorted in global memory), [3]=tiles above 512 */
    size_t rec;         /* float[NV*P][24]  Tu3 Tv3 Tw3 | xy2 opacity | normal3 | r | bbox x0 x1 y0 y1 | g b sign - */
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

/* Bytes of scratch the backward wants: NV*P*GA_RASTER_GRAD_FLOATS floats.  Only the leading
 * batch*P*GA_RASTER_ROW_FLOATS floats are used (zeroed, then summed into); a larger buffer is accepted and the rest
 * of it is not touched. */
size_t ga_raster_backward_scratch_bytes(int batch, int P, int views);

/*
 * Backward.  dL_dcolor [NV][3][H][W], dL_dallmap [NV][7][H][W]; grad_gauss13
 * [batch][P][13] is OVERWRITTEN with the gradient summed over the views of
 * each batch item (same column order as gauss13).  workspace and list_k must
 * be the ones the matching ga_raster_forward_ex filled and used.  scratch must
 * be 16-byte aligned.  radii is the forward's out_radii; it must not be NULL,
 * but the gradient does not depend on it.
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
    void *out;                /* modes 0-3, 5 */
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
 * lda, ldw multiples of 8.  Arguments are checked by ga_gemm_validate before anything is launched. */
int ga_gemm_bf16_tn(const void *A, int lda, const void *W, int ldw, int M, int N, int K,
                    const GaGemmEpilogue *epi, int block_n, void *stream);
/* Host only, no CUDA call: 0 when ga_gemm_bf16_tn accepts the arguments, else GA_ERR_BADARG.  The rules:
 *   A, W, epi non-NULL; M, N, K > 0; A and W 16-byte aligned; lda, ldw multiples of 8 and >= K;
 *   block_n in {64, 128, 192, 256}; mode in 0..5;
 *   modes 0-3, 5: out non-NULL; ld_out >= N (N / 2 for GEGLU, where N is even); out aligned to 16 bytes (modes 2, 3),
 *     8 bytes (modes 0, 1) or 4 bytes (mode 5);
 *   mode 3 with a gate: rows_per_batch >= 1 and gate_ld >= N (a NULL gate reads neither);
 *   mode 4: block_n 128 or 256; heads >= 1; N a multiple of 64 * heads; first_part 0 or 1 and first_part +
 *     N / (64 * heads) <= 3; q, k, vt non-NULL and 16-byte aligned for each part the columns reach (q for part 0,
 *     k for 1, vt for 2); rows_per_batch >= 1 and tok_pitch >= rows_per_batch. */
int ga_gemm_validate(const void *A, int lda, const void *W, int ldw, int M, int N, int K,
                     const GaGemmEpilogue *epi, int block_n);

/* softmax(Q K^T * softmax_scale) V, head_dim 64.  Q [B*H, pitch_q, 64], K [B*H, pitch_k, 64],
 * Vt [B*H, 64, pitch_k] (bf16, padding beyond Nk must be finite); out [B, Nq, H*64] bf16.
 * pitch_k must be a multiple of 128. */
int ga_attention_bf16(const void *Q, const void *K, const void *Vt, void *out, int batch, int heads,
                      int Nq, int Nk, int pitch_q, int pitch_k, float softmax_scale, float score_bound,
                      void *stream);
/* score_bound: an upper bound of |q.k| * softmax_scale over all (q, k) pairs, or <= 0 if unknown.  With
 * RMS-normalised q and k (the DiT's qk-norm) it is 64 * max|w_q| * max|w_k| * softmax_scale; when given
 * (and <= 40) the kernel uses it instead of a running row maximum (same result, one pass over the scores). */
/* Causal ga_attention_bf16 (same arguments and layouts, Nq == Nk): query i attends to keys 0..i only.  Row i's
 * output does not depend on K or V of any key above i (the CLIP text tower's attn_mask). */
int ga_attention_causal_bf16(const void *Q, const void *K, const void *Vt, void *out, int batch, int heads,
                             int Nq, int Nk, int pitch_q, int pitch_k, float softmax_scale, float score_bound,
                             void *stream);
/* Host only, no CUDA call: the argument check both attention entry points make first (causal != 0 for the causal
 * one).  GA_ERR_BADARG unless Q, K, Vt, out are non-NULL; batch, heads, Nq, Nk > 0; pitch_q >= Nq; pitch_k >= Nk and
 * a multiple of 128; Nq == Nk when causal; Q, K, Vt 16-byte and out 4-byte aligned.  GA_ERR_SIZE when
 * batch * heads > 65535 (one grid row per (batch, head)).  0 otherwise. */
int ga_attention_validate(const void *Q, const void *K, const void *Vt, const void *out, int batch, int heads,
                          int Nq, int Nk, int pitch_q, int pitch_k, int causal);

/* out_bf16[r,:] = RMSNorm(x[r,:]; eps) * w [* (1 + scale[b,:]) + shift[b,:]], b = r / rows_per_batch;
 * shift/scale both NULL or both set, rows mod_ld apart (mod_ld % 4 == 0).  D % 4 == 0; x, w, shift, scale 16-byte
 * and out_bf16 8-byte aligned (GA_ERR_BADARG otherwise). */
int ga_rmsnorm_modulate(const float *x, const float *w, const float *shift, const float *scale,
                        int mod_ld, int rows_per_batch, void *out_bf16, int R, int D, float eps, void *stream);

/* y[b,n] (+)= act_out(bias[n] + sum_k act_in(x[b,k]) W[n,k]);  rows <= 16; act: 0 none, 1 SiLU (other codes
 * GA_ERR_BADARG).  SiLU is applied to the sum, then y's old value added.  When K % 128 == 0 and K <= 1024, x and W
 * must be 16-byte aligned. */
int ga_linear_small(const float *x, const float *W, const float *bias, float *y, int rows, int N, int K,
                    int act_in, int act_out, int accumulate, void *stream);
/* out[r] = [cos(t[r] f_i) | sin(t[r] f_i)], f_i = exp(-ln(1e4) i / (dim / 2)), i < dim / 2; dim even, <= 2048 */
int ga_timestep_sinusoid(const float *t, float *out, int rows, int dim, void *stream);
/* y[r] = LayerNorm(x[r]; eps) [* w [+ b]], fp32; b needs w.  When D % 4 == 0 and D <= 1024, x, w, b and y must be
 * 16-byte aligned. */
int ga_layernorm_rows(const float *x, const float *w, const float *b, float *y, int R, int D, float eps, void *stream);
/* mod[l,b,e] = tables[l,e] + t0[b, e % t0_ld], e in [0, JD) */
int ga_add_tables(const float *tables, const float *t0, float *mod, int L, int rows, int JD, int t0_ld, void *stream);
/* h = gelu_tanh(W1 [xin2 | xin] + b1) -> bf16 [R, D] (token embedder, first layer); Cx > 0, C2 >= 0 */
int ga_embed_fc1(const float *xin, int Cx, const float *xin2, int C2, const float *W1, const float *b1,
                 void *h_bf16, int R, int D, void *stream);
/* NeRF positional encoding of xyz (63 features, padded to 64) -> bf16 [R, 64] */
int ga_xyz_posenc(const float *xyz, void *out_bf16, int R, void *stream);
/* y[r,c] = bias[c] + sum_d (LayerNorm(x[r])[d] (1 + scale[b,d]) + shift[b,d]) W[c,d]; mod [B,2,D]; Cout <= 16;
 * b = r / rows_per_batch, rows_per_batch > 0.  When D % 4 == 0 and D <= 1024, x, mod and W must be 16-byte aligned. */
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
 * D % 4 == 0, D <= 1024; bias needs w; mod_ld % 4 == 0.  x, w, bias, shift, scale 16-byte and out_bf16 8-byte
 * aligned. */
int ga_layernorm_modulate(const float *x, const float *w, const float *bias, const float *shift, const float *scale,
                          int mod_ld, int rows_per_batch, void *out_bf16, int R, int D, float eps, void *stream);
/* y[r, c] = bias[c] + sum_d f(x[r])[d] W[c, d], f = optional LayerNorm (ln_w, ln_b) then optional SiLU; C <= 16;
 * D % 4 == 0, D <= 1024; x, ln_w, ln_b, W 16-byte aligned */
int ga_thin_linear(const float *x, const float *ln_w, const float *ln_b, int apply_silu, const float *W,
                   const float *bias, float *y, int R, int D, int C, float eps, void *stream);
/* attention over S sequences of L <= 16 tokens: qkv bf16 [S*L, 3*H*64] ("(K H D)" columns), q/k RMS-normalised per
 * head with weights qn_w / kn_w [64], softmax(q k^T / 8) v -> out bf16 [S*L, H*64].  qkv and out 4-byte, qn_w and
 * kn_w 8-byte aligned. */
int ga_micro_attention_bf16(const void *qkv, const float *qn_w, const float *kn_w, void *out, int S, int L, int H,
                            float eps, void *stream);
/* seq [S, 1+f, D] fp32: row 0 = the parent token (prev_f == 0: parents[s]; else child s % prev_f of sequence
 * s / prev_f of the previous stage's [S/prev_f, 1+prev_f, D] buffer), rows 1..f = queries [f, D]; D % 4 == 0,
 * D <= 1024; parents, queries, seq 16-byte aligned */
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
 * patch_out [batch * n_patch, D] + pos_embed[1 ..] ; pos_embed [1 + n_patch, D], D % 4 == 0; every pointer 16-byte
 * aligned */
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
 * out_f32 and / or out_bf16 (either may be NULL, not both).  x and w_packed 16-byte, residual and out_f32 8-byte
 * (float2), out_bf16 4-byte (__nv_bfloat162) aligned. */
int ga_conv3x3_bf16(const void *x, int n, int H, int W, int Cin, const void *w_packed, int k_pitch,
                    const float *bias, int Cout, int stride, const float *residual, float *out_f32,
                    void *out_bf16, void *stream);
/* Bytes of scratch ga_group_norm_nhwc needs for n images of HW pixels.  Host-only. */
size_t ga_group_norm_scratch_bytes(int n, int HW);
/* GroupNorm(32 groups) over x fp32 NHWC [n, HW, C] (statistics per image and group: per pixel chunk, fp32 sums of
 * the values less the chunk's first pixel, formed into the chunk's (mean, M2) in fp64 and merged in fp64, so a
 * group's |mean| / std costs no precision), * gamma + beta, then SiLU if silu != 0; out bf16 (out_bf16 != 0) or
 * fp32, same layout.  0 < C <= 1024, C % 32 == 0.  x 16-byte aligned; out 16-byte (fp32) or 8-byte (bf16) aligned.
 * Deterministic. */
int ga_group_norm_nhwc(const float *x, const float *gamma, const float *beta, int n, int HW, int C, float eps,
                       int silu, void *out, int out_bf16, void *scratch, size_t scratch_bytes, void *stream);
/* Farthest-point sampling, one CTA per sample: pcd fp32 [batch, N, 3], N <= 16384, K <= min(N, 1024).  Point 0 is
 * start_idx[b]; point k is the one with the largest distance to the points already chosen, distances fp32
 * (dx*dx + dy*dy) + dz*dz with each operation rounded on its own, ties to the lowest index.  idx_out int32
 * [batch, K], xyz_out fp32 [batch, K, 3] (the gathered points). */
int ga_fps(const float *pcd, int batch, int N, int K, const int32_t *start_idx, int32_t *idx_out,
           float *xyz_out, void *stream);
/* img fp32 NCHW [n, C, H, W] -> x_bf16 NHWC [n, H, W, c_pad] (channels from C on zero; c_pad % 8 == 0), and, when
 * token_xyz is not NULL, token_xyz fp32 ["(n ty tx)", 3] = img[:, xyz_c:xyz_c+3, off::step, off::step].  x_bf16
 * 4-byte aligned.  Every argument, token_xyz's included, is checked before anything is written. */
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
 * be NULL), latent = mean + std * noise (noise fp32 [R, zc]; NULL gives latent = mean; latent may be NULL).
 * GA_ERR_SIZE when (D + hid + 6 zc) * 4 bytes of shared memory, plus the kernel's 32 static bytes, exceed 48 KiB. */
int ga_vae_enc_head(const GaVaeEncHead *p, const float *x, const float *noise, int R, int D, int hid, int zc,
                    float *h_out, float *mean, float *logvar, float *stdv, float *latent, void *stream);

/*
 * ---------------------------------------------------------------------------
 * Part 6: text conditioner (OpenCLIP ViT-L/14 text tower, the reference's FrozenOpenCLIPEmbedder2,
 * /root/reference/sgm/modules/encoders/modules.py:416-512).  The residual blocks run on the Part 2 entry points
 * (ga_layernorm_modulate, ga_gemm_bf16_tn, ga_attention_causal_bf16) plus ga_quick_gelu_bf16 after c_fc; ln_final
 * on ga_layernorm_rows and the text projection on ga_linear_small.
 * ---------------------------------------------------------------------------
 */
/* x fp32 [batch * ctx_len, D] = token_embedding[ids[r]] (fp32 [vocab, D]) + positional_embedding[r % ctx_len]
 * (fp32 [ctx_len, D]); ids int32 [batch, ctx_len].  The caller rejects ids outside [0, vocab); such a row is
 * written as NaN. */
int ga_clip_text_embed(const int32_t *ids, const float *token_embedding, const float *positional_embedding,
                       float *x, int batch, int ctx_len, int D, int vocab, void *stream);
/* out fp32 [batch, D] = x[b * ctx_len + p_b], p_b = the first position of the largest id of row b (the end-of-text
 * token, open_clip's text.argmax(dim=-1)). */
int ga_clip_text_eot_gather(const int32_t *ids, const float *x, float *out, int batch, int ctx_len, int D,
                            void *stream);
/* In place on bf16 x [n]: x = x * sigmoid(1.702 x) (QuickGELU, computed in fp32). */
int ga_quick_gelu_bf16(void *x, int64_t n, void *stream);

/*
 * ---------------------------------------------------------------------------
 * Part 7: 3D VAE reconstruction from G-buffer chunk folders (the reference's vae-3d.sh input:
 * datasets/g_buffer_objaverse.py read_chunk :3225-3302 and PostProcess._post_process_sample_batch :481-702, at
 * reso == reso_encoder == the files' size, frame_0_as_canonical=False, append_xyz, plucker_embedding, read_normal).
 * Both kernels are compiled without FMA contraction: every operation below is rounded to fp32 on its own, in the
 * order written.
 * ---------------------------------------------------------------------------
 */
/* One launch, one thread per four pixels of a row (16-byte stores).  Inputs as the chunk's files decode, the n_chunk
 * views side by side: raw_img, normal uint8 [H, n_chunk * W, 3], alpha uint8 [H, n_chunk * W] (may be NULL without
 * targets), depth fp32 [n_chunk, H, W], cams fp32 [n_chunk, 25] (c2w row-major 16 | K 9, normalised by the image
 * size), views int32 [n_views] in [0, n_chunk) (the caller checks the range).  W % 4 == 0, W <= 1024.
 * img_to_encoder fp32 [n_views, 15, H, W], row s from view views[s]:
 *   0-2   (rgb / 255 - mean) / std, mean = (0.485, 0.456, 0.406), std = (0.229, 0.224, 0.225): the ImageNet
 *         Normalize of PostProcess.__init__ (:156-160); load_eval_data's chunk branch leaves imgnet_normalize=True
 *   3-5   n = (u8 / 255) * 2 - 1, then (-n.x, -n.z, n.y) (unity2blender_fix)
 *   6-11  cross(o, d), d: o = c2w[:3, 3]; d = c2w[:3, :3] g, g = (gx, gy, 1) / sqrt(gx gx + gy gy + 1),
 *         gx = ((x + 0.5) / W - cx) / fx, gy = ((y + 0.5) / H - cy) / fy  (gen_rays; sums left to right)
 *   12-14 p = o + depth * r, r = q / max(|q|, 1e-12), q = (c2w (lx, ly, 1, 1))[:3] - o,
 *         lx = (u - cx + cy sk / fy - sk v / fy) / fx, ly = (v - cy) / fy, u = (x + 0.5) / W, v = (y + 0.5) / H
 *         (RaySampler); p clipped to [-0.45, 0.45], then 0 where |p| == 0.45.  A background pixel (depth 0) gives
 *         p = o: removed only where the camera origin's coordinate is outside the clip, as in the reference.
 * Targets, all four or none: t_img fp32 [n_views, 3, H, W] = (rgb / 255) * 2 - 1; t_alpha [n_views, 1, H, W] =
 * alpha / 255; t_depth [n_views, 1, H, W] = depth; t_mask [n_views, 1, H, W] = depth > 0 as 1.0 / 0.0. */
int ga_gbuffer_pack(const uint8_t *raw_img, const uint8_t *normal, const uint8_t *alpha, const float *depth,
                    const float *cams, int n_chunk, int H, int W, const int32_t *views, int n_views,
                    float *img_to_encoder, float *t_img, float *t_alpha, float *t_depth, float *t_mask,
                    void *stream);
/* Blocks per view of the first stage of ga_recon_metrics: partial is fp32 [n_views, GA_RECON_METRICS_BLOCKS, 8]. */
#define GA_RECON_METRICS_BLOCKS 64
/* Per-view sums over the H * W pixels of rendered maps against targets, table fp32 [n_views, 8]:
 *   [0] sum over 3 channels of (image - (t_img + 1) / 2)^2      image in [0, 1], t_img in [-1, 1]
 *   [1] sum of t_mask * |depth - t_depth|                        [2] sum of t_mask
 *   [3] sum of t_mask * (1 - <rend_normal, t_normal>)            (nsr/train_nv_util.py:2162 on the foreground)
 *   [4] sum of |alpha - t_alpha|
 *   [5], [6] pixels where alpha > 0.5 and / or t_alpha > 0.5     [7] H * W
 * image, rend_normal, t_img fp32 [n_views, 3, H, W]; depth, alpha, t_depth, t_alpha, t_mask [n_views, 1, H, W];
 * t_normal fp32, view v at t_normal + v * t_normal_stride, [3, H, W] (channels 3-5 of img_to_encoder with stride
 * 15 H W).  H * W <= 2^24, so the counts are exact.  Two stages in a fixed order (per-block partial sums, then one
 * block per view adds them in block order), no atomics: the same inputs give the same bits. */
int ga_recon_metrics(const float *image, const float *depth, const float *alpha, const float *rend_normal,
                     const float *t_img, const float *t_depth, const float *t_alpha, const float *t_mask,
                     const float *t_normal, int64_t t_normal_stride, int n_views, int H, int W, float *partial,
                     float *table, void *stream);

/*
 * ---------------------------------------------------------------------------
 * Part 8: image-quality metrics.  LPIPS with the VGG16 backbone (the network and formulas of the reference's
 * sgm/modules/autoencoding/lpips/loss/lpips.py, i.e. lpips.LPIPS(net="vgg", version="0.1") as nsr/losses/builder.py
 * uses it) and SSIM (_ssim of nsr/losses/builder.py:23-55, size_average=False).  Inference only.
 * LPIPS: ga_lpips_pack, then VGG16's 13 convolutions on ga_conv3x3_relu_bf16 (bf16 operands and activations, fp32
 * accumulation) with ga_maxpool2x2_bf16 between the stages, ga_lpips_head on each of the five taps (relu1_2,
 * relu2_2, relu3_3, relu4_3, relu5_3), then ga_lpips_reduce.  The head and the reduction run in fp32, SSIM's
 * window sums in fp64.
 * This file's kernels (lpips_ops.cu) are compiled without FMA contraction: every operation below is rounded to fp32 on
 * its own, in the order written.
 * ---------------------------------------------------------------------------
 */
/* ga_conv3x3_bf16 at stride 1 with no residual and a ReLU epilogue: out_bf16[m, :] = bf16(max(bias + conv, 0)),
 * fp32 up to the final rounding.  Same arguments and checks as ga_conv3x3_bf16 (bias may be NULL; out_bf16 4-byte
 * aligned). */
int ga_conv3x3_relu_bf16(const void *x, int n, int H, int W, int Cin, const void *w_packed, int k_pitch,
                         const float *bias, int Cout, void *out_bf16, void *stream);
/* The two images of n pairs, in0 and in1 fp32 NCHW [n, 3, H, W] each -> out bf16 NHWC [2n, H, W, 8] (16-byte
 * aligned): images 0..n-1 from in0, n..2n-1 from in1.  Per value x: x = 2 x - 1 when normalize != 0 (the package's
 * normalize=True for [0, 1] input), then bf16((x - shift[c]) / scale[c]) (one fp32 subtraction and one fp32 division;
 * shift, scale fp32 [3], device); channels 3-7 are 0.  The first VGG convolution then runs with Cin 8 (K 72,
 * k_pitch 128) and zero weights for channels 3-7. */
int ga_lpips_pack(const float *in0, const float *in1, int n, int H, int W, int normalize, const float *shift,
                  const float *scale, void *out, void *stream);
/* nn.MaxPool2d(2, 2) on bf16 NHWC: x [n, H, W, C] -> out [n, H / 2, W / 2, C] (floor), the max of each 2x2 window.
 * Bit-exact for finite input.  C % 8 == 0, H, W >= 2, x and out 16-byte aligned. */
int ga_maxpool2x2_bf16(const void *x, int n, int H, int W, int C, void *out, void *stream);
#define GA_LPIPS_TAPS 5
/* Blocks per pair of ga_lpips_head: its partial is fp32 [n, GA_LPIPS_HEAD_BLOCKS] per tap. */
#define GA_LPIPS_HEAD_BLOCKS 128
/* One LPIPS tap: feat bf16 NHWC [2n, H, W, C] (a ReLU output, 16-byte aligned), C in {64, 128, 256, 512};
 * lin_w fp32 [C] (the tap's bias-free 1x1 NetLinLayer).  For pair i at each pixel, f0 = feat[i], f1 = feat[i + n]:
 *   n0 = sqrt(sum_c f0_c * f0_c) + 1e-10,  n1 likewise          (NormalizeTensor, eps 1e-10)
 *   d  = sum_c w_c * (t_c * t_c),  t_c = f0_c / n0 - f1_c / n1
 * Channel sums: each of G = min(32, C / 8) lanes adds its channels in increasing order, then an xor butterfly
 * over the G lanes.  partial[i * GA_LPIPS_HEAD_BLOCKS + b] = sum of d over pixels [b * per, (b + 1) * per) (per =
 * ceil(H W / GA_LPIPS_HEAD_BLOCKS)) in a fixed order that depends on H and W only, so a pair's partials are the
 * same bits whatever n is.  Swapping the two images gives the same bits; equal images give exactly 0.  No atomics. */
int ga_lpips_head(const void *feat, int n, int H, int W, int C, const float *lin_w, float *partial, void *stream);
/* partial fp32 [GA_LPIPS_TAPS, n, GA_LPIPS_HEAD_BLOCKS] (ga_lpips_head's output for tap k at partial + k n
 * GA_LPIPS_HEAD_BLOCKS) -> out fp32 [n, GA_LPIPS_TAPS + 1]: out[i, k] = fp32(the fp64 sum of the tap's partials in
 * block order / ((H >> k) (W >> k))), the tap's spatial mean (H, W: the input size; tap k is (H >> k) x (W >> k));
 * out[i, 5] = (((out[i,0] + out[i,1]) + out[i,2]) + out[i,3]) + out[i,4] in fp32.  H >> 4 and W >> 4 >= 1. */
int ga_lpips_reduce(const float *partial, int n, int H, int W, float *out, void *stream);
#define GA_SSIM_WINDOW 11
/* Bytes of scratch ga_ssim needs.  Host-only. */
size_t ga_ssim_scratch_bytes(int n, int H, int W);
/* SSIM of n image pairs, img1 and img2 fp32 [n, 3, H, W] -> out fp32 [n], the mean of the SSIM map over C, H and W.
 * window fp32 [11, 11] (device): create_window(11, .)'s values, g g^T of the normalised fp32 Gaussian (sigma 1.5),
 * computed by the caller.  The kernel uses this 2D window (not the separable form).  With zero padding of 5, in fp64
 * (the fp32 window and pixels widened; E[x^2] - mu^2 in fp32 would cancel to SSIM errors of ~2e-5):
 *   mu1 = sum w x, mu2 = sum w y, e11 = sum w (x x), e22 = sum w (y y), e12 = sum w (x y)
 *        taps in row-major order, each step one fp64 fma (x x, y y, x y are exact in fp64)
 *   mu1_sq = mu1 mu1, mu2_sq = mu2 mu2, mu1_mu2 = mu1 mu2
 *   s1 = e11 - mu1_sq, s2 = e22 - mu2_sq, s12 = e12 - mu1_mu2
 *   map = fp32(((2 mu1_mu2 + C1) (2 s12 + C2)) / ((mu1_sq + mu2_sq + C1) (s1 + s2 + C2))), C1 = 0.01^2, C2 = 0.03^2
 * The map is summed per 16 x 16 block in fp32 (fixed order), the block sums of an image in fp64, and out =
 * fp32(sum / (3 H W)).  Equal images give exactly 1; the same inputs give the same bits.  n <= 21845. */
int ga_ssim(const float *img1, const float *img2, int n, int H, int W, const float *window, void *scratch,
            size_t scratch_bytes, float *out, void *stream);

/*
 * ---------------------------------------------------------------------------
 * Part 9: LPIPS backward, the input gradients of Part 8's LPIPS (the network is frozen: no weight gradients).  For
 * the per-pair values v_i of the forward and upstream weights g_i (fp32, device; autograd's incoming gradient), the
 * gradient of sum_i g_i v_i with respect to the images of one side: side 0 is in0 (images 0..n-1 of the packed
 * batch), side 1 is in1 (images n..2n-1), each computed only when asked for.  Per side, from the last layer down:
 *   tap 4:  ga_lpips_tap_backward without dpool -> the gradient at conv 12's pre-activation (bf16)
 *   inside a slice: ga_conv3x3_mask_bf16 with the flipped weights of the conv above and the ReLU output of the conv
 *           below as mask -> the gradient at the lower conv's pre-activation (bf16)
 *   the first conv of slices 1-4: ga_conv3x3_bf16 (stride 1, no bias, out_f32) with its flipped weights -> the
 *           gradient at the pooled map (fp32), then ga_lpips_tap_backward of the tap below with that dpool
 *   conv 0: ga_lpips_input_backward -> fp32 NCHW gradients of the images.
 * Flipped weights of a conv with weight W [Co, Ci, 3, 3]: the Part 5 packed layout with Cout = Ci and Cin = Co,
 * W'[ci, (ky * 3 + kx) * Co + co] = bf16(W[co, ci, 2 - ky, 2 - kx]): the dgrad of a stride-1 pad-1 3x3 convolution is
 * the stride-1 pad-1 3x3 convolution with these weights.  Accumulation in fp32; no atomics and no loss scaling (bf16
 * has fp32's exponent range), so the same inputs give the same bits whatever n and the chunking.
 * lpips_grad.cu is compiled without FMA contraction: every operation below is rounded to fp32 on its own, in the
 * order written.  The convolutions follow Part 5 (fp32 accumulation in the wgmma's order).
 * ---------------------------------------------------------------------------
 */
/* ga_conv3x3_bf16 at stride 1 with no bias or residual and a ReLU-mask epilogue: out_bf16[m, c] =
 * bf16(mask[m, c] > 0 ? conv : 0), a select (a non-finite conv value never leaks through a masked zero).  mask bf16
 * [n, H, W, Cout] (4-byte aligned).  Other arguments and checks as ga_conv3x3_bf16. */
int ga_conv3x3_mask_bf16(const void *x, int n, int H, int W, int Cin, const void *w_packed, int k_pitch, int Cout,
                         const void *mask, void *out_bf16, void *stream);
/* One tap's backward for one side.  feat: the tap, bf16 NHWC [2n, H, W, C] as ga_lpips_head reads it (16-byte
 * aligned), C in {64, 128, 256, 512}; lin_w fp32 [C]; g fp32 [n] (device).  For pair i at each pixel, f = feat[side n
 * + i] (this side), f' = feat[(1 - side) n + i] (the other), with the head's channel sums (G lanes, each in increasing
 * channel order, then an xor butterfly):
 *   r = sqrt(sum_c f_c f_c), nf = r + 1e-10, nf' = sqrt(sum_c f'_c f'_c) + 1e-10
 *   t_c = f_c / nf - f'_c / nf',  u_c = 2 (w_c t_c),  S = sum_c u_c f_c,  s = g_i / fp32(H W),  q = (S / nf) / nf
 *   head_c = s (u_c / nf - (f_c / r) q)  where r > 0, else 0 (the reference's normalize_tensor gives NaN at an all-zero
 *            vector, and its ReLU backward, a select, turns that into 0)
 * The same code serves both sides, so swapping the two images swaps the sides' gradients with the same bits.
 * dpool: NULL, or the fp32 gradient at this tap's 2x2 max pool, NHWC [n, H / 2, W / 2, C] (16-byte aligned): the
 * pooled gradient goes to the window's first maximum of f in row-major order (torch's max_pool2d rule); the row and
 * column the floor drops (odd H or W) get none.  Out: grad bf16 NHWC [n, H, W, C] (16-byte aligned) =
 *   bf16(f_c > 0 ? routed_c + head_c : 0),
 * the gradient at the pre-activation of the conv whose ReLU output the tap is.  H W <= 2^24. */
int ga_lpips_tap_backward(const void *feat, int n, int H, int W, int C, int side, const float *lin_w, const float *g,
                          const float *dpool, void *grad, void *stream);
/* The dgrad of VGG's first convolution (3 -> 64) fused with the backward of ga_lpips_pack.  g0 bf16 NHWC
 * [n, H, W, 64] (16-byte aligned): the gradient at conv 0's pre-activation; w_flip fp32 [9, 64, 3] (device),
 * w_flip[ky * 3 + kx, co, c] = bf16(W0[co, c, 2 - ky, 2 - kx]) as fp32.  Per pixel and c < 3:
 *   acc_c = sum over taps (ky, kx) in row-major order, inside the image, of sum over co in increasing order of
 *           w_flip[ky * 3 + kx, co, c] * g0[y + ky - 1, x + kx - 1, co]
 *   dx[i, c, y, x] = acc_c / scale[c], then * 2 when normalize != 0        (fp32 NCHW [n, 3, H, W])
 * (the straight-through gradient of the pack's bf16 rounding).  n <= 65535. */
int ga_lpips_input_backward(const void *g0, int n, int H, int W, const float *w_flip, const float *scale,
                            int normalize, float *dx, void *stream);

/*
 * ---------------------------------------------------------------------------
 * Part 10: surface point clouds, the inputs the reference's scripts/save_pcd.py (save_pcd_from_depth :323-403) and
 * scripts/save_pcd_from_gs.py (:158-185) make with pytorch3d.ops.sample_farthest_points: a G-buffer chunk's depth
 * maps fused into one cloud, and farthest-point sampling of clouds of up to 4M points.
 * pcd_ops.cu is compiled without FMA contraction: every operation below is rounded to fp32 on its own.
 * ---------------------------------------------------------------------------
 */
/* ga_fps's range: the one-CTA kernel holds a cloud in registers. */
#define GA_FPS_MAX_N 16384
#define GA_FPS_MAX_K 1024
/* ga_fps_ex's range. */
#define GA_FPS_EX_MAX_N 4194304
#define GA_FPS_EX_MAX_K 32768
/* Bytes of the workspace ga_fps_ex needs: a 64-bit slot per (cloud, round) and the running minimum distance of
 * every point.  Host-only, no CUDA call. */
size_t ga_fps_ex_workspace_bytes(int batch, int N, int K);
/* Farthest-point sampling with ga_fps's selection rule (Part 5: point 0 is start_idx[b], point k the one farthest
 * from the points already chosen, distance (dx*dx + dy*dy) + dz*dz with each operation rounded on its own, ties to the
 * lowest index) over clouds of different lengths, as pytorch3d's sample_farthest_points pads them.
 * pcd fp32 [batch, N, 3]; lengths int32 [batch] (device) or NULL: cloud b is its first min(lengths[b], N) points
 * (every cloud has N points when NULL); start_idx int32 [batch] in [0, lengths[b]) (device; not read for an empty
 * cloud).  idx_out int32 [batch, K], xyz_out fp32 [batch, K, 3]: the first min(K, lengths[b]) entries of cloud b
 * are its samples, the rest -1 and (0, 0, 0).  N <= GA_FPS_EX_MAX_N and K <= GA_FPS_EX_MAX_K (GA_ERR_SIZE above).
 * Without lengths, where N <= GA_FPS_MAX_N and K <= min(N, GA_FPS_MAX_K), this is ga_fps (the workspace is not read
 * and may be NULL).  Otherwise one cooperative launch: each cloud gets several CTAs that keep a slice of its points
 * in registers (the rest, and their distances, in the workspace), and each round is reduced by a 64-bit atomicMax
 * of (distance bits << 32 | ~index) into the round's slot, then one grid-wide barrier.  GA_ERR_SIZE when the device
 * cannot hold batch CTAs of it at once (batch > 132 on an H100 SXM).  The same inputs give the same bits. */
int ga_fps_ex(const float *pcd, const int32_t *lengths, int batch, int N, int K, const int32_t *start_idx,
              int32_t *idx_out, float *xyz_out, void *workspace, size_t workspace_bytes, void *stream);
/* Bytes of scratch ga_chunk_surface_points needs.  Host-only, no CUDA call. */
size_t ga_chunk_surface_points_scratch_bytes(int n_views, int H, int W);
/* The surface points of a chunk's views, fused.  alpha uint8 [H, n_chunk * W] and depth fp32 [n_chunk, H, W],
 * cams fp32 [n_chunk, 25] as ga_gbuffer_pack takes them; views int32 [n_views] in [0, n_chunk) (the caller checks
 * the range).  W % 4 == 0.  Pixel (x, y) of view views[s] is unprojected exactly as ga_gbuffer_pack's encoder
 * channels 12-14 (the same device code: RaySampler, clip to [-0.45, 0.45], 0 where |p| == 0.45) and kept where
 *   alpha >= alpha_min  and  depth >= min_depth  and  all three coordinates != 0
 * (save_pcd_from_depth with alpha_min 255, its alpha_mask == 1, and min_depth 1.05: a kept coordinate is strictly
 * inside +-0.45).  points fp32 [n_views * H * W, 3] (room for every pixel) receives the kept points in view order
 * (s), then row-major pixel order; count int32 [1] (device) = their number.  Three launches (count per block, scan,
 * emit), no atomics. */
int ga_chunk_surface_points(const uint8_t *alpha, const float *depth, const float *cams, int n_chunk, int H, int W,
                            const int32_t *views, int n_views, int alpha_min, float min_depth, float *points,
                            int32_t *count, void *scratch, size_t scratch_bytes, void *stream);

/*
 * ---------------------------------------------------------------------------
 * Part 11: PatchGAN discriminator, the reference's nsr/losses/disc.py NLayerDiscriminator(input_nc=3, ndf=64,
 * n_layers=3, use_actnorm=False): five 4x4 convolutions with pad 1 (strides 2, 2, 2, 1, 1; channels 3 -> 64 -> 128 ->
 * 256 -> 512 -> 1), BatchNorm2d after convs 2-4, LeakyReLU(0.2) after convs 1-4; forward in training and eval mode,
 * input and weight gradients.  Activations NHWC; every weight is repacked from the fp32 parameters on every call.
 *   conv 1: the image packed by ga_vae_enc_input (c_pad 8, bf16), ga_conv4x4_lrelu_bf16 -> a1 bf16
 *   conv k = 2..4: ga_conv4x4_stats -> z_k fp32 and per-CTA partials, ga_disc_bn_forward -> a_k bf16
 *   conv 5: ga_disc_conv5 -> fp32 logits
 * Packed weights of a 4x4 conv W [Co, Ci, 4, 4]: bf16 [Co, k_pitch], column (ky * 4 + kx) * Ci' + ci = W[co, ci, ky, kx]
 * (Ci' = 8 for conv 1, channels 3-7 zero), k_pitch = 16 Ci' rounded up to 64.
 * Backward, from the logits' fp32 gradient g5:
 *   ga_disc_conv5_backward -> gy4 = dL/dy4 (y4 = BN 4's output) fp32, BN 4's partials, dW5
 *   ga_disc_bn_backward    -> dgamma, dbeta, dz4 = dL/dz4 bf16
 *   ga_disc_wgrad(dz_k, a_{k-1}) -> dW_k;  ga_disc_dgrad(dz_k, flipped W_k) -> gy_{k-1} fp32 (k = 3, 4) or dz1 bf16
 *   conv 1: ga_disc_wgrad(dz1, packed image) -> dW1, ga_disc_colsum(dz1) -> db1, ga_disc_input_backward -> dx.
 * dgrad weights: stride 1 (conv 4), the 4x4 conv of the gradient padded by 2: bf16 [Ci, k_pitch], column
 * (ky * 4 + kx) * Co + co = W[co, ci, 3 - ky, 3 - kx].  Stride 2 (convs 2, 3): the input pixel (2a + py, 2b + px) of
 * parity class (py, px) receives a 2x2 stride-1 conv of the gradient at rows a - 1 + py + ty (ty = 0, 1) and columns
 * b - 1 + px + tx with W[co, ci, 3 - py - 2 ty, 3 - px - 2 tx]; four packs [4 = 2 py + px][Ci, k_pitch], column
 * (ty * 2 + tx) * Co + co, k_pitch = 4 Co rounded up to 64.
 * Rounding: bf16 operands (activations a_k, packed weights, dz_k), fp32 accumulation in the wgmma's order; z_k, gy_k
 * and the logits fp32; conv 5's weights fp32.  disc_ops.cu is compiled without FMA contraction: every operation of
 * the non-GEMM kernels below is rounded to fp32 on its own, in the order written.  No atomics: the same inputs give
 * the same bits.
 * Alignment (GA_ERR_BADARG otherwise): the bf16 NHWC inputs of the convolutions and g1 of ga_disc_input_backward
 * 16 bytes; every fp32 tensor read or written as float2 8 bytes (z of ga_conv4x4_stats; z and partial of
 * ga_disc_bn_forward; z4, gy4, bn_partial and dw_partial of ga_disc_conv5_backward; z, gy_out and partial of
 * ga_disc_dgrad; gy, z, partial and k_scratch of ga_disc_bn_backward; the workspace of ga_disc_wgrad); every bf16
 * tensor read or written in pairs 4 bytes (the bf16 outputs of ga_conv4x4_lrelu_bf16, ga_disc_bn_forward,
 * ga_disc_dgrad and ga_disc_bn_backward; act of ga_disc_dgrad; a4 of ga_disc_conv5_backward).
 * BatchNorm statistics: each conv CTA (128 output pixels) writes its channel mean m_b (fp32 sum / count) and
 * M2_b = sum (z - m_b)^2 (fp32, from the accumulator registers); the finalize merges them in fp64 with Chan's rule
 * (mean += d n_b / n, M2 += M2_b + d^2 n_a n_b / n), so no E[z^2] - mean^2 cancellation: thread t of 128 merges CTAs
 * t, t + 128, ... in order, then the 128 states are merged by a fixed tree (t with t + s, s = 64, 32, ..., 1).
 * var = M2 / M.  The backward's sums (sum gy, sum gy xhat) are added in fp64 in the same fixed pattern.
 * Test bounds: the bf16-emulating oracle (oracle/disc_oracle.py) rounds where these kernels round, with every sum in
 * fp64.  Its relative L2 distance from fp64 was measured on the golden cases (tests/golden/disc_small.npz, 64 x 64 /
 * 50 x 70, 4 images, the d-step of make_disc_golden.py), and the GPU tests allow 1.5 times it plus 1e-5:
 *   logits, train mode: real 5.1e-3 / 5.1e-3, fake 7.1e-3 / 6.9e-3; eval mode 1.9e-3 / 2.2e-3
 *   input gradient of the g-loss 0.143 / 0.144
 *   d-loss parameter gradients: conv 1 weight 0.096 / 0.133, bias 0.104 / 0.156; conv 2 0.104 / 0.111;
 *   BN 2 weight 0.097 / 0.104, bias 0.121 / 0.114; conv 3 0.088 / 0.097; BN 3 weight 0.065 / 0.071, bias 0.101 /
 *   0.099; conv 4 0.066 / 0.073; BN 4 weight 3.0e-3 / 4.4e-3, bias 0.017 / 0.029; conv 5 weight 3.1e-3 / 4.6e-3,
 *   bias 0 / 0.
 * The gradients are far from fp64 because, with random weights, BatchNorm's backward subtracts nearly equal terms,
 * and bf16 rounding of the activations decides them.  Timings: profiles/disc_h100.md (H100 80GB HBM3, 700 W).
 * ---------------------------------------------------------------------------
 */
/* Output size of a 4x4 pad-1 convolution: (H - 2) / stride + 1, stride 1 or 2; GA_ERR_BADARG when H < 2.  Host only. */
int ga_conv4x4_out_size(int H, int stride);
/* 4x4 pad-1 convolution (Part 5's implicit GEMM generalised to 4x4 taps) with bias and LeakyReLU(0.2):
 * out_bf16[m, c] = bf16(v > 0 ? v : 0.2 v), v = bias[c] + conv.  x bf16 NHWC [n, H, W, Cin], Cin % 8 == 0;
 * w_packed as above; Cout % 64 == 0; out [n, Ho, Wo, Cout]. */
int ga_conv4x4_lrelu_bf16(const void *x, int n, int H, int W, int Cin, const void *w_packed, int k_pitch,
                          const float *bias, int Cout, int stride, void *out_bf16, void *stream);
/* 4x4 pad-1 convolution without bias: z fp32 [M = n Ho Wo, Cout], and partial float2 [ceil(M / 128), Cout]: CTA b's
 * (m_b, M2_b) over rows [128 b, 128 b + 128) as stated above.  partial NULL: z only (eval mode). */
int ga_conv4x4_stats(const void *x, int n, int H, int W, int Cin, const void *w_packed, int k_pitch, int Cout,
                     int stride, float *z, void *partial, void *stream);
/* BatchNorm2d + LeakyReLU(0.2) on z fp32 [M, C].  training != 0: mean and var (biased) from ga_conv4x4_stats's
 * partials (Chan, fp64), rstd = fp32(1 / sqrt(var + eps)) in fp64; running_mean = fp32((1 - momentum) rm + momentum
 * mean), running_var = fp32((1 - momentum) rv + momentum M2 / (M - 1)), in fp64 (M >= 2).  training == 0: mean =
 * running_mean, rstd from running_var; the running stats are not written.  mean_out, rstd_out fp32 [C];
 * a_out bf16 [M, C] = bf16(lrelu(((z - mean) rstd) gamma + beta)). */
int ga_disc_bn_forward(const float *z, const void *partial, int64_t M, int C, const float *gamma, const float *beta,
                       int training, float momentum, float eps, float *running_mean, float *running_var,
                       float *mean_out, float *rstd_out, void *a_out, void *stream);
/* Conv 5 (512 -> 1, 4x4, pad 1, stride 1): x bf16 NHWC [n, H, W, 512], w5 fp32 [16, 512] (w5[ky * 4 + kx, ci] =
 * W5[0, ci, ky, kx]), bias fp32 [1] (device).  out fp32 [n, H - 1, W - 1] = bias + sum over taps in row-major order
 * of (lane sums of channels 8 l .. 8 l + 7 then 256 + 8 l .., increasing), then an xor butterfly over 32 lanes. */
int ga_disc_conv5(const void *x, int n, int H, int W, const float *w5, const float *bias, float *out, void *stream);
/* Number of partial rows ga_disc_conv5_backward writes for conv 5's input [n, H, W]. */
int ga_disc_conv5_partials(int n, int H, int W);
/* Conv 5's backward through LeakyReLU 4 to BatchNorm 4's output.  g5 fp32 [n, H - 1, W - 1]; a4 bf16 and z4 fp32
 * [n, H, W, 512]; mean4, rstd4 BN 4's.  Per input pixel p and channel c: ga = sum over taps (row-major) of g5[o] w5[tap,
 * c] where o is the output the tap reaches; gy4[p, c] = a4 > 0 ? ga : 0.2 ga.  Block b of 256 pixels: bn_partial float2
 * [b, 512] = (sum gy4, sum gy4 xhat) in pixel order, xhat = (z4 - mean4) rstd4; dw_partial fp32 [b, 16, 512] = sum
 * g5[o] a4[p]; dw5 fp32 [16, 512] = the fp64 sum of dw_partial over blocks in order (both NULL: no weight
 * gradient is formed). */
int ga_disc_conv5_backward(const float *g5, int n, int H, int W, const float *w5, const void *a4, const float *z4,
                           const float *mean4, const float *rstd4, float *gy4, void *bn_partial, float *dw_partial,
                           float *dw5, void *stream);
/* Number of partial rows ga_disc_dgrad writes for an output (the forward's input) of [n, H, W]. */
int ga_disc_dgrad_partials(int n, int H, int W, int stride);
/* dgrad of a 4x4 pad-1 convolution whose input is [n, H, W, Cout] (its gradient is this call's output) and whose
 * output gradient is g bf16 [n, Ho, Wo, Cg]; w_packed: the flipped packs above (Cout = the forward's Ci).  act bf16
 * [n, H, W, Cout]: the LeakyReLU output at the forward's input.  With v the dgrad:
 *   z == NULL: out_bf16 = bf16(act > 0 ? v : 0.2 v)                      (conv 1's LeakyReLU, no BatchNorm)
 *   z != NULL: gy_out fp32 = act > 0 ? v : 0.2 v, and per CTA (class by class for stride 2, classes in order 2 py +
 *              px) partial float2 [ga_disc_dgrad_partials, Cout] = (sum gy, sum gy xhat), xhat = (z - mean) rstd. */
int ga_disc_dgrad(const void *g, int n, int H, int W, int Cg, const void *w_packed, int k_pitch, int Cout, int stride,
                  const void *act, const float *z, const float *mean, const float *rstd, float *gy_out, void *partial,
                  void *out_bf16, void *stream);
/* BatchNorm backward on gy fp32 [M, C] (the gradient at the BN output): sums S = sum gy, T = sum gy xhat over the
 * n_partial rows of partial (fp64, the fixed pattern above); dbeta = fp32(S), dgamma = fp32(T) (either may be NULL); k = (fp32(S / M),
 * fp32(T / M)) in training mode, (0, 0) in eval mode (fixed statistics), into k_scratch (float2 [C]);
 * dz_bf16 [M, C] = bf16((gamma rstd) ((gy - k.x) - xhat k.y)). */
int ga_disc_bn_backward(const float *gy, const float *z, int64_t M, int C, const float *mean, const float *rstd,
                        const float *gamma, const void *partial, int n_partial, int training, float *dgamma, float *dbeta,
                        void *k_scratch, void *dz_bf16, void *stream);
/* Bytes of workspace ga_disc_wgrad needs.  Host only. */
size_t ga_disc_wgrad_workspace_bytes(int n, int Ho, int Wo, int Co, int Cin);
/* Weight gradient of a 4x4 pad-1 convolution: dy bf16 [n, Ho, Wo, Co] (Co % 64 == 0), x bf16 NHWC [n, H, W, Cin]
 * (Cin % 8 == 0).  D[co, (ky * 4 + kx) Cin + ci] = sum over output pixels p of dy[p, co] x[p's tap, ci]: a GEMM whose
 * K is the pixel count, both operands MN-major; they are staged with cp.async as they lie and transposed by
 * ldmatrix.trans into mma.sync m16n8k16 (fp32 accumulation).  Split over pixels into S fp32 partials (S from the
 * shapes only), summed in split order in fp64: dw fp32 [Co, cin_out, 4, 4] (the parameter layout, channels past
 * cin_out dropped). */
int ga_disc_wgrad(const void *dy, const void *x, int n, int H, int W, int Cin, int Co, int stride, int cin_out,
                  void *workspace, size_t workspace_bytes, float *dw, void *stream);
/* Bytes of scratch ga_disc_colsum needs.  Host only. */
size_t ga_disc_colsum_scratch_bytes(int64_t rows, int C);
/* out fp32 [C] = column sums of x [rows, C] (bf16 when is_bf16, else fp32), 256 % C == 0: blocks of 1024 rows summed
 * in fp32 in a fixed order, the blocks in order in fp64. */
int ga_disc_colsum(const void *x, int is_bf16, int64_t rows, int C, void *scratch, size_t scratch_bytes, float *out,
                   void *stream);
/* Conv 1's dgrad to the image: g1 bf16 [n, Ho, Wo, 64] (dz1), w1 fp32 [16, 64, 3] (w1[ky * 4 + kx, co, c] =
 * bf16(W1[co, c, ky, kx]) as fp32).  dx fp32 NCHW [n, 3, H, W]: per pixel the taps reaching it in row-major order,
 * within a tap co increasing (the straight-through gradient of the input's bf16 rounding). */
int ga_disc_input_backward(const void *g1, int n, int H, int W, const float *w1, float *dx, void *stream);

/*
 * ---------------------------------------------------------------------------
 * Part 12: differentiable attention, xformers.ops.memory_efficient_attention for training (csrc/attention_grad.cu).
 * O = softmax(S) V with S = q k^T * scale, lse[bh, i] = ln sum_j exp(S_ij) (fp32), and the backward
 *   Delta_i = sum_c dO_ic O_ic,  P = exp(S - lse),  dV = P^T dO,  dS = P o (dO V^T - Delta),  dK = scale dS^T q,
 *   dQ = scale dS k.
 * Tensors are bf16 and addressed where they lie: element (b, n, h, c) of tensor t at t + b s0 + n s1 + h s2 + c, with
 * strides = int64 [8][3] (host) for q, k, v, o, dout, dq, dk, dv in that order, in elements (a 3-D [B, N, d] tensor:
 * heads 1, s2 0).  Every stride a multiple of 8 and every tensor 16-byte aligned.  Head dimensions d_qk (q, k) and
 * d_v (v, o) are 32 or 64; 32 is zero-padded to 64 in shared memory, which is exact.  lse and delta fp32
 * [batch * heads, Nq].  Any Nq, Nk >= 1; rows past the end are zero-filled on load and masked, never read.
 * Nq <= 16 and Nk <= 16: one warp per (sequence, head) on CUDA cores, bf16 operands and fp32 arithmetic.  Otherwise
 * wgmma m64n64k16 (bf16 operands, fp32 accumulation) over 64 x 64 tiles; P is rounded to bf16 before P V and
 * P^T dO, dS before dS^T q and dS k.  The backward runs a Delta pass, a dK/dV kernel (one CTA per key block over all
 * query blocks) and a dQ kernel (one CTA per query block over all key blocks): no atomics, the same inputs give the
 * same bits.  The grid is one-dimensional, so batch * heads may exceed 65535.
 * Test bounds (tests/attention_grad_ref.py): a bf16-emulating fp64 reference rounds where the tiled kernels round;
 * the GPU result is held to 1.5 times its measured distance from fp64.  Timings: profiles/attention_grad_h100.md.
 * ---------------------------------------------------------------------------
 */
/* Host only, no CUDA call: 0 when the arguments are accepted, else GA_ERR_BADARG (a NULL q, k, v, o, lse or strides;
 * batch, heads, Nq or Nk < 1; d_qk or d_v not 32 or 64; backward with a NULL dout or delta; a misaligned tensor or
 * a negative or non-multiple-of-8 stride of a tensor in use; a zero stride of o, dq, dk or dv on a dimension of size
 * > 1, where CTAs would write the same elements) or GA_ERR_SIZE (more than 2^31 - 1 CTAs).  dq, dk, dv
 * may each be NULL: that gradient is not formed. */
int ga_attention_grad_validate(const void *q, const void *k, const void *v, const void *o, const float *lse,
                               const void *dout, const float *delta, const void *dq, const void *dk, const void *dv,
                               int batch, int heads, int Nq, int Nk, int d_qk, int d_v, const int64_t *strides,
                               int backward);
/* Forward: o (written, strides row 3) and lse. */
int ga_attention_fwd_lse_bf16(const void *q, const void *k, const void *v, void *o, float *lse, int batch, int heads,
                              int Nq, int Nk, int d_qk, int d_v, const int64_t *strides, float scale, void *stream);
/* Backward from the forward's o and lse and the output gradient dout; delta is fp32 scratch [batch * heads, Nq].
 * The dQ kernel is skipped when dq is NULL, the dK/dV kernel when dk and dv are both NULL; with dk and dq NULL (dV
 * alone) neither the Delta pass nor dS is formed. */
int ga_attention_bwd_bf16(const void *q, const void *k, const void *v, const void *o, const float *lse,
                          const void *dout, float *delta, void *dq, void *dk, void *dv, int batch, int heads, int Nq,
                          int Nk, int d_qk, int d_v, const int64_t *strides, float scale, void *stream);

/*
 * ---------------------------------------------------------------------------
 * Part 13: linear-layer gradients and a differentiable FusedMLP (xformers' FusedMLP: Linear(D -> hidden, no bias),
 * bias + exact GELU, Linear(hidden -> D, no bias), bias; csrc/linear_grad.cu and csrc/dit_gemm.cu).
 * For y = x W^T + b with x [M, K], W [N, K] (the nn.Linear parameter layout) and the output gradient G = dy [M, N]:
 *   dx = G W          (dgrad: contracts W along its rows)
 *   dW = G^T x        (wgrad: contracts both along the M rows)
 *   db = sum_m G[m, :]
 * The MLP forward for training keeps fc1's pre-activation: v = x W1^T + b1, Z = bf16(v), H = bf16(gelu_erf(v)),
 * y = H W2^T + b2.  Its backward: db2 = colsum(dY), dW2 = dY^T H, dZ = bf16((dY W2) o gelu'(Z)), db1 = colsum(dZ),
 * dW1 = dZ^T x, dx = dZ W1, with gelu'(z) = Phi(z) + z phi(z) evaluated in fp32 from the bf16 Z.
 * Rounding: every GEMM operand is bf16 (x, W1, W2, H, dY, dZ; the fp32 parameters are packed to bf16 row-major on
 * every call), products are accumulated in fp32 by wgmma; Z and H are stored as bf16; dgrad outputs are bf16 or fp32
 * as asked; dW and db are fp32.  No atomics anywhere: the same inputs give the same bits on any H100.
 * Every row count M >= 1 is accepted; N and K (and every pitch, which equals the row length) are multiples of 8, the
 * TMA pitch; rows and columns past the end of a tile are zero-filled by TMA and never written.
 * wgrad splits the M rows into S consecutive ranges of 64-row blocks (S from ga_linear_wgrad_splits: the shapes only,
 * never the SM count), each range's fp32 partial [N, K] is written to the workspace, and dW = the partials added in
 * fp32 in split order (S = 1 writes dW directly).  Bias gradients (ga_linear_bias_grad_bf16) sum the bf16 matrix
 * given (dY for db2, the bf16 dZ for db1) in fp32: within a chunk of 256 rows, warp w (0..7) adds rows w, w + 8, ...
 * in increasing order, the eight warp sums are added in warp order, then the chunks are added in chunk order.
 * Test bounds (tests/mlp_grad_ref.py): a bf16-emulating fp64 reference rounds where these kernels round; the GPU
 * results are held to 1.5 times its measured distance from fp64.  Timings: profiles/mlp_grad_h100.md.
 * ---------------------------------------------------------------------------
 */
#define GA_LINEAR_FC1    0   /* ga_linear_fc1_gelu_bf16 */
#define GA_LINEAR_DGRAD  1   /* ga_linear_dgrad_bf16 */
#define GA_LINEAR_WGRAD  2   /* ga_linear_wgrad_bf16 */
#define GA_LINEAR_BGRAD  3   /* ga_linear_bias_grad_bf16 */
/* Host only, no CUDA call: 0 when the entry point `op` (GA_LINEAR_*) accepts the arguments, else GA_ERR_BADARG.
 * The arguments of each op (a, b, aux, out as below; every pointer given must be 16-byte aligned):
 *   FC1:   a = x [M, K], b = W1 [N, K], aux = Z, out = H [M, N]; all non-NULL; out_f32 == 0; block_n in {64, 128,
 *          192, 256} (ga_gemm_bf16_tn's tile widths);
 *   DGRAD: a = G [M, N], b = W [N, K], out [M, K] (fp32 when out_f32, else bf16) non-NULL; aux = Z [M, K] or NULL,
 *          and with Z the output is bf16 (out_f32 == 0); out_f32 0 or 1;
 *   WGRAD: a = G [M, N], b = x [M, K], out = dW fp32 [N, K] non-NULL; out_f32 == 1; workspace_bytes >=
 *          ga_linear_wgrad_workspace_bytes(M, N, K), and the workspace non-NULL when that is > 0;
 *   BGRAD: a = G [M, N] non-NULL, out = db fp32 [N] non-NULL; out_f32 == 1; K is ignored; workspace as for WGRAD
 *          with ga_linear_bias_grad_workspace_bytes(M, N).
 * M >= 1; N >= 8 and K >= 8 multiples of 8 (K unused by BGRAD); M * max(N, K) < 2^31. */
int ga_linear_grad_validate(int op, const void *a, const void *b, const void *aux, const void *out, int out_f32, int M,
                            int N, int K, int block_n, const void *workspace, size_t workspace_bytes);
/* fc1 of the MLP for training: v = x W1^T + b1 (b1 fp32 [N] or NULL), H = bf16(gelu_erf(v)), Z = bf16(v), both bf16
 * [M, N] (row pitch N).  x bf16 [M, K], W1 bf16 [N, K].  ga_gemm_bf16_tn's GEMM at tile width block_n, with an
 * epilogue that writes both outputs from one accumulator; gelu_erf is GA_EPI_GELU_BF16's. */
int ga_linear_fc1_gelu_bf16(const void *x, const void *w1, const float *b1, void *h, void *z, int M, int N, int K,
                            int block_n, void *stream);
/* dgrad: out[M, K] = G[M, N] W[N, K], G and W bf16 row-major (W as stored, the parameter packed to bf16).  z == NULL:
 * out = the fp32 product (out_f32) or its bf16 rounding.  z bf16 [M, K]: out bf16 = bf16(v gelu'(z)), v the fp32
 * product (fc2's dgrad fused with the GELU backward: dZ). */
int ga_linear_dgrad_bf16(const void *g, const void *w, const void *z, void *out, int out_f32, int M, int N, int K,
                         void *stream);
/* Number of M splits ga_linear_wgrad_bf16 uses for these shapes (>= 1).  Host only. */
int ga_linear_wgrad_splits(int M, int N, int K);
/* Bytes of workspace ga_linear_wgrad_bf16 needs (0 when there is one split).  Host only. */
size_t ga_linear_wgrad_workspace_bytes(int M, int N, int K);
/* wgrad: dW fp32 [N, K] = G^T x, G bf16 [M, N], x bf16 [M, K], split over M as stated above. */
int ga_linear_wgrad_bf16(const void *g, const void *x, float *dw, int M, int N, int K, void *workspace,
                         size_t workspace_bytes, void *stream);
/* Bytes of workspace ga_linear_bias_grad_bf16 needs (0 when M <= 256).  Host only. */
size_t ga_linear_bias_grad_workspace_bytes(int M, int N);
/* db fp32 [N] = column sums of G bf16 [M, N], in the order stated above. */
int ga_linear_bias_grad_bf16(const void *g, float *db, int M, int N, void *workspace, size_t workspace_bytes,
                             void *stream);

/*
 * ---------------------------------------------------------------------------
 * Part 14: the row kernels of a trainable image-to-3D DiT block (ImageCondDiTBlockPixelArtRMSNormClayLRM,
 * gaussiananything_b200/dit_grad.py; csrc/dit_grad.cu).  With mod = scale_shift_table + t [B, 6 D] in the chunk order
 * shift_msa, scale_msa, gate_msa, shift_mlp, scale_mlp, gate_mlp, and b = r / rows_per_batch the batch item of row r:
 *   RMSNorm-modulate   h = n w (1 + scale[b]) + shift[b],  n = x rstd,  rstd = (mean(x^2) + eps)^-1/2  (x fp32)
 *     backward         dy0 = dh (1 + scale[b]),  dw = sum_r dy0 n,  dscale[b] = sum_{r in b} dh n w,
 *                      dshift[b] = sum_{r in b} dh,  dx = dx_in + rstd (dy0 w - n mean(dy0 w n))
 *                      (without modulation: scale = shift = 0 and no dscale, dshift)
 *   q/k RMSNorm        per 64-column head: qn = bf16(n w), n = q rstd over the head's 64 values (q bf16)
 *     backward         dq = bf16(rstd (dn - n mean(dn n))), dn = dqn w;  dw = sum over rows and heads of dqn n
 *   gated residual     x_out = x + gate[b] a (a fp32, the GEMM's output), optionally followed in the same pass by
 *                      h = bf16(RMSNorm-modulate(x_out))
 *     backward         da = bf16(gate[b] dy),  dgate[b] = sum_{r in b} dy a
 * All arithmetic is fp32; the only bf16 roundings are of the outputs named bf16 above (h, qn, dq, da).  rstd is
 * recomputed from x (or q) in the backward, nothing is saved but the inputs.
 * Layouts: row-major, fp32 rows of D columns (D % 4 == 0, D <= 1024) at pitch D; modulation chunks are [B, mod_ld]
 * pointers already offset to their chunk (shift = mod + 0 D, ...); q/k matrices are bf16 [rows, ld] with head h of
 * part p (p = 0: the q or first block, 1: the k block) at columns 64 (p heads + h) .. + 63, the "(K H D)" layout of a
 * qkv or kv GEMM output.  Columns past parts * heads * 64 (v, padding) are never read or written.
 * Determinism, no atomics: sums over rows are taken in chunks of 32 rows, a chunk never crossing a batch item.  The
 * row kernels (norm and gate backward) run one CTA per chunk, warp w (0..7) adding rows w, w + 8, ... of the chunk in
 * increasing order, the eight warp sums then added in warp order into partial p = b * ceil(rows_per_batch / 32) + c
 * (ga_dit_grad_partials(R, rows_per_batch) partials in all).  The q/k backward runs one CTA per chunk of 32 rows
 * (ga_dit_grad_partials(rows, rows) of them); its 32 slots of 8 lanes take the chunk's (row, head) items s, s + 32,
 * ... in row-major order and the slot sums are added in slot order; partial [part, chunk, 64].  ga_dit_grad_reduce
 * then adds partials in index order.  The same inputs give the same bits on any H100.
 * Test bounds (tests/dit_grad_ref.py): a bf16-emulating fp64 reference rounds where these kernels and Parts 12 and 13
 * round; the GPU results are held to 1.5 times its distance from fp64.  Timings: profiles/dit_block_grad_h100.md.
 * ---------------------------------------------------------------------------
 */
/* Number of partials of a row sum over `rows` rows in batch items of rows_per_batch rows (0 when rows is not a
 * positive multiple of rows_per_batch).  Host only. */
int ga_dit_grad_partials(int rows, int rows_per_batch);
/* Host only, no CUDA call: 0 when ga_dit_rmsnorm_bwd accepts the arguments, else GA_ERR_BADARG.  R a positive multiple
 * of rows_per_batch >= 1; 4 <= D <= 1024, D % 4 == 0; R D < 2^31; dh, x, w, part_dw non-NULL; dx_in only with dx_out;
 * with scale: mod_ld >= D, part_dshift and part_dscale non-NULL, part_ld >= D, both lds multiples of 4; without
 * scale: part_dshift and part_dscale NULL.  Every pointer given 16-byte aligned. */
int ga_dit_rmsnorm_bwd_validate(const float *dh, const float *x, const float *w, const float *scale, int mod_ld,
                                const float *dx_in, const float *dx_out, const float *part_dw,
                                const float *part_dshift, const float *part_dscale, int part_ld, int rows_per_batch,
                                int R, int D);
/* RMSNorm(-modulate) backward as above.  dh, x, dx fp32 [R, D]; scale [B, mod_ld] (NULL: no modulation); dx_out =
 * dx_in + dRMSNorm (dx_in NULL: 0; dx_out NULL: dx is not formed; dx_in may be dx_out); partials part_dw [P, D] and,
 * with scale, part_dshift / part_dscale [P, part_ld], P = ga_dit_grad_partials(R, rows_per_batch). */
int ga_dit_rmsnorm_bwd(const float *dh, const float *x, const float *w, const float *scale, int mod_ld,
                       const float *dx_in, float *dx_out, float *part_dw, float *part_dshift, float *part_dscale,
                       int part_ld, int rows_per_batch, int R, int D, float eps, void *stream);
/* Host only: as ga_dit_rmsnorm_bwd_validate for ga_dit_gate_bwd; dy, a, gate, part_dgate non-NULL and 16-byte
 * aligned, da_bf16 non-NULL and 8-byte aligned, gate_ld and part_ld >= D and multiples of 4. */
int ga_dit_gate_bwd_validate(const float *dy, const float *a, const float *gate, int gate_ld, const void *da_bf16,
                             const float *part_dgate, int part_ld, int rows_per_batch, int R, int D);
/* Gate backward: da bf16 [R, D] = bf16(gate[b] dy), part_dgate [P, part_ld] the chunk sums of dy a. */
int ga_dit_gate_bwd(const float *dy, const float *a, const float *gate, int gate_ld, void *da_bf16, float *part_dgate,
                    int part_ld, int rows_per_batch, int R, int D, void *stream);
/* Host only: 0 when ga_dit_gate_residual accepts the arguments.  Rows as above; x, a, x_out non-NULL; a gate given
 * with gate_ld >= D; w NULL: shift, scale and h_bf16 NULL too; w given: h_bf16 non-NULL (8-byte aligned), shift and
 * scale both NULL or both given with mod_ld >= D; fp32 pointers 16-byte aligned, lds multiples of 4. */
int ga_dit_gate_residual_validate(const float *x, const float *a, const float *gate, int gate_ld, const float *x_out,
                                  const float *w, const float *shift, const float *scale, int mod_ld,
                                  const void *h_bf16, int rows_per_batch, int R, int D);
/* x_out [R, D] = x + gate[b] a (gate NULL: x + a); with w, also h_bf16 = RMSNorm(x_out) w [(1 + scale[b]) +
 * shift[b]] (ga_rmsnorm_modulate's formula, on the fp32 x_out). */
int ga_dit_gate_residual(const float *x, const float *a, const float *gate, int gate_ld, float *x_out, const float *w,
                         const float *shift, const float *scale, int mod_ld, void *h_bf16, int rows_per_batch, int R,
                         int D, float eps, void *stream);
/* Host only: 0 when the q/k RMSNorm forward (backward = 0: dout, ld_dout and part_dw unused and dout, part_dw NULL)
 * or backward (1; out is din) accepts the arguments.  rows, heads >= 1; parts 1 (w1 NULL) or 2 (w1 non-NULL); every
 * ld >= 64 heads parts and a multiple of 8; in, out, dout, w0, w1, part_dw 16-byte aligned. */
int ga_dit_qk_norm_validate(int backward, const void *in, int ld_in, const void *dout, int ld_dout, const void *out,
                            int ld_out, const float *w0, const float *w1, const float *part_dw, int rows, int heads,
                            int parts);
/* q/k RMSNorm forward: out = bf16(n w) per head, w = w0 [64] for part 0 and w1 [64] for part 1.  out may be in. */
int ga_dit_qk_norm_fwd_bf16(const void *in, int ld_in, void *out, int ld_out, const float *w0, const float *w1,
                            int rows, int heads, int parts, float eps, void *stream);
/* q/k RMSNorm backward: in = the pre-norm q/k, dout = the attention's dq/dk (bf16), din = the pre-norm gradient
 * (bf16; din may be dout); part_dw fp32 [parts, ga_dit_grad_partials(rows, rows), 64]. */
int ga_dit_qk_norm_bwd_bf16(const void *in, int ld_in, const void *dout, int ld_dout, void *din, int ld_din,
                            const float *w0, const float *w1, float *part_dw, int rows, int heads, int parts,
                            float eps, void *stream);
/* Host only: 0 when part and out are non-NULL and groups, parts, cols >= 1. */
int ga_dit_grad_reduce_validate(const float *part, const float *out, int groups, int parts, int cols);
/* out [groups, cols] = sum over p = 0, 1, ..., parts - 1 (in that order, fp32) of part [groups, parts, cols]. */
int ga_dit_grad_reduce(const float *part, float *out, int groups, int parts, int cols, void *stream);

/*
 * ---------------------------------------------------------------------------
 * Part 15: the backwards of the image-to-3D DiT outside its blocks (DiT_I23D_PCD_PixelArt_noclip and its stage-2
 * model, gaussiananything_b200/dit_grad.py model_forward; csrc/dit_model_grad.cu).  The forward runs on the Part 2
 * launches the inference engine uses:
 *   stem     sinus = timestep_embedding(t, 256); a1 = sinus W0^T + b0; temb = silu(a1) W2^T + b2
 *            + (LayerNorm(vec) Wv^T + bv); t0 = silu(temb) Wa^T + ba [B, 6 D]            (fp32, ga_linear_small)
 *   tokens   e1 = bf16(gelu_tanh([xyz | x] W1^T + b1)); xres = e1 Wf2^T + bf2 (+ bf16(posenc(xyz)) Wxyz^T + bxyz)
 *   head     y = (LN(xres) (1 + scale[b]) + shift[b]) Wf^T + bf,  [shift | scale] = table + temb  (eps 1e-6)
 * Its backward: fc2's and the xyz projection's dW and db and fc2's dgrad are Part 13 GEMMs on bf16(dxres); the
 * kernels below do the rest in fp32.  As in Part 14 nothing uses atomics: sums over the R token rows are written as
 * one partial per chunk of 32 rows of one batch item (ga_dit_grad_partials(R, rows_per_batch) of them), rows added in
 * a stated order, and ga_dit_grad_reduce adds the partials in index order; sums over the B stem rows are taken in
 * row order.  The same inputs give the same bits on any H100.  Every entry point checks its arguments with its
 * host-only *_validate first (0, or GA_ERR_BADARG).
 * Test bounds (tests/dit_model_grad_ref.py): the GPU gradients are held to 1.5 times a bf16-emulating fp64
 * reference's distance from fp64.  Timings: profiles/dit_train_h100.md.
 * ---------------------------------------------------------------------------
 */
/* Host only: R a positive multiple of rows_per_batch; 4 <= D <= 1024, D % 4 == 0; 1 <= Cout <= 16; R D < 2^31;
 * x, mod, W non-NULL; dy non-NULL; part_dw and part_db both NULL or both given; x, mod, W, dx, part_dmod, part_dw
 * 16-byte aligned, dy and part_db 4-byte aligned. */
int ga_dit_final_layer_bwd_validate(const float *x, const float *mod, const float *W, const float *dy,
                                    const float *dx, const float *part_dmod, const float *part_dw,
                                    const float *part_db, int rows_per_batch, int R, int D, int Cout);
/* Final-layer backward: x fp32 [R, D] (the residual stream), mod [B, 2 D] = [shift | scale], W [Cout, D], dy
 * [R, Cout].  With n = LN(x) recomputed and dh = dy W: dx [R, D] = rstd (dn - mean(dn) - n mean(dn n)),
 * dn = dh (1 + scale[b]) (NULL: not formed); part_dmod [P, 2 D] = the chunk sums of [dh | dh n] (NULL: not formed);
 * part_dw [P, Cout, D] and part_db [P, Cout] = the chunk sums of dy h and dy, h = n (1 + scale[b]) + shift[b], rows
 * in increasing order.  P = ga_dit_grad_partials(R, rows_per_batch). */
int ga_dit_final_layer_bwd(const float *x, const float *mod, const float *W, const float *dy, float *dx,
                           float *part_dmod, float *part_dw, float *part_db, int rows_per_batch, int R, int D,
                           int Cout, float eps, void *stream);
/* Host only: R >= 1; 1 <= D <= 1024; Cx >= 1, C2 >= 0, Cx + C2 <= 16; R D < 2^31; xin2 given iff C2 > 0; xin, W1,
 * b1, de1, part_dw1, part_db1 non-NULL; every pointer 4-byte aligned. */
int ga_dit_embed_fc1_bwd_validate(const float *xin, int Cx, const float *xin2, int C2, const float *W1,
                                  const float *b1, const float *de1, const float *part_dw1, const float *part_db1,
                                  const float *dxin, int R, int D);
/* Token-embedder fc1 backward (ga_embed_fc1's layer, K = C2 + Cx inputs [xin2 | xin]): v recomputed in fp32, dv =
 * de1 gelu_tanh'(v) with de1 fp32 [R, D]; part_dw1 [P, D, K] and part_db1 [P, D] the chunk sums of dv [xin2 | xin]
 * and dv over rows in increasing order (P = ga_dit_grad_partials(R, R)); dxin [R, Cx] = dv W1[:, C2:] (NULL: not
 * formed; the xin2 columns get no gradient). */
int ga_dit_embed_fc1_bwd(const float *xin, int Cx, const float *xin2, int C2, const float *W1, const float *b1,
                         const float *de1, float *part_dw1, float *part_db1, float *dxin, int R, int D, void *stream);
/* Host only: rows, N >= 1; K >= 4, K % 4 == 0; act_in 0 or 1; N K < 2^31 and P rows K < 2^31; x, W non-NULL and
 * 16-byte aligned; dy non-NULL; dW 16-byte aligned; dx given: part non-NULL and 16-byte aligned; dx NULL: part and
 * dx_in NULL; dy, db, dx, dx_in 4-byte aligned. */
int ga_dit_linear_small_bwd_validate(const float *x, int act_in, const float *W, const float *dy, const float *dW,
                                     const float *db, const float *part, const float *dx_in, const float *dx,
                                     int rows, int N, int K);
/* Backward of ga_linear_small's y = act(x) W^T + b for any number of rows: x [rows, K], W [N, K], dy [rows, N], act
 * SiLU when act_in.  dW [N, K] = sum over b = 0, 1, ... of dy[b]^T act(x[b]); db [N] likewise; dx [rows, K] = dx_in +
 * act'(x) (dy W) (dx_in NULL: 0; dx_in may be dx), dy W summed over chunks of 32 rows of W (P =
 * ga_dit_grad_partials(N, N) partials [P, rows, K] in part, rows of a chunk in increasing order) then over the
 * chunks in order.  Any output may be NULL.  Byte floor: W read once and dW written once, 8 N K bytes, plus 8 P rows K
 * bytes of partials when dx is formed. */
int ga_dit_linear_small_bwd(const float *x, int act_in, const float *W, const float *dy, float *dW, float *db,
                            float *part, const float *dx_in, float *dx, int rows, int N, int K, void *stream);
/* Host only: R >= 1; 4 <= D <= 1024, D % 4 == 0; R D < 2^31; x, w, dy non-NULL; every pointer 16-byte aligned. */
int ga_dit_layernorm_rows_bwd_validate(const float *x, const float *w, const float *dy, const float *dx,
                                       const float *dw, const float *db, int R, int D);
/* Backward of ga_layernorm_rows with affine w (the pooled vector's LayerNorm): n = (x - mean) rstd, dn = dy w;
 * dx [R, D] = rstd (dn - mean(dn) - n mean(dn n)); dw = sum_r dy n, db = sum_r dy, rows in increasing order (one
 * CTA).  Any output may be NULL. */
int ga_dit_layernorm_rows_bwd(const float *x, const float *w, const float *dy, float *dx, float *dw, float *db,
                              int R, int D, float eps, void *stream);

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
