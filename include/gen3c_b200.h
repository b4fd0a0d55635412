/*
 * gen3c_b200 — C ABI of libgen3c_b200.so (sm_90a, H100).
 *
 * The reference (nv-tlabs/GEN3C) has no FFI: its seams are Python call sites.  Each entry point
 * below replaces one of them; the citation is the reference file:line whose arithmetic it
 * reproduces.  Conventions: every pointer is a DEVICE pointer owned by the caller unless noted;
 * `stream` is a cudaStream_t passed as void*; functions enqueue on that stream and return
 * immediately; return 0 on success, <0 on error (G3C_E*), message via g3c_last_error() (thread
 * local).  No hidden allocations after a *_create / *_set_shape / *_set_deterministic / g3c_dit_set_linear_fp8 call.  Handles are not thread
 * safe; distinct handles are independent.  There is no CPU fallback anywhere in this library.
 */
#ifndef GEN3C_B200_H_
#define GEN3C_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define G3C_OK 0
#define G3C_EINVAL (-1)
#define G3C_ECUDA (-2)
#define G3C_ENOMEM (-3)
#define G3C_ESTATE (-4)
#define G3C_ENCCL (-5)

const char* g3c_last_error(void);
int g3c_version(void);
int g3c_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ===================================== Path R: 3D-cache render ================================= */

typedef struct g3c_render g3c_render_t;

/* Workspace for H x W frames: accumulation buffers for `max_items_per_pass` frames kept L2
 * resident between the splat and the normalise pass. */
int g3c_render_create(int H, int W, int max_items_per_pass, g3c_render_t** out);
int g3c_render_destroy(g3c_render_t* r);

/* on != 0: g3c_forward_warp, g3c_render_cache and g3c_bilinear_splatting on this handle splat in a fixed order and are
 * bitwise reproducible whatever the pass size or the run (torch.use_deterministic_algorithms(True) for the
 * reference's index_put_(accumulate=True)).  Each destination texel sums its contributions sequentially in fp32 from
 * 0, corner-major (nw, sw, ne, se, reference :659-675), then in ascending source pixel, with the reference's weight
 * arithmetic; no float atomics.  The first enable allocates the sort workspace, about 76 B per pixel of one frame
 * (69 MB at 704 x 1280); g3c_render_destroy frees it.  on = 0 returns to the default atomic splat.
 * Every other Path R entry point is deterministic already: the log-depth maxima and the foreground z-buffer are
 * atomicMax / atomicMin on float bits, which do not depend on order, and every other output has one writer. */
int g3c_render_set_deterministic(g3c_render_t* r, int on);

#define G3C_WARP_RENDER_DEPTH 1 /* also splat z (forward_warp render_depth=True)            */
#define G3C_WARP_NOT_IMAGE 2    /* is_image=False: fill 0 instead of -1, no clamp to [-1,1] */

/* forward_warp(frame1, mask1, depth1=None, transformation2=w2c, intrinsic2=K, world_points1=points)
 * reference: cosmos_predict1/diffusion/inference/forward_warp_utils_pytorch.py:171-336 (the
 * depth1=None branch :219-224, :244-250, :281-284) incl. project_points :462-486 and
 * bilinear_splatting :576-695.  The log-depth max is taken over all `b` items of the call.
 *   points [b,H,W,3] f32, image [b,C,H,W] f32 (C<=3), mask [b,1,H,W] f32 or NULL (= ones),
 *   w2c [b,4,4], K [b,3,3]  ->  warped [b,C,H,W], mask_out [b,1,H,W],
 *   depth_out [b,H,W] (iff G3C_WARP_RENDER_DEPTH), flow_out [b,2,H,W] or NULL. */
int g3c_forward_warp(g3c_render_t* r, const float* points, const float* image, const float* mask,
                     const float* w2c, const float* K, int b, int C, int flags, float* warped,
                     float* mask_out, float* depth_out, float* flow_out, void* stream);

/* Cache3D_Base.render_cache — reference: cosmos_predict1/diffusion/inference/cache_3d.py:151-236.
 * Items are flattened (B F N) with N fastest and warped in chunks of 2 that share one log-depth
 * max, exactly as the reference loop (:175,:183).  The cache stays on the GPU.
 *   points [B,src_frames,N,H,W,3], images [B,src_frames,N,3,H,W], masks [B,src_frames,N,1,H,W] or
 *   NULL, src_frames = 1 (broadcast over targets) or F_target; w2cs [B,F_target,4,4],
 *   Ks [B,F_target,3,3] -> pixels [B,F,N,3,H,W], masks_out [B,F,N,1,H,W],
 *   depth_out [B,F,N,H,W] iff render_depth. */
int g3c_render_cache(g3c_render_t* r, const float* points, const float* images, const float* masks,
                     const float* w2cs, const float* Ks, int B, int F_target, int N, int src_frames,
                     int render_depth, float* pixels, float* masks_out, float* depth_out,
                     void* stream);

/* bilinear_splatting(frame1, mask1, depth1, flow12, None, is_image) — reference :576-695.
 *   frame [b,C,H,W], mask [b,1,H,W] or NULL, depth [b,1,H,W], flow [b,2,H,W] -> out, mask_out */
int g3c_bilinear_splatting(g3c_render_t* r, const float* frame, const float* mask,
                           const float* depth, const float* flow, int b, int C, int is_image,
                           float* out, float* mask_out, void* stream);

/* The integer part of bilinear_splatting (:605-621): idx [b,4,H,W] int32 =
 * {floor_x, floor_y, ceil_x, ceil_y} after clamping; the same device function the splat uses. */
int g3c_splat_indices(const float* flow, int b, int H, int W, int32_t* idx, void* stream);

/* unproject_points(depth, w2c, K, is_depth, mask) — reference :410-460.
 *   depth [b,1,H,W], mask [b,H,W] uint8 or NULL (= depth>0) -> points [b,H,W,3] */
int g3c_unproject_points(const float* depth, const float* w2c, const float* K, const uint8_t* mask,
                         int b, int H, int W, int is_depth, float* points, void* stream);

/* reliable_depth_mask_range_batch — reference :338-353.  out [b,H,W] uint8 */
int g3c_reliable_depth_mask(const float* depth, int b, int H, int W, int window, float ratio_thresh,
                            float eps, uint8_t* out, void* stream);

/* Second stage of align_depth(..., alignment_method="non_rigid") as called by Cache3D_Buffer.update_cache (reference:
 * cosmos_predict1/diffusion/inference/camera_utils.py:292-345, cache_3d.py:262-282): a per-pixel scale map fitted with
 * `num_iters` Adam steps (lr, betas .9/.999, eps 1e-8) to
 *     mean |unproject(depth*sc) - unproject(target_depth)| over target_mask  +  lambda_arap * mean |box3(sc) - sc| ,
 * gradient in closed form, one stencil kernel per iteration.  `depth` is the source depth AFTER the rigid (affine
 * inverse-depth) stage; `c2w` is the matrix the reference hands to unproject_points (which inverts it).
 *   depth, target_depth [H,W] f32, target_mask [H,W] u8, K [9], c2w [16] (device)  ->  out_depth [H,W] = depth * sc */
int g3c_align_depth_nonrigid(const float* depth, const float* target_depth, const uint8_t* target_mask, const float* K,
                             const float* c2w, int H, int W, int num_iters, float lambda_arap, float lr,
                             float* out_depth, void* stream);

/* The foreground-masking occlusion pass of
 * forward_warp(foreground_masking=True, boundary_mask=...) — reference forward_warp_utils_pytorch.py:285-335 with
 * points_to_mesh :49-132, get_camera_rays :151-168 and the NVIDIA-Warp kernel ray_triangle_intersection_warp.py:23-105.
 * Post-processes the outputs of g3c_forward_warp(..., G3C_WARP_RENDER_DEPTH): pixels whose 1/4-resolution boundary mesh
 * lies more than 0.02 in front of the splatted depth are cleared (mask 0, image -1, depth 0).
 *   points [b,H,W,3] f32 world points, boundary [b,H,W] u8, w2c [b,4,4], K [b,3,3]; in/out warped [b,C,H,W],
 *   mask [b,1,H,W], depth [b,H,W]. */
int g3c_foreground_occlusion(const float* points, const unsigned char* boundary, const float* w2c, const float* K, int b,
                             int C, int H, int W, float* warped, float* mask, float* depth, void* stream);

/* The same pass over the items of a cache render (Cache3D_Base.render_cache with foreground_masking=True, reference
 * cache_3d.py:168-215): items (B F N) as in g3c_render_cache, each with its source frame's points / boundary mask and its
 * target camera.  In/out: the pixels / masks / depth that g3c_render_cache(render_depth=1) wrote. */
int g3c_render_cache_occlusion(const float* points, const unsigned char* boundary, const float* w2cs, const float* Ks, int B,
                               int F_target, int N, int src_frames, float* pixels, float* masks, float* depth, int H, int W,
                               void* stream);

/* ===================================== Path D: DiT denoise step =============================== */

#define G3C_EPI_BF16 0               /* D (bf16) = acc                          */
#define G3C_EPI_GELU_BF16 1          /* D (bf16) = gelu_erf(acc)                */
#define G3C_EPI_GATED_RESIDUAL_F32 2 /* D (f32) += gate[n] * acc                */
#define G3C_EPI_F32 3                /* D (f32) = acc                           */

/* D[M,N] = A[M,K] . B[N,K]^T, bf16 operands (K contiguous), fp32 accumulation on wgmma (Hopper tensor cores).
 * Replaces every nn.Linear of the net (reference: module/attention.py:263-266,289,91-102;
 * module/blocks.py:153-163,228-241).  block_n: 0 = auto, or 64/128/256.  epilogue: one of the four G3C_EPI_* above
 * (any other value is G3C_EINVAL; the fused RMSNorm/RoPE epilogue has its own entry point below). */
int g3c_gemm_bf16(const void* A, const void* B, void* D, int M, int N, int K, int lda, int ldb,
                  int ldd, int epilogue, const float* gate, int block_n, void* stream);

/* D (bf16) [M,N] = RoPE(RMSNorm_head(A . B^T) * gamma): the to_q / to_k projection of the reference
 * (`nn.Sequential(Linear, RMSNorm)`, module/attention.py:263-266) followed by the rotate-half RoPE (:268-283), with the
 * norm and the rotation applied to the fp32 accumulators of each 128-wide head in the GEMM epilogue.  gamma [128] f32,
 * cos_sin [M][128] f32 (cos of the 64 angles | sin) or NULL for no rotation; N must be a multiple of 128. */
int g3c_gemm_norm_rope_bf16(const void* A, const void* B, void* D, int M, int N, int K, int lda, int ldb, int ldd,
                            const float* gamma, const float* cos_sin, float eps, void* stream);

/* FP8 (e4m3) Linear path.  Row quantisation of bf16 x [R, C] (leading dimension ld): amax_r = max_c |x[r,c]|,
 * codes[r,c] = e4m3_rn_satfinite(x[r,c] * (448 / amax_r)) (fp32 multiply), scales[r] = amax_r / 448; a zero row gets
 * codes 0 and scale 1.  C must be a multiple of 16, ld of 8, ldq (>= C) of 16; x, codes, scales 16-byte aligned. */
int g3c_quantize_rows_fp8(const void* x_bf16, int ld, int R, int C, void* codes, int ldq, float* scales, void* stream);

/* D[M,N] = (A8[M,K] . B8[N,K]^T) * scale_A[m] * scale_B[n], then `epilogue` as in g3c_gemm_bf16: e4m3 codes (K
 * contiguous) from g3c_quantize_rows_fp8, on the fp8 wgmma; each 128-code k-block's partial sum is added into fp32
 * accumulators (the instruction's own sum is not full fp32), and tiles are at most 128 columns wide (block_n 256 runs 128).  The scales multiply the accumulators
 * before any epilogue arithmetic.  K, lda and ldb must be multiples of 16; scale_A [M] and scale_B [N] non-NULL and
 * 16-byte aligned. */
int g3c_gemm_fp8(const void* A8, const float* scale_A, const void* B8, const float* scale_B, void* D, int M, int N,
                 int K, int lda, int ldb, int ldd, int epilogue, const float* gate, int block_n, void* stream);

/* g3c_gemm_norm_rope_bf16 on e4m3 operands: the RMSNorm sees the dequantised accumulators. */
int g3c_gemm_norm_rope_fp8(const void* A8, const float* scale_A, const void* B8, const float* scale_B, void* D, int M,
                           int N, int K, int lda, int ldb, int ldd, const float* gamma, const float* cos_sin, float eps,
                           void* stream);

/* O = softmax(Q K^T * scale) V, head_dim 128, no mask — the attention operator behind
 * Attention.cal_attn (reference: module/attention.py:282-297, TE DotProductAttention :228-238;
 * also usable as an `attn_op`, :136-139).
 *   q [Lq, heads*128] (ld ldq), k [Lk, heads*128] (ld ldk), vt [Lk/vt_chunk_len][heads*128]
 *   [vt_chunk_len] (V transposed, keys contiguous; vt_chunk_len <= 0 means Lk), o [Lq, heads*128].
 *   Lk must be a multiple of 128.
 *   scale = ln 2 (0.6931472) declares that Q already carries softmax_scale * log2(e) (the DiT engine folds it into
 *   the query RMSNorm gain): the scores are then exponentiated as 2^s without a multiply per score.
 *   block_n of g3c_gemm_bf16: 0 chooses (256 when N % 256 == 0, else 128 or 64); 512 is accepted and runs 256. */
int g3c_attn_fwd(const void* q, const void* k, const void* vt, void* o, int Lq, int Lk, int heads,
                 int ldq, int ldk, int ldo, int vt_chunk_len, float scale, void* stream);

/* The same operator on the layout of TE DotProductAttention(qkv_format="sbhd") — the reference's `attn_op` seam
 * (module/attention.py:136-139,288) — with V as given and any key count.
 *   q [Lq][batch*heads*128] (ld ldq), k and v [Lk][batch*heads*128] (ld ldk, ldv), o [Lq][batch*heads*128] (ld ldo):
 *   the token rows of [s, b, h, 128] tensors whose (b, h, d) block is contiguous, so batch x heads are one launch's
 *   heads.  Lq, Lk >= 1 (no multiple-of-128 rule: the keys past Lk in the last KV tile are masked).  Leading
 *   dimensions in elements, multiples of 8 and >= batch*heads*128; pointers 16-byte aligned; batch*heads <= 65535.
 *   scale as in g3c_attn_fwd (1/sqrt(128) for TE's default; ln 2 when Q already carries softmax_scale * log2(e)). */
int g3c_attn_fwd_sbhd(const void* q, const void* k, const void* v, void* o, int Lq, int Lk, int batch, int heads,
                      int ldq, int ldk, int ldv, int ldo, float scale, void* stream);

/* g3c_attn_fwd_sbhd that also stores, per (head, query row), the row's log-sum-exp for g3c_attn_bwd_sbhd:
 *   lse f32 [batch*heads][Lq] (head-major, 4-byte aligned, non-NULL) = m + log2(l) in log2 units of s * sl2, where
 *   s = q . k and sl2 = scale * log2(e) (exactly 1 for scale = ln 2), so softmax_j = 2^(s_j sl2 - lse).
 *   O is bitwise equal to g3c_attn_fwd_sbhd's. */
int g3c_attn_fwd_sbhd_lse(const void* q, const void* k, const void* v, void* o, float* lse, int Lq, int Lk, int batch,
                          int heads, int ldq, int ldk, int ldv, int ldo, float scale, void* stream);

/* Backward of g3c_attn_fwd_sbhd_lse: given dout = dL/dO, writes dq, dk, dv (bf16, the same sbhd token rows as q, k, v;
 * leading dimensions lddq, lddk, lddv).  With P = 2^(s sl2 - lse) and Delta_i = sum_d dout_id o_id (fp32, from the
 * bf16 o the forward returned):
 *   dV = P^T dout,  dS = P o (dout V^T - Delta),  dQ = scale * dS K,  dK = scale * dS^T Q
 * where scale is the natural-log softmax scale given to the forward (ln 2 under its log2 convention).  P and dS enter
 * the MMAs as bf16, the products accumulate in fp32.  delta_ws is a caller-supplied f32 [batch*heads][Lq] workspace
 * (overwritten with Delta); nothing is allocated.  Every gradient element has one writer (no atomics), so the result
 * is bitwise reproducible.  Three launches on `stream`: Delta, then dK/dV (one CTA per 128 keys of a head), then dQ
 * (one CTA per 128 queries of a head); S = q k^T and dout V^T are computed in both of the last two.  Sizes, strides
 * and alignment as in g3c_attn_fwd_sbhd, for all ten tensors; lse and delta_ws 4-byte aligned. */
int g3c_attn_bwd_sbhd(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                      float* delta_ws, void* dq, void* dk, void* dv, int Lq, int Lk, int batch, int heads, int ldq,
                      int ldk, int ldv, int ldo, int lddo, int lddq, int lddk, int lddv, float scale, void* stream);

/* Profiling aid: when a device buffer of 3*64*8 uint64 is registered, the next g3c_attn_fwd launches run a
 * traced build of the kernel in which CTA (0,0) records clock64() stamps per KV step j (first 64 steps): roles 1/2 =
 * the two consumer warpgroups; slots 0 turn acquired, 1 MMAs of the step issued (S_j and P_{j-1} V_{j-1}), 2 S_j
 * complete, 3 softmax of S_j done, 4 P_{j-1} V_{j-1} complete.  Step 0 has no P.V; step n_kv (the last P.V) stamps
 * slots 0, 1 and 4 only.  NULL switches tracing off. */
int g3c_attn_set_trace(unsigned long long* device_buffer);

/* x (f32 [L,D]) += pos (bf16, optional) ; y (bf16) = LayerNorm_eps(x) * (1 + scale) + shift
 * reference: module/blocks.py:339-341, :547-548 */
int g3c_ln_modulate(float* x, const void* pos_bf16, const float* shift, const float* scale,
                    void* y_bf16, int L, int D, float eps, void* stream);

/* g3c_ln_modulate with the modulated fp32 rows quantised as in g3c_quantize_rows_fp8: y_codes e4m3 [L,D], y_scales
 * [L] f32 (both 16-byte aligned, D a multiple of 16).  x is updated as by g3c_ln_modulate. */
int g3c_ln_modulate_fp8(float* x, const void* pos_bf16, const float* shift, const float* scale, void* y_codes,
                        float* y_scales, int L, int D, float eps, void* stream);

/* in-place per-head RMSNorm (eps, gamma[128]) and optional rotate-half RoPE (cos_sin [L,128] =
 * cos(angles[0:64]) | sin(angles[0:64])) on bf16 [L, heads*128]
 * reference: module/attention.py:274-279 */
int g3c_rmsnorm_rope(void* qk_bf16, int ld, int L, int heads, const float* gamma,
                     const float* cos_sin, float eps, void* stream);

typedef struct g3c_dit g3c_dit_t;

typedef struct g3c_dit_config {
  int model_channels;      /* 4096 (multiple of 128; heads = model_channels / 128) */
  int num_blocks;          /* 28, each FA-CA-MLP */
  int num_heads;           /* 32 (head_dim is fixed to 128) */
  int ffn_dim;             /* 16384 */
  int context_dim;         /* 1024 */
  int adaln_lora_dim;      /* 256 */
  int in_channels;         /* 81 = 16 latent + 1 condition mask + 64 pose, padding mask excluded */
  int out_channels;        /* 16 */
  int concat_padding_mask; /* 1 */
  int max_frames;          /* 128: rows of extra_pos_embedder.pos_emb_t */
  int max_h, max_w;        /* 120, 120: rows of pos_emb_h / pos_emb_w (max_img / patch) */
  float rope_h_ratio, rope_w_ratio, rope_t_ratio; /* 1, 1, 2 */
  int base_fps;            /* 24 */
} g3c_dit_config;

#define G3C_DTYPE_BF16 0
#define G3C_DTYPE_F32 1

/* The network VideoExtendGeneralDIT (reference: networks/general_dit_video_conditioned.py:58-217,
 * networks/general_dit.py:272-358,439-522).  Weights are registered under the reference's
 * state-dict key names (SURVEY.md §5) and are NOT copied: the caller keeps them alive. */
int g3c_dit_create(const g3c_dit_config* cfg, g3c_dit_t** out);
int g3c_dit_destroy(g3c_dit_t* h);
int g3c_dit_load(g3c_dit_t* h, const char* name, const void* ptr, const int64_t* shape, int ndim,
                 int dtype);

/* Context parallelism over the latent-frame axis (reference: general_dit.py:524-543 +
 * module/parallel.py:25-87).  nccl_unique_id: 128 bytes from g3c_nccl_unique_id on rank 0. */
int g3c_nccl_unique_id(void* out128);
/* nccl_unique_id == NULL selects the default mode: the K / V^T projections store their tiles straight into every
 * rank's buffers through NVLink peer memory (fused compute -> all-gather) and attention consumes the chunks as
 * their arrival flags are raised.  After g3c_dit_set_shape every rank exports the IPC handle of its region
 * (g3c_dit_cp_export, 64 bytes) and imports the handles of all ranks in rank order (g3c_dit_cp_import).
 * A non-NULL id selects the baseline mode: one in-place ncclAllGather of K and of V^T per layer. */
int g3c_dit_enable_cp(g3c_dit_t* h, const void* nccl_unique_id, int cp_rank, int cp_size);
int g3c_dit_cp_export(g3c_dit_t* h, void* out_handle64);
int g3c_dit_cp_import(g3c_dit_t* h, const void* handles, int n);
int g3c_dit_cp_mode(const g3c_dit_t* h); /* 0 = off, 1 = peer-memory (fused), 2 = NCCL */
int g3c_dit_disable_cp(g3c_dit_t* h);

/* Classifier-free-guidance parallelism (an extension; SURVEY.md §8e "CFG x CP hybrid"): the two forwards of a denoise
 * step (model_v2w.py:141-142) run on two ranks that hold the SAME latent slice — role 0 evaluates the conditional
 * branch, role 1 the unconditional one — and g3c_denoise_step exchanges the two network outputs through peer memory
 * (one copy-engine push of 16*T*H*W bf16 per rank and step, a system-scope flag, a one-warp wait kernel) before both
 * ranks apply the identical sampler update.  Composes with context parallelism (cfg 2 x cp N/2).  role < 0 disables.
 * After g3c_dit_set_shape: g3c_dit_cfg_export (64-byte IPC handle of this rank's exchange region) and
 * g3c_dit_cfg_import (the partner's handle). */
int g3c_dit_enable_cfg_parallel(g3c_dit_t* h, int role);
int g3c_dit_cfg_export(g3c_dit_t* h, void* out_handle64);
int g3c_dit_cfg_import(g3c_dit_t* h, const void* partner_handle64);

/* FP8 Linear mode (off by default).  on != 0: the eight large Linears of every block (self-attention to_q, to_k,
 * to_v, to_out; cross-attention to_q, to_out; MLP layer1, layer2) run on e4m3 operands with per-row scales: the
 * weights per output channel, the activations per token (g3c_quantize_rows_fp8 arithmetic).  Allocates the e4m3
 * weight copies now (about 235 MB per block of the 7B net, 6.6 GB for its 28 blocks); the next forward quantises them
 * from the registered bf16 weights, and again after every g3c_dit_load.  Frees the shape's workspace: call
 * g3c_dit_set_shape again (it then also allocates the fp8 activation buffers).  on = 0 frees the copies and returns to the bf16 forward.  Composes with context and CFG
 * parallelism (K and V^T stay bf16). */
int g3c_dit_set_linear_fp8(g3c_dit_t* h, int on);

/* Fix the token grid: T_local latent frames on this rank (of T_local*cp_size), latent H x W,
 * context length, fps.  Allocates the workspace and precomputes the abs-pos / RoPE tables. */
int g3c_dit_set_shape(g3c_dit_t* h, int T_local, int H_latent, int W_latent, int ctx_len, float fps);

/* net(x, timesteps, crossattn_emb, condition_video_input_mask, condition_video_pose, padding_mask)
 *   x [16,T,H,W], cond_mask [1,T,H,W], cond_pose [64,T,H,W] or NULL (zeros), padding_mask [H,W]
 *   (already at latent resolution) or NULL (zeros), ctx [ctx_len, context_dim]; all bf16, this
 *   rank's T slice.  out bf16 [16,T,H,W]. */
int g3c_dit_forward(g3c_dit_t* h, const void* x, const void* cond_mask, const void* cond_pose,
                    const void* padding_mask, float timestep, const void* ctx, void* out,
                    void* stream);

typedef struct g3c_step_args {
  const void* xt;        /* bf16 [16,T,H,W]                                                   */
  const void* gt_latent; /* bf16 [16,T,H,W]  condition.gt_latent                              */
  const float* aug_noise;/* f32  [16,T,H,W]  arch_invariant_rand(seed) slice (utils/misc.py:133) */
  const float* indicator;/* f32  [T]         condition_video_indicator                         */
  const void* cond_mask; /* bf16 [1,T,H,W]   condition_video_input_mask                        */
  const void* pose_cond; /* bf16 [64,T,H,W]  condition_video_pose (cond) ; uncond uses zeros   */
  const void* padding_mask; /* bf16 [H,W] or NULL */
  const void* ctx_cond;  /* bf16 [ctx_len, context_dim] */
  const void* ctx_uncond;
  float sigma, sigma_next, sigma_data, sigma_aug, guidance;
  void* xt_next;         /* bf16 [16,T,H,W] */
  const void* cond_mask_uncond; /* bf16 [1,T,H,W] uncondition.condition_video_input_mask (all zeros with
                                   add_input_frames_guidance, model_v2w.py:76-80) or NULL = same as cond_mask */
  void* net_output;      /* optional out, bf16 [16,T,H,W]: net_output_cond + guidance * (cond - uncond)
                            (model_v2w.py:143) before the indicator replacement; NULL = not stored */
} g3c_step_args;

/* One loop body of DiffusionV2WModel.generate_samples_from_batch (reference:
 * model/model_v2w.py:130-149 with _augment_noise_with_latent :201-247, _reverse_precondition_*
 * :249-259 and the EDM Euler step of diffusers 0.32.2): two DiT forwards + sampler glue. */
int g3c_denoise_step(g3c_dit_t* h, const g3c_step_args* a, void* stream);

/* Device-side timing by kernel category for bench.py's roofline: with profiling enabled every launch
 * of g3c_dit_forward is bracketed by CUDA events on the launching stream.  Categories:
 * 0 GEMM, 1 self-attention, 2 cross-attention, 3 elementwise, 4 comm, 5 B=1 vector ops.
 * g3c_dit_profile_read synchronises, sums elapsed ms / launch counts per category and resets. */
/* g3c_dit_profile_wait_ms: mean time per CTA and launch (ms, summed over the launches since the last read) that the
 * attention kernel's TMA warps spent polling a peer's K/V arrival flag under context parallelism — an upper bound of the
 * exposed exchange (the ring may still hold tiles for the MMA warp while the loader waits). */
int g3c_dit_profile_wait_ms(g3c_dit_t* h, float* ms);
#define G3C_PROFILE_CATEGORIES 6
int g3c_dit_profile(g3c_dit_t* h, int enable);
int g3c_dit_profile_read(g3c_dit_t* h, float* ms_by_category, int* launches_by_category, int ncat);

/* bytes of device workspace currently held by the handle */
int64_t g3c_dit_workspace_bytes(const g3c_dit_t* h);
/* number of kernels the last g3c_dit_forward enqueued (for bench.py's gpu_launches) */
int g3c_dit_last_launch_count(const g3c_dit_t* h);

/* ---- test hooks: read back what the forward derives from the weights, the shape and the timestep ---- */
/* The position tables of the current shape (g3c_dit_set_shape), built as a rank whose first latent frame is t0 builds
 * them: rope f32 [L,128] = cos | sin of the angles (t | h | w columns 22 | 21 | 21, token (t*Hp + h)*Wp + w), pos bf16
 * [L,D] the per-block abs-pos embedding.  The forward uses t0 = cp_rank * T_local.  t0 + T_local > max_frames is
 * G3C_EINVAL.  Leaves the forward's own tables untouched. */
int g3c_dit_read_tables(g3c_dit_t* h, int t0, float* rope, void* pos, void* stream);
/* The adaLN modulation vectors a forward at `timestep` uses: mods f32 [num_blocks*3][3D] (shift | scale | gate of
 * block i, sub-block j at row i*3 + j), modf f32 [2D] (final layer shift | scale).  Goes through the forward's
 * per-timestep cache (a forward right after at the same timestep reuses the vectors). */
int g3c_dit_read_modulation(g3c_dit_t* h, float timestep, float* mods, float* modf, void* stream);
/* The four bf16 [16,T,H,W] latents of the last g3c_denoise_step: x~ and x_in as sampler_pre wrote them, and the cond /
 * uncond network outputs sampler_post read (under CFG parallelism one of them is the partner's copy in the exchange
 * region).  G3C_ESTATE when no step has completed since the last g3c_dit_set_shape or g3c_dit_set_linear_fp8. */
int g3c_dit_read_step(g3c_dit_t* h, void* xtilde, void* xin, void* oc, void* ou, void* stream);
/* g3c_attn_fwd with the context-parallel chunk gate of the engine's peer-memory mode: the KV tiles are visited chunk by
 * chunk (chunks of vt_chunk_len keys, in K and in V^T) starting with chunk `first`, and the TMA loader of each CTA reads
 * a chunk c != first only once flags[c] >= seq (a system-scope acquire; flags is device memory of Lk / vt_chunk_len
 * uint32, typically raised by a copy after the chunk's data).  The local chunk `first` is never gated.  wait_ns (device,
 * optional): += ns each CTA's loader spent polling.  A flag that stays below seq traps the kernel after the peer timeout
 * (G3C_PEER_TIMEOUT_S, 600 s). */
int g3c_attn_fwd_gated(const void* q, const void* k, const void* vt, void* o, int Lq, int Lk, int heads,
                       int ldq, int ldk, int ldo, int vt_chunk_len, float scale,
                       const uint32_t* flags, uint32_t seq, int first, unsigned long long* wait_ns, void* stream);
/* The two peer-memory exchanges of the engine wired inside one process, so that every rank's handle can run on one
 * device, one after another.  g3c_dit_cp_region: this rank's context-parallel region (peer-memory mode, after
 * g3c_dit_set_shape) and its layout, as byte offsets from base: K of layer-parity set s (set = seq & 1 of the
 * self-attention layer) bf16 [cp][L][D] at off_k2[s], V^T bf16 [cp][D][L] at off_vt2[s], and uint32 arrival flags
 * [2][8] at off_flags (flags[s*8 + r] = seq of the last layer whose rank-r chunk landed in set s).  G3C_ESTATE without
 * such a region.  g3c_dit_cp_attach: g3c_dit_cp_import with the device pointers of the n = cp_size regions (from
 * g3c_dit_cp_region of each rank's handle, in rank order; entry cp_rank must be this handle's own region) instead of IPC
 * handles; G3C_ESTATE without a region or after g3c_dit_cp_import, G3C_EINVAL for a wrong n or entry.  Attached
 * pointers are never unmapped by this handle; the regions belong to their own handles, so every handle must be
 * synchronised before another one's region is freed. */
int g3c_dit_cp_region(g3c_dit_t* h, void** base, int64_t* off_k2, int64_t* off_vt2, int64_t* off_flags);
int g3c_dit_cp_attach(g3c_dit_t* h, const void* const* bases, int n);
/* The same for CFG parallelism: this rank's exchange region (2 slots of slot_bytes, the partner's output of step seq in
 * slot seq & 1, then uint32 flags [2] = seq of the output in each slot) and g3c_dit_cfg_import with the partner's region
 * pointer.  G3C_ESTATE without an exchange region (enable_cfg_parallel, then set_shape) or after g3c_dit_cfg_import. */
int g3c_dit_cfg_region(g3c_dit_t* h, void** base, int64_t* slot_bytes);
int g3c_dit_cfg_attach(g3c_dit_t* h, const void* partner_base);

#ifdef __cplusplus
}
#endif
#endif /* GEN3C_B200_H_ */
