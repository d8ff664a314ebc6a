/* aab200.h — C-ABI of libaab200.so: the sm_90a (Hopper) kernels of the animate-anything denoising hot path.
 *
 * The reference (alibaba/animate-anything) has no FFI of its own: its hot path is Python composing
 * `diffusers==0.24.0` leaf modules that bottom out in cuDNN / cuBLAS / SDPA calls.  Each entry point below is what a
 * binding for that path attaches to; the reference call site it replaces is cited as file:line (relative to the
 * reference tree; "diffusers:" = the leaf module of diffusers 0.24.0 invoked from that line).
 *
 * Conventions
 *   - plain pointers and sizes only (no torch types); all pointers are DEVICE pointers unless noted;
 *   - 16-bit tensors are fp16 or bf16 (`is_bf16`), activations are channels-last: rows ordered (b, t, y, x);
 *   - every call enqueues work on `stream` (a cudaStream_t passed as void*), allocates nothing, never synchronises;
 *   - return value: 0 ok, 1 bad argument, 2 CUDA launch error, 3 driver (TMA descriptor) error;
 *   - no ownership transfer; workspaces are provided by the caller.
 */
#ifndef AAB200_H
#define AAB200_H

#include "../animate_anything_b200/csrc/igemm.h" /* AabIgemmDesc, AAB_ACT_*, AAB_F_* */

#ifdef __cplusplus
extern "C" {
#endif

/* Implicit GEMM on wgmma (TMA-fed, register accumulators): Linear, conv3x3 (pad 1), conv3x3 stride 2, Conv3d (3,1,1),
 * batched Q.K^T / P.V.  Replaces cuBLAS/cuDNN under diffusers ResnetBlock2D.conv1/conv2/conv_shortcut/time_emb_proj,
 * TemporalConvLayer.conv1..4, Downsample2D.conv, Upsample2D.conv, Attention.to_q/k/v/to_out, GEGLU.proj (fused gate),
 * FeedForward.net[2], Transformer*.proj_in/out, AutoencoderKL convs
 * (models/unet_3d_blocks.py:262-306,425-476,564-591,660-709,794-819; models/unet_3d_condition_mask.py:137-168,264). */
int aab_igemm(const AabIgemmDesc* desc, void* stream);
/* 1 when this launch will write desc->colstats (per m-tile column sums of the rounded outputs: the statistics of the GroupNorm
 * that follows, diffusers ResnetBlock2D.norm2 / TemporalConvLayer / Transformer*Model.norm, taken in the producing GEMM's
 * epilogue), 0 when its epilogue cannot (direct-store variants, GEGLU) and the caller must run the statistics pass. */
int aab_igemm_emits_colstats(const AabIgemmDesc* desc);

/* Spatial self-attention / text cross-attention, head_dim 64, flash-style on wgmma
 * (diffusers AttnProcessor2_0 -> F.scaled_dot_product_attention; installed by train.py:124-138, blocks built at
 * models/unet_3d_blocks.py:287-296,446-456,681-691).  q: [nb*lq, ldq] with head h at columns q_col0 + 64 h;
 * k, v: columns k_col0 / v_col0 of kv [nb_kv*lk, ldkv]; query batch b reads kv batch b / kv_batch_div.
 * `is_bf16` bit 0: bfloat16 (else float16); bit 1: causal mask (key j visible to query i iff j <= i; needs lq == lk <= 128):
 * the CLIP text tower's self-attention (transformers CLIPAttention + causal_attention_mask), reached from
 * models/pipeline.py:136 `_encode_prompt`.
 * Rejected with 1: col0 + 64 heads past q_cols / kv_cols, (nb - 1) / kv_batch_div >= nb_kv, q / kv / out not 16-byte aligned,
 * row or batch strides not multiples of 8. */
int aab_flash_attn_d64(const void* q, long ldq, long q_batch_stride, int q_cols, int q_col0, const void* kv, long ldkv,
                       long kv_batch_stride, int kv_cols, int k_col0, int v_col0, void* out, long ld_out,
                       long out_batch_stride, int out_col0, int nb, int nb_kv, int kv_batch_div, int heads, int lq, int lk,
                       float scale, int is_bf16, void* stream);

/* The same attention for head_dim 80, bidirectional (no causal bit: `is_bf16` must be 0 or 1): the self-attention of the CLIP
 * ViT-H/14 image tower (transformers CLIPAttention, 16 heads x 80, 257 tokens) that the SVD pipelines' `_encode_image` runs
 * (models/pipeline.py:347,597).  Same arguments as aab_flash_attn_d64 with head h at columns col0 + 80 h; additionally
 * col0 + 80 heads must fit the given column counts, q / kv / out 16-byte aligned, batch strides multiples of 8. */
int aab_flash_attn_d80(const void* q, long ldq, long q_batch_stride, int q_cols, int q_col0, const void* kv, long ldkv,
                       long kv_batch_stride, int kv_cols, int k_col0, int v_col0, void* out, long ld_out,
                       long out_batch_stride, int out_col0, int nb, int nb_kv, int kv_batch_div, int heads, int lq, int lk,
                       float scale, int is_bf16, void* stream);

/* CLIP image preprocessing + patchify, the input of the CLIP image tower's patch-embedding GEMM (diffusers 0.24
 * StableVideoDiffusionPipeline._encode_image, models/pipeline.py:347,597; restated at train_svd.py:384-395).
 * src [b, 3, h, w] by element strides; src_type 0 = uint8 (a PIL image: strides h*w*3, 1, w*3, 3), 1 = float32, 2 = float16,
 * 3 = bfloat16.  uint8: x = u8/255, 2x - 1, separable Gaussian blur with reflect padding (taps_x [ks_x] along x first, then
 * taps_y [ks_y] along y; fp32, odd sizes), bicubic resize (align_corners) to out_size^2, (x + 1)/2, (x - mean)/std with
 * mean_std = fp32 [mean r, g, b, std r, g, b] -- all in fp32.  Float sources are the CLIP pixel values themselves
 * (h == w == out_size; taps and mean_std unused): rounding only.
 * out [b * (1 + (out_size/patch)^2), ld_out] 16-bit: row 0 of each image's block is zeros (the class-token slot), row 1 + p
 * is patch p (row-major grid) in the column order of patch_embedding.weight.flatten(1); columns >= 3 patch^2 are zeros. */
int aab_clip_image_prep(const void* src, int src_type, long sb, long sc, long sy, long sx, int b, int h, int w,
                        const float* taps_y, int ks_y, const float* taps_x, int ks_x, const float* mean_std, int out_size,
                        int patch, void* out, long ld_out, int is_bf16, void* stream);

/* Self-attention over the frame axis without the (b t) c h w -> (b h w) t c permutes
 * (diffusers TransformerTemporalModel.forward; models/unet_3d_blocks.py:299-306,459-467,694-701).
 * qkv rows ((b t) hw, ld); head h of q / k / v at columns col0 + 64 h.  is_bf16 bit 0: bf16 (else fp16); bit 1: the long-clip
 * kernel, t in 1..128 (without it t in 1..32, the v2 kernel).  Rejected with 1: any other is_bf16 bit, t outside the
 * selected range, b, hw or heads < 1, col0 + 64 heads > ld, 64 heads > ld_out, ld / ld_out / col0 not multiples of 8,
 * qkv / out not 16-byte aligned. */
int aab_temporal_attn_d64(const void* qkv, long ld, int q_col0, int k_col0, int v_col0, void* out, long ld_out, int b, int t,
                          int hw, int heads, float scale, int is_bf16, void* stream);

/* GroupNorm (+ optional SiLU) over `rows` x (C/groups) per (sample, group); x2 != NULL = virtual channel concat
 * (torch.cat at models/unet_3d_blocks.py:731,828).  Deterministic reductions.  `workspace` must hold
 * aab_groupnorm_workspace_bytes(...) bytes, zero-initialised once (the kernel leaves it reusable).
 * (diffusers ResnetBlock2D.norm1/norm2, TemporalConvLayer GroupNorms, Transformer*.norm, conv_norm_out :514-516).
 * Returns 1 before any launch when: x1, y or workspace is NULL, or x2 when c2 > 0; x1, y or (c2 > 0) x2 is not 16-byte
 * aligned; gamma or beta is NULL; c1, c2, ld1, ld2 or ldy is not a multiple of 8; groups is outside 1..256 or does not
 * divide c1 + c2; samples < 1, samples > 4096 or rows < 1. */
long aab_groupnorm_workspace_bytes(long samples, long rows, int c, int groups);
int aab_groupnorm(const void* x1, long ld1, int c1, const void* x2, long ld2, int c2, long samples, long rows, int groups,
                  const float* gamma, const float* beta, float eps, int silu, void* y, long ldy, void* workspace,
                  int is_bf16, void* stream);
/* Same GroupNorm with the statistics pass replaced by the column sums the PRODUCING implicit GEMM wrote (AabIgemmDesc.colstats,
 * [rows_total / 128][c][2] fp32): a tiny finalize kernel + the apply pass.  rows % 128 == 0 (every 128-row tile inside one sample).
 * Same rejections as aab_groupnorm, plus a NULL colstats1 (or colstats2 when c2 > 0) and rows % 128 != 0. */
int aab_groupnorm_colstats(const void* x1, long ld1, int c1, const float* colstats1, const void* x2, long ld2, int c2,
                           const float* colstats2, long samples, long rows, int groups, const float* gamma, const float* beta,
                           float eps, int silu, void* y, long ldy, void* workspace, int is_bf16, void* stream);

/* LayerNorm over C per row (diffusers BasicTransformerBlock.norm1/2/3).  Returns 1 before any launch when: x, y, gamma or
 * beta is NULL or not 16-byte aligned; c is not a multiple of 8 or above 2048; ldx or ldy is not a multiple of 8; rows < 1. */
int aab_layernorm(const void* x, long ldx, void* y, long ldy, const float* gamma, const float* beta, long rows, int c,
                  float eps, int is_bf16, void* stream);

/* fp32 scores -> 16-bit probabilities, row softmax (AutoencoderKL mid-block attention, upcast_softmax).  The probability
 * rows are ldp wide: columns l..ldp-1 are written as +0 (K padding of the following P.V GEMM).  Returns 1 before any launch
 * when: s or p is NULL; rows < 1; l < 1; lds < l or ldp < l. */
int aab_softmax_rows(const float* s, long lds, void* p, long ldp, long rows, int l, int is_bf16, void* stream);

/* UNet boundary: frame concat + mask channel + (b f) permute in one pass (models/unet_3d_condition_mask.py:376,424-431)
 * and its inverse with frame 0 dropped (:521-522).  Strides are in elements, order (b, c, f, y, x). */
int aab_unet_in_assemble(const void* sample, const long* s_strides, const void* cond, const long* c_strides,
                         const void* mask, const long* m_strides, int mask_batch, void* out, int b, int t, int h, int w,
                         int is_bf16, void* stream);
int aab_unet_out_finalize(const float* y, int ldc, void* out, int b, int t, int h, int w, int is_bf16, void* stream);

/* Sinusoidal timestep / motion embedding, flip_sin_to_cos=True, shift 0 (models/unet_3d_condition_mask.py:146,156,408,415). */
int aab_timestep_embed(const float* t, int t_count, void* out, int b, int dim, int is_bf16, void* stream);

/* CLIP text embeddings (transformers CLIPTextEmbeddings.forward; models/pipeline.py:136 _encode_prompt):
 * out[r, :] = tok_emb[ids[r], :] + pos_emb[r % seq_len, :]; ids int64 [rows], 16-bit tables, c % 8 == 0. */
int aab_embed_tokens(const long long* ids, const void* tok_emb, const void* pos_emb, void* out, long rows, int seq_len,
                     int c, int vocab, int is_bf16, void* stream);

/* SVD path (config 4; models/pipeline.py:223-466 driving diffusers' UNetSpatioTemporalConditionModel):
 * 9-channel UNet input [N, C<=16, H, W] -> channels-last padded to 16 (:422 cat([mask, latents, image_latents], dim=2));
 * out[r] = x[r] + vec[idx(r)], out may alias x (single-key cross-attention = per-sample vector; frame position embedding; mode 1 = the
 * (h*w, batch)-ordered time_context quirk of TransformerSpatioTemporalModel.forward);
 * AlphaBlender out = a*x + b*y for fp32 a, b: each product and the sum rounded to 16 bits, as torch computes `a * x + b * y`
 * for Python-float a, b (the caller passes alpha = sigmoid(mix_factor) in fp32; the stock 16-bit AlphaBlender would first
 * round alpha to the model dtype); conv_out -> [B, F, 4, H, W]. */
int aab_image_to_nhwc16(const void* img, long sn, long sc, long sy, long sx, void* out, long n, int c, int h, int w,
                        int is_bf16, void* stream);
int aab_add_rowvec(const void* x, long ldx, void* out, long ldo, const float* vec, long ldv, long rows, int cols,
                   long rows_per_vec, int mod, int mode, int mod2, int is_bf16, void* stream);
int aab_axpby(const void* x, const void* y, void* out, long n_elems, float a, float b, int is_bf16, void* stream);
int aab_svd_out_finalize(const float* y, int ldc, void* out, long bf, int h, int w, int is_bf16, void* stream);
/* SVD loop boundary kernels (models/pipeline.py:416-439): scale_model_input + CFG duplication + 9-channel cat in one pass;
 * per-frame guidance + Euler step (v-prediction) in one pass.  gs: fp32 [f] = linspace(min, max, f) (:405-408).
 * Guidance: v = v_u + g (v_c - v_u) with the 16-bit roundings of torch (pred, gs and every op rounded); the Euler step is
 * then fp32 throughout, including v * (-sigma / sqrt(sigma^2 + 1)), which diffusers would round to 16 bits for a 16-bit v. */
int aab_svd_in_assemble(const void* x, const void* img_lat, const void* mask, float inv_scale, void* out, int b, int f, int h,
                        int w, int cfg, int is_bf16, void* stream);
/* General form for TextStableVideoDiffusionPipeline.__call__ (models/pipeline.py:596-606 conditioning latents per frame, either
 * `_encode_vae_image` output (zero_uncond = 1) or the caller's `condition_latent` duplicated for both halves; :590 mask
 * `torch.cat([mask] * 2)`, per frame; :654-661 cat([mask, x, cond], dim=2) or, for an 8-channel UNet (mask == NULL), cat([x, cond])).
 * Strides in elements; 0 = broadcast. */
int aab_svd_in_assemble_frames(const void* x, const void* cond, long cond_half_stride, long cond_batch_stride,
                               long cond_frame_stride, int zero_uncond, const void* mask, long mask_batch_stride,
                               long mask_frame_stride, float inv_scale, void* out, int b, int f, int h, int w, int cfg, int is_bf16,
                               void* stream);
int aab_svd_cfg_euler_step(const float* pred, int ldc, int cfg, const float* gs, const void* x, void* x_out, float sigma,
                           float sigma_next, int b, int f, int h, int w, int is_bf16, void* stream);

/* Unfused fallbacks / helpers: GEGLU gate (diffusers GEGLU.forward), nearest 2x upsample (Upsample2D), copies. */
int aab_geglu(const void* x, long ldx, void* out, long ldo, long rows, int nh, int is_bf16, void* stream);
int aab_upsample2x(const void* x, void* y, long n, int h, int w, int c, void* stream);
/* Upsample2D with output_size (F.interpolate(size=, mode="nearest")) and bottom/right zero padding to even sizes for the
 * stride-2 conv: the latent-size-not-a-multiple-of-8 path, models/unet_3d_condition_mask.py:377-383,486-491. */
int aab_upsample_nearest(const void* x, void* y, long n, int h, int w, int oh, int ow, int c, void* stream);
int aab_pad_br(const void* x, void* y, long n, int h, int w, int ph, int pw, int c, void* stream);
int aab_copy2d(const void* src, long lds, void* dst, long ldd, long rows, int cols, void* stream);
/* dst[0:bytes] = dst[bytes:2*bytes] = src: batch duplication for the shared CFG prefix (torch.cat([latents] * 2), models/pipeline.py:165) */
int aab_dup_rows(const void* src, void* dst, long bytes, void* stream);
int aab_transpose(const void* src, long lds, long src_batch, void* dst, int nb, int rows, int cols, int ldd, void* stream);

/* Classifier-free guidance + scheduler step + layout shuffles in one kernel (models/pipeline.py:180-192):
 * eps = e_u + g (e_t - e_u); x0 = k0 x + k1 eps; x' = k2 x + k3 eps + k4 x0 + k5 x0_prev.  coef: device [steps][6]. */
int aab_cfg_scheduler_step(const float* eps, int ldc, int cfg, float guidance, const void* x, void* x_out, float* x0_hist,
                           const float* coef, const int* step_idx, int n, int f, int h, int w, int is_bf16, void* stream);

/* VAE boundary ops (utils/common.py:12-20; diffusers decode_latents called at models/pipeline.py:200). */
int aab_image_to_nhwc8(const void* img, long sn, long sc, long sy, long sx, void* out, long n, int c, int h, int w,
                       int is_bf16, void* stream);
int aab_vae_enc_finalize(const void* mom, int ldm, const float* wq, const float* bq, float scale, void* out, int b, int f,
                         int h, int w, int is_bf16, void* stream);
int aab_vae_dec_in(const void* lat, float inv_scale, const float* wp, const float* bp, void* out, int b, int f, int h, int w,
                   int is_bf16, void* stream);
int aab_vae_dec_finalize(const float* y, int ldc, float* out, int b, int f, int h, int w, int is_bf16, void* stream);
/* decoder tail fused with diffusers tensor2vid (models/pipeline.py:205): uint8 frames [f, h, b*w, 3].  is_bf16 bit 0: bf16
 * model; bit 1: round the scaled value half to even (the SVD pipelines' postprocess) instead of truncating; any other bit
 * returns 1 before a launch. */
int aab_vae_dec_finalize_u8(const float* y, int ldc, void* out, int b, int f, int h, int w, int is_bf16, void* stream);

/* Forward-diffuse the image latent to the first kept timestep: out = sa * repeat(x0 over f) + sb * noise with torch's
 * per-op 16-bit roundings (utils/common.py:32-48 DDPM_forward_timesteps -> DDPMScheduler.add_noise; :22-30 DDPM_forward).
 * x0 [bc, fx, hw] with fx in {1, f}; noise, out [bc, f, hw]. */
int aab_add_noise(const void* x0, const void* noise, float sa, float sb, void* out, long bc, int f, int fx, long hw,
                  int is_bf16, void* stream);

/* Transparent-video branch (SURVEY row f4): models/pipeline_stage2.py:171-337 MaskedLatentToVideoPipeline.__call__ +
 * models/layerdiffuse_VAE.py:44-177 UNet384 (the alpha decoder; its convolutions / GroupNorm(4) / head-dim-8 attention run on
 * aab_igemm / aab_groupnorm / aab_flash_attn_d64 with zero-padded heads).
 * :305 `video_tensor.permute(0,2,1,3,4).reshape(b*f,c,h,w).to(dtype)`: fp32 video [b, c<=8, f, h, w] (strides in elements)
 *      -> channels-last 16-bit [b*f, h, w, 8], zero padded;
 * :311-324 RGBA post-processing of the decoder's conv_out result y [pixels, ldc] (fp32, channels r g b alpha) -> uint8
 *      [pixels, 4]: alpha*255 thresholded at 127 to {0,255}, (fg+1)*127.5 with torch's 16-bit roundings, clip, truncate;
 * pad_cols: dst [rows, dst_cols] = src [rows, cols] | zeros (32-channel activations in front of a stride-2 conv, whose
 *      space-to-depth K block is 64 channels wide). */
int aab_video_f32_to_nhwc8(const float* video, long sb, long sc, long sf, long sy, long sx, void* out, int b, int c, int f,
                           int h, int w, int is_bf16, void* stream);
int aab_rgba_finalize_u8(const float* y, int ldc, void* out, long pixels, int is_bf16, void* stream);
int aab_pad_cols(const void* src, long lds, void* dst, long rows, int cols, int dst_cols, void* stream);

int aab_cast_f32(const float* x, void* y, long n, int is_bf16, void* stream);
int aab_num_sms(void);

#ifdef __cplusplus
}
#endif
#endif /* AAB200_H */
