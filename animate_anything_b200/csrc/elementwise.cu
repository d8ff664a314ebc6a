// Small HBM/launch-bound kernels that sit between the implicit GEMMs: layout assembly at the model boundaries
// (reference layouts are [b, c, f, h, w]; internal layout is channels-last [b, t, h, w, c]), sinusoidal timestep
// embedding, GEGLU (unfused fallback), nearest 2x upsample, the fused classifier-free-guidance + scheduler step, and
// the VAE boundary ops.  Each cites the reference line it replaces.
#include "common.cuh"

namespace aab {

// ------------------------------------------------------------------------------------------------
// UNet input assembly  (models/unet_3d_condition_mask.py:376 cat(condition_latent, sample) on frames;
// :424-427 mask repeat + cat on channels + permute to (b f) c h w).  Output [B, T, H, W, 8] 16-bit, channel order
// (mask, c0..c3, 0, 0, 0) when mask != NULL, else (c0..c3, 0...).
struct Strides5 { long b, c, f, y, x; };

template <bool BF16>
__global__ void unet_in_assemble_kernel(const void* __restrict__ sample, Strides5 ss, const void* __restrict__ cond,
                                        Strides5 cs, const void* __restrict__ mask, Strides5 ms, int mask_batch,
                                        void* __restrict__ out, int B, int T, int H, int W) {
  const long total = static_cast<long>(B) * T * H * W;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = i % W;
  long r = i / W;
  const int y = r % H;
  r /= H;
  const int t = r % T;
  const int b = r / T;
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = 0.f;
  int o = 0;
  if (mask != nullptr) {
    v[0] = load_elem(mask, (b % mask_batch) * ms.b + y * ms.y + x * ms.x, BF16);
    o = 1;
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    v[o + c] = (t == 0) ? load_elem(cond, b * cs.b + c * cs.c + y * cs.y + x * cs.x, BF16)
                        : load_elem(sample, b * ss.b + c * ss.c + (t - 1) * ss.f + y * ss.y + x * ss.x, BF16);
  }
  uint4 u;
  u.x = pack2(v[0], v[1], BF16);
  u.y = pack2(v[2], v[3], BF16);
  u.z = pack2(v[4], v[5], BF16);
  u.w = pack2(v[6], v[7], BF16);
  reinterpret_cast<uint4*>(out)[i] = u;
}

// UNet output: conv_out result [B, T, H, W, ldc] (fp32, 4 valid channels) -> [B, 4, T-1, H, W] 16-bit, frame 0 dropped
// (models/unet_3d_condition_mask.py:521-522).
template <bool BF16>
__global__ void unet_out_finalize_kernel(const float* __restrict__ y, int ldc, void* __restrict__ out, int B, int T,
                                         int H, int W) {
  const int F = T - 1;
  const long total = static_cast<long>(B) * 4 * F * H * W;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = i % W;
  long r = i / W;
  const int yy = r % H;
  r /= H;
  const int f = r % F;
  r /= F;
  const int c = r % 4;
  const int b = r / 4;
  const float v = y[(((static_cast<long>(b) * T + f + 1) * H + yy) * W + x) * ldc + c];
  store_elem(out, i, v, BF16);
}

// ------------------------------------------------------------------------------------------------
// Sinusoidal embedding, diffusers Timesteps(num_channels, flip_sin_to_cos=True, downscale_freq_shift=0)
// (models/unet_3d_condition_mask.py:146,156,408,415): out[b, j] = cos(t * w_j) for j < half, sin(t * w_{j-half}) after.
template <bool BF16>
__global__ void timestep_embed_kernel(const float* __restrict__ t, int t_count, void* __restrict__ out, int B, int dim) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * dim) return;
  const int b = i / dim;
  const int j = i % dim;
  const int half = dim / 2;
  const int k = (j < half) ? j : j - half;
  const float tv = t[b % t_count];        // t_count in {1, B, B/2 (CFG pair: [uncond..., text...])}
  const float freq = expf(-9.210340371976184f * static_cast<float>(k) / static_cast<float>(half));
  const float a = tv * freq;
  const float v = (j < half) ? cosf(a) : sinf(a);
  store_elem(out, i, v, BF16);
}

// CLIP text embeddings (transformers CLIPTextEmbeddings.forward, reached from models/pipeline.py:136 _encode_prompt):
// out[r, :] = token_embedding[ids[r], :] + position_embedding[r % L, :], one 16-byte octet per thread.
template <bool BF16>
__global__ void embed_tokens_kernel(const long long* __restrict__ ids, const uint4* __restrict__ tok,
                                    const uint4* __restrict__ pos, uint4* __restrict__ out, long rows, int L, int V8,
                                    int vocab) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= rows * V8) return;
  const long r = i / V8;
  const int o = static_cast<int>(i % V8);
  long long id = ids[r];
  if (id < 0) id = 0;
  if (id >= vocab) id = vocab - 1;
  const uint4 a = __ldg(tok + id * V8 + o);
  const uint4 b = __ldg(pos + (r % L) * V8 + o);
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
  const uint32_t bw[4] = {b.x, b.y, b.z, b.w};
  uint32_t w[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 fa = unpack2(aw[e], BF16);
    const float2 fb = unpack2(bw[e], BF16);
    w[e] = pack2(fa.x + fb.x, fa.y + fb.y, BF16);
  }
  out[i] = make_uint4(w[0], w[1], w[2], w[3]);
}

// GEGLU fallback: out[r, j] = x[r, j] * gelu(x[r, nh + j])   (diffusers GEGLU.forward)
template <bool BF16>
__global__ void geglu_kernel(const void* __restrict__ x, long ldx, void* __restrict__ out, long ldo, long rows, int nh) {
  const long total = rows * (nh / 8);
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long r = i / (nh / 8);
  const int c = (i % (nh / 8)) * 8;
  const uint4 a = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(x) + (r * ldx + c) * 2);
  const uint4 g = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(x) + (r * ldx + nh + c) * 2);
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
  const uint32_t gw[4] = {g.x, g.y, g.z, g.w};
  uint32_t o[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 af = unpack2(aw[e], BF16);
    const float2 gf = unpack2(gw[e], BF16);
    o[e] = pack2(af.x * gelu_erf_f(gf.x), af.y * gelu_erf_f(gf.y), BF16);
  }
  *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(out) + (r * ldo + c) * 2) = make_uint4(o[0], o[1], o[2], o[3]);
}

// nearest-neighbour 2x upsample on channels-last [N, H, W, C] -> [N, 2H, 2W, C]  (diffusers Upsample2D, F.interpolate)
__global__ void upsample2x_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, long n, int H, int W, int V) {
  const long total = n * 2 * H * 2 * W * V;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int v = i % V;
  long r = i / V;
  const int ox = r % (2 * W);
  r /= (2 * W);
  const int oy = r % (2 * H);
  const long nn = r / (2 * H);
  y[i] = __ldg(&x[((nn * H + (oy >> 1)) * W + (ox >> 1)) * V + v]);
}

// nearest-neighbour resize to an arbitrary output size (diffusers Upsample2D with `output_size`, i.e.
// F.interpolate(x, size=(OH, OW), mode="nearest"): src = min(floor(dst * (in / out)), in - 1) with the scale in fp32, as ATen
// computes it).  Reached when the latent size is not a multiple of 8 (models/unet_3d_condition_mask.py:377-383,486-491).
__global__ void upsample_nearest_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, long n, int H, int W, int OH,
                                        int OW, int V) {
  const long total = n * OH * OW * V;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int v = i % V;
  long r = i / V;
  const int ox = r % OW;
  r /= OW;
  const int oy = r % OH;
  const long nn = r / OH;
  const float sh = static_cast<float>(H) / static_cast<float>(OH);
  const float sw = static_cast<float>(W) / static_cast<float>(OW);
  int sy = static_cast<int>(floorf(static_cast<float>(oy) * sh));
  int sx = static_cast<int>(floorf(static_cast<float>(ox) * sw));
  sy = sy < H - 1 ? sy : H - 1;
  sx = sx < W - 1 ? sx : W - 1;
  y[i] = __ldg(&x[((nn * H + sy) * W + sx) * V + v]);
}

// zero padding at the bottom / right: [N, H, W, C] -> [N, H + ph, W + pw, C].  Makes an odd-sized activation even so that the
// stride-2 convolution can use its space-to-depth view; the added zeros are exactly the conv's own zero padding.
__global__ void pad_br_kernel(const uint4* __restrict__ x, uint4* __restrict__ y, long n, int H, int W, int PH, int PW, int V) {
  const long total = n * PH * PW * V;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int v = i % V;
  long r = i / V;
  const int ox = r % PW;
  r /= PW;
  const int oy = r % PH;
  const long nn = r / PH;
  uint4 val = make_uint4(0, 0, 0, 0);
  if (oy < H && ox < W) val = __ldg(&x[((nn * H + oy) * W + ox) * V + v]);
  y[i] = val;
}

// strided 16-bit copy of a [rows, cols] block (used for K/V^T staging and channel concat fallbacks)
__global__ void copy2d_kernel(const uint16_t* __restrict__ src, long lds, uint16_t* __restrict__ dst, long ldd, long rows,
                              int cols) {
  const long total = rows * cols;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long r = i / cols;
  const int c = i % cols;
  dst[r * ldd + c] = src[r * lds + c];
}

// same copy in 16-byte units (cols, both row strides and both base addresses multiples of 8 elements)
__global__ void copy2d_v8_kernel(const uint4* __restrict__ src, long lds8, uint4* __restrict__ dst, long ldd8, long rows, int cols8) {
  const long total = rows * cols8;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long r = i / cols8;
  const int c = static_cast<int>(i % cols8);
  dst[r * ldd8 + c] = src[r * lds8 + c];
}

// out[0:n16] = out[n16:2*n16] = src (16-byte units): duplicates the rows of the unconditional half for the text half when
// the CFG pair shares its prefix (see UNet3DConditionModel.forward, `_cfg_shared_prefix`)
__global__ void dup_rows_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, long n16) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n16) return;
  const uint4 v = __ldg(src + i);
  dst[i] = v;
  dst[i + n16] = v;
}

// batched transpose: src [nb][rows][lds] (cols used) -> dst [nb][cols][ldd]; dst columns rows..ldd-1 are zero-filled
// (ldd = rows rounded up to a multiple of 8 so that the result can be a TMA operand when rows % 8 != 0)
__global__ void transpose_kernel(const uint16_t* __restrict__ src, long lds, long src_batch, uint16_t* __restrict__ dst,
                                 int rows, int cols, int ldd) {
  __shared__ uint16_t tile[32][33];
  const int b = blockIdx.z;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int r = r0 + j, c = c0 + threadIdx.x;
    if (r < rows && c < cols) tile[j][threadIdx.x] = src[b * src_batch + static_cast<long>(r) * lds + c];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (r < ldd && c < cols) dst[(static_cast<long>(b) * cols + c) * ldd + r] = (r < rows) ? tile[threadIdx.x][j] : uint16_t(0);
  }
}

// ------------------------------------------------------------------------------------------------
// Fused classifier-free guidance + scheduler step + layout shuffles (models/pipeline.py:180-192).
//   eps  = e_u + g * (e_t - e_u)            (or e directly when no CFG)
//   x0   = k0 * x + k1 * eps
//   x'   = k2 * x + k3 * eps + k4 * x0 + k5 * x0_prev ;  x0_prev <- x0
// covers DDIM (k2, k3) and DPM-Solver++(2M) (k0, k1, k2, k4, k5).  `coef` is a device table [steps][6]; the row is
// selected by *step_idx (device) so the same captured CUDA graph serves every step.
// eps comes straight from conv_out: fp32 [Bu, T, H, W, ldc]; latents are [n, 4, F, H, W] 16-bit.
template <bool BF16>
__global__ void cfg_step_kernel(const float* __restrict__ eps, int ldc, int cfg, float guidance,
                                const void* __restrict__ x, void* __restrict__ x_out, float* __restrict__ x0_hist,
                                const float* __restrict__ coef, const int* __restrict__ step_idx, int n, int F, int H,
                                int W) {
  const long total = static_cast<long>(n) * 4 * F * H * W;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float* k = coef + (step_idx ? *step_idx : 0) * 6;
  const int xw = i % W;
  long r = i / W;
  const int y = r % H;
  r /= H;
  const int f = r % F;
  r /= F;
  const int c = r % 4;
  const int b = r / 4;
  const int T = F + 1;
  const long pix = ((static_cast<long>(f + 1)) * H + y) * W + xw;
  const long per_b = static_cast<long>(T) * H * W;
  float e;
  if (cfg) {
    const float eu = eps[(b * per_b + pix) * ldc + c];
    const float et = eps[((b + n) * per_b + pix) * ldc + c];
    e = eu + guidance * (et - eu);
  } else {
    e = eps[(b * per_b + pix) * ldc + c];
  }
  const float xv = load_elem(x, i, BF16);
  const float x0 = k[0] * xv + k[1] * e;
  float xn = k[2] * xv + k[3] * e + k[4] * x0;
  if (x0_hist != nullptr) {
    xn += k[5] * x0_hist[i];
    x0_hist[i] = x0;
  }
  store_elem(x_out, i, xn, BF16);
}

// ------------------------------------------------------------------------------------------------ VAE boundary ops
// image [N, 3, H, W] (strided, 16-bit) -> channels-last [N, H, W, 8] zero padded   (AutoencoderKL.encode input)
template <bool BF16>
__global__ void image_to_nhwc8_kernel(const void* __restrict__ img, long sn, long sc, long sy, long sx,
                                      void* __restrict__ out, long N, int C, int H, int W) {
  const long total = N * H * W;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = i % W;
  long r = i / W;
  const int y = r % H;
  const long nn = r / H;
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = (j < C) ? load_elem(img, nn * sn + j * sc + y * sy + x * sx, BF16) : 0.f;
  reinterpret_cast<uint4*>(out)[i] =
      make_uint4(pack2(v[0], v[1], BF16), pack2(v[2], v[3], BF16), pack2(v[4], v[5], BF16), pack2(v[6], v[7], BF16));
}

// SVD UNet input (models/pipeline.py:422 cat([mask, latents, image_latents], dim=2) -> conv_in of
// UNetSpatioTemporalConditionModel): x [N, C, H, W] (strided, 16-bit, C <= 16) -> channels-last [N, H, W, 16] zero padded
template <bool BF16>
__global__ void image_to_nhwc16_kernel(const void* __restrict__ img, long sn, long sc, long sy, long sx,
                                       void* __restrict__ out, long N, int C, int H, int W) {
  const long total = N * H * W * 2;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int half = i & 1;
  long r = i >> 1;
  const int x = r % W;
  r /= W;
  const int y = r % H;
  const long nn = r / H;
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = half * 8 + j;
    v[j] = (c < C) ? load_elem(img, nn * sn + c * sc + y * sy + x * sx, BF16) : 0.f;
  }
  reinterpret_cast<uint4*>(out)[i] =
      make_uint4(pack2(v[0], v[1], BF16), pack2(v[2], v[3], BF16), pack2(v[4], v[5], BF16), pack2(v[6], v[7], BF16));
}

// out[r, :] = x[r, :] + vec[idx(r), :]   (out may alias x; 16-bit x / out, fp32 vec rows of `cols` values)
//   mode 0: idx = (r / rows_per_vec) % mod   -- per-sample / per-frame vectors: the single-key cross-attention of the SVD
//           transformer blocks (one image embedding per sample => softmax over ONE key is 1, the attention output is
//           to_out(to_v(context)) for every token) and the frame position embedding of TransformerSpatioTemporalModel
//   mode 1: rows are (b, f, s) with S = rows_per_vec, F = mod2; idx = (b * S + s) % mod -- the (h*w, batch)-ordered
//           `time_context` of diffusers' TransformerSpatioTemporalModel.forward read by (batch, h*w)-ordered tokens
template <bool BF16>
__global__ void add_rowvec_kernel(const void* x, long ldx, void* out, long ldo, const float* __restrict__ vec, long ldv, long rows,
                                  int cols, long rows_per_vec, int mod, int mode, int mod2) {
  const int V = cols >> 3;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= rows * V) return;
  const long r = i / V;
  const int c = static_cast<int>(i % V) * 8;
  long idx;
  if (mode == 0) {
    idx = (r / rows_per_vec) % mod;
  } else {
    const long s = r % rows_per_vec;
    const long b = r / (rows_per_vec * mod2);
    idx = (b * rows_per_vec + s) % mod;
  }
  const uint4 u = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(x) + (r * ldx + c) * 2);
  uint4* px = reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(out) + (r * ldo + c) * 2);
  const float4 a = __ldg(reinterpret_cast<const float4*>(vec + idx * ldv + c));
  const float4 b4 = __ldg(reinterpret_cast<const float4*>(vec + idx * ldv + c) + 1);
  const float add[8] = {a.x, a.y, a.z, a.w, b4.x, b4.y, b4.z, b4.w};
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
  uint32_t o[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 f = unpack2(w[e], BF16);
    o[e] = pack2(f.x + add[2 * e], f.y + add[2 * e + 1], BF16);
  }
  *px = make_uint4(o[0], o[1], o[2], o[3]);
}

// out = a * x + b * y for fp32 a, b with each product and the sum rounded to 16 bits: torch's `a * x + b * y` for Python-float
// a, b on 16-bit tensors (diffusers AlphaBlender.forward: `alpha * x_spatial + (1 - alpha) * x_temporal`).  The coefficients
// are used as given: the caller passes sigmoid(mix_factor) in fp32, where the stock 16-bit module rounds alpha to the model
// dtype first and computes 1 - alpha in that dtype.
template <bool BF16>
__global__ void axpby_kernel(const uint4* __restrict__ x, const uint4* __restrict__ y, uint4* __restrict__ out, long n16,
                             float a, float b) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n16) return;
  const uint4 ux = __ldg(x + i), uy = __ldg(y + i);
  const uint32_t wx[4] = {ux.x, ux.y, ux.z, ux.w};
  const uint32_t wy[4] = {uy.x, uy.y, uy.z, uy.w};
  uint32_t o[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 fx = unpack2(wx[e], BF16);
    const float2 fy = unpack2(wy[e], BF16);
    o[e] = pack2(round16(a * fx.x, BF16) + round16(b * fy.x, BF16), round16(a * fx.y, BF16) + round16(b * fy.y, BF16), BF16);
  }
  out[i] = make_uint4(o[0], o[1], o[2], o[3]);
}

// conv_out result [B*F*H*W, ldc] fp32 (4 valid channels) -> [B, F, 4, H, W] 16-bit
// (UNetSpatioTemporalConditionModel.forward tail: sample.reshape(batch, frames, C, H, W))
template <bool BF16>
__global__ void svd_out_finalize_kernel(const float* __restrict__ y, int ldc, void* __restrict__ out, long BF, int H, int W) {
  const long total = BF * 4 * H * W;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = i % W;
  long r = i / W;
  const int yy = r % H;
  r /= H;
  const int c = r % 4;
  const long n = r / 4;
  store_elem(out, i, y[((n * H + yy) * W + x) * ldc + c], BF16);
}

// SVD loop, input side (models/pipeline.py:418-422): latent_model_input = cat([latents] * 2) / sqrt(sigma^2 + 1)
// (EulerDiscreteScheduler.scale_model_input), then cat([mask, latent_model_input, image_latents], dim=2) with the
// unconditional half seeing ZERO image latents (_encode_vae_image) -> channels-last [2B*F, h, w, 16] (9 used).
// x [B, F, 4, h, w]; img_lat [B, 4, h, w] (positive half); mask [h, w]; `cfg` = 1: two halves, 0: one.
// General form (TextStableVideoDiffusionPipeline, models/pipeline.py:596-606,654-661): the conditioning latents may differ per frame
// and per CFG half (element strides cond_hs / cond_bs / cond_fs; 0 = broadcast), the unconditional half sees zeros only when they
// come from `_encode_vae_image` (zero_uncond), the mask is per frame ([B, F, h, w], strides mask_bs / mask_fs) or absent (8-channel
// UNet: cat([x, cond], dim=2)).
template <bool BF16>
__global__ void svd_in_assemble_kernel(const void* __restrict__ x, const void* __restrict__ img_lat, const void* __restrict__ mask,
                                       float inv_scale, void* __restrict__ out, int B, int F, int H, int W, int cfg, long cond_hs,
                                       long cond_bs, long cond_fs, int zero_uncond, long mask_bs, long mask_fs) {
  const long per_half = static_cast<long>(B) * F * H * W;
  const long total = per_half * (cfg ? 2 : 1) * 2;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int half8 = i & 1;                       // which 8-channel octet of the 16
  long r = i >> 1;
  const int cond = (cfg && r >= per_half) ? 1 : (cfg ? 0 : 1);
  if (r >= per_half) r -= per_half;
  const int xx = r % W;
  long q = r / W;
  const int yy = q % H;
  q /= H;
  const int f = q % F;
  const int b = q / F;
  const int c_x = mask ? 1 : 0;                  // first latent channel
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = half8 * 8 + j;
    float val = 0.f;
    if (c < c_x) {
      val = load_elem(mask, b * mask_bs + f * mask_fs + static_cast<long>(yy) * W + xx, BF16);
    } else if (c < c_x + 4) {
      // torch: 16-bit tensor / 0-d fp32 tensor -> computed in fp32, rounded once to the 16-bit dtype
      val = load_elem(x, (((static_cast<long>(b) * F + f) * 4 + (c - c_x)) * H + yy) * W + xx, BF16) * inv_scale;
    } else if (c < c_x + 8) {
      if (cond || !zero_uncond)
        val = load_elem(img_lat, (cond && cfg ? cond_hs : 0) + b * cond_bs + f * cond_fs +
                                     (static_cast<long>(c - c_x - 4) * H + yy) * W + xx, BF16);
    }
    v[j] = val;
  }
  reinterpret_cast<uint4*>(out)[i] =
      make_uint4(pack2(v[0], v[1], BF16), pack2(v[2], v[3], BF16), pack2(v[4], v[5], BF16), pack2(v[6], v[7], BF16));
}

// SVD loop, output side (models/pipeline.py:433-439): per-frame classifier-free guidance
//   v = v_u + g_f (v_c - v_u), g_f = linspace(min, max, F)[f]      (16-bit roundings of every op, as torch does on fp16)
// then EulerDiscreteScheduler.step with v-prediction, all in fp32:
//   x0 = v * (-sigma / sqrt(sigma^2 + 1)) + x / (sigma^2 + 1);  x' = x + (x - x0) / sigma * (sigma_next - sigma)
// The product v * (-sigma / ...) is not rounded to 16 bits.  diffusers rounds it when the model output is 16-bit (16-bit tensor
// times 0-d fp32 tensor); keeping fp32 is what the fp32 pipeline computes.
// pred: fp32 [2B*F*h*w, ldc] channels-last straight from conv_out (rows: uncond half then cond half); x, x_out [B, F, 4, h, w].
template <bool BF16>
__global__ void svd_cfg_euler_step_kernel(const float* __restrict__ pred, int ldc, int cfg, const float* __restrict__ gs,
                                          const void* __restrict__ x, void* __restrict__ x_out, float sigma, float sigma_next,
                                          int B, int F, int H, int W) {
  const long total = static_cast<long>(B) * F * 4 * H * W;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int xx = i % W;
  long r = i / W;
  const int yy = r % H;
  r /= H;
  const int c = r % 4;
  r /= 4;
  const int f = r % F;
  const int b = r / F;
  const long row = ((static_cast<long>(b) * F + f) * H + yy) * W + xx;
  const long per_half = static_cast<long>(B) * F * H * W;
  float v;
  if (cfg) {
    const float vu = round16(pred[row * ldc + c], BF16);                  // the UNet's 16-bit output
    const float vc = round16(pred[(per_half + row) * ldc + c], BF16);
    const float g = round16(gs[f], BF16);                                 // guidance_scale.to(latents.dtype)
    v = round16(vu + round16(g * round16(vc - vu, BF16), BF16), BF16);
  } else {
    v = round16(pred[row * ldc + c], BF16);
  }
  const float xs = load_elem(x, i, BF16);                                 // sample.to(float32)
  const float s2 = sigma * sigma + 1.0f;
  const float x0 = v * (-sigma / sqrtf(s2)) + xs / s2;
  const float d = (xs - x0) / sigma;
  store_elem(x_out, i, xs + d * (sigma_next - sigma), BF16);
}

// encoder tail: conv_out result [N, h, w, ldm] (8 ch) -> quant_conv (1x1, 8->8) -> moments [N, 8, h, w] (NCHW, 16-bit)
// (AutoencoderKL.encode: `moments = self.quant_conv(h)`; DiagonalGaussianDistribution.mode() is channels 0..3)
template <bool BF16>
__global__ void vae_enc_finalize_kernel(const void* __restrict__ mom, int ldm, const float* __restrict__ wq /*[8][8]*/,
                                        const float* __restrict__ bq, float scale, void* __restrict__ out, int B, int F,
                                        int H, int W) {
  const long total = static_cast<long>(B) * F * H * W;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = i % W;
  long r = i / W;
  const int y = r % H;
  r /= H;
  const int f = r % F;
  const int b = r / F;
  float m[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) m[j] = load_elem(mom, i * ldm + j, BF16);
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    float acc = bq[c];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc = fmaf(wq[c * 8 + j], m[j], acc);
    // scale != 1: the reference multiplies the 16-bit moments by 0.18215 afterwards (utils/common.py:18) -> two roundings
    const float v = (scale == 1.0f) ? acc : round16(acc, BF16) * scale;
    store_elem(out, (((static_cast<long>(b) * 8 + c) * F + f) * H + y) * W + x, v, BF16);
  }
}

// decoder head: latents [B, 4, F, h, w] -> z/scaling -> post_quant_conv (1x1, 4->4) -> channels-last [B*F, h, w, 8]
// (TextToVideoSDPipeline.decode_latents + AutoencoderKL._decode)
template <bool BF16>
__global__ void vae_dec_in_kernel(const void* __restrict__ lat, float inv_scale, const float* __restrict__ wp /*[4][4]*/,
                                  const float* __restrict__ bp, void* __restrict__ out, int B, int F, int H, int W) {
  const long total = static_cast<long>(B) * F * H * W;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = i % W;
  long r = i / W;
  const int y = r % H;
  r /= H;
  const int f = r % F;
  const int b = r / F;
  float z[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const float raw = load_elem(lat, (((static_cast<long>(b) * 4 + c) * F + f) * H + y) * W + x, BF16) * inv_scale;
    z[c] = BF16 ? __bfloat162float(__float2bfloat16_rn(raw)) : __half2float(__float2half_rn(raw));
  }
  float v[8];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    float acc = bp[c];
#pragma unroll
    for (int j = 0; j < 4; ++j) acc = fmaf(wp[c * 4 + j], z[j], acc);
    v[c] = acc;
  }
#pragma unroll
  for (int c = 4; c < 8; ++c) v[c] = 0.f;
  reinterpret_cast<uint4*>(out)[i] =
      make_uint4(pack2(v[0], v[1], BF16), pack2(v[2], v[3], BF16), pack2(v[4], v[5], BF16), pack2(v[6], v[7], BF16));
}

// decoder tail: conv_out result [B*F, H, W, ldc] (3 valid channels, fp32) -> video [B, 3, F, H, W] float32
// (decode_latents: reshape + permute + .float()).  The value is first rounded to the model dtype like the reference.
template <bool BF16>
__global__ void vae_dec_finalize_kernel(const float* __restrict__ y, int ldc, float* __restrict__ out, int B, int F,
                                        int H, int W) {
  const long total = static_cast<long>(B) * 3 * F * H * W;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = i % W;
  long r = i / W;
  const int yy = r % H;
  r /= H;
  const int f = r % F;
  r /= F;
  const int c = r % 3;
  const int b = r / 3;
  const float v = y[(((static_cast<long>(b) * F + f) * H + yy) * W + x) * ldc + c];
  out[i] = BF16 ? __bfloat162float(__float2bfloat16_rn(v)) : __half2float(__float2half_rn(v));
}

// decoder tail fused with diffusers tensor2vid (models/pipeline.py:205): conv_out result [B*F, H, W, ldc] (fp32) ->
// uint8 frames [F, H, B*W, 3]:  x -> round to model dtype -> x*0.5 -> +0.5 -> clamp(0,1) -> *255 -> truncate
// (separate fp32 multiply and add, like `video.mul_(std).add_(mean)`; numpy `astype("uint8")` truncates).
// RINT: the SVD pipelines' `postprocess(..., "pil")` instead -- `(x / 2 + 0.5).clamp(0, 1)` in fp32, then numpy's
// `(images * 255).round().astype("uint8")`: the fp32 product rounded half to even.  x / 2 and x * 0.5 are the same exact
// value, so the steps before the last one are shared.
template <bool BF16, bool RINT>
__global__ void vae_dec_finalize_u8_kernel(const float* __restrict__ y, int ldc, uint8_t* __restrict__ out, int B, int F,
                                           int H, int W) {
  const long total = static_cast<long>(F) * H * B * W;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = i % W;
  long r = i / W;
  const int b = r % B;
  r /= B;
  const int yy = r % H;
  const int f = r / H;
  const float* src = y + (((static_cast<long>(b) * F + f) * H + yy) * W + x) * ldc;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v = src[c];
    v = BF16 ? __bfloat162float(__float2bfloat16_rn(v)) : __half2float(__float2half_rn(v));
    v = __fadd_rn(__fmul_rn(v, 0.5f), 0.5f);
    v = fminf(fmaxf(v, 0.0f), 1.0f);
    const float s = __fmul_rn(v, 255.0f);
    out[i * 3 + c] = static_cast<uint8_t>(RINT ? rintf(s) : s);
  }
}

// x_t = sa * repeat(x0 over frames) + sb * noise, each product and the sum rounded to 16 bits like the three torch ops of
// DDPMScheduler.add_noise (utils/common.py:40-47: repeat 'b c 1 h w -> b c f h w' + scheduler.add_noise).
// x0 [B*C, FX, HW] with FX in {1, F}; noise / out [B*C, F, HW].
template <bool BF16>
__global__ void add_noise_kernel(const void* __restrict__ x0, const void* __restrict__ noise, float sa, float sb,
                                 void* __restrict__ out, long bc, int F, int FX, long HW) {
  const long total = bc * F * HW;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long p = i % HW;
  const long r = i / HW;
  const int f = static_cast<int>(r % F);
  const long q = r / F;
  const float x = load_elem(x0, (q * FX + (FX == 1 ? 0 : f)) * HW + p, BF16);
  const float n = load_elem(noise, i, BF16);
  const float t1 = round16(__fmul_rn(sa, x), BF16);
  const float t2 = round16(__fmul_rn(sb, n), BF16);
  store_elem(out, i, __fadd_rn(t1, t2), BF16);
}

// fp32 -> 16-bit convert (weights / small tensors)
template <bool BF16>
__global__ void cast_f32_kernel(const float* __restrict__ x, void* __restrict__ y, long n) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) store_elem(y, i, x[i], BF16);
}

// ------------------------------------------------------------------------------------------------ transparent-video branch
// decode_latents output (fp32 video [B, 3, F, H, W], any strides) -> channels-last 16-bit [B*F, H, W, 8] zero padded: the
// `video_tensor.permute(0, 2, 1, 3, 4).reshape(b*f, c, h, w).to(dtype)` of models/pipeline_stage2.py:305 fused with the
// layout change the alpha decoder's conv_in wants.
template <bool BF16>
__global__ void video_f32_to_nhwc8_kernel(const float* __restrict__ v, long sb, long sc, long sf, long sy, long sx,
                                          void* __restrict__ out, int B, int C, int F, int H, int W) {
  const long total = static_cast<long>(B) * F * H * W;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int x = i % W;
  long r = i / W;
  const int y = r % H;
  r /= H;
  const int f = r % F;
  const long b = r / F;
  const float* src = v + b * sb + f * sf + y * sy + x * sx;
  float e[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) e[j] = (j < C) ? src[j * sc] : 0.f;
  reinterpret_cast<uint4*>(out)[i] =
      make_uint4(pack2(e[0], e[1], BF16), pack2(e[2], e[3], BF16), pack2(e[4], e[5], BF16), pack2(e[6], e[7], BF16));
}

// RGBA post-processing of MaskedLatentToVideoPipeline.__call__ (models/pipeline_stage2.py:311-324) on the alpha decoder's
// conv_out result y [pixels, ldc] (fp32 accumulators, 4 valid channels: r, g, b, alpha) -> uint8 [pixels, 4]:
//   v     = round16(y)                       (the decoder output in the model dtype)
//   alpha = round16(v3 * 255);  alpha > 127 -> 255, else 0
//   fg    = round16(round16(v + 1) * 127.5)  -> float -> clip(0, 255) -> truncate   (numpy astype(uint8))
template <bool BF16>
__global__ void rgba_finalize_u8_kernel(const float* __restrict__ y, int ldc, uint8_t* __restrict__ out, long pixels) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= pixels) return;
  const float* src = y + i * ldc;
  uint32_t px = 0;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v = round16(src[c], BF16);
    v = round16(__fadd_rn(v, 1.0f), BF16);
    v = round16(__fmul_rn(v, 127.5f), BF16);
    v = fminf(fmaxf(v, 0.0f), 255.0f);
    px |= static_cast<uint32_t>(static_cast<uint8_t>(v)) << (8 * c);
  }
  const float a = round16(__fmul_rn(round16(src[3], BF16), 255.0f), BF16);
  if (a > 127.0f) px |= 0xFF000000u;
  reinterpret_cast<uint32_t*>(out)[i] = px;
}

// dst [rows, ldd] = src [rows, cols] with columns cols..dcols-1 zero: widens a 32-channel activation to the 64-channel K
// block of the stride-2 implicit GEMM (UNet384 level-0 Downsample2D, LatentTransparencyOffsetEncoder 32 -> 64 conv).
__global__ void pad_cols_kernel(const uint4* __restrict__ src, long lds8, uint4* __restrict__ dst, long rows, int cols8, int dcols8) {
  const long total = rows * dcols8;
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = static_cast<int>(i % dcols8);
  const long r = i / dcols8;
  dst[i] = c < cols8 ? src[r * lds8 + c] : make_uint4(0, 0, 0, 0);
}

}  // namespace aab

using namespace aab;

#define AAB_GRID(total, threads) static_cast<unsigned>(((total) + (threads)-1) / (threads))
#define AAB_LAUNCH_RET() return cudaGetLastError() == cudaSuccess ? AAB_OK : AAB_ERR_CUDA

extern "C" int aab_unet_in_assemble(const void* sample, const long* s_strides /*b,c,f,y,x*/, const void* cond,
                                    const long* c_strides, const void* mask, const long* m_strides, int mask_batch,
                                    void* out, int b, int t, int h, int w, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!sample || !cond || !out) return AAB_ERR_ARG;
  Strides5 ss{s_strides[0], s_strides[1], s_strides[2], s_strides[3], s_strides[4]};
  Strides5 cs{c_strides[0], c_strides[1], c_strides[2], c_strides[3], c_strides[4]};
  Strides5 ms{0, 0, 0, 0, 0};
  if (mask) ms = Strides5{m_strides[0], m_strides[1], m_strides[2], m_strides[3], m_strides[4]};
  const long total = static_cast<long>(b) * t * h * w;
  if (is_bf16)
    unet_in_assemble_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(sample, ss, cond, cs, mask, ms,
                                                                            mask_batch > 0 ? mask_batch : 1, out, b, t, h, w);
  else
    unet_in_assemble_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(sample, ss, cond, cs, mask, ms,
                                                                             mask_batch > 0 ? mask_batch : 1, out, b, t, h, w);
  AAB_LAUNCH_RET();
}

extern "C" int aab_unet_out_finalize(const float* y, int ldc, void* out, int b, int t, int h, int w, int is_bf16,
                                     void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long total = static_cast<long>(b) * 4 * (t - 1) * h * w;
  if (is_bf16) unet_out_finalize_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(y, ldc, out, b, t, h, w);
  else unet_out_finalize_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(y, ldc, out, b, t, h, w);
  AAB_LAUNCH_RET();
}

extern "C" int aab_timestep_embed(const float* t, int t_count, void* out, int b, int dim, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  // one value per batch item, one shared value, or one per prompt under CFG (B = 2 x prompts); anything else would
  // index out of bounds (the reference raises a broadcast error in that case)
  if (!t || !out || (dim & 1) || t_count < 1 || b < 1 || (b % t_count) != 0) return AAB_ERR_ARG;
  const long total = static_cast<long>(b) * dim;
  if (is_bf16) timestep_embed_kernel<true><<<dim3(AAB_GRID(total, 128)), dim3(128), 0, stream>>>(t, t_count, out, b, dim);
  else timestep_embed_kernel<false><<<dim3(AAB_GRID(total, 128)), dim3(128), 0, stream>>>(t, t_count, out, b, dim);
  AAB_LAUNCH_RET();
}

extern "C" int aab_embed_tokens(const long long* ids, const void* tok_emb, const void* pos_emb, void* out, long rows,
                                int seq_len, int c, int vocab, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!ids || !tok_emb || !pos_emb || !out || (c % 8) || seq_len < 1 || vocab < 1) return AAB_ERR_ARG;
  const long total = rows * (c / 8);
  if (is_bf16)
    embed_tokens_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(
        ids, reinterpret_cast<const uint4*>(tok_emb), reinterpret_cast<const uint4*>(pos_emb),
        reinterpret_cast<uint4*>(out), rows, seq_len, c / 8, vocab);
  else
    embed_tokens_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(
        ids, reinterpret_cast<const uint4*>(tok_emb), reinterpret_cast<const uint4*>(pos_emb),
        reinterpret_cast<uint4*>(out), rows, seq_len, c / 8, vocab);
  AAB_LAUNCH_RET();
}

extern "C" int aab_geglu(const void* x, long ldx, void* out, long ldo, long rows, int nh, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if ((nh % 8) || (ldx % 8) || (ldo % 8)) return AAB_ERR_ARG;
  const long total = rows * (nh / 8);
  if (is_bf16) geglu_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(x, ldx, out, ldo, rows, nh);
  else geglu_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(x, ldx, out, ldo, rows, nh);
  AAB_LAUNCH_RET();
}

extern "C" int aab_upsample2x(const void* x, void* y, long n, int h, int w, int c, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (c % 8) return AAB_ERR_ARG;
  const long total = n * 2 * h * 2 * w * (c / 8);
  upsample2x_kernel<<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(reinterpret_cast<const uint4*>(x),
                                                               reinterpret_cast<uint4*>(y), n, h, w, c / 8);
  AAB_LAUNCH_RET();
}

extern "C" int aab_upsample_nearest(const void* x, void* y, long n, int h, int w, int oh, int ow, int c, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !y || (c % 8) || h < 1 || w < 1 || oh < 1 || ow < 1) return AAB_ERR_ARG;
  const long total = n * oh * ow * (c / 8);
  upsample_nearest_kernel<<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(reinterpret_cast<const uint4*>(x),
                                                                     reinterpret_cast<uint4*>(y), n, h, w, oh, ow, c / 8);
  AAB_LAUNCH_RET();
}

extern "C" int aab_pad_br(const void* x, void* y, long n, int h, int w, int ph, int pw, int c, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !y || (c % 8) || ph < h || pw < w) return AAB_ERR_ARG;
  const long total = n * ph * pw * (c / 8);
  pad_br_kernel<<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(y), n,
                                                           h, w, ph, pw, c / 8);
  AAB_LAUNCH_RET();
}

extern "C" int aab_copy2d(const void* src, long lds, void* dst, long ldd, long rows, int cols, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long total = rows * cols;
  if (cols % 8 == 0 && lds % 8 == 0 && ldd % 8 == 0 && (reinterpret_cast<uintptr_t>(src) % 16) == 0 &&
      (reinterpret_cast<uintptr_t>(dst) % 16) == 0) {
    copy2d_v8_kernel<<<dim3(AAB_GRID(total / 8, 256)), dim3(256), 0, stream>>>(reinterpret_cast<const uint4*>(src), lds / 8,
             reinterpret_cast<uint4*>(dst), ldd / 8, rows, cols / 8);
    AAB_LAUNCH_RET();
  }
  copy2d_kernel<<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(reinterpret_cast<const uint16_t*>(src), lds,
                                                          reinterpret_cast<uint16_t*>(dst), ldd, rows, cols);
  AAB_LAUNCH_RET();
}

extern "C" int aab_dup_rows(const void* src, void* dst, long bytes, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!src || !dst || (bytes % 16)) return AAB_ERR_ARG;
  const long n16 = bytes / 16;
  dup_rows_kernel<<<dim3(AAB_GRID(n16, 256)), dim3(256), 0, stream>>>(reinterpret_cast<const uint4*>(src),
                                                         reinterpret_cast<uint4*>(dst), n16);
  AAB_LAUNCH_RET();
}

extern "C" int aab_transpose(const void* src, long lds, long src_batch, void* dst, int nb, int rows, int cols, int ldd,
                             void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!src || !dst || ldd < rows) return AAB_ERR_ARG;
  dim3 grid((cols + 31) / 32, (ldd + 31) / 32, nb);
  transpose_kernel<<<dim3(grid), dim3(dim3(32, 8)), 0, stream>>>(reinterpret_cast<const uint16_t*>(src), lds, src_batch,
                                                     reinterpret_cast<uint16_t*>(dst), rows, cols, ldd);
  AAB_LAUNCH_RET();
}

extern "C" int aab_cfg_scheduler_step(const float* eps, int ldc, int cfg, float guidance, const void* x, void* x_out,
                                      float* x0_hist, const float* coef, const int* step_idx, int n, int f, int h, int w,
                                      int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!eps || !x || !x_out || !coef) return AAB_ERR_ARG;
  const long total = static_cast<long>(n) * 4 * f * h * w;
  if (is_bf16)
    cfg_step_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(eps, ldc, cfg, guidance, x, x_out, x0_hist, coef,
                                                                    step_idx, n, f, h, w);
  else
    cfg_step_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(eps, ldc, cfg, guidance, x, x_out, x0_hist, coef,
                                                                     step_idx, n, f, h, w);
  AAB_LAUNCH_RET();
}

extern "C" int aab_image_to_nhwc8(const void* img, long sn, long sc, long sy, long sx, void* out, long n, int c, int h,
                                  int w, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (c > 8) return AAB_ERR_ARG;
  const long total = n * h * w;
  if (is_bf16) image_to_nhwc8_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(img, sn, sc, sy, sx, out, n, c, h, w);
  else image_to_nhwc8_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(img, sn, sc, sy, sx, out, n, c, h, w);
  AAB_LAUNCH_RET();
}

extern "C" int aab_image_to_nhwc16(const void* img, long sn, long sc, long sy, long sx, void* out, long n, int c, int h, int w,
                                   int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!img || !out || c > 16 || c < 1) return AAB_ERR_ARG;
  const long total = n * h * w * 2;
  if (is_bf16) image_to_nhwc16_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(img, sn, sc, sy, sx, out, n, c, h, w);
  else image_to_nhwc16_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(img, sn, sc, sy, sx, out, n, c, h, w);
  AAB_LAUNCH_RET();
}

extern "C" int aab_add_rowvec(const void* x, long ldx, void* out, long ldo, const float* vec, long ldv, long rows, int cols,
                              long rows_per_vec, int mod, int mode, int mod2, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !out || !vec || (cols % 8) || (ldx % 8) || (ldo % 8) || (ldv % 4) || rows_per_vec < 1 || mod < 1 ||
      (mode == 1 && mod2 < 1))
    return AAB_ERR_ARG;
  const long total = rows * (cols / 8);
  if (is_bf16)
    add_rowvec_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(x, ldx, out, ldo, vec, ldv, rows, cols, rows_per_vec, mod,
                                                                     mode, mod2);
  else
    add_rowvec_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(x, ldx, out, ldo, vec, ldv, rows, cols, rows_per_vec, mod,
                                                                      mode, mod2);
  AAB_LAUNCH_RET();
}

extern "C" int aab_axpby(const void* x, const void* y, void* out, long n_elems, float a, float b, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !y || !out || (n_elems % 8)) return AAB_ERR_ARG;
  const long n16 = n_elems / 8;
  if (is_bf16)
    axpby_kernel<true><<<dim3(AAB_GRID(n16, 256)), dim3(256), 0, stream>>>(reinterpret_cast<const uint4*>(x),
                                                                 reinterpret_cast<const uint4*>(y),
                                                                 reinterpret_cast<uint4*>(out), n16, a, b);
  else
    axpby_kernel<false><<<dim3(AAB_GRID(n16, 256)), dim3(256), 0, stream>>>(reinterpret_cast<const uint4*>(x),
                                                                  reinterpret_cast<const uint4*>(y),
                                                                  reinterpret_cast<uint4*>(out), n16, a, b);
  AAB_LAUNCH_RET();
}

extern "C" int aab_svd_out_finalize(const float* y, int ldc, void* out, long bf, int h, int w, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!y || !out || ldc < 4) return AAB_ERR_ARG;
  const long total = bf * 4 * h * w;
  if (is_bf16) svd_out_finalize_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(y, ldc, out, bf, h, w);
  else svd_out_finalize_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(y, ldc, out, bf, h, w);
  AAB_LAUNCH_RET();
}

extern "C" int aab_svd_in_assemble(const void* x, const void* img_lat, const void* mask, float inv_scale, void* out, int b, int f,
                                   int h, int w, int cfg, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !img_lat || !mask || !out) return AAB_ERR_ARG;
  const long total = static_cast<long>(b) * f * h * w * (cfg ? 2 : 1) * 2;
  const long hw4 = 4L * h * w;
  if (is_bf16) svd_in_assemble_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(x, img_lat, mask, inv_scale, out, b, f, h, w, cfg, 0L, hw4, 0L, 1, 0L, 0L);
  else svd_in_assemble_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(x, img_lat, mask, inv_scale, out, b, f, h, w, cfg, 0L, hw4, 0L, 1, 0L, 0L);
  AAB_LAUNCH_RET();
}

extern "C" int aab_svd_in_assemble_frames(const void* x, const void* cond, long cond_half_stride, long cond_batch_stride,
                                          long cond_frame_stride, int zero_uncond, const void* mask, long mask_batch_stride,
                                          long mask_frame_stride, float inv_scale, void* out, int b, int f, int h, int w, int cfg,
                                          int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !cond || !out) return AAB_ERR_ARG;
  const long total = static_cast<long>(b) * f * h * w * (cfg ? 2 : 1) * 2;
  if (is_bf16) svd_in_assemble_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(x, cond, mask, inv_scale, out, b, f, h, w, cfg, cond_half_stride, cond_batch_stride, cond_frame_stride, zero_uncond, mask_batch_stride, mask_frame_stride);
  else svd_in_assemble_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(x, cond, mask, inv_scale, out, b, f, h, w, cfg, cond_half_stride, cond_batch_stride, cond_frame_stride, zero_uncond, mask_batch_stride, mask_frame_stride);
  AAB_LAUNCH_RET();
}

extern "C" int aab_svd_cfg_euler_step(const float* pred, int ldc, int cfg, const float* gs, const void* x, void* x_out,
                                      float sigma, float sigma_next, int b, int f, int h, int w, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!pred || !x || !x_out || (cfg && !gs) || ldc < 4 || sigma <= 0.f) return AAB_ERR_ARG;
  const long total = static_cast<long>(b) * f * 4 * h * w;
  if (is_bf16)
    svd_cfg_euler_step_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(pred, ldc, cfg, gs, x, x_out, sigma, sigma_next, b,
                                                                             f, h, w);
  else
    svd_cfg_euler_step_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(pred, ldc, cfg, gs, x, x_out, sigma, sigma_next, b,
                                                                              f, h, w);
  AAB_LAUNCH_RET();
}

extern "C" int aab_vae_enc_finalize(const void* mom, int ldm, const float* wq, const float* bq, float scale, void* out,
                                    int b, int f, int h, int w, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long total = static_cast<long>(b) * f * h * w;
  if (is_bf16) vae_enc_finalize_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(mom, ldm, wq, bq, scale, out, b, f, h, w);
  else vae_enc_finalize_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(mom, ldm, wq, bq, scale, out, b, f, h, w);
  AAB_LAUNCH_RET();
}

extern "C" int aab_vae_dec_in(const void* lat, float inv_scale, const float* wp, const float* bp, void* out, int b, int f,
                              int h, int w, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long total = static_cast<long>(b) * f * h * w;
  if (is_bf16) vae_dec_in_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(lat, inv_scale, wp, bp, out, b, f, h, w);
  else vae_dec_in_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(lat, inv_scale, wp, bp, out, b, f, h, w);
  AAB_LAUNCH_RET();
}

extern "C" int aab_vae_dec_finalize(const float* y, int ldc, float* out, int b, int f, int h, int w, int is_bf16,
                                    void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long total = static_cast<long>(b) * 3 * f * h * w;
  if (is_bf16) vae_dec_finalize_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(y, ldc, out, b, f, h, w);
  else vae_dec_finalize_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(y, ldc, out, b, f, h, w);
  AAB_LAUNCH_RET();
}

extern "C" int aab_vae_dec_finalize_u8(const float* y, int ldc, void* out, int b, int f, int h, int w, int is_bf16,
                                       void* stream_) {
  // bit 0: bf16 model; bit 1: round to nearest even (SVD postprocess) instead of truncating (tensor2vid)
  if (is_bf16 & ~3) return AAB_ERR_ARG;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const long total = static_cast<long>(b) * f * h * w;
  uint8_t* o = reinterpret_cast<uint8_t*>(out);
  const dim3 grid(AAB_GRID(total, 256)), block(256);
  switch (is_bf16) {
    case 0: vae_dec_finalize_u8_kernel<false, false><<<grid, block, 0, stream>>>(y, ldc, o, b, f, h, w); break;
    case 1: vae_dec_finalize_u8_kernel<true, false><<<grid, block, 0, stream>>>(y, ldc, o, b, f, h, w); break;
    case 2: vae_dec_finalize_u8_kernel<false, true><<<grid, block, 0, stream>>>(y, ldc, o, b, f, h, w); break;
    default: vae_dec_finalize_u8_kernel<true, true><<<grid, block, 0, stream>>>(y, ldc, o, b, f, h, w); break;
  }
  AAB_LAUNCH_RET();
}

extern "C" int aab_add_noise(const void* x0, const void* noise, float sa, float sb, void* out, long bc, int f, int fx,
                             long hw, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x0 || !noise || !out || bc < 1 || f < 1 || hw < 1 || (fx != 1 && fx != f)) return AAB_ERR_ARG;
  const long total = bc * f * hw;
  if (is_bf16) add_noise_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(x0, noise, sa, sb, out, bc, f, fx, hw);
  else add_noise_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(x0, noise, sa, sb, out, bc, f, fx, hw);
  AAB_LAUNCH_RET();
}

extern "C" int aab_cast_f32(const float* x, void* y, long n, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (is_bf16) cast_f32_kernel<true><<<dim3(AAB_GRID(n, 256)), dim3(256), 0, stream>>>(x, y, n);
  else cast_f32_kernel<false><<<dim3(AAB_GRID(n, 256)), dim3(256), 0, stream>>>(x, y, n);
  AAB_LAUNCH_RET();
}

extern "C" int aab_video_f32_to_nhwc8(const float* video, long sb, long sc, long sf, long sy, long sx, void* out, int b, int c,
                                      int f, int h, int w, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!video || !out || c < 1 || c > 8 || b < 1 || f < 1 || h < 1 || w < 1) return AAB_ERR_ARG;
  const long total = static_cast<long>(b) * f * h * w;
  if (is_bf16) video_f32_to_nhwc8_kernel<true><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(video, sb, sc, sf, sy, sx, out, b, c, f, h, w);
  else video_f32_to_nhwc8_kernel<false><<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(video, sb, sc, sf, sy, sx, out, b, c, f, h, w);
  AAB_LAUNCH_RET();
}

extern "C" int aab_rgba_finalize_u8(const float* y, int ldc, void* out, long pixels, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!y || !out || ldc < 4 || pixels < 1) return AAB_ERR_ARG;
  if (is_bf16) rgba_finalize_u8_kernel<true><<<dim3(AAB_GRID(pixels, 256)), dim3(256), 0, stream>>>(y, ldc, reinterpret_cast<uint8_t*>(out), pixels);
  else rgba_finalize_u8_kernel<false><<<dim3(AAB_GRID(pixels, 256)), dim3(256), 0, stream>>>(y, ldc, reinterpret_cast<uint8_t*>(out), pixels);
  AAB_LAUNCH_RET();
}

extern "C" int aab_pad_cols(const void* src, long lds, void* dst, long rows, int cols, int dst_cols, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!src || !dst || rows < 1 || (cols % 8) || (dst_cols % 8) || (lds % 8) || cols > dst_cols || cols < 8) return AAB_ERR_ARG;
  const long total = rows * (dst_cols / 8);
  pad_cols_kernel<<<dim3(AAB_GRID(total, 256)), dim3(256), 0, stream>>>(reinterpret_cast<const uint4*>(src), lds / 8,
           reinterpret_cast<uint4*>(dst), rows, cols / 8, dst_cols / 8);
  AAB_LAUNCH_RET();
}
