// CLIP image preprocessing + patchify: the front end of the CLIP ViT image tower behind the SVD pipelines' `_encode_image`
// (models/pipeline.py:347,597; diffusers 0.24 StableVideoDiffusionPipeline._encode_image, restated by the reference itself
// at train_svd.py:384-395).  One thread per output pixel (3 channels), one CTA per patch row of the GEMM operand.
//
// uint8 source (a PIL image, pil_to_numpy), per image, in fp32:
//   x = u8 / 255;  x = 2 x - 1;
//   _resize_with_antialiasing(x, (S, S)): separable Gaussian blur (x axis first, then y; reflect padding; taps computed on
//   the host by the caller) followed by F.interpolate(mode="bicubic", align_corners=True);
//   x = (x + 1) / 2;  x = (x - mean) / std  (CLIPImageProcessor normalisation).
// float source: the tensor already is the CLIP pixel values (diffusers passes tensors straight to the encoder): rounding only.
// Every step is a separately rounded fp32 operation (the __f*_rn intrinsics keep nvcc from contracting them into FMAs): the
// sums run tap by tap in a fixed order, so a plain-torch restatement of the same order reproduces the kernel bit for bit in
// fp32, and differs from torch's own conv / interpolate kernels only by their summation order.
#include "common.cuh"

namespace aab {

struct ClipPrepParams {
  const void* src;
  int src_type;                  // 0 uint8, 1 float32, 2 float16, 3 bfloat16
  long sb, sc, sy, sx;           // element strides of [b, 3, h, w]
  int h, w;
  const float* taps_y;
  int ks_y;
  const float* taps_x;
  int ks_x;
  const float* mean_std;         // [6]: mean r g b, std r g b
  int S, patch, grid;            // output size, patch edge, patches per side
  void* out;
  long ld_out;
};

__device__ __forceinline__ int reflect_idx(int i, int n) {
  i = i < 0 ? -i : i;
  return i >= n ? 2 * (n - 1) - i : i;
}

// torch upsample_bicubic2d (A = -0.75) weights of the four taps around fractional offset t, op by op:
// cc1(x) = ((A + 2) x - (A + 3)) x x + 1,  cc2(x) = ((A x - 5A) x + 8A) x - 4A
__device__ __forceinline__ float cubic_cc1(float x) {
  return __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(1.25f, x), 2.25f), x), x), 1.0f);
}
__device__ __forceinline__ float cubic_cc2(float x) {
  return __fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(-0.75f, x), 3.75f), x), 6.0f), x), 3.0f);
}
__device__ __forceinline__ void cubic_coeffs(float c[4], float t) {
  c[0] = cubic_cc2(__fadd_rn(t, 1.0f));
  c[1] = cubic_cc1(t);
  c[2] = cubic_cc1(__fsub_rn(1.0f, t));
  c[3] = cubic_cc2(__fsub_rn(2.0f, t));
}

__device__ __forceinline__ float u8_to_signed_unit(uint8_t v) {
  return __fsub_rn(__fmul_rn(__fdiv_rn(static_cast<float>(v), 255.0f), 2.0f), 1.0f);
}

template <bool BF16>
__global__ void __launch_bounds__(256) clip_image_prep_kernel(const ClipPrepParams p) {
  const int row = blockIdx.x;                      // 0: class slot, 1 + patch index
  const int b = blockIdx.y;
  const int pp = p.patch * p.patch;
  uint8_t* orow = reinterpret_cast<uint8_t*>(p.out) + ((static_cast<long>(b) * (1 + p.grid * p.grid) + row) * p.ld_out) * 2;
  if (row == 0) {
    for (long c = threadIdx.x; c < p.ld_out; c += blockDim.x) store_elem(orow, c, 0.f, BF16);
    return;
  }
  for (long c = 3 * pp + threadIdx.x; c < p.ld_out; c += blockDim.x) store_elem(orow, c, 0.f, BF16);
  const int pidx = row - 1;
  for (int t = threadIdx.x; t < pp; t += blockDim.x) {
    const int oy = (pidx / p.grid) * p.patch + t / p.patch;
    const int ox = (pidx % p.grid) * p.patch + t % p.patch;
    float v[3];
    if (p.src_type != 0) {
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const long i = b * p.sb + ch * p.sc + oy * p.sy + ox * p.sx;
        v[ch] = p.src_type == 1 ? reinterpret_cast<const float*>(p.src)[i]
                                : load_elem(p.src, static_cast<size_t>(i), p.src_type == 3);
      }
    } else {
      const uint8_t* img = reinterpret_cast<const uint8_t*>(p.src) + b * p.sb;
      // bicubic source position (align_corners=True) of this output pixel
      const float scy = p.S > 1 ? static_cast<float>(p.h - 1) / static_cast<float>(p.S - 1) : 0.f;
      const float scx = p.S > 1 ? static_cast<float>(p.w - 1) / static_cast<float>(p.S - 1) : 0.f;
      const float ry = __fmul_rn(scy, static_cast<float>(oy));
      const float rx = __fmul_rn(scx, static_cast<float>(ox));
      const int iy = static_cast<int>(floorf(ry));
      const int ix = static_cast<int>(floorf(rx));
      float wy[4], wx[4];
      cubic_coeffs(wy, __fsub_rn(ry, static_cast<float>(iy)));
      cubic_coeffs(wx, __fsub_rn(rx, static_cast<float>(ix)));
      const int pad_y = (p.ks_y - 1) / 2, pad_x = (p.ks_x - 1) / 2;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int yy = min(max(iy - 1 + k, 0), p.h - 1);
          float racc = 0.f;
#pragma unroll
          for (int l = 0; l < 4; ++l) {
            const int xx = min(max(ix - 1 + l, 0), p.w - 1);
            // blurred value at (yy, xx): y taps over x-blurred rows
            float by = 0.f;
            for (int ky = 0; ky < p.ks_y; ++ky) {
              const uint8_t* r = img + reflect_idx(yy + ky - pad_y, p.h) * p.sy + ch * p.sc;
              float bx = 0.f;
              for (int kx = 0; kx < p.ks_x; ++kx)
                bx = __fadd_rn(bx, __fmul_rn(__ldg(p.taps_x + kx), u8_to_signed_unit(r[reflect_idx(xx + kx - pad_x, p.w) * p.sx])));
              by = __fadd_rn(by, __fmul_rn(__ldg(p.taps_y + ky), bx));
            }
            racc = __fadd_rn(racc, __fmul_rn(by, wx[l]));
          }
          acc = __fadd_rn(acc, __fmul_rn(racc, wy[k]));
        }
        const float unit = __fdiv_rn(__fadd_rn(acc, 1.0f), 2.0f);
        v[ch] = __fdiv_rn(__fsub_rn(unit, __ldg(p.mean_std + ch)), __ldg(p.mean_std + 3 + ch));
      }
    }
    const int col = (oy % p.patch) * p.patch + ox % p.patch;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) store_elem(orow, static_cast<size_t>(ch) * pp + col, v[ch], BF16);
  }
}

}  // namespace aab

using namespace aab;

extern "C" int aab_clip_image_prep(const void* src, int src_type, long sb, long sc, long sy, long sx, int b, int h, int w,
                                   const float* taps_y, int ks_y, const float* taps_x, int ks_x, const float* mean_std,
                                   int out_size, int patch, void* out, long ld_out, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!src || !out || src_type < 0 || src_type > 3 || b < 1 || h < 1 || w < 1 || patch < 1 || out_size < patch ||
      out_size % patch || ld_out < 3L * patch * patch || ld_out % 8 || (reinterpret_cast<uintptr_t>(out) % 16))
    return AAB_ERR_ARG;
  if (src_type == 0) {
    // the blur pads by (ks - 1) / 2 with reflection, which needs that many pixels on each side (torch's reflect pad rule)
    if (!taps_y || !taps_x || !mean_std || ks_y < 1 || ks_x < 1 || !(ks_y & 1) || !(ks_x & 1) || (ks_y - 1) / 2 >= h ||
        (ks_x - 1) / 2 >= w)
      return AAB_ERR_ARG;
  } else if (h != out_size || w != out_size) {
    return AAB_ERR_ARG;                      // the model's input size: transformers raises for any other
  }
  ClipPrepParams p;
  p.src = src;
  p.src_type = src_type;
  p.sb = sb;
  p.sc = sc;
  p.sy = sy;
  p.sx = sx;
  p.h = h;
  p.w = w;
  p.taps_y = taps_y;
  p.ks_y = ks_y;
  p.taps_x = taps_x;
  p.ks_x = ks_x;
  p.mean_std = mean_std;
  p.S = out_size;
  p.patch = patch;
  p.grid = out_size / patch;
  p.out = out;
  p.ld_out = ld_out;
  const dim3 grid(1 + p.grid * p.grid, b);
  if (is_bf16)
    clip_image_prep_kernel<true><<<grid, dim3(256), 0, stream>>>(p);
  else
    clip_image_prep_kernel<false><<<grid, dim3(256), 0, stream>>>(p);
  return cudaGetLastError() == cudaSuccess ? AAB_OK : AAB_ERR_CUDA;
}
