// Internal + C-ABI structures of the implicit-GEMM kernel (see include/aab200.h for the public declaration).
#pragma once
#include <stdint.h>

#define AAB_MAX_TAPS 9

#define AAB_ACT_NONE 0
#define AAB_ACT_SILU 1
#define AAB_ACT_GELU 2
#define AAB_ACT_QUICK_GELU 3   /* x * sigmoid(1.702 x): transformers 'quick_gelu' (CLIP text MLP) */

#define AAB_F_BF16 1      /* 16-bit type is bfloat16 (else float16) */
#define AAB_F_DIRECT 2    /* generic epilogue: any n_out, fp32 output, every flag combination, per-element masks */
#define AAB_F_OUT_F32 4   /* output is float32 (direct store only) */
#define AAB_F_SCALE_ACC 16 /* out = act(acc + bias + bias2) * out_scale + residual (scale BEFORE the residual; direct store only) */
#define AAB_F_GEGLU 8     /* B rows [0,N/2) are values, [N/2,N) gates: out = value * gelu(gate), N/2 columns */
#define AAB_F_TWO_CTA 64  /* two CTAs per SM (3-stage ring, 80 registers): block_n 64, not GEGLU */

#ifdef __cplusplus
extern "C" {
#endif

// Caller-side description of one implicit-GEMM launch. Pixel dims are innermost-first; "dim 0" of A is channels.
typedef struct AabIgemmDesc {
  const void* a;            // activation tensor, 16-bit, viewed as 5-D [a_dims[4]]...[a_dims[0]=channels]
  long a_dims[5];
  long a_strides[5];        // in elements; a_strides[0] == 1, others multiples of 8
  const void* a2;           // optional second source (virtual channel concat): channels [kc1, kc) come from a2
  long a2_dims[5];
  long a2_strides[5];
  int kc;                   // reduction length per tap (channels)
  int kc1;                  // channels taken from `a` when a2 != NULL (multiple of 64)
  int num_taps;
  int tap_off[AAB_MAX_TAPS][5];  // per tap: offset added to (channel, pix0, pix1, pix2, pix3) coordinates of A
  const void* b;            // weights [b_batch][n][num_taps*kc], K contiguous
  long ld_b;                // row stride of b in elements
  int b_batch;              // 0/1: shared weights; >1: batched B (e.g. K^T of attention)
  long b_batch_stride;
  int b_batch_dim;          // which pixel dim (0..3) indexes the B batch, -1 for none
  int n;                    // rows of b (for GEGLU: 2 x output columns)
  int dim_d[4];             // output pixel dims (innermost first); tile grid is derived from these
  int box[4];               // pixels per tile along each dim, product must be 128
  void* out;                // [prod(dim_d)][ld_out]
  long ld_out;
  const float* bias;        // [n] fp32 or NULL
  const float* bias2;       // [*, ld_bias2] fp32 per-sample bias (row / rows_per_bias2 selects the sample) or NULL
  int rows_per_bias2;
  long ld_bias2;
  const void* residual;     // [prod(dim_d)][ld_res] 16-bit or NULL
  long ld_res;
  float out_scale;
  int act;
  int flags;
  int block_n;              // 32 / 64 / 128 / 160 / 192 / 256 (GEGLU: 128 / 256)
  float* colstats;          // optional [num_m_tiles][n_out][2] fp32: per m-tile column sums (sum, sum of squares) of the ROUNDED
                            // 16-bit outputs over the tile's valid rows -- the statistics of the GroupNorm that follows, taken
                            // where the data already is in registers (staged epilogues only), or NULL
} AabIgemmDesc;

#ifdef __cplusplus
}
#endif

#ifdef __CUDACC__
namespace aab {
struct IgemmParams {
  int dimD[4];
  int box[4];
  int tiles[4];
  int num_m_tiles, num_n_tiles;
  int N, n_out, Kc, Kc1, num_taps, kb_per_tap;
  int tap_off[AAB_MAX_TAPS][5];
  int b_batch_dim;
  const float* bias;
  const float* bias2;
  int rows_per_bias2;
  long ld_bias2;
  const void* residual;
  long ld_res;
  void* out;
  long ld_out;
  float out_scale;
  int act;
  int flags;
  float* colstats;
};
int make_tmap_16(CUtensorMap* out, const void* base, int rank, const long* dims, const long* strides, const int* box,
                 int is_bf16, int swizzle_bytes = 128);
int num_sms();
}  // namespace aab
#endif
