// HBM-bound normalisation kernels on channels-last activations [samples][rows][C]:
//   * GroupNorm statistics (fp32 partial sums per thread, fp64 atomics per (sample, group)), with the statistics
//     extent a parameter: rows = H*W gives torch.nn.GroupNorm on [(b t), C, H, W] (ResnetBlock2D / Transformer2DModel
//     norms), rows = T*H*W gives GroupNorm on [b, C, T, H, W] (TemporalConvLayer / TransformerTemporalModel norms,
//     reference: diffusers resnet.TemporalConvLayer, transformer_temporal.py; call sites models/unet_3d_blocks.py:276,299).
//   * GroupNorm apply (+ optional SiLU) writing the 16-bit operand of the following implicit GEMM; the input may be
//     the *virtual* channel concatenation of two tensors (skip connections, models/unet_3d_blocks.py:731,828), so
//     torch.cat is never materialised for the norm path.
//   * LayerNorm over C (one warp per token row, exact two-pass variance in registers).
// Algorithmic bytes: stats = 1 read of the activation; apply = 1 read + 1 write; layernorm = 1 read + 1 write.
#include "common.cuh"
#include "igemm.h"
#include <stdlib.h>

namespace aab {

__device__ __forceinline__ uint4 ldg16(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// thread mapping shared by stats/apply: V = C/8 channel octets per row; blockDim = V * rpi (rows per iteration)
struct GnArgs {
  const void* x1;
  const void* x2;     // optional second source (channels C1..C)
  int C1, C2;         // C = C1 + C2
  long ld1, ld2;      // row strides (elements)
  long rows;          // rows per sample (statistics extent)
  int groups;
  int rows_per_cta;
  int bf16;
};

// Deterministic (bitwise reproducible) statistics: fixed-order reductions only.  Each CTA reduces its row chunk to one
// (sum, sumsq) pair per group and stores it to `partial`; the last CTA of a sample (atomic ticket, self-resetting)
// adds the chunk partials in index order and publishes mean / rstd.
__global__ void gn_stats_kernel(GnArgs a, double* __restrict__ partial /* [S][chunks][G][2] */,
                                float* __restrict__ mean_rstd /* [S][G][2] */, unsigned int* __restrict__ ticket /* [S] */,
                                float eps) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ float sh[];   // [rpi][C] sums, [rpi][C] squares
  __shared__ bool is_last;
  const int C = a.C1 + a.C2;
  const int V = C >> 3;
  const int oct = threadIdx.x % V;
  const int rsub = threadIdx.x / V;
  const int rpi = blockDim.x / V;
  const int s = blockIdx.y;
  const int chunks = gridDim.x;
  const long r0 = static_cast<long>(blockIdx.x) * a.rows_per_cta;
  long r1 = r0 + a.rows_per_cta;
  if (r1 > a.rows) r1 = a.rows;
  float sum[8], sq[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) sum[j] = sq[j] = 0.f;
  const bool bf = a.bf16 != 0;
  const int c0 = oct * 8;
  const uint8_t* base;
  long ld;
  int cc;
  if (c0 < a.C1) { base = reinterpret_cast<const uint8_t*>(a.x1); ld = a.ld1; cc = c0; }
  else { base = reinterpret_cast<const uint8_t*>(a.x2); ld = a.ld2; cc = c0 - a.C1; }
  // 8 independent 16-byte loads in flight per thread, and the NEXT batch of 8 is requested before the current one is
  // accumulated (register double buffering): the kernel is latency-bound otherwise
  auto load8 = [&](uint4 (&u)[8], long r) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const long rk = r + static_cast<long>(k) * rpi;
      u[k] = make_uint4(0, 0, 0, 0);
      if (rk < r1) u[k] = ldg16(base + ((static_cast<long>(s) * a.rows + rk) * ld + cc) * 2);
    }
  };
  uint4 u[8], un[8];
  load8(u, r0 + rsub);
  for (long r = r0 + rsub; r < r1; r += 8 * rpi) {
    const bool more = r + 8 * rpi < r1;
    if (more) load8(un, r + 8 * rpi);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const uint32_t w[4] = {u[k].x, u[k].y, u[k].z, u[k].w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack2(w[e], bf);
        sum[2 * e] += f.x; sq[2 * e] += f.x * f.x;
        sum[2 * e + 1] += f.y; sq[2 * e + 1] += f.y * f.y;
      }
    }
    if (more) {
#pragma unroll
      for (int k = 0; k < 8; ++k) u[k] = un[k];
    }
  }
  float* shs = sh;
  float* shq = sh + rpi * C;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    shs[rsub * C + c0 + j] = sum[j];
    shq[rsub * C + c0 + j] = sq[j];
  }
  __syncthreads();
  const int cpg = C / a.groups;
  if (threadIdx.x < a.groups) {
    // fixed-order fp32 combine of the <= rows_per_cta x cpg values of this CTA (two independent chains per quantity),
    // fp64 only across CTAs
    const int g = threadIdx.x;
    float fs0 = 0.f, fs1 = 0.f, fq0 = 0.f, fq1 = 0.f;
    for (int r = 0; r < rpi; ++r) {
      int c = g * cpg;
      for (; c + 1 < (g + 1) * cpg; c += 2) {
        fs0 += shs[r * C + c];
        fs1 += shs[r * C + c + 1];
        fq0 += shq[r * C + c];
        fq1 += shq[r * C + c + 1];
      }
      if (c < (g + 1) * cpg) {
        fs0 += shs[r * C + c];
        fq0 += shq[r * C + c];
      }
    }
    double* pp = partial + ((static_cast<long>(s) * chunks + blockIdx.x) * a.groups + g) * 2;
    pp[0] = static_cast<double>(fs0) + static_cast<double>(fs1);
    pp[1] = static_cast<double>(fq0) + static_cast<double>(fq1);
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int t = atomicAdd(&ticket[s], 1u);
    is_last = (t == static_cast<unsigned int>(chunks - 1));
    if (is_last) ticket[s] = 0;          // self-reset for the next launch
  }
  __syncthreads();
  if (is_last) {
    // final, fixed-order reduction over the chunk partials, spread over the whole CTA:
    // part p of group g adds chunks p, p+P, p+2P, ... ; then the P parts are added in index order.
    __threadfence();
    const int P = blockDim.x / a.groups;                 // >= 1 (blockDim >= groups is guaranteed by the host)
    double* red = reinterpret_cast<double*>(sh);         // [P][groups][2] doubles (fits: P*groups*16 B <= smem)
    const int g = threadIdx.x % a.groups;
    const int part = threadIdx.x / a.groups;
    if (part < P) {
      // 8 independent L2 loads in flight per thread (a dependent load->add chain over ~80 partials costs ~30 us);
      // the summation order stays fixed: lane k of the 8 accumulators always takes chunks part + (8 i + k) P
      double ds[8], dq[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) ds[k] = dq[k] = 0.0;
      const double* pp = partial + (static_cast<long>(s) * chunks * a.groups + g) * 2;
      for (int ch = part; ch < chunks; ch += 8 * P) {
        double2 v[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int c2 = ch + k * P;
          v[k] = make_double2(0.0, 0.0);
          if (c2 < chunks) v[k] = __ldcg(reinterpret_cast<const double2*>(pp + static_cast<long>(c2) * a.groups * 2));
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          ds[k] += v[k].x;
          dq[k] += v[k].y;
        }
      }
      red[(part * a.groups + g) * 2] = ((ds[0] + ds[1]) + (ds[2] + ds[3])) + ((ds[4] + ds[5]) + (ds[6] + ds[7]));
      red[(part * a.groups + g) * 2 + 1] = ((dq[0] + dq[1]) + (dq[2] + dq[3])) + ((dq[4] + dq[5]) + (dq[6] + dq[7]));
    }
    __syncthreads();
    if (threadIdx.x < a.groups) {
      double ds = 0.0, dq = 0.0;
      for (int q = 0; q < P; ++q) {
        ds += red[(q * a.groups + g) * 2];
        dq += red[(q * a.groups + g) * 2 + 1];
      }
      const double n = static_cast<double>(a.rows) * cpg;
      const double m = ds / n;
      double var = dq / n - m * m;
      if (var < 0) var = 0;
      mean_rstd[(static_cast<long>(s) * a.groups + g) * 2] = static_cast<float>(m);
      mean_rstd[(static_cast<long>(s) * a.groups + g) * 2 + 1] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
    }
  }
}

__global__ void gn_apply_kernel(GnArgs a, const float* __restrict__ mean_rstd, const float* __restrict__ gamma,
                                const float* __restrict__ beta, int silu, void* __restrict__ y, long ldy) {
  pdl_trigger();
  pdl_wait();
  const int C = a.C1 + a.C2;
  const int V = C >> 3;
  const int oct = threadIdx.x % V;
  const int rsub = threadIdx.x / V;
  const int rpi = blockDim.x / V;
  const int s = blockIdx.y;
  const long r0 = static_cast<long>(blockIdx.x) * a.rows_per_cta;
  long r1 = r0 + a.rows_per_cta;
  if (r1 > a.rows) r1 = a.rows;
  const bool bf = a.bf16 != 0;
  const int c0 = oct * 8;
  const int cpg = C / a.groups;
  float sc[8], sf[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int g = (c0 + j) / cpg;
    const float m = mean_rstd[(static_cast<long>(s) * a.groups + g) * 2];
    const float rstd = mean_rstd[(static_cast<long>(s) * a.groups + g) * 2 + 1];
    const float gm = gamma[c0 + j];
    sc[j] = rstd * gm;
    sf[j] = beta[c0 + j] - m * rstd * gm;
  }
  const uint8_t* base;
  long ld;
  int cc;
  if (c0 < a.C1) { base = reinterpret_cast<const uint8_t*>(a.x1); ld = a.ld1; cc = c0; }
  else { base = reinterpret_cast<const uint8_t*>(a.x2); ld = a.ld2; cc = c0 - a.C1; }
  auto load4 = [&](uint4 (&u)[4], long r) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const long rk = r + static_cast<long>(k) * rpi;
      u[k] = make_uint4(0, 0, 0, 0);
      if (rk < r1) u[k] = ldg16(base + ((static_cast<long>(s) * a.rows + rk) * ld + cc) * 2);
    }
  };
  uint4 u[4], un[4];
  load4(u, r0 + rsub);
  for (long r = r0 + rsub; r < r1; r += 4 * rpi) {
    const bool more = r + 4 * rpi < r1;
    if (more) load4(un, r + 4 * rpi);       // next batch in flight while this one is normalised and stored
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const long rk = r + static_cast<long>(k) * rpi;
      if (rk >= r1) break;
      const uint32_t w[4] = {u[k].x, u[k].y, u[k].z, u[k].w};
      uint32_t o[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack2(w[e], bf);
        float v0 = fmaf(f.x, sc[2 * e], sf[2 * e]);
        float v1 = fmaf(f.y, sc[2 * e + 1], sf[2 * e + 1]);
        if (silu) { v0 = silu_fast_f(v0); v1 = silu_fast_f(v1); }
        o[e] = pack2(v0, v1, bf);
      }
      *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(y) + ((static_cast<long>(s) * a.rows + rk) * ldy + c0) * 2) =
          make_uint4(o[0], o[1], o[2], o[3]);
    }
    if (more) {
#pragma unroll
      for (int k = 0; k < 4; ++k) u[k] = un[k];
    }
  }
}

// GroupNorm statistics from the column sums the producing GEMM left behind (igemm `colstats`: [m-tiles][C][2] fp32, one
// (sum, sumsq) per 128-row tile and column).  CTA (sample s, group g) adds the tps tiles of the sample x the cpg columns of the
// group in a fixed order (fp64) and publishes mean / rstd -- the 89 MB statistics read of a level-0 GroupNorm becomes a 2.8 MB
// one.  Two sources = virtual channel concat (channels [0, C1) from cs1, [C1, C1+C2) from cs2).
__global__ void gn_finalize_kernel(const float* __restrict__ cs1, int C1, const float* __restrict__ cs2, int C2, int tps, long rows,
                                   int groups, float eps, float* __restrict__ mean_rstd) {
  pdl_trigger();
  pdl_wait();
  __shared__ double red[2][256];
  const int s = blockIdx.y;
  const int g = blockIdx.x;
  const int C = C1 + C2;
  const int cpg = C / groups;
  const int n = tps * cpg;                       // (tile, column) pairs of this (sample, group)
  double ds = 0.0, dq = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int t = i / cpg;
    const int c = g * cpg + (i - t * cpg);
    const long tile = static_cast<long>(s) * tps + t;
    const float2 v = (c < C1) ? __ldg(reinterpret_cast<const float2*>(cs1 + (tile * C1 + c) * 2))
                              : __ldg(reinterpret_cast<const float2*>(cs2 + (tile * C2 + (c - C1)) * 2));
    ds += static_cast<double>(v.x);
    dq += static_cast<double>(v.y);
  }
  red[0][threadIdx.x] = ds;
  red[1][threadIdx.x] = dq;
  __syncthreads();
  for (int off = blockDim.x >> 1; off > 0; off >>= 1) {      // fixed-order tree
    if (threadIdx.x < off) {
      red[0][threadIdx.x] += red[0][threadIdx.x + off];
      red[1][threadIdx.x] += red[1][threadIdx.x + off];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double cnt = static_cast<double>(rows) * cpg;
    const double m = red[0][0] / cnt;
    double var = red[1][0] / cnt - m * m;
    if (var < 0) var = 0;
    mean_rstd[(static_cast<long>(s) * groups + g) * 2] = static_cast<float>(m);
    mean_rstd[(static_cast<long>(s) * groups + g) * 2 + 1] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  }
}

// One warp handles R consecutive rows at a time (all loads of the R rows are issued before any reduction, so that
// enough bytes are in flight per SM); OPL = 16-byte octets per lane = ceil(C/8/32).  C % 8 == 0, C <= 2048.
template <int OPL, int R>
__global__ void __launch_bounds__(256)
layernorm_kernel(const void* __restrict__ x, long ldx, void* __restrict__ y, long ldy, const float* __restrict__ gamma,
                 const float* __restrict__ beta, long rows, int C, float eps, int bf16) {
  pdl_trigger();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const long warp_global = static_cast<long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long row0 = warp_global * R;
  if (row0 >= rows) return;
  const bool bf = bf16 != 0;
  const int V = C >> 3;
  uint4 raw[R][OPL];
#pragma unroll
  for (int r = 0; r < R; ++r) {
#pragma unroll
    for (int i = 0; i < OPL; ++i) {
      const int o = lane + i * 32;
      raw[r][i] = make_uint4(0, 0, 0, 0);
      if (o < V && row0 + r < rows)
        raw[r][i] = ldg16(reinterpret_cast<const uint8_t*>(x) + ((row0 + r) * ldx + o * 8) * 2);
    }
  }
  const float invc = 1.0f / C;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    if (row0 + r >= rows) break;
    float v[OPL][8];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < OPL; ++i) {
      const uint32_t w[4] = {raw[r][i].x, raw[r][i].y, raw[r][i].z, raw[r][i].w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack2(w[e], bf);
        v[i][2 * e] = f.x; v[i][2 * e + 1] = f.y;
        sum += f.x + f.y;                 // lanes beyond V hold zeros
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
    const float mean = sum * invc;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < OPL; ++i) {
      if (lane + i * 32 < V) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; sq += d * d; }
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, off);
    const float rstd = rsqrtf(sq * invc + eps);
#pragma unroll
    for (int i = 0; i < OPL; ++i) {
      const int o = lane + i * 32;
      if (o < V) {
        const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + o * 8));
        const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + o * 8) + 1);
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + o * 8));
        const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + o * 8) + 1);
        const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        uint32_t ow[4];
#pragma unroll
        for (int e = 0; e < 4; ++e)
          ow[e] = pack2((v[i][2 * e] - mean) * rstd * gg[2 * e] + bb[2 * e],
                        (v[i][2 * e + 1] - mean) * rstd * gg[2 * e + 1] + bb[2 * e + 1], bf);
        *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(y) + ((row0 + r) * ldy + o * 8) * 2) =
            make_uint4(ow[0], ow[1], ow[2], ow[3]);
      }
    }
  }
}

// LayerNorm v2 (v1 leaves lanes idle for C = 320 / 640): LPR lanes share one row (LPR = 8 / 16 / 32 chosen so that
// ceil(C/8 / LPR) octets per lane waste no lanes: C=320 -> 8 lanes x 5 octets, 640 -> 16 x 5, 1280 -> 32 x 5), a warp
// normalises 32/LPR rows at once, persistent warps walk the row groups and the NEXT group's loads are issued before the
// current group is reduced (register double buffering), so every warp always has loads in flight.  Exact two-pass
// variance in registers as before; results are per-row (batch-invariant).
template <int OPL, int LPR>
__global__ void __launch_bounds__(256)
layernorm_v2_kernel(const void* __restrict__ x, long ldx, void* __restrict__ y, long ldy, const float* __restrict__ gamma,
                    const float* __restrict__ beta, long rows, int C, float eps, int bf16) {
  pdl_trigger();
  pdl_wait();
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPR;
  const int slot = lane / LPR;
  const long nwarps = static_cast<long>(gridDim.x) * (blockDim.x >> 5);
  long grp = static_cast<long>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long ngroups = (rows + RPW - 1) / RPW;
  if (grp >= ngroups) return;
  const bool bf = bf16 != 0;
  const int V = C >> 3;
  const float invc = 1.0f / C;
  auto load = [&](uint4 (&buf)[OPL], long g) {
    const long row = g * RPW + slot;
#pragma unroll
    for (int i = 0; i < OPL; ++i) {
      const int o = sub + i * LPR;
      buf[i] = make_uint4(0, 0, 0, 0);
      if (o < V && row < rows) buf[i] = ldg16(reinterpret_cast<const uint8_t*>(x) + (row * ldx + o * 8) * 2);
    }
  };
  uint4 cur[OPL], nxt[OPL];
  load(cur, grp);
  for (; grp < ngroups; grp += nwarps) {
    const long ng = grp + nwarps;
    if (ng < ngroups) load(nxt, ng);
    const long row = grp * RPW + slot;
    float v[OPL][8];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < OPL; ++i) {
      const uint32_t w[4] = {cur[i].x, cur[i].y, cur[i].z, cur[i].w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack2(w[e], bf);
        v[i][2 * e] = f.x; v[i][2 * e + 1] = f.y;
        sum += f.x + f.y;                   // octets beyond V hold zeros
      }
    }
#pragma unroll
    for (int off = LPR / 2; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
    const float mean = sum * invc;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < OPL; ++i) {
      if (sub + i * LPR < V) {
#pragma unroll
        for (int j = 0; j < 8; ++j) { const float d = v[i][j] - mean; sq += d * d; }
      }
    }
#pragma unroll
    for (int off = LPR / 2; off > 0; off >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, off);
    const float rstd = rsqrtf(sq * invc + eps);
    if (row < rows) {
#pragma unroll
      for (int i = 0; i < OPL; ++i) {
        const int o = sub + i * LPR;
        if (o < V) {
          const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + o * 8));
          const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + o * 8) + 1);
          const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + o * 8));
          const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + o * 8) + 1);
          const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
          const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
          uint32_t ow[4];
#pragma unroll
          for (int e = 0; e < 4; ++e)
            ow[e] = pack2((v[i][2 * e] - mean) * rstd * gg[2 * e] + bb[2 * e],
                          (v[i][2 * e + 1] - mean) * rstd * gg[2 * e + 1] + bb[2 * e + 1], bf);
          *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(y) + (row * ldy + o * 8) * 2) =
              make_uint4(ow[0], ow[1], ow[2], ow[3]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < OPL; ++i) cur[i] = nxt[i];
  }
}

// row softmax: fp32 scores [rows][L] -> 16-bit probabilities (VAE mid-block attention, upcast_softmax semantics)
__global__ void softmax_rows_kernel(const float* __restrict__ s, long lds, void* __restrict__ p, long ldp, int L, int Lpad,
                                    int bf16) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  const long row = blockIdx.x;
  const float* sr = s + row * lds;
  float mx = -INFINITY;
  for (int i = threadIdx.x; i < L; i += blockDim.x) mx = fmaxf(mx, sr[i]);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < (blockDim.x >> 5); ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int i = threadIdx.x; i < L; i += blockDim.x) sum += __expf(sr[i] - mx);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
  for (int i = 0; i < (blockDim.x >> 5); ++i) sum += red[i];
  const float inv = 1.f / sum;
  for (int i = threadIdx.x; i < L; i += blockDim.x) store_elem(p, row * ldp + i, __expf(sr[i] - mx) * inv, bf16 != 0);
  // columns L .. Lpad-1 (K padding of the following P.V GEMM when L % 8 != 0) are zero
  for (int i = L + threadIdx.x; i < Lpad; i += blockDim.x) store_elem(p, row * ldp + i, 0.f, bf16 != 0);
}

}  // namespace aab

using namespace aab;

static int gn_launch_cfg(int C, long samples, long rows, int* threads, int* rows_per_cta, int* chunks) {
  if (C % 8) return AAB_ERR_ARG;
  const int V = C / 8;
  if (V > 1024) return AAB_ERR_ARG;
  int rpi = 256 / V;
  if (rpi < 1) rpi = 1;
  *threads = V * rpi;
  // The row partition depends on (rows, C) only -- never on the number of samples -- so a sample's statistics are
  // summed in the same order whatever batch it arrives in (CFG halves split over two GPUs stay bit-identical to the
  // batched evaluation).  Elements per CTA: 72K for the wide-row levels (C <= 640, or very large samples), 18K where C >= 1280 (few rows per sample: CTA count matters),
  // 12K for tiny samples; at least 8 row-iterations per CTA; at most 1024 chunks per sample.
  (void)samples;
  const long elems = rows * C;
  long tgt = 73728;
  if (elems < (1L << 18)) tgt = 12288;
  else if (C >= 1280 && elems < (1L << 23)) tgt = 18432;
  long rpc = (tgt + C - 1) / C;
  if (rpc < 8L * rpi) rpc = 8L * rpi;
  if ((rows + rpc - 1) / rpc > 1024) rpc = (rows + 1023) / 1024;
  rpc = ((rpc + rpi - 1) / rpi) * rpi;
  *rows_per_cta = static_cast<int>(rpc);
  *chunks = static_cast<int>((rows + rpc - 1) / rpc);
  return AAB_OK;
}

// The apply pass is elementwise: its row partition is free (unlike the statistics pass, whose partition fixes the summation
// order).  The statistics partition can leave a partly filled last wave of CTAs; here the rows are cut so that the launch is
// ~3 waves of CTAs (AAB_GN_APPLY_WAVES; 0 = the statistics partition), each thread still walking >= 4 rows.
static int gn_apply_rows_per_cta(int C, long samples, long rows, int stats_rpc) {
  static int waves = -1;
  if (waves < 0) {
    const char* e = getenv("AAB_GN_APPLY_WAVES");
    waves = e ? atoi(e) : 3;
  }
  if (waves <= 0) return stats_rpc;
  const int V = C / 8;
  int rpi = 256 / V;
  if (rpi < 1) rpi = 1;
  const long slots = 3L * num_sms() * waves;
  long rpc = (rows * samples + slots - 1) / slots;
  if (rpc < 4L * rpi) rpc = 4L * rpi;
  rpc = ((rpc + rpi - 1) / rpi) * rpi;
  if (rpc > stats_rpc) rpc = stats_rpc;
  return static_cast<int>(rpc);
}

// Workspace layout (bytes): a FIXED 16 KiB header of tickets (one u32 per sample) that must be zero before the first use
// and is self-resetting afterwards (fixed offset: calls with different sample counts share one workspace, and a ticket must
// never alias another call's statistics); then mean/rstd floats [samples*groups*2], then double partials
// [samples*chunks*groups*2].
static const long GN_MAX_SAMPLES = 4096;
static const long GN_HEADER_BYTES = GN_MAX_SAMPLES * 4;
extern "C" long aab_groupnorm_workspace_bytes(long samples, long rows, int c, int groups) {
  int threads, rpc, chunks;
  if (gn_launch_cfg(c, samples, rows, &threads, &rpc, &chunks)) return -1;
  if (samples > GN_MAX_SAMPLES) return -1;
  long off = GN_HEADER_BYTES;
  off += ((samples * groups * 2 * 4 + 255) / 256) * 256;
  off += samples * chunks * groups * 2 * 8;
  return off;
}

extern "C" int aab_groupnorm(const void* x1, long ld1, int c1, const void* x2, long ld2, int c2, long samples, long rows,
                             int groups, const float* gamma, const float* beta, float eps, int silu, void* y, long ldy,
                             void* workspace, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int C = c1 + c2;
  if (!x1 || !y || !workspace || groups < 1 || groups > 256 || C % groups || (c1 % 8) || (c2 % 8) || (ld1 % 8) ||
      (ldy % 8))
    return AAB_ERR_ARG;
  if (c2 > 0 && (!x2 || (ld2 % 8))) return AAB_ERR_ARG;
  int threads, rpc, chunks;
  int r = gn_launch_cfg(C, samples, rows, &threads, &rpc, &chunks);
  if (r) return r;
  GnArgs a;
  a.x1 = x1; a.x2 = x2; a.C1 = c1; a.C2 = c2; a.ld1 = ld1; a.ld2 = ld2; a.rows = rows; a.groups = groups;
  a.rows_per_cta = rpc; a.bf16 = is_bf16;
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  if (samples > GN_MAX_SAMPLES) return AAB_ERR_ARG;
  unsigned int* ticket = reinterpret_cast<unsigned int*>(ws);
  long off = GN_HEADER_BYTES;
  float* mean_rstd = reinterpret_cast<float*>(ws + off);
  off += ((samples * groups * 2 * 4 + 255) / 256) * 256;
  double* partial = reinterpret_cast<double*>(ws + off);
  const int rpi = threads / (C / 8);
  size_t smem = static_cast<size_t>(2) * rpi * C * sizeof(float);
  const size_t smem_red = static_cast<size_t>(threads / groups) * groups * 2 * sizeof(double);
  if (smem_red > smem) smem = smem_red;
  if (smem > 48 * 1024 || threads < groups) return AAB_ERR_ARG;
  // Two launches rather than one cooperative grid (statistics -> per-sample flag -> apply): a flag wait would serialise the
  // two phases inside every CTA, while two plain launches let the hardware overlap the tail of one with the head of the next.
  dim3 grid(static_cast<unsigned>(chunks), static_cast<unsigned>(samples));
  launch_k(gn_stats_kernel, dim3(grid), dim3(threads), smem, stream, a, partial, mean_rstd, ticket, eps);
  {
    GnArgs aa = a;
    aa.rows_per_cta = gn_apply_rows_per_cta(C, samples, rows, rpc);
    dim3 ga(static_cast<unsigned>((rows + aa.rows_per_cta - 1) / aa.rows_per_cta), static_cast<unsigned>(samples));
    launch_k(gn_apply_kernel, dim3(ga), dim3(threads), 0, stream, aa, mean_rstd, gamma, beta, silu, y, ldy);
  }
  return cudaGetLastError() == cudaSuccess ? AAB_OK : AAB_ERR_CUDA;
}

// GroupNorm with the statistics pass replaced by the producer's column sums (see gn_finalize_kernel).  colstats1 / colstats2:
// [samples * rows / 128][c1 | c2][2] fp32 as written by aab_igemm (each 128-row tile must lie inside one sample: rows % 128 == 0).
extern "C" int aab_groupnorm_colstats(const void* x1, long ld1, int c1, const float* colstats1, const void* x2, long ld2, int c2,
                                      const float* colstats2, long samples, long rows, int groups, const float* gamma,
                                      const float* beta, float eps, int silu, void* y, long ldy, void* workspace, int is_bf16,
                                      void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const int C = c1 + c2;
  if (!x1 || !y || !workspace || !colstats1 || groups < 1 || groups > 256 || C % groups || (c1 % 8) || (c2 % 8) || (ld1 % 8) ||
      (ldy % 8) || (rows % 128) || samples > GN_MAX_SAMPLES)
    return AAB_ERR_ARG;
  if (c2 > 0 && (!x2 || !colstats2 || (ld2 % 8))) return AAB_ERR_ARG;
  int threads, rpc, chunks;
  int r = gn_launch_cfg(C, samples, rows, &threads, &rpc, &chunks);
  if (r) return r;
  GnArgs a;
  a.x1 = x1; a.x2 = x2; a.C1 = c1; a.C2 = c2; a.ld1 = ld1; a.ld2 = ld2; a.rows = rows; a.groups = groups;
  a.rows_per_cta = rpc; a.bf16 = is_bf16;
  float* mean_rstd = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + GN_HEADER_BYTES);
  const int tps = static_cast<int>(rows / 128);
  const int n = tps * (C / groups);
  int fthreads = 32;
  while (fthreads < n && fthreads < 256) fthreads <<= 1;
  launch_k(gn_finalize_kernel, dim3(static_cast<unsigned>(groups), static_cast<unsigned>(samples)), dim3(fthreads), 0, stream,
           colstats1, c1, colstats2, c2, tps, rows, groups, eps, mean_rstd);
  dim3 grid(static_cast<unsigned>(chunks), static_cast<unsigned>(samples));
  {
    GnArgs aa = a;
    aa.rows_per_cta = gn_apply_rows_per_cta(C, samples, rows, rpc);
    dim3 ga(static_cast<unsigned>((rows + aa.rows_per_cta - 1) / aa.rows_per_cta), static_cast<unsigned>(samples));
    launch_k(gn_apply_kernel, dim3(ga), dim3(threads), 0, stream, aa, mean_rstd, gamma, beta, silu, y, ldy);
  }
  return cudaGetLastError() == cudaSuccess ? AAB_OK : AAB_ERR_CUDA;
}

template <int OPL, int R>
static void launch_ln(const void* x, long ldx, void* y, long ldy, const float* gamma, const float* beta, long rows, int c,
                      float eps, int is_bf16, cudaStream_t stream) {
  const int wpb = 8;
  const long warps = (rows + R - 1) / R;
  launch_k(layernorm_kernel<OPL, R>, dim3(static_cast<unsigned>((warps + wpb - 1) / wpb)), dim3(wpb * 32), 0, stream, 
      x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16);
}

template <int OPL, int LPR>
static void launch_ln2(const void* x, long ldx, void* y, long ldy, const float* gamma, const float* beta, long rows, int c,
                       float eps, int is_bf16, cudaStream_t stream) {
  constexpr int RPW = 32 / LPR;
  const int wpb = 8;
  const long groups = (rows + RPW - 1) / RPW;
  long ctas = (groups + wpb - 1) / wpb;
  const long cap = 6L * aab::num_sms();                 // persistent: ~6 CTAs of 8 warps per SM
  if (ctas > cap) ctas = cap;
  launch_k(layernorm_v2_kernel<OPL, LPR>, dim3(static_cast<unsigned>(ctas)), dim3(wpb * 32), 0, stream, x, ldx, y, ldy, gamma, beta, rows, c,
                                                                                     eps, is_bf16);
}

extern "C" int aab_layernorm(const void* x, long ldx, void* y, long ldy, const float* gamma, const float* beta,
                             long rows, int c, float eps, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !y || (c % 8) || c > 2048 || (ldx % 8) || (ldy % 8)) return AAB_ERR_ARG;
  const int V = c / 8;
  static int use_v1 = -1;                 // AAB_LN_V1=1: the round-1 kernel (A/B measurements)
  if (use_v1 < 0) {
    const char* e = getenv("AAB_LN_V1");
    use_v1 = (e && e[0] == '1') ? 1 : 0;
  }
  if (!use_v1) {
    // lanes per row: the smallest of 8 / 16 / 32 that keeps <= 8 octets per lane, preferring exact fits
    if (V <= 8) launch_ln2<1, 8>(x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16, stream);
    else if (V <= 16) launch_ln2<2, 8>(x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16, stream);
    else if (V <= 24) launch_ln2<3, 8>(x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16, stream);
    else if (V <= 32) launch_ln2<4, 8>(x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16, stream);
    else if (V <= 40) launch_ln2<5, 8>(x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16, stream);
    else if (V <= 64) launch_ln2<4, 16>(x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16, stream);
    else if (V <= 80) launch_ln2<5, 16>(x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16, stream);
    else if (V <= 128) launch_ln2<4, 32>(x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16, stream);
    else if (V <= 160) launch_ln2<5, 32>(x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16, stream);
    else launch_ln2<8, 32>(x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16, stream);
    return cudaGetLastError() == cudaSuccess ? AAB_OK : AAB_ERR_CUDA;
  }
  if (V <= 64) launch_ln<2, 4>(x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16, stream);
  else if (V <= 96) launch_ln<3, 4>(x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16, stream);
  else if (V <= 160) launch_ln<5, 2>(x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16, stream);
  else launch_ln<8, 1>(x, ldx, y, ldy, gamma, beta, rows, c, eps, is_bf16, stream);
  return cudaGetLastError() == cudaSuccess ? AAB_OK : AAB_ERR_CUDA;
}

extern "C" int aab_softmax_rows(const float* s, long lds, void* p, long ldp, long rows, int l, int is_bf16,
                                void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!s || !p || ldp < l) return AAB_ERR_ARG;
  // the probability rows are `ldp` wide: columns l..ldp-1 are written as zeros
  launch_k(softmax_rows_kernel, dim3(static_cast<unsigned>(rows)), dim3(256), 0, stream, s, lds, p, ldp, l, static_cast<int>(ldp), is_bf16);
  return cudaGetLastError() == cudaSuccess ? AAB_OK : AAB_ERR_CUDA;
}
