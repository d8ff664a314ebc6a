// Attention kernels of the denoising path.
//
// 1. aab_flash_attn_d64 — spatial self-attention and text cross-attention of diffusers' BasicTransformerBlock
//    (head_dim 64; reference call sites: Transformer2DModel built at models/unet_3d_blocks.py:287-296,446-456,
//    681-691, processor AttnProcessor2_0 -> F.scaled_dot_product_attention installed by train.py:124-138).
//    Flash-style on the Hopper warpgroup MMA: one CTA owns 128 query rows of one (batch, head), split between two
//    consumer warpgroups of 64 rows.  S = Q.K^T (wgmma, both operands in shared memory) lands in registers, the online
//    softmax (exp2, fp32 running max / sum) runs on those registers, and P is fed back as the register A operand of
//    O += P.V (wgmma, V MN-major in shared memory).  64-key K/V blocks are TMA-loaded into a 3-stage ring by a producer
//    warp.  Keys past Lk (e.g. 77 text tokens) are masked to -inf.
//
// 2. aab_temporal_attn_d64 — self-attention over the frame axis (T <= 32) of TransformerTemporalModel
//    (models/unet_3d_blocks.py:299-306,459-467,694-701; called without encoder_hidden_states so both attn1 and attn2
//    are self-attention over T).  Activations stay in [B, T, H*W, C] order; the kernel gathers the T rows of one
//    (b, position, head) with stride H*W*ld, so no permute to [B*H*W, T, C] is ever materialised.  0.1 % of the
//    FLOPs: CUDA cores, one warp per (position, head).
#include "common.cuh"
#include "igemm.h"
#include "wgmma.cuh"
#include <stdlib.h>

namespace aab {

constexpr int FA_THREADS = 288;       // warpgroups 0, 1: 64 query rows each; warp 8: TMA producer
constexpr int FA_BKV = 64;            // keys per K/V block
constexpr int FA_KV_STAGES = 3;
constexpr int FA_Q_BYTES = 128 * 64 * 2;       // 16 KiB: [128 x 64] 16-bit
constexpr int FA_KV_BYTES = FA_BKV * 64 * 2;   // 8 KiB: [64 x 64] 16-bit
constexpr int FA_SMEM_BYTES = FA_Q_BYTES + FA_KV_STAGES * 2 * FA_KV_BYTES + 1024 + 256;

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

struct FaParams {
  int Lq, Lk, heads, kv_batch_div;
  int q_col0, k_col0, v_col0;
  void* out;
  long ld_out;
  long out_batch_stride;   // elements between consecutive batches of the output
  int out_col0;
  float scale_log2;
  int causal;              // key j visible to query i iff j <= i (CLIP text tower); host guarantees Lq == Lk <= 128
};

// Fragment layout of an m64nN fp32 accumulator (and of the register A operand): thread `lane` of warp `wq` in the warpgroup
// holds, for i in [0, N/2), row 16 wq + lane / 4 + 8 ((i >> 1) & 1) and column 8 (i >> 2) + 2 (lane & 3) + (i & 1).
template <bool BF16>
__global__ void __launch_bounds__(FA_THREADS, 2)
flash_attn_d64_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                      const __grid_constant__ CUtensorMap tmV, const FaParams p) {
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smQ = smem;
  uint8_t* smK = smQ + FA_Q_BYTES;                        // [ST][8K]
  uint8_t* smV = smK + FA_KV_STAGES * FA_KV_BYTES;        // [ST][8K]
  uint64_t* bars = reinterpret_cast<uint64_t*>(smV + FA_KV_STAGES * FA_KV_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;
  uint64_t* kv_empty = kv_full + FA_KV_STAGES;

  const int warp = static_cast<int>(threadIdx.x) >> 5;
  const int q0 = blockIdx.x * 128;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int bkv = b / p.kv_batch_div;
  const int nkv = (p.Lk + FA_BKV - 1) / FA_BKV;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmQ);
    prefetch_tmap(&tmK);
    prefetch_tmap(&tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < FA_KV_STAGES; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 8);         // lane 0 of each consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == 8) {
    if (elect_one()) {
      mbar_arrive_expect_tx(q_full, FA_Q_BYTES);
      tma_load_3d(smQ, &tmQ, q_full, p.q_col0 + head * 64, q0, b);
      for (int j = 0; j < nkv; ++j) {
        const int s = j % FA_KV_STAGES;
        mbar_wait(&kv_empty[s], ((j / FA_KV_STAGES) & 1) ^ 1);
        mbar_arrive_expect_tx(&kv_full[s], 2 * FA_KV_BYTES);
        tma_load_3d(smK + s * FA_KV_BYTES, &tmK, &kv_full[s], p.k_col0 + head * 64, j * FA_BKV, bkv);
        tma_load_3d(smV + s * FA_KV_BYTES, &tmV, &kv_full[s], p.v_col0 + head * 64, j * FA_BKV, bkv);
      }
    }
    return;
  }

  const int cw = warp >> 2;                   // consumer warpgroup: query rows q0 + 64 cw ...
  const int wq = warp & 3;
  const int lane = static_cast<int>(lane_id());
  const int row0 = 64 * cw + 16 * wq + (lane >> 2);     // tile rows row0 and row0 + 8
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const uint32_t qa = smem_u32(smQ + cw * 64 * 128);
  mbar_wait(q_full, 0);

  for (int j = 0; j < nkv; ++j) {
    const int s = j % FA_KV_STAGES;
    mbar_wait(&kv_full[s], (j / FA_KV_STAGES) & 1);
    // ---------------- S = Q K^T   [64 x 64 keys]
    float sc[32];
    const uint32_t ka = smem_u32(smK + s * FA_KV_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma_ss<64, BF16>(sc, make_desc_kmajor_sw128(qa + k * 32), make_desc_kmajor_sw128(ka + k * 32), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<32>(sc);
    // ---------------- mask keys past Lk (and, causal, past the query)
    const int kbase = j * FA_BKV;
    if (p.causal || p.Lk - kbase < FA_BKV) {
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int key = kbase + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
        const int q = q0 + row0 + 8 * ((i >> 1) & 1);
        if (key >= p.Lk || (p.causal && key > q)) sc[i] = -INFINITY;
      }
    }
    // ---------------- online softmax on the two rows of this thread (a row's 64 keys live in the 4 lanes of a quad)
    float alpha[2], m_new[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (((i >> 1) & 1) == h) mx = fmaxf(mx, sc[i]);
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      m_new[h] = fmaxf(m_run[h], mx * p.scale_log2);
      alpha[h] = fast_exp2(m_run[h] - m_new[h]);
      m_run[h] = m_new[h];
    }
    float lsum[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int h = (i >> 1) & 1;
      sc[i] = fast_exp2(fmaf(sc[i], p.scale_log2, -m_new[h]));
      lsum[h] += sc[i];
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) l_run[h] = l_run[h] * alpha[h] + lsum[h];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
    // ---------------- O += P V: P (16-bit) as the register A operand, 16 keys per wgmma
    uint32_t pf[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      pf[kk][0] = pack2(sc[8 * kk + 0], sc[8 * kk + 1], BF16);
      pf[kk][1] = pack2(sc[8 * kk + 2], sc[8 * kk + 3], BF16);
      pf[kk][2] = pack2(sc[8 * kk + 4], sc[8 * kk + 5], BF16);
      pf[kk][3] = pack2(sc[8 * kk + 6], sc[8 * kk + 7], BF16);
    }
    const uint32_t va = smem_u32(smV + s * FA_KV_BYTES);
    fence_regs<32>(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_rs_tb<64, BF16>(o, pf[kk], make_desc_mnmajor_sw128(va + kk * 2048));
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<32>(o);
    if (lane == 0) mbar_arrive(&kv_empty[s]);
  }
  // ---------------- normalise and store
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
    const int q = q0 + row0 + 8 * h;
    if (q < p.Lq) {
      const float inv = 1.0f / l_run[h];
      uint8_t* op = reinterpret_cast<uint8_t*>(p.out) +
                    (static_cast<long>(b) * p.out_batch_stride + static_cast<long>(q) * p.ld_out + p.out_col0 + head * 64 +
                     2 * (lane & 3)) * 2;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(op + jj * 16) = pack2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv, BF16);
    }
  }
}

// ------------------------------------------------------------------------------------------------ temporal
// q/k/v rows of frame t of (b, position pos): base + ((b*T + t)*HW + pos)*ld + col0 + head*64
// One warp per (b, pixel, head).  T <= 32 is far below the 64-row wgmma tile, so the two tiny GEMMs
// (S = Q.K^T: 32x32x64, O = P.V: 32x64x32, T zero-padded to 32) run on warp-level mma.sync m16n8k16 with the online
// softmax on the accumulator fragments (the S fragments are re-used as the A operand of P.V).  Q/K/V rows are gathered
// with coalesced 8-byte loads into padded shared memory (row stride 144 B: conflict-free fragment loads).
template <bool BF16>
__device__ __forceinline__ void mma_16816(float* c, const uint32_t* a, const uint32_t* b) {
  if (BF16)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

constexpr int TA_ROW = 72;                    // halves per smem row (64 + 8 pad)
constexpr int TA_WARP_HALVES = 3 * 32 * TA_ROW;

template <bool BF16>
__global__ void __launch_bounds__(128)
temporal_attn_d64_kernel(const void* __restrict__ qkv, long ld, int q_col0, int k_col0, int v_col0, void* __restrict__ out,
                         long ld_out, int B, int T, int HW, int heads, float scale) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ uint16_t sm16[];
  const int w = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const long item = static_cast<long>(blockIdx.x) * 4 + w;
  const long total = static_cast<long>(B) * HW * heads;
  if (item >= total) return;
  uint16_t* sQ = sm16 + static_cast<size_t>(w) * TA_WARP_HALVES;
  uint16_t* sK = sQ + 32 * TA_ROW;
  uint16_t* sV = sK + 32 * TA_ROW;
  const int head = item % heads;
  const long bp = item / heads;
  const int pos = bp % HW;
  const int b = bp / HW;
  // gather: 16 lanes cover one 128-byte row (8 B per lane), two rows per iteration; rows >= T are zero
  const int sub = lane & 15;
  for (int t = lane >> 4; t < 32; t += 2) {
    uint2 qu = make_uint2(0, 0), ku = make_uint2(0, 0), vu = make_uint2(0, 0);
    if (t < T) {
      const uint8_t* rowp = reinterpret_cast<const uint8_t*>(qkv) +
                            (((static_cast<long>(b) * T + t) * HW + pos) * ld + head * 64 + sub * 4) * 2;
      qu = *reinterpret_cast<const uint2*>(rowp + q_col0 * 2);
      ku = *reinterpret_cast<const uint2*>(rowp + k_col0 * 2);
      vu = *reinterpret_cast<const uint2*>(rowp + v_col0 * 2);
    }
    *reinterpret_cast<uint2*>(sQ + t * TA_ROW + sub * 4) = qu;
    *reinterpret_cast<uint2*>(sK + t * TA_ROW + sub * 4) = ku;
    *reinterpret_cast<uint2*>(sV + t * TA_ROW + sub * 4) = vu;
  }
  __syncwarp();
  const int g = lane >> 2;      // fragment row group
  const int t4 = lane & 3;      // fragment column pair
  // ---------------- S = Q K^T  (2 m-tiles x 4 n-tiles)
  float S[2][4][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int nj = 0; nj < 4; ++nj)
#pragma unroll
      for (int e = 0; e < 4; ++e) S[mi][nj][e] = 0.f;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    uint32_t afr[2][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi) {
      const uint16_t* base = sQ + (16 * mi + g) * TA_ROW + 16 * kk + 2 * t4;
      afr[mi][0] = *reinterpret_cast<const uint32_t*>(base);
      afr[mi][1] = *reinterpret_cast<const uint32_t*>(base + 8 * TA_ROW);
      afr[mi][2] = *reinterpret_cast<const uint32_t*>(base + 8);
      afr[mi][3] = *reinterpret_cast<const uint32_t*>(base + 8 * TA_ROW + 8);
    }
#pragma unroll
    for (int nj = 0; nj < 4; ++nj) {
      uint32_t bfr[2];
      const uint16_t* kb = sK + (8 * nj + g) * TA_ROW + 16 * kk + 2 * t4;
      bfr[0] = *reinterpret_cast<const uint32_t*>(kb);
      bfr[1] = *reinterpret_cast<const uint32_t*>(kb + 8);
      mma_16816<BF16>(S[0][nj], afr[0], bfr);
      mma_16816<BF16>(S[1][nj], afr[1], bfr);
    }
  }
  // ---------------- softmax over the key axis (columns), rows (16 mi + g) and (16 mi + g + 8)
  const float sl2 = scale * 1.4426950408889634f;
  float inv_l[2][2];
  uint32_t pfr[2][2][4];       // P as A fragments: [m-tile][k-step of 16 keys][4]
#pragma unroll
  for (int mi = 0; mi < 2; ++mi) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {          // h = 0: row g, h = 1: row g + 8
      float mx = -INFINITY;
#pragma unroll
      for (int nj = 0; nj < 4; ++nj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * nj + 2 * t4 + e;
          float v = S[mi][nj][2 * h + e] * sl2;
          v = (col < T) ? v : -INFINITY;
          S[mi][nj][2 * h + e] = v;
          mx = fmaxf(mx, v);
        }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      float l = 0.f;
#pragma unroll
      for (int nj = 0; nj < 4; ++nj)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float pv = fast_exp2(S[mi][nj][2 * h + e] - mx);
          S[mi][nj][2 * h + e] = pv;
          l += pv;
        }
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      inv_l[mi][h] = 1.0f / l;
    }
#pragma unroll
    for (int k2 = 0; k2 < 2; ++k2) {
      pfr[mi][k2][0] = pack2(S[mi][2 * k2][0], S[mi][2 * k2][1], BF16);
      pfr[mi][k2][1] = pack2(S[mi][2 * k2][2], S[mi][2 * k2][3], BF16);
      pfr[mi][k2][2] = pack2(S[mi][2 * k2 + 1][0], S[mi][2 * k2 + 1][1], BF16);
      pfr[mi][k2][3] = pack2(S[mi][2 * k2 + 1][2], S[mi][2 * k2 + 1][3], BF16);
    }
  }
  // ---------------- O = P V  (2 m-tiles x 8 n-tiles of d, 2 k-steps of 16 keys)
  float O[2][8][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int dj = 0; dj < 8; ++dj)
#pragma unroll
      for (int e = 0; e < 4; ++e) O[mi][dj][e] = 0.f;
#pragma unroll
  for (int k2 = 0; k2 < 2; ++k2) {
#pragma unroll
    for (int dj = 0; dj < 8; ++dj) {
      const uint16_t* vb = sV + (16 * k2 + 2 * t4) * TA_ROW + 8 * dj + g;
      uint32_t bfr[2];
      bfr[0] = static_cast<uint32_t>(vb[0]) | (static_cast<uint32_t>(vb[TA_ROW]) << 16);
      bfr[1] = static_cast<uint32_t>(vb[8 * TA_ROW]) | (static_cast<uint32_t>(vb[9 * TA_ROW]) << 16);
      mma_16816<BF16>(O[0][dj], pfr[0][k2], bfr);
      mma_16816<BF16>(O[1][dj], pfr[1][k2], bfr);
    }
  }
  // ---------------- normalise and store rows < T
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = 16 * mi + g + 8 * h;
      if (row < T) {
        const float il = inv_l[mi][h];
        uint8_t* op = reinterpret_cast<uint8_t*>(out) +
                      (((static_cast<long>(b) * T + row) * HW + pos) * ld_out + head * 64 + 2 * t4) * 2;
#pragma unroll
        for (int dj = 0; dj < 8; ++dj)
          *reinterpret_cast<uint32_t*>(op + dj * 16) = pack2(O[mi][dj][2 * h] * il, O[mi][dj][2 * h + 1] * il, BF16);
      }
    }
}


// ------------------------------------------------------------------------------------------------ temporal v2
// Same math as temporal_attn_d64_kernel (bit-identical results), restructured for HBM throughput.  Persistent warps walk the
// (b, pixel, head) items;
// the Q/K/V rows of the NEXT item are fetched with 16-byte cp.async copies straight into the second shared-memory buffer
// (408 copies in flight per warp, no registers involved) while the current item is computed; the normalised output is
// staged in shared memory and written with 16-byte stores (one 128-byte row per 8 lanes).
__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

template <bool BF16>
__global__ void __launch_bounds__(128)
temporal_attn_d64_v2_kernel(const void* __restrict__ qkv, long ld, int q_col0, int k_col0, int v_col0,
                            void* __restrict__ out, long ld_out, int B, int T, int HW, int heads, float scale) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ uint16_t sm16[];
  const int w = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const long total = static_cast<long>(B) * HW * heads;
  const long stride = static_cast<long>(gridDim.x) * 4;
  long item = static_cast<long>(blockIdx.x) * 4 + w;
  uint16_t* wbase = sm16 + static_cast<size_t>(w) * 2 * TA_WARP_HALVES;      // two buffers of (Q, K, V)[32][72]
  // rows T..31 of every buffer stay zero for the whole kernel (cp.async only ever writes rows < T)
  for (int i = lane; i < 2 * TA_WARP_HALVES / 8; i += 32) reinterpret_cast<uint4*>(wbase)[i] = make_uint4(0, 0, 0, 0);
  __syncwarp();
  const int col_off[3] = {q_col0, k_col0, v_col0};
  auto prefetch = [&](long it, int buf) {
    const int head = static_cast<int>(it % heads);
    const long bp = it / heads;
    const int pos = static_cast<int>(bp % HW);
    const int b = static_cast<int>(bp / HW);
    uint16_t* dst = wbase + buf * TA_WARP_HALVES;
    const int nchunks = T * 24;                 // T rows x 3 tensors x 8 pieces of 16 bytes
    for (int c = lane; c < nchunks; c += 32) {
      const int t = c / 24;
      const int rem = c - t * 24;
      const int seg = rem >> 3;
      const int part = rem & 7;
      const uint8_t* src = reinterpret_cast<const uint8_t*>(qkv) +
                           (((static_cast<long>(b) * T + t) * HW + pos) * ld + col_off[seg] + head * 64 + part * 8) * 2;
      cp_async_16(dst + seg * 32 * TA_ROW + t * TA_ROW + part * 8, src);
    }
  };
  int buf = 0;
  if (item < total) prefetch(item, 0);
  cp_async_commit();
  const int g = lane >> 2;
  const int t4 = lane & 3;
  const float sl2 = scale * 1.4426950408889634f;
  for (; item < total; item += stride, buf ^= 1) {
    const long nxt = item + stride;
    if (nxt < total) prefetch(nxt, buf ^ 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncwarp();
    uint16_t* sQ = wbase + buf * TA_WARP_HALVES;
    uint16_t* sK = sQ + 32 * TA_ROW;
    uint16_t* sV = sK + 32 * TA_ROW;
    // ---------------- S = Q K^T
    float S[2][4][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int nj = 0; nj < 4; ++nj)
#pragma unroll
        for (int e = 0; e < 4; ++e) S[mi][nj][e] = 0.f;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t afr[2][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const uint16_t* base = sQ + (16 * mi + g) * TA_ROW + 16 * kk + 2 * t4;
        afr[mi][0] = *reinterpret_cast<const uint32_t*>(base);
        afr[mi][1] = *reinterpret_cast<const uint32_t*>(base + 8 * TA_ROW);
        afr[mi][2] = *reinterpret_cast<const uint32_t*>(base + 8);
        afr[mi][3] = *reinterpret_cast<const uint32_t*>(base + 8 * TA_ROW + 8);
      }
#pragma unroll
      for (int nj = 0; nj < 4; ++nj) {
        uint32_t bfr[2];
        const uint16_t* kb = sK + (8 * nj + g) * TA_ROW + 16 * kk + 2 * t4;
        bfr[0] = *reinterpret_cast<const uint32_t*>(kb);
        bfr[1] = *reinterpret_cast<const uint32_t*>(kb + 8);
        mma_16816<BF16>(S[0][nj], afr[0], bfr);
        mma_16816<BF16>(S[1][nj], afr[1], bfr);
      }
    }
    // ---------------- softmax over the keys
    float inv_l[2][2];
    uint32_t pfr[2][2][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float mx = -INFINITY;
#pragma unroll
        for (int nj = 0; nj < 4; ++nj)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * nj + 2 * t4 + e;
            float v = S[mi][nj][2 * h + e] * sl2;
            v = (col < T) ? v : -INFINITY;
            S[mi][nj][2 * h + e] = v;
            mx = fmaxf(mx, v);
          }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        float l = 0.f;
#pragma unroll
        for (int nj = 0; nj < 4; ++nj)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float pv = fast_exp2(S[mi][nj][2 * h + e] - mx);
            S[mi][nj][2 * h + e] = pv;
            l += pv;
          }
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        inv_l[mi][h] = 1.0f / l;
      }
#pragma unroll
      for (int k2 = 0; k2 < 2; ++k2) {
        pfr[mi][k2][0] = pack2(S[mi][2 * k2][0], S[mi][2 * k2][1], BF16);
        pfr[mi][k2][1] = pack2(S[mi][2 * k2][2], S[mi][2 * k2][3], BF16);
        pfr[mi][k2][2] = pack2(S[mi][2 * k2 + 1][0], S[mi][2 * k2 + 1][1], BF16);
        pfr[mi][k2][3] = pack2(S[mi][2 * k2 + 1][2], S[mi][2 * k2 + 1][3], BF16);
      }
    }
    // ---------------- O = P V
    float O[2][8][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int dj = 0; dj < 8; ++dj)
#pragma unroll
        for (int e = 0; e < 4; ++e) O[mi][dj][e] = 0.f;
#pragma unroll
    for (int k2 = 0; k2 < 2; ++k2) {
#pragma unroll
      for (int dj = 0; dj < 8; ++dj) {
        const uint16_t* vb = sV + (16 * k2 + 2 * t4) * TA_ROW + 8 * dj + g;
        uint32_t bfr[2];
        bfr[0] = static_cast<uint32_t>(vb[0]) | (static_cast<uint32_t>(vb[TA_ROW]) << 16);
        bfr[1] = static_cast<uint32_t>(vb[8 * TA_ROW]) | (static_cast<uint32_t>(vb[9 * TA_ROW]) << 16);
        mma_16816<BF16>(O[0][dj], pfr[0][k2], bfr);
        mma_16816<BF16>(O[1][dj], pfr[1][k2], bfr);
      }
    }
    // ---------------- normalise -> stage in the Q buffer (all Q reads of this warp are done) -> 16-byte row stores
    __syncwarp();
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = 16 * mi + g + 8 * h;
        const float il = inv_l[mi][h];
        uint16_t* orow = sQ + row * TA_ROW + 2 * t4;
#pragma unroll
        for (int dj = 0; dj < 8; ++dj)
          *reinterpret_cast<uint32_t*>(orow + dj * 8) = pack2(O[mi][dj][2 * h] * il, O[mi][dj][2 * h + 1] * il, BF16);
      }
    __syncwarp();
    {
      const int head = static_cast<int>(item % heads);
      const long bp = item / heads;
      const int pos = static_cast<int>(bp % HW);
      const int b = static_cast<int>(bp / HW);
      for (int c = lane; c < T * 8; c += 32) {
        const int t = c >> 3;
        const int part = c & 7;
        const uint4 v = *reinterpret_cast<const uint4*>(sQ + t * TA_ROW + part * 8);
        *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(out) +
                                  (((static_cast<long>(b) * T + t) * HW + pos) * ld_out + head * 64 + part * 8) * 2) = v;
      }
    }
    __syncwarp();
    // rows >= T of the Q buffer were overwritten by the staging (rows 16 mi + g + 8 h cover all 32): zero them again
    for (int c = lane; c < (32 - T) * 9; c += 32) {
      const int r = T + c / 9;
      reinterpret_cast<uint4*>(sQ + r * TA_ROW)[c % 9] = make_uint4(0, 0, 0, 0);
    }
    __syncwarp();
  }
  cp_async_wait<0>();
}

}  // namespace aab

using namespace aab;

extern "C" int aab_flash_attn_d64(const void* q, long ldq, long q_batch_stride, int q_cols, int q_col0,
                                  const void* kv, long ldkv, long kv_batch_stride, int kv_cols, int k_col0, int v_col0,
                                  void* out, long ld_out, long out_batch_stride, int out_col0, int nb, int nb_kv,
                                  int kv_batch_div, int heads, int lq, int lk, float scale, int is_bf16, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  // bit 1 of `is_bf16` selects the causal variant (CLIP text self-attention, transformers CLIPAttention with
  // causal_attention_mask; reached from models/pipeline.py:136 _encode_prompt); one KV block only
  const int causal = (is_bf16 >> 1) & 1;
  is_bf16 &= 1;
  if (causal && (lq != lk || lk > 128)) return AAB_ERR_ARG;
  if (!q || !kv || !out || lq < 1 || lk < 1 || heads < 1 || nb < 1 || kv_batch_div < 1) return AAB_ERR_ARG;
  if ((ldq % 8) || (ldkv % 8) || (ld_out % 8) || (out_col0 % 8)) return AAB_ERR_ARG;
  CUtensorMap tmQ, tmK, tmV;
  {
    long dims[3] = {q_cols, lq, nb};
    long strides[3] = {1, ldq, q_batch_stride};
    int box[3] = {64, 128, 1};
    int r = make_tmap_16(&tmQ, q, 3, dims, strides, box, is_bf16);
    if (r) return r;
  }
  {
    long dims[3] = {kv_cols, lk, nb_kv};
    long strides[3] = {1, ldkv, kv_batch_stride};
    int box[3] = {64, FA_BKV, 1};
    int r = make_tmap_16(&tmK, kv, 3, dims, strides, box, is_bf16);
    if (r) return r;
    tmV = tmK;
  }
  FaParams p;
  p.Lq = lq;
  p.Lk = lk;
  p.heads = heads;
  p.kv_batch_div = kv_batch_div;
  p.q_col0 = q_col0;
  p.k_col0 = k_col0;
  p.v_col0 = v_col0;
  p.out = out;
  p.ld_out = ld_out;
  p.out_batch_stride = out_batch_stride;
  p.out_col0 = out_col0;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.causal = causal;
  const dim3 grid((lq + 127) / 128, heads, nb);
  if (is_bf16) {
    static std::atomic<unsigned long long> attr_b{0};
    if (int r = ensure_dyn_smem(flash_attn_d64_kernel<true>, FA_SMEM_BYTES, attr_b)) return r;
    launch_k(flash_attn_d64_kernel<true>, grid, dim3(FA_THREADS), FA_SMEM_BYTES, stream, tmQ, tmK, tmV, p);
  } else {
    static std::atomic<unsigned long long> attr_h{0};
    if (int r = ensure_dyn_smem(flash_attn_d64_kernel<false>, FA_SMEM_BYTES, attr_h)) return r;
    launch_k(flash_attn_d64_kernel<false>, grid, dim3(FA_THREADS), FA_SMEM_BYTES, stream, tmQ, tmK, tmV, p);
  }
  return cudaGetLastError() == cudaSuccess ? AAB_OK : AAB_ERR_CUDA;
}

extern "C" int aab_temporal_attn_d64(const void* qkv, long ld, int q_col0, int k_col0, int v_col0, void* out,
                                     long ld_out, int b, int t, int hw, int heads, float scale, int is_bf16,
                                     void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!qkv || !out || t < 1 || t > 32 || (ld % 8) || (ld_out % 8)) return AAB_ERR_ARG;
  const long total = static_cast<long>(b) * hw * heads;
  static int use_v1 = -1;                 // AAB_TATTN_V1=1: the round-1 kernel (A/B measurements)
  if (use_v1 < 0) {
    const char* e = getenv("AAB_TATTN_V1");
    use_v1 = (e && e[0] == '1') ? 1 : 0;
  }
  if (!use_v1) {
    if ((q_col0 | k_col0 | v_col0) % 8) return AAB_ERR_ARG;     // 16-byte cp.async pieces
    const size_t smem2 = static_cast<size_t>(4) * 2 * TA_WARP_HALVES * sizeof(uint16_t);   // 108 KiB: double-buffered Q, K, V
    static std::atomic<unsigned long long> a2t{0}, a2f{0};
    if (int r = ensure_dyn_smem(temporal_attn_d64_v2_kernel<true>, static_cast<int>(smem2), a2t)) return r;
    if (int r = ensure_dyn_smem(temporal_attn_d64_v2_kernel<false>, static_cast<int>(smem2), a2f)) return r;
    long ctas = (total + 3) / 4;
    const long cap = 2L * num_sms();                              // two 108 KiB CTAs per SM, persistent
    const int grid2 = static_cast<int>(ctas < cap ? ctas : cap);
    if (is_bf16)
      launch_k(temporal_attn_d64_v2_kernel<true>, dim3(grid2), dim3(128), smem2, stream, qkv, ld, q_col0, k_col0, v_col0, out, ld_out, b, t, hw,
                                                                       heads, scale);
    else
      launch_k(temporal_attn_d64_v2_kernel<false>, dim3(grid2), dim3(128), smem2, stream, qkv, ld, q_col0, k_col0, v_col0, out, ld_out, b, t, hw,
                                                                        heads, scale);
    return cudaGetLastError() == cudaSuccess ? AAB_OK : AAB_ERR_CUDA;
  }
  const int grid = static_cast<int>((total + 3) / 4);
  const size_t smem = static_cast<size_t>(4) * TA_WARP_HALVES * sizeof(uint16_t);   // 54 KiB: Q, K, V padded to 32 rows
  static std::atomic<unsigned long long> attr_t{0}, attr_f{0};
  if (int r = ensure_dyn_smem(temporal_attn_d64_kernel<true>, 65536, attr_t)) return r;
  if (int r = ensure_dyn_smem(temporal_attn_d64_kernel<false>, 65536, attr_f)) return r;
  if (is_bf16)
    launch_k(temporal_attn_d64_kernel<true>, dim3(grid), dim3(128), smem, stream, qkv, ld, q_col0, k_col0, v_col0, out, ld_out, b, t, hw,
                                                                heads, scale);
  else
    launch_k(temporal_attn_d64_kernel<false>, dim3(grid), dim3(128), smem, stream, qkv, ld, q_col0, k_col0, v_col0, out, ld_out, b, t, hw,
                                                                 heads, scale);
  return cudaGetLastError() == cudaSuccess ? AAB_OK : AAB_ERR_CUDA;
}
