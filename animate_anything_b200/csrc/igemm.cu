// Implicit-GEMM on the Hopper warpgroup MMA (wgmma) for every dense contraction of the denoising path:
//   Linear / 1x1 conv (1 tap), conv3x3 (9 taps over H,W), temporal conv (3,1,1) (3 taps over T),
//   stride-2 conv (9 taps over a space-to-depth view), batched Q.K^T / P.V for the VAE attention.
//
//   D[pixels, N] = act( sum_taps A_tap[pixels, Kc] . B[N, tap*Kc : (tap+1)*Kc]^T + bias + bias2[sample] + residual ) * s
//
// * A (activations, channels-last) is never im2col'd: every tap is a TMA box load of the same 5-D tensor map at a
//   shifted pixel coordinate; out-of-bounds pixels are zero-filled by the TMA unit (= conv zero padding).
// * B (weights, [N, K] K-contiguous) is TMA-loaded; both land in shared memory in the 128B-swizzled K-major layout
//   that wgmma reads through matrix descriptors.  A stage ring of mbarrier-guarded buffers feeds the tensor cores.
// * Warp specialisation: warp 0 of warpgroup 0 is the TMA producer (one elected thread), warps 1 - 3 of warpgroup 0 are
//   the epilogue warps, warpgroups 1 and 2 each own 64 rows of the 128 x BN tile and keep their accumulators in registers
//   (m64nBNk16 wgmma, fp32).
// * Persistent CTAs (one per SM) walk the tile list n-fastest so that the CTAs running concurrently share the same
//   A rows (L2 hits) while the weights stay L2-resident; the producer runs ahead into the next tile while the
//   consumers finish the epilogue of the current one.
// * Two CTAs per SM (AAB_F_TWO_CTA, template MINB = 2, 64-column tiles, 3-stage ring, 80 registers per thread) for the
//   1-tap launches with K <= 640 (ops.pick_two_cta): their main loop is only 5 - 10 k-blocks, so with one CTA the tensor
//   cores idle through every ring refill; the second CTA's MMAs run under it.  Same control flow, K order and epilogue:
//   bit-identical to one CTA per SM.
// * Tile widths 32 / 64 / 128 / 160 / 192 / 256: the caller fits the width to N and to the number of tiles per wave, because
//   a ragged last N tile costs no traffic (TMA zero-fill) but issues every wgmma of its dead columns.
// * Staged epilogue (16-bit outputs TMA can address): the consumers add bias / per-sample bias (time embedding) / residual,
//   apply SiLU or the GEGLU gate and round, writing in place over the residual in a 128 x OUT_BN shared-memory staging tile,
//   and go straight back to the main loop of their next tile.  The producer thread loads the residual into the staging tile
//   by TMA; the epilogue warps stage the tile's bias rows in shared memory, take the per-tile column statistics for the
//   GroupNorm that follows from the staged 16-bit values, and store the tile by TMA.  fp32 / odd-N / scaled outputs are
//   stored per element from the registers (direct epilogue).
//
// Replaces, for the reference path (SURVEY.md section 8a): cuDNN conv2d/conv3d and cuBLAS linear calls made by
// diffusers ResnetBlock2D / TemporalConvLayer / Transformer2DModel / TransformerTemporalModel / AutoencoderKL
// (models/unet_3d_blocks.py:262-306,425-467,564-583,660-701,794-813).
#include "common.cuh"
#include "igemm.h"
#include "wgmma.cuh"

namespace aab {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;       // 16 KiB
constexpr int NUM_CONSUMERS = 2;                 // consumer warpgroups, 64 tile rows each
constexpr int NUM_THREADS = 128 * (1 + NUM_CONSUMERS);
constexpr int NUM_CONSUMER_THREADS = 128 * NUM_CONSUMERS;
constexpr int NUM_EPI_THREADS = 96;              // warps 1 - 3 of warpgroup 0: column statistics and the output store

// staged epilogue: the 128 x OUT_BN 16-bit output tile sits in shared memory as OUT_BN / 32 sub-tiles of 128 rows x 64 bytes
// in the TMA SWIZZLE_64B layout (16-byte chunk c of row r at chunk c ^ ((r >> 1) & 3)): one TMA box each way, and a warp's
// accumulator-layout 4-byte accesses (8 rows x 4 words of one chunk) fall on 32 distinct banks
constexpr int SUB_COLS = 32;
constexpr int SUB_BYTES = BM * SUB_COLS * 2;     // 8 KiB

// Shared-memory ring and register split per tile width, CTAs per SM (MINB) and GEGLU (half as many output columns).
//   MINB = 1: the ring, the output staging tile (128 x OUT_BN x 2 bytes) and the tile's bias rows inside the 227 KiB a block
//             may use; the producer warpgroup gives registers to the consumers (56 / 224: the epilogue warps spill below 56).
//             BN 256 keeps 3 stages (212.3 KiB), BN 192 4 (211.5), BN 160 5 (223.1), BN 128 6 (226.8), BN 64 8 (210),
//             GEGLU 256 4 (226.8), GEGLU 128 6 (210).
//   MINB = 2: the short-K 1-tap launches (ops.pick_two_cta), 64-column tiles only: two CTAs per SM, so that one CTA's
//             main loop runs while the other waits for its ring refill.  Shared memory: a CTA gets at most 113 KiB (half of
//             the SM's 228 KiB less the 1 KiB reserved per CTA); 3 stages = 72 KiB of operands + 16 KiB staging tile + bias +
//             pad = 90 KiB (a fourth stage would need 114).  Registers: __launch_bounds__(384, 2) caps every thread at
//             80 (2 x 384 x 80 <= 64 K), 30 720 per CTA >= producer 56 + consumers 88.  The compiler allocates the consumer
//             code within the 80 of the launch bounds: the 32 accumulators of BN = 64 fit with no spill, the 64 of
//             BN = 128 (and so GEGLU) do not compile.  The producer and epilogue warps spill below 56.
template <int BN, int MINB = 1, bool GEGLU = false>
struct Cfg {
  static_assert(MINB == 1 || (MINB == 2 && BN == 64 && !GEGLU), "two CTAs per SM are instantiated at BN = 64 only");
  static constexpr int OUT_BN = GEGLU ? BN / 2 : BN;
  static constexpr int STAGES = (MINB == 2) ? 3 : (BN == 256) ? (GEGLU ? 4 : 3) : (BN == 192) ? 4 : (BN == 160) ? 5
                                : (BN == 128) ? 6 : 8;
  static constexpr int PRODUCER_REGS = 56;
  static constexpr int CONSUMER_REGS = (MINB == 2) ? 88 : 224;
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int OUT_BYTES = BM * OUT_BN * 2;
  static constexpr int BIAS_FLOATS = 3 * OUT_BN;   // bias | per-sample bias of the tile's first and last sample (GEGLU: bias of values | gates)
  static constexpr int SMEM_BYTES = STAGES * (A_STAGE_BYTES + B_STAGE_BYTES) + OUT_BYTES + BIAS_FLOATS * 4 +
                                    1024 /*align*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= (MINB == 2 ? 113 : 227) * 1024, "tile configuration exceeds the shared memory of an SM");
  static_assert(B_STAGE_BYTES % 1024 == 0, "the staging tile must stay 1024-byte aligned for its swizzle");
  static_assert(128 * PRODUCER_REGS + 128 * NUM_CONSUMERS * CONSUMER_REGS <= NUM_THREADS * (MINB == 2 ? 80 : 168),
                "setmaxnreg split exceeds the registers the launch bounds give a CTA");
};

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == AAB_ACT_SILU) return silu_f(x);
  if (act == AAB_ACT_GELU) return gelu_erf_f(x);
  if (act == AAB_ACT_QUICK_GELU) return quick_gelu_f(x);
  return x;
}

template <int BN, bool BF16>
__device__ __forceinline__ void mma_kblock(float* acc, uint32_t a_addr, uint32_t b_addr, bool first) {
#pragma unroll
  for (int k = 0; k < BK / 16; ++k) {
    const uint64_t da = make_desc_kmajor_sw128(a_addr + k * 32);
    const uint64_t db = make_desc_kmajor_sw128(b_addr + k * 32);
    const uint32_t sc = (first && k == 0) ? 0u : 1u;
    wgmma_ss<BN, BF16>(acc, da, db, sc);
  }
}

// byte offset of the 4-byte word (row r, column pair cp) in the staging tile
__device__ __forceinline__ int stage_word_off(int r, int cp) {
  return (cp >> 4) * SUB_BYTES + r * (SUB_COLS * 2) + ((((cp >> 2) & 3) ^ ((r >> 1) & 3)) << 4) + (cp & 3) * 4;
}

// GEGLU: B tile = [values | gates] (BN/2 rows each), out = value * gelu(gate), BN/2 columns.
// Epilogue flavours (runtime, uniform per launch):
//   staged  (no AAB_F_DIRECT): n_out % 32 == 0, 16-bit output, rows TMA can address, at most one of residual / per-sample
//                              bias / SiLU, no scaling; the consumers convert into the shared-memory staging tile and go
//                              back to their main loop, warps 1 - 3 take the column statistics and store the tile by TMA;
//                              the residual comes in by TMA
//   direct  (AAB_F_DIRECT):    any n_out, fp32 or 16-bit output, every flag combination, masked per element
//
// Staged epilogue barriers, one phase per tile of the CTA (j = the CTA's tile count so far, parity j & 1):
//   free  (96 arrivals):       the epilogue warps have read tile j's staging tile and its TMA store has read it too.  The
//                              producer waits for phase j - 1 (parity (j & 1) ^ 1: passes at once for j = 0) after it has
//                              issued every k-block of tile j, so the ring never waits for an epilogue.
//   ready (1 + 96 arrivals):   the producer (with the residual's TMA bytes, 0 without a residual) and the epilogue warps
//                              (tile j's bias rows are in shared memory); the consumers wait for it after their main loop.
//   full  (256 arrivals):      every consumer thread has written its part of tile j (and fenced it for the async proxy);
//                              the epilogue warps wait for it.  They stage tile j + 1's bias only after it, so the bias
//                              buffer is single.
// Each barrier's phase j + 1 can only start after phase j has completed (ready(j + 1) follows full(j), full(j + 1) follows
// ready(j + 1), free(j + 1) follows full(j + 1)), so one parity bit per barrier is enough.  A ragged last n-tile moves only
// its n_out - n0 columns (whole sub-tiles); rows outside the tensor are zero-filled on the residual load and clipped on the
// store by the TMA unit, and the column statistics skip them.  A CTA with no tile runs none of this.
template <int BN, int MINB, bool GEGLU, bool BF16>
__global__ void __launch_bounds__(NUM_THREADS, MINB)
igemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
             const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmOut,
             const __grid_constant__ CUtensorMap tmRes, const IgemmParams p) {
  using CF = Cfg<BN, MINB, GEGLU>;
  constexpr int STAGES = CF::STAGES;
  constexpr int OUT_BN = CF::OUT_BN;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smA = smem;
  uint8_t* smB = smA + STAGES * A_STAGE_BYTES;
  uint8_t* stile = smB + STAGES * CF::B_STAGE_BYTES;
  float* sbias = reinterpret_cast<float*>(stile + CF::OUT_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(sbias + CF::BIAS_FLOATS);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;
  uint64_t* free_bar = bars + 2 * STAGES;
  uint64_t* ready_bar = free_bar + 1;
  uint64_t* out_full_bar = free_bar + 2;

  const int wg = static_cast<int>(threadIdx.x) >> 7;
  const int warp = static_cast<int>(threadIdx.x) >> 5;
  constexpr bool bf16 = BF16;
  const int tile_first = static_cast<int>(blockIdx.x);
  const int tile_step = static_cast<int>(gridDim.x);
  const int num_tiles = p.num_m_tiles * p.num_n_tiles;
  const int kb_per_tap = p.kb_per_tap;
  const int k_iters = p.num_taps * kb_per_tap;
  const bool direct = (p.flags & AAB_F_DIRECT) != 0;
  const bool staged = BN >= 64 && (GEGLU || !direct);
  const bool has_res = !GEGLU && p.residual != nullptr;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmA2);
    prefetch_tmap(&tmB);
    if (staged) {
      prefetch_tmap(&tmOut);
      if (has_res) prefetch_tmap(&tmRes);
    }
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], NUM_CONSUMERS * 4);   // lane 0 of every consumer warp releases a stage
    }
    mbar_init(free_bar, NUM_EPI_THREADS);
    mbar_init(ready_bar, 1 + NUM_EPI_THREADS);
    mbar_init(out_full_bar, NUM_CONSUMER_THREADS);
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<CF::PRODUCER_REGS>();
    if (warp == 0) {
      // ===================================================== TMA producer
      if (!elect_one()) return;
      // the weight tile is fetched in NS row slices of BN / NS rows (GEGLU: values and gates are separate slices)
      constexpr int NS = GEGLU ? 2 : 1;
      constexpr int slice_rows = BN / NS;
      uint32_t it = 0, j = 0;
      for (int tile = tile_first; tile < num_tiles; tile += tile_step) {
        const int nt = tile % p.num_n_tiles;
        int mt = tile / p.num_n_tiles;
        int cb[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          cb[i] = (mt % p.tiles[i]) * p.box[i];
          mt /= p.tiles[i];
        }
        const int bbatch = (p.b_batch_dim >= 0) ? cb[p.b_batch_dim] : 0;
        const int n0 = nt * OUT_BN;
        for (int tap = 0; tap < p.num_taps; ++tap) {
          const int o0 = p.tap_off[tap][0], o1 = p.tap_off[tap][1], o2 = p.tap_off[tap][2], o3 = p.tap_off[tap][3],
                    o4 = p.tap_off[tap][4];
          for (int kb = 0; kb < kb_per_tap; ++kb, ++it) {
            const int s = it % STAGES;
            const uint32_t ph = (it / STAGES) & 1;
            mbar_wait(&empty_bar[s], ph ^ 1);
            const int kc = kb * BK;
            const int kg = tap * p.Kc + kc;
            mbar_arrive_expect_tx(&full_bar[s], A_STAGE_BYTES + CF::B_STAGE_BYTES);
            if (kc < p.Kc1)
              tma_load_5d(smA + s * A_STAGE_BYTES, &tmA, &full_bar[s], kc + o0, cb[0] + o1, cb[1] + o2, cb[2] + o3,
                          cb[3] + o4);
            else
              tma_load_5d(smA + s * A_STAGE_BYTES, &tmA2, &full_bar[s], kc - p.Kc1 + o0, cb[0] + o1, cb[1] + o2,
                          cb[2] + o3, cb[3] + o4);
#pragma unroll
            for (int jn = 0; jn < NS; ++jn) {
              const int t0 = jn * slice_rows;                       // first tile row of the slice
              const int row = (GEGLU && t0 >= BN / 2) ? p.N / 2 + n0 + (t0 - BN / 2) : n0 + t0;
              tma_load_3d(smB + s * CF::B_STAGE_BYTES + t0 * 128, &tmB, &full_bar[s], kg, row, bbatch);
            }
          }
        }
        if (staged) {
          // this tile's staging tile, once the previous tile's has been stored, with the residual in it
          mbar_wait(free_bar, (j & 1) ^ 1);
          const int nsub = min(OUT_BN, p.n_out - n0) / SUB_COLS;
          if (has_res) {
            mbar_arrive_expect_tx(ready_bar, nsub * SUB_BYTES);
            for (int s = 0; s < nsub; ++s)
              tma_load_5d(stile + s * SUB_BYTES, &tmRes, ready_bar, n0 + s * SUB_COLS, cb[0], cb[1], cb[2], cb[3]);
          } else {
            mbar_arrive(ready_bar);
          }
          ++j;
        }
      }
      return;
    }
    if (!staged) return;
    // ===================================================== epilogue warps: bias rows in, column statistics, TMA store out
    const int et = static_cast<int>(threadIdx.x) - 32;
    const bool stats = !GEGLU && p.colstats != nullptr;
    uint32_t j = 0;
    for (int tile = tile_first; tile < num_tiles; tile += tile_step, ++j) {
      const int nt = tile % p.num_n_tiles;
      int mt = tile / p.num_n_tiles;
      const int mt_lin = mt;                                   // linear m-tile index (row of the column-statistics table)
      int cb[4], lim[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        cb[i] = (mt % p.tiles[i]) * p.box[i];
        mt /= p.tiles[i];
        lim[i] = min(p.box[i], p.dimD[i] - cb[i]);             // rows of the tile inside the tensor along dim i
      }
      const int n0 = nt * OUT_BN;
      const int ncols = min(OUT_BN, p.n_out - n0);
      // this tile's bias (GEGLU: values | gates) and the per-sample bias of its first and last row's sample (host: a tile
      // spans at most two samples); the consumers have read the previous tile's (full barrier below)
      if (p.bias != nullptr)
        for (int c = et; c < ncols; c += NUM_EPI_THREADS) {
          sbias[c] = __ldg(p.bias + n0 + c);
          if (GEGLU) sbias[OUT_BN + c] = __ldg(p.bias + p.N / 2 + n0 + c);
        }
      if (!GEGLU && p.bias2 != nullptr) {
        // (the host keeps the output rows of a staged launch below 2^31)
        const int g_first = ((cb[3] * p.dimD[2] + cb[2]) * p.dimD[1] + cb[1]) * p.dimD[0] + cb[0];
        const int g_last = ((((cb[3] + lim[3] - 1) * p.dimD[2] + cb[2] + lim[2] - 1) * p.dimD[1] + cb[1] + lim[1] - 1) *
                            p.dimD[0]) + cb[0] + lim[0] - 1;
        const float* b0 = p.bias2 + static_cast<long>(g_first / p.rows_per_bias2) * p.ld_bias2 + n0;
        const float* b1 = p.bias2 + static_cast<long>(g_last / p.rows_per_bias2) * p.ld_bias2 + n0;
        for (int c = et; c < ncols; c += NUM_EPI_THREADS) {
          sbias[OUT_BN + c] = __ldg(b0 + c);
          sbias[2 * OUT_BN + c] = __ldg(b1 + c);
        }
      }
      mbar_arrive(ready_bar);
      mbar_wait(out_full_bar, j & 1);
      if (et == 0) {
        for (int s = 0; s < ncols / SUB_COLS; ++s)
          tma_store_5d(&tmOut, stile + s * SUB_BYTES, n0 + s * SUB_COLS, cb[0], cb[1], cb[2], cb[3]);
        tma_store_commit();
      }
      if (stats) {
        // one column per thread, in the float order of the accumulator layout: consumer warp w holds rows 16 w .. 16 w + 15,
        // its lane-row r (0..7) sums (0 + v[r]) + v[r + 8] over valid rows, the xor-4 / 8 / 16 butterfly combines the lane-rows
        // as ((p0 + p1) + (p2 + p3)) + ((p4 + p5) + (p6 + p7)), and the 8 warps are added in order
        uint32_t vmask[4];                                     // bit r & 31 of word r >> 5: tile row r is inside the tensor
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          int r = static_cast<int>(lane_id()) + 32 * k;
          bool v = true;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            v = v && (r % p.box[i] < lim[i]);
            r /= p.box[i];
          }
          vmask[k] = __ballot_sync(0xffffffffu, v);
        }
        for (int c = et; c < ncols; c += NUM_EPI_THREADS) {
          auto ld = [&](int r) {
            const uint16_t u = *reinterpret_cast<const uint16_t*>(stile + stage_word_off(r, c >> 1) + 2 * (c & 1));
            return bf16 ? __uint_as_float(static_cast<uint32_t>(u) << 16) : __half2float(__ushort_as_half(u));
          };
          float tot_s = 0.f, tot_q = 0.f;
#pragma unroll 1
          for (int w = 0; w < NUM_CONSUMERS * 4; ++w) {
            const uint32_t vw = w < 2 ? vmask[0] : w < 4 ? vmask[1] : w < 6 ? vmask[2] : vmask[3];
            const uint32_t vrows = (w & 1) ? vw >> 16 : vw;    // rows 16 w .. 16 w + 15
            float ts[4], tq[4];                                // (p0 + p1), (p2 + p3), (p4 + p5), (p6 + p7)
#pragma unroll
            for (int r = 0; r < 8; r += 2) {
              float s2[2], q2[2];
#pragma unroll
              for (int u = 0; u < 2; ++u) {
                float s = 0.f, q = 0.f;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const int row = 16 * w + r + u + 8 * h;
                  if ((vrows >> (r + u + 8 * h)) & 1) {
                    const float v = ld(row);
                    s += v;
                    q = fmaf(v, v, q);
                  }
                }
                s2[u] = s;
                q2[u] = q;
              }
              ts[r / 2] = s2[0] + s2[1];
              tq[r / 2] = q2[0] + q2[1];
            }
            tot_s += (ts[0] + ts[1]) + (ts[2] + ts[3]);
            tot_q += (tq[0] + tq[1]) + (tq[2] + tq[3]);
          }
          float* cs = p.colstats + (static_cast<long>(mt_lin) * p.n_out + n0 + c) * 2;
          cs[0] = tot_s;
          cs[1] = tot_q;
        }
      }
      if (et == 0) tma_store_wait_read<0>();
      mbar_arrive(free_bar);
    }
    return;
  }

  // ===================================================== consumers: warpgroup cw owns tile rows [64 cw, 64 cw + 64)
  setmaxnreg_inc<CF::CONSUMER_REGS>();
  const int cw = wg - 1;
  const int wq = warp & 3;
  const int lane = static_cast<int>(lane_id());
  const bool out_f32 = (p.flags & AAB_F_OUT_F32) != 0;
  const bool scale_acc = (p.flags & AAB_F_SCALE_ACC) != 0;
  uint32_t it = 0, j = 0;

  for (int tile = tile_first; tile < num_tiles; tile += tile_step) {
    float acc[BN / 2];                  // the first wgmma of a tile overwrites it (scale-d = 0)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    // ---------------- main loop: one k-block of wgmmas in flight while the previous one retires and frees its stage
    for (int ki = 0; ki < k_iters; ++ki, ++it) {
      const int s = it % STAGES;
      mbar_wait(&full_bar[s], (it / STAGES) & 1);
      fence_regs<BN / 2>(acc);
      wgmma_fence();
      mma_kblock<BN, BF16>(acc, smem_u32(smA + s * A_STAGE_BYTES + cw * 64 * 128),
                           smem_u32(smB + s * CF::B_STAGE_BYTES), ki == 0);
      wgmma_commit();
      fence_regs<BN / 2>(acc);
      if (ki > 0) {
        wgmma_wait<1>();
        fence_regs<BN / 2>(acc);
        if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
      }
    }
    wgmma_wait<0>();
    fence_regs<BN / 2>(acc);
    if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);

    // ---------------- epilogue
    const int nt = tile % p.num_n_tiles;
    int mt = tile / p.num_n_tiles;
    int cb[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      cb[i] = (mt % p.tiles[i]) * p.box[i];
      mt /= p.tiles[i];
    }
    // this thread's two accumulator rows: r and r + 8 of the tile
    long grow[2];
    bool rvalid[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      int rr = cw * 64 + wq * 16 + (lane >> 2) + 8 * h;
      int g[4];
      bool v = true;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        g[i] = cb[i] + rr % p.box[i];
        rr /= p.box[i];
        v = v && (g[i] < p.dimD[i]);
      }
      rvalid[h] = v;
      grow[h] = ((static_cast<long>(g[3]) * p.dimD[2] + g[2]) * p.dimD[1] + g[1]) * p.dimD[0] + g[0];
    }
    const int n0 = nt * OUT_BN;
    const bool has_bias2 = p.bias2 != nullptr;

    if (GEGLU || !direct) {
      if constexpr (BN >= 64) {
        // ---- staged: bias, per-sample bias, residual, activation and rounding in the accumulator layout, written in place
        // over the residual in the staging tile; the warps 1 - 3 of warpgroup 0 take it from there
        const int q = lane & 3;
        const int r0 = cw * 64 + wq * 16 + (lane >> 2);        // tile rows r0 and r0 + 8
        const int nslab = min(OUT_BN, p.n_out - n0) / SUB_COLS;   // n_out is a multiple of 32
        int bsel[2] = {0, 0};                                  // per-sample bias row of each accumulator row (0: first sample)
        if (!GEGLU && has_bias2) {
          const long s_first =
              (((static_cast<long>(cb[3]) * p.dimD[2] + cb[2]) * p.dimD[1] + cb[1]) * p.dimD[0] + cb[0]) / p.rows_per_bias2;
#pragma unroll
          for (int h = 0; h < 2; ++h) bsel[h] = (grow[h] / p.rows_per_bias2 > s_first) ? 2 * OUT_BN : OUT_BN;
        }
        mbar_wait(ready_bar, j & 1);
#pragma unroll
        for (int s = 0; s < OUT_BN / SUB_COLS; ++s) {
          if (s >= nslab) break;                               // warp-uniform: a ragged last n-tile
#pragma unroll
          for (int jc = 0; jc < SUB_COLS / 8; ++jc) {
            const int jj = s * (SUB_COLS / 8) + jc;
            const int cl = jj * 8 + 2 * q;                     // tile column of this thread's pair
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float x[2] = {acc[4 * jj + 2 * h], acc[4 * jj + 2 * h + 1]};
              uint32_t* wp = reinterpret_cast<uint32_t*>(stile + stage_word_off(r0 + 8 * h, cl >> 1));
              if (GEGLU) {
                float g[2] = {acc[4 * (jj + BN / 16) + 2 * h], acc[4 * (jj + BN / 16) + 2 * h + 1]};
                if (p.bias != nullptr) {
                  const float2 bv = *reinterpret_cast<const float2*>(sbias + cl);
                  const float2 bg = *reinterpret_cast<const float2*>(sbias + OUT_BN + cl);
                  x[0] += bv.x; x[1] += bv.y;
                  g[0] += bg.x; g[1] += bg.y;
                }
                *wp = pack2(x[0] * gelu_fast_f(g[0]), x[1] * gelu_fast_f(g[1]), bf16);
              } else {
                if (p.bias != nullptr) {
                  const float2 b = *reinterpret_cast<const float2*>(sbias + cl);
                  x[0] += b.x; x[1] += b.y;
                }
                if (has_bias2 && rvalid[h]) {
                  const float2 b = *reinterpret_cast<const float2*>(sbias + bsel[h] + cl);
                  x[0] += b.x; x[1] += b.y;
                }
                if (has_res) {
                  const float2 r = unpack2(*wp, bf16);
                  x[0] += r.x; x[1] += r.y;
                }
                if (p.act == AAB_ACT_SILU) {
                  x[0] = silu_fast_f(x[0]);
                  x[1] = silu_fast_f(x[1]);
                }
                *wp = pack2(x[0], x[1], bf16);
              }
            }
          }
        }
        fence_proxy_async_smem();                              // the TMA store reads what this thread wrote
        mbar_arrive(out_full_bar);
        ++j;
      }
    } else if constexpr (!GEGLU) {
      auto bias2row = [&](int h) { return p.bias2 + (grow[h] / p.rows_per_bias2) * p.ld_bias2; };
      auto resrow = [&](int h) { return reinterpret_cast<const uint8_t*>(p.residual) + grow[h] * p.ld_res * 2; };
      // ---- direct: masked per element, straight from the accumulator registers
#pragma unroll
      for (int jj = 0; jj < OUT_BN / 8; ++jj) {
        const int col = n0 + jj * 8 + 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (col + e < p.n_out) {
              float v = acc[4 * jj + 2 * h + e];
              if (p.bias != nullptr) v += __ldg(p.bias + col + e);
              if (has_bias2 && rvalid[h]) v += __ldg(bias2row(h) + col + e);
              if (scale_acc) {
                v = apply_act(v, p.act) * p.out_scale;
                if (p.residual != nullptr && rvalid[h]) v += load_elem(resrow(h), col + e, bf16);
              } else {
                if (p.residual != nullptr && rvalid[h]) v += load_elem(resrow(h), col + e, bf16);
                v = apply_act(v, p.act) * p.out_scale;
              }
              if (rvalid[h]) {
                if (out_f32) reinterpret_cast<float*>(p.out)[grow[h] * p.ld_out + col + e] = v;
                else store_elem(p.out, grow[h] * p.ld_out + col + e, v, bf16);
              }
            }
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || ptr == nullptr) return nullptr;
  fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  return fn;
}

// rank-`rank` 16-bit tensor map, dims/strides innermost first (strides in elements, strides[0] must be 1)
int make_tmap_16(CUtensorMap* out, const void* base, int rank, const long* dims, const long* strides, const int* box,
                 int is_bf16, int swizzle_bytes) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return AAB_ERR_DRIVER;
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = static_cast<cuuint64_t>(dims[i]);
    bx[i] = static_cast<cuuint32_t>(box[i]);
    es[i] = 1;
    if (i > 0) gstr[i - 1] = static_cast<cuuint64_t>(strides[i]) * 2;
  }
  CUresult r = enc(out, is_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                   static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim, gstr, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle_bytes == 32   ? CU_TENSOR_MAP_SWIZZLE_32B
                   : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                         : CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? AAB_OK : AAB_ERR_DRIVER;
}

static int g_num_sms = 0;
int num_sms() {
  if (g_num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}

template <int BN, int MINB, bool GEGLU, bool BF16>
static int launch_t(const CUtensorMap& a, const CUtensorMap& a2, const CUtensorMap& b, const CUtensorMap& o,
                    const CUtensorMap& r, const IgemmParams& p, cudaStream_t stream) {
  using CF = Cfg<BN, MINB, GEGLU>;
  static std::atomic<unsigned long long> attr_done{0};
  if (int r = ensure_dyn_smem(igemm_kernel<BN, MINB, GEGLU, BF16>, CF::SMEM_BYTES, attr_done)) return r;
  const int tiles = p.num_m_tiles * p.num_n_tiles;
  int ctas = num_sms() * MINB;     // persistent: MINB CTAs per SM
  if (tiles < ctas) ctas = tiles;
  igemm_kernel<BN, MINB, GEGLU, BF16><<<ctas, NUM_THREADS, CF::SMEM_BYTES, stream>>>(a, a2, b, o, r, p);
  return cudaGetLastError() == cudaSuccess ? AAB_OK : AAB_ERR_CUDA;
}

template <int BN, bool GEGLU, int MINB = 1>
static int launch_bn(const CUtensorMap& a, const CUtensorMap& a2, const CUtensorMap& b, const CUtensorMap& o,
                     const CUtensorMap& r, const IgemmParams& p, cudaStream_t stream) {
  if (p.flags & AAB_F_BF16) return launch_t<BN, MINB, GEGLU, true>(a, a2, b, o, r, p, stream);
  return launch_t<BN, MINB, GEGLU, false>(a, a2, b, o, r, p, stream);
}

}  // namespace aab

using namespace aab;

// 1 when this launch takes a staged epilogue -- the only ones that can emit `colstats` -- else 0
static int igemm_is_staged(const AabIgemmDesc* d) {
  const bool geglu = (d->flags & AAB_F_GEGLU) != 0;
  const int bn = d->block_n;
  const int n_out = geglu ? d->n / 2 : d->n;
  if ((d->flags & (AAB_F_DIRECT | AAB_F_OUT_F32 | AAB_F_SCALE_ACC)) || bn == 32 || (d->ld_out % 8) || (n_out % 32)) return 0;
  // the output (and the residual) move as TMA boxes of a 5-D map [pixel dims][n_out]: 16-byte aligned base, row strides a
  // multiple of 16 bytes, every stride below 2^40 bytes; fewer than 2^31 rows (32-bit row arithmetic in the epilogue warps)
  long rows = 1;
  for (int i = 0; i < 4; ++i) rows *= d->dim_d[i] > 0 ? d->dim_d[i] : 1;
  if (rows >= (1l << 31) || reinterpret_cast<uintptr_t>(d->out) % 16 || rows * d->ld_out * 2 >= (1l << 40)) return 0;
  if (d->residual && ((d->ld_res % 8) || reinterpret_cast<uintptr_t>(d->residual) % 16 || rows * d->ld_res * 2 >= (1l << 40)))
    return 0;
  if (d->bias2) {
    // the epilogue holds the per-sample bias of two samples per tile: the rows a tile can span must fit in one sample
    long span = 1, pitch = 1;
    for (int i = 0; i < 4; ++i) {
      span += static_cast<long>(d->box[i] - 1) * pitch;
      pitch *= d->dim_d[i];
    }
    if (span > (d->rows_per_bias2 > 0 ? d->rows_per_bias2 : 1)) return 0;
  }
  if ((d->act == AAB_ACT_GELU || d->act == AAB_ACT_QUICK_GELU) && !geglu) return 0;
  const int extras = (d->residual ? 1 : 0) + (d->bias2 ? 1 : 0) + (d->act == AAB_ACT_SILU ? 1 : 0);
  if (!geglu && (extras > 1 || d->out_scale != 1.0f)) return 0;
  return 1;
}

extern "C" int aab_igemm_emits_colstats(const AabIgemmDesc* d) {
  return (d && d->colstats && !(d->flags & AAB_F_GEGLU) && igemm_is_staged(d)) ? 1 : 0;
}

extern "C" int aab_igemm(const AabIgemmDesc* d, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!d || !d->a || !d->b || !d->out) return AAB_ERR_ARG;
  if (d->flags & ~(AAB_F_BF16 | AAB_F_DIRECT | AAB_F_OUT_F32 | AAB_F_GEGLU | AAB_F_SCALE_ACC | AAB_F_TWO_CTA)) return AAB_ERR_ARG;
  const int is_bf16 = (d->flags & AAB_F_BF16) ? 1 : 0;
  const bool geglu = (d->flags & AAB_F_GEGLU) != 0;
  int bn = d->block_n;
  if (bn != 32 && bn != 64 && bn != 128 && bn != 160 && bn != 192 && bn != 256) return AAB_ERR_ARG;
  const int n_out = geglu ? d->n / 2 : d->n;
  // staged: one extra term (residual | per-sample bias | SiLU), no output scaling, output and residual addressable by TMA
  const bool direct = !igemm_is_staged(d);
  if (geglu) {   // the gate half of the tile must be a whole number of 64-column blocks; GEGLU only has the staged epilogue
    if ((bn != 128 && bn != 256) || direct || d->residual || d->bias2 || d->act == AAB_ACT_SILU || d->out_scale != 1.0f)
      return AAB_ERR_ARG;
  }
  const bool two_cta = (d->flags & AAB_F_TWO_CTA) != 0;
  if (two_cta && (bn != 64 || geglu)) return AAB_ERR_ARG;   // the one width instantiated with MINB = 2
  if (d->num_taps < 1 || d->num_taps > AAB_MAX_TAPS) return AAB_ERR_ARG;
  if (d->kc % 8 != 0) return AAB_ERR_ARG;
  if (d->a2 && (d->kc1 % 64 != 0)) return AAB_ERR_ARG;

  IgemmParams p;
  memset(&p, 0, sizeof(p));
  long box_prod = 1;
  p.num_m_tiles = 1;
  for (int i = 0; i < 4; ++i) {
    p.dimD[i] = d->dim_d[i];
    p.box[i] = d->box[i];
    if (p.box[i] < 1 || p.dimD[i] < 1) return AAB_ERR_ARG;
    p.tiles[i] = (p.dimD[i] + p.box[i] - 1) / p.box[i];
    p.num_m_tiles *= p.tiles[i];
    box_prod *= p.box[i];
  }
  if (box_prod != BM) return AAB_ERR_ARG;
  const int out_bn = geglu ? bn / 2 : bn;
  p.num_n_tiles = (n_out + out_bn - 1) / out_bn;
  p.N = d->n;
  p.n_out = n_out;
  p.Kc = d->kc;
  p.Kc1 = d->a2 ? d->kc1 : (1 << 30);
  p.num_taps = d->num_taps;
  p.kb_per_tap = (d->kc + BK - 1) / BK;
  for (int t = 0; t < d->num_taps; ++t)
    for (int j = 0; j < 5; ++j) p.tap_off[t][j] = d->tap_off[t][j];
  p.b_batch_dim = d->b_batch_dim;
  p.bias = d->bias;
  p.bias2 = d->bias2;
  p.rows_per_bias2 = d->rows_per_bias2 > 0 ? d->rows_per_bias2 : 1;
  p.ld_bias2 = d->ld_bias2;
  p.residual = d->residual;
  p.ld_res = d->ld_res;
  p.out = d->out;
  p.ld_out = d->ld_out;
  p.out_scale = d->out_scale;
  p.act = d->act;
  p.flags = d->flags | (direct ? AAB_F_DIRECT : 0);
  p.colstats = direct ? nullptr : d->colstats;   // staged epilogues only (the caller checks the result of aab_igemm_emits_colstats)

  CUtensorMap tmA, tmA2, tmB;
  {
    int box[5] = {BK, d->box[0], d->box[1], d->box[2], d->box[3]};
    int r = make_tmap_16(&tmA, d->a, 5, d->a_dims, d->a_strides, box, is_bf16, 128);
    if (r) return r;
    if (d->a2) {
      r = make_tmap_16(&tmA2, d->a2, 5, d->a2_dims, d->a2_strides, box, is_bf16, 128);
      if (r) return r;
    } else {
      tmA2 = tmA;
    }
  }
  {
    long dims[3] = {static_cast<long>(d->num_taps) * d->kc, d->n, d->b_batch > 0 ? d->b_batch : 1};
    long strides[3] = {1, d->ld_b, d->b_batch_stride > 0 ? d->b_batch_stride : static_cast<long>(d->n) * d->ld_b};
    int box[3] = {BK, geglu ? bn / 2 : bn, 1};      // one weight-tile slice (GEGLU: values and gates, see the producer)
    int r = make_tmap_16(&tmB, d->b, 3, dims, strides, box, is_bf16, 128);
    if (r) return r;
  }
  CUtensorMap tmOut = tmA, tmRes = tmA;   // staged epilogue only: the output tile leaves and the residual comes in by TMA
  if (!direct) {
    long dims[5] = {n_out, d->dim_d[0], d->dim_d[1], d->dim_d[2], d->dim_d[3]};
    long strides[5] = {1, d->ld_out, 0, 0, 0};
    for (int i = 2; i < 5; ++i) strides[i] = strides[i - 1] * dims[i - 1];
    int box[5] = {SUB_COLS, d->box[0], d->box[1], d->box[2], d->box[3]};
    int r = make_tmap_16(&tmOut, d->out, 5, dims, strides, box, is_bf16, 64);
    if (r) return r;
    if (d->residual && !geglu) {
      strides[1] = d->ld_res;
      for (int i = 2; i < 5; ++i) strides[i] = strides[i - 1] * dims[i - 1];
      r = make_tmap_16(&tmRes, d->residual, 5, dims, strides, box, is_bf16, 64);
      if (r) return r;
    }
  }
  if (two_cta) return launch_bn<64, false, 2>(tmA, tmA2, tmB, tmOut, tmRes, p, stream);
  if (geglu) {
    if (bn == 128) return launch_bn<128, true>(tmA, tmA2, tmB, tmOut, tmRes, p, stream);
    return launch_bn<256, true>(tmA, tmA2, tmB, tmOut, tmRes, p, stream);
  }
  switch (bn) {
    case 32: return launch_bn<32, false>(tmA, tmA2, tmB, tmOut, tmRes, p, stream);
    case 64: return launch_bn<64, false>(tmA, tmA2, tmB, tmOut, tmRes, p, stream);
    case 128: return launch_bn<128, false>(tmA, tmA2, tmB, tmOut, tmRes, p, stream);
    case 160: return launch_bn<160, false>(tmA, tmA2, tmB, tmOut, tmRes, p, stream);
    case 192: return launch_bn<192, false>(tmA, tmA2, tmB, tmOut, tmRes, p, stream);
    default: return launch_bn<256, false>(tmA, tmA2, tmB, tmOut, tmRes, p, stream);
  }
}

extern "C" int aab_num_sms(void) { return aab::num_sms(); }
