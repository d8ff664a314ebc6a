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
// * Warp specialisation: warpgroup 0 is the TMA producer (one elected thread), warpgroups 1 and 2 each own 64 rows of
//   the 128 x BN tile and keep their accumulators in registers (m64nBNk16 wgmma, fp32).
// * Persistent CTAs (one per SM) walk the tile list n-fastest so that the CTAs running concurrently share the same
//   A rows (L2 hits) while the weights stay L2-resident; the producer runs ahead into the next tile while the
//   consumers finish the epilogue of the current one.
// * Clusters (IgemmParams::cluster = 2 or 4, 256-column tiles): the CTAs of a cluster take consecutive m-tiles of the same
//   n-tile; each fetches 1/cluster of the weight tile and multicasts it to all of them, so a k-block reads the weights from
//   L2 once per cluster instead of once per CTA.  A stage is refilled only after the consumers of every CTA of the cluster
//   have released it.  Same K order, same epilogue: bit-identical to single CTAs.
// * Epilogue straight from the accumulator registers: bias / per-sample bias (time embedding) / residual / activation
//   / GEGLU gate -> 16-bit (or fp32) stores, masked at the tile edges, plus optional per-tile column statistics for the
//   GroupNorm that follows.
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
constexpr int NUM_CONSUMER_WARPS = 4 * NUM_CONSUMERS;

// smem ring depth per tile width: 192 KiB (160 KiB for BN = 32) of operands in flight whatever BN, plus the column-statistics
// scratch, inside the 227 KiB a block may use
template <int BN>
struct Cfg {
  static constexpr int STAGES = (BN == 256) ? 4 : (BN == 128) ? 6 : 8;
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STATS_BYTES = NUM_CONSUMER_WARPS * BN * 2 * 4;   // per-warp (sum, sum of squares) per column
  static constexpr int SMEM_BYTES = STAGES * (A_STAGE_BYTES + B_STAGE_BYTES) + STATS_BYTES + 1024 /*align*/ +
                                    256 /*barriers*/;
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

// GEGLU: B tile = [values | gates] (BN/2 rows each), out = value * gelu(gate), BN/2 columns.
// Epilogue flavours (runtime, uniform per launch):
//   staged  (no AAB_F_DIRECT): n_out % 32 == 0, 16-bit output, at most one of residual / per-sample bias / SiLU, no scaling;
//                              column pairs are stored as 32-bit words; may emit column statistics
//   direct  (AAB_F_DIRECT):    any n_out, fp32 or 16-bit output, every flag combination, masked per element
template <int BN, bool GEGLU, bool BF16>
__global__ void __launch_bounds__(NUM_THREADS, 1)
igemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
             const __grid_constant__ CUtensorMap tmB, const IgemmParams p) {
  pdl_trigger();
  using CF = Cfg<BN>;
  constexpr int STAGES = CF::STAGES;
  constexpr int OUT_BN = GEGLU ? BN / 2 : BN;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smA = smem;
  uint8_t* smB = smA + STAGES * A_STAGE_BYTES;
  float* sstats = reinterpret_cast<float*>(smB + STAGES * CF::B_STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sstats) + CF::STATS_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;

  const int wg = static_cast<int>(threadIdx.x) >> 7;
  const int warp = static_cast<int>(threadIdx.x) >> 5;
  constexpr bool bf16 = BF16;
  // cluster tiles: CL consecutive m-tiles x one n-tile; this CTA owns m-tile CL * (tile / num_n_tiles) + crank.  With a
  // number of m-tiles that CL does not divide, the CTAs past the end load m-tile 0 (the cluster moves in lockstep) and
  // store nothing.
  const int CL = p.cluster;
  const int crank = CL > 1 ? static_cast<int>(cluster_ctarank()) : 0;
  const int tile_first = static_cast<int>(blockIdx.x) / CL;
  const int tile_step = static_cast<int>(gridDim.x) / CL;
  const int num_tiles = ((p.num_m_tiles + CL - 1) / CL) * p.num_n_tiles;
  const int kb_per_tap = p.kb_per_tap;
  const int k_iters = p.num_taps * kb_per_tap;

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmA2);
    prefetch_tmap(&tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], NUM_CONSUMER_WARPS * CL);   // lane 0 of every consumer warp of the cluster releases a stage
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (CL > 1) cluster_sync_all();     // the other CTAs' barriers are initialised before anything is signalled into them
  pdl_wait();       // everything above (barriers, descriptor prefetch) overlapped the previous kernel's tail

  if (wg == 0) {
    // ===================================================== TMA producer
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      // the weight tile is fetched in NS row slices of BN / NS rows (GEGLU: values and gates are separate slices); CTA crank
      // of the cluster fetches slices crank, crank + CL, ... and multicasts them
      const int NS = (CL > 1 || !GEGLU) ? CL : 2;
      const int slice_rows = BN / (NS > 1 ? NS : 1);
      const uint16_t mask = static_cast<uint16_t>((1u << CL) - 1u);
      uint32_t it = 0;
      for (int tile = tile_first; tile < num_tiles; tile += tile_step) {
        const int nt = tile % p.num_n_tiles;
        int mt = (tile / p.num_n_tiles) * CL + crank;
        if (mt >= p.num_m_tiles) mt = 0;
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
            mbar_wait_cluster(&empty_bar[s], ph ^ 1);
            const int kc = kb * BK;
            const int kg = tap * p.Kc + kc;
            mbar_arrive_expect_tx(&full_bar[s], A_STAGE_BYTES + CF::B_STAGE_BYTES);
            if (kc < p.Kc1)
              tma_load_5d(smA + s * A_STAGE_BYTES, &tmA, &full_bar[s], kc + o0, cb[0] + o1, cb[1] + o2, cb[2] + o3,
                          cb[3] + o4);
            else
              tma_load_5d(smA + s * A_STAGE_BYTES, &tmA2, &full_bar[s], kc - p.Kc1 + o0, cb[0] + o1, cb[1] + o2,
                          cb[2] + o3, cb[3] + o4);
            for (int j = crank; j < (NS > 1 ? NS : 1); j += CL) {
              const int t0 = j * slice_rows;                        // first tile row of the slice
              const int row = (GEGLU && t0 >= BN / 2) ? p.N / 2 + n0 + (t0 - BN / 2) : n0 + t0;
              uint8_t* dst = smB + s * CF::B_STAGE_BYTES + t0 * 128;
              if (CL > 1) tma_load_3d_mcast(dst, &tmB, &full_bar[s], kg, row, bbatch, mask);
              else tma_load_3d(dst, &tmB, &full_bar[s], kg, row, bbatch);
            }
          }
        }
      }
    }
    if (CL > 1) {                     // no CTA leaves while a peer may still multicast into it or release its stages
      __syncwarp();
      cluster_sync_all();
    }
    return;
  }

  // ===================================================== consumers: warpgroup cw owns tile rows [64 cw, 64 cw + 64)
  setmaxnreg_inc<232>();
  const int cw = wg - 1;
  const int wq = warp & 3;
  const int lane = static_cast<int>(lane_id());
  const bool direct = (p.flags & AAB_F_DIRECT) != 0;
  const bool out_f32 = (p.flags & AAB_F_OUT_F32) != 0;
  const bool scale_acc = (p.flags & AAB_F_SCALE_ACC) != 0;
  const bool stats = !GEGLU && !direct && p.colstats != nullptr;
  uint32_t it = 0;

  auto release = [&](uint32_t stage) {
    if (lane != 0) return;
    if (CL > 1) {
      for (int r = 0; r < CL; ++r) mbar_arrive_cluster(&empty_bar[stage], static_cast<uint32_t>(r));
    } else {
      mbar_arrive(&empty_bar[stage]);
    }
  };

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
        release((it - 1) % STAGES);
      }
    }
    wgmma_wait<0>();
    fence_regs<BN / 2>(acc);
    release((it - 1) % STAGES);

    // ---------------- epilogue
    const int nt = tile % p.num_n_tiles;
    int mt = (tile / p.num_n_tiles) * CL + crank;
    const bool tile_ok = mt < p.num_m_tiles;                 // a cluster CTA past the last m-tile stores nothing
    if (!tile_ok) mt = 0;
    const int mt_lin = mt;                                  // linear m-tile index (row of the column-statistics table)
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
      rvalid[h] = v && tile_ok;
      grow[h] = ((static_cast<long>(g[3]) * p.dimD[2] + g[2]) * p.dimD[1] + g[1]) * p.dimD[0] + g[0];
    }
    const int n0 = nt * OUT_BN;
    const float* bias2row[2];
    const uint8_t* resrow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      bias2row[h] = (p.bias2 != nullptr && rvalid[h]) ? p.bias2 + (grow[h] / p.rows_per_bias2) * p.ld_bias2 : nullptr;
      resrow[h] = (p.residual != nullptr && rvalid[h])
                      ? reinterpret_cast<const uint8_t*>(p.residual) + grow[h] * p.ld_res * 2
                      : nullptr;
    }
    if (stats) named_bar_sync(1, 128 * NUM_CONSUMERS);     // the previous tile's statistics scratch has been read

#pragma unroll
    for (int jj = 0; jj < OUT_BN / 8; ++jj) {
      const int cl = jj * 8 + 2 * (lane & 3);                // tile column of this thread's pair
      const int col = n0 + cl;
      float ssum[2] = {0.f, 0.f}, ssq[2] = {0.f, 0.f};
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float x[2] = {acc[4 * jj + 2 * h], acc[4 * jj + 2 * h + 1]};
        if (GEGLU) {
          float g[2] = {acc[4 * (jj + BN / 16) + 2 * h], acc[4 * (jj + BN / 16) + 2 * h + 1]};
          if (col < p.n_out) {
            if (p.bias != nullptr) {
              const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + col));
              const float2 bg = __ldg(reinterpret_cast<const float2*>(p.bias + p.N / 2 + col));
              x[0] += bv.x; x[1] += bv.y;
              g[0] += bg.x; g[1] += bg.y;
            }
            if (rvalid[h]) {
              const uint32_t o = pack2(x[0] * gelu_fast_f(g[0]), x[1] * gelu_fast_f(g[1]), bf16);
              *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(p.out) + (grow[h] * p.ld_out + col) * 2) = o;
            }
          }
        } else if (!direct) {
          if (col < p.n_out) {
            if (p.bias != nullptr) {
              const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + col));
              x[0] += b.x; x[1] += b.y;
            }
            if (bias2row[h] != nullptr) {
              const float2 b = __ldg(reinterpret_cast<const float2*>(bias2row[h] + col));
              x[0] += b.x; x[1] += b.y;
            }
            if (resrow[h] != nullptr) {
              const float2 r = unpack2(__ldg(reinterpret_cast<const unsigned int*>(resrow[h] + col * 2)), bf16);
              x[0] += r.x; x[1] += r.y;
            }
            if (p.act == AAB_ACT_SILU) {
              x[0] = silu_fast_f(x[0]);
              x[1] = silu_fast_f(x[1]);
            }
            const uint32_t o = pack2(x[0], x[1], bf16);
            if (rvalid[h]) {
              *reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(p.out) + (grow[h] * p.ld_out + col) * 2) = o;
              if (stats) {
                const float2 f = unpack2(o, bf16);           // statistics of the ROUNDED 16-bit outputs
                ssum[0] += f.x; ssq[0] = fmaf(f.x, f.x, ssq[0]);
                ssum[1] += f.y; ssq[1] = fmaf(f.y, f.y, ssq[1]);
              }
            }
          }
        } else {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (col + e < p.n_out) {
              float v = x[e];
              if (p.bias != nullptr) v += __ldg(p.bias + col + e);
              if (bias2row[h] != nullptr) v += __ldg(bias2row[h] + col + e);
              if (scale_acc) {
                v = apply_act(v, p.act) * p.out_scale;
                if (resrow[h] != nullptr) v += load_elem(resrow[h], col + e, bf16);
              } else {
                if (resrow[h] != nullptr) v += load_elem(resrow[h], col + e, bf16);
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
      if (stats) {
        // sum over the warp's 16 rows: the 8 lanes sharing (lane & 3) hold this column pair; fixed-order butterfly
#pragma unroll
        for (int off = 4; off < 32; off <<= 1) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            ssum[e] += __shfl_xor_sync(0xffffffffu, ssum[e], off);
            ssq[e] += __shfl_xor_sync(0xffffffffu, ssq[e], off);
          }
        }
        if (lane < 4) {
          float* sp = sstats + ((cw * 4 + wq) * BN + cl) * 2;
          sp[0] = ssum[0]; sp[1] = ssq[0]; sp[2] = ssum[1]; sp[3] = ssq[1];
        }
      }
    }
    if (stats) {
      // the eight warps' partial sums, added in warp order -> one (sum, sumsq) pair per column and m-tile, reproducible
      named_bar_sync(1, 128 * NUM_CONSUMERS);
      for (int c = static_cast<int>(threadIdx.x) - 128; c < OUT_BN && tile_ok; c += 128 * NUM_CONSUMERS) {
        if (n0 + c >= p.n_out) break;
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int w = 0; w < NUM_CONSUMER_WARPS; ++w) {
          s0 += sstats[(w * BN + c) * 2];
          s1 += sstats[(w * BN + c) * 2 + 1];
        }
        p.colstats[(static_cast<long>(mt_lin) * p.n_out + n0 + c) * 2] = s0;
        p.colstats[(static_cast<long>(mt_lin) * p.n_out + n0 + c) * 2 + 1] = s1;
      }
    }
  }
  if (CL > 1) cluster_sync_all();
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
                   swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
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

template <int BN, bool GEGLU, bool BF16>
static int launch_t(const CUtensorMap& a, const CUtensorMap& a2, const CUtensorMap& b, const IgemmParams& p,
                    int max_ctas, cudaStream_t stream) {
  using CF = Cfg<BN>;
  static std::atomic<unsigned long long> attr_done{0};
  if (int r = ensure_dyn_smem(igemm_kernel<BN, GEGLU, BF16>, CF::SMEM_BYTES, attr_done)) return r;
  const int cl = p.cluster;
  const int tiles = ((p.num_m_tiles + cl - 1) / cl) * p.num_n_tiles;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.blockDim = dim3(NUM_THREADS);
  cfg.dynamicSmemBytes = CF::SMEM_BYTES;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int na = 0;
  if (cl > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = static_cast<unsigned>(cl);
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  if (pdl_enabled()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  int clusters = num_sms() / cl;
  if (cl > 1) {
    // a cluster's CTAs must fit inside one GPC: ask the driver how many clusters can be resident at once (cached per device)
    static std::atomic<int> max_clusters[64];
    int dev = 0;
    cudaGetDevice(&dev);
    int mc = max_clusters[dev & 63].load(std::memory_order_acquire);
    if (mc == 0) {
      cfg.gridDim = dim3(static_cast<unsigned>(cl * clusters));
      int n = 0;
      if (cudaOccupancyMaxActiveClusters(&n, igemm_kernel<BN, GEGLU, BF16>, &cfg) != cudaSuccess || n < 1) {
        cudaGetLastError();
        n = 1;
      }
      mc = n;
      max_clusters[dev & 63].store(mc, std::memory_order_release);
    }
    if (clusters > mc) clusters = mc;
  }
  if (tiles < clusters) clusters = tiles;
  if (max_ctas > 0 && clusters > max_ctas / cl) clusters = max_ctas / cl > 0 ? max_ctas / cl : 1;
  cfg.gridDim = dim3(static_cast<unsigned>(cl * clusters));
  const cudaError_t e = cudaLaunchKernelEx(&cfg, igemm_kernel<BN, GEGLU, BF16>, a, a2, b, p);
  return e == cudaSuccess ? AAB_OK : AAB_ERR_CUDA;
}

template <int BN, bool GEGLU>
static int launch_bn(const CUtensorMap& a, const CUtensorMap& a2, const CUtensorMap& b, const IgemmParams& p,
                     int max_ctas, cudaStream_t stream) {
  if (p.flags & AAB_F_BF16) return launch_t<BN, GEGLU, true>(a, a2, b, p, max_ctas, stream);
  return launch_t<BN, GEGLU, false>(a, a2, b, p, max_ctas, stream);
}

}  // namespace aab

using namespace aab;

// 1 when this launch takes a staged epilogue -- the only ones that can emit `colstats` -- else 0
static int igemm_is_staged(const AabIgemmDesc* d) {
  const bool geglu = (d->flags & AAB_F_GEGLU) != 0;
  const int bn = d->block_n;
  const int n_out = geglu ? d->n / 2 : d->n;
  if ((d->flags & (AAB_F_DIRECT | AAB_F_OUT_F32 | AAB_F_SCALE_ACC)) || bn == 32 || (d->ld_out % 8) || (n_out % 32)) return 0;
  if (d->residual && (d->ld_res % 8)) return 0;
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
  const int is_bf16 = (d->flags & AAB_F_BF16) ? 1 : 0;
  const bool geglu = (d->flags & AAB_F_GEGLU) != 0;
  int bn = d->block_n;
  if (bn != 32 && bn != 64 && bn != 128 && bn != 256) return AAB_ERR_ARG;
  bool direct = (d->flags & AAB_F_DIRECT) != 0;
  const int n_out = geglu ? d->n / 2 : d->n;
  if (bn == 32 || (d->ld_out % 8) != 0 || (n_out % 32) != 0 || (d->flags & AAB_F_OUT_F32)) direct = true;
  if (geglu && (bn < 128 || direct)) return AAB_ERR_ARG;   // the gate half of the tile must be a whole number of 64-column blocks
  if (d->residual && (d->ld_res % 8) != 0 && !direct) direct = true;
  if (d->flags & AAB_F_SCALE_ACC) direct = true;
  if ((d->act == AAB_ACT_GELU || d->act == AAB_ACT_QUICK_GELU) && !geglu) direct = true;
  {   // the staged epilogue covers one extra term (residual | per-sample bias | SiLU) and no output scaling
    const int extras = (d->residual ? 1 : 0) + (d->bias2 ? 1 : 0) + (d->act == AAB_ACT_SILU ? 1 : 0);
    if (!geglu && (extras > 1 || d->out_scale != 1.0f)) direct = true;
    if (geglu && (extras > 0 || d->out_scale != 1.0f)) return AAB_ERR_ARG;
  }
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
  // clusters sharing each weight tile: 256-column staged tiles with unbatched weights and at least two m-tiles
  const bool pair = (d->flags & AAB_F_PAIR) != 0 && bn == 256 && !direct && d->b_batch_dim < 0 && p.num_m_tiles >= 2;
  p.cluster = pair ? (((d->flags & AAB_F_QUAD) && p.num_m_tiles >= 4) ? 4 : 2) : 1;
  {
    long dims[3] = {static_cast<long>(d->num_taps) * d->kc, d->n, d->b_batch > 0 ? d->b_batch : 1};
    long strides[3] = {1, d->ld_b, d->b_batch_stride > 0 ? d->b_batch_stride : static_cast<long>(d->n) * d->ld_b};
    const int slices = p.cluster > 1 ? p.cluster : (geglu ? 2 : 1);   // rows of one weight-tile slice (see the producer)
    int box[3] = {BK, bn / slices, 1};
    int r = make_tmap_16(&tmB, d->b, 3, dims, strides, box, is_bf16, 128);
    if (r) return r;
  }
  if (geglu) {
    if (bn == 128) return launch_bn<128, true>(tmA, tmA2, tmB, p, d->max_ctas, stream);
    return launch_bn<256, true>(tmA, tmA2, tmB, p, d->max_ctas, stream);
  }
  switch (bn) {
    case 32: return launch_bn<32, false>(tmA, tmA2, tmB, p, d->max_ctas, stream);
    case 64: return launch_bn<64, false>(tmA, tmA2, tmB, p, d->max_ctas, stream);
    case 128: return launch_bn<128, false>(tmA, tmA2, tmB, p, d->max_ctas, stream);
    default: return launch_bn<256, false>(tmA, tmA2, tmB, p, d->max_ctas, stream);
  }
}

extern "C" int aab_num_sms(void) { return aab::num_sms(); }
