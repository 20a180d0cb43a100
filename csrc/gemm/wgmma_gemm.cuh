// Persistent warp-specialised wgmma GEMM for sm_90a:
//
//     D[M,N] (+)= sum_{src} sum_k A_src[M,k] * B_src[N,k]       bf16 x bf16 -> fp32 (registers)
//
// * operands staged by TMA into 128B-swizzled shared memory, 64-wide K blocks, N-stage mbarrier ring
// * two consumer warpgroups each issue wgmma 64 x BN x 16 on their half of the 128-row tile and run the fused epilogue
//   straight from their accumulator registers while the producer already fills the ring for the next tile
// * either operand may be K-major ([rows][K]) or MN-major ([K][rows]) — the latter is what makes the
//   weight-gradient / sufficient-factor outer product  dW = Uᵀ·V  a plain TMA GEMM with no transposes
// * the reduction may span several *sources* (one tensor map per source): for SFB the sources are the
//   peers' symmetric (u, v) buffers read over NVLink, gated by per-peer epoch flags
// * for implicit-GEMM convolution one operand is fetched by the TMA engine in im2col mode (IM2COL_A / IM2COL_B) or, where
//   the channel count does not allow that, built by cp.async gather warps (GATHER_A / GATHER_B, see conv_gather.cuh)
// * CTA pairs (CG = 2): a (2,1,1) cluster whose CTAs own two m-blocks of the same n-block; each fetches half of the
//   shared B tile and multicasts it to both, halving the B traffic per SM
// * the TMA-producer loop runs warp-uniform with one elected issuing lane (operands in uniform registers)
// * fused epilogues: bias + ReLU (+ mask) -> bf16 ; fp32 store / split-K partials ; in-place SGD update
//
// Replaces the reference's cublasSgemm call sites (src/caffe/util/math_functions.cu:15-45) used by
// InnerProduct fwd/bwd (layers/inner_product_layer.cu:13-52), the per-image conv GEMMs
// (layers/conv_layer.cu:23-119) and ComputeGradientFromSV_gpu (layers/inner_product_layer.cu:55-64).
#pragma once
#include "sm90_prims.cuh"
#include "conv_gather.cuh"
#include <cuda_fp8.h>
#include <type_traits>

namespace psd {

constexpr int kMaxSrc = 8;
constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;
constexpr int MMA_K = 16;
constexpr int kEpiWarps = 8;              // two consumer warpgroups; warp e owns rows [16e, 16e + 16) of the tile
constexpr int kNumThreads = 128 + 32 * kEpiWarps;   // warp0 TMA, warps1-3 idle (warpgroup alignment), warps4-11 MMA + epilogue
constexpr int kEpiWarp0 = 4;
constexpr int kGatherWarp0 = kEpiWarp0 + kEpiWarps;  // conv kernels: 4 more warps gather the implicit-im2col operand
constexpr int kGatherThreads = 128;
// Widest tile of the gather kernels: 512 threads leave 128 registers per thread, enough for 64 fp32 accumulators.
constexpr int kGatherMaxBN = 128;
// GATHER_A / GATHER_B: operand built by the cp.async gather warps (any channel count, ROW mode).
// IM2COL_A / IM2COL_B: operand fetched by the TMA engine in im2col mode (C_g % 64 == 0): no gather warps at all.
// TILED_WGRAD: the fp8 weight gradient over batch-innermost CHWN copies — both operands K-major plain tiled 3-D boxes,
// the producer decoding each k block into (output row, column run, image chunk) (see wgmma_fp8_wgrad_kernel).
enum GatherMode : int { GATHER_NONE = 0, GATHER_A = 1, GATHER_B = 2, IM2COL_A = 3, IM2COL_B = 4, TILED_WGRAD = 5 };
__host__ __device__ constexpr bool has_gather_warps(int g) { return g == GATHER_A || g == GATHER_B; }

enum EpiMode : int { EPI_BF16 = 0, EPI_F32 = 1, EPI_SGD = 2 };

// Tensor-map encoders (gemm_ops.cu).  dtype: bf16 operands, or CU_TENSOR_MAP_DATA_TYPE_UINT8 for e4m3 ones.
void encode_tmap_2d(CUtensorMap* map, const void* base, int64_t inner, int64_t outer, int64_t ld, int box_inner,
                    int box_outer, CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
void encode_tmap_im2col(CUtensorMap* map, const void* base, int64_t C, int64_t W, int64_t H, int64_t N, int64_t pitch,
                        int lower_w, int lower_h, int upper_w, int upper_h, int pixels, int stride_w, int stride_h,
                        CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);

struct TmapSet {
  CUtensorMap a[kMaxSrc];
  CUtensorMap b[kMaxSrc];
};

struct GemmParams {
  int M, N;              // output extent
  int kb_per_src;        // number of 64-wide k blocks per source
  int num_src;
  int split_k;           // >1: the reduction is split over CTAs (EPI_F32 only; see split_stride)
  long split_stride;     // EPI_F32, split_k > 1: split s stores its partial tile to c_f32 + s * split_stride (plain stores,
                         // summed in split order afterwards, so the result does not depend on CTA timing)
  int src_rot;           // first source to visit (own rank for SFB: local data needs no flag wait)
  int cluster;           // CTAs per cluster sharing the TMA operand by multicast (1 = no clusters); conv kernels only
  int max_stages;        // experiment knob: use only this many ring stages (0 = all that fit)
  int no_bulk_epi;       // experiment knob: bit 0 / bit 1 = fp32 / bf16 output through the per-warp 16x32 walk instead of bulk row stores
  // --- epilogue operands
  __nv_bfloat16* c_bf16; // EPI_BF16 output [M, ldc]
  float* c_f32;          // EPI_F32 output [M, ldc]
  long ldc;
  const float* bias;     // optional, per output column (N)
  const __nv_bfloat16* mask;  // optional [M, ldc]: zero the output where mask <= 0 (fused ReLU backward)
  int relu;              // EPI_BF16: apply max(0, x) (negative_slope below)
  float relu_slope;
  int atomic;            // EPI_F32: atomicAdd instead of store
  int col_cg, col_cgk;   // EPI_F32 (conv wgrad over channel-padded K): output column (tap*cgk + c) -> tap*cg + c, c >= cg dropped
  float alpha;           // scale applied to the accumulator
  // --- EPI_SGD: W[M,N] fp32 master, H history, Wb bf16 shadow, in place
  float* w;
  float* h;
  __nv_bfloat16* wb;
  float lr, momentum, decay;
  const float* lr_dev;   // optional device-resident global learning rate (multiplies lr)
  int rule;              // 0 SGD, 1 Nesterov, 2 AdaGrad
  int l1;
  float delta;
  // --- peer gating (SFB): flag[src] must reach `epoch` before src's tiles are read
  const uint32_t* flags;
  uint32_t epoch;
  const uint32_t* epoch_dev;   // optional device-resident step counter added to `epoch` (CUDA-graph replays)
};

// CG = CTAs per B tile (1, or 2 = a CTA pair that shares the B tile by multicast: each CTA fetches BN/2 of its rows).
template <int BN, int CG = 1>
struct GemmSmem {
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;     // 16 KB
  static constexpr int kBBytes = BN * BLOCK_K * 2;          // the whole B tile (CG == 2: half of it written by the peer)
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kBarBytes = 256;
  // epilogue staging: per-warp 16 x 32 fp32 tiles (walk), or one 32-row quadrant slab (SGD / fp32 bulk / two bf16 slabs)
  static constexpr int cmax(int a, int b) { return a > b ? a : b; }
  static constexpr int kEpiStageBytes =
      cmax(cmax(kEpiWarps * 16 * 33 * 4, 32 * (BN + 4) * 4), 2 * 32 * (BN * 2 + 16));
  // as many ring stages as fit beside the barriers and the epilogue staging (at most 8: 4 @ BN 256, 6 @ 128, 8 @ <= 64)
  static constexpr int kFit = (232448 - 1024 - kBarBytes - kEpiStageBytes) / kStageBytes;
  static constexpr int kStages = kFit > 8 ? 8 : kFit;
  static constexpr int kTotal = kStages * kStageBytes + kBarBytes + kEpiStageBytes + 1024;  // +1024 alignment slack
  static_assert(kTotal <= 232448, "shared memory budget (227 KB per CTA)");
};

__device__ __forceinline__ float sgd_apply(float acc, float& w, float& h, const GemmParams& p, float lr) {
  float g = acc;
  if (p.decay != 0.f) g += p.decay * (p.l1 ? (w > 0.f ? 1.f : (w < 0.f ? -1.f : 0.f)) : w);
  float step;
  if (p.rule == 0) {
    h = lr * g + p.momentum * h;
    step = h;
  } else if (p.rule == 1) {
    float h_old = h;
    h = lr * g + p.momentum * h;
    step = (1.f + p.momentum) * h - p.momentum * h_old;
  } else {
    h = h + g * g;
    step = lr * g / (sqrtf(h) + p.delta);
  }
  w -= step;
  return w;
}

// Epilogue of one 16 x 32 accumulator sub-tile of a warp, already transposed into the warp's padded staging tile
// (`stage[r * 33 + c]`), so that every global access of the warp is row-contiguous (64-128 B segments).
// DEQ (fp8 operands, EPI_BF16): the accumulator is first scaled by sx * sw[col], before bias and activation.
template <int EPI, bool DEQ = false>
__device__ __forceinline__ void epilogue_tile16(const GemmParams& p, float* c_f32, const float* stage, int lane, int row0,
                                                int col0, float sx = 0.f, const float* sw = nullptr) {
  constexpr int ROWS = 16;
  const int nrows = min(ROWS, p.M - row0);
  const int ncols = min(32, p.N - col0);
  if constexpr (EPI == EPI_BF16) {
    // two rows per pass: lanes 0-15 -> row 2i, lanes 16-31 -> row 2i+1, each lane a column pair
    const int half = lane >> 4, cp = (lane & 15) * 2;
    const bool c0 = cp < ncols, c1 = cp + 1 < ncols;
    float b0 = 0.f, b1 = 0.f;
    if (p.bias != nullptr) {
      if (c0) b0 = __ldg(p.bias + col0 + cp);
      if (c1) b1 = __ldg(p.bias + col0 + cp + 1);
    }
    [[maybe_unused]] float q0 = 0.f, q1 = 0.f;
    if constexpr (DEQ) {
      if (c0) q0 = sx * __ldg(sw + col0 + cp);
      if (c1) q1 = sx * __ldg(sw + col0 + cp + 1);
    }
    const bool pair_ok = c1 && ((p.ldc & 1) == 0) && (((col0 + cp) & 1) == 0);
    // fused ReLU-backward mask: issue all loads of this lane up front (they are independent), then combine
    uint32_t mk[ROWS / 2];
    if (p.mask != nullptr) {
#pragma unroll
      for (int i = 0; i < ROWS / 2; ++i) {
        const int rr = 2 * i + half;
        const long off = static_cast<long>(row0 + rr) * p.ldc + col0 + cp;
        uint32_t v = 0x3f803f80u;                                      // (1.0, 1.0): keep
        if (rr < nrows) {
          if (pair_ok) v = *reinterpret_cast<const uint32_t*>(p.mask + off);
          else {
            const uint32_t lo = c0 ? __bfloat16_as_ushort(p.mask[off]) : 0x3f80u;
            const uint32_t hi = c1 ? __bfloat16_as_ushort(p.mask[off + 1]) : 0x3f80u;
            v = lo | (hi << 16);
          }
        }
        mk[i] = v;
      }
    }
#pragma unroll
    for (int i = 0; i < ROWS / 2; ++i) {
      const int rr = 2 * i + half;
      if (rr >= nrows) continue;
      float x0, x1;
      if constexpr (DEQ) {
        x0 = stage[rr * 33 + cp] * q0 + b0;
        x1 = stage[rr * 33 + cp + 1] * q1 + b1;
      } else {
        x0 = stage[rr * 33 + cp] + b0;
        x1 = stage[rr * 33 + cp + 1] + b1;
      }
      if (p.relu) {
        x0 = x0 > 0.f ? x0 : x0 * p.relu_slope;
        x1 = x1 > 0.f ? x1 : x1 * p.relu_slope;
      }
      const long off = static_cast<long>(row0 + rr) * p.ldc + col0 + cp;
      if (p.mask != nullptr) {
        const float m0 = __uint_as_float(mk[i] << 16), m1 = __uint_as_float(mk[i] & 0xffff0000u);
        if (!(m0 > 0.f)) x0 *= p.relu_slope;
        if (!(m1 > 0.f)) x1 *= p.relu_slope;
      }
      if (pair_ok) {
        *reinterpret_cast<__nv_bfloat162*>(p.c_bf16 + off) = __floats2bfloat162_rn(x0, x1);
      } else {
        if (c0) p.c_bf16[off] = __float2bfloat16(x0);
        if (c1) p.c_bf16[off + 1] = __float2bfloat16(x1);
      }
    }
  } else if constexpr (EPI == EPI_F32) {
    int col = col0 + lane;
    bool col_ok = lane < ncols;
    if (p.col_cgk > 0) {
      const int tap = col / p.col_cgk, c = col - tap * p.col_cgk;
      col_ok = col_ok && c < p.col_cg;
      col = tap * p.col_cg + c;
    }
    if (col_ok) {
#pragma unroll 4
      for (int rr = 0; rr < nrows; ++rr) {
        float* dst = c_f32 + static_cast<long>(row0 + rr) * p.ldc + col;
        const float v = stage[rr * 33 + lane];
        if (p.atomic) atomicAdd(dst, v);
        else *dst = v;
      }
    }
  }
  // EPI_SGD does not come through here: see sgd_rows_from_slab (CTA-cooperative, row-contiguous).
}

// Write this warp's 16 x BN accumulator fragment (wgmma layout, see Wgmma) into rows [r0, r0 + 16) of an fp32 slab of
// row pitch LD, scaled by alpha.
template <int BN, int LD>
__device__ __forceinline__ void frag_to_slab(const float (&acc)[BN / 2], float* slab, int r0, int lane, float alpha) {
  const int r = r0 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < BN / 8; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float2* dst = reinterpret_cast<float2*>(slab + (r + 8 * h) * LD + 8 * i + c);
      if constexpr (LD % 2 == 0) *dst = make_float2(acc[4 * i + 2 * h] * alpha, acc[4 * i + 2 * h + 1] * alpha);
      else {
        slab[(r + 8 * h) * LD + 8 * i + c] = acc[4 * i + 2 * h] * alpha;
        slab[(r + 8 * h) * LD + 8 * i + c + 1] = acc[4 * i + 2 * h + 1] * alpha;
      }
    }
  }
}

// EPI_SGD, CTA-cooperative form.  The optimizer step is pure HBM streaming (18 B per weight), and DRAM only streams
// at full rate when whole rows of the tile (BN * 4 B = 1 KB) are touched back to back: a per-warp sub-tile walk would
// issue isolated 128-byte pieces 36 KB apart, far from the rate of the same update as a linear stream.  Here the two
// warps that own a 32-row quadrant of the tile dump its 32 x BN accumulators into one shared slab, then ALL epilogue
// warps update 4 full rows each: every warp issues BN/32 consecutive 128-byte accesses per row and array (one
// contiguous 1 KB burst), with 8 * BN/32 independent loads in flight.
template <int BN>
__device__ __forceinline__ void sgd_rows_from_slab(const GemmParams& p, const float* slab, int e, int lane, int row0,
                                                   int col0, float lr_eff) {
  constexpr int LD = BN + 1;
  constexpr int NC = BN / 32;
  constexpr int RW = 32 / kEpiWarps;                 // rows of the slab per warp
  float wv[RW][NC], hv[RW][NC];
#pragma unroll
  for (int k = 0; k < RW; ++k) {
    const int row = row0 + e * RW + k;
    const long off0 = static_cast<long>(row) * p.ldc + col0 + lane;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      const bool ok = row < p.M && col0 + lane + 32 * i < p.N;
      wv[k][i] = ok ? p.w[off0 + 32 * i] : 0.f;
      hv[k][i] = ok ? p.h[off0 + 32 * i] : 0.f;
    }
  }
#pragma unroll
  for (int k = 0; k < RW; ++k) {
    const int row = row0 + e * RW + k;
    const long off0 = static_cast<long>(row) * p.ldc + col0 + lane;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
      if (row < p.M && col0 + lane + 32 * i < p.N) {
        sgd_apply(slab[(e * RW + k) * LD + lane + 32 * i], wv[k][i], hv[k][i], p, lr_eff);
        p.w[off0 + 32 * i] = wv[k][i];
        p.h[off0 + 32 * i] = hv[k][i];
        if (p.wb != nullptr) p.wb[off0 + 32 * i] = __float2bfloat16(wv[k][i]);
      }
    }
  }
}
__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kEpiWarps * 32) : "memory"); }


// Producer policy: both operands via TMA.  CG == 2: this CTA fetches rows / columns [crank * BN/2, (crank + 1) * BN/2) of
// the B tile and multicasts them into both CTAs of the pair (same shared-memory offset, same barrier offset).
template <int CG>
__device__ __forceinline__ void tma_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int x, int y) {
  if constexpr (CG == 2) tma_load_2d_mcast_u32(dst, map, bar, x, y, 0x3);
  else tma_load_2d_u32(dst, map, bar, x, y);
}
// KB: elements per k block (one 128-byte row: 64 bf16 or 128 fp8).
template <int BN, bool A_MN, bool B_MN, int CG = 1, int KB = BLOCK_K>
struct TmaProducer {
  static_assert(CG == 1 || !B_MN || (BN / CG) % 64 == 0, "MN-major B: each CTA's share must be whole 64-column chunks");
  __device__ static void load_a(const TmapSet& tm, int src, int kb, int m_blk, uint32_t sa, uint32_t bar) {
    const int k0 = kb * KB;
    if constexpr (!A_MN) {
      tma_load_2d_u32(sa, &tm.a[src], bar, k0, m_blk * BLOCK_M);
    } else {
#pragma unroll
      for (int c = 0; c < BLOCK_M / 64; ++c) tma_load_2d_u32(sa + c * 8192, &tm.a[src], bar, m_blk * BLOCK_M + 64 * c, k0);
    }
  }
  __device__ static void load_b(const TmapSet& tm, int src, int kb, int n_blk, int crank, uint32_t sb, uint32_t bar) {
    const int k0 = kb * KB;
    const int n0 = n_blk * BN + crank * (BN / CG);
    const uint32_t dst = sb + crank * (BN / CG) * 128;         // K-major: BN/CG rows of 128 B; MN-major: BN/CG/64 chunks
    if constexpr (!B_MN) {
      tma_2d<CG>(dst, &tm.b[src], bar, k0, n0);                // tensor-map box: BN / CG rows
    } else {
#pragma unroll
      for (int c = 0; c < BN / CG / 64; ++c) tma_2d<CG>(dst + c * 8192, &tm.b[src], bar, n0 + 64 * c, k0);
    }
  }
  __device__ static void load_stage(const TmapSet& tm, int src, int kb, int m_blk, int n_blk, int crank, uint32_t sa,
                                    uint32_t sb, uint32_t bar) {
    load_a(tm, src, kb, m_blk, sa, bar);
    load_b(tm, src, kb, n_blk, crank, sb, bar);
  }
};

// Tile enumeration.  Without clusters: tile -> (m fastest, then n, then split).  With a cluster of C CTAs the
// cluster walks "cluster tiles"; its CTAs take C consecutive blocks along the dimension the multicast (TMA)
// operand does NOT depend on: m for fprop/dgrad (weights shared), n for wgrad (dY slice shared).  Blocks past
// the edge are harmless: loads zero-fill / are out of range and the epilogue skips them.
struct TileCoord {
  int m_blk, n_blk, split;
};
// NFAST (optimizer-step epilogue): n fastest, so that the CTAs running at the same time update whole rows of W —
// one contiguous region of memory — instead of a 1 KB column slab with a row-sized stride between pieces.
template <int GATHER>
__device__ __forceinline__ TileCoord tile_coord(int t, int m_blocks, int n_blocks, int C, int crank, bool nfast) {
  TileCoord tc;
  if (nfast) {
    tc.n_blk = t % n_blocks;
    const int rest = t / n_blocks;
    tc.m_blk = rest % m_blocks;
    tc.split = rest / m_blocks;
  } else if (GATHER == GATHER_B || GATHER == IM2COL_A) {
    const int n_groups = (n_blocks + C - 1) / C;
    tc.m_blk = t % m_blocks;
    const int rest = t / m_blocks;
    tc.n_blk = (rest % n_groups) * C + crank;
    tc.split = rest / n_groups;
  } else {
    const int m_groups = (m_blocks + C - 1) / C;
    tc.m_blk = (t % m_groups) * C + crank;
    const int rest = t / m_groups;
    tc.n_blk = rest % n_blocks;
    tc.split = rest / n_blocks;
  }
  return tc;
}

// CTA pairs: the pair walks (pair of m-blocks, n-block, split) tiles; CTA `crank` of the pair owns m-block 2*mp + crank.
// A phantom m-block past the edge (odd m_blocks) is harmless: its loads are out of range (zero-filled) and its
// epilogue rows are skipped.
__device__ __forceinline__ TileCoord tile_coord_pair(int t, int m_pairs, int n_blocks, int crank, bool nfast) {
  TileCoord tc;
  int mp;
  if (nfast) {
    tc.n_blk = t % n_blocks;
    const int rest = t / n_blocks;
    mp = rest % m_pairs;
    tc.split = rest / m_pairs;
  } else {
    mp = t % m_pairs;
    const int rest = t / m_pairs;
    tc.n_blk = rest % n_blocks;
    tc.split = rest / n_blocks;
  }
  tc.m_blk = 2 * mp + crank;
  return tc;
}

// Body of the GEMM kernels below.  TA / TB: operand elements, both __nv_bfloat16, or fp8 (A __nv_fp8_e4m3 or
// __nv_fp8_e5m2, B __nv_fp8_e4m3).  A k block is one 128-byte swizzled row either way (64 bf16 or 128 fp8), so the ring,
// the descriptors and the TMA boxes keep their byte geometry; fp8 issues k32 MMAs (still 4 per k block) and dequantises
// in the epilogue (scale_x * scale_w[col], ConvGeom).
template <int BN, bool A_MN, bool B_MN, int EPI, int GATHER, int CG, typename TA, typename TB>
__device__ __forceinline__ void wgmma_gemm_body(const TmapSet& tm, const GemmParams p, const ConvGeom cg) {
  constexpr bool kFp8 = sizeof(TA) == 1;
  constexpr bool kE5M2A = std::is_same<TA, __nv_fp8_e5m2>::value;
  constexpr int KB = 128 / static_cast<int>(sizeof(TA));    // elements per k block
  static_assert(sizeof(TA) == sizeof(TB), "both operands bf16, or both fp8");
  static_assert(!kFp8 || std::is_same<TB, __nv_fp8_e4m3>::value, "fp8 B operand: e4m3");
  static_assert(!kFp8 || (!A_MN && !B_MN && BN <= 128 &&
                          ((GATHER == IM2COL_A && EPI == EPI_BF16) || (GATHER == TILED_WGRAD && EPI == EPI_F32))),
                "fp8 operands: K-major im2col convolution with the bf16 epilogue, or the tiled weight gradient (fp32)");
  static_assert(GATHER != TILED_WGRAD || kFp8, "the tiled weight-gradient producer reads fp8 CHWN copies");
  static_assert(CG == 1 || CG == 2, "one CTA or a CTA pair per B tile");
  static_assert(CG == 1 || !has_gather_warps(GATHER), "CTA pairs share a TMA-fetched B tile");
  static_assert(!has_gather_warps(GATHER) || BN <= kGatherMaxBN, "gather kernels: accumulator register budget");
  static_assert(GATHER != GATHER_A || !A_MN, "gathered A is produced K-major");
  static_assert(GATHER != GATHER_B || B_MN, "gathered B is produced MN-major");
  static_assert(GATHER != IM2COL_A || !A_MN, "im2col A is K-major");
  static_assert(GATHER != IM2COL_B || B_MN, "im2col B is MN-major");
  static_assert(BN % 32 == 0 && (!B_MN || BN % 64 == 0), "tile width");
  using S = GemmSmem<BN, CG>;
  constexpr int kStages = S::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* bar_base = smem + kStages * S::kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(bar_base);
  uint64_t* empty_bar = full_bar + kStages;
  float* epi_stage = reinterpret_cast<float*>(bar_base + S::kBarBytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nst = (p.max_stages > 0 && p.max_stages < kStages) ? p.max_stages : kStages;     // ring depth in use

  const int m_blocks = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int n_blocks = (p.N + BN - 1) / BN;
  const int total_kb = p.kb_per_src * p.num_src;
  // CTAs per cluster sharing one operand by TMA multicast (CG == 1 only): the cp.async gather modes share the TMA (weight /
  // dY) operand; the im2col-TMA modes share the IM2COL operand itself, each CTA of the cluster fetching 1/C of its rows.
  const int C = (CG == 1 && GATHER != GATHER_NONE && p.cluster > 1) ? p.cluster : 1;
  const int crank = (C > 1 || CG == 2) ? static_cast<int>(cluster_ctarank()) : 0;
  const int share = CG == 2 ? 2 : C;                    // CTAs whose producers write into this CTA's ring
  const int prank = CG == 2 ? crank : 0;                // which half of the B tile this CTA fetches (CTA pairs only)
  const uint16_t cmask = static_cast<uint16_t>((1u << C) - 1);
  // cluster-level tile space and stride
  const int m_pairs = (m_blocks + 1) / 2;
  const int num_tiles = CG == 2 ? m_pairs * n_blocks * p.split_k
                                : ((GATHER == GATHER_B || GATHER == IM2COL_A) ? m_blocks * ((n_blocks + C - 1) / C)
                                                                              : ((m_blocks + C - 1) / C) * n_blocks) * p.split_k;
  const int tile0 = blockIdx.x / (C * CG), tile_step = gridDim.x / (C * CG);
  // n fastest for the epilogues that stream whole fp32 rows (optimizer step; plain fp32 output of the inner-product weight
  // gradient): the CTAs running at the same time then cover complete rows — one contiguous region of memory
  // (not for the form that adds onto the output with atomics: there the m-blocks of one weight tile run back to back)
  const bool nfast = EPI == EPI_SGD || (EPI == EPI_F32 && GATHER == GATHER_NONE && !p.atomic);
  auto coord = [&](int t) -> TileCoord {
    if constexpr (CG == 2) return tile_coord_pair(t, m_pairs, n_blocks, crank, nfast);
    else return tile_coord<GATHER>(t, m_blocks, n_blocks, C, crank, nfast);
  };

  if (warp == 0 && lane == 0) {
    for (int s = 0; s < p.num_src; ++s) {
      tma_prefetch_desc(&tm.a[s]);
      tma_prefetch_desc(&tm.b[s]);
    }
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1 + (has_gather_warps(GATHER) ? kGatherThreads : 0));
      mbar_init(&empty_bar[s], (kEpiWarps / 4) * share);   // one arrive per consumer warpgroup of every sharing CTA
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (share > 1) cluster_sync_all();   // peers' barriers exist before any remote arrive / multicast

  if (warp == 0) {
    // ===================== TMA producer =====================
    // The whole warp runs the loop with uniform control flow and ONE elected lane issues the TMA / barrier
    // instructions: the operands then live in uniform registers, whereas a loop under `if (lane == 0)` is divergent code
    // in which every issue needs a register-to-uniform waterfall.
    {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = tile0; tile < num_tiles; tile += tile_step) {
        const TileCoord tc = coord(tile);
        const int m_blk = tc.m_blk, n_blk = tc.n_blk, split = tc.split;
        const int g0 = static_cast<int>(static_cast<long>(total_kb) * split / p.split_k);
        const int g1 = static_cast<int>(static_cast<long>(total_kb) * (split + 1) / p.split_k);
        // im2col modes: coordinates of the tile's first base pixel (A) / tap decode of the tile's k-columns (B)
        [[maybe_unused]] int im_w = 0, im_h = 0, im_n = 0;
        [[maybe_unused]] const int im_org_w = cg.off_w - (cg.dr < 0 ? cg.S - 1 : 0);
        [[maybe_unused]] const int im_org_h = cg.off_h - (cg.dr < 0 ? cg.R - 1 : 0);
        [[maybe_unused]] int im_c0[BN / 64 > 0 ? BN / 64 : 1];
        [[maybe_unused]] uint16_t im_offw[BN / 64 > 0 ? BN / 64 : 1], im_offh[BN / 64 > 0 ? BN / 64 : 1];
        if constexpr (GATHER == IM2COL_A) {
          // first base pixel this CTA fetches: the tile's, or (cluster multicast) that of its 128 / C pixel slice
          const uint32_t m0 = static_cast<uint32_t>(m_blk) * BLOCK_M + (C > 1 ? static_cast<uint32_t>(crank * (BLOCK_M / C)) : 0u);
          const uint32_t n_img = fdiv(m0, cg.div_ohow);
          const uint32_t rem = m0 - n_img * static_cast<uint32_t>(cg.OH * cg.OW);
          const uint32_t oh = fdiv(rem, cg.div_ow);
          const uint32_t ow = rem - oh * static_cast<uint32_t>(cg.OW);
          im_w = static_cast<int>(ow) * cg.sw + im_org_w;
          im_h = static_cast<int>(oh) * cg.sh + im_org_h;
          im_n = static_cast<int>(n_img);
        }
        if constexpr (GATHER == IM2COL_B) {
#pragma unroll
          for (int c = 0; c < BN / 64; ++c) {
            int kc = n_blk * BN + c * 64;
            if (kc >= cg.K) kc = 0;                      // columns past K are dropped by the epilogue: load anything valid
            const int tap = static_cast<int>(fdiv(static_cast<uint32_t>(kc), cg.div_cg));
            im_c0[c] = kc - tap * cg.Cgk;
            const int r = static_cast<int>(fdiv(static_cast<uint32_t>(tap), cg.div_s));
            im_offh[c] = static_cast<uint16_t>(r);
            im_offw[c] = static_cast<uint16_t>(tap - r * cg.S);
          }
        }
        // TILED_WGRAD: k block g0 -> (output row, column run, image chunk), then advanced incrementally; per B box of
        // this CTA (rows [prank * BN/CG, ...) of the tile, kRowsB each) its tap displacement and first channel
        constexpr int kRowsB = BN / CG < 64 ? BN / CG : 64;       // rows per B box: 64 columns of one tap, or half
        constexpr int kBoxesB = GATHER == TILED_WGRAD ? BN / CG / kRowsB : 1;
        [[maybe_unused]] int wg_n = 0, wg_w = 0, wg_h = 0, wg_dw[kBoxesB], wg_dh[kBoxesB], wg_c[kBoxesB];
        if constexpr (GATHER == TILED_WGRAD) {
          wg_n = g0 % cg.wg_nch;
          const int rest = g0 / cg.wg_nch;
          wg_w = rest % cg.wg_owr;
          wg_h = rest / cg.wg_owr;
#pragma unroll
          for (int j = 0; j < kBoxesB; ++j) {
            const int row0 = prank * (BN / CG) + j * kRowsB;
            int kc = n_blk * BN + (row0 & ~63);
            if (kc >= cg.K) kc = 0;                      // columns past K are dropped by the epilogue: load anything valid
            const int tap = static_cast<int>(fdiv(static_cast<uint32_t>(kc), cg.div_cg));
            const int r = static_cast<int>(fdiv(static_cast<uint32_t>(tap), cg.div_s));
            wg_c[j] = kc - tap * cg.Cgk + (row0 & 63);
            wg_dh[j] = r + im_org_h;
            wg_dw[j] = tap - r * cg.S + im_org_w;
          }
        }
        // (source, k-block) advance incrementally: no divisions in the single-thread producer loop
        int src_lin = g0 / p.kb_per_src;
        int kb = g0 - src_lin * p.kb_per_src;
        int src = (src_lin + p.src_rot) % p.num_src;
        bool new_src = true;
        for (int g = g0; g < g1; ++g) {
          if (new_src) {
            if (p.flags != nullptr) {
              if (lane == 0) {
                const uint32_t ep = p.epoch + (p.epoch_dev != nullptr ? *reinterpret_cast<const volatile uint32_t*>(p.epoch_dev) : 0u);
                wait_flag_ge(p.flags + src, ep);
              }
              __syncwarp();
            }
            new_src = false;
          }
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * S::kStageBytes;
          if (elect_one()) {
          const uint32_t fbar = smem_u32(&full_bar[stage]);
          const uint32_t sa32 = smem_u32(sa), sb32 = sa32 + S::kABytes;
          if constexpr (GATHER == GATHER_NONE) {
            mbar_arrive_expect_tx(&full_bar[stage], S::kStageBytes);
            TmaProducer<BN, A_MN, B_MN, CG>::load_stage(tm, src, kb, m_blk, n_blk, prank, sa32, sb32, fbar);
          } else if constexpr (GATHER == IM2COL_A) {
            // A tile = 128 output pixels x 64 channels of tap (r, s): one im2col-mode TMA instruction
            const int k0 = g * KB;
            const int tap = static_cast<int>(fdiv(static_cast<uint32_t>(k0), cg.div_cg));
            const int c0 = k0 - tap * cg.Cgk;
            const int r = static_cast<int>(fdiv(static_cast<uint32_t>(tap), cg.div_s));
            const int sx = tap - r * cg.S;
            const bool in_k = k0 < cg.K;
            const int offw = cg.dr > 0 ? sx : cg.S - 1 - sx, offh = cg.dr > 0 ? r : cg.R - 1 - r;
            mbar_arrive_expect_tx(&full_bar[stage], S::kStageBytes);
            // k-blocks past K (K % 64 != 0 never happens here: C_g % 64 == 0) — keep the guard cheap
            if (C > 1)       // this CTA's 128 / C pixel rows of the shared A tile, delivered to the whole cluster
              tma_load_im2col_4d_mcast(sa32 + crank * (BLOCK_M / C) * 128, &tm.a[0], fbar, in_k ? c0 : 0, im_w, im_h, im_n,
                                       static_cast<uint16_t>(in_k ? offw : 0), static_cast<uint16_t>(in_k ? offh : 0), cmask);
            else
              tma_load_im2col_4d(sa32, &tm.a[0], fbar, in_k ? c0 : 0, im_w, im_h, im_n,
                                 static_cast<uint16_t>(in_k ? offw : 0), static_cast<uint16_t>(in_k ? offh : 0));
            if constexpr (B_MN) {
              // dgrad straight from the FPROP weight layout [co][tap][ci] (no packed copy): the B tile of k-block
              // (tap, co0..co0+63) is BN/64 boxes {64 ci, 64 co, 1 tap} of a 3-D map — ci contiguous = MN-major B;
              // output channels past Cout_g and input channels past C_g are zero-filled by the TMA.  CTA pairs: this
              // CTA fetches boxes [crank * BN/128, (crank + 1) * BN/128) for both.
              const int n0 = n_blk * BN;
#pragma unroll
              for (int c = prank * (BN / CG / 64); c < (prank + 1) * (BN / CG / 64); ++c) {
                if constexpr (CG == 2)
                  tma_load_3d_mcast_u32(sb32 + c * 8192, &tm.b[0], fbar, n0 + 64 * c, in_k ? c0 : 0, in_k ? tap : 0, 0x3);
                else tma_load_3d_u32(sb32 + c * 8192, &tm.b[0], fbar, n0 + 64 * c, in_k ? c0 : 0, in_k ? tap : 0);
              }
            } else {
              TmaProducer<BN, A_MN, B_MN, CG, KB>::load_b(tm, src, kb, n_blk, prank, sb32, fbar);
            }
          } else if constexpr (GATHER == IM2COL_B) {
            // B tile = BN/64 chunks of [64 reduction pixels][64 channels of one tap]; the pixels advance with g.
            // A cluster (C CTAs along Cout, or a CTA pair) shares the tile: chunk c is fetched by CTA c % share.
            const uint32_t m0 = static_cast<uint32_t>(g) * BLOCK_K;
            const uint32_t n_img = fdiv(m0, cg.div_ohow);
            const uint32_t rem = m0 - n_img * static_cast<uint32_t>(cg.OH * cg.OW);
            const uint32_t oh = fdiv(rem, cg.div_ow);
            const uint32_t ow = rem - oh * static_cast<uint32_t>(cg.OW);
            const int bw = static_cast<int>(ow) * cg.sw + im_org_w, bh = static_cast<int>(oh) * cg.sh + im_org_h;
            mbar_arrive_expect_tx(&full_bar[stage], S::kStageBytes);
#pragma unroll
            for (int c = 0; c < BN / 64; ++c) {
              if (share > 1) {
                if (c % share == crank)
                  tma_load_im2col_4d_mcast(sb32 + c * 8192, &tm.b[0], fbar, im_c0[c], bw, bh, static_cast<int>(n_img),
                                           im_offw[c], im_offh[c], static_cast<uint16_t>((1u << share) - 1));
              } else {
                tma_load_im2col_4d(sb32 + c * 8192, &tm.b[0], fbar, im_c0[c], bw, bh, static_cast<int>(n_img), im_offw[c],
                                   im_offh[c]);
              }
            }
            TmaProducer<BN, A_MN, B_MN, CG>::load_a(tm, src, kb, m_blk, sa32, fbar);
          } else if constexpr (GATHER == TILED_WGRAD) {
            // One k block = 128 bytes of the (column, image) row of output row wg_h, starting at column w0, image n0.
            // A = dYᵀ rows (output channels): box {128 B, 1, 128 co} of [Cout_g][OH][OW * Np]; columns past OW and
            // channels past Cout_g are zero-filled, so a partial last column run adds nothing.
            // B = X rows (tap, ci): per 64-column chunk, a box {128 B, 1, rows} of [Cg][H][W * Np] displaced by the tap;
            // the zero fill outside the image (negative or past-the-end coordinates) is the convolution's padding.
            // CTA pairs: this CTA fetches rows [prank * BN/2, (prank + 1) * BN/2) of the B tile for both.
            const int x0 = wg_w * cg.wg_wr * cg.wg_np + wg_n * 128;
            mbar_arrive_expect_tx(&full_bar[stage], S::kStageBytes);
            tma_load_3d_u32(sa32, &tm.a[0], fbar, x0, wg_h, m_blk * BLOCK_M);
#pragma unroll
            for (int j = 0; j < kBoxesB; ++j) {
              const uint32_t dst = sb32 + (prank * (BN / CG) + j * kRowsB) * 128;
              const int xb = x0 + wg_dw[j] * cg.wg_np;
              if constexpr (CG == 2) tma_load_3d_mcast_u32(dst, &tm.b[0], fbar, xb, wg_h + wg_dh[j], wg_c[j], 0x3);
              else tma_load_3d_u32(dst, &tm.b[0], fbar, xb, wg_h + wg_dh[j], wg_c[j]);
            }
          } else if constexpr (GATHER == GATHER_A) {
            mbar_arrive_expect_tx(&full_bar[stage], S::kBBytes);     // the whole B tile lands here (C slices)
            if (C == 1) {
              TmaProducer<BN, A_MN, B_MN>::load_b(tm, src, kb, n_blk, 0, sb32, fbar);
            } else {
              // this CTA fetches rows [crank*BN/C, (crank+1)*BN/C) of the K-major weight tile for the whole cluster
              const int rows = BN / C;
              tma_load_2d_mcast(sa + S::kABytes + crank * rows * 128, &tm.b[src], &full_bar[stage], kb * BLOCK_K,
                                n_blk * BN + crank * rows, cmask);
            }
          } else {
            mbar_arrive_expect_tx(&full_bar[stage], S::kABytes);
            if (C == 1) {
              TmaProducer<BN, A_MN, B_MN>::load_a(tm, src, kb, m_blk, sa32, fbar);
            } else {
              // dY^T tile (MN-major: 2 chunks of [64 k-rows][64 cout]); CTA `crank` fetches k-rows [crank*64/C, ...)
              const int krows = BLOCK_K / C;
#pragma unroll
              for (int c = 0; c < BLOCK_M / 64; ++c)
                tma_load_2d_mcast(sa + c * 8192 + crank * krows * 128, &tm.a[src], &full_bar[stage],
                                  m_blk * BLOCK_M + 64 * c, kb * BLOCK_K + crank * krows, cmask);
            }
          }
          }  // elect_one
          __syncwarp();
          if constexpr (GATHER == TILED_WGRAD) {
            if (++wg_n == cg.wg_nch) {
              wg_n = 0;
              if (++wg_w == cg.wg_owr) { wg_w = 0; ++wg_h; }
            }
          }
          if (++stage == nst) { stage = 0; phase ^= 1; }
          if (++kb == p.kb_per_src) {
            kb = 0;
            if (++src == p.num_src) src = 0;
            new_src = true;
          }
        }
      }
    }
  } else if (has_gather_warps(GATHER) && warp >= kGatherWarp0) {
    // ===================== gather producers: implicit im2col -> swizzled smem via cp.async =====================
    const int gt = threadIdx.x - kGatherWarp0 * 32;      // 0..kGatherThreads-1
    const int j = gt & 7;                                 // this thread's 16-byte chunk column
    const int rg = gt >> 3;                               // first row; further rows every kGatherThreads/8
    constexpr int kRowStep = kGatherThreads / 8;      // 16: row r and r + 16 share (r & 7), i.e. the same swizzle
    const GatherRegs gr = load_gather_regs(cg);
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = tile0; tile < num_tiles; tile += tile_step) {
      const TileCoord tc = coord(tile);
      const int m_blk = tc.m_blk, n_blk = tc.n_blk, split = tc.split;
      const int g0 = static_cast<int>(static_cast<long>(total_kb) * split / p.split_k);
      const int g1 = static_cast<int>(static_cast<long>(total_kb) * (split + 1) / p.split_k);
      if constexpr (GATHER == GATHER_A) {
        // rows of the A tile are fixed along K: fetch their row-table entries once per tile
        constexpr int kRows = BLOCK_M / kRowStep;
        RowPos pos[kRows];
#pragma unroll
        for (int i = 0; i < kRows; ++i) pos[i] = load_row(gr, static_cast<long>(m_blk) * BLOCK_M + rg + i * kRowStep);
        for (int g = g0; g < g1; ++g) {
          const ChunkOff t = decode_chunk_off(gr, g * BLOCK_K + j * 8);
          mbar_wait(&empty_bar[stage], phase ^ 1);
          const uint32_t sa = smem_u32(smem + stage * S::kStageBytes) + rg * 128 + ((j ^ (rg & 7)) << 4);
          if (gr.mode == 0) {
#pragma unroll
            for (int i = 0; i < kRows; ++i) gather_chunk_tap(gr, sa + i * (kRowStep * 128), pos[i], t);
          } else {
#pragma unroll
            for (int i = 0; i < kRows; ++i) gather_chunk_row(gr, sa + i * (kRowStep * 128), pos[i], t);
          }
          cp_async_mbar_arrive_noinc(&full_bar[stage]);
          if (++stage == nst) { stage = 0; phase ^= 1; }
        }
      } else {
        // B tile (MN-major): BN/64 chunk-columns of [64 reduction rows (m)][64 k-columns]; the k-columns are
        // fixed per tile (decode the taps once), the rows advance with the reduction index g — their row-table
        // entries for k-block g+1 are fetched before waiting for the slot of k-block g
        constexpr int kChunks = BN / 64 > 0 ? BN / 64 : 1;      // (BN < 64 is never instantiated with gather warps)
        constexpr int kRows = 64 / kRowStep;
        ChunkOff taps[kChunks];
#pragma unroll
        for (int c = 0; c < kChunks; ++c) taps[c] = decode_chunk_off(gr, n_blk * BN + c * 64 + j * 8);
        RowPos pos[kRows], nxt[kRows];
#pragma unroll
        for (int i = 0; i < kRows; ++i) nxt[i] = load_row(gr, static_cast<long>(g0) * BLOCK_K + rg + i * kRowStep);
        for (int g = g0; g < g1; ++g) {
#pragma unroll
          for (int i = 0; i < kRows; ++i) {
            pos[i] = nxt[i];
            nxt[i] = load_row(gr, static_cast<long>(g + 1) * BLOCK_K + rg + i * kRowStep);
          }
          mbar_wait(&empty_bar[stage], phase ^ 1);
          const uint32_t sb = smem_u32(smem + stage * S::kStageBytes) + S::kABytes + rg * 128 + ((j ^ (rg & 7)) << 4);
#pragma unroll
          for (int c = 0; c < kChunks; ++c) {
#pragma unroll
            for (int i = 0; i < kRows; ++i) {
              if (gr.mode == 0) gather_chunk_tap(gr, sb + c * 8192 + i * (kRowStep * 128), pos[i], taps[c]);
              else gather_chunk_row(gr, sb + c * 8192 + i * (kRowStep * 128), pos[i], taps[c]);
            }
          }
          cp_async_mbar_arrive_noinc(&full_bar[stage]);
          if (++stage == nst) { stage = 0; phase ^= 1; }
        }
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
  } else if (warp >= kEpiWarp0 && warp < kEpiWarp0 + kEpiWarps) {
    // ===================== consumer warpgroups: wgmma main loop, then the epilogue from registers =====================
    const int e = warp - kEpiWarp0;               // rows [16e, 16e + 16) of the tile
    const int wg = e >> 2;                        // warpgroup: rows [64 wg, 64 wg + 64)
    const bool wg_leader = (e & 3) == 0 && lane == 0;
    // release a ring slot in every CTA whose producer writes into it
    auto release = [&](int s) {
      if (wg_leader) {
        if (share == 1) mbar_arrive(&empty_bar[s]);
        else
          for (int r = 0; r < share; ++r) mbar_arrive_remote(&empty_bar[s], static_cast<uint32_t>(r));
      }
    };
    [[maybe_unused]] const bool bulk_f32 = EPI == EPI_F32 && !p.atomic && !(p.no_bulk_epi & 1) && p.col_cgk == 0 && (p.N & 3) == 0 &&
                                           (p.ldc & 3) == 0 &&
                                           (reinterpret_cast<uintptr_t>(p.c_f32) & 15) == 0 && (p.split_stride & 3) == 0;
    [[maybe_unused]] const bool bulk_bf16 = EPI == EPI_BF16 && !kFp8 && !(p.no_bulk_epi & 2) && (p.N & 7) == 0 && (p.ldc & 7) == 0 &&
                                            (reinterpret_cast<uintptr_t>(p.c_bf16) & 15) == 0 &&
                                            (p.mask == nullptr || (reinterpret_cast<uintptr_t>(p.mask) & 15) == 0);
    int stage = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    for (int tile = tile0; tile < num_tiles; tile += tile_step) {
      const TileCoord tc = coord(tile);
      const int m_blk = tc.m_blk, n_blk = tc.n_blk, split = tc.split;
      const int g0 = static_cast<int>(static_cast<long>(total_kb) * split / p.split_k);
      const int g1 = static_cast<int>(static_cast<long>(total_kb) * (split + 1) / p.split_k);
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int g = g0; g < g1; ++g) {
        mbar_wait(&full_bar[stage], phase);
        // the gather warps wrote this slot through the generic proxy; wgmma reads it through the async proxy
        if constexpr (has_gather_warps(GATHER)) fence_proxy_async_smem();
        const uint32_t a_addr = smem_u32(smem + stage * S::kStageBytes) + wg * 8192;   // this warpgroup's 64 rows of A
        const uint32_t b_addr = smem_u32(smem + stage * S::kStageBytes) + S::kABytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / MMA_K; ++k) {
          const uint64_t da = A_MN ? make_smem_desc(a_addr + k * (MMA_K * 128), 8192, 1024)
                                   : make_smem_desc(a_addr + k * (MMA_K * 2), 16, 1024);
          const uint64_t db = B_MN ? make_smem_desc(b_addr + k * (MMA_K * 128), 8192, 1024)
                                   : make_smem_desc(b_addr + k * (MMA_K * 2), 16, 1024);
          if constexpr (kE5M2A) WgmmaFp8E5M2<BN>::mma(acc, da, db, 1u);
          else if constexpr (kFp8) WgmmaFp8<BN>::mma(acc, da, db, 1u);
          else Wgmma<BN, A_MN ? 1 : 0, B_MN ? 1 : 0>::mma(acc, da, db, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();                          // the previous k-block's MMAs have retired: its slot is free
        wgmma_fence_regs(acc);
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == nst) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev >= 0) release(prev);
      // fp8 weight gradient: the fp32 epilogue scales by s_dy * s_x * alpha (one scale each, no per-column factor)
      [[maybe_unused]] float alpha_w = 0.f;
      if constexpr (GATHER == TILED_WGRAD) alpha_w = __ldg(cg.scale_x) * __ldg(cg.scale_w) * p.alpha;

      const int col0 = n_blk * BN;
      [[maybe_unused]] float* const c_f32 = p.c_f32 + (p.split_stride > 0 ? split * p.split_stride : 0);   // this split's slice
      if constexpr (EPI == EPI_SGD) {
        static_assert(32 * (BN + 1) * 4 <= S::kEpiStageBytes, "SGD slab must fit the epilogue staging buffer");
        const float lr_eff = p.lr_dev != nullptr ? p.lr * __ldg(p.lr_dev) : p.lr;
#pragma unroll 1
        for (int qq = 0; qq < 4; ++qq) {
          if ((e >> 1) == qq) frag_to_slab<BN, BN + 1>(acc, epi_stage, (e & 1) * 16, lane, p.alpha);   // the quadrant's owners
          epi_bar_sync();
          sgd_rows_from_slab<BN>(p, epi_stage, e, lane, m_blk * BLOCK_M + qq * 32, col0, lr_eff);
          epi_bar_sync();                                 // slab free for the next quadrant
        }
      } else {
        bool stored = false;
        if constexpr (EPI == EPI_F32) {
          // Plain fp32 output (inner-product weight gradients, the SFB reconstruct in its two-pass form): pure HBM
          // streaming — a 128 x BN tile is 128 KB of output for as little as 4 k-blocks of MMA.  A 32-row quadrant is laid
          // down in ONE shared slab (row pitch BN + 4 floats: 16-byte aligned rows) and leaves as 32 bulk-async (TMA) row
          // stores of up to 1 KB each; the issuing lanes only wait until the copy engine has READ the slab, so the global
          // writes of one quadrant overlap the fill of the next.
          if (bulk_f32) {
            constexpr int LDS = BN + 4;
            static_assert(32 * LDS * 4 <= S::kEpiStageBytes, "fp32 slab must fit the epilogue staging buffer");
            constexpr int RW = 32 / kEpiWarps;
            const int ncols = min(BN, p.N - col0);
#pragma unroll 1
            for (int qq = 0; qq < 4; ++qq) {
              if ((e >> 1) == qq) {
                frag_to_slab<BN, LDS>(acc, epi_stage, (e & 1) * 16, lane, GATHER == TILED_WGRAD ? alpha_w : p.alpha);
                fence_proxy_async_smem();               // generic-proxy writes -> visible to the bulk-copy engine
              }
              epi_bar_sync();
              if (lane < RW) {
                const int rr = e * RW + lane;
                const int row = m_blk * BLOCK_M + qq * 32 + rr;
                if (row < p.M && ncols > 0)
                  bulk_store_row(c_f32 + static_cast<long>(row) * p.ldc + col0, epi_stage + rr * LDS,
                                 static_cast<uint32_t>(ncols) * 4u);
                bulk_commit_wait_read();                 // the slab may be overwritten once the engine has read it
              }
              epi_bar_sync();
            }
            stored = true;
          }
        }
        if constexpr (EPI == EPI_BF16) {
          // bf16 activations / data gradients through TWO half-size slabs (32 rows x BN bf16, row pitch BN * 2 + 16 bytes).
          // Bias, (leaky) ReLU and the producer's ReLU mask are applied in registers; quadrant qq + 1 is converted into the
          // other slab while the copy engine still reads quadrant qq, and rows leave as up-to-512-byte bulk stores.
          // Off by default (set_bulk_epilogue(3) turns it on; its numerics test compares it with the per-warp walk).
          if (bulk_bf16) {
            constexpr int LDB = BN * 2 + 16;
            static_assert(2 * 32 * LDB <= S::kEpiStageBytes, "two bf16 slabs must fit the epilogue staging buffer");
            constexpr int RW = 32 / kEpiWarps;
            uint8_t* slabs = reinterpret_cast<uint8_t*>(epi_stage);
            const int ncols = min(BN, p.N - col0);
#pragma unroll 1
            for (int qq = 0; qq < 4; ++qq) {
              uint8_t* slab = slabs + (qq & 1) * (32 * LDB);
              if ((e >> 1) == qq) {
                const int sr = (e & 1) * 16 + (lane >> 2);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const long grow = static_cast<long>(m_blk) * BLOCK_M + qq * 32 + sr + 8 * h;
#pragma unroll
                  for (int i = 0; i < BN / 8; ++i) {
                    const int c = 8 * i + 2 * (lane & 3);
                    const int cb = col0 + c;
                    if (cb >= p.N) continue;               // past N: never stored (N % 8 == 0: both columns are past)
                    float x0 = acc[4 * i + 2 * h] * p.alpha, x1 = acc[4 * i + 2 * h + 1] * p.alpha;
                    if (p.bias != nullptr) {
                      x0 += __ldg(p.bias + cb);
                      x1 += __ldg(p.bias + cb + 1);
                    }
                    if (p.relu) {
                      x0 = x0 > 0.f ? x0 : x0 * p.relu_slope;
                      x1 = x1 > 0.f ? x1 : x1 * p.relu_slope;
                    }
                    if (p.mask != nullptr && grow < p.M) {
                      const uint32_t m = __ldg(reinterpret_cast<const unsigned int*>(p.mask + grow * p.ldc + cb));
                      if (!(__uint_as_float(m << 16) > 0.f)) x0 *= p.relu_slope;
                      if (!(__uint_as_float(m & 0xffff0000u) > 0.f)) x1 *= p.relu_slope;
                    }
                    const __nv_bfloat162 v = __floats2bfloat162_rn(x0, x1);
                    *reinterpret_cast<__nv_bfloat162*>(slab + (sr + 8 * h) * LDB + c * 2) = v;
                  }
                }
                fence_proxy_async_smem();                 // generic-proxy writes -> visible to the bulk-copy engine
              }
              // every bulk group issued so far has been read (the other slab, quadrant qq - 1): after the barrier
              // below that slab is free for quadrant qq + 1
              if (lane < RW) bulk_wait_read_all();
              epi_bar_sync();
              if (lane < RW) {
                const int rr = e * RW + lane;
                const long row = static_cast<long>(m_blk) * BLOCK_M + qq * 32 + rr;
                if (row < p.M && ncols > 0)
                  bulk_store_row(p.c_bf16 + row * p.ldc + col0, slab + rr * LDB, static_cast<uint32_t>(ncols) * 2u);
                bulk_commit();
              }
            }
            stored = true;
          }
        }
        if (!stored) {
          // per-warp walk: 16 x 32 sub-tiles transposed through the warp's padded staging tile
          float* stage_w = epi_stage + e * (16 * 33);
          const int row0 = m_blk * BLOCK_M + 16 * e;
          [[maybe_unused]] float sx = 0.f;
          if constexpr (kFp8) sx = __ldg(cg.scale_x);
          if (row0 < p.M) {                               // warp-uniform
#pragma unroll
            for (int c = 0; c < BN / 32; ++c) {
              if (col0 + 32 * c >= p.N) break;            // warp-uniform
#pragma unroll
              for (int i = 0; i < 4; ++i) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  float* dst = stage_w + ((lane >> 2) + 8 * h) * 33 + 8 * i + 2 * (lane & 3);
                  dst[0] = acc[4 * (4 * c + i) + 2 * h] * (GATHER == TILED_WGRAD ? alpha_w : p.alpha);
                  dst[1] = acc[4 * (4 * c + i) + 2 * h + 1] * (GATHER == TILED_WGRAD ? alpha_w : p.alpha);
                }
              }
              __syncwarp();
              if constexpr (kFp8) epilogue_tile16<EPI, true>(p, c_f32, stage_w, lane, row0, col0 + 32 * c, sx, cg.scale_w);
              else epilogue_tile16<EPI>(p, c_f32, stage_w, lane, row0, col0 + 32 * c);
              __syncwarp();
            }
          }
        }
      }
    }
    if constexpr (EPI != EPI_SGD) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // bulk row stores have landed
  }

  __syncthreads();
  if (share > 1) cluster_sync_all();   // no CTA leaves while a peer may still arrive on its barriers / multicast into it
}

template <int BN, bool A_MN, bool B_MN, int EPI, int GATHER = GATHER_NONE, int CG = 1>
__global__ void __launch_bounds__(kNumThreads + (has_gather_warps(GATHER) ? kGatherThreads : 0), 1)
wgmma_gemm_kernel(const __grid_constant__ TmapSet tm, const GemmParams p, const ConvGeom cg) {
  wgmma_gemm_body<BN, A_MN, B_MN, EPI, GATHER, CG, __nv_bfloat16, __nv_bfloat16>(tm, p, cg);
}

// e4m3 operands: the forward convolution with the im2col-TMA activation operand and the bf16 epilogue (conv_fprop_fp8).
template <int BN, int CG>
__global__ void __launch_bounds__(kNumThreads, 1)
wgmma_fp8_conv_kernel(const __grid_constant__ TmapSet tm, const GemmParams p, const ConvGeom cg) {
  wgmma_gemm_body<BN, false, false, EPI_BF16, IM2COL_A, CG, __nv_fp8_e4m3, __nv_fp8_e4m3>(tm, p, cg);
}

// e5m2 dY x e4m3 weights: the stride-1 data gradient (conv_dgrad_fp8) — the same im2col-A GEMM with the mirrored tap walk
// (ConvGeom::dr = -1); the epilogue dequantises per input channel and applies the producer's ReLU mask (p.mask).
template <int BN, int CG>
__global__ void __launch_bounds__(kNumThreads, 1)
wgmma_fp8_dgrad_kernel(const __grid_constant__ TmapSet tm, const GemmParams p, const ConvGeom cg) {
  wgmma_gemm_body<BN, false, false, EPI_BF16, IM2COL_A, CG, __nv_fp8_e5m2, __nv_fp8_e4m3>(tm, p, cg);
}

// e5m2 dY x e4m3 X: the stride-1 weight gradient (conv_wgrad_fp8).  Rows = output channels, columns = (tap, ci), the
// reduction runs over pixels with the batch innermost, read from CHWN copies as plain tiled boxes (TILED_WGRAD); fp32
// epilogue (split-K partials / add onto dw) scaled by s_dy * s_x * alpha.
template <int BN, int CG>
__global__ void __launch_bounds__(kNumThreads, 1)
wgmma_fp8_wgrad_kernel(const __grid_constant__ TmapSet tm, const GemmParams p, const ConvGeom cg) {
  wgmma_gemm_body<BN, false, false, EPI_F32, TILED_WGRAD, CG, __nv_fp8_e5m2, __nv_fp8_e4m3>(tm, p, cg);
}

// Persistent kernels on clusters: a grid holding more clusters than the GPU can run at once would leave its last clusters
// to run after all the others have finished (GPCs whose SM count is not a multiple of the cluster size strand SMs, so
// sms / cluster clusters do not always fit).  Largest grid, in CTAs, whose clusters are all resident together.
template <typename Kern>
inline int resident_cluster_ctas(Kern kern, int threads, int smem, int cluster) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(cluster);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kern, &cfg) != cudaSuccess || n < 1) {
    (void)cudaGetLastError();
    return cluster;
  }
  return n * cluster;
}

}  // namespace psd
