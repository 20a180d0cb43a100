// Halo-tiled data gradient for stride-1 convolutions with narrow input groups (AlexNet conv2: 48 input channels per group,
// 5x5 taps).  The im2col schedule of conv_dgrad_w fetches a 128-pixel x 64-channel tile of dY for every (tap, channel
// chunk): each dY pixel crosses L2 -> SM R*S times, and with only 64 output columns there is too little MMA work per
// operand byte to hide it.  Here a CTA loads the dY halo of a tile ONCE into shared memory and walks the taps as address
// offsets into it.
//
// * Tile: T rows of one image's dX, laid out with the halo's pitch P = W + S - 1.  In that padded-pitch pixel space, tap
//   (r, s) of tile row m reads halo pixel m + (R-1-r)*P + (S-1-s) (the mirrored walk of the transposed convolution): a pure
//   shift.  Columns x >= W, rows past T or past the image are computed and never stored.  The tile is M = 64 * (NB0 + NB1)
//   rows: consumer warpgroup 0 owns 64-row blocks [0, NB0), warpgroup 1 blocks [NB0, NB0 + NB1).
// * Halo layout: no swizzle, K-major core matrices [channel / 8][pixel][8 channels]: 8 consecutive pixels x 16 B are one
//   contiguous 128-byte core matrix, so the A descriptor of (tap, 64-row block, k16 step) is valid at any pixel shift
//   (LBO = one 8-channel slab, SBO = 128 B).  One tiled TMA box per 8-channel slab ({8 ch, P, Hb rows, 1 image}); negative
//   and past-the-end coordinates are zero-filled, which is the convolution's padding.  Hb covers every pixel the dead rows
//   of the tile read, so all reads stay inside the box.
// * B: the fprop weight shadow [Cout][R][S][Cg] through the 3-D map conv_dgrad_w uses (MN-major, 128B swizzle, input
//   channels past Cg zero-filled); the two CTAs of a cluster pair walk the same k-block sequence on different tiles and
//   each fetches 32 of the 64 output-channel rows of a k block, multicast to both.
// * K order: taps in order, then 64-channel chunks of dY, then k16 steps — the order of the im2col kernel, so every dX
//   element is accumulated from the same products in the same order: bit-identical results.
// * Epilogue: that of conv_dgrad_w's bf16 per-warp walk (alpha 1, no bias; the producer's ReLU mask with its slope).
#pragma once
#include "sm90_prims.cuh"

namespace psd {

constexpr int kHaloThreads = 384;          // warp 0 TMA producer, warps 1-3 idle (warpgroup alignment), warps 4-11 MMA
constexpr int kHaloConsumerWarp0 = 4;
constexpr int kHaloStages = 8;             // B ring
constexpr int kHaloBStageBytes = 64 * 64 * 2;
constexpr int kHaloBarBytes = 256;
constexpr int kHaloSmemLimit = 232448;

struct HaloDgradParams {
  int N, H, W;              // dX extent
  int P, T;                 // halo row pitch (W + S - 1); dX rows per tile
  int tiles_per_img, num_tiles;
  int R, S, kcb;            // filter extent; 64-channel chunks of dY per tap
  int slabs, Hb, HP;        // 8-channel slabs; halo rows per box; slab stride in pixels (Hb * P rounded up to 8)
  int h_org, w_org;         // dY row / column of halo pixel 0, relative to the tile's first dX row and column 0
  uint32_t halo_bytes;      // transaction bytes of one halo (slabs * Hb * P * 16)
  __nv_bfloat16* dx;        // this group's first channel
  long ldc;                 // dX pixel pitch
  const __nv_bfloat16* mask;  // optional, laid out like dX
  float slope;
  int Cg;                   // output columns stored
};

__device__ __forceinline__ void tma_load_4d_u32(uint32_t smem_dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                                int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

// Shared-memory matrix descriptor without swizzle (layout field 0).
__device__ __forceinline__ uint64_t halo_smem_desc(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return static_cast<uint64_t>((addr & 0x3FFFF) >> 4) | (static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16) |
         (static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32);
}

// One warpgroup's share of a tile: NB 64-row blocks starting at block blk0.
template <int NB>
__device__ __forceinline__ void halo_consume_tile(const HaloDgradParams& p, float (&acc)[NB][32], uint64_t* full_bar,
                                                  uint64_t* empty_bar, uint32_t sb, uint32_t sh, int blk0, bool leader,
                                                  int& stage, uint32_t& phase) {
#pragma unroll
  for (int j = 0; j < NB; ++j)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[j][i] = 0.f;
  const uint64_t a0 = halo_smem_desc(sh, static_cast<uint32_t>(p.HP) * 16u, 128u) + static_cast<uint64_t>(blk0 * 64);
  int prev = -1;
  int r = 0, s = 0;
  for (int tap = 0; tap < p.R * p.S; ++tap) {
    const int shift = (p.R - 1 - r) * p.P + (p.S - 1 - s);
    for (int c = 0; c < p.kcb; ++c) {
      mbar_wait(&full_bar[stage], phase);
      const uint64_t b0 = make_smem_desc(sb + stage * kHaloBStageBytes, 8192, 1024);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        // channels [64c + 16kk, +16): slabs 8c + 2kk and 8c + 2kk + 1 (LBO apart)
        const uint64_t da = a0 + static_cast<uint64_t>((8 * c + 2 * kk) * p.HP + shift);
        const uint64_t db = b0 + static_cast<uint64_t>(kk * (16 * 128 / 16));
#pragma unroll
        for (int j = 0; j < NB; ++j) Wgmma<64, 0, 1>::mma(acc[j], da + static_cast<uint64_t>(j * 64), db, 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();                          // the previous k block's MMAs have retired: its slot is free
#pragma unroll
      for (int j = 0; j < NB; ++j) wgmma_fence_regs(acc[j]);
      if (prev >= 0 && leader) {
        mbar_arrive_remote(&empty_bar[prev], 0);
        mbar_arrive_remote(&empty_bar[prev], 1);
      }
      prev = stage;
      if (++stage == kHaloStages) { stage = 0; phase ^= 1; }
    }
    if (++s == p.S) { s = 0; ++r; }
  }
  wgmma_wait<0>();
#pragma unroll
  for (int j = 0; j < NB; ++j) wgmma_fence_regs(acc[j]);
  if (prev >= 0 && leader) {
    mbar_arrive_remote(&empty_bar[prev], 0);
    mbar_arrive_remote(&empty_bar[prev], 1);
  }
}

// dX rows of the warp's 16-row slice of each block, straight from the accumulator fragment (see Wgmma): lane holds rows
// (lane / 4) and (lane / 4) + 8, column pairs 8i + 2 (lane % 4).  Numerics of conv_dgrad_w's per-warp walk: acc * 1 + 0,
// then the mask's slope where the producer's output was <= 0, then round to bf16.
template <int NB>
__device__ __forceinline__ void halo_store_tile(const HaloDgradParams& p, const float (&acc)[NB][32], int blk0, int w4, int lane,
                                                int n, int h0) {
#pragma unroll
  for (int j = 0; j < NB; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = (blk0 + j) * 64 + 16 * w4 + (lane >> 2) + 8 * h;
      const int tr = m / p.P, x = m - tr * p.P;
      if (x >= p.W || tr >= p.T || h0 + tr >= p.H) continue;
      const long off = ((static_cast<long>(n) * p.H + h0 + tr) * p.W + x) * p.ldc;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int col = 8 * i + 2 * (lane & 3);
        if (col >= p.Cg) continue;              // Cg % 8 == 0: both columns of the pair are in range or both are not
        float x0 = acc[j][4 * i + 2 * h] + 0.f, x1 = acc[j][4 * i + 2 * h + 1] + 0.f;
        if (p.mask != nullptr) {
          const uint32_t mk = __ldg(reinterpret_cast<const unsigned int*>(p.mask + off + col));
          if (!(__uint_as_float(mk << 16) > 0.f)) x0 *= p.slope;
          if (!(__uint_as_float(mk & 0xffff0000u) > 0.f)) x1 *= p.slope;
        }
        *reinterpret_cast<__nv_bfloat162*>(p.dx + off + col) = __floats2bfloat162_rn(x0, x1);
      }
    }
  }
}

// Launched on (2,1,1) clusters; the grid is a multiple of 2.  The pair walks pair-tiles; CTA `rank` owns tile
// 2 * pair_tile + rank (a phantom tile past the end loads the last real tile's halo and stores nothing).
template <int NB0, int NB1>
__global__ void __launch_bounds__(kHaloThreads, 1)
halo_dgrad_kernel(const __grid_constant__ CUtensorMap halo_map, const __grid_constant__ CUtensorMap w_map,
                  const HaloDgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sb = smem_u32(smem);                                   // B ring (1024-aligned: 128B swizzle)
  const uint32_t sh = sb + kHaloStages * kHaloBStageBytes;              // halo slabs
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kHaloStages * kHaloBStageBytes + p.slabs * p.HP * 16);
  uint64_t* empty_bar = full_bar + kHaloStages;
  uint64_t* halo_full = empty_bar + kHaloStages;
  uint64_t* halo_empty = halo_full + 1;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int crank = static_cast<int>(cluster_ctarank());
  const int pair_tiles = (p.num_tiles + 1) / 2;
  const int kb_per_tile = p.R * p.S * p.kcb;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&halo_map);
    tma_prefetch_desc(&w_map);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kHaloStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2 * 2);          // one arrive per consumer warpgroup of both CTAs
    }
    mbar_init(halo_full, 1);
    mbar_init(halo_empty, 2);                   // both consumer warpgroups of this CTA
    fence_barrier_init();
  }
  __syncthreads();
  cluster_sync_all();                           // the peer's barriers exist before any multicast / remote arrive

  if (warp == 0) {
    // ===================== TMA producer (warp-uniform loop, one elected lane issues) =====================
    int stage = 0;
    uint32_t phase = 0, hphase = 0;
    for (int pt = blockIdx.x / 2; pt < pair_tiles; pt += gridDim.x / 2) {
      const int tile = min(2 * pt + crank, p.num_tiles - 1);
      const int n = tile / p.tiles_per_img, h0 = (tile - n * p.tiles_per_img) * p.T;
      mbar_wait(halo_empty, hphase ^ 1);        // the previous tile's MMAs have all retired
      if (elect_one()) {
        mbar_arrive_expect_tx(halo_full, p.halo_bytes);
        for (int sl = 0; sl < p.slabs; ++sl)
          tma_load_4d_u32(sh + sl * p.HP * 16, &halo_map, smem_u32(halo_full), 8 * sl, p.w_org, h0 + p.h_org, n);
      }
      __syncwarp();
      hphase ^= 1;
      int tap = 0, c = 0;
      for (int kb = 0; kb < kb_per_tile; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (elect_one()) {
          const uint32_t fb = smem_u32(&full_bar[stage]);
          mbar_arrive_expect_tx(&full_bar[stage], kHaloBStageBytes);
          // rows [32 rank, 32 rank + 32) of the k block's 64 output channels, into both CTAs of the pair
          tma_load_3d_mcast_u32(sb + stage * kHaloBStageBytes + crank * (32 * 128), &w_map, fb, 0, 64 * c + 32 * crank, tap,
                                0x3);
        }
        __syncwarp();
        if (++c == p.kcb) { c = 0; ++tap; }
        if (++stage == kHaloStages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= kHaloConsumerWarp0) {
    // ===================== consumer warpgroups =====================
    const int e = warp - kHaloConsumerWarp0;
    const int wg = e >> 2, w4 = e & 3;
    const bool leader = w4 == 0 && lane == 0;
    int stage = 0;
    uint32_t phase = 0, hphase = 0;
    for (int pt = blockIdx.x / 2; pt < pair_tiles; pt += gridDim.x / 2) {
      const int tile = 2 * pt + crank;
      const int n = tile / p.tiles_per_img, h0 = (tile - n * p.tiles_per_img) * p.T;
      mbar_wait(halo_full, hphase);
      hphase ^= 1;
      if (wg == 0) {
        float acc[NB0][32];
        halo_consume_tile<NB0>(p, acc, full_bar, empty_bar, sb, sh, 0, leader, stage, phase);
        if (leader) mbar_arrive(halo_empty);
        if (tile < p.num_tiles) halo_store_tile<NB0>(p, acc, 0, w4, lane, n, h0);
      } else {
        float acc[NB1][32];
        halo_consume_tile<NB1>(p, acc, full_bar, empty_bar, sb, sh, NB0, leader, stage, phase);
        if (leader) mbar_arrive(halo_empty);
        if (tile < p.num_tiles) halo_store_tile<NB1>(p, acc, NB0, w4, lane, n, h0);
      }
    }
  }
  __syncthreads();
  cluster_sync_all();                           // no CTA leaves while its peer may still multicast into it / arrive on it
}

// ------------------------------------------------------------------------------------------------------------------------
// Halo-tiled forward for stride-1 convolutions with narrow input groups (AlexNet conv2: 48 channels per group, 5x5 taps).
// The gather schedule of conv_fprop builds a 128-pixel x 64-channel A tile per 64-wide k block, so every input pixel
// crosses L2 -> SM R*S times.  Here a CTA loads the input halo of a tile once and walks the taps as descriptor shifts.
//
// * Tile: T rows of one image's output in a pixel space of pitch P = OW + S - 1; tap (r, s) of tile row m reads halo pixel
//   m + r*P + s.  Columns x >= OW, rows past T or past OH are computed and never stored.  M = 64 * (NB0 + NB1) rows as in
//   the data gradient; each CTA computes one 64-wide block of the group's output channels (wgmma m64n64k16).
// * Halo: Cg / 8 non-swizzled [pixel][8 ch] slabs, one tiled TMA box per slab with origin (row h0 - ph, column -pw); the
//   zero fill outside the image is the padding.  Two halo buffers: the next tile's halo loads while this tile's MMAs run.
// * B: the forward weight shadow wb [Cout][R*S*Cg] through a 2-D K-major map (128B swizzle), in the 64-column k blocks the
//   gather kernel reads (the last one zero-filled past K).  The two CTAs of a pair take different spatial tiles of the
//   same 64 output channels; each fetches 32 of the 64 rows of a k block and multicasts them to both.
// * K order: k16 step j covers K columns [16j, 16j + 16) = tap j / (Cg/16), slabs 2 (j mod Cg/16) and +1, B slice j mod 4
//   of k block j / 4 (Cg % 16 == 0: no step straddles a tap).  Steps run in order over whole k blocks; those past K (the
//   tail of the last block, B zero-filled) read A from 2 KB of zeros.  That is the gather kernel's sequence of products,
//   zero tail included, so every output is accumulated from the same products in the same order: bit-identical results.
// * Epilogue: the arithmetic of epilogue_tile16<EPI_BF16> at alpha 1 (acc + bias, leaky ReLU, round to bf16).
// * One launch covers every group: the halo map spans all input channels (the group sets the channel coordinate) and the
//   weight map all output channels.
constexpr int kHaloZeroBytes = 2048;       // halo forward: 64 rows x 16 channels of zeros (the A operand of steps past K)

struct HaloFpropParams {
  int OH, OW;               // output extent
  int P, T;                 // halo row pitch (OW + S - 1); output rows per tile
  int tiles_per_img, num_tiles;   // spatial tiles per image; per (group, channel block)
  int nblk, cblocks;        // 64-wide output-channel blocks per group; groups * nblk
  int S, Cg, Cout_g;
  int steps, kb_per_tile;   // k16 steps per tile (R*S*Cg/16); 64-wide k blocks per tile
  int slabs, Hb, HP;        // 8-channel slabs; halo rows per box; slab stride in pixels (Hb * P rounded up to 8)
  int ph, pw;
  uint32_t halo_bytes;      // transaction bytes of one halo (slabs * Hb * P * 16)
  __nv_bfloat16* y;         // output, first channel
  long ldc;                 // output pixel pitch
  const float* bias;        // optional, per output channel
  int relu;
  float slope;
};

// One warpgroup's share of a tile: NB 64-row blocks starting at block blk0, halo at shared address sh, 2 KB of zeros at sz.
template <int NB>
__device__ __forceinline__ void halo_fprop_consume(const HaloFpropParams& p, float (&acc)[NB][32], uint64_t* full_bar,
                                                   uint64_t* empty_bar, uint32_t sb, uint32_t sh, uint32_t sz, int blk0,
                                                   bool leader, int& stage, uint32_t& phase) {
#pragma unroll
  for (int j = 0; j < NB; ++j)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[j][i] = 0.f;
  const uint64_t a0 = halo_smem_desc(sh, static_cast<uint32_t>(p.HP) * 16u, 128u) + static_cast<uint64_t>(blk0 * 64);
  const int cpt = p.Cg / 16;                    // k16 steps per tap
  const uint64_t az = halo_smem_desc(sz, 1024u, 128u);   // 64 rows x 16 channels of zeros
  int prev = -1, step = 0;
  int cp = 0, r = 0, s = 0;                     // channel pair, tap row and tap column of the next k16 step
  for (int kb = 0; kb < p.kb_per_tile; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint64_t b0 = make_smem_desc(sb + stage * kHaloBStageBytes, 16, 1024);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk, ++step) {
      // steps past K (the tail of the last k block, whose B is zero-filled) multiply zeros, as the gather kernel's do
      const bool in_k = step < p.steps;
      const uint64_t da = a0 + static_cast<uint64_t>(2 * cp * p.HP + r * p.P + s);
      const uint64_t db = b0 + static_cast<uint64_t>(kk * (16 * 2 / 16));
#pragma unroll
      for (int j = 0; j < NB; ++j) Wgmma<64, 0, 0>::mma(acc[j], in_k ? da + static_cast<uint64_t>(j * 64) : az, db, 1u);
      if (++cp == cpt) {
        cp = 0;
        if (++s == p.S) { s = 0; ++r; }
      }
    }
    wgmma_commit();
    wgmma_wait<1>();                            // the previous k block's MMAs have retired: its slot is free
#pragma unroll
    for (int j = 0; j < NB; ++j) wgmma_fence_regs(acc[j]);
    if (prev >= 0 && leader) {
      mbar_arrive_remote(&empty_bar[prev], 0);
      mbar_arrive_remote(&empty_bar[prev], 1);
    }
    prev = stage;
    if (++stage == kHaloStages) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
#pragma unroll
  for (int j = 0; j < NB; ++j) wgmma_fence_regs(acc[j]);
  if (prev >= 0 && leader) {
    mbar_arrive_remote(&empty_bar[prev], 0);
    mbar_arrive_remote(&empty_bar[prev], 1);
  }
}

// Output rows of the warp's 16-row slice of each block, straight from the accumulator fragment (lane holds rows (lane / 4)
// and (lane / 4) + 8, column pairs 8i + 2 (lane % 4)); y points at the tile's first output channel.
template <int NB>
__device__ __forceinline__ void halo_fprop_store(const HaloFpropParams& p, const float (&acc)[NB][32], int blk0, int w4,
                                                 int lane, int n, int h0, __nv_bfloat16* y, const float* bias) {
#pragma unroll
  for (int j = 0; j < NB; ++j) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = (blk0 + j) * 64 + 16 * w4 + (lane >> 2) + 8 * h;
      const int tr = m / p.P, x = m - tr * p.P;
      if (x >= p.OW || tr >= p.T || h0 + tr >= p.OH) continue;
      const long off = ((static_cast<long>(n) * p.OH + h0 + tr) * p.OW + x) * p.ldc;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int col = 8 * i + 2 * (lane & 3);
        float b0 = 0.f, b1 = 0.f;
        if (bias != nullptr) {
          b0 = __ldg(bias + col);
          b1 = __ldg(bias + col + 1);
        }
        float x0 = acc[j][4 * i + 2 * h] + b0, x1 = acc[j][4 * i + 2 * h + 1] + b1;
        if (p.relu) {
          x0 = x0 > 0.f ? x0 : x0 * p.slope;
          x1 = x1 > 0.f ? x1 : x1 * p.slope;
        }
        *reinterpret_cast<__nv_bfloat162*>(y + off + col) = __floats2bfloat162_rn(x0, x1);
      }
    }
  }
}

// Launched on (2,1,1) clusters; the grid is a multiple of 2.  The pair walks pair-tiles, channel block fastest (the CTAs
// running at the same time read the same input halos); CTA `rank` owns spatial tile 2 * spatial_pair + rank (a phantom
// tile past the end loads the last real tile's halo and stores nothing).
template <int NB0, int NB1>
__global__ void __launch_bounds__(kHaloThreads, 1)
halo_fprop_kernel(const __grid_constant__ CUtensorMap halo_map, const __grid_constant__ CUtensorMap w_map,
                  const HaloFpropParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t halo_buf = static_cast<uint32_t>(p.slabs * p.HP * 16);
  const uint32_t sb = smem_u32(smem);                                   // B ring (1024-aligned: 128B swizzle)
  const uint32_t sh = sb + kHaloStages * kHaloBStageBytes;              // two halo buffers
  const uint32_t sz = sh + 2 * halo_buf;                                // A operand of the steps past K
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kHaloStages * kHaloBStageBytes + 2 * halo_buf + kHaloZeroBytes);
  uint64_t* empty_bar = full_bar + kHaloStages;
  uint64_t* halo_full = empty_bar + kHaloStages;    // [2]
  uint64_t* halo_empty = halo_full + 2;             // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int crank = static_cast<int>(cluster_ctarank());
  const int pair_tiles = (p.num_tiles + 1) / 2 * p.cblocks;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&halo_map);
    tma_prefetch_desc(&w_map);
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kHaloStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2 * 2);          // one arrive per consumer warpgroup of both CTAs
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(&halo_full[b], 1);
      mbar_init(&halo_empty[b], 2);             // both consumer warpgroups of this CTA
    }
    fence_barrier_init();
  }
  if (threadIdx.x >= kHaloConsumerWarp0 * 32) {
    for (int i = threadIdx.x - kHaloConsumerWarp0 * 32; i < kHaloZeroBytes / 16; i += kHaloThreads - kHaloConsumerWarp0 * 32)
      *reinterpret_cast<uint4*>(smem + (sz - sb) + 16 * i) = make_uint4(0, 0, 0, 0);
    fence_proxy_async_smem();                   // generic-proxy writes -> visible to wgmma
  }
  __syncthreads();
  cluster_sync_all();                           // the peer's barriers exist before any multicast / remote arrive

  if (warp == 0) {
    // ===================== TMA producer (warp-uniform loop, one elected lane issues) =====================
    int stage = 0, it = 0;
    uint32_t phase = 0;
    for (int pt = blockIdx.x / 2; pt < pair_tiles; pt += gridDim.x / 2, ++it) {
      const int cb = pt % p.cblocks, g = cb / p.nblk;
      const int tile = min(2 * (pt / p.cblocks) + crank, p.num_tiles - 1);
      const int n = tile / p.tiles_per_img, h0 = (tile - n * p.tiles_per_img) * p.T;
      const int buf = it & 1;
      mbar_wait(&halo_empty[buf], ((it >> 1) & 1) ^ 1);   // the MMAs of the tile before last (same buffer) have retired
      if (elect_one()) {
        mbar_arrive_expect_tx(&halo_full[buf], p.halo_bytes);
        for (int sl = 0; sl < p.slabs; ++sl)
          tma_load_4d_u32(sh + buf * halo_buf + sl * p.HP * 16, &halo_map, smem_u32(&halo_full[buf]), g * p.Cg + 8 * sl,
                          -p.pw, h0 - p.ph, n);
      }
      __syncwarp();
      const int row0 = g * p.Cout_g + (cb - g * p.nblk) * 64 + 32 * crank;
      for (int kb = 0; kb < p.kb_per_tile; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        if (elect_one()) {
          const uint32_t fb = smem_u32(&full_bar[stage]);
          mbar_arrive_expect_tx(&full_bar[stage], kHaloBStageBytes);
          // rows [32 rank, 32 rank + 32) of the block's 64 output channels, into both CTAs of the pair
          tma_load_2d_mcast_u32(sb + stage * kHaloBStageBytes + crank * (32 * 128), &w_map, fb, 64 * kb, row0, 0x3);
        }
        __syncwarp();
        if (++stage == kHaloStages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= kHaloConsumerWarp0) {
    // ===================== consumer warpgroups =====================
    const int e = warp - kHaloConsumerWarp0;
    const int wg = e >> 2, w4 = e & 3;
    const bool leader = w4 == 0 && lane == 0;
    int stage = 0, it = 0;
    uint32_t phase = 0;
    for (int pt = blockIdx.x / 2; pt < pair_tiles; pt += gridDim.x / 2, ++it) {
      const int cb = pt % p.cblocks, g = cb / p.nblk;
      const int tile = 2 * (pt / p.cblocks) + crank;
      const int n = tile / p.tiles_per_img, h0 = (tile - n * p.tiles_per_img) * p.T;
      const int c0 = g * p.Cout_g + (cb - g * p.nblk) * 64;
      const int buf = it & 1;
      mbar_wait(&halo_full[buf], (it >> 1) & 1);
      const uint32_t hb = sh + buf * halo_buf;
      __nv_bfloat16* y = p.y + c0;
      const float* bias = p.bias != nullptr ? p.bias + c0 : nullptr;
      if (wg == 0) {
        float acc[NB0][32];
        halo_fprop_consume<NB0>(p, acc, full_bar, empty_bar, sb, hb, sz, 0, leader, stage, phase);
        if (leader) mbar_arrive(&halo_empty[buf]);
        if (tile < p.num_tiles) halo_fprop_store<NB0>(p, acc, 0, w4, lane, n, h0, y, bias);
      } else {
        float acc[NB1][32];
        halo_fprop_consume<NB1>(p, acc, full_bar, empty_bar, sb, hb, sz, NB0, leader, stage, phase);
        if (leader) mbar_arrive(&halo_empty[buf]);
        if (tile < p.num_tiles) halo_fprop_store<NB1>(p, acc, NB0, w4, lane, n, h0, y, bias);
      }
    }
  }
  __syncthreads();
  cluster_sync_all();                           // no CTA leaves while its peer may still multicast into it / arrive on it
}

}  // namespace psd
