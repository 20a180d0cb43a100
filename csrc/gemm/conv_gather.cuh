// Implicit-GEMM convolution operand gather (im2col never materialised).
//
// Four producer warps (128 threads) build, directly in the 128B-swizzled shared-memory layout the wgmma
// descriptors expect, 64-element K slices of the virtual im2col matrix
//        A[m, k],   m = (n, oh, ow),   k = (r, s, c)          (NHWC input, channels innermost)
// with 16-byte cp.async copies (zero-fill for padding taps / tails).  Two addressing modes:
//   TAP : C_g % 8 == 0.  A 16-byte chunk is 8 channels of one tap.
//   ROW : first layers (C padded to 4): the S*C elements of one kernel row are contiguous in memory, so
//         K is organised as [R][Lp] (Lp = S*C rounded up to 8; the pad multiplies zero weights).
//
// Thread mapping (coalescing): thread t owns chunk column j = t & 7 and rows (t >> 3) + 16*i.  A warp-level
// cp.async therefore covers 4 rows x 128 contiguous bytes (4-8 L1 wavefronts) instead of 32 scattered 16-byte
// pieces (32 wavefronts).
//
// The producers are instruction-issue bound, so everything that depends only on the row m is taken out of the loop: a
// per-geometry ROW TABLE (8 bytes per output pixel, built once by conv_rowtab_kernel and cached on the host side)
// holds the element offset of tap (0,0) and a validity bit mask per kernel row / kernel column.  Per chunk the
// producer then needs one AND/compare for the bounds check and one add for the address.
//
// The same routine feeds fprop (A operand, K-major: 128 rows x 64 k), dgrad (gathers dY with mirrored taps)
// and wgrad (B operand, MN-major: 64 reduction rows x 64 k-columns per chunk).
//
// Replaces im2col_gpu_kernel/col2im_gpu_kernel + per-image cublasSgemm loops
// (reference: src/caffe/util/im2col.cu:12-132, src/caffe/layers/conv_layer.cu:13-119).
#pragma once
#include "fastdiv.cuh"
#include "sm90_prims.cuh"

namespace psd {

// Row-table entry for row m = (n, oh, ow) of the virtual im2col matrix.
//   base : element offset (from ConvGeom::x) of input element (n, ih0, iw0, 0), ih0 = oh*sh + off_h, iw0 = ow*sw + off_w
//          (may be negative / outside the image; only dereferenced for valid taps)
//   info : TAP mode: bit r       = kernel row r hits the image   (ih0 + r*dr in [0, H))
//                    bit 16 + s  = kernel column s hits the image (iw0 + s*dr in [0, W))
//          ROW mode: bit r as above, bits 16..31 = number of valid elements of a kernel row inside the image row
//   rows m >= M have info = 0 (all taps invalid -> zero fill)
struct RowPos {
  int base;
  uint32_t info;
};

struct ConvGeom {
  const __nv_bfloat16* x;   // gathered tensor (activations for fprop/wgrad, dY for dgrad), group offset applied
  const int2* rowtab;       // [Mtab] row table (see RowPos)
  int Mtab;
  int N, H, W;              // its spatial extent
  long pitch;               // pixel pitch in elements
  int Cg;                   // channels per group (TAP) / padded channels (ROW)
  int Cgk;                  // K-slots per tap (>= Cg: rounded up to 64 when the im2col-TMA path pads the channels; the
                            // tensor map's channel extent stays Cg, so slots [Cg, Cgk) are zero-filled by the TMA)
  int OH, OW;               // extent of the row index m = (n, oh, ow)
  int R, S, sh, sw;
  int off_h, off_w;         // ih = oh*sh + off_h + r*dr  (fprop: off=-pad, dr=+1 ; dgrad: off=+pad, dr=-1)
  int dr;
  int mode;                 // 0 TAP, 1 ROW
  int L, Lp;                // ROW: valid / padded elements per kernel row
  int K;                    // total reduction length (multiple of 8)
  long M;                   // N*OH*OW
  FastDiv div_ow, div_ohow, div_cg, div_s, div_lp;
  // fp8 kernels only: dequantisation scales read by the epilogue (device memory, so a captured graph sees each step's
  // values).  Kept last so that the kernel-parameter offsets of every other field stay those of the bf16 kernels.
  const float* scale_x;     // one float: the activation (fprop) / dY (dgrad) scale
  const float* scale_w;     // per output column of this group (output channel / input channel)
};

// Builds the row table (one thread per row).
static __global__ void conv_rowtab_kernel(ConvGeom g, int2* __restrict__ tab, int Mtab) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= Mtab) return;
  int2 e = make_int2(0, 0);
  if (m < g.M) {
    const uint32_t mm = static_cast<uint32_t>(m);
    const uint32_t n = fdiv(mm, g.div_ohow);
    const uint32_t rem = mm - n * static_cast<uint32_t>(g.OH * g.OW);
    const uint32_t oh = fdiv(rem, g.div_ow);
    const uint32_t ow = rem - oh * static_cast<uint32_t>(g.OW);
    const int ih0 = static_cast<int>(oh) * g.sh + g.off_h;
    const int iw0 = static_cast<int>(ow) * g.sw + g.off_w;
    const long base = (static_cast<long>(n) * g.H + ih0) * g.W * g.pitch + static_cast<long>(iw0) * g.pitch;
    uint32_t info = 0;
    for (int r = 0; r < g.R; ++r)
      if (static_cast<unsigned>(ih0 + r * g.dr) < static_cast<unsigned>(g.H)) info |= 1u << r;
    if (g.mode == 0) {
      for (int s = 0; s < g.S; ++s)
        if (static_cast<unsigned>(iw0 + s * g.dr) < static_cast<unsigned>(g.W)) info |= 1u << (16 + s);
    } else {
      const int lim = max(0, min(g.L, (g.W - iw0) * g.Cg));
      info |= static_cast<uint32_t>(lim) << 16;
    }
    e = make_int2(static_cast<int>(base), static_cast<int>(info));
  }
  tab[m] = e;
}

// The geometry fields the inner loops need, hoisted into registers once per role (the asm memory clobbers of
// cp.async would otherwise make the compiler re-read the kernel-parameter bank on every use).
struct GatherRegs {
  const __nv_bfloat16* x;
  const int2* rowtab;
  int Mtab, S, dr, Cg, Lp, K, mode, pitch;
  int row_step;               // elements between consecutive input rows (W * pitch)
  FastDiv div_cg, div_s, div_lp;
};
__device__ __forceinline__ GatherRegs load_gather_regs(const ConvGeom& g) {
  GatherRegs r;
  r.x = g.x; r.rowtab = g.rowtab; r.Mtab = g.Mtab; r.S = g.S; r.dr = g.dr; r.Cg = g.Cg; r.Lp = g.Lp; r.K = g.K;
  r.mode = g.mode; r.pitch = static_cast<int>(g.pitch);
  r.row_step = static_cast<int>(g.W * g.pitch);
  r.div_cg = g.div_cg; r.div_s = g.div_s; r.div_lp = g.div_lp;
  return r;
}

__device__ __forceinline__ RowPos load_row(const GatherRegs& g, long m) {
  RowPos p;
  p.base = 0;
  p.info = 0;
  if (m < g.Mtab) {
    const int2 e = __ldg(g.rowtab + m);
    p.base = e.x;
    p.info = static_cast<uint32_t>(e.y);
  }
  return p;
}

// Per-thread, per-k-block chunk decode with everything the row loop needs precomputed.
struct ChunkOff {
  uint32_t bits;     // TAP: (1 << r) | (1 << (16 + s)); ROW: (1 << r).  0 marks k >= K (never valid)
  int off;           // element offset from the row's base to this chunk
  int c;             // ROW mode: element offset inside the padded kernel row
};
__device__ __forceinline__ ChunkOff decode_chunk_off(const GatherRegs& g, int k) {
  ChunkOff t;
  if (g.mode == 0) {
    const uint32_t tap = fdiv(static_cast<uint32_t>(k), g.div_cg);
    const int c = k - static_cast<int>(tap) * g.Cg;
    const int r = static_cast<int>(fdiv(tap, g.div_s));
    const int s = static_cast<int>(tap) - r * g.S;
    t.bits = (1u << r) | (1u << (16 + s));
    t.off = (r * g.row_step + s * g.pitch) * g.dr + c;
    t.c = c;
  } else {
    const int r = static_cast<int>(fdiv(static_cast<uint32_t>(k), g.div_lp));
    t.c = k - r * g.Lp;
    t.bits = 1u << r;
    t.off = r * g.row_step + t.c;
  }
  if (k >= g.K) t.bits = 0xffffffffu;     // never matches: R, S <= 15, so no row has bits 15 / 31 set
  return t;
}

// One 16-byte chunk of one row: a handful of integer instructions + the cp.async.
__device__ __forceinline__ void gather_chunk_tap(const GatherRegs& g, uint32_t dst, const RowPos& pos, const ChunkOff& t) {
  const bool ok = (pos.info & t.bits) == t.bits;
  cp_async_16(dst, g.x + (ok ? pos.base + t.off : 0), ok ? 16u : 0u);
}
__device__ __forceinline__ void gather_chunk_row(const GatherRegs& g, uint32_t dst, const RowPos& pos, const ChunkOff& t) {
  const bool okh = (pos.info & 0xffffu & t.bits) == t.bits;
  int valid = min(8, static_cast<int>(pos.info >> 16) - t.c);
  if (!okh || valid < 0) valid = 0;
  cp_async_16(dst, g.x + (valid > 0 ? pos.base + t.off : 0), static_cast<uint32_t>(valid * 2));
}

}  // namespace psd
