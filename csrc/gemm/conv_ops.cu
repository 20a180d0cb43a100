// Implicit-GEMM convolution on the wgmma GEMM core: fprop, dgrad (stride 1), wgrad (split-K, partials summed in order).
//
// Layouts (sm100 engine): activations NHWC bf16 (pixel pitch may exceed C for channel-slice views);
// weights fp32 master + bf16 shadow as [Cout][R][S][Cg] ("KRSC", K-major rows of length R*S*Cg), or
// [Cout][R][Lp] for first layers in ROW mode (see conv_gather.cuh).
//
// reference semantics: src/caffe/layers/conv_layer.cpp:114-155 (output size, groups),
// conv_layer.cu:13-44 (fprop + bias), :48-119 (bias / weight / data gradients).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/library.h>
#include <torch/types.h>

#include <array>
#include <map>
#include <mutex>
#include <type_traits>
#include <vector>

#include "../ops/nhwc_common.cuh"
#include "wgmma_gemm.cuh"

namespace psd {

void encode_tmap_bf16_3d(CUtensorMap* map, const void* base, int64_t d0, int64_t d1, int64_t d2, int64_t stride1, int64_t stride2,
                         int box0, int box1, int box2);
void splitk_reduce(const at::Tensor& ws, int splits, float* out, long ldo, int M, int N, bool accumulate,
                   cudaStream_t stream);

static int g_conv_im2col = 1;      // TMA im2col-mode operand fetch where the geometry allows it (C_g % 64 == 0)

static int g_conv_cluster = 1;     // CTAs per cluster sharing the TMA operand by multicast (1 = off)

int pair_cta_enabled();
extern int g_max_stages;
extern int g_no_bulk_epi;

template <int BN, bool A_MN, bool B_MN, int EPI, int GATHER, int CG = 1, typename T = __nv_bfloat16>
static void launch_conv(const TmapSet& tm, const GemmParams& p, const ConvGeom& cg, int grid, cudaStream_t stream) {
  auto kern = [] {
    if constexpr (std::is_same<T, __nv_fp8_e5m2>::value) return wgmma_fp8_dgrad_kernel<BN, CG>;
    else if constexpr (sizeof(T) == 1) return wgmma_fp8_conv_kernel<BN, CG>;
    else return wgmma_gemm_kernel<BN, A_MN, B_MN, EPI, GATHER, CG>;
  }();
  constexpr int smem = GemmSmem<BN, CG>::kTotal;
  static bool configured = false;
  if (!configured) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  constexpr int threads = kNumThreads + (has_gather_warps(GATHER) ? kGatherThreads : 0);
  const int cluster = CG == 2 ? 2 : p.cluster;
  if (cluster <= 1) {
    kern<<<grid, threads, smem, stream>>>(tm, p, cg);
  } else {
    static std::map<int, int> resident;                 // per cluster size (conv clusters come in 2, 3 and 4)
    static std::mutex mu;
    {
      std::lock_guard<std::mutex> lock(mu);
      auto it = resident.find(cluster);
      if (it == resident.end()) it = resident.emplace(cluster, resident_cluster_ctas(kern, threads, smem, cluster)).first;
      grid = std::min(grid, it->second);
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = cluster;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    C10_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, tm, p, cg));
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// Grid of a CTA-pair launch: one CTA pair per pair-tile, at most sms/2 pairs.
static int pair_grid(long m_blocks, long n_blocks, long split, int sms) {
  const long pair_tiles = ((m_blocks + 1) / 2) * n_blocks * split;
  return static_cast<int>(2 * std::max<long>(1, std::min<long>(pair_tiles, sms / 2)));
}

static int g_conv_mcast = 1;       // CTAs per cluster sharing the im2col operand by TMA multicast (1 = off, the default:
                                   // every SM still ingests the whole tile)
static int g_conv_pair = 1;        // CTA pairs sharing the weight / im2col B tile for the im2col convolution kernels

// Launch the im2col-A kernel (fprop / dgrad) for tile width bn; CG = 2: CTA pairs, else cluster multicast (p.cluster).
template <int CG>
static void launch_im2col_a(int bn, const TmapSet& tm, const GemmParams& p, const ConvGeom& cg, int grid, cudaStream_t stream) {
  switch (bn) {
    case 32:
      if constexpr (CG == 1) launch_conv<32, false, false, EPI_BF16, IM2COL_A, 1>(tm, p, cg, grid, stream);
      else TORCH_CHECK(false, "CTA pairs: BLOCK_N >= 64");
      break;
    case 64: launch_conv<64, false, false, EPI_BF16, IM2COL_A, CG>(tm, p, cg, grid, stream); break;
    case 96:
      if constexpr (CG == 1) launch_conv<96, false, false, EPI_BF16, IM2COL_A, 1>(tm, p, cg, grid, stream);
      else TORCH_CHECK(false, "CTA pairs: BLOCK_N 96 is not instantiated");
      break;
    case 128: launch_conv<128, false, false, EPI_BF16, IM2COL_A, CG>(tm, p, cg, grid, stream); break;
    case 192: launch_conv<192, false, false, EPI_BF16, IM2COL_A, CG>(tm, p, cg, grid, stream); break;
    case 256: launch_conv<256, false, false, EPI_BF16, IM2COL_A, CG>(tm, p, cg, grid, stream); break;
    default: TORCH_CHECK(false, "unsupported conv BLOCK_N ", bn);
  }
}

// Multicast plan for an im2col-A convolution with n_cols output columns: the cluster's C CTAs take C consecutive column
// blocks of the SAME pixel tile and each fetches 128 / C of its pixel rows.  The tile width is the narrowest
// instantiated one that covers n_cols / C.  Returns C (1 = no multicast) and sets *bn, *grid.
static int plan_im2col_mcast(long n_cols, long m_blocks, int sms, int* bn, int* grid) {
  int c = g_conv_mcast;
  if (c <= 1 || n_cols < 32) return 1;
  while (c > 1 && n_cols < 32L * c) c >>= 1;
  if (c <= 1) return 1;
  const long want = (n_cols + c - 1) / c;
  int w = 256;
  for (int cand : {256, 192, 128, 96, 64, 32})
    if (cand >= want) w = cand;
  *bn = w;
  const long n_blocks = (n_cols + w - 1) / w;
  const long cluster_tiles = m_blocks * ((n_blocks + c - 1) / c);
  const int usable = (sms / c) * c;             // launch_conv caps the grid at the clusters that fit at once
  *grid = static_cast<int>(std::max<long>(c, std::min<long>(cluster_tiles * c, (usable / c) * c)));
  return c;
}

// cluster size to use for a tile space of `tiles_along` blocks along the cluster dimension, and the grid
static int pick_cluster(long tiles_along, long tiles_total, int sms, int* grid) {
  int c = g_conv_cluster;
  while (c > 1 && tiles_along < c) c >>= 1;
  const int usable = sms;                       // launch_conv caps the grid at the clusters that fit at once
  const long ctiles = (tiles_total + c - 1) / c;              // cluster tiles (upper bound incl. edge padding)
  long g = std::min<long>(ctiles * c, (usable / c) * c);
  g = std::max<long>(c, (g / c) * c);
  *grid = static_cast<int>(g);
  return c;
}

// Row tables (conv_gather.cuh) depend only on the geometry, not on the data pointer: built once per distinct
// (device, geometry) and kept for the life of the process (8 bytes per output pixel).  The first call for a geometry
// happens in the warm-up iterations, i.e. outside any CUDA-graph capture.
static void attach_rowtab(ConvGeom& g, int device) {
  using Key = std::array<long, 18>;
  static std::map<Key, at::Tensor> cache;
  static std::mutex mu;
  const Key key{device, g.N, g.H, g.W, g.pitch, g.Cg, g.OH, g.OW, g.R, g.S, g.sh, g.sw, g.off_h, g.off_w, g.dr, g.mode, g.L, g.M};
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it == cache.end()) {
    const long mtab = (g.M + BLOCK_M - 1) / BLOCK_M * BLOCK_M;
    at::Tensor tab = at::empty({mtab, 2}, at::TensorOptions().dtype(at::kInt).device(at::kCUDA, device));
    g.rowtab = nullptr;
    g.Mtab = static_cast<int>(mtab);
    conv_rowtab_kernel<<<static_cast<unsigned>((mtab + 255) / 256), 256, 0, at::cuda::getCurrentCUDAStream()>>>(
        g, reinterpret_cast<int2*>(tab.data_ptr<int>()), static_cast<int>(mtab));
    C10_CUDA_KERNEL_LAUNCH_CHECK();
    it = cache.emplace(key, tab).first;
  }
  g.rowtab = reinterpret_cast<const int2*>(it->second.data_ptr<int>());
  g.Mtab = static_cast<int>(it->second.size(0));
}

struct ConvDesc {
  int R, S, sh, sw, ph, pw, groups;
  int mode;      // 0 TAP, 1 ROW
};

static ConvGeom make_geom(const at::Tensor& x, const NhwcView& xv, int c_off, int Cg, int OH, int OW, const ConvDesc& d,
                          bool dgrad, int Cgk = 0) {
  ConvGeom g{};
  g.x = reinterpret_cast<const __nv_bfloat16*>(x.data_ptr()) + c_off;
  g.N = xv.N; g.H = xv.H; g.W = xv.W;
  g.pitch = xv.pitch;
  g.Cg = Cg;
  g.Cgk = Cgk > 0 ? Cgk : Cg;
  g.OH = OH; g.OW = OW;
  g.R = d.R; g.S = d.S;
  g.sh = dgrad ? 1 : d.sh; g.sw = dgrad ? 1 : d.sw;
  g.off_h = dgrad ? d.ph : -d.ph;
  g.off_w = dgrad ? d.pw : -d.pw;
  g.dr = dgrad ? -1 : 1;
  g.mode = d.mode;
  g.L = d.S * Cg;
  g.Lp = (g.L + 7) / 8 * 8;
  g.K = d.mode == 1 ? d.R * g.Lp : d.R * d.S * g.Cgk;
  g.M = static_cast<long>(xv.N) * OH * OW;
  TORCH_CHECK(g.M < (1L << 31), "conv: N*OH*OW must fit in 31 bits");
  g.div_ow = make_fastdiv(OW);
  g.div_ohow = make_fastdiv(static_cast<uint32_t>(OH) * OW);
  g.div_cg = make_fastdiv(g.Cgk);
  g.div_s = make_fastdiv(d.S);
  g.div_lp = make_fastdiv(g.Lp);
  TORCH_CHECK(d.R <= 15 && d.S <= 15, "conv: kernel extents up to 15 are supported");
  TORCH_CHECK(static_cast<long>(xv.N) * xv.H * xv.W * xv.pitch < (1L << 31), "conv: gathered tensor must have < 2^31 elements");
  if (d.mode == 1) {
    TORCH_CHECK(xv.pitch == Cg, "ROW-mode conv needs a dense input (pitch == channels)");
    TORCH_CHECK(d.ph == 0 && d.pw == 0, "ROW-mode conv expects a pre-padded input");
    TORCH_CHECK((d.sw * Cg) % 8 == 0 && (xv.W * Cg) % 8 == 0, "ROW-mode conv: 16-byte alignment of kernel rows");
  } else {
    TORCH_CHECK(Cg % 8 == 0 && xv.pitch % 8 == 0 && c_off % 8 == 0, "TAP-mode conv: channels must be multiples of 8");
  }
  attach_rowtab(g, x.device().index());
  return g;
}

// TMA im2col eligibility: TAP mode, K slices of one 128-byte row (64 bf16 / 128 fp8 channels, `es` bytes per element)
// never straddle a tap, corner offsets fit the descriptor.
// On success fills `map` for boxes of `pixels` base pixels x 128 bytes of channels over the gathered tensor.
static bool im2col_ok(const ConvGeom& g, int es = 2) {
  if (!g_conv_im2col || g.mode != 0 || g.Cgk % (128 / es) != 0) return false;
  const int org_w = g.off_w - (g.dr < 0 ? g.S - 1 : 0), org_h = g.off_h - (g.dr < 0 ? g.R - 1 : 0);
  // the bounding box must enumerate exactly OW x OH base pixels: extent + upper - lower - 1 = (O - 1) * stride
  const int up_w = (g.OW - 1) * g.sw + 1 + org_w - g.W, up_h = (g.OH - 1) * g.sh + 1 + org_h - g.H;
  auto ok = [](int v) { return v >= -128 && v <= 127; };
  if (!ok(org_w) || !ok(org_h) || !ok(up_w) || !ok(up_h) || g.sw > 8 || g.sh > 8) return false;
  return (reinterpret_cast<uintptr_t>(g.x) & 15) == 0 && (g.pitch * es) % 16 == 0;
}
static bool try_im2col_map(CUtensorMap* map, const ConvGeom& g, int pixels, int es = 2) {
  if (!im2col_ok(g, es)) return false;
  const int org_w = g.off_w - (g.dr < 0 ? g.S - 1 : 0), org_h = g.off_h - (g.dr < 0 ? g.R - 1 : 0);
  const int up_w = (g.OW - 1) * g.sw + 1 + org_w - g.W, up_h = (g.OH - 1) * g.sh + 1 + org_h - g.H;
  encode_tmap_im2col(map, g.x, g.Cg, g.W, g.H, g.N, g.pitch, org_w, org_h, up_w, up_h, pixels, g.sw, g.sh,
                     es == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
  return true;
}

// Widest N tile that does not over-pad the channel count and still yields a full wave of CTAs; small problems
// (GoogLeNet's 14x14 / 7x7 stages at batch 32) take the narrowest tile so that more SMs get work.
static int pick_conv_bn(int64_t n_cols, int64_t m_blocks, int sms) {
  // candidates widest first; 192 only where it removes >= 15 % padding (a narrower tile pays the A operand again)
  int best = 64;
  long best_pad = -1;
  for (int bn : {256, 192, 128, 64}) {
    const long padded = (n_cols + bn - 1) / bn * bn;
    if (best_pad < 0 || padded * 100 < best_pad * (bn == 192 ? 85 : 100)) {
      if (best_pad < 0 || padded < best_pad) { best = bn; best_pad = padded; }
    }
  }
  // small problems (GoogLeNet's 14x14 / 7x7 stages at batch 32): narrow the tile until a full wave of CTAs has work
  int bn = best;
  while (bn > 64 && m_blocks * ((n_cols + bn - 1) / bn) < sms) bn = (bn == 256 ? 128 : (bn == 192 ? 128 : 64));
  return bn;
}

// y[N, Cout, OH, OW] (NHWC bf16) = act(conv(x, w) + bias).  wb: [Cout, Kw] bf16 (Kw = R*S*Cg or R*Lp).
at::Tensor conv_fprop(const at::Tensor& x, const at::Tensor& wb, const c10::optional<at::Tensor>& bias, at::IntArrayRef kernel,
                      at::IntArrayRef stride, at::IntArrayRef pad, int64_t groups, int64_t mode, int64_t OH, int64_t OW,
                      bool relu, double slope, c10::optional<at::Tensor> out) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && wb.scalar_type() == at::kBFloat16 && wb.dim() == 2);
  c10::cuda::CUDAGuard guard(x.device());
  NhwcView xv = nhwc_view(x);
  ConvDesc d{static_cast<int>(kernel[0]), static_cast<int>(kernel[1]), static_cast<int>(stride[0]), static_cast<int>(stride[1]),
             static_cast<int>(pad[0]), static_cast<int>(pad[1]), static_cast<int>(groups), static_cast<int>(mode)};
  const int Cout = wb.size(0), Cout_g = Cout / groups, Cg = xv.C / groups;
  at::Tensor y = out.has_value() ? *out : empty_nhwc(xv.N, Cout, OH, OW, x.options());
  NhwcView yv = nhwc_view(y);
  TORCH_CHECK(yv.C == Cout && yv.H == OH && yv.W == OW && yv.N == xv.N, "conv_fprop: bad output tensor");
  auto stream = at::cuda::getCurrentCUDAStream();
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  for (int gidx = 0; gidx < groups; ++gidx) {
    // channel-padded operand (R*S*Cgk columns, Cgk = Cg rounded up to 64): the TMA im2col path zero-fills slots >= Cg
    const int Cgk = (d.mode == 0 && wb.size(1) != static_cast<int64_t>(d.R) * d.S * Cg) ? static_cast<int>(wb.size(1) / (d.R * d.S)) : 0;
    ConvGeom cg = make_geom(x, xv, gidx * Cg, Cg, OH, OW, d, false, Cgk);
    TORCH_CHECK(wb.size(1) == cg.K, "conv_fprop: weight K ", wb.size(1), " != expected ", cg.K);
    const long m_blocks = (cg.M + BLOCK_M - 1) / BLOCK_M;
    int bn = pick_conv_bn(Cout_g, m_blocks, sms);
    if (!(g_conv_cluster == 1 && im2col_ok(cg))) bn = std::min(bn, kGatherMaxBN);
    const long n_blocks = (Cout_g + bn - 1) / bn;
    int grid = 0;
    const int cl = pick_cluster(m_blocks, m_blocks * n_blocks, sms, &grid);
    TmapSet tm;
    const __nv_bfloat16* wptr = reinterpret_cast<const __nv_bfloat16*>(wb.data_ptr()) + static_cast<long>(gidx) * Cout_g * cg.K;
    encode_tmap_2d(&tm.b[0], wptr, cg.K, Cout_g, cg.K, BLOCK_K, bn / cl);     // each CTA multicasts 1/cl of the rows
    tm.a[0] = tm.b[0];
    GemmParams p{};
    p.max_stages = g_max_stages;
    p.no_bulk_epi = g_no_bulk_epi;
    p.cluster = cl;
    p.M = static_cast<int>(cg.M);
    p.N = Cout_g;
    p.kb_per_src = (cg.K + BLOCK_K - 1) / BLOCK_K;
    p.num_src = 1;
    p.split_k = 1;
    p.c_bf16 = reinterpret_cast<__nv_bfloat16*>(y.data_ptr()) + gidx * Cout_g;
    p.ldc = yv.pitch;
    p.bias = bias.has_value() ? bias->data_ptr<float>() + gidx * Cout_g : nullptr;
    p.relu = relu;
    p.relu_slope = static_cast<float>(slope);
    p.alpha = 1.f;
    if (cl == 1 && try_im2col_map(&tm.a[0], cg, BLOCK_M)) {
      int mbn = bn, mgrid = grid;
      const int mc = plan_im2col_mcast(Cout_g, m_blocks, sms, &mbn, &mgrid);
      if (mc > 1) {
        // cluster multicast of the im2col operand: every CTA fetches 128 / mc pixel rows of the shared A tile
        TORCH_CHECK(try_im2col_map(&tm.a[0], cg, BLOCK_M / mc), "im2col map");
        encode_tmap_2d(&tm.b[0], wptr, cg.K, Cout_g, cg.K, BLOCK_K, mbn);
        p.cluster = mc;
        launch_im2col_a<1>(mbn, tm, p, cg, mgrid, stream);
        continue;
      }
      if (g_conv_pair && pair_cta_enabled() && m_blocks >= 2 && bn >= 64) {
        // CTA pairs: two pixel blocks share every weight tile; each CTA fetches BN/2 weight rows for both
        encode_tmap_2d(&tm.b[0], wptr, cg.K, Cout_g, cg.K, BLOCK_K, bn / 2);
        launch_im2col_a<2>(bn, tm, p, cg, pair_grid(m_blocks, n_blocks, 1, sms), stream);
        continue;
      }
      launch_im2col_a<1>(bn, tm, p, cg, grid, stream);
      continue;
    }
    TORCH_CHECK(cg.Cgk == cg.Cg, "conv_fprop: channel-padded operand needs the TMA im2col path");
    if (bn == 64) launch_conv<64, false, false, EPI_BF16, GATHER_A>(tm, p, cg, grid, stream);
    else launch_conv<128, false, false, EPI_BF16, GATHER_A>(tm, p, cg, grid, stream);
  }
  return y;
}

// y[N, Cout, OH, OW] (NHWC bf16) = act(conv(x8, w8) * s_x * s_w[co] + bias[co]) with e4m3 operands (fp8_quant.cu):
//   x8 : e4m3 NHWC, pixel pitch a multiple of 16 bytes;  w8 : [Cout, R*S*Cgk] e4m3, Cgk = per-tap slots (multiple of 128,
//   slots >= Cg zero);  s_x : one float;  s_w : [Cout] floats.  `out` may be a channel slice of a concat slab.
// TMA im2col path only: single CTAs, or CTA pairs sharing the weight tile (the default for >= 2 pixel blocks).
at::Tensor conv_fprop_fp8(const at::Tensor& x8, const at::Tensor& w8, const at::Tensor& s_x, const at::Tensor& s_w,
                          const c10::optional<at::Tensor>& bias, at::IntArrayRef kernel, at::IntArrayRef stride,
                          at::IntArrayRef pad, int64_t groups, int64_t OH, int64_t OW, bool relu, double slope,
                          c10::optional<at::Tensor> out) {
  TORCH_CHECK(x8.is_cuda() && x8.scalar_type() == at::kFloat8_e4m3fn && w8.scalar_type() == at::kFloat8_e4m3fn &&
              w8.dim() == 2 && w8.is_contiguous(), "conv_fprop_fp8: e4m3 NHWC x8 and contiguous [Cout, K] e4m3 w8 expected");
  TORCH_CHECK(s_x.scalar_type() == at::kFloat && s_x.numel() == 1 && s_x.is_cuda(), "conv_fprop_fp8: s_x must be one float");
  TORCH_CHECK(s_w.scalar_type() == at::kFloat && s_w.is_contiguous() && s_w.numel() == w8.size(0) && s_w.is_cuda(),
              "conv_fprop_fp8: s_w must hold one float per output channel");
  TORCH_CHECK(!bias.has_value() || (bias->scalar_type() == at::kFloat && bias->is_contiguous() && bias->numel() == w8.size(0)),
              "conv_fprop_fp8: bias must be fp32 [Cout]");
  TORCH_CHECK(g_conv_cluster == 1, "conv_fprop_fp8: the gather multicast-cluster schedule (set_conv_cluster) is bf16-only");
  TORCH_CHECK(g_conv_mcast == 1, "conv_fprop_fp8: the im2col multicast-cluster schedule (set_conv_mcast) is bf16-only");
  NhwcView xv = nhwc_view(x8);
  const int R = static_cast<int>(kernel[0]), S = static_cast<int>(kernel[1]);
  TORCH_CHECK(groups >= 1 && w8.size(0) % groups == 0 && xv.C % groups == 0, "conv_fprop_fp8: channel counts");
  const int Cout = w8.size(0), Cout_g = Cout / groups, Cg = xv.C / groups;
  TORCH_CHECK(Cg % 8 == 0 && R >= 1 && S >= 1, "conv_fprop_fp8: channels per group must be a multiple of 8");
  TORCH_CHECK(w8.size(1) % (R * S) == 0, "conv_fprop_fp8: weight columns must be R*S*Cgk");
  const int Cgk = static_cast<int>(w8.size(1) / (R * S));
  TORCH_CHECK(Cgk % 128 == 0 && Cgk >= Cg, "conv_fprop_fp8: per-tap slots Cgk must be a multiple of 128 and >= Cg");
  TORCH_CHECK(R <= 15 && S <= 15, "conv_fprop_fp8: kernel extents up to 15 are supported");
  NhwcView yv{};
  if (out.has_value()) {
    yv = nhwc_view(*out);
    TORCH_CHECK(out->scalar_type() == at::kBFloat16 && yv.C == Cout && yv.H == OH && yv.W == OW && yv.N == xv.N,
                "conv_fprop_fp8: bad output tensor");
  }
  // every group's geometry is validated before any device work
  std::vector<ConvGeom> geoms(groups);
  for (int gidx = 0; gidx < groups; ++gidx) {
    ConvGeom& cg = geoms[gidx];
    cg.x = reinterpret_cast<const __nv_bfloat16*>(reinterpret_cast<const uint8_t*>(x8.data_ptr()) + gidx * Cg);
    cg.N = xv.N; cg.H = xv.H; cg.W = xv.W;
    cg.pitch = xv.pitch;
    cg.Cg = Cg;
    cg.Cgk = Cgk;
    cg.OH = static_cast<int>(OH); cg.OW = static_cast<int>(OW);
    cg.R = R; cg.S = S;
    cg.sh = static_cast<int>(stride[0]); cg.sw = static_cast<int>(stride[1]);
    cg.off_h = -static_cast<int>(pad[0]); cg.off_w = -static_cast<int>(pad[1]);
    cg.dr = 1;
    cg.mode = 0;
    cg.K = R * S * Cgk;
    cg.M = static_cast<long>(xv.N) * OH * OW;
    TORCH_CHECK(cg.M < (1L << 31), "conv_fprop_fp8: N*OH*OW must fit in 31 bits");
    TORCH_CHECK(im2col_ok(cg, 1), "conv_fprop_fp8: geometry outside the im2col-TMA limits (stride <= 8, corner offsets in "
                "[-128, 127], 16-byte aligned group slices and pixels)");
    cg.div_ow = make_fastdiv(static_cast<uint32_t>(OW));
    cg.div_ohow = make_fastdiv(static_cast<uint32_t>(OH * OW));
    cg.div_cg = make_fastdiv(Cgk);
    cg.div_s = make_fastdiv(S);
    cg.scale_x = s_x.data_ptr<float>();
    cg.scale_w = s_w.data_ptr<float>() + gidx * Cout_g;
  }
  c10::cuda::CUDAGuard guard(x8.device());
  at::Tensor y = out.has_value() ? *out : empty_nhwc(xv.N, Cout, OH, OW, x8.options().dtype(at::kBFloat16));
  if (!out.has_value()) yv = nhwc_view(y);
  auto stream = at::cuda::getCurrentCUDAStream();
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  for (int gidx = 0; gidx < groups; ++gidx) {
    const ConvGeom& cg = geoms[gidx];
    TmapSet tm;
    TORCH_CHECK(try_im2col_map(&tm.a[0], cg, BLOCK_M, 1), "conv_fprop_fp8: im2col map");
    const long m_blocks = (cg.M + BLOCK_M - 1) / BLOCK_M;
    const int bn = std::min(pick_conv_bn(Cout_g, m_blocks, sms), 128);
    const long n_blocks = (Cout_g + bn - 1) / bn;
    const uint8_t* wptr = reinterpret_cast<const uint8_t*>(w8.data_ptr()) + static_cast<long>(gidx) * Cout_g * cg.K;
    GemmParams p{};
    p.max_stages = g_max_stages;
    p.no_bulk_epi = g_no_bulk_epi;
    p.cluster = 1;
    p.M = static_cast<int>(cg.M);
    p.N = Cout_g;
    p.kb_per_src = cg.K / 128;
    p.num_src = 1;
    p.split_k = 1;
    p.c_bf16 = reinterpret_cast<__nv_bfloat16*>(y.data_ptr()) + gidx * Cout_g;
    p.ldc = yv.pitch;
    p.bias = bias.has_value() ? bias->data_ptr<float>() + gidx * Cout_g : nullptr;
    p.relu = relu;
    p.relu_slope = static_cast<float>(slope);
    p.alpha = 1.f;
    const bool pair = g_conv_pair && pair_cta_enabled() && m_blocks >= 2;
    encode_tmap_2d(&tm.b[0], wptr, cg.K, Cout_g, cg.K, 128, pair ? bn / 2 : bn, CU_TENSOR_MAP_DATA_TYPE_UINT8);
    if (pair) {
      const int grid = pair_grid(m_blocks, n_blocks, 1, sms);
      if (bn == 64) launch_conv<64, false, false, EPI_BF16, IM2COL_A, 2, __nv_fp8_e4m3>(tm, p, cg, grid, stream);
      else launch_conv<128, false, false, EPI_BF16, IM2COL_A, 2, __nv_fp8_e4m3>(tm, p, cg, grid, stream);
    } else {
      const int grid = static_cast<int>(std::max<long>(1, std::min<long>(m_blocks * n_blocks, sms)));
      if (bn == 64) launch_conv<64, false, false, EPI_BF16, IM2COL_A, 1, __nv_fp8_e4m3>(tm, p, cg, grid, stream);
      else launch_conv<128, false, false, EPI_BF16, IM2COL_A, 1, __nv_fp8_e4m3>(tm, p, cg, grid, stream);
    }
  }
  return y;
}

// dx[N, Cin, H, W] = conv_transpose(dy, w) for stride-1 convolutions; wt: [groups*Cg, R*S*Cout_g] bf16
// (per group: rows = input channel, K = (r, s, co)).  Optional mask = forward output of the producer layer
// (fused ReLU backward: dx is zeroed / scaled by slope where mask <= 0).
at::Tensor conv_dgrad(const at::Tensor& dy, const at::Tensor& wt, at::IntArrayRef kernel, at::IntArrayRef pad, int64_t groups,
                      int64_t H, int64_t W, const c10::optional<at::Tensor>& mask, double slope) {
  TORCH_CHECK(dy.is_cuda() && dy.scalar_type() == at::kBFloat16 && wt.scalar_type() == at::kBFloat16 && wt.dim() == 2);
  c10::cuda::CUDAGuard guard(dy.device());
  NhwcView dv = nhwc_view(dy);
  ConvDesc d{static_cast<int>(kernel[0]), static_cast<int>(kernel[1]), 1, 1, static_cast<int>(pad[0]), static_cast<int>(pad[1]),
             static_cast<int>(groups), 0};
  const int Cin = wt.size(0), Cg = Cin / groups, Cout_g = dv.C / groups;
  at::Tensor dx = empty_nhwc(dv.N, Cin, H, W, dy.options());
  NhwcView xv = nhwc_view(dx);
  auto stream = at::cuda::getCurrentCUDAStream();
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  long mask_pitch = 0;
  if (mask.has_value()) {
    NhwcView mv = nhwc_view(*mask);
    TORCH_CHECK(mv.C == Cin && mv.H == H && mv.W == W && mv.pitch == xv.pitch, "conv_dgrad: mask must match dx layout");
    mask_pitch = mv.pitch;
  }
  for (int gidx = 0; gidx < groups; ++gidx) {
    const int Cok = wt.size(1) != static_cast<int64_t>(d.R) * d.S * Cout_g ? static_cast<int>(wt.size(1) / (d.R * d.S)) : 0;
    ConvGeom cg = make_geom(dy, dv, gidx * Cout_g, Cout_g, H, W, d, true, Cok);
    TORCH_CHECK(wt.size(1) == cg.K, "conv_dgrad: packed weight K mismatch");
    const long m_blocks = (cg.M + BLOCK_M - 1) / BLOCK_M;
    int bn = pick_conv_bn(Cg, m_blocks, sms);
    if (!(g_conv_cluster == 1 && im2col_ok(cg))) bn = std::min(bn, kGatherMaxBN);
    const long n_blocks = (Cg + bn - 1) / bn;
    int grid = 0;
    const int cl = pick_cluster(m_blocks, m_blocks * n_blocks, sms, &grid);
    TmapSet tm;
    const __nv_bfloat16* wptr = reinterpret_cast<const __nv_bfloat16*>(wt.data_ptr()) + static_cast<long>(gidx) * Cg * cg.K;
    encode_tmap_2d(&tm.b[0], wptr, cg.K, Cg, cg.K, BLOCK_K, bn / cl);
    tm.a[0] = tm.b[0];
    GemmParams p{};
    p.max_stages = g_max_stages;
    p.no_bulk_epi = g_no_bulk_epi;
    p.cluster = cl;
    p.M = static_cast<int>(cg.M);
    p.N = Cg;
    p.kb_per_src = (cg.K + BLOCK_K - 1) / BLOCK_K;
    p.num_src = 1;
    p.split_k = 1;
    p.c_bf16 = reinterpret_cast<__nv_bfloat16*>(dx.data_ptr()) + gidx * Cg;
    p.ldc = xv.pitch;
    p.mask = mask.has_value() ? reinterpret_cast<const __nv_bfloat16*>(mask->data_ptr()) + gidx * Cg : nullptr;
    p.relu_slope = static_cast<float>(slope);
    p.alpha = 1.f;
    (void)mask_pitch;
    if (cl == 1 && try_im2col_map(&tm.a[0], cg, BLOCK_M)) {
      int mbn = bn, mgrid = grid;
      const int mc = plan_im2col_mcast(Cg, m_blocks, sms, &mbn, &mgrid);
      if (mc > 1) {
        TORCH_CHECK(try_im2col_map(&tm.a[0], cg, BLOCK_M / mc), "im2col map");
        encode_tmap_2d(&tm.b[0], wptr, cg.K, Cg, cg.K, BLOCK_K, mbn);
        p.cluster = mc;
        launch_im2col_a<1>(mbn, tm, p, cg, mgrid, stream);
        continue;
      }
      if (g_conv_pair && pair_cta_enabled() && m_blocks >= 2 && bn >= 64) {
        encode_tmap_2d(&tm.b[0], wptr, cg.K, Cg, cg.K, BLOCK_K, bn / 2);
        launch_im2col_a<2>(bn, tm, p, cg, pair_grid(m_blocks, n_blocks, 1, sms), stream);
        continue;
      }
      launch_im2col_a<1>(bn, tm, p, cg, grid, stream);
      continue;
    }
    TORCH_CHECK(cg.Cgk == cg.Cg, "conv_dgrad: channel-padded operand needs the TMA im2col path");
    if (bn == 64) launch_conv<64, false, false, EPI_BF16, GATHER_A>(tm, p, cg, grid, stream);
    else launch_conv<128, false, false, EPI_BF16, GATHER_A>(tm, p, cg, grid, stream);
  }
  return dx;
}

// dx[N, Cin, H, W] (NHWC bf16, dense) = conv_transpose(dy8, wt8) * s_dy * s_wt[ci] for stride-1 convolutions, with e5m2 dY
// and e4m3 weights (fp8_quant.cu):
//   dy8 : e5m2 NHWC [N, Cout, OH, OW], pixel pitch a multiple of 16 bytes;  wt8 : [groups*Cg, R*S*Cok] e4m3 in
//   conv_pack_dgrad's order (per group: rows = input channel, K = (r, s, co)), Cok a multiple of 128, slots >= Cout_g zero;
//   s_dy : one float;  s_wt : [Cin] floats.  Optional mask = forward output of the producer layer, laid out like dx
//   (fused ReLU backward, as in conv_dgrad).  TMA im2col path only: single CTAs, or CTA pairs sharing the weight tile.
at::Tensor conv_dgrad_fp8(const at::Tensor& dy8, const at::Tensor& wt8, const at::Tensor& s_dy, const at::Tensor& s_wt,
                          at::IntArrayRef kernel, at::IntArrayRef pad, int64_t groups, int64_t H, int64_t W,
                          const c10::optional<at::Tensor>& mask, double slope) {
  TORCH_CHECK(dy8.is_cuda() && dy8.scalar_type() == at::kFloat8_e5m2 && wt8.is_cuda() &&
              wt8.scalar_type() == at::kFloat8_e4m3fn && wt8.dim() == 2 && wt8.is_contiguous(),
              "conv_dgrad_fp8: e5m2 NHWC dy8 and contiguous [Cin, K] e4m3 wt8 expected");
  TORCH_CHECK(s_dy.is_cuda() && s_dy.scalar_type() == at::kFloat && s_dy.numel() == 1, "conv_dgrad_fp8: s_dy must be one float");
  TORCH_CHECK(s_wt.is_cuda() && s_wt.scalar_type() == at::kFloat && s_wt.is_contiguous() && s_wt.numel() == wt8.size(0),
              "conv_dgrad_fp8: s_wt must hold one float per input channel");
  TORCH_CHECK(kernel.size() == 2 && pad.size() == 2, "conv_dgrad_fp8: kernel and pad take two values");
  TORCH_CHECK(g_conv_cluster == 1, "conv_dgrad_fp8: the gather multicast-cluster schedule (set_conv_cluster) is bf16-only");
  TORCH_CHECK(g_conv_mcast == 1, "conv_dgrad_fp8: the im2col multicast-cluster schedule (set_conv_mcast) is bf16-only");
  NhwcView dv = nhwc_view(dy8);
  const int R = static_cast<int>(kernel[0]), S = static_cast<int>(kernel[1]);
  const int ph = static_cast<int>(pad[0]), pw = static_cast<int>(pad[1]);
  TORCH_CHECK(R >= 1 && S >= 1 && R <= 15 && S <= 15, "conv_dgrad_fp8: kernel extents from 1 to 15 are supported");
  TORCH_CHECK(ph >= 0 && pw >= 0 && H >= 1 && W >= 1, "conv_dgrad_fp8: bad padding or input extent");
  TORCH_CHECK(dv.H == H + 2 * ph - R + 1 && dv.W == W + 2 * pw - S + 1,
              "conv_dgrad_fp8: dY extent is not that of a stride-1 convolution over H x W");
  TORCH_CHECK(groups >= 1 && wt8.size(0) % groups == 0 && dv.C % groups == 0, "conv_dgrad_fp8: channel counts");
  const int Cin = static_cast<int>(wt8.size(0)), Cg = Cin / static_cast<int>(groups), Cout_g = dv.C / static_cast<int>(groups);
  TORCH_CHECK(Cg % 8 == 0 && Cout_g % 8 == 0, "conv_dgrad_fp8: channels per group must be multiples of 8");
  TORCH_CHECK(wt8.size(1) % (R * S) == 0, "conv_dgrad_fp8: weight columns must be R*S*Cok");
  const int Cok = static_cast<int>(wt8.size(1) / (R * S));
  TORCH_CHECK(Cok % 128 == 0 && Cok >= Cout_g, "conv_dgrad_fp8: per-tap slots Cok must be a multiple of 128 and >= Cout_g");
  if (mask.has_value()) {
    TORCH_CHECK(mask->is_cuda() && mask->scalar_type() == at::kBFloat16, "conv_dgrad_fp8: bf16 mask expected");
    NhwcView mv = nhwc_view(*mask);
    TORCH_CHECK(mv.N == dv.N && mv.C == Cin && mv.H == H && mv.W == W && mv.pitch == Cin,
                "conv_dgrad_fp8: mask must match dx layout");
  }
  // every group's geometry is validated before any device work
  std::vector<ConvGeom> geoms(groups);
  for (int gidx = 0; gidx < groups; ++gidx) {
    ConvGeom& cg = geoms[gidx];
    cg.x = reinterpret_cast<const __nv_bfloat16*>(reinterpret_cast<const uint8_t*>(dy8.data_ptr()) + gidx * Cout_g);
    cg.N = dv.N; cg.H = dv.H; cg.W = dv.W;
    cg.pitch = dv.pitch;
    cg.Cg = Cout_g;
    cg.Cgk = Cok;
    cg.OH = static_cast<int>(H); cg.OW = static_cast<int>(W);
    cg.R = R; cg.S = S;
    cg.sh = 1; cg.sw = 1;
    cg.off_h = ph; cg.off_w = pw;
    cg.dr = -1;                                 // mirrored tap walk: the transposed convolution
    cg.mode = 0;
    cg.K = R * S * Cok;
    cg.M = static_cast<long>(dv.N) * H * W;
    TORCH_CHECK(cg.M < (1L << 31), "conv_dgrad_fp8: N*H*W must fit in 31 bits");
    TORCH_CHECK(im2col_ok(cg, 1), "conv_dgrad_fp8: geometry outside the im2col-TMA limits (mirrored corner offsets in "
                "[-128, 127], 16-byte aligned group slices and pixels)");
    cg.div_ow = make_fastdiv(static_cast<uint32_t>(W));
    cg.div_ohow = make_fastdiv(static_cast<uint32_t>(H * W));
    cg.div_cg = make_fastdiv(Cok);
    cg.div_s = make_fastdiv(S);
    cg.scale_x = s_dy.data_ptr<float>();
    cg.scale_w = s_wt.data_ptr<float>() + gidx * Cg;
  }
  c10::cuda::CUDAGuard guard(dy8.device());
  at::Tensor dx = empty_nhwc(dv.N, Cin, H, W, dy8.options().dtype(at::kBFloat16));
  auto stream = at::cuda::getCurrentCUDAStream();
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  for (int gidx = 0; gidx < groups; ++gidx) {
    const ConvGeom& cg = geoms[gidx];
    TmapSet tm;
    TORCH_CHECK(try_im2col_map(&tm.a[0], cg, BLOCK_M, 1), "conv_dgrad_fp8: im2col map");
    const long m_blocks = (cg.M + BLOCK_M - 1) / BLOCK_M;
    const int bn = std::min(pick_conv_bn(Cg, m_blocks, sms), 128);
    const long n_blocks = (Cg + bn - 1) / bn;
    const uint8_t* wptr = reinterpret_cast<const uint8_t*>(wt8.data_ptr()) + static_cast<long>(gidx) * Cg * cg.K;
    GemmParams p{};
    p.max_stages = g_max_stages;
    p.no_bulk_epi = g_no_bulk_epi;
    p.cluster = 1;
    p.M = static_cast<int>(cg.M);
    p.N = Cg;
    p.kb_per_src = cg.K / 128;
    p.num_src = 1;
    p.split_k = 1;
    p.c_bf16 = reinterpret_cast<__nv_bfloat16*>(dx.data_ptr()) + gidx * Cg;
    p.ldc = Cin;
    p.mask = mask.has_value() ? reinterpret_cast<const __nv_bfloat16*>(mask->data_ptr()) + gidx * Cg : nullptr;
    p.relu_slope = static_cast<float>(slope);
    p.alpha = 1.f;
    const bool pair = g_conv_pair && pair_cta_enabled() && m_blocks >= 2;
    encode_tmap_2d(&tm.b[0], wptr, cg.K, Cg, cg.K, 128, pair ? bn / 2 : bn, CU_TENSOR_MAP_DATA_TYPE_UINT8);
    if (pair) {
      const int grid = pair_grid(m_blocks, n_blocks, 1, sms);
      if (bn == 64) launch_conv<64, false, false, EPI_BF16, IM2COL_A, 2, __nv_fp8_e5m2>(tm, p, cg, grid, stream);
      else launch_conv<128, false, false, EPI_BF16, IM2COL_A, 2, __nv_fp8_e5m2>(tm, p, cg, grid, stream);
    } else {
      const int grid = static_cast<int>(std::max<long>(1, std::min<long>(m_blocks * n_blocks, sms)));
      if (bn == 64) launch_conv<64, false, false, EPI_BF16, IM2COL_A, 1, __nv_fp8_e5m2>(tm, p, cg, grid, stream);
      else launch_conv<128, false, false, EPI_BF16, IM2COL_A, 1, __nv_fp8_e5m2>(tm, p, cg, grid, stream);
    }
  }
  return dx;
}

// Data gradient of a stride-1 convolution read straight from the FPROP weight operand wb [Cout][R][S][Cg] (bf16): no
// packed [Cin][R][S][Cout] copy, no pack kernel per step.  K = (tap, co) with Cok = round64(Cout_g) slots per tap; the
// surplus slots are zero on both sides (im2col channel overrun on dY, row overrun of the 3-D weight map).  Any Cout_g,
// C_g that are multiples of 8 take this (TMA) path; returns false if the geometry does not fit the im2col descriptor.
bool conv_dgrad_w_impl(const at::Tensor& dy, const at::Tensor& wb, at::IntArrayRef kernel, at::IntArrayRef pad, int64_t groups,
                       int64_t H, int64_t W, const c10::optional<at::Tensor>& mask, double slope, at::Tensor& dx) {
  NhwcView dv = nhwc_view(dy);
  ConvDesc d{static_cast<int>(kernel[0]), static_cast<int>(kernel[1]), 1, 1, static_cast<int>(pad[0]), static_cast<int>(pad[1]),
             static_cast<int>(groups), 0};
  const int Cout = wb.size(0), Cout_g = Cout / groups, RS = d.R * d.S;
  const int Cg = static_cast<int>(wb.size(1) / RS), Cin = Cg * groups;
  if (Cout_g % 8 != 0 || Cg % 8 != 0 || dv.C != Cout) return false;
  const int Cok = (Cout_g + 63) / 64 * 64;
  NhwcView xv = nhwc_view(dx);
  auto stream = at::cuda::getCurrentCUDAStream();
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  for (int gidx = 0; gidx < groups; ++gidx) {
    ConvGeom cg = make_geom(dy, dv, gidx * Cout_g, Cout_g, H, W, d, true, Cok);
    TmapSet tm;
    if (!try_im2col_map(&tm.a[0], cg, BLOCK_M)) return false;
    const long m_blocks = (cg.M + BLOCK_M - 1) / BLOCK_M;
    int bn = pick_conv_bn(Cg, m_blocks, sms);
    if (bn == 192) bn = 256;                       // MN-major B: whole 64-column chunks per CTA pair half
    const long n_blocks = (Cg + bn - 1) / bn;
    const __nv_bfloat16* wptr = reinterpret_cast<const __nv_bfloat16*>(wb.data_ptr()) + static_cast<long>(gidx) * Cout_g * RS * Cg;
    encode_tmap_bf16_3d(&tm.b[0], wptr, Cg, Cout_g, RS, static_cast<int64_t>(RS) * Cg, Cg, 64, 64, 1);
    GemmParams p{};
    p.max_stages = g_max_stages;
    p.no_bulk_epi = g_no_bulk_epi;
    p.cluster = 1;
    p.M = static_cast<int>(cg.M);
    p.N = Cg;
    p.kb_per_src = (cg.K + BLOCK_K - 1) / BLOCK_K;
    p.num_src = 1;
    p.split_k = 1;
    p.c_bf16 = reinterpret_cast<__nv_bfloat16*>(dx.data_ptr()) + gidx * Cg;
    p.ldc = xv.pitch;
    p.mask = mask.has_value() ? reinterpret_cast<const __nv_bfloat16*>(mask->data_ptr()) + gidx * Cg : nullptr;
    p.relu_slope = static_cast<float>(slope);
    p.alpha = 1.f;
    const bool pair = g_conv_pair && pair_cta_enabled() && m_blocks >= 2 && bn >= 128;
    if (pair) {
      const int pgrid = pair_grid(m_blocks, n_blocks, 1, sms);
      if (bn == 128) launch_conv<128, false, true, EPI_BF16, IM2COL_A, 2>(tm, p, cg, pgrid, stream);
      else launch_conv<256, false, true, EPI_BF16, IM2COL_A, 2>(tm, p, cg, pgrid, stream);
    } else {
      const int grid = static_cast<int>(std::max<long>(1, std::min<long>(m_blocks * n_blocks, sms)));
      if (bn == 64) launch_conv<64, false, true, EPI_BF16, IM2COL_A, 1>(tm, p, cg, grid, stream);
      else if (bn == 128) launch_conv<128, false, true, EPI_BF16, IM2COL_A, 1>(tm, p, cg, grid, stream);
      else launch_conv<256, false, true, EPI_BF16, IM2COL_A, 1>(tm, p, cg, grid, stream);
    }
  }
  return true;
}

at::Tensor conv_dgrad_w(const at::Tensor& dy, const at::Tensor& wb, at::IntArrayRef kernel, at::IntArrayRef pad, int64_t groups,
                        int64_t H, int64_t W, const c10::optional<at::Tensor>& mask, double slope) {
  TORCH_CHECK(dy.is_cuda() && dy.scalar_type() == at::kBFloat16 && wb.scalar_type() == at::kBFloat16 && wb.dim() == 2 &&
              wb.is_contiguous(), "conv_dgrad_w: bf16 dY and the contiguous fprop weight operand expected");
  c10::cuda::CUDAGuard guard(dy.device());
  NhwcView dv = nhwc_view(dy);
  const int RS = static_cast<int>(kernel[0] * kernel[1]);
  const int64_t Cin = wb.size(1) / RS * groups;
  at::Tensor dx = empty_nhwc(dv.N, Cin, H, W, dy.options());
  if (mask.has_value()) {
    NhwcView mv = nhwc_view(*mask), xv = nhwc_view(dx);
    TORCH_CHECK(mv.C == Cin && mv.H == H && mv.W == W && mv.pitch == xv.pitch, "conv_dgrad_w: mask must match dx layout");
  }
  TORCH_CHECK(conv_dgrad_w_impl(dy, wb, kernel, pad, groups, H, W, mask, slope, dx),
              "conv_dgrad_w: geometry outside the im2col-TMA limits (use conv_dgrad with the packed operand)");
  return dx;
}

// dw[Cout, Kw] fp32 += alpha * dYᵀ · im2col(x)   (split-K over the N*OH*OW reduction, partials summed in a fixed order;
// dw pre-zeroed unless accumulating into an existing gradient).
void conv_wgrad(const at::Tensor& x, const at::Tensor& dy, at::Tensor dw, at::IntArrayRef kernel, at::IntArrayRef stride,
                at::IntArrayRef pad, int64_t groups, int64_t mode, double alpha, int64_t cgk) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && dy.scalar_type() == at::kBFloat16);
  TORCH_CHECK(dw.scalar_type() == at::kFloat && dw.dim() == 2 && dw.is_contiguous());
  c10::cuda::CUDAGuard guard(x.device());
  NhwcView xv = nhwc_view(x), dv = nhwc_view(dy);
  ConvDesc d{static_cast<int>(kernel[0]), static_cast<int>(kernel[1]), static_cast<int>(stride[0]), static_cast<int>(stride[1]),
             static_cast<int>(pad[0]), static_cast<int>(pad[1]), static_cast<int>(groups), static_cast<int>(mode)};
  const int Cout = dv.C, Cout_g = Cout / groups, Cg = xv.C / groups;
  TORCH_CHECK(dv.pitch % 8 == 0 && Cout_g % 8 == 0, "conv_wgrad: output channels must be multiples of 8");
  auto stream = at::cuda::getCurrentCUDAStream();
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  for (int gidx = 0; gidx < groups; ++gidx) {
    // cgk > Cg: the reduction's k-columns are channel-padded per tap (im2col TMA); dw itself stays unpadded and the
    // epilogue maps column tap*cgk + c -> tap*Cg + c, dropping the pad
    ConvGeom cg = make_geom(x, xv, gidx * Cg, Cg, dv.H, dv.W, d, false, (mode == 0 && cgk > Cg) ? static_cast<int>(cgk) : 0);
    const int64_t k_real = mode == 1 ? cg.K : static_cast<int64_t>(d.R) * d.S * Cg;
    TORCH_CHECK(dw.size(0) == Cout && dw.size(1) == k_real, "conv_wgrad: dw shape mismatch");
    int bn = cg.K > 128 ? 256 : (cg.K > 64 ? 128 : 64);
    if (bn == 256 && ((cg.K + 191) / 192 * 192) * 100 < ((cg.K + 255) / 256 * 256) * 85) bn = 192;   // e.g. K = 576
    if (!(g_conv_cluster == 1 && im2col_ok(cg))) bn = std::min(bn, kGatherMaxBN);
    TmapSet tm;
    // A = dYᵀ: MN-major, inner = Cout_g channels of this group, outer = M pixels, pitch = dy pixel pitch
    const __nv_bfloat16* dyp = reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr()) + gidx * Cout_g;
    GemmParams p{};
    p.max_stages = g_max_stages;
    p.no_bulk_epi = g_no_bulk_epi;
    p.M = Cout_g;
    p.N = cg.K;
    p.kb_per_src = static_cast<int>((cg.M + BLOCK_K - 1) / BLOCK_K);
    p.num_src = 1;
    const long n_blocks = (cg.K + bn - 1) / bn;
    const long tiles = ((Cout_g + BLOCK_M - 1) / BLOCK_M) * n_blocks;
    long split = std::max<long>(1, (2L * sms + tiles - 1) / tiles);
    split = std::min<long>(split, std::max<long>(1, p.kb_per_src / 8));
    p.split_k = static_cast<int>(split);
    int grid = 0;
    const int cl = pick_cluster(n_blocks, tiles * split, sms, &grid);
    p.cluster = cl;
    encode_tmap_2d(&tm.a[0], dyp, Cout_g, cg.M, dv.pitch, 64, BLOCK_K / cl);      // each CTA multicasts 1/cl of the k-rows
    tm.b[0] = tm.a[0];
    p.c_f32 = dw.data_ptr<float>() + static_cast<long>(gidx) * Cout_g * k_real;
    p.ldc = k_real;
    if (cg.Cgk != cg.Cg) { p.col_cg = cg.Cg; p.col_cgk = cg.Cgk; }
    p.atomic = 1;
    p.alpha = static_cast<float>(alpha);
    // Split reduction: each split stores its partial to its own workspace slice (plain stores) and the slices are added
    // onto dw in split order afterwards, so the gradient does not depend on which CTA finishes first.  One split adds
    // onto dw directly (one add per element).
    float* const dwg = p.c_f32;
    at::Tensor ws;
    if (split > 1) {
      ws = at::empty({split, Cout_g, k_real}, dw.options());
      p.c_f32 = ws.data_ptr<float>();
      p.split_stride = static_cast<long>(Cout_g) * k_real;
      p.atomic = 0;
    }
    [&] {
      if (cl == 1 && try_im2col_map(&tm.b[0], cg, BLOCK_K)) {
        const long m_blocks = (Cout_g + BLOCK_M - 1) / BLOCK_M;
        if (g_conv_mcast > 1 && m_blocks >= 2 && bn >= 128) {
          // cluster along Cout: its CTAs need the same im2col B tile (bn / 64 boxes of 64 pixels x 64 channels per k-block)
          // — each fetches every C-th box and multicasts it
          const int mc = (m_blocks % 3 == 0 && bn >= 192) ? 3 : 2;
          const long ctiles = ((m_blocks + mc - 1) / mc) * n_blocks * split;
          p.cluster = mc;
          const int mgrid = static_cast<int>(std::max<long>(1, std::min<long>(ctiles, sms / mc))) * mc;
          switch (bn) {
            case 128: launch_conv<128, true, true, EPI_F32, IM2COL_B>(tm, p, cg, mgrid, stream); break;
            case 192: launch_conv<192, true, true, EPI_F32, IM2COL_B>(tm, p, cg, mgrid, stream); break;
            default: launch_conv<256, true, true, EPI_F32, IM2COL_B>(tm, p, cg, mgrid, stream); break;
          }
          return;
        }
        if (g_conv_pair && pair_cta_enabled() && m_blocks >= 2 && m_blocks % 2 == 0 && (bn == 128 || bn == 256)) {
          // CTA pairs along Cout (even block counts only: a phantom block would waste a third of conv3's MMA work)
          const int pgrid = pair_grid(m_blocks, n_blocks, split, sms);
          if (bn == 128) launch_conv<128, true, true, EPI_F32, IM2COL_B, 2>(tm, p, cg, pgrid, stream);
          else launch_conv<256, true, true, EPI_F32, IM2COL_B, 2>(tm, p, cg, pgrid, stream);
          return;
        }
        switch (bn) {
          case 64: launch_conv<64, true, true, EPI_F32, IM2COL_B>(tm, p, cg, grid, stream); break;
          case 128: launch_conv<128, true, true, EPI_F32, IM2COL_B>(tm, p, cg, grid, stream); break;
          case 192: launch_conv<192, true, true, EPI_F32, IM2COL_B>(tm, p, cg, grid, stream); break;
          default: launch_conv<256, true, true, EPI_F32, IM2COL_B>(tm, p, cg, grid, stream); break;
        }
        return;
      }
      TORCH_CHECK(cg.Cgk == cg.Cg, "conv_wgrad: channel-padded reduction needs the TMA im2col path");
      if (bn == 64) launch_conv<64, true, true, EPI_F32, GATHER_B>(tm, p, cg, grid, stream);
      else launch_conv<128, true, true, EPI_F32, GATHER_B>(tm, p, cg, grid, stream);
    }();
    if (split > 1) splitk_reduce(ws, static_cast<int>(split), dwg, k_real, Cout_g, static_cast<int>(k_real), true, stream);
  }
}

// Pack the dgrad operand from the fp32 master weights: w [Cout][R][S][Cg] -> wt [groups][Cg][R][S][Cop] bf16, where
// Cop >= Cout_g is the per-tap slot count (Cout_g rounded up to 64 on the channel-padded im2col path; pad = 0).
__global__ void pack_dgrad_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ wt, int Cout, int RS, int Cg,
                                  int groups, int Cop) {
  const int Cout_g = Cout / groups;
  const long total = static_cast<long>(groups) * Cg * RS * Cop;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    // i indexes wt: (((g*Cg + ci)*RS + tap)*Cop + co)
    const int co = static_cast<int>(i % Cop);
    long t = i / Cop;
    const int tap = static_cast<int>(t % RS); t /= RS;
    const int ci = static_cast<int>(t % Cg);
    const int g = static_cast<int>(t / Cg);
    wt[i] = co < Cout_g ? __float2bfloat16(w[((static_cast<long>(g) * Cout_g + co) * RS + tap) * Cg + ci])
                        : __float2bfloat16(0.f);
  }
}

at::Tensor conv_pack_dgrad(const at::Tensor& w, int64_t Cout, int64_t RS, int64_t Cg, int64_t groups,
                           c10::optional<at::Tensor> out, int64_t cop) {
  TORCH_CHECK(w.is_cuda() && w.scalar_type() == at::kFloat && w.numel() == Cout * RS * Cg);
  c10::cuda::CUDAGuard guard(w.device());
  const int64_t Cop = cop > 0 ? cop : Cout / groups;
  TORCH_CHECK(Cop >= Cout / groups);
  at::Tensor wt = out.has_value() ? *out : at::empty({groups * Cg, RS * Cop}, w.options().dtype(at::kBFloat16));
  TORCH_CHECK(wt.numel() == groups * Cg * RS * Cop, "conv_pack_dgrad: output shape mismatch");
  const long total = groups * Cg * RS * Cop;
  pack_dgrad_kernel<<<grid_for(total, 256), 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      w.data_ptr<float>(), reinterpret_cast<__nv_bfloat16*>(wt.data_ptr()), Cout, RS, Cg, groups, static_cast<int>(Cop));
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return wt;
}

// Channel-padded fprop / wgrad operand: wb [Cout][RS][Cg] bf16 -> [Cout][RS][Cgk] bf16 (slots >= Cg zero).
__global__ void pack_pad_channels_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst, long rows,
                                         int Cg, int Cgk) {
  const long total = rows * Cgk;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long r = i / Cgk;
    const int c = static_cast<int>(i - r * Cgk);
    dst[i] = c < Cg ? src[r * Cg + c] : __float2bfloat16(0.f);
  }
}
at::Tensor conv_pack_padded(const at::Tensor& wb, int64_t Cout, int64_t RS, int64_t Cg, int64_t Cgk,
                            c10::optional<at::Tensor> out) {
  TORCH_CHECK(wb.is_cuda() && wb.scalar_type() == at::kBFloat16 && wb.is_contiguous() && wb.numel() == Cout * RS * Cg);
  c10::cuda::CUDAGuard guard(wb.device());
  at::Tensor dst = out.has_value() ? *out : at::empty({Cout, RS * Cgk}, wb.options());
  TORCH_CHECK(dst.numel() == Cout * RS * Cgk && dst.is_contiguous());
  const long rows = Cout * RS;
  pack_pad_channels_kernel<<<grid_for(rows * Cgk, 256), 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const __nv_bfloat16*>(wb.data_ptr()), reinterpret_cast<__nv_bfloat16*>(dst.data_ptr()), rows,
      static_cast<int>(Cg), static_cast<int>(Cgk));
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return dst;
}

}  // namespace psd

namespace psd {
void set_conv_im2col(int64_t on) { g_conv_im2col = on != 0; }
void set_conv_pair(int64_t on) { g_conv_pair = on != 0; }
void set_conv_mcast(int64_t c) {
  TORCH_CHECK(c == 1 || c == 2 || c == 4, "im2col multicast cluster size must be 1, 2 or 4");
  g_conv_mcast = static_cast<int>(c);
}
void set_conv_cluster(int64_t c) {
  TORCH_CHECK(c == 1 || c == 2 || c == 4, "cluster size must be 1, 2 or 4");
  g_conv_cluster = static_cast<int>(c);
}
}  // namespace psd

TORCH_LIBRARY_FRAGMENT(poseidon, m) {
  m.def("set_conv_cluster(int c) -> ()", &psd::set_conv_cluster);
  m.def("set_conv_im2col(int on) -> ()", &psd::set_conv_im2col);
  m.def("set_conv_mcast(int c) -> ()", &psd::set_conv_mcast);
  m.def("set_conv_pair(int on) -> ()", &psd::set_conv_pair);
  m.def("conv_fprop(Tensor x, Tensor wb, Tensor? bias, int[] kernel, int[] stride, int[] pad, int groups, int mode, "
        "int OH, int OW, bool relu, float slope, Tensor? out) -> Tensor", &psd::conv_fprop);
  m.def("conv_fprop_fp8(Tensor x8, Tensor w8, Tensor s_x, Tensor s_w, Tensor? bias, int[] kernel, int[] stride, int[] pad, "
        "int groups, int OH, int OW, bool relu, float slope, Tensor? out) -> Tensor", &psd::conv_fprop_fp8);
  m.def("conv_dgrad_fp8(Tensor dy8, Tensor wt8, Tensor s_dy, Tensor s_wt, int[] kernel, int[] pad, int groups, int H, int W, "
        "Tensor? mask, float slope) -> Tensor", &psd::conv_dgrad_fp8);
  m.def("conv_dgrad(Tensor dy, Tensor wt, int[] kernel, int[] pad, int groups, int H, int W, Tensor? mask, float slope) "
        "-> Tensor", &psd::conv_dgrad);
  m.def("conv_dgrad_w(Tensor dy, Tensor wb, int[] kernel, int[] pad, int groups, int H, int W, Tensor? mask, float slope) "
        "-> Tensor", &psd::conv_dgrad_w);
  m.def("conv_wgrad(Tensor x, Tensor dy, Tensor(a!) dw, int[] kernel, int[] stride, int[] pad, int groups, int mode, "
        "float alpha, int cgk) -> ()", &psd::conv_wgrad);
  m.def("conv_pack_dgrad(Tensor w, int Cout, int RS, int Cg, int groups, Tensor? out, int cop) -> Tensor", &psd::conv_pack_dgrad);
  m.def("conv_pack_padded(Tensor wb, int Cout, int RS, int Cg, int Cgk, Tensor? out) -> Tensor", &psd::conv_pack_padded);
}
