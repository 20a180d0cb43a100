// Host side of the halo-tiled data gradient and forward (halo_conv.cuh): geometry selection, tensor maps, launch, the A/B
// switches.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/library.h>
#include <torch/types.h>

#include <atomic>

#include "../ops/nhwc_common.cuh"
#include "halo_conv.cuh"
#include "wgmma_gemm.cuh"

namespace psd {

void encode_tmap_bf16_3d(CUtensorMap* map, const void* base, int64_t d0, int64_t d1, int64_t d2, int64_t stride1, int64_t stride2,
                         int box0, int box1, int box2);

// set_conv_halo: 0 off (im2col schedule only), 1 where the geometry selects it (default), 2 wherever the kernel can run
// (also tiles that are mostly padding, and problems with fewer than two tiles per SM: for tests)
static int g_conv_halo = 1;
static std::atomic<int64_t> g_halo_launches{0};   // kernel launches so far (conv_halo_launches: which schedule ran)

namespace {

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn encode_fn() {
  static EncodeFn fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    TORCH_CHECK(e == cudaSuccess && qres == cudaDriverEntryPointSuccess && ptr != nullptr,
                "cuTensorMapEncodeTiled not available from the driver");
    fn = reinterpret_cast<EncodeFn>(ptr);
  }
  return fn;
}

// dY of one group as a 4-D tiled map {channel, column, row, image} (strides in elements), boxes of {8 channels, P columns,
// Hb rows, 1 image}, no swizzle: one box is one [pixel][8 channels] slab of the halo.
void encode_halo_map(CUtensorMap* map, const void* base, const NhwcView& v, int channels, int P, int Hb) {
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(channels), static_cast<cuuint64_t>(v.W), static_cast<cuuint64_t>(v.H),
                        static_cast<cuuint64_t>(v.N)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(v.pitch) * 2, static_cast<cuuint64_t>(v.row) * 2,
                           static_cast<cuuint64_t>(v.img) * 2};
  cuuint32_t box[4] = {8, static_cast<cuuint32_t>(P), static_cast<cuuint32_t>(Hb), 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = encode_fn()(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  TORCH_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (halo) failed: ", static_cast<int>(r));
}

// Tile shapes (64-row blocks of the two consumer warpgroups) that are instantiated.
struct HaloShape {
  int nb0, nb1;
};
constexpr HaloShape kShapes[] = {{4, 3}, {4, 4}};

template <int NB0, int NB1>
void launch(const CUtensorMap& hm, const CUtensorMap& wm, const HaloDgradParams& p, int smem, int sms, cudaStream_t stream) {
  auto kern = halo_dgrad_kernel<NB0, NB1>;
  static int resident = 0;
  if (resident == 0) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kHaloSmemLimit));
    resident = resident_cluster_ctas(kern, kHaloThreads, kHaloSmemLimit, 2);
  }
  const long pair_tiles = (p.num_tiles + 1) / 2;
  const int grid = static_cast<int>(2 * std::max<long>(1, std::min<long>(pair_tiles, std::min(resident, sms) / 2)));
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kHaloThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  C10_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, hm, wm, p));
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  g_halo_launches.fetch_add(1, std::memory_order_relaxed);
}

}  // namespace

// Plan of the halo schedule for one geometry; false when it does not apply.  The kernel runs stride-1 data gradients with at
// most 64 input channels per group (one 64-wide N block), whole 64-channel chunks of dY per group and a halo that fits shared
// memory beside the B ring.  It is selected where it also has at least 3x3 taps, at least 32 k blocks per tile (the halo of
// the next tile loads while the epilogue runs, not while MMAs run: VGG-16 conv1_2, 9 k blocks per tile, measured slower than
// the im2col schedule), at most 30 % padded tile rows and at least two tiles per SM (below that the im2col schedule spreads
// the work over more SMs).
static bool halo_dgrad_plan(int N, int H, int W, int R, int S, int Cg, int Cout_g, int sms, HaloDgradParams* out, int* shape,
                            int* smem_out) {
  if (!g_conv_halo || Cg > 64 || Cg % 8 != 0 || Cout_g % 64 != 0) return false;
  const int P = W + S - 1;
  if (P > 256) return false;
  long best_cost = -1;
  for (int si = 0; si < static_cast<int>(sizeof(kShapes) / sizeof(kShapes[0])); ++si) {
    const int M = 64 * (kShapes[si].nb0 + kShapes[si].nb1);
    int T = std::min(H, M / P);
    if (T < 1) continue;
    const int tiles = (H + T - 1) / T;
    T = (H + tiles - 1) / tiles;                  // same tile count, rows spread evenly
    const int Hb = (M + (R - 1) * P + S - 1 + P - 1) / P;
    const int HP = (Hb * P + 7) / 8 * 8;
    const int slabs = Cout_g / 8;
    const long smem = 1024L + kHaloStages * kHaloBStageBytes + static_cast<long>(slabs) * HP * 16 + kHaloBarBytes;
    if (Hb > 256 || smem > kHaloSmemLimit) continue;
    const long cost = static_cast<long>(tiles) * M;
    if (best_cost >= 0 && cost >= best_cost) continue;
    best_cost = cost;
    HaloDgradParams& p = *out;
    p = HaloDgradParams{};
    p.N = N; p.H = H; p.W = W;
    p.P = P; p.T = T;
    p.tiles_per_img = tiles;
    p.num_tiles = N * tiles;
    p.R = R; p.S = S;
    p.kcb = Cout_g / 64;
    p.slabs = slabs; p.Hb = Hb; p.HP = HP;
    p.halo_bytes = static_cast<uint32_t>(slabs) * Hb * P * 16;
    p.Cg = Cg;
    *shape = si;
    *smem_out = static_cast<int>(smem);
  }
  if (best_cost < 0) return false;
  if (g_conv_halo == 2) return true;
  return R * S >= 9 && R * S * out->kcb >= 32 && best_cost * 10 <= 13L * H * W &&
         static_cast<long>(N) * out->tiles_per_img >= 2L * sms;
}

// conv_dgrad_w on the halo schedule when the geometry selects it (see halo_dgrad_plan); false (nothing launched) otherwise.
// dy: NHWC bf16 [N, groups * Cout_g, OH, OW]; wb: fprop shadow [groups * Cout_g][R][S][Cg]; dx: NHWC bf16 [N, groups * Cg, H, W].
bool conv_dgrad_halo(const at::Tensor& dy, const at::Tensor& wb, int R, int S, int ph, int pw, int groups, int H, int W,
                     const c10::optional<at::Tensor>& mask, double slope, at::Tensor& dx) {
  const NhwcView dv = nhwc_view(dy), xv = nhwc_view(dx);
  const int Cout_g = dv.C / groups, Cg = xv.C / groups;
  if ((dv.pitch * 2) % 16 != 0 || xv.pitch % 2 != 0) return false;
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  HaloDgradParams p;
  int shape = 0, smem = 0;
  if (!halo_dgrad_plan(dv.N, H, W, R, S, Cg, Cout_g, sms, &p, &shape, &smem)) return false;
  for (int gidx = 0; gidx < groups; ++gidx) {
    const auto* dyp = reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr()) + gidx * Cout_g;
    if ((reinterpret_cast<uintptr_t>(dyp) & 15) != 0) return false;
  }
  p.h_org = ph - (R - 1);
  p.w_org = pw - (S - 1);
  p.ldc = xv.pitch;
  p.slope = static_cast<float>(slope);
  auto stream = at::cuda::getCurrentCUDAStream();
  const int RS = R * S;
  for (int gidx = 0; gidx < groups; ++gidx) {
    CUtensorMap hm, wm;
    encode_halo_map(&hm, reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr()) + gidx * Cout_g, dv, Cout_g, p.P, p.Hb);
    const __nv_bfloat16* wptr = reinterpret_cast<const __nv_bfloat16*>(wb.data_ptr()) + static_cast<long>(gidx) * Cout_g * RS * Cg;
    encode_tmap_bf16_3d(&wm, wptr, Cg, Cout_g, RS, static_cast<int64_t>(RS) * Cg, Cg, 64, 32, 1);
    p.dx = reinterpret_cast<__nv_bfloat16*>(dx.data_ptr()) + gidx * Cg;
    p.mask = mask.has_value() ? reinterpret_cast<const __nv_bfloat16*>(mask->data_ptr()) + gidx * Cg : nullptr;
    if (shape == 0) launch<4, 3>(hm, wm, p, smem, sms, stream);
    else launch<4, 4>(hm, wm, p, smem, sms, stream);
  }
  return true;
}

// set_conv_halo_fprop: 0 off (gather schedule only), 1 where the geometry selects it (default), 2 wherever it can run
static int g_conv_halo_fprop = 1;
static std::atomic<int64_t> g_halo_fprop_launches{0};

// Plan of the halo forward for one geometry; false when it does not apply.  The kernel runs stride-1 forwards with at most
// 64 input channels per group in whole k16 steps per tap (Cg % 16 == 0), whole 64-channel blocks of output per group and
// two halos that fit shared memory beside the B ring.  It is selected where it also has at least 3x3 taps, at most 30 %
// padded tile rows and at least two CTA tiles per SM.
static bool halo_fprop_plan(int N, int OH, int OW, int R, int S, int Cg, int Cout_g, int groups, int sms, HaloFpropParams* out,
                            int* smem_out) {
  if (!g_conv_halo_fprop || Cg % 16 != 0 || Cg > 64 || Cout_g % 64 != 0) return false;
  const int P = OW + S - 1;
  constexpr int M = 64 * (4 + 3);
  int T = std::min(OH, M / P);
  if (P > 256 || T < 1) return false;
  const int tiles = (OH + T - 1) / T;
  T = (OH + tiles - 1) / tiles;                 // same tile count, rows spread evenly
  const int Hb = (M + (R - 1) * P + S - 1 + P - 1) / P;
  const int HP = (Hb * P + 7) / 8 * 8;
  const int slabs = Cg / 8;
  const long smem = 1024L + kHaloStages * kHaloBStageBytes + 2L * slabs * HP * 16 + kHaloZeroBytes + kHaloBarBytes;
  if (Hb > 256 || smem > kHaloSmemLimit) return false;
  HaloFpropParams& p = *out;
  p = HaloFpropParams{};
  p.OH = OH; p.OW = OW;
  p.P = P; p.T = T;
  p.tiles_per_img = tiles;
  p.num_tiles = N * tiles;
  p.nblk = Cout_g / 64;
  p.cblocks = groups * p.nblk;
  p.S = S; p.Cg = Cg; p.Cout_g = Cout_g;
  p.steps = R * S * Cg / 16;
  p.kb_per_tile = (p.steps + 3) / 4;
  p.slabs = slabs; p.Hb = Hb; p.HP = HP;
  p.halo_bytes = static_cast<uint32_t>(slabs) * Hb * P * 16;
  *smem_out = static_cast<int>(smem);
  if (g_conv_halo_fprop == 2) return true;
  return R * S >= 9 && static_cast<long>(tiles) * M * 10 <= 13L * OH * OW &&
         static_cast<long>(p.num_tiles) * p.cblocks >= 2L * sms;
}

// conv_fprop on the halo schedule when the geometry selects it (see halo_fprop_plan); false (nothing launched) otherwise.
// The caller has established a stride-1 TAP-mode convolution without channel-padded weights that the gather kernel would
// run.  x: NHWC bf16 [N, groups * Cg, H, W]; wb: [groups * Cout_g][R][S][Cg]; y: NHWC bf16 [N, groups * Cout_g, OH, OW].
bool conv_fprop_halo(const at::Tensor& x, const at::Tensor& wb, const c10::optional<at::Tensor>& bias, int R, int S, int ph,
                     int pw, int groups, bool relu, double slope, at::Tensor& y) {
  const NhwcView xv = nhwc_view(x), yv = nhwc_view(y);
  const int Cg = xv.C / groups, Cout_g = yv.C / groups;
  if ((xv.pitch * 2) % 16 != 0 || (reinterpret_cast<uintptr_t>(x.data_ptr()) & 15) != 0 || yv.pitch % 2 != 0 ||
      (reinterpret_cast<uintptr_t>(y.data_ptr()) & 3) != 0 || (reinterpret_cast<uintptr_t>(wb.data_ptr()) & 15) != 0)
    return false;
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  HaloFpropParams p;
  int smem = 0;
  if (!halo_fprop_plan(xv.N, yv.H, yv.W, R, S, Cg, Cout_g, groups, sms, &p, &smem)) return false;
  p.ph = ph;
  p.pw = pw;
  p.y = reinterpret_cast<__nv_bfloat16*>(y.data_ptr());
  p.ldc = yv.pitch;
  p.bias = bias.has_value() ? bias->data_ptr<float>() : nullptr;
  p.relu = relu;
  p.slope = static_cast<float>(slope);
  const int K = R * S * Cg;
  CUtensorMap hm, wm;
  encode_halo_map(&hm, x.data_ptr(), xv, xv.C, p.P, p.Hb);
  encode_tmap_2d(&wm, wb.data_ptr(), K, static_cast<int64_t>(groups) * Cout_g, K, 64, 32);
  auto kern = halo_fprop_kernel<4, 3>;
  static int resident = 0;
  if (resident == 0) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kHaloSmemLimit));
    resident = resident_cluster_ctas(kern, kHaloThreads, kHaloSmemLimit, 2);
  }
  const long pair_tiles = static_cast<long>(p.num_tiles + 1) / 2 * p.cblocks;
  const int grid = static_cast<int>(2 * std::max<long>(1, std::min<long>(pair_tiles, std::min(resident, sms) / 2)));
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kHaloThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = at::cuda::getCurrentCUDAStream();
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  C10_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, hm, wm, p));
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  g_halo_fprop_launches.fetch_add(1, std::memory_order_relaxed);
  return true;
}

void set_conv_halo_fprop(int64_t mode) {
  TORCH_CHECK(mode >= 0 && mode <= 2,
              "set_conv_halo_fprop: 0 (off), 1 (where the geometry selects it) or 2 (wherever it can run)");
  g_conv_halo_fprop = static_cast<int>(mode);
}

int64_t conv_halo_fprop_launches() { return g_halo_fprop_launches.load(std::memory_order_relaxed); }

void set_conv_halo(int64_t mode) {
  TORCH_CHECK(mode >= 0 && mode <= 2, "set_conv_halo: 0 (off), 1 (where the geometry selects it) or 2 (wherever it can run)");
  g_conv_halo = static_cast<int>(mode);
}

int64_t conv_halo_launches() { return g_halo_launches.load(std::memory_order_relaxed); }

}  // namespace psd

TORCH_LIBRARY_FRAGMENT(poseidon, m) {
  m.def("set_conv_halo(int mode) -> ()", &psd::set_conv_halo);
  m.def("conv_halo_launches() -> int", &psd::conv_halo_launches);
  m.def("set_conv_halo_fprop(int mode) -> ()", &psd::set_conv_halo_fprop);
  m.def("conv_halo_fprop_launches() -> int", &psd::conv_halo_fprop_launches);
}
