// Host side of the halo-tiled data gradient (halo_conv.cuh): geometry selection, tensor maps, launch, the A/B switch.
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

void set_conv_halo(int64_t mode) {
  TORCH_CHECK(mode >= 0 && mode <= 2, "set_conv_halo: 0 (off), 1 (where the geometry selects it) or 2 (wherever it can run)");
  g_conv_halo = static_cast<int>(mode);
}

int64_t conv_halo_launches() { return g_halo_launches.load(std::memory_order_relaxed); }

}  // namespace psd

TORCH_LIBRARY_FRAGMENT(poseidon, m) {
  m.def("set_conv_halo(int mode) -> ()", &psd::set_conv_halo);
  m.def("conv_halo_launches() -> int", &psd::conv_halo_launches);
}
