// Host side of the wgmma GEMM family: tensor-map encoding, template dispatch, torch op registration.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/library.h>
#include <torch/types.h>

#include "wgmma_gemm.cuh"

namespace psd {

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                              const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                              CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeFn get_encode_fn() {
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

static int64_t tmap_elem_bytes(CUtensorMapDataType dtype) {
  TORCH_CHECK(dtype == CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 || dtype == CU_TENSOR_MAP_DATA_TYPE_UINT8,
              "tensor maps: bf16 or 8-bit elements");
  return dtype == CU_TENSOR_MAP_DATA_TYPE_UINT8 ? 1 : 2;
}

// 2-D tensor map: `inner` contiguous elements, `outer` rows `ld` elements apart, 128B swizzle.  dtype: bf16, or UINT8 for
// e4m3 operands (the TMA only moves bytes).
void encode_tmap_2d(CUtensorMap* map, const void* base, int64_t inner, int64_t outer, int64_t ld,
                    int box_inner, int box_outer, CUtensorMapDataType dtype) {
  const int64_t es = tmap_elem_bytes(dtype);
  TORCH_CHECK((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base must be 16-byte aligned");
  TORCH_CHECK((ld * es) % 16 == 0, "TMA row pitch must be a multiple of 16 bytes (ld=", ld, ")");
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(inner), static_cast<cuuint64_t>(outer)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld * es)};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_inner), static_cast<cuuint32_t>(box_outer)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode_fn()(map, dtype, 2, const_cast<void*>(base), dims, strides,
                               box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  TORCH_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed: ", static_cast<int>(r), " inner=", inner,
              " outer=", outer, " ld=", ld);
}

// 3-D bf16 tensor map (innermost dimension contiguous), 128B swizzle; strides in elements for dims 1 and 2.
void encode_tmap_bf16_3d(CUtensorMap* map, const void* base, int64_t d0, int64_t d1, int64_t d2, int64_t stride1, int64_t stride2,
                         int box0, int box1, int box2) {
  TORCH_CHECK((reinterpret_cast<uintptr_t>(base) & 15) == 0 && (stride1 * 2) % 16 == 0 && (stride2 * 2) % 16 == 0,
              "3-D TMA map: 16-byte alignment of base and strides");
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(d0), static_cast<cuuint64_t>(d1), static_cast<cuuint64_t>(d2)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(stride1) * 2, static_cast<cuuint64_t>(stride2) * 2};
  cuuint32_t box[3] = {static_cast<cuuint32_t>(box0), static_cast<cuuint32_t>(box1), static_cast<cuuint32_t>(box2)};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = get_encode_fn()(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  TORCH_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (3-D) failed: ", static_cast<int>(r));
}

// 3-D 8-bit tensor map [d2][d1][d0] (d0 contiguous), 128B swizzle, boxes of {128 bytes, 1, box2}: the fp8 weight-gradient
// operands [C][H][W * Np].  strides in bytes.
void encode_tmap_u8_3d(CUtensorMap* map, const void* base, int64_t d0, int64_t d1, int64_t d2, int64_t stride1,
                       int64_t stride2, int box2) {
  TORCH_CHECK((reinterpret_cast<uintptr_t>(base) & 15) == 0 && stride1 % 16 == 0 && stride2 % 16 == 0,
              "3-D TMA map: 16-byte alignment of base and strides");
  cuuint64_t dims[3] = {static_cast<cuuint64_t>(d0), static_cast<cuuint64_t>(d1), static_cast<cuuint64_t>(d2)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(stride1), static_cast<cuuint64_t>(stride2)};
  cuuint32_t box[3] = {128, 1, static_cast<cuuint32_t>(box2)};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = get_encode_fn()(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  TORCH_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (3-D, 8-bit) failed");
}

// 4-D im2col-mode tensor map over an NHWC tensor (channels innermost, pixel pitch `pitch` elements).
//   lower / upper : bounding-box corner offsets {w, h} (cuTensorMapEncodeIm2col semantics: base pixels run from
//                   `lower` to `extent + upper - 1` in steps of the traversal stride)
//   box           : `pixels` base pixels x 128 bytes of channels (64 bf16 / 128 e4m3 as UINT8), 128B swizzle
void encode_tmap_im2col(CUtensorMap* map, const void* base, int64_t C, int64_t W, int64_t H, int64_t N, int64_t pitch,
                        int lower_w, int lower_h, int upper_w, int upper_h, int pixels, int stride_w, int stride_h,
                        CUtensorMapDataType dtype) {
  const int64_t es = tmap_elem_bytes(dtype);
  using Im2colFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static Im2colFn fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &ptr, cudaEnableDefault, &qres);
    TORCH_CHECK(e == cudaSuccess && qres == cudaDriverEntryPointSuccess && ptr != nullptr,
                "cuTensorMapEncodeIm2col not available from the driver");
    fn = reinterpret_cast<Im2colFn>(ptr);
  }
  TORCH_CHECK((reinterpret_cast<uintptr_t>(base) & 15) == 0 && (pitch * es) % 16 == 0, "im2col TMA: 16-byte alignment");
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H),
                        static_cast<cuuint64_t>(N)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(pitch * es), static_cast<cuuint64_t>(pitch * W * es),
                           static_cast<cuuint64_t>(pitch * W * H * es)};
  int lower[2] = {lower_w, lower_h}, upper[2] = {upper_w, upper_h};
  cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(stride_w), static_cast<cuuint32_t>(stride_h), 1};
  CUresult r = fn(map, dtype, 4, const_cast<void*>(base), dims, strides, lower, upper, static_cast<cuuint32_t>(128 / es),
                  static_cast<cuuint32_t>(pixels), estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  TORCH_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeIm2col failed: ", static_cast<int>(r), " C=", C, " W=", W, " H=", H,
              " N=", N, " lower=", lower_w, ",", lower_h, " upper=", upper_w, ",", upper_h);
}

int g_no_bulk_epi = 2;             // bit 0 / 1: fp32 / bf16 outputs NOT through the bulk-store epilogue (bf16: off by default)
int g_max_stages = 0;             // experiment knob (set_max_stages): ring stages actually used, 0 = all
static int g_pair_cta = 1;        // CTA pairs sharing the B tile by multicast where the tile space allows it; 0 = single CTAs
int pair_cta_enabled() { return g_pair_cta; }

// Launch on a (CG,1,1) cluster.  grid is a multiple of CG.
template <typename Kern>
static void launch_clustered(Kern kern, int grid, int threads, int smem, int cluster, int resident, cudaStream_t stream,
                             const TmapSet& tm, const GemmParams& p, const ConvGeom& cg) {
  if (cluster <= 1) {
    kern<<<grid, threads, smem, stream>>>(tm, p, cg);
  } else {
    grid = std::min(grid, resident);
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

template <int BN, bool A_MN, bool B_MN, int EPI, int CG>
static void launch(const TmapSet& tm, const GemmParams& p, int grid, cudaStream_t stream) {
  auto kern = wgmma_gemm_kernel<BN, A_MN, B_MN, EPI, GATHER_NONE, CG>;
  constexpr int smem = GemmSmem<BN, CG>::kTotal;
  static bool configured = false;
  static int resident = 0;
  if (!configured) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    if (CG > 1) resident = resident_cluster_ctas(kern, kNumThreads, smem, CG);
    configured = true;
  }
  launch_clustered(kern, grid, kNumThreads, smem, CG, resident, stream, tm, p, ConvGeom{});
}

template <bool A_MN, bool B_MN, int EPI>
static void dispatch_bn(int bn, int cg, const TmapSet& tm, const GemmParams& p, int grid, cudaStream_t s) {
  if (cg == 2) {
    switch (bn) {
      case 64:
        if constexpr (!B_MN) launch<64, A_MN, B_MN, EPI, 2>(tm, p, grid, s);
        else TORCH_CHECK(false, "paired CTAs with an MN-major B need BLOCK_N >= 128");
        break;
      case 128: launch<128, A_MN, B_MN, EPI, 2>(tm, p, grid, s); break;
      case 256: launch<256, A_MN, B_MN, EPI, 2>(tm, p, grid, s); break;
      default: TORCH_CHECK(false, "unsupported BLOCK_N ", bn);
    }
    return;
  }
  switch (bn) {
    case 64: launch<64, A_MN, B_MN, EPI, 1>(tm, p, grid, s); break;
    case 128: launch<128, A_MN, B_MN, EPI, 1>(tm, p, grid, s); break;
    case 256: launch<256, A_MN, B_MN, EPI, 1>(tm, p, grid, s); break;
    default: TORCH_CHECK(false, "unsupported BLOCK_N ", bn);
  }
}

int pick_bn(int64_t M, int64_t N, int sms) {
  // Largest N tile that still fills the machine; when even BN=64 cannot, take the tile that launches most CTAs
  // (small-M GEMMs such as the FC forward are bandwidth/latency bound: more CTAs = more TMA streams in flight).
  const int64_t mb = (M + BLOCK_M - 1) / BLOCK_M;
  for (int bn : {256, 128, 64}) {
    if (N >= bn && mb * ((N + bn - 1) / bn) >= sms) return bn;
  }
  return N > 128 ? 64 : (N > 64 ? 128 : 64);
}

// The one entry point.  Operands are described by raw device pointers so that peer (symmetric-memory)
// buffers can be passed exactly like local ones.
//   a_ptrs[i] : A of source i.  a_mn=false: [M, K] row-major (ld = lda) ; a_mn=true: [K, M] row-major.
//   b_ptrs[i] : B of source i, same convention with N.
//   K         : reduction length per source.
void gemm_launch(const std::vector<int64_t>& a_ptrs, bool a_mn, int64_t lda, const std::vector<int64_t>& b_ptrs,
                 bool b_mn, int64_t ldb, int64_t M, int64_t N, int64_t K, int epi, GemmParams p, int bn,
                 int max_ctas, cudaStream_t stream) {
  const int nsrc = static_cast<int>(a_ptrs.size());
  TORCH_CHECK(nsrc >= 1 && nsrc <= kMaxSrc && b_ptrs.size() == a_ptrs.size(), "1..8 sources expected");
  const auto* prop = at::cuda::getCurrentDeviceProperties();
  const int sms = prop->multiProcessorCount;
  if (bn <= 0) bn = pick_bn(M, N, sms);
  const int64_t m_blocks = (M + BLOCK_M - 1) / BLOCK_M;
  // CTA pairs: two m-blocks share every B tile.  Needs >= 2 m-blocks, an even CTA budget, and — for an
  // MN-major B — a half tile made of whole 64-column chunks.
  int cgp = (g_pair_cta && m_blocks >= 2 && (!b_mn || bn >= 128) && (max_ctas <= 0 || max_ctas >= 2)) ? 2 : 1;
  TmapSet tm;
  for (int s = 0; s < nsrc; ++s) {
    if (!a_mn) encode_tmap_2d(&tm.a[s], reinterpret_cast<void*>(a_ptrs[s]), K, M, lda, BLOCK_K, BLOCK_M);
    else       encode_tmap_2d(&tm.a[s], reinterpret_cast<void*>(a_ptrs[s]), M, K, lda, 64, BLOCK_K);
    if (!b_mn) encode_tmap_2d(&tm.b[s], reinterpret_cast<void*>(b_ptrs[s]), K, N, ldb, BLOCK_K, bn / cgp);
    else       encode_tmap_2d(&tm.b[s], reinterpret_cast<void*>(b_ptrs[s]), N, K, ldb, 64, BLOCK_K);
  }
  p.M = static_cast<int>(M);
  p.N = static_cast<int>(N);
  p.max_stages = g_max_stages;
  p.no_bulk_epi = g_no_bulk_epi;
  p.kb_per_src = static_cast<int>((K + BLOCK_K - 1) / BLOCK_K);
  p.num_src = nsrc;
  if (p.split_k < 1) p.split_k = 1;
  p.split_k = std::min(p.split_k, p.kb_per_src * nsrc);
  const int64_t m_units = cgp == 2 ? (m_blocks + 1) / 2 : m_blocks;
  const int64_t tiles = m_units * ((N + bn - 1) / bn) * p.split_k;          // CTA (or CTA-pair) tiles
  const int budget = (max_ctas > 0 ? max_ctas : sms) / cgp;
  int grid = static_cast<int>(std::min<int64_t>(tiles, budget)) * cgp;
  if (!a_mn && !b_mn) {
    if (epi == EPI_BF16) dispatch_bn<false, false, EPI_BF16>(bn, cgp, tm, p, grid, stream);
    else if (epi == EPI_F32) dispatch_bn<false, false, EPI_F32>(bn, cgp, tm, p, grid, stream);
    else TORCH_CHECK(false, "EPI_SGD requires MN-major operands");
  } else if (!a_mn && b_mn) {
    if (epi == EPI_BF16) dispatch_bn<false, true, EPI_BF16>(bn, cgp, tm, p, grid, stream);
    else if (epi == EPI_F32) dispatch_bn<false, true, EPI_F32>(bn, cgp, tm, p, grid, stream);
    else TORCH_CHECK(false, "K-major x MN-major supports the bf16 / fp32 epilogues");
  } else if (a_mn && b_mn) {
    if (epi == EPI_F32) dispatch_bn<true, true, EPI_F32>(bn, cgp, tm, p, grid, stream);
    else if (epi == EPI_SGD) dispatch_bn<true, true, EPI_SGD>(bn, cgp, tm, p, grid, stream);
    else TORCH_CHECK(false, "MN-major x MN-major supports fp32 / SGD epilogues");
  } else {
    TORCH_CHECK(false, "MN-major A with K-major B is not instantiated");
  }
}

// Split-K finish: out = act(sum_s ws[s] + bias) (optionally ReLU-masked) -> bf16.  ws holds one dense [M, N] fp32 partial per
// split, summed in split order: the result does not depend on which CTA finished first.  Four columns per thread (16-byte
// loads / stores, 32-bit index math); the scalar form serves N or ldc that are not multiples of 4.
__global__ void __launch_bounds__(256)
splitk_finish_kernel(const float* __restrict__ ws, long split_stride, int splits, __nv_bfloat16* __restrict__ out, long ldc,
                     const float* __restrict__ bias, const __nv_bfloat16* __restrict__ mask, int relu, float slope, int M, int N) {
  if ((N & 3) == 0 && (ldc & 3) == 0) {
    const uint32_t n4 = static_cast<uint32_t>(N) >> 2;
    const uint32_t total4 = static_cast<uint32_t>(M) * n4;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += gridDim.x * blockDim.x) {
      const uint32_t m = i / n4, c = (i - m * n4) << 2;
      float4 v = reinterpret_cast<const float4*>(ws)[i];
      for (int sp = 1; sp < splits; ++sp) {
        const float4 w = reinterpret_cast<const float4*>(ws + sp * split_stride)[i];
        v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
      }
      if (bias != nullptr) {
        const float4 b = *reinterpret_cast<const float4*>(bias + c);
        v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
      }
      if (relu) {
        v.x = v.x > 0.f ? v.x : v.x * slope; v.y = v.y > 0.f ? v.y : v.y * slope;
        v.z = v.z > 0.f ? v.z : v.z * slope; v.w = v.w > 0.f ? v.w : v.w * slope;
      }
      const long o = static_cast<long>(m) * ldc + c;
      if (mask != nullptr) {
        const uint2 mk = *reinterpret_cast<const uint2*>(mask + o);
        if (!(__uint_as_float(mk.x << 16) > 0.f)) v.x *= slope;
        if (!(__uint_as_float(mk.x & 0xffff0000u) > 0.f)) v.y *= slope;
        if (!(__uint_as_float(mk.y << 16) > 0.f)) v.z *= slope;
        if (!(__uint_as_float(mk.y & 0xffff0000u) > 0.f)) v.w *= slope;
      }
      __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
      uint2 pk;
      pk.x = *reinterpret_cast<uint32_t*>(&lo);
      pk.y = *reinterpret_cast<uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(out + o) = pk;
    }
    return;
  }
  const long total = static_cast<long>(M) * N;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int m = static_cast<int>(i / N), n = static_cast<int>(i - static_cast<long>(m) * N);
    float v = ws[i];
    for (int sp = 1; sp < splits; ++sp) v += ws[sp * split_stride + i];
    if (bias != nullptr) v += bias[n];
    if (relu) v = v > 0.f ? v : v * slope;
    if (mask != nullptr && !(__bfloat162float(mask[m * ldc + n]) > 0.f)) v *= slope;
    out[m * ldc + n] = __float2bfloat16(v);
  }
}

// out[m, n] (+)= sum_s ws[s][m, n] in split order (ws: `splits` dense [M, N] fp32 partials, split_stride elements apart).
// accumulate = 0 overwrites out: gemm_f32(accumulate=False) with split_k > 1 used to add onto whatever out held.
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ ws, long split_stride, int splits, float* __restrict__ out, long ldo, int M, int N,
                     int accumulate) {
  const long total = static_cast<long>(M) * N;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long m = i / N, n = i - m * N;
    float v = ws[i];
    for (int sp = 1; sp < splits; ++sp) v += ws[sp * split_stride + i];
    if (accumulate) out[m * ldo + n] += v;
    else out[m * ldo + n] = v;
  }
}

void splitk_reduce(const at::Tensor& ws, int splits, float* out, long ldo, int M, int N, bool accumulate, cudaStream_t stream) {
  const long total = static_cast<long>(M) * N;
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  const int grid = static_cast<int>(std::max<long>(1, std::min<long>((total + 255) / 256, sms * 8L)));
  splitk_reduce_kernel<<<grid, 256, 0, stream>>>(ws.data_ptr<float>(), total, splits, out, ldo, M, N, accumulate ? 1 : 0);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------ torch ops
static const void* opt_ptr(const c10::optional<at::Tensor>& t) { return t.has_value() ? t->data_ptr() : nullptr; }

// C[M,N] bf16 = act(alpha * A·Bᵀ + bias) (optionally masked).  a: [M,K] (or [K,M] if a_mn), b: [N,K] (or [K,N]).
at::Tensor gemm_bf16(const at::Tensor& a, bool a_mn, const at::Tensor& b, bool b_mn,
                     const c10::optional<at::Tensor>& bias, bool relu, double slope,
                     const c10::optional<at::Tensor>& mask, c10::optional<at::Tensor> out, int64_t bn) {
  TORCH_CHECK(a.is_cuda() && b.is_cuda() && a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16);
  TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && a.stride(1) == 1 && b.stride(1) == 1);
  c10::cuda::CUDAGuard guard(a.device());
  const int64_t M = a_mn ? a.size(1) : a.size(0), K = a_mn ? a.size(0) : a.size(1);
  const int64_t N = b_mn ? b.size(1) : b.size(0);
  TORCH_CHECK((b_mn ? b.size(0) : b.size(1)) == K, "K mismatch");
  at::Tensor c = out.has_value() ? *out : at::empty({M, N}, a.options());
  TORCH_CHECK(c.scalar_type() == at::kBFloat16 && c.size(0) == M && c.size(1) == N && c.stride(1) == 1);
  GemmParams p{};
  p.c_bf16 = reinterpret_cast<__nv_bfloat16*>(c.data_ptr());
  p.ldc = c.stride(0);
  p.bias = reinterpret_cast<const float*>(opt_ptr(bias));
  if (bias.has_value()) TORCH_CHECK(bias->scalar_type() == at::kFloat && bias->numel() == N);
  p.mask = reinterpret_cast<const __nv_bfloat16*>(opt_ptr(mask));
  if (mask.has_value()) TORCH_CHECK(mask->scalar_type() == at::kBFloat16 && mask->stride(0) == p.ldc);
  p.relu = relu;
  p.relu_slope = static_cast<float>(slope);
  p.alpha = 1.f;
  p.split_k = 1;
  auto stream = at::cuda::getCurrentCUDAStream();
  // Small-M GEMMs (the inner-product forward / data-gradient at batch 256): two M blocks cannot fill the SMs with wide
  // tiles, and narrow tiles re-read the activation panel once per 64 output columns.  Split the reduction over the idle
  // SMs into an fp32 workspace, then one finishing pass.
  if (bn <= 0 && !a_mn) {
    const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
    const int bn_s = N >= 256 ? 256 : (N > 64 ? 128 : 64);
    const int64_t tiles = ((M + BLOCK_M - 1) / BLOCK_M) * ((N + bn_s - 1) / bn_s);
    const int64_t kb = (K + BLOCK_K - 1) / BLOCK_K;
    const int64_t split = std::min<int64_t>(sms / std::max<int64_t>(tiles, 1), kb / 8);
    if (tiles * 2 <= sms && split >= 2) {
      // one fp32 partial per split, written with plain stores and summed in split order by the finishing kernel
      at::Tensor ws = at::empty({split, M, N}, a.options().dtype(at::kFloat));
      GemmParams q{};
      q.c_f32 = ws.data_ptr<float>();
      q.ldc = N;
      q.alpha = 1.f;
      q.split_k = static_cast<int>(split);
      q.split_stride = M * N;
      gemm_launch({reinterpret_cast<int64_t>(a.data_ptr())}, a_mn, a.stride(0),
                  {reinterpret_cast<int64_t>(b.data_ptr())}, b_mn, b.stride(0), M, N, K, EPI_F32, q, bn_s, 0, stream);
      const long total = (N % 4 == 0 && p.ldc % 4 == 0) ? M * N / 4 : M * N;
      const int grid = static_cast<int>(std::min<long>((total + 255) / 256, sms * 8L));
      splitk_finish_kernel<<<grid, 256, 0, stream>>>(ws.data_ptr<float>(), M * N, static_cast<int>(split), p.c_bf16, p.ldc,
                                                     p.bias, p.mask, p.relu ? 1 : 0, p.relu_slope, static_cast<int>(M),
                                                     static_cast<int>(N));
      C10_CUDA_KERNEL_LAUNCH_CHECK();
      return c;
    }
  }
  gemm_launch({reinterpret_cast<int64_t>(a.data_ptr())}, a_mn, a.stride(0),
              {reinterpret_cast<int64_t>(b.data_ptr())}, b_mn, b.stride(0), M, N, K, EPI_BF16, p,
              static_cast<int>(bn), 0, stream);
  return c;
}

// out[M,N] fp32 = alpha * A·Bᵀ, or out += alpha * A·Bᵀ with accumulate, for every split_k.  split_k > 1: the splits' partials
// go to a workspace and are summed in split order, then stored into (or added onto) out in one pass.
void gemm_f32(const at::Tensor& a, bool a_mn, const at::Tensor& b, bool b_mn, at::Tensor out, double alpha,
              bool accumulate, int64_t split_k, int64_t bn) {
  TORCH_CHECK(a.is_cuda() && a.scalar_type() == at::kBFloat16 && b.scalar_type() == at::kBFloat16);
  TORCH_CHECK(a.dim() == 2 && b.dim() == 2 && a.stride(1) == 1 && b.stride(1) == 1);
  TORCH_CHECK(out.scalar_type() == at::kFloat && out.dim() == 2 && out.stride(1) == 1);
  c10::cuda::CUDAGuard guard(a.device());
  const int64_t M = a_mn ? a.size(1) : a.size(0), K = a_mn ? a.size(0) : a.size(1);
  const int64_t N = b_mn ? b.size(1) : b.size(0);
  TORCH_CHECK((b_mn ? b.size(0) : b.size(1)) == K && out.size(0) == M && out.size(1) == N, "shape mismatch");
  auto stream = at::cuda::getCurrentCUDAStream();
  const int64_t splits = std::max<int64_t>(1, std::min<int64_t>(split_k, (K + BLOCK_K - 1) / BLOCK_K));
  GemmParams p{};
  p.alpha = static_cast<float>(alpha);
  p.split_k = static_cast<int>(splits);
  if (splits == 1) {
    p.c_f32 = out.data_ptr<float>();
    p.ldc = out.stride(0);
    p.atomic = accumulate ? 1 : 0;           // one add per element onto the existing value
    gemm_launch({reinterpret_cast<int64_t>(a.data_ptr())}, a_mn, a.stride(0),
                {reinterpret_cast<int64_t>(b.data_ptr())}, b_mn, b.stride(0), M, N, K, EPI_F32, p, static_cast<int>(bn), 0,
                stream);
    return;
  }
  at::Tensor ws = at::empty({splits, M, N}, out.options());
  p.c_f32 = ws.data_ptr<float>();
  p.ldc = N;
  p.split_stride = M * N;
  gemm_launch({reinterpret_cast<int64_t>(a.data_ptr())}, a_mn, a.stride(0),
              {reinterpret_cast<int64_t>(b.data_ptr())}, b_mn, b.stride(0), M, N, K, EPI_F32, p, static_cast<int>(bn), 0,
              stream);
  splitk_reduce(ws, static_cast<int>(splits), out.data_ptr<float>(), out.stride(0), static_cast<int>(M), static_cast<int>(N),
                accumulate, stream);
}

// The sufficient-factor outer product with the optimizer fused into the epilogue:
//   ΔW[N,K] = alpha * Σ_src U_srcᵀ[N,Mb] · V_src[Mb,K];   (W, H, Wb) <- step(W, H, ΔW)   in place.
// u_ptrs / v_ptrs are device addresses (local or NVLink-peer-mapped) of [Mb, N] / [Mb, K] bf16 buffers.
// With one source this is the local weight-gradient + update kernel (no dense dW is ever materialised).
void sfb_outer_sgd(std::vector<int64_t> u_ptrs, std::vector<int64_t> v_ptrs, int64_t Mb, int64_t N, int64_t K,
                   at::Tensor w, at::Tensor h, c10::optional<at::Tensor> wb, double alpha, double lr,
                   double momentum, double decay, int64_t rule, bool l1, double delta,
                   const c10::optional<at::Tensor>& flags, int64_t epoch, int64_t src_rot, int64_t bn,
                   int64_t max_ctas, const c10::optional<at::Tensor>& lr_dev, const c10::optional<at::Tensor>& epoch_dev) {
  TORCH_CHECK(w.is_cuda() && w.scalar_type() == at::kFloat && h.scalar_type() == at::kFloat);
  TORCH_CHECK(w.numel() == N * K && h.numel() == N * K && w.is_contiguous() && h.is_contiguous());
  c10::cuda::CUDAGuard guard(w.device());
  GemmParams p{};
  p.w = w.data_ptr<float>();
  p.h = h.data_ptr<float>();
  p.wb = wb.has_value() ? reinterpret_cast<__nv_bfloat16*>(wb->data_ptr()) : nullptr;
  p.ldc = K;
  p.alpha = static_cast<float>(alpha);
  p.lr = static_cast<float>(lr);
  p.lr_dev = lr_dev.has_value() ? lr_dev->data_ptr<float>() : nullptr;
  p.momentum = static_cast<float>(momentum);
  p.decay = static_cast<float>(decay);
  p.rule = static_cast<int>(rule);
  p.l1 = l1;
  p.delta = static_cast<float>(delta);
  p.split_k = 1;
  p.src_rot = static_cast<int>(src_rot);
  if (flags.has_value()) {
    TORCH_CHECK(flags->scalar_type() == at::kInt && flags->numel() >= static_cast<int64_t>(u_ptrs.size()));
    p.flags = reinterpret_cast<const uint32_t*>(flags->data_ptr());
    p.epoch = static_cast<uint32_t>(epoch);
    p.epoch_dev = epoch_dev.has_value() ? reinterpret_cast<const uint32_t*>(epoch_dev->data_ptr()) : nullptr;
  }
  // A = Uᵀ : MN-major with "M" = N_out ; B = Vᵀ... : MN-major with "N" = K_in ; reduction = Mb rows.
  gemm_launch(u_ptrs, true, N, v_ptrs, true, K, N, K, Mb, EPI_SGD, p, static_cast<int>(bn),
              static_cast<int>(max_ctas), at::cuda::getCurrentCUDAStream());
}

// Same reduction over the P sufficient-factor slots, but into a dense fp32 buffer (no optimizer step): the
// two-pass form  out = alpha * Σ_src U_srcᵀ V_src ; fused_update(out)  which streams W/H at full HBM rate.
void sfb_outer_f32(std::vector<int64_t> u_ptrs, std::vector<int64_t> v_ptrs, int64_t Mb, int64_t N, int64_t K,
                   at::Tensor out, double alpha, const c10::optional<at::Tensor>& flags, int64_t epoch, int64_t src_rot,
                   int64_t bn, int64_t max_ctas, const c10::optional<at::Tensor>& epoch_dev) {
  TORCH_CHECK(out.is_cuda() && out.scalar_type() == at::kFloat && out.numel() == N * K && out.is_contiguous());
  c10::cuda::CUDAGuard guard(out.device());
  GemmParams p{};
  p.c_f32 = out.data_ptr<float>();
  p.ldc = K;
  p.alpha = static_cast<float>(alpha);
  p.split_k = 1;
  p.src_rot = static_cast<int>(src_rot);
  if (flags.has_value()) {
    TORCH_CHECK(flags->scalar_type() == at::kInt && flags->numel() >= static_cast<int64_t>(u_ptrs.size()));
    p.flags = reinterpret_cast<const uint32_t*>(flags->data_ptr());
    p.epoch = static_cast<uint32_t>(epoch);
    p.epoch_dev = epoch_dev.has_value() ? reinterpret_cast<const uint32_t*>(epoch_dev->data_ptr()) : nullptr;
  }
  gemm_launch(u_ptrs, true, N, v_ptrs, true, K, N, K, Mb, EPI_F32, p, static_cast<int>(bn), static_cast<int>(max_ctas),
              at::cuda::getCurrentCUDAStream());
}

void set_pair_cta(int64_t on) { g_pair_cta = on != 0; }
void set_max_stages(int64_t n) { g_max_stages = static_cast<int>(n); }
// bit 0: fp32 outputs, bit 1: bf16 outputs leave through shared slabs + bulk row stores (default 1: fp32 only)
void set_bulk_epilogue(int64_t on) { g_no_bulk_epi = static_cast<int>(~on & 3); }

}  // namespace psd

TORCH_LIBRARY_FRAGMENT(poseidon, m) {
  m.def("set_pair_cta(int on) -> ()", &psd::set_pair_cta);
  m.def("set_max_stages(int n) -> ()", &psd::set_max_stages);
  m.def("set_bulk_epilogue(int on) -> ()", &psd::set_bulk_epilogue);
  m.def("sfb_outer_f32(int[] u_ptrs, int[] v_ptrs, int Mb, int N, int K, Tensor(a!) out, float alpha, Tensor? flags, "
        "int epoch, int src_rot, int bn, int max_ctas, Tensor? epoch_dev) -> ()", &psd::sfb_outer_f32);
  m.def("gemm_bf16(Tensor a, bool a_mn, Tensor b, bool b_mn, Tensor? bias, bool relu, float slope, Tensor? mask, "
        "Tensor? out, int bn) -> Tensor", &psd::gemm_bf16);
  m.def("gemm_f32(Tensor a, bool a_mn, Tensor b, bool b_mn, Tensor(a!) out, float alpha, bool accumulate, "
        "int split_k, int bn) -> ()", &psd::gemm_f32);
  m.def("sfb_outer_sgd(int[] u_ptrs, int[] v_ptrs, int Mb, int N, int K, Tensor(a!) w, Tensor(b!) h, "
        "Tensor(c!)? wb, float alpha, float lr, float momentum, float decay, int rule, bool l1, float delta, "
        "Tensor? flags, int epoch, int src_rot, int bn, int max_ctas, Tensor? lr_dev, Tensor? epoch_dev) -> ()", &psd::sfb_outer_sgd);
}
