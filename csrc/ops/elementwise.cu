// Small memory-bound kernels of the sm100 engine: data transform (uint8 NCHW -> bf16 NHWC), standalone
// ReLU, counter-based dropout, bias gradient (column sums), fp32 -> bf16 shadow cast.
//
// reference: src/caffe/data_transformer.cpp:10-125 (CPU per-datum loop), layers/relu_layer.cu:10-42,
// layers/dropout_layer.cu:15-50 (separate cuRAND mask generation + kernel), caffe_gpu_gemv bias gradient
// (layers/conv_layer.cu:66-70, inner_product_layer.cu:38-43).
#include "nhwc_common.cuh"

namespace psd {

// ------------------------------------------------------------------ data transform
// out[n, oh+opad, ow+opad, 0..Cp) = (x[n, c, h_off+oh, w_off+(flip ? OW-1-ow : ow)] - mean) * scale, channels >= C zero.
// Each thread produces PX consecutive output pixels of one row: PX*C independent loads in flight, and the PX
// packed pixels leave as one or two 16-byte stores.
// Threads walk the PHYSICAL output (border and alignment columns included) so the kernel itself writes the zeros —
// no separate memset pass over the 100 MB activation — with 32-bit indices and magic-number divides (the first
// version spent most of its instructions per thread on three 64-bit divisions and was issue-bound).
template <typename TIn, int CP, int PX>
__global__ void __launch_bounds__(256)
transform_kernel(const TIn* __restrict__ x, __nv_bfloat16* __restrict__ out, const int* __restrict__ h_off,
                 const int* __restrict__ w_off, const uint8_t* __restrict__ flip, const float* __restrict__ mean,
                 int mean_mode, float scale, int C, int H, int W, int OH, int OW, int opad, int OWp, FastDiv d_owg,
                 FastDiv d_ohp, uint32_t total, int s2d) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const uint32_t t = fdiv(i, d_owg);
    const int owg = static_cast<int>(i - t * d_owg.d);
    const uint32_t n = fdiv(t, d_ohp);
    const int ohp = static_cast<int>(t - n * d_ohp.d);
    const int oh = ohp - opad;
    const bool row_ok = static_cast<unsigned>(oh) < static_cast<unsigned>(OH);
    const int h = h_off[n] + oh;
    const int wo = w_off[n];
    const bool fl = flip[n] != 0;
    const TIn* xn = x + static_cast<long>(n) * C * H * W + static_cast<long>(h) * W;
    uint32_t packed[PX][CP / 2];
#pragma unroll
    for (int q = 0; q < PX; ++q) {
      const int ow = owg * PX + q - opad;
      const bool ok = row_ok && static_cast<unsigned>(ow) < static_cast<unsigned>(OW);
      const int w = wo + (fl ? (OW - 1 - ow) : ow);
      float v[CP];
#pragma unroll
      for (int c = 0; c < CP; ++c) {
        float f = 0.f;
        if (ok && c < C) {
          f = static_cast<float>(xn[c * (H * W) + w]);
          if (mean_mode == 1) f -= mean[c];
          else if (mean_mode == 2) f -= mean[(c * H + h) * W + w];
          f *= scale;
        }
        v[c] = f;
      }
#pragma unroll
      for (int c = 0; c < CP / 2; ++c) {
        const __nv_bfloat162 b2 = __floats2bfloat162_rn(v[2 * c], v[2 * c + 1]);
        packed[q][c] = *reinterpret_cast<const uint32_t*>(&b2);
      }
    }
    __nv_bfloat16* o = out + (static_cast<long>(t) * OWp + owg * PX) * CP;      // t = n * OHp + ohp
    if (s2d) {
      // space-to-depth by 4 (stride-4 first layers): pixel (y, x), channel c -> block (y/4, x/4), channel
      // (y%4)*16 + (x%4)*4 + c.  This thread's 4 pixels are one block row: 16 contiguous elements.
      const int OHq = static_cast<int>(d_ohp.d) >> 2, OWq = OWp >> 2;
      o = out + ((static_cast<long>(n) * OHq + (ohp >> 2)) * OWq + owg) * 64 + (ohp & 3) * 16;
    }
    const int left = OWp - owg * PX;
    if (CP == 4 && left >= PX && PX == 4) {
      // 4 pixels x 4 channels = 32 bytes, 16-byte aligned (OWp is even and the group starts at a multiple of 4)
      *reinterpret_cast<uint4*>(o) = make_uint4(packed[0][0], packed[0][1], packed[1][0], packed[1][1]);
      *reinterpret_cast<uint4*>(o + 8) = make_uint4(packed[2][0], packed[2][1], packed[3][0], packed[3][1]);
    } else {
#pragma unroll
      for (int q = 0; q < PX; ++q) {
        if (q >= left) break;
        if constexpr (CP == 4) {
          *reinterpret_cast<uint2*>(o + q * CP) = make_uint2(packed[q][0], packed[q][1]);
        } else {
          *reinterpret_cast<uint4*>(o + q * CP) = make_uint4(packed[q][0], packed[q][1], packed[q][2], packed[q][3]);
        }
      }
    }
  }
}

// x: [N,C,H,W] uint8|float32 contiguous -> [N, Cp, OH+2opad, OW+2opad] bf16 channels-last (border zero).
at::Tensor transform_nhwc(const at::Tensor& x, const at::Tensor& h_off, const at::Tensor& w_off, const at::Tensor& flip,
                          const c10::optional<at::Tensor>& mean, double scale, int64_t OH, int64_t OW, int64_t cp,
                          int64_t opad, int64_t wextra, int64_t hextra, bool s2d) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 4 && x.is_contiguous());
  TORCH_CHECK(h_off.scalar_type() == at::kInt && w_off.scalar_type() == at::kInt && flip.scalar_type() == at::kByte);
  c10::cuda::CUDAGuard guard(x.device());
  const int N = x.size(0), C = x.size(1), H = x.size(2), W = x.size(3);
  TORCH_CHECK(C <= cp && (cp == 4 || cp == 8), "transform: channel padding must be 4 or 8");
  const int OHp = OH + 2 * opad + hextra, OWp = OW + 2 * opad + wextra;
  TORCH_CHECK(!s2d || (cp == 4 && OHp % 4 == 0 && OWp % 4 == 0), "transform: space-to-depth needs 4 channels and /4 extents");
  at::Tensor out = s2d ? empty_nhwc(N, 64, OHp / 4, OWp / 4, x.options().dtype(at::kBFloat16))
                       : empty_nhwc(N, cp, OHp, OWp, x.options().dtype(at::kBFloat16));
  int mean_mode = 0;
  const float* mp = nullptr;
  if (mean.has_value()) {
    TORCH_CHECK(mean->scalar_type() == at::kFloat && mean->is_contiguous());
    mp = mean->data_ptr<float>();
    mean_mode = mean->numel() == C ? 1 : 2;
    if (mean_mode == 2) TORCH_CHECK(mean->numel() == static_cast<int64_t>(C) * H * W, "mean image shape mismatch");
  }
  auto stream = at::cuda::getCurrentCUDAStream();
  constexpr int kPx = 4;
  const int owg = (OWp + kPx - 1) / kPx;
  const long total = static_cast<long>(N) * OHp * owg;
  TORCH_CHECK(total < (1L << 31) && static_cast<long>(C) * H * W < (1L << 31), "transform: batch too large for 32-bit indexing");
  TORCH_CHECK(cp == 8 || OWp % 2 == 0, "transform: padded width must be even for 4-channel outputs");
  const FastDiv d_owg = make_fastdiv(owg), d_ohp = make_fastdiv(OHp);
  auto op = reinterpret_cast<__nv_bfloat16*>(out.data_ptr());
#define PSD_XF(T, CPV)                                                                                          \
  transform_kernel<T, CPV, kPx><<<grid_for(total, 256, 132 * 32), 256, 0, stream>>>(                                         \
      x.data_ptr<T>(), op, h_off.data_ptr<int>(), w_off.data_ptr<int>(), flip.data_ptr<uint8_t>(), mp, mean_mode, \
      static_cast<float>(scale), C, H, W, OH, OW, opad, OWp, d_owg, d_ohp, static_cast<uint32_t>(total), s2d ? 1 : 0)
  if (x.scalar_type() == at::kByte) {
    if (cp == 4) PSD_XF(uint8_t, 4); else PSD_XF(uint8_t, 8);
  } else {
    TORCH_CHECK(x.scalar_type() == at::kFloat, "transform: uint8 or float32 input");
    if (cp == 4) PSD_XF(float, 4); else PSD_XF(float, 8);
  }
#undef PSD_XF
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return out;
}

// ------------------------------------------------------------------ ReLU (standalone; normally fused into epilogues)
__global__ void relu_fwd_kernel(const bf16x8* __restrict__ x, bf16x8* __restrict__ y, long n8, float slope) {
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < n8; i += static_cast<long>(gridDim.x) * blockDim.x) {
    float f[8];
    unpack8(x[i], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = f[j] > 0.f ? f[j] : f[j] * slope;
    y[i] = pack8(f);
  }
}
__global__ void relu_bwd_kernel(const bf16x8* __restrict__ y, const bf16x8* __restrict__ dy, bf16x8* __restrict__ dx, long n8,
                                float slope) {
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < n8; i += static_cast<long>(gridDim.x) * blockDim.x) {
    float f[8], d[8];
    unpack8(y[i], f);
    unpack8(dy[i], d);
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] = f[j] > 0.f ? d[j] : d[j] * slope;
    dx[i] = pack8(d);
  }
}

static void check_dense8(const at::Tensor& t) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kBFloat16 && t.numel() % 8 == 0, "dense bf16 tensor, numel % 8 == 0");
  TORCH_CHECK(t.is_contiguous() || t.is_contiguous(at::MemoryFormat::ChannelsLast), "dense tensor expected");
}

at::Tensor relu_fwd(const at::Tensor& x, double slope) {
  check_dense8(x);
  c10::cuda::CUDAGuard guard(x.device());
  at::Tensor y = at::empty_like(x);
  const long n8 = x.numel() / 8;
  relu_fwd_kernel<<<grid_for(n8, 256), 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const bf16x8*>(x.data_ptr()), reinterpret_cast<bf16x8*>(y.data_ptr()), n8, static_cast<float>(slope));
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return y;
}
at::Tensor relu_bwd(const at::Tensor& y, const at::Tensor& dy, double slope) {
  check_dense8(y);
  check_dense8(dy);
  TORCH_CHECK(y.strides() == dy.strides(), "relu_bwd: layout mismatch");
  c10::cuda::CUDAGuard guard(y.device());
  at::Tensor dx = at::empty_like(y);
  const long n8 = y.numel() / 8;
  relu_bwd_kernel<<<grid_for(n8, 256), 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const bf16x8*>(y.data_ptr()), reinterpret_cast<const bf16x8*>(dy.data_ptr()),
      reinterpret_cast<bf16x8*>(dx.data_ptr()), n8, static_cast<float>(slope));
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return dx;
}

// ReLU backward for NHWC tensors that are channel slices of wider buffers (zero-copy concat: a branch convolution's
// output y lives inside the concat slab, its incoming gradient dy is a channel slice of the slab's gradient): rows are
// pixels, C contiguous channels, independent pixel pitches.  Output dense NHWC.
__global__ void relu_bwd_pitch_kernel(const __nv_bfloat16* __restrict__ y, const __nv_bfloat16* __restrict__ dy,
                                      __nv_bfloat16* __restrict__ dx, long total8, int c8n, long py, long pdy, float slope) {
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total8; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long pix = i / c8n;
    const int c0 = static_cast<int>(i - pix * c8n) * 8;
    float f[8], d[8];
    unpack8(ld8(y + pix * py + c0), f);
    unpack8(ld8(dy + pix * pdy + c0), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) d[j] = f[j] > 0.f ? d[j] : d[j] * slope;
    st8(dx + pix * (static_cast<long>(c8n) * 8) + c0, pack8(d));
  }
}
at::Tensor relu_bwd_nhwc(const at::Tensor& y, const at::Tensor& dy, double slope) {
  TORCH_CHECK(y.is_cuda() && y.scalar_type() == at::kBFloat16 && dy.scalar_type() == at::kBFloat16);
  c10::cuda::CUDAGuard guard(y.device());
  NhwcView vy = nhwc_view(y), vd = nhwc_view(dy);
  TORCH_CHECK(vy.N == vd.N && vy.C == vd.C && vy.H == vd.H && vy.W == vd.W && vy.C % 8 == 0 && vy.pitch % 8 == 0 &&
              vd.pitch % 8 == 0, "relu_bwd_nhwc: shapes must match, channels in multiples of 8");
  at::Tensor dx = empty_nhwc(vy.N, vy.C, vy.H, vy.W, y.options());
  const long total8 = static_cast<long>(vy.N) * vy.H * vy.W * (vy.C / 8);
  relu_bwd_pitch_kernel<<<grid_for(total8, 256), 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const __nv_bfloat16*>(y.data_ptr()), reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr()),
      reinterpret_cast<__nv_bfloat16*>(dx.data_ptr()), total8, vy.C / 8, vy.pitch, vd.pitch, static_cast<float>(slope));
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return dx;
}

// ------------------------------------------------------------------ dropout (mask regenerated from (seed, index))
__device__ __forceinline__ uint32_t mix32(uint32_t a, uint32_t b) {
  uint32_t h = a * 0x9E3779B1u ^ (b + 0x7F4A7C15u);
  h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
  return h;
}
// keep iff hash > threshold, threshold = UINT_MAX * ratio (same test as the reference's uint mask).
__global__ void dropout_kernel(const bf16x8* __restrict__ x, bf16x8* __restrict__ y, long n8, uint32_t seed_lo, uint32_t seed_hi,
                               uint32_t threshold, float scale, const long long* __restrict__ seed_dev) {
  if (seed_dev != nullptr) {                       // per-iteration counter kept on the device (CUDA-graph replay safe)
    const unsigned long long s = static_cast<unsigned long long>(*seed_dev) * 0x9E3779B97F4A7C15ull;
    seed_lo ^= static_cast<uint32_t>(s);
    seed_hi ^= static_cast<uint32_t>(s >> 32);
  }
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < n8; i += static_cast<long>(gridDim.x) * blockDim.x) {
    float f[8];
    unpack8(x[i], f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint64_t e = static_cast<uint64_t>(i) * 8 + j;
      const uint32_t r = mix32(mix32(static_cast<uint32_t>(e), seed_lo), static_cast<uint32_t>(e >> 32) ^ seed_hi);
      f[j] = r > threshold ? f[j] * scale : 0.f;
    }
    y[i] = pack8(f);
  }
}
// forward and backward are the same map applied to x resp. dy.
at::Tensor dropout_apply(const at::Tensor& x, double ratio, int64_t seed, const c10::optional<at::Tensor>& seed_dev) {
  check_dense8(x);
  c10::cuda::CUDAGuard guard(x.device());
  at::Tensor y = at::empty_like(x);
  const long n8 = x.numel() / 8;
  const uint32_t thr = static_cast<uint32_t>(4294967295.0 * ratio);
  dropout_kernel<<<grid_for(n8, 256), 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const bf16x8*>(x.data_ptr()), reinterpret_cast<bf16x8*>(y.data_ptr()), n8,
      static_cast<uint32_t>(seed), static_cast<uint32_t>(static_cast<uint64_t>(seed) >> 32), thr,
      static_cast<float>(1.0 / (1.0 - ratio)),
      seed_dev.has_value() ? reinterpret_cast<const long long*>(seed_dev->data_ptr<int64_t>()) : nullptr);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return y;
}

// ------------------------------------------------------------------ bias gradient: out[c] (+)= sum_rows dy[row, c]
// Pass 1: block (x, y) sums the rows of split y for 64 columns into part[y][c]; pass 2 adds the splits onto out in split
// order (no atomics: the sum does not depend on which block finishes first).
__global__ void __launch_bounds__(256)
colsum_kernel(const __nv_bfloat16* __restrict__ dy, long ld, long rows, int C, float* __restrict__ part) {
  // blockDim = (8 vec-columns, 32 row lanes); grid = (ceil(C/64), row splits)
  __shared__ float red[32][65];
  const int v = threadIdx.x, ry = threadIdx.y;
  const int c0 = blockIdx.x * 64 + v * 8;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (c0 < C) {
    for (long r = static_cast<long>(blockIdx.y) * 32 + ry; r < rows; r += static_cast<long>(gridDim.y) * 32) {
      float f[8];
      unpack8(ld8(dy + r * ld + c0), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[ry][v * 8 + j] = acc[j];
  __syncthreads();
  const int t = ry * 8 + v;
  if (t < 64) {
    float s = 0.f;
#pragma unroll 8
    for (int r = 0; r < 32; ++r) s += red[r][t];
    const int c = blockIdx.x * 64 + t;
    if (c < C) part[static_cast<long>(blockIdx.y) * C + c] = s;
  }
}

__global__ void __launch_bounds__(256)
colsum_finish_kernel(const float* __restrict__ part, int splits, int C, float* __restrict__ out, float alpha, int accumulate) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int y = 0; y < splits; ++y) s += part[static_cast<long>(y) * C + c];
  out[c] = (accumulate ? out[c] : 0.f) + s * alpha;
}

// dy viewed as [rows, C] with row pitch ld (C % 8 == 0); out fp32 [C] (zeroed unless accumulate).
void colsum(const at::Tensor& dy, int64_t rows, int64_t C, int64_t ld, at::Tensor out, double alpha, bool accumulate) {
  TORCH_CHECK(dy.is_cuda() && dy.scalar_type() == at::kBFloat16 && out.scalar_type() == at::kFloat && out.numel() == C);
  TORCH_CHECK(C % 8 == 0 && ld % 8 == 0, "colsum: C and pitch must be multiples of 8");
  c10::cuda::CUDAGuard guard(dy.device());
  auto stream = at::cuda::getCurrentCUDAStream();
  dim3 block(8, 32);
  const int gx = (C + 63) / 64;
  const int gy = static_cast<int>(std::max<long>(1, std::min<long>((rows + 255) / 256, std::max(1, 592 / gx))));
  at::Tensor part = at::empty({gy, C}, out.options());
  colsum_kernel<<<dim3(gx, gy), block, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr()), ld, rows, C,
                                                    part.data_ptr<float>());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  colsum_finish_kernel<<<(C + 255) / 256, 256, 0, stream>>>(part.data_ptr<float>(), gy, C, out.data_ptr<float>(),
                                                            static_cast<float>(alpha), accumulate ? 1 : 0);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

}  // namespace psd

TORCH_LIBRARY_FRAGMENT(poseidon, m) {
  m.def("transform_nhwc(Tensor x, Tensor h_off, Tensor w_off, Tensor flip, Tensor? mean, float scale, int OH, int OW, "
        "int cp, int opad, int wextra, int hextra, bool s2d) -> Tensor", &psd::transform_nhwc);
  m.def("relu_fwd(Tensor x, float slope) -> Tensor", &psd::relu_fwd);
  m.def("relu_bwd(Tensor y, Tensor dy, float slope) -> Tensor", &psd::relu_bwd);
  m.def("relu_bwd_nhwc(Tensor y, Tensor dy, float slope) -> Tensor", &psd::relu_bwd_nhwc);
  m.def("dropout_apply(Tensor x, float ratio, int seed, Tensor? seed_dev) -> Tensor", &psd::dropout_apply);
  m.def("colsum(Tensor dy, int rows, int C, int ld, Tensor(a!) out, float alpha, bool accumulate) -> ()", &psd::colsum);
}
