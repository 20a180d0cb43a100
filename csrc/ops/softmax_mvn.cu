// Softmax (over channels) and MVN (mean-variance normalisation) of the sm100 engine: bf16 storage, fp32 math.
//
// Softmax: Caffe normalises over the channel axis at every (n, h, w) position (src/caffe/layers/softmax_layer.cu:14-149).
// With NHWC memory that is a row softmax over C contiguous values — one warp per row, the row held in registers.
//   forward   y = exp(x - max) / sum           backward   dx = y * (dy - sum(dy * y))
//
// MVN: per (n, c) plane — or per image with across_channels — subtract the mean and (optionally) divide by
// (sqrt(var) + eps), eps = 1e-10 (src/caffe/layers/mvn_layer.cu:15-135).  Three launches: per-(n, c) partial sums
// (coalesced over channels), a tiny finishing kernel that turns them into mean / 1/(std+eps) for either grouping, and an
// elementwise apply.  Backward uses the same reduction on (dy, dy*y):
//   normalize_variance:  dx = (dy - mean(dy) - y * mean(dy * y)) / (std + eps)      else  dx = dy - mean(dy)
#include "nhwc_common.cuh"

namespace psd {

constexpr int kSoftmaxMaxPerLane = 32;      // rows up to 32 * 32 = 1024 channels stay in registers

// rows x C, row r starts at r * ld.  One warp per row (grid-stride).
template <bool BWD>
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ b, __nv_bfloat16* __restrict__ out,
                    long rows, int C, long ld_a, long ld_b, long ld_o) {
  const int lane = threadIdx.x & 31;
  const long warp = (blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x) >> 5;
  const long nwarps = (static_cast<long>(gridDim.x) * blockDim.x) >> 5;
  for (long r = warp; r < rows; r += nwarps) {
    const __nv_bfloat16* ap = a + r * ld_a;
    float v[kSoftmaxMaxPerLane], w[kSoftmaxMaxPerLane];
    if constexpr (!BWD) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < kSoftmaxMaxPerLane; ++i) {
        const int c = lane + 32 * i;
        v[i] = c < C ? __bfloat162float(ap[c]) : -INFINITY;
        mx = fmaxf(mx, v[i]);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < kSoftmaxMaxPerLane; ++i) {
        v[i] = (lane + 32 * i) < C ? __expf(v[i] - mx) : 0.f;
        sum += v[i];
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      const float inv = 1.f / sum;
#pragma unroll
      for (int i = 0; i < kSoftmaxMaxPerLane; ++i) {
        const int c = lane + 32 * i;
        if (c < C) out[r * ld_o + c] = __float2bfloat16(v[i] * inv);
      }
    } else {
      // a = y, b = dy
      const __nv_bfloat16* bp = b + r * ld_b;
      float dot = 0.f;
#pragma unroll
      for (int i = 0; i < kSoftmaxMaxPerLane; ++i) {
        const int c = lane + 32 * i;
        v[i] = c < C ? __bfloat162float(ap[c]) : 0.f;
        w[i] = c < C ? __bfloat162float(bp[c]) : 0.f;
        dot += v[i] * w[i];
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
#pragma unroll
      for (int i = 0; i < kSoftmaxMaxPerLane; ++i) {
        const int c = lane + 32 * i;
        if (c < C) out[r * ld_o + c] = __float2bfloat16(v[i] * (w[i] - dot));
      }
    }
  }
}

// Rows of any length (C > 1024): one block per row, three passes over global memory.
template <bool BWD>
__global__ void __launch_bounds__(256)
softmax_long_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ b, __nv_bfloat16* __restrict__ out,
                    long rows, int C, long ld_a, long ld_b, long ld_o) {
  __shared__ float red[32];
  auto block_reduce = [&](float v, bool is_max) -> float {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float t = __shfl_xor_sync(0xffffffffu, v, o);
      v = is_max ? fmaxf(v, t) : v + t;
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = is_max ? -INFINITY : 0.f;
    for (int i = 0; i < static_cast<int>(blockDim.x >> 5); ++i) r = is_max ? fmaxf(r, red[i]) : r + red[i];
    return r;
  };
  for (long r = blockIdx.x; r < rows; r += gridDim.x) {
    const __nv_bfloat16* ap = a + r * ld_a;
    if constexpr (!BWD) {
      float mx = -INFINITY;
      for (int c = threadIdx.x; c < C; c += blockDim.x) mx = fmaxf(mx, __bfloat162float(ap[c]));
      mx = block_reduce(mx, true);
      float sum = 0.f;
      for (int c = threadIdx.x; c < C; c += blockDim.x) sum += __expf(__bfloat162float(ap[c]) - mx);
      sum = block_reduce(sum, false);
      const float inv = 1.f / sum;
      for (int c = threadIdx.x; c < C; c += blockDim.x) out[r * ld_o + c] = __float2bfloat16(__expf(__bfloat162float(ap[c]) - mx) * inv);
    } else {
      const __nv_bfloat16* bp = b + r * ld_b;
      float dot = 0.f;
      for (int c = threadIdx.x; c < C; c += blockDim.x) dot += __bfloat162float(ap[c]) * __bfloat162float(bp[c]);
      dot = block_reduce(dot, false);
      for (int c = threadIdx.x; c < C; c += blockDim.x)
        out[r * ld_o + c] = __float2bfloat16(__bfloat162float(ap[c]) * (__bfloat162float(bp[c]) - dot));
    }
  }
}

struct RowsView {
  long rows, ld;
  int C;
};
// (N, C) row-major or (N, C, H, W) channels-last (pixel pitch >= C): rows of C contiguous values.
static RowsView rows_view(const at::Tensor& t, const char* what) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kBFloat16, what, ": bf16 CUDA tensor expected");
  RowsView v;
  if (t.dim() == 2) {
    TORCH_CHECK(t.stride(1) == 1, what, ": rows must be contiguous");
    v.rows = t.size(0); v.C = static_cast<int>(t.size(1)); v.ld = t.stride(0);
  } else {
    NhwcView n = nhwc_view(t);
    v.rows = static_cast<long>(n.N) * n.H * n.W; v.C = n.C; v.ld = n.pitch;
  }
  return v;
}

template <bool BWD>
static void launch_softmax(const at::Tensor& a, const at::Tensor* b, at::Tensor& out) {
  RowsView va = rows_view(a, "softmax"), vo = rows_view(out, "softmax");
  RowsView vb = b != nullptr ? rows_view(*b, "softmax") : va;
  TORCH_CHECK(va.rows == vo.rows && va.C == vo.C && vb.rows == va.rows && vb.C == va.C, "softmax: shape mismatch");
  auto st = at::cuda::getCurrentCUDAStream();
  auto* ap = reinterpret_cast<const __nv_bfloat16*>(a.data_ptr());
  auto* bp = b != nullptr ? reinterpret_cast<const __nv_bfloat16*>(b->data_ptr()) : nullptr;
  auto* op = reinterpret_cast<__nv_bfloat16*>(out.data_ptr());
  if (va.C <= 32 * kSoftmaxMaxPerLane) {
    const int grid = grid_for(va.rows * 32, 256);
    softmax_rows_kernel<BWD><<<grid, 256, 0, st>>>(ap, bp, op, va.rows, va.C, va.ld, vb.ld, vo.ld);
  } else {
    const int grid = static_cast<int>(std::min<long>(va.rows, 132L * 8));
    softmax_long_kernel<BWD><<<grid, 256, 0, st>>>(ap, bp, op, va.rows, va.C, va.ld, vb.ld, vo.ld);
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

at::Tensor softmax_fwd(const at::Tensor& x) {
  c10::cuda::CUDAGuard guard(x.device());
  at::Tensor y = at::empty_like(x);
  launch_softmax<false>(x, nullptr, y);
  return y;
}
at::Tensor softmax_bwd(const at::Tensor& y, const at::Tensor& dy) {
  c10::cuda::CUDAGuard guard(y.device());
  at::Tensor dx = at::empty_like(y);
  launch_softmax<true>(y, &dy, dx);
  return dx;
}

// ------------------------------------------------------------------------------------------------ MVN
// sums[n][c] = (sum_p a, sum_p a*b)   over the H*W pixels of plane (n, c);  b == nullptr: a*a.
// Block = 32 pixel lanes x 8 channel vectors (64 channels); grid = (ceil(C/64), N).
__global__ void __launch_bounds__(256)
plane_sums_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ b, float2* __restrict__ sums, int C,
                  int HW, long pitch_a, long pitch_b) {
  __shared__ float sm[2][8][32][8 + 1];
  const int cv = threadIdx.x & 7, pl = threadIdx.x >> 3;     // channel vector (8 channels), pixel lane
  const int c0 = (blockIdx.x * 8 + cv) * 8;
  const int n = blockIdx.y;
  float s1[8], s2[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) s1[k] = s2[k] = 0.f;
  if (c0 < C) {
    const __nv_bfloat16* ap = a + static_cast<long>(n) * HW * pitch_a + c0;
    const __nv_bfloat16* bp = b != nullptr ? b + static_cast<long>(n) * HW * pitch_b + c0 : nullptr;
    for (int p = pl; p < HW; p += 32) {
      float va[8], vb[8];
      unpack8(ld8(ap + p * pitch_a), va);
      if (bp != nullptr) unpack8(ld8(bp + p * pitch_b), vb);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        s1[k] += va[k];
        s2[k] += va[k] * (bp != nullptr ? vb[k] : va[k]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) { sm[0][cv][pl][k] = s1[k]; sm[1][cv][pl][k] = s2[k]; }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int v = threadIdx.x >> 3, k = threadIdx.x & 7;
    float t1 = 0.f, t2 = 0.f;
    for (int p = 0; p < 32; ++p) { t1 += sm[0][v][p][k]; t2 += sm[1][v][p][k]; }
    const int c = (blockIdx.x * 8 + v) * 8 + k;
    if (c < C) sums[static_cast<long>(n) * C + c] = make_float2(t1, t2);
  }
}

// stats[n][c] = (m1, m2): means of the two sums over the group (plane, or whole image with across_channels); for the
// forward m2 is turned into 1 / (sqrt(var) + eps) (or 1 without variance normalisation).
__global__ void mvn_finish_kernel(const float2* __restrict__ sums, float2* __restrict__ stats, int C, int HW, int across,
                                  int forward, int normalize_variance, float eps) {
  const int n = blockIdx.x;
  __shared__ float r1[256], r2[256];
  float g1 = 0.f, g2 = 0.f;
  if (across) {
    for (int c = threadIdx.x; c < C; c += blockDim.x) { const float2 s = sums[static_cast<long>(n) * C + c]; g1 += s.x; g2 += s.y; }
    r1[threadIdx.x] = g1; r2[threadIdx.x] = g2;
    __syncthreads();
    for (int o = blockDim.x >> 1; o > 0; o >>= 1) {
      if (threadIdx.x < o) { r1[threadIdx.x] += r1[threadIdx.x + o]; r2[threadIdx.x] += r2[threadIdx.x + o]; }
      __syncthreads();
    }
    g1 = r1[0]; g2 = r2[0];
  }
  const float cnt = across ? static_cast<float>(HW) * C : static_cast<float>(HW);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float2 s = sums[static_cast<long>(n) * C + c];
    if (across) s = make_float2(g1, g2);
    float m1 = s.x / cnt, m2 = s.y / cnt;
    if (forward) {
      const float var = fmaxf(m2 - m1 * m1, 0.f);
      m2 = normalize_variance ? 1.f / (sqrtf(var) + eps) : 1.f;
    }
    stats[static_cast<long>(n) * C + c] = make_float2(m1, m2);
  }
}

// forward:  y = (x - mean) * inv
// backward: dx = (dy - m1 - y * m2) * inv   (normalize_variance)   |   dx = dy - m1
__global__ void __launch_bounds__(256)
mvn_apply_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ out,
                 const float2* __restrict__ stats, const float2* __restrict__ fwd_stats, int C, int HW, long total8,
                 long pitch_a, long pitch_y, long pitch_o, int backward, int normalize_variance) {
  const int c8n = C >> 3;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total8; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long pix = i / c8n;
    const int c0 = static_cast<int>(i - pix * c8n) * 8;
    const long n = pix / HW;
    float va[8], vy[8], o[8];
    unpack8(ld8(a + pix * pitch_a + c0), va);
    if (backward && normalize_variance) unpack8(ld8(y + pix * pitch_y + c0), vy);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float2 s = stats[n * C + c0 + k];
      if (!backward) o[k] = (va[k] - s.x) * s.y;
      else if (normalize_variance) o[k] = (va[k] - s.x - vy[k] * s.y) * fwd_stats[n * C + c0 + k].y;
      else o[k] = va[k] - s.x;
    }
    st8(out + pix * pitch_o + c0, pack8(o));
  }
}

static void mvn_stats(const at::Tensor& a, const at::Tensor* b, at::Tensor& stats, bool across, bool forward, bool nv) {
  NhwcView va = nhwc_view(a);
  TORCH_CHECK(va.C % 8 == 0 && va.pitch % 8 == 0, "mvn: channels must be a multiple of 8");
  at::Tensor sums = at::empty({va.N, va.C, 2}, a.options().dtype(at::kFloat));
  auto st = at::cuda::getCurrentCUDAStream();
  dim3 grid((va.C + 63) / 64, va.N);
  long pb = 0;
  const __nv_bfloat16* bp = nullptr;
  if (b != nullptr) { NhwcView vb = nhwc_view(*b); pb = vb.pitch; bp = reinterpret_cast<const __nv_bfloat16*>(b->data_ptr()); }
  plane_sums_kernel<<<grid, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(a.data_ptr()), bp,
                                          reinterpret_cast<float2*>(sums.data_ptr<float>()), va.C, va.H * va.W, va.pitch, pb);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  mvn_finish_kernel<<<va.N, 256, 0, st>>>(reinterpret_cast<const float2*>(sums.data_ptr<float>()),
                                          reinterpret_cast<float2*>(stats.data_ptr<float>()), va.C, va.H * va.W, across ? 1 : 0,
                                          forward ? 1 : 0, nv ? 1 : 0, 1e-10f);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// returns (y, stats[N, C, 2] = mean, 1/(std+eps))
std::tuple<at::Tensor, at::Tensor> mvn_fwd(const at::Tensor& x, bool normalize_variance, bool across_channels) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16, "mvn_fwd: bf16 CUDA tensor expected");
  c10::cuda::CUDAGuard guard(x.device());
  NhwcView v = nhwc_view(x);
  at::Tensor stats = at::empty({v.N, v.C, 2}, x.options().dtype(at::kFloat));
  mvn_stats(x, nullptr, stats, across_channels, true, normalize_variance);
  at::Tensor y = empty_nhwc(v.N, v.C, v.H, v.W, x.options());
  const long total8 = static_cast<long>(v.N) * v.H * v.W * (v.C / 8);
  mvn_apply_kernel<<<grid_for(total8, 256), 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const __nv_bfloat16*>(x.data_ptr()), nullptr, reinterpret_cast<__nv_bfloat16*>(y.data_ptr()),
      reinterpret_cast<const float2*>(stats.data_ptr<float>()), nullptr, v.C, v.H * v.W, total8, v.pitch, 0, v.C, 0,
      normalize_variance ? 1 : 0);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return {y, stats};
}

at::Tensor mvn_bwd(const at::Tensor& y, const at::Tensor& dy, const at::Tensor& fwd_stats, bool normalize_variance,
                   bool across_channels) {
  TORCH_CHECK(y.is_cuda() && y.scalar_type() == at::kBFloat16 && dy.scalar_type() == at::kBFloat16);
  c10::cuda::CUDAGuard guard(y.device());
  NhwcView v = nhwc_view(dy), vy = nhwc_view(y);
  TORCH_CHECK(vy.N == v.N && vy.C == v.C && vy.H == v.H && vy.W == v.W, "mvn_bwd: shape mismatch");
  at::Tensor stats = at::empty({v.N, v.C, 2}, y.options().dtype(at::kFloat));
  mvn_stats(dy, &y, stats, across_channels, false, normalize_variance);       // (mean(dy), mean(dy * y))
  at::Tensor dx = empty_nhwc(v.N, v.C, v.H, v.W, y.options());
  const long total8 = static_cast<long>(v.N) * v.H * v.W * (v.C / 8);
  mvn_apply_kernel<<<grid_for(total8, 256), 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr()), reinterpret_cast<const __nv_bfloat16*>(y.data_ptr()),
      reinterpret_cast<__nv_bfloat16*>(dx.data_ptr()), reinterpret_cast<const float2*>(stats.data_ptr<float>()),
      reinterpret_cast<const float2*>(fwd_stats.data_ptr<float>()), v.C, v.H * v.W, total8, v.pitch, vy.pitch, v.C, 1,
      normalize_variance ? 1 : 0);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return dx;
}

}  // namespace psd

TORCH_LIBRARY_FRAGMENT(poseidon, m) {
  m.def("softmax_fwd(Tensor x) -> Tensor", &psd::softmax_fwd);
  m.def("softmax_bwd(Tensor y, Tensor dy) -> Tensor", &psd::softmax_bwd);
  m.def("mvn_fwd(Tensor x, bool normalize_variance, bool across_channels) -> (Tensor, Tensor)", &psd::mvn_fwd);
  m.def("mvn_bwd(Tensor y, Tensor dy, Tensor stats, bool normalize_variance, bool across_channels) -> Tensor", &psd::mvn_bwd);
}
