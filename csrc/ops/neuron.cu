// Elementwise layer kernels of the sm100 engine: Sigmoid / TanH / AbsVal / BNLL / Power / Threshold (forward + backward)
// and Eltwise PROD / SUM / MAX over up to 8 bottoms.  bf16 in, bf16 out, fp32 math, 16-byte accesses, any dense layout
// (the tensors of one call share their strides, so the kernels walk storage order).
//
// reference semantics (file:line of the fp32 originals):
//   src/caffe/layers/sigmoid_layer.cu:10-55   y = 1/(1+e^-x)            dx = dy * y * (1 - y)
//   src/caffe/layers/tanh_layer.cu:13-55      y = tanh(x)               dx = dy * (1 - y^2)
//   src/caffe/layers/absval_layer.cu:11-36    y = |x|                   dx = dy * sign(x)
//   src/caffe/layers/bnll_layer.cu:13-57      y = x>0 ? x+log(1+e^-x) : log(1+e^x)    dx = dy * e/(e+1), e = exp(min(x, 50))
//   src/caffe/layers/power_layer.cu:13-87     y = (shift + scale*x)^power              dx = dy * power*scale*(shift+scale*x)^(power-1)
//   src/caffe/layers/threshold_layer.cu:11-30 y = x > t ? 1 : 0                        (no gradient)
//   src/caffe/layers/eltwise_layer.cu:11-90   PROD / SUM (coefficients) / MAX (arg-max mask for backward)
#include "nhwc_common.cuh"

namespace psd {

enum UnaryOp : int { U_SIGMOID = 0, U_TANH = 1, U_ABSVAL = 2, U_BNLL = 3, U_POWER = 4, U_THRESHOLD = 5 };

struct UnaryParams {
  float a, b, c;      // POWER: a = power, b = scale, c = shift ; THRESHOLD: a = threshold
};

template <int OP>
__device__ __forceinline__ float unary_fwd(float x, const UnaryParams& p) {
  if constexpr (OP == U_SIGMOID) return 1.f / (1.f + __expf(-x));
  if constexpr (OP == U_TANH) return tanhf(x);
  if constexpr (OP == U_ABSVAL) return fabsf(x);
  if constexpr (OP == U_BNLL) return x > 0.f ? x + log1pf(__expf(-x)) : log1pf(__expf(x));
  if constexpr (OP == U_POWER) {
    const float v = p.c + p.b * x;
    if (p.a == 1.f) return v;
    if (p.a == 2.f) return v * v;
    return powf(v, p.a);
  }
  if constexpr (OP == U_THRESHOLD) return x > p.a ? 1.f : 0.f;
  return x;
}

// `s` is the saved tensor of the backward: the OUTPUT y for sigmoid / tanh, the INPUT x for the others.
template <int OP>
__device__ __forceinline__ float unary_bwd(float s, float dy, const UnaryParams& p) {
  if constexpr (OP == U_SIGMOID) return dy * s * (1.f - s);
  if constexpr (OP == U_TANH) return dy * (1.f - s * s);
  if constexpr (OP == U_ABSVAL) return dy * (s > 0.f ? 1.f : (s < 0.f ? -1.f : 0.f));
  if constexpr (OP == U_BNLL) {
    const float e = __expf(fminf(s, 50.f));
    return dy * e / (e + 1.f);
  }
  if constexpr (OP == U_POWER) {
    if (p.a * p.b == 0.f) return dy * 0.f;      // power_layer.cu:42: powf(0, a - 1) would make 0 * inf = NaN
    if (p.a == 1.f) return dy * p.b;
    const float v = p.c + p.b * s;
    if (p.a == 2.f) return dy * 2.f * p.b * v;
    return dy * p.a * p.b * powf(v, p.a - 1.f);
  }
  return 0.f;
}

template <int OP, bool BWD>
__global__ void __launch_bounds__(256)
unary_kernel(const __nv_bfloat16* __restrict__ s, const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ out, long n,
             UnaryParams p) {
  const long n8 = n >> 3;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < n8; i += static_cast<long>(gridDim.x) * blockDim.x) {
    float a[8], g[8], o[8];
    unpack8(ld8(s + 8 * i), a);
    if constexpr (BWD) unpack8(ld8(dy + 8 * i), g);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = BWD ? unary_bwd<OP>(a[k], g[k], p) : unary_fwd<OP>(a[k], p);
    st8(out + 8 * i, pack8(o));
  }
  for (long i = (n8 << 3) + blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const float a = __bfloat162float(s[i]);
    out[i] = __float2bfloat16(BWD ? unary_bwd<OP>(a, __bfloat162float(dy[i]), p) : unary_fwd<OP>(a, p));
  }
}

static void check_dense_bf16(const at::Tensor& t, const char* what) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kBFloat16 && t.is_non_overlapping_and_dense(), what,
              ": dense bf16 CUDA tensor expected");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0, what, ": 16-byte aligned storage expected");
}

template <bool BWD>
static void launch_unary(int op, const __nv_bfloat16* s, const __nv_bfloat16* dy, __nv_bfloat16* out, long n, UnaryParams p,
                         cudaStream_t st) {
  const int grid = grid_for((n + 7) / 8, 256);
  switch (op) {
    case U_SIGMOID: unary_kernel<U_SIGMOID, BWD><<<grid, 256, 0, st>>>(s, dy, out, n, p); break;
    case U_TANH: unary_kernel<U_TANH, BWD><<<grid, 256, 0, st>>>(s, dy, out, n, p); break;
    case U_ABSVAL: unary_kernel<U_ABSVAL, BWD><<<grid, 256, 0, st>>>(s, dy, out, n, p); break;
    case U_BNLL: unary_kernel<U_BNLL, BWD><<<grid, 256, 0, st>>>(s, dy, out, n, p); break;
    case U_POWER: unary_kernel<U_POWER, BWD><<<grid, 256, 0, st>>>(s, dy, out, n, p); break;
    case U_THRESHOLD: unary_kernel<U_THRESHOLD, BWD><<<grid, 256, 0, st>>>(s, dy, out, n, p); break;
    default: TORCH_CHECK(false, "unknown unary op ", op);
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

at::Tensor unary_fwd_op(const at::Tensor& x, int64_t op, double a, double b, double c) {
  check_dense_bf16(x, "unary_fwd");
  c10::cuda::CUDAGuard guard(x.device());
  at::Tensor y = at::empty_like(x);
  launch_unary<false>(static_cast<int>(op), reinterpret_cast<const __nv_bfloat16*>(x.data_ptr()), nullptr,
                      reinterpret_cast<__nv_bfloat16*>(y.data_ptr()), x.numel(),
                      UnaryParams{static_cast<float>(a), static_cast<float>(b), static_cast<float>(c)},
                      at::cuda::getCurrentCUDAStream());
  return y;
}

at::Tensor unary_bwd_op(const at::Tensor& saved, const at::Tensor& dy, int64_t op, double a, double b, double c) {
  check_dense_bf16(saved, "unary_bwd");
  check_dense_bf16(dy, "unary_bwd");
  TORCH_CHECK(saved.sizes() == dy.sizes() && saved.strides() == dy.strides(), "unary_bwd: saved tensor and dy must share a layout");
  c10::cuda::CUDAGuard guard(dy.device());
  at::Tensor dx = at::empty_like(dy);
  launch_unary<true>(static_cast<int>(op), reinterpret_cast<const __nv_bfloat16*>(saved.data_ptr()),
                     reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr()), reinterpret_cast<__nv_bfloat16*>(dx.data_ptr()),
                     dy.numel(), UnaryParams{static_cast<float>(a), static_cast<float>(b), static_cast<float>(c)},
                     at::cuda::getCurrentCUDAStream());
  return dx;
}

// ------------------------------------------------------------------------------------------------ Eltwise
constexpr int kMaxEltwise = 8;
enum EltOp : int { E_PROD = 0, E_SUM = 1, E_MAX = 2 };

struct EltPtrs {
  const __nv_bfloat16* x[kMaxEltwise];
  __nv_bfloat16* dx[kMaxEltwise];
  float coeff[kMaxEltwise];
  int n;
};

template <int OP>
__global__ void __launch_bounds__(256)
eltwise_fwd_kernel(EltPtrs pp, __nv_bfloat16* __restrict__ y, uint8_t* __restrict__ mask, long n8) {
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < n8; i += static_cast<long>(gridDim.x) * blockDim.x) {
    float acc[8], v[8];
    unpack8(ld8(pp.x[0] + 8 * i), acc);
    alignas(8) uint8_t arg[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if constexpr (OP == E_SUM) {
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] *= pp.coeff[0];
    }
    for (int j = 1; j < pp.n; ++j) {
      unpack8(ld8(pp.x[j] + 8 * i), v);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        if constexpr (OP == E_PROD) acc[k] *= v[k];
        if constexpr (OP == E_SUM) acc[k] += pp.coeff[j] * v[k];
        if constexpr (OP == E_MAX) {
          if (v[k] > acc[k]) { acc[k] = v[k]; arg[k] = static_cast<uint8_t>(j); }     // ties keep the earlier bottom (reference)
        }
      }
    }
    st8(y + 8 * i, pack8(acc));
    if constexpr (OP == E_MAX) {
      if (mask != nullptr) *reinterpret_cast<uint2*>(mask + 8 * i) = *reinterpret_cast<const uint2*>(arg);
    }
  }
}

// dx_j = dy * prod_{k != j} x_k (PROD; the reference's stable form) | coeff_j * dy (SUM) | dy where the arg-max is j (MAX)
template <int OP>
__global__ void __launch_bounds__(256)
eltwise_bwd_kernel(EltPtrs pp, const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ mask, long n8) {
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < n8; i += static_cast<long>(gridDim.x) * blockDim.x) {
    float g[8];
    unpack8(ld8(dy + 8 * i), g);
    if constexpr (OP == E_PROD) {
      float xs[kMaxEltwise][8];
      for (int j = 0; j < pp.n; ++j) unpack8(ld8(pp.x[j] + 8 * i), xs[j]);
      for (int j = 0; j < pp.n; ++j) {
        if (pp.dx[j] == nullptr) continue;
        float o[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          float pr = g[k];
          for (int q = 0; q < pp.n; ++q)
            if (q != j) pr *= xs[q][k];
          o[k] = pr;
        }
        st8(pp.dx[j] + 8 * i, pack8(o));
      }
    } else {
      alignas(8) uint8_t arg[8];
      if constexpr (OP == E_MAX) *reinterpret_cast<uint2*>(arg) = *reinterpret_cast<const uint2*>(mask + 8 * i);
      for (int j = 0; j < pp.n; ++j) {
        if (pp.dx[j] == nullptr) continue;
        float o[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = OP == E_SUM ? pp.coeff[j] * g[k] : (arg[k] == j ? g[k] : 0.f);
        st8(pp.dx[j] + 8 * i, pack8(o));
      }
    }
  }
}

// xs: 2..8 dense bf16 tensors of one layout, numel % 8 == 0.  Returns (y, mask) — mask (uint8 arg-max) only for MAX.
std::tuple<at::Tensor, at::Tensor> eltwise_fwd(std::vector<at::Tensor> xs, int64_t op, std::vector<double> coeffs, bool want_mask) {
  const int n = static_cast<int>(xs.size());
  TORCH_CHECK(n >= 2 && n <= kMaxEltwise, "eltwise: 2..8 bottoms");
  c10::cuda::CUDAGuard guard(xs[0].device());
  EltPtrs pp{};
  pp.n = n;
  for (int j = 0; j < n; ++j) {
    check_dense_bf16(xs[j], "eltwise_fwd");
    TORCH_CHECK(xs[j].sizes() == xs[0].sizes() && xs[j].strides() == xs[0].strides(), "eltwise: bottoms must share a layout");
    pp.x[j] = reinterpret_cast<const __nv_bfloat16*>(xs[j].data_ptr());
    pp.coeff[j] = coeffs.empty() ? 1.f : static_cast<float>(coeffs[j]);
  }
  const long numel = xs[0].numel();
  TORCH_CHECK(numel % 8 == 0, "eltwise: element count must be a multiple of 8");
  at::Tensor y = at::empty_like(xs[0]);
  at::Tensor mask = at::empty({(op == E_MAX && want_mask) ? numel : 0L}, xs[0].options().dtype(at::kByte));
  auto st = at::cuda::getCurrentCUDAStream();
  const int grid = grid_for(numel / 8, 256);
  auto* yp = reinterpret_cast<__nv_bfloat16*>(y.data_ptr());
  uint8_t* mp = mask.numel() ? mask.data_ptr<uint8_t>() : nullptr;
  if (op == E_PROD) eltwise_fwd_kernel<E_PROD><<<grid, 256, 0, st>>>(pp, yp, mp, numel / 8);
  else if (op == E_SUM) eltwise_fwd_kernel<E_SUM><<<grid, 256, 0, st>>>(pp, yp, mp, numel / 8);
  else if (op == E_MAX) eltwise_fwd_kernel<E_MAX><<<grid, 256, 0, st>>>(pp, yp, mp, numel / 8);
  else TORCH_CHECK(false, "eltwise: unknown op ", op);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return {y, mask};
}

std::vector<at::Tensor> eltwise_bwd(std::vector<at::Tensor> xs, const at::Tensor& dy, const at::Tensor& mask, int64_t op,
                                    std::vector<double> coeffs, std::vector<int64_t> need) {
  const int n = static_cast<int>(xs.size());
  TORCH_CHECK(n >= 2 && n <= kMaxEltwise && static_cast<int>(need.size()) == n, "eltwise_bwd: 2..8 bottoms");
  check_dense_bf16(dy, "eltwise_bwd");
  c10::cuda::CUDAGuard guard(dy.device());
  EltPtrs pp{};
  pp.n = n;
  std::vector<at::Tensor> out(n);
  for (int j = 0; j < n; ++j) {
    check_dense_bf16(xs[j], "eltwise_bwd");
    TORCH_CHECK(xs[j].sizes() == dy.sizes() && xs[j].strides() == dy.strides(), "eltwise_bwd: layouts must match");
    pp.x[j] = reinterpret_cast<const __nv_bfloat16*>(xs[j].data_ptr());
    pp.coeff[j] = coeffs.empty() ? 1.f : static_cast<float>(coeffs[j]);
    if (need[j]) {
      out[j] = at::empty_like(dy);
      pp.dx[j] = reinterpret_cast<__nv_bfloat16*>(out[j].data_ptr());
    } else {
      out[j] = at::empty({0}, dy.options());
    }
  }
  const long numel = dy.numel();
  TORCH_CHECK(numel % 8 == 0, "eltwise: element count must be a multiple of 8");
  if (op == E_MAX) TORCH_CHECK(mask.numel() == numel && mask.scalar_type() == at::kByte, "eltwise_bwd: MAX needs the forward mask");
  auto st = at::cuda::getCurrentCUDAStream();
  const int grid = grid_for(numel / 8, 256);
  auto* gp = reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr());
  const uint8_t* mp = mask.numel() ? mask.data_ptr<uint8_t>() : nullptr;
  if (op == E_PROD) eltwise_bwd_kernel<E_PROD><<<grid, 256, 0, st>>>(pp, gp, mp, numel / 8);
  else if (op == E_SUM) eltwise_bwd_kernel<E_SUM><<<grid, 256, 0, st>>>(pp, gp, mp, numel / 8);
  else if (op == E_MAX) eltwise_bwd_kernel<E_MAX><<<grid, 256, 0, st>>>(pp, gp, mp, numel / 8);
  else TORCH_CHECK(false, "eltwise: unknown op ", op);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return out;
}

}  // namespace psd

TORCH_LIBRARY_FRAGMENT(poseidon, m) {
  m.def("unary_fwd(Tensor x, int op, float a, float b, float c) -> Tensor", &psd::unary_fwd_op);
  m.def("unary_bwd(Tensor saved, Tensor dy, int op, float a, float b, float c) -> Tensor", &psd::unary_bwd_op);
  m.def("eltwise_fwd(Tensor[] xs, int op, float[] coeffs, bool want_mask) -> (Tensor, Tensor)", &psd::eltwise_fwd);
  m.def("eltwise_bwd(Tensor[] xs, Tensor dy, Tensor mask, int op, float[] coeffs, int[] need) -> Tensor[]", &psd::eltwise_bwd);
}
