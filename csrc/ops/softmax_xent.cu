// Fused softmax + multinomial-logistic loss + gradient, one CTA per row, everything stays on the GPU.
//
//   prob = softmax(x[row, :]);  loss += -log(max(prob[label], FLT_MIN)) / rows
//   dx[row, c] = (prob[c] - [c == label]) * grad_scale / rows          (bf16, written in the same pass)
//
// The reference's SoftmaxWithLoss GPU path calls the CPU implementation, forcing a D2H of the logits
// and an H2D of the gradient every iteration (src/caffe/layers/softmax_loss_layer.cu:11-22,
// softmax_loss_layer.cpp:38-87); the standalone softmax is 5 kernels (softmax_layer.cu:14-149).
#include "nhwc_common.cuh"

namespace psd {

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffff, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffff, v, o);
  return v;
}

template <typename T>
__device__ __forceinline__ float to_f(T v);
template <>
__device__ __forceinline__ float to_f<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T>
__global__ void __launch_bounds__(256)
softmax_xent_kernel(const T* __restrict__ x, long ldx, const float* __restrict__ label, T* __restrict__ dx, long lddx,
                    float* __restrict__ prob, float* __restrict__ row_loss, int rows, int C, float grad_scale) {
  __shared__ float red[8];
  __shared__ float bc;
  const int row = blockIdx.x;
  const T* xr = x + static_cast<long>(row) * ldx;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  float m = -3.402823466e38f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) m = fmaxf(m, to_f(xr[c]));
  m = warp_max(m);
  if (lane == 0) red[warp] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = red[0];
    for (int i = 1; i < nw; ++i) t = fmaxf(t, red[i]);
    bc = t;
  }
  __syncthreads();
  m = bc;
  float s = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) s += __expf(to_f(xr[c]) - m);
  s = warp_sum(s);
  __syncthreads();
  if (lane == 0) red[warp] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < nw; ++i) t += red[i];
    bc = t;
  }
  __syncthreads();
  const float inv = 1.f / bc;
  const int lab = static_cast<int>(label[row]);
  const float gs = grad_scale / static_cast<float>(rows);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float p = __expf(to_f(xr[c]) - m) * inv;
    if (prob != nullptr) prob[static_cast<long>(row) * C + c] = p;
    if (dx != nullptr) {
      const float g = (p - (c == lab ? 1.f : 0.f)) * gs;
      if constexpr (sizeof(T) == 2) dx[static_cast<long>(row) * lddx + c] = __float2bfloat16(g);
      else dx[static_cast<long>(row) * lddx + c] = g;
    }
    if (c == lab) row_loss[row] = -__logf(fmaxf(p, 1.17549435e-38f));
  }
}

// loss = mean of the per-row losses, summed in a fixed order (strided per thread, then a fixed tree): no atomics, so the
// loss is the same in every run.
__global__ void __launch_bounds__(256)
mean_rows_kernel(const float* __restrict__ row_loss, int rows, float* __restrict__ loss) {
  __shared__ float red[256];
  float s = 0.f;
  for (int r = threadIdx.x; r < rows; r += blockDim.x) s += row_loss[r];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = blockDim.x / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] = red[0] / static_cast<float>(rows);
}

// x: [rows, C] (bf16 or fp32), label: [rows] fp32 class ids.  Returns (loss[1] fp32, dx like x, prob fp32 or empty).
std::tuple<at::Tensor, at::Tensor, at::Tensor> softmax_xent(const at::Tensor& x, const at::Tensor& label, double grad_scale,
                                                            bool want_grad, bool want_prob) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.stride(1) == 1);
  TORCH_CHECK(label.scalar_type() == at::kFloat && label.numel() == x.size(0) && label.is_contiguous());
  c10::cuda::CUDAGuard guard(x.device());
  const int rows = x.size(0), C = x.size(1);
  at::Tensor loss = at::empty({1}, x.options().dtype(at::kFloat));
  at::Tensor row_loss = at::zeros({rows}, x.options().dtype(at::kFloat));   // rows whose label is out of range add 0
  at::Tensor dx = want_grad ? at::empty({rows, C}, x.options()) : at::Tensor();
  at::Tensor prob = want_prob ? at::empty({rows, C}, x.options().dtype(at::kFloat)) : at::Tensor();
  auto stream = at::cuda::getCurrentCUDAStream();
  float* pp = want_prob ? prob.data_ptr<float>() : nullptr;
  if (x.scalar_type() == at::kBFloat16) {
    softmax_xent_kernel<__nv_bfloat16><<<rows, 256, 0, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(x.data_ptr()), x.stride(0), label.data_ptr<float>(),
        want_grad ? reinterpret_cast<__nv_bfloat16*>(dx.data_ptr()) : nullptr, C, pp, row_loss.data_ptr<float>(), rows, C,
        static_cast<float>(grad_scale));
  } else {
    TORCH_CHECK(x.scalar_type() == at::kFloat, "softmax_xent: bf16 or fp32 logits");
    softmax_xent_kernel<float><<<rows, 256, 0, stream>>>(x.data_ptr<float>(), x.stride(0), label.data_ptr<float>(),
                                                         want_grad ? dx.data_ptr<float>() : nullptr, C, pp,
                                                         row_loss.data_ptr<float>(), rows, C, static_cast<float>(grad_scale));
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  mean_rows_kernel<<<1, 256, 0, stream>>>(row_loss.data_ptr<float>(), rows, loss.data_ptr<float>());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return {loss, want_grad ? dx : at::empty({0}, x.options()), want_prob ? prob : at::empty({0}, x.options())};
}

}  // namespace psd

TORCH_LIBRARY_FRAGMENT(poseidon, m) {
  m.def("softmax_xent(Tensor x, Tensor label, float grad_scale, bool want_grad, bool want_prob) -> (Tensor, Tensor, Tensor)",
        &psd::softmax_xent);
}
