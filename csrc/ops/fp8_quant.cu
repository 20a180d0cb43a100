// Per-tensor fp8 quantisation of the fp8 convolution operands (conv_fprop_fp8 / conv_dgrad_fp8 in gemm/conv_ops.cu).
//
//   fp8_quant_act    : bf16 NHWC activations (pixel pitch may exceed C: concat-slab slices) -> dense e4m3 NHWC whose pixel
//                      pitch is C rounded up to 16 bytes (the TMA stride rule); one scale for the whole tensor.
//   fp8_quant_weight : fp32 master weights, physically [Cout][R][S][Cg] -> [Cout][R*S*Cgk] e4m3 (slots >= Cg zero), one
//                      scale per output channel.  Reading the master (not the bf16 shadow) rounds once, and the result
//                      does not depend on when a shadow was last refreshed.
//   fp8_quant_grad   : bf16 NHWC dY (pitched) -> dense e5m2 NHWC, one scale for the whole tensor; optionally applies the
//                      layer's own ReLU backward first (mask = forward output y) and returns that masked bf16 dY.
//   fp8_quant_weight_dgrad : fp32 master -> e4m3 in conv_pack_dgrad's order, [groups*Cg][R*S*Cok] (input-channel rows,
//                      K = (tap, co), slots >= Cout_g zero), one scale per input channel: the input channel is the output
//                      column of the data gradient, so its scale factors out of the accumulation.
//
// Scaling is just in time: s = MAX / amax(|v|) (MAX = 448 for e4m3, 57344 for e5m2; 1 when amax == 0),
// q = cvt.rn.satfinite(v * s), and 1 / s is stored for the GEMM epilogue.  amax uses fmaxf, which skips NaN, so a NaN
// element stays NaN after the multiply and the cast (satfinite keeps NaN); an infinite element makes s = 0 and comes out
// NaN.  Max is order-independent and the partial maxima are reduced by the cast kernel, so results are identical bit for
// bit from run to run, with no host sync.
#include <cfloat>
#include <type_traits>

#include "nhwc_common.cuh"

namespace psd {

constexpr int kQuantThreads = 256;
constexpr int kAmaxMaxBlocks = 264;      // 2 waves of 132 SMs; the cast kernel reduces these partials

__device__ __forceinline__ float block_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();                                   // red may still be read by a previous call
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = lane < static_cast<int>(blockDim.x >> 5) ? red[lane] : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// fp8 formats: the largest finite value sets the scale
struct E4M3 { static constexpr float kMax = 448.f; };
struct E5M2 { static constexpr float kMax = 57344.f; };

template <typename F>
__device__ __forceinline__ float quant_scale(float amax) {
  return amax > 0.f ? fminf(F::kMax / amax, FLT_MAX) : 1.f;
}

// two floats -> two fp8 bytes, `lo` at the lower address
template <typename F>
__device__ __forceinline__ uint32_t cvt_fp8x2(float lo, float hi) {
  uint16_t r;
  if constexpr (std::is_same<F, E5M2>::value) asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  else asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}

__global__ void __launch_bounds__(kQuantThreads) amax_nhwc_kernel(const __nv_bfloat16* __restrict__ x, long pixels, int C,
                                                                  long pitch, float* __restrict__ partial) {
  __shared__ float red[kQuantThreads / 32];
  const int vpp = C / 8;
  const long items = pixels * vpp;
  float m = 0.f;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < items; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long px = i / vpp;
    const int v = static_cast<int>(i - px * vpp);
    float f[8];
    unpack8(ld8(x + px * pitch + v * 8), f);
#pragma unroll
    for (int k = 0; k < 8; ++k) m = fmaxf(m, fabsf(f[k]));
  }
  m = block_max(m, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = m;
}

template <typename F>
__global__ void __launch_bounds__(kQuantThreads) cast_fp8_nhwc_kernel(const __nv_bfloat16* __restrict__ x, long pixels, int C,
                                                                      long pitch, int pitch8, const float* __restrict__ partial,
                                                                      int nparts, uint8_t* __restrict__ y,
                                                                      float* __restrict__ s_x) {
  __shared__ float red[kQuantThreads / 32];
  float m = 0.f;
  for (int i = threadIdx.x; i < nparts; i += blockDim.x) m = fmaxf(m, partial[i]);
  const float s = quant_scale<F>(block_max(m, red));
  if (blockIdx.x == 0 && threadIdx.x == 0) *s_x = 1.f / s;
  const int cpp = pitch8 / 16;                       // 16-byte output chunks per pixel
  const long items = pixels * cpp;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < items; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long px = i / cpp;
    const int c0 = static_cast<int>(i - px * cpp) * 16;
    float a[8], b[8];
    unpack8(ld8(x + px * pitch + c0), a);            // c0 < C: pitch8 is C rounded up to 16
    if (c0 + 8 < C) {
      unpack8(ld8(x + px * pitch + c0 + 8), b);
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) b[k] = 0.f;        // pad channels (C % 16 == 8)
    }
    uint4 q;
    q.x = cvt_fp8x2<F>(a[0] * s, a[1] * s) | (cvt_fp8x2<F>(a[2] * s, a[3] * s) << 16);
    q.y = cvt_fp8x2<F>(a[4] * s, a[5] * s) | (cvt_fp8x2<F>(a[6] * s, a[7] * s) << 16);
    q.z = cvt_fp8x2<F>(b[0] * s, b[1] * s) | (cvt_fp8x2<F>(b[2] * s, b[3] * s) << 16);
    q.w = cvt_fp8x2<F>(b[4] * s, b[5] * s) | (cvt_fp8x2<F>(b[6] * s, b[7] * s) << 16);
    *reinterpret_cast<uint4*>(y + px * pitch8 + c0) = q;
  }
}

// One CTA per output channel: amax over its R*S*Cg weights, then the padded e4m3 row.
__global__ void __launch_bounds__(kQuantThreads) quant_weight_kernel(const float* __restrict__ w, int RS, int Cg, int Cgk,
                                                                     uint8_t* __restrict__ w8, float* __restrict__ s_w) {
  __shared__ float red[kQuantThreads / 32];
  const int co = blockIdx.x;
  const float* row = w + static_cast<long>(co) * RS * Cg;
  const int n = RS * Cg;
  float m = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(row[i]));
  const float s = quant_scale<E4M3>(block_max(m, red));
  if (threadIdx.x == 0) s_w[co] = 1.f / s;
  uint8_t* out = w8 + static_cast<long>(co) * RS * Cgk;
  const int pairs = RS * Cgk / 2;
  for (int j = threadIdx.x; j < pairs; j += blockDim.x) {
    const int k = 2 * j;
    const int tap = k / Cgk, c = k - tap * Cgk;      // Cg and Cgk are even: a pair never straddles the pad boundary
    const float v0 = c < Cg ? row[tap * Cg + c] * s : 0.f;
    const float v1 = c < Cg ? row[tap * Cg + c + 1] * s : 0.f;
    *reinterpret_cast<uint16_t*>(out + k) = static_cast<uint16_t>(cvt_fp8x2<E4M3>(v0, v1));
  }
}

// x: bf16 NHWC (logical [N, C, H, W], channels-last, pixel pitch >= C); s_x_out: one float, receives 1 / s.
// Returns e4m3 [N, C, H, W] as a channel slice of a channels-last [N, round16(C), H, W] tensor (pad channels zero).
at::Tensor fp8_quant_act(const at::Tensor& x, at::Tensor s_x_out) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16, "fp8_quant_act: bf16 CUDA input expected");
  TORCH_CHECK(s_x_out.is_cuda() && s_x_out.scalar_type() == at::kFloat && s_x_out.numel() == 1 && s_x_out.is_contiguous(),
              "fp8_quant_act: s_x_out must be one fp32 element");
  c10::cuda::CUDAGuard guard(x.device());
  const NhwcView xv = nhwc_view(x);
  TORCH_CHECK(xv.C % 8 == 0 && xv.pitch % 8 == 0 && (reinterpret_cast<uintptr_t>(x.data_ptr()) & 15) == 0,
              "fp8_quant_act: channels and pixel pitch must be multiples of 8 (16-byte vectors)");
  const int pitch8 = (xv.C + 15) / 16 * 16;
  at::Tensor full = empty_nhwc(xv.N, pitch8, xv.H, xv.W, x.options().dtype(at::kFloat8_e4m3fn));
  const long pixels = static_cast<long>(xv.N) * xv.H * xv.W;
  auto stream = at::cuda::getCurrentCUDAStream();
  const int blocks = grid_for(pixels * (xv.C / 8), kQuantThreads, kAmaxMaxBlocks);
  at::Tensor partial = at::empty({blocks}, x.options().dtype(at::kFloat));
  const auto* xp = reinterpret_cast<const __nv_bfloat16*>(x.data_ptr());
  amax_nhwc_kernel<<<blocks, kQuantThreads, 0, stream>>>(xp, pixels, xv.C, xv.pitch, partial.data_ptr<float>());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  cast_fp8_nhwc_kernel<E4M3><<<grid_for(pixels * (pitch8 / 16), kQuantThreads), kQuantThreads, 0, stream>>>(
      xp, pixels, xv.C, xv.pitch, pitch8, partial.data_ptr<float>(), blocks,
      reinterpret_cast<uint8_t*>(full.data_ptr()), s_x_out.data_ptr<float>());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return full.narrow(1, 0, xv.C);
}

// w: fp32 master, logical [Cout, Cg, R, S] stored channels-last (physically [Cout][R][S][Cg]); cgk: per-tap slots of the
// result (>= Cg, even); s_w_out: [Cout] floats, receives 1 / s per output channel.  Returns [Cout, R*S*cgk] e4m3.
at::Tensor fp8_quant_weight(const at::Tensor& w, int64_t cgk, at::Tensor s_w_out) {
  TORCH_CHECK(w.is_cuda() && w.scalar_type() == at::kFloat && w.dim() == 4 &&
              w.is_contiguous(at::MemoryFormat::ChannelsLast), "fp8_quant_weight: fp32 channels-last [Cout, Cg, R, S] master expected");
  const int64_t Cout = w.size(0), Cg = w.size(1), RS = w.size(2) * w.size(3);
  TORCH_CHECK(cgk >= Cg && cgk % 2 == 0 && Cg % 2 == 0, "fp8_quant_weight: cgk must be even and >= Cg");
  TORCH_CHECK(s_w_out.is_cuda() && s_w_out.scalar_type() == at::kFloat && s_w_out.numel() == Cout && s_w_out.is_contiguous(),
              "fp8_quant_weight: s_w_out must hold Cout fp32 elements");
  TORCH_CHECK(RS * cgk < (1L << 31) && RS * Cg < (1L << 31), "fp8_quant_weight: row too long");
  c10::cuda::CUDAGuard guard(w.device());
  at::Tensor w8 = at::empty({Cout, RS * cgk}, w.options().dtype(at::kFloat8_e4m3fn));
  if (Cout == 0) return w8;
  quant_weight_kernel<<<static_cast<unsigned>(Cout), kQuantThreads, 0, at::cuda::getCurrentCUDAStream()>>>(
      w.data_ptr<float>(), static_cast<int>(RS), static_cast<int>(Cg), static_cast<int>(cgk),
      reinterpret_cast<uint8_t*>(w8.data_ptr()), s_w_out.data_ptr<float>());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return w8;
}

// amax pass of fp8_quant_grad with the layer's own ReLU backward fused in: d = y > 0 ? dy : dy * slope (relu_bwd's
// formula, so the masked tensor is the same bits), written dense (pixel pitch C); the partial maxima are those of d.
__global__ void __launch_bounds__(kQuantThreads) mask_amax_nhwc_kernel(const __nv_bfloat16* __restrict__ dy, long pitch_dy,
                                                                       const __nv_bfloat16* __restrict__ y, long pitch_y,
                                                                       float slope, long pixels, int C,
                                                                       __nv_bfloat16* __restrict__ out,
                                                                       float* __restrict__ partial) {
  __shared__ float red[kQuantThreads / 32];
  const int vpp = C / 8;
  const long items = pixels * vpp;
  float m = 0.f;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < items; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long px = i / vpp;
    const int v = static_cast<int>(i - px * vpp);
    float f[8], d[8];
    unpack8(ld8(y + px * pitch_y + v * 8), f);
    unpack8(ld8(dy + px * pitch_dy + v * 8), d);
#pragma unroll
    for (int k = 0; k < 8; ++k) d[k] = f[k] > 0.f ? d[k] : d[k] * slope;
    const bf16x8 q = pack8(d);
    st8(out + px * C + v * 8, q);
    unpack8(q, d);                                    // the maximum of what the cast pass reads back
#pragma unroll
    for (int k = 0; k < 8; ++k) m = fmaxf(m, fabsf(d[k]));
  }
  m = block_max(m, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = m;
}

// One CTA per input-channel row of the data-gradient operand: amax over the R*S*Cout_g weights that feed input channel ci
// of group g, then the padded e4m3 row (tap, co) with Cok slots per tap.
__global__ void __launch_bounds__(kQuantThreads) quant_weight_dgrad_kernel(const float* __restrict__ w, int RS, int Cg,
                                                                           int Cout_g, int Cok, uint8_t* __restrict__ w8,
                                                                           float* __restrict__ s_w) {
  __shared__ float red[kQuantThreads / 32];
  const int row = blockIdx.x;                         // g * Cg + ci
  const int g = row / Cg, ci = row - g * Cg;
  const float* base = w + static_cast<long>(g) * Cout_g * RS * Cg + ci;      // + (co * RS + tap) * Cg
  const int n = RS * Cout_g;
  float m = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(base[static_cast<long>(i) * Cg]));
  const float s = quant_scale<E4M3>(block_max(m, red));
  if (threadIdx.x == 0) s_w[row] = 1.f / s;
  uint8_t* out = w8 + static_cast<long>(row) * RS * Cok;
  const int pairs = RS * Cok / 2;
  for (int j = threadIdx.x; j < pairs; j += blockDim.x) {
    const int k = 2 * j;
    const int tap = k / Cok, co = k - tap * Cok;      // Cout_g and Cok are even: a pair never straddles the pad boundary
    const float v0 = co < Cout_g ? base[(static_cast<long>(co) * RS + tap) * Cg] * s : 0.f;
    const float v1 = co < Cout_g ? base[(static_cast<long>(co + 1) * RS + tap) * Cg] * s : 0.f;
    *reinterpret_cast<uint16_t*>(out + k) = static_cast<uint16_t>(cvt_fp8x2<E4M3>(v0, v1));
  }
}

// dy: bf16 NHWC (logical [N, C, H, W], pixel pitch >= C); s_out: one float, receives 1 / s (s = 57344 / amax).
// y (optional): the layer's forward output (same logical shape, any pixel pitch): dY is first masked as relu_bwd does it.
// Returns (e5m2 [N, C, H, W] as a channel slice of a channels-last [N, round16(C), H, W] tensor, the bf16 dY the cast read:
// `dy` itself, or the masked dense copy).
std::tuple<at::Tensor, at::Tensor> fp8_quant_grad(const at::Tensor& dy, at::Tensor s_out, const c10::optional<at::Tensor>& y,
                                                  double slope) {
  TORCH_CHECK(dy.is_cuda() && dy.scalar_type() == at::kBFloat16, "fp8_quant_grad: bf16 CUDA dY expected");
  TORCH_CHECK(s_out.is_cuda() && s_out.scalar_type() == at::kFloat && s_out.numel() == 1 && s_out.is_contiguous(),
              "fp8_quant_grad: s_out must be one fp32 element");
  c10::cuda::CUDAGuard guard(dy.device());
  const NhwcView dv = nhwc_view(dy);
  TORCH_CHECK(dv.C % 8 == 0 && dv.pitch % 8 == 0 && (reinterpret_cast<uintptr_t>(dy.data_ptr()) & 15) == 0,
              "fp8_quant_grad: channels and pixel pitch must be multiples of 8 (16-byte vectors)");
  NhwcView yv{};
  if (y.has_value()) {
    TORCH_CHECK(y->is_cuda() && y->scalar_type() == at::kBFloat16, "fp8_quant_grad: bf16 CUDA mask y expected");
    yv = nhwc_view(*y);
    TORCH_CHECK(yv.N == dv.N && yv.C == dv.C && yv.H == dv.H && yv.W == dv.W && yv.pitch % 8 == 0 &&
                (reinterpret_cast<uintptr_t>(y->data_ptr()) & 15) == 0, "fp8_quant_grad: y must match dY (pitch a multiple of 8)");
  }
  const int pitch8 = (dv.C + 15) / 16 * 16;
  at::Tensor full = empty_nhwc(dv.N, pitch8, dv.H, dv.W, dy.options().dtype(at::kFloat8_e5m2));
  const long pixels = static_cast<long>(dv.N) * dv.H * dv.W;
  auto stream = at::cuda::getCurrentCUDAStream();
  const int blocks = grid_for(pixels * (dv.C / 8), kQuantThreads, kAmaxMaxBlocks);
  at::Tensor partial = at::empty({blocks}, dy.options().dtype(at::kFloat));
  at::Tensor src = dy;
  long src_pitch = dv.pitch;
  if (y.has_value()) {
    src = empty_nhwc(dv.N, dv.C, dv.H, dv.W, dy.options());
    src_pitch = dv.C;
    mask_amax_nhwc_kernel<<<blocks, kQuantThreads, 0, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr()), dv.pitch, reinterpret_cast<const __nv_bfloat16*>(y->data_ptr()),
        yv.pitch, static_cast<float>(slope), pixels, dv.C, reinterpret_cast<__nv_bfloat16*>(src.data_ptr()),
        partial.data_ptr<float>());
  } else {
    amax_nhwc_kernel<<<blocks, kQuantThreads, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr()), pixels,
                                                           dv.C, dv.pitch, partial.data_ptr<float>());
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  cast_fp8_nhwc_kernel<E5M2><<<grid_for(pixels * (pitch8 / 16), kQuantThreads), kQuantThreads, 0, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(src.data_ptr()), pixels, dv.C, src_pitch, pitch8, partial.data_ptr<float>(),
      blocks, reinterpret_cast<uint8_t*>(full.data_ptr()), s_out.data_ptr<float>());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return {full.narrow(1, 0, dv.C), src};
}

// w: fp32 master, logical [Cout, Cg, R, S] stored channels-last (physically [Cout][R][S][Cg]); groups: Cout = groups * Cout_g;
// cok: per-tap slots (>= Cout_g, even); s_out: [groups * Cg] floats, receives 1 / s per input channel.
// Returns [groups * Cg, R*S*cok] e4m3 in conv_pack_dgrad's order.
at::Tensor fp8_quant_weight_dgrad(const at::Tensor& w, int64_t groups, int64_t cok, at::Tensor s_out) {
  TORCH_CHECK(w.is_cuda() && w.scalar_type() == at::kFloat && w.dim() == 4 &&
              w.is_contiguous(at::MemoryFormat::ChannelsLast), "fp8_quant_weight_dgrad: fp32 channels-last [Cout, Cg, R, S] master expected");
  TORCH_CHECK(groups >= 1 && w.size(0) % groups == 0, "fp8_quant_weight_dgrad: Cout must be a multiple of groups");
  const int64_t Cout_g = w.size(0) / groups, Cg = w.size(1), RS = w.size(2) * w.size(3);
  TORCH_CHECK(cok >= Cout_g && cok % 2 == 0 && Cout_g % 2 == 0, "fp8_quant_weight_dgrad: cok must be even and >= Cout_g");
  TORCH_CHECK(s_out.is_cuda() && s_out.scalar_type() == at::kFloat && s_out.numel() == groups * Cg && s_out.is_contiguous(),
              "fp8_quant_weight_dgrad: s_out must hold groups * Cg fp32 elements");
  TORCH_CHECK(RS * cok < (1L << 31) && RS * Cout_g < (1L << 31) && w.numel() < (1L << 31), "fp8_quant_weight_dgrad: too large");
  c10::cuda::CUDAGuard guard(w.device());
  at::Tensor w8 = at::empty({groups * Cg, RS * cok}, w.options().dtype(at::kFloat8_e4m3fn));
  if (groups * Cg == 0) return w8;
  quant_weight_dgrad_kernel<<<static_cast<unsigned>(groups * Cg), kQuantThreads, 0, at::cuda::getCurrentCUDAStream()>>>(
      w.data_ptr<float>(), static_cast<int>(RS), static_cast<int>(Cg), static_cast<int>(Cout_g), static_cast<int>(cok),
      reinterpret_cast<uint8_t*>(w8.data_ptr()), s_out.data_ptr<float>());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return w8;
}

}  // namespace psd

TORCH_LIBRARY_FRAGMENT(poseidon, m) {
  m.def("fp8_quant_act(Tensor x, Tensor(a!) s_x_out) -> Tensor", &psd::fp8_quant_act);
  m.def("fp8_quant_weight(Tensor w, int cgk, Tensor(a!) s_w_out) -> Tensor", &psd::fp8_quant_weight);
  m.def("fp8_quant_grad(Tensor dy, Tensor(a!) s_out, Tensor? y, float slope) -> (Tensor, Tensor)", &psd::fp8_quant_grad);
  m.def("fp8_quant_weight_dgrad(Tensor w, int groups, int cok, Tensor(a!) s_out) -> Tensor", &psd::fp8_quant_weight_dgrad);
}
