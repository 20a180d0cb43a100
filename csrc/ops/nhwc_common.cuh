// Shared helpers for the NHWC bf16 layer kernels (8 channels = one 16-byte vector per access).
#pragma once
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <torch/library.h>
#include <torch/types.h>

#include "../gemm/fastdiv.cuh"

namespace psd {

struct alignas(16) bf16x8 {
  __nv_bfloat162 v[4];
};

__device__ __forceinline__ void unpack8(const bf16x8& p, float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(p.v[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ bf16x8 pack8(const float (&f)[8]) {
  bf16x8 p;
#pragma unroll
  for (int i = 0; i < 4; ++i) p.v[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return p;
}
// MUFU approximations (the layer kernels feed bf16 outputs; inputs here are >= 1, no denormal handling needed)
__device__ __forceinline__ float fast_lg2(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ bf16x8 ld8(const __nv_bfloat16* p) { return *reinterpret_cast<const bf16x8*>(p); }
__device__ __forceinline__ void st8(__nv_bfloat16* p, const bf16x8& v) { *reinterpret_cast<bf16x8*>(p) = v; }

// Logical NCHW tensor stored channels-last: returns (N, C, H, W) and the pixel pitch in elements.
struct NhwcView {
  int N, C, H, W;
  long pitch;     // elements between consecutive pixels (>= C; > C for channel-slice views)
  long img;       // elements between consecutive images
  long row;       // elements between consecutive rows
};

inline NhwcView nhwc_view(const at::Tensor& t) {
  TORCH_CHECK(t.dim() == 4, "expected a 4-D tensor");
  TORCH_CHECK(t.stride(1) == 1 || t.size(1) == 1, "expected channels-last (NHWC) memory layout");
  NhwcView v;
  v.N = t.size(0); v.C = t.size(1); v.H = t.size(2); v.W = t.size(3);
  v.pitch = v.W > 1 ? t.stride(3) : (v.H > 1 ? t.stride(2) : (v.N > 1 ? t.stride(0) : v.C));
  v.row = v.pitch * v.W;
  v.img = v.row * v.H;
  TORCH_CHECK(v.pitch >= v.C, "bad NHWC pixel pitch");
  if (v.H > 1 && v.W > 1) TORCH_CHECK(t.stride(2) == v.row, "NHWC tensor must be dense in H,W (pixel pitch only)");
  if (v.N > 1) TORCH_CHECK(t.stride(0) == v.img, "NHWC tensor must be dense in N (pixel pitch only)");
  return v;
}

inline at::Tensor empty_nhwc(int64_t n, int64_t c, int64_t h, int64_t w, const at::TensorOptions& opt) {
  return at::empty({n, c, h, w}, opt.memory_format(at::MemoryFormat::ChannelsLast));
}

inline int grid_for(long work, int block, int max_blocks = 132 * 16) {
  long g = (work + block - 1) / block;
  return static_cast<int>(std::max<long>(1, std::min<long>(g, max_blocks)));
}

}  // namespace psd
