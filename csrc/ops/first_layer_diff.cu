// First-layer data gradient back to the logical blob: the inverse of the layouts the transform kernel writes for a
// first-layer convolution (elementwise.cu transform_nhwc), applied to that convolution's data gradient.
//
//   pad8 (8-channel pad):      dx[n, c, y, x] = src[n, c, y, x]                                    (c < C of the Cp channels)
//   ROW (spatially pre-padded): dx[n, c, y, x] = src[n, c, y + ph, x + pw]      (drops the border and the even-width column)
//   s2d (space-to-depth by 4): dx[n, c, y, x] = src[n, ((y+p)%4)*16 + ((x+p)%4)*4 + c, (y+p)/4, (x+p)/4]
//
// A pure gather (no arithmetic), so the result is exact.  The reference has no counterpart: its data layer writes the
// logical blob and conv_layer.cu computes that blob's diff directly.
#include "nhwc_common.cuh"

namespace psd {

// One thread per logical pixel (n, y, x): it reads the pixel's C channels from the NHWC source (contiguous, or one
// s2d slot of them) and writes them to C planes of the NCHW output, so neighbouring threads store neighbouring x.
template <typename TOut>
__global__ void __launch_bounds__(256)
first_layer_diff_kernel(const __nv_bfloat16* __restrict__ src, TOut* __restrict__ dx, int C, int H, int W, int ph, int pw,
                        long pitch, long row, long img, int s2d, FastDiv d_w, FastDiv d_h, uint32_t total) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const uint32_t t = fdiv(i, d_w);
    const int x = static_cast<int>(i - t * d_w.d);
    const uint32_t n = fdiv(t, d_h);
    const int y = static_cast<int>(t - n * d_h.d);
    int sy = y + ph, sx = x + pw, c0 = 0;
    if (s2d) {
      c0 = (sy & 3) * 16 + (sx & 3) * 4;
      sy >>= 2;
      sx >>= 2;
    }
    const __nv_bfloat16* s = src + n * img + sy * row + sx * pitch + c0;
    TOut* o = dx + (static_cast<long>(n) * C * H + y) * W + x;
    for (int c = 0; c < C; ++c) {
      const float v = __bfloat162float(s[c]);
      if constexpr (sizeof(TOut) == 4) {
        o[static_cast<long>(c) * H * W] = v;
      } else {
        o[static_cast<long>(c) * H * W] = __float2bfloat16_rn(v);     // exact: v came from a bf16
      }
    }
  }
}

// src: the first layer's data gradient, bf16 channels-last (pixel pitch may exceed the channel count: a channel slice of a
// padded scratch).  Returns [N, C, H, W] contiguous, float32 when out_float else bf16.
at::Tensor first_layer_diff(const at::Tensor& src, int64_t C, int64_t H, int64_t W, int64_t ph, int64_t pw, bool s2d,
                            bool out_float) {
  TORCH_CHECK(src.is_cuda() && src.scalar_type() == at::kBFloat16, "first_layer_diff: bf16 CUDA source expected");
  c10::cuda::CUDAGuard guard(src.device());
  const NhwcView v = nhwc_view(src);
  TORCH_CHECK(C >= 1 && H >= 1 && W >= 1 && ph >= 0 && pw >= 0, "first_layer_diff: bad logical geometry");
  if (s2d) {
    TORCH_CHECK(v.C == 64 && C <= 4 && ph == pw, "first_layer_diff: s2d source must have 64 channels, C <= 4, one pad");
    TORCH_CHECK((H - 1 + ph) / 4 < v.H && (W - 1 + pw) / 4 < v.W, "first_layer_diff: s2d source too small");
  } else {
    TORCH_CHECK(C <= v.C && H + ph <= v.H && W + pw <= v.W, "first_layer_diff: source smaller than the logical blob");
  }
  at::Tensor dx = at::empty({v.N, C, H, W}, src.options().dtype(out_float ? at::kFloat : at::kBFloat16));
  const long total = static_cast<long>(v.N) * H * W;
  TORCH_CHECK(total < (1L << 31), "first_layer_diff: batch too large for 32-bit indexing");
  if (total == 0) return dx;
  const FastDiv d_w = make_fastdiv(static_cast<uint32_t>(W)), d_h = make_fastdiv(static_cast<uint32_t>(H));
  auto stream = at::cuda::getCurrentCUDAStream();
  const auto* sp = reinterpret_cast<const __nv_bfloat16*>(src.data_ptr());
  if (out_float) {
    first_layer_diff_kernel<float><<<grid_for(total, 256, 132 * 32), 256, 0, stream>>>(
        sp, dx.data_ptr<float>(), C, H, W, ph, pw, v.pitch, v.row, v.img, s2d ? 1 : 0, d_w, d_h,
        static_cast<uint32_t>(total));
  } else {
    first_layer_diff_kernel<__nv_bfloat16><<<grid_for(total, 256, 132 * 32), 256, 0, stream>>>(
        sp, reinterpret_cast<__nv_bfloat16*>(dx.data_ptr()), C, H, W, ph, pw, v.pitch, v.row, v.img, s2d ? 1 : 0, d_w,
        d_h, static_cast<uint32_t>(total));
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return dx;
}

}  // namespace psd

TORCH_LIBRARY_FRAGMENT(poseidon, m) {
  m.def("first_layer_diff(Tensor src, int C, int H, int W, int ph, int pw, bool s2d, bool out_float) -> Tensor",
        &psd::first_layer_diff);
}
