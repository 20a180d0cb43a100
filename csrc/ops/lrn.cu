// Across-channel local response normalisation, NHWC bf16, single pass fwd / single pass bwd.
//
//   scale_c = 1 + (alpha/n) * sum_{c' in [c-pre, c+n-1-pre]} x_c'^2 ,   y_c = x_c * scale_c^-beta
//   dx_c    = dy_c * scale_c^-beta - (2*alpha*beta/n) * x_c * sum_{c' window} dy_c' * y_c' / scale_c'
//
// In NHWC the channel window of a pixel is contiguous, so a CTA stages a strip of pixels in shared
// memory (fp32) and every thread produces 8 channels of one pixel with 16-byte global accesses.  The
// backward recomputes `scale` from x instead of storing it (the reference keeps a full `scale_` blob).
//
// reference: src/caffe/layers/lrn_layer.cu:10-53 (LRNFillScale), :73-78 (LRNComputeOutput), :119-177
// (LRNComputeDiff) — three kernels with one thread per (n,h,w) walking all channels.
#include "nhwc_common.cuh"

namespace psd {

constexpr int kLrnThreads = 256;

template <bool BWD>
__global__ void __launch_bounds__(kLrnThreads)
lrn_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ out,
           long npix, int C, long xpitch, long dpitch, long opitch, int size, float alpha_over_n, float beta,
           int pix_per_cta, int fuse_relu) {
  extern __shared__ float sm[];
  const int pre = (size - 1) / 2;
  const int post = size - 1 - pre;
  const int CP = C + size - 1;          // padded row: [pre zeros | C | post zeros]
  float* sx = sm;                        // x      [pix][CP]
  float* sr = sm + pix_per_cta * CP;     // bwd: r = dy * x * scale^(-beta-1)   [pix][CP]
  const int c8 = C / 8;
  for (long p0 = static_cast<long>(blockIdx.x) * pix_per_cta; p0 < npix; p0 += static_cast<long>(gridDim.x) * pix_per_cta) {
    const long rem = npix - p0;
    const int np = rem < pix_per_cta ? static_cast<int>(rem) : pix_per_cta;
    // stage x (optionally with a fused ReLU on the way in)
    for (int i = threadIdx.x; i < np * c8; i += blockDim.x) {
      const int p = i / c8, v = i - p * c8;
      float f[8];
      unpack8(ld8(x + (p0 + p) * xpitch + v * 8), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) sx[p * CP + pre + v * 8 + j] = fuse_relu ? fmaxf(f[j], 0.f) : f[j];
    }
    for (int i = threadIdx.x; i < np * (size - 1); i += blockDim.x) {
      const int p = i / (size - 1), k = i - p * (size - 1);
      const int idx = k < pre ? k : C + k;   // k>=pre -> pre + C + (k - pre)
      sx[p * CP + idx] = 0.f;
      if (BWD) sr[p * CP + idx] = 0.f;
    }
    __syncthreads();
    if constexpr (!BWD) {
      for (int i = threadIdx.x; i < np * c8; i += blockDim.x) {
        const int p = i / c8, v = i - p * c8;
        const float* row = sx + p * CP + v * 8;   // row[j + pre] is channel v*8+j
        float acc = 0.f;
#pragma unroll 4
        for (int k = 0; k < size - 1; ++k) acc += row[k] * row[k];
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float hi = row[j + size - 1];
          acc += hi * hi;
          const float scale = 1.f + alpha_over_n * acc;
          o[j] = row[j + pre] * exp2f(-beta * log2f(scale));
          acc -= row[j] * row[j];
        }
        st8(out + (p0 + p) * opitch + v * 8, pack8(o));
      }
    } else {
      // pass 1: r_c = dy_c * x_c * scale_c^(-beta-1)
      for (int i = threadIdx.x; i < np * c8; i += blockDim.x) {
        const int p = i / c8, v = i - p * c8;
        const float* row = sx + p * CP + v * 8;
        float d[8];
        unpack8(ld8(dy + (p0 + p) * dpitch + v * 8), d);
        float acc = 0.f;
#pragma unroll 4
        for (int k = 0; k < size - 1; ++k) acc += row[k] * row[k];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float hi = row[j + size - 1];
          acc += hi * hi;
          const float scale = 1.f + alpha_over_n * acc;
          sr[p * CP + pre + v * 8 + j] = d[j] * row[j + pre] * exp2f((-beta - 1.f) * log2f(scale));
          acc -= row[j] * row[j];
        }
      }
      __syncthreads();
      // pass 2: dx_c = dy_c * scale_c^-beta - 2*alpha*beta/n * x_c * sum_{c' : c in window(c')} r_c'
      const float cache_ratio = 2.f * alpha_over_n * beta;
      for (int i = threadIdx.x; i < np * c8; i += blockDim.x) {
        const int p = i / c8, v = i - p * c8;
        const float* row = sx + p * CP + v * 8;
        const float* rr = sr + p * CP + v * 8;
        float d[8];
        unpack8(ld8(dy + (p0 + p) * dpitch + v * 8), d);
        float acc = 0.f, racc = 0.f;
        // scale window of c: [c-pre, c+post]; r window of c (channels whose window contains c): [c-post, c+pre]
#pragma unroll 4
        for (int k = 0; k < size - 1; ++k) acc += row[k] * row[k];
        for (int k = 0; k < size - 1; ++k) racc += rr[k + pre - post];
        float o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float hi = row[j + size - 1];
          acc += hi * hi;
          racc += rr[j + size - 1 + pre - post];
          const float scale = 1.f + alpha_over_n * acc;
          const float xc = row[j + pre];
          float g = d[j] * exp2f(-beta * log2f(scale)) - cache_ratio * xc * racc;
          if (fuse_relu && !(xc > 0.f)) g = 0.f;
          o[j] = g;
          acc -= row[j] * row[j];
          racc -= rr[j + pre - post];
        }
        st8(out + (p0 + p) * opitch + v * 8, pack8(o));
      }
    }
    __syncthreads();
  }
}

// Register/L1 variant for the usual small windows (local_size <= 9): each thread owns 8 channels of one pixel and
// reads the neighbouring 16-byte vectors directly (they are L1 hits: the same lines are being read by the
// adjacent threads), so there is no shared-memory staging, no bank conflicts and DRAM sees every byte once.
// Register-resident variant (local_size <= 9): one thread = 8 channels of one pixel, neighbours' vectors loaded
// directly (the channel window of a pixel is contiguous in NHWC).  The first version was issue-bound: 64-bit index
// divisions, libm log2f/exp2f and 5-tap re-summation.  This version uses a magic-number divide, MUFU lg2/ex2 and sliding-window sums.
template <int N>
__device__ __forceinline__ void load_window(const __nv_bfloat16* p, int v, int c8, float (&w)[24]) {
  float t[8];
  bf16x8 z;
#pragma unroll
  for (int i = 0; i < 4; ++i) z.v[i] = __floats2bfloat162_rn(0.f, 0.f);
  unpack8(v > 0 ? ld8(p - 8) : z, t);
#pragma unroll
  for (int j = 0; j < 8; ++j) w[j] = t[j];
  unpack8(ld8(p), t);
#pragma unroll
  for (int j = 0; j < 8; ++j) w[8 + j] = t[j];
  unpack8(v + 1 < c8 ? ld8(p + 8) : z, t);
#pragma unroll
  for (int j = 0; j < 8; ++j) w[16 + j] = t[j];
}

template <bool BWD, int PRE>
__global__ void __launch_bounds__(256)
lrn_reg_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ dy, __nv_bfloat16* __restrict__ out,
               uint32_t total, FastDiv div_c8, int xpitch, int dpitch, int opitch, float alpha_over_n, float beta,
               int mask_relu) {
  constexpr int pre = PRE;             // compile-time window: all register-array indices below are static
  const int c8 = static_cast<int>(div_c8.d);
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const uint32_t p = fdiv(i, div_c8);
    const int v = static_cast<int>(i - p * div_c8.d);
    float xw[24];                                 // channels [8v-8, 8v+16)
    load_window<0>(x + static_cast<long>(p) * xpitch + v * 8, v, c8, xw);
    if (mask_relu) {                              // the op is applied to ReLU(x), as in the shared-memory kernel
#pragma unroll
      for (int q = 0; q < 24; ++q) xw[q] = fmaxf(xw[q], 0.f);
    }
    float o[8];
    if constexpr (!BWD) {
      // sliding window over the squares of channels [8v-pre, 8v+7+pre]
      float sq[8 + 2 * pre];
#pragma unroll
      for (int q = 0; q < 8 + 2 * pre; ++q) sq[q] = xw[8 - pre + q] * xw[8 - pre + q];
      float acc = 0.f;
#pragma unroll
      for (int q = 0; q < 2 * pre; ++q) acc += sq[q];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        acc += sq[j + 2 * pre];
        o[j] = xw[8 + j] * fast_ex2(-beta * fast_lg2(fmaf(alpha_over_n, acc, 1.f)));
        acc -= sq[j];
      }
    } else {
      float dw[24];
      load_window<1>(dy + static_cast<long>(p) * dpitch + v * 8, v, c8, dw);
      // squares of channels [8v-2pre, 8v+7+2pre] (zero outside the loaded 24: needs pre <= 4)
      constexpr int NS = 8 + 4 * pre;
      float sq[NS];
#pragma unroll
      for (int q = 0; q < NS; ++q) sq[q] = xw[8 - 2 * pre + q] * xw[8 - 2 * pre + q];
      // r_c = dy_c * x_c * scale_c^(-beta-1) for c in [8v-pre, 8v+7+pre]; keep scale_c^-beta of the centre 8
      constexpr int NR = 8 + 2 * pre;
      float rr[NR], sb[8];
      float acc = 0.f;
#pragma unroll
      for (int q = 0; q < 2 * pre; ++q) acc += sq[q];
#pragma unroll
      for (int q = 0; q < NR; ++q) {
        acc += sq[q + 2 * pre];
        const float s = fmaf(alpha_over_n, acc, 1.f);
        const float t = fast_ex2(-beta * fast_lg2(s));            // scale^-beta
        rr[q] = dw[8 - pre + q] * xw[8 - pre + q] * __fdividef(t, s);
        if (q >= pre && q < pre + 8) sb[q - pre] = t;
        acc -= sq[q];
      }
      const float ratio = 2.f * alpha_over_n * beta;
      float racc = 0.f;
#pragma unroll
      for (int q = 0; q < 2 * pre; ++q) racc += rr[q];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        racc += rr[j + 2 * pre];
        const float xc = xw[8 + j];
        float g = fmaf(dw[8 + j], sb[j], -ratio * xc * racc);
        if (mask_relu && !(xc > 0.f)) g = 0.f;
        o[j] = g;
        racc -= rr[j];
      }
    }
    st8(out + static_cast<long>(p) * opitch + v * 8, pack8(o));
  }
}

static void lrn_launch(bool bwd, const at::Tensor& x, const at::Tensor* dy, at::Tensor& out, int64_t size, double alpha,
                       double beta, bool fuse_relu) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16, "lrn: bf16 CUDA tensor expected");
  TORCH_CHECK(size % 2 == 1, "lrn: pre == post requires an odd local_size");
  c10::cuda::CUDAGuard guard(x.device());
  NhwcView v = nhwc_view(x), o = nhwc_view(out);
  TORCH_CHECK(v.C % 8 == 0, "lrn: channels must be a multiple of 8");
  const long npix = static_cast<long>(v.N) * v.H * v.W;
  const int CP = v.C + size - 1;
  const int arrays = bwd ? 2 : 1;
  int pix = std::max(1, std::min(64, static_cast<int>((96 * 1024) / (arrays * CP * 4))));
  const size_t smem = static_cast<size_t>(arrays) * pix * CP * sizeof(float);
  auto stream = at::cuda::getCurrentCUDAStream();
  const int grid = static_cast<int>(std::min<long>((npix + pix - 1) / pix, 132 * 8));
  long dpitch = 0;
  const __nv_bfloat16* dyp = nullptr;
  if (bwd) {
    NhwcView d = nhwc_view(*dy);
    dpitch = d.pitch;
    dyp = reinterpret_cast<const __nv_bfloat16*>(dy->data_ptr());
  }
  auto xp = reinterpret_cast<const __nv_bfloat16*>(x.data_ptr());
  auto op = reinterpret_cast<__nv_bfloat16*>(out.data_ptr());
  if (size <= 9) {
    const long total = npix * (v.C / 8);
    TORCH_CHECK(total < (1L << 31) && v.pitch < (1L << 31), "lrn: tensor too large for 32-bit indexing");
    const int g2 = grid_for(total, 256, 132 * 32);
    const float aon = static_cast<float>(alpha / size), bt = static_cast<float>(beta);
    const FastDiv dc8 = make_fastdiv(static_cast<uint32_t>(v.C / 8));
    const uint32_t tot = static_cast<uint32_t>(total);
    const int xpi = static_cast<int>(v.pitch), dpi = static_cast<int>(dpitch), opi = static_cast<int>(o.pitch);
#define PSD_LRN(PRE)                                                                                                   \
  if (bwd) lrn_reg_kernel<true, PRE><<<g2, 256, 0, stream>>>(xp, dyp, op, tot, dc8, xpi, dpi, opi, aon, bt, fuse_relu); \
  else lrn_reg_kernel<false, PRE><<<g2, 256, 0, stream>>>(xp, nullptr, op, tot, dc8, xpi, 0, opi, aon, bt, fuse_relu)
    switch ((size - 1) / 2) {
      case 0: PSD_LRN(0); break;
      case 1: PSD_LRN(1); break;
      case 2: PSD_LRN(2); break;
      case 3: PSD_LRN(3); break;
      default: PSD_LRN(4); break;
    }
#undef PSD_LRN
    C10_CUDA_KERNEL_LAUNCH_CHECK();
    return;
  }
  if (bwd) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(lrn_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    lrn_kernel<true><<<grid, kLrnThreads, smem, stream>>>(xp, dyp, op, npix, v.C, v.pitch, dpitch, o.pitch,
                                                          static_cast<int>(size), static_cast<float>(alpha / size),
                                                          static_cast<float>(beta), pix, fuse_relu);
  } else {
    C10_CUDA_CHECK(cudaFuncSetAttribute(lrn_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    lrn_kernel<false><<<grid, kLrnThreads, smem, stream>>>(xp, nullptr, op, npix, v.C, v.pitch, 0, o.pitch,
                                                           static_cast<int>(size), static_cast<float>(alpha / size),
                                                           static_cast<float>(beta), pix, fuse_relu);
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

at::Tensor lrn_fwd(const at::Tensor& x, int64_t size, double alpha, double beta, bool fuse_relu) {
  at::Tensor y = empty_nhwc(x.size(0), x.size(1), x.size(2), x.size(3), x.options());
  lrn_launch(false, x, nullptr, y, size, alpha, beta, fuse_relu);
  return y;
}

at::Tensor lrn_bwd(const at::Tensor& x, const at::Tensor& dy, int64_t size, double alpha, double beta, bool fuse_relu) {
  at::Tensor dx = empty_nhwc(x.size(0), x.size(1), x.size(2), x.size(3), x.options());
  lrn_launch(true, x, &dy, dx, size, alpha, beta, fuse_relu);
  return dx;
}

}  // namespace psd

TORCH_LIBRARY_FRAGMENT(poseidon, m) {
  m.def("lrn_fwd(Tensor x, int size, float alpha, float beta, bool fuse_relu) -> Tensor", &psd::lrn_fwd);
  m.def("lrn_bwd(Tensor x, Tensor dy, int size, float alpha, float beta, bool fuse_relu) -> Tensor", &psd::lrn_bwd);
}
