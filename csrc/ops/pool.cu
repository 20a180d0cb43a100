// MAX / AVE pooling, NHWC bf16, 8 channels per thread (16-byte accesses), Caffe window semantics
// (ceil output size computed by the caller; AVE divisor = window clipped to the padded extent).
//
// MAX forward stores the arg-max as the in-window tap index (uint8) so backward is a pure gather:
// every input pixel sums dy over the output windows whose recorded tap points at it — no atomics,
// deterministic.  AVE backward is the matching gather.
//
// reference: src/caffe/layers/pooling_layer.cu:12-47 (MaxPoolForward), :50-78 (AvePoolForward),
// :213-256 (MaxPoolBackward), :259-293 (AvePoolBackward).
#include "nhwc_common.cuh"

namespace psd {

struct PoolGeom {
  int N, C, H, W, OH, OW, kh, kw, sh, sw, ph, pw;
  int xpitch, ypitch;    // pixel pitches of the input-side and output-side tensors
  FastDiv d_c8, d_ow, d_oh, d_w, d_h, d_sh, d_sw;
};

// The first versions of these kernels were issue-bound: 64-bit index divisions and per-channel fp32 compare/select chains.  Now: 32-bit
// indices with magic-number divides, MAX forward entirely in packed bf16x2 (max + compare-mask + one LOP3 per channel
// pair and tap; bf16 compares are exact, so the result equals the fp32 computation), MAX backward with SIMD byte compares.

__device__ __forceinline__ uint32_t bf2_as_u32(const __nv_bfloat162& v) { return *reinterpret_cast<const uint32_t*>(&v); }
__device__ __forceinline__ __nv_bfloat162 u32_as_bf2(uint32_t v) { return *reinterpret_cast<const __nv_bfloat162*>(&v); }

// KT > 0: compile-time square window (fully unrolled, all window loads issued before use); KT == 0: generic.
template <bool MAXP, int KT>
__global__ void __launch_bounds__(256)
pool_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, uint8_t* __restrict__ idx,
                PoolGeom g, uint32_t total) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    uint32_t t = fdiv(i, g.d_c8);
    const int v = static_cast<int>(i - t * g.d_c8.d);
    const uint32_t opix = t;
    uint32_t q = fdiv(t, g.d_ow);
    const int ow = static_cast<int>(t - q * g.d_ow.d);
    const uint32_t n = fdiv(q, g.d_oh);
    const int oh = static_cast<int>(q - n * g.d_oh.d);
    const int hs = oh * g.sh - g.ph, ws = ow * g.sw - g.pw;
    const __nv_bfloat16* xb = x + static_cast<long>(n) * (g.H * g.W) * g.xpitch + v * 8;
    if constexpr (MAXP) {
      const __nv_bfloat162 ninf = __halves2bfloat162(__ushort_as_bfloat16(0xff80), __ushort_as_bfloat16(0xff80));
      __nv_bfloat162 cur[4] = {ninf, ninf, ninf, ninf};
      uint32_t best[4] = {0u, 0u, 0u, 0u};            // two 16-bit tap indices per register
      auto take = [&](const bf16x8& w, uint32_t tap) {
        const uint32_t tt = tap | (tap << 16);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint32_t m = __hgt2_mask(w.v[k], cur[k]);      // 0xffff per half where the new value is larger
          cur[k] = __hmax2(cur[k], w.v[k]);
          best[k] = (best[k] & ~m) | (tt & m);
        }
      };
      if constexpr (KT > 0) {
        bf16x8 win[KT * KT];
        bool ok[KT * KT];
#pragma unroll
        for (int dh = 0; dh < KT; ++dh) {
#pragma unroll
          for (int dw = 0; dw < KT; ++dw) {
            const int h = hs + dh, w = ws + dw;
            ok[dh * KT + dw] = static_cast<unsigned>(h) < static_cast<unsigned>(g.H) &&
                               static_cast<unsigned>(w) < static_cast<unsigned>(g.W);
            if (ok[dh * KT + dw]) win[dh * KT + dw] = ld8(xb + static_cast<long>(h * g.W + w) * g.xpitch);
          }
        }
#pragma unroll
        for (int tp = 0; tp < KT * KT; ++tp)
          if (ok[tp]) take(win[tp], tp);
      } else {
        const int he = min(hs + g.kh, g.H), we = min(ws + g.kw, g.W);
        for (int h = max(hs, 0); h < he; ++h)
          for (int w = max(ws, 0); w < we; ++w)
            take(ld8(xb + static_cast<long>(h * g.W + w) * g.xpitch), static_cast<uint32_t>((h - hs) * g.kw + (w - ws)));
      }
      bf16x8 o;
#pragma unroll
      for (int k = 0; k < 4; ++k) o.v[k] = cur[k];
      st8(y + static_cast<long>(opix) * g.ypitch + v * 8, o);
      if (idx != nullptr) {
        uint2 pk;                                        // byte j = tap of channel j
        pk.x = __byte_perm(best[0], best[1], 0x6420);
        pk.y = __byte_perm(best[2], best[3], 0x6420);
        *reinterpret_cast<uint2*>(idx + static_cast<long>(opix) * g.C + v * 8) = pk;
      }
    } else {
      const int he_pad = min(hs + g.kh, g.H + g.ph), we_pad = min(ws + g.kw, g.W + g.pw);
      const int he = min(he_pad, g.H), we = min(we_pad, g.W);
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = 0.f;
      for (int h = max(hs, 0); h < he; ++h) {
        for (int w = max(ws, 0); w < we; ++w) {
          float f[8];
          unpack8(ld8(xb + static_cast<long>(h * g.W + w) * g.xpitch), f);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] += f[j];
        }
      }
      const float inv = 1.f / static_cast<float>((he_pad - hs) * (we_pad - ws));
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] *= inv;
      st8(y + static_cast<long>(opix) * g.ypitch + v * 8, pack8(acc));
    }
  }
}

// NC > 0: at most NC x NC output windows cover an input pixel (NC = ceil(k / stride)), loops unrolled with
// predicates so every dy / index load is in flight before the accumulation; NC == 0: generic.
template <bool MAXP, int NC>
__global__ void __launch_bounds__(256)
pool_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ idx, __nv_bfloat16* __restrict__ dx,
                PoolGeom g, uint32_t total) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    uint32_t t = fdiv(i, g.d_c8);
    const int v = static_cast<int>(i - t * g.d_c8.d);
    const uint32_t ipix = t;
    uint32_t q = fdiv(t, g.d_w);
    const int w = static_cast<int>(t - q * g.d_w.d);
    const uint32_t n = fdiv(q, g.d_h);
    const int h = static_cast<int>(q - n * g.d_h.d);
    // output windows that cover (h, w)
    const int hp = h + g.ph, wp = w + g.pw;
    const int oh0 = hp < g.kh ? 0 : static_cast<int>(fdiv(static_cast<uint32_t>(hp - g.kh), g.d_sh)) + 1;
    const int oh1 = min(static_cast<int>(fdiv(static_cast<uint32_t>(hp), g.d_sh)) + 1, g.OH);
    const int ow0 = wp < g.kw ? 0 : static_cast<int>(fdiv(static_cast<uint32_t>(wp - g.kw), g.d_sw)) + 1;
    const int ow1 = min(static_cast<int>(fdiv(static_cast<uint32_t>(wp), g.d_sw)) + 1, g.OW);
    const uint32_t obase = n * static_cast<uint32_t>(g.OH * g.OW);
    float acc[8];
    // MAX: an input pixel is the arg-max of at most NC*NC windows and usually of one — the masked dy values are summed as
    // packed bf16 pairs (4 HADD2 per window instead of 8 unpack + 8 FADD; the result is rounded to bf16 anyway)
    __nv_bfloat162 acc2[4];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) acc2[k] = u32_as_bf2(0u);
    auto accumulate = [&](int oh, int ow, const bf16x8& dv, const uint2& pk) {
      const int hs = oh * g.sh - g.ph, ws = ow * g.sw - g.pw;
      if (MAXP) {
        // keep dy only where the recorded arg-max tap is this pixel: SIMD byte compare -> 16-bit lane masks
        const uint32_t tap = static_cast<uint32_t>((h - hs) * g.kw + (w - ws)) * 0x01010101u;
        const uint32_t m0 = __vcmpeq4(pk.x, tap), m1 = __vcmpeq4(pk.y, tap);
        const uint32_t mk[4] = {__byte_perm(m0, 0, 0x1100), __byte_perm(m0, 0, 0x3322), __byte_perm(m1, 0, 0x1100),
                                __byte_perm(m1, 0, 0x3322)};
#pragma unroll
        for (int k = 0; k < 4; ++k) acc2[k] = __hadd2(acc2[k], u32_as_bf2(bf2_as_u32(dv.v[k]) & mk[k]));
      } else {
        float d[8];
        unpack8(dv, d);
        const int he_pad = min(hs + g.kh, g.H + g.ph), we_pad = min(ws + g.kw, g.W + g.pw);
        const float inv = 1.f / static_cast<float>((he_pad - hs) * (we_pad - ws));
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += d[j] * inv;
      }
    };
    if constexpr (NC > 0) {
      bf16x8 dv[NC * NC];
      uint2 pk[NC * NC];
      bool ok[NC * NC];
#pragma unroll
      for (int a = 0; a < NC; ++a) {
#pragma unroll
        for (int b = 0; b < NC; ++b) {
          const int oh = oh0 + a, ow = ow0 + b;
          const int tt = a * NC + b;
          ok[tt] = oh < oh1 && ow < ow1;
          pk[tt] = make_uint2(0, 0);
          if (ok[tt]) {
            const uint32_t opix = obase + static_cast<uint32_t>(oh * g.OW + ow);
            dv[tt] = ld8(dy + static_cast<long>(opix) * g.ypitch + v * 8);
            if (MAXP) pk[tt] = *reinterpret_cast<const uint2*>(idx + static_cast<long>(opix) * g.C + v * 8);
          }
        }
      }
#pragma unroll
      for (int a = 0; a < NC; ++a) {
#pragma unroll
        for (int b = 0; b < NC; ++b)
          if (ok[a * NC + b]) accumulate(oh0 + a, ow0 + b, dv[a * NC + b], pk[a * NC + b]);
      }
    } else {
      for (int oh = oh0; oh < oh1; ++oh) {
        for (int ow = ow0; ow < ow1; ++ow) {
          const uint32_t opix = obase + static_cast<uint32_t>(oh * g.OW + ow);
          const bf16x8 dv = ld8(dy + static_cast<long>(opix) * g.ypitch + v * 8);
          uint2 pk = make_uint2(0, 0);
          if (MAXP) pk = *reinterpret_cast<const uint2*>(idx + static_cast<long>(opix) * g.C + v * 8);
          accumulate(oh, ow, dv, pk);
        }
      }
    }
    if (MAXP) {
      bf16x8 o;
#pragma unroll
      for (int k = 0; k < 4; ++k) o.v[k] = acc2[k];
      st8(dx + static_cast<long>(ipix) * g.xpitch + v * 8, o);
    } else {
      st8(dx + static_cast<long>(ipix) * g.xpitch + v * 8, pack8(acc));
    }
  }
}

static PoolGeom make_geom(const NhwcView& x, int64_t oh, int64_t ow, at::IntArrayRef k, at::IntArrayRef s,
                          at::IntArrayRef p) {
  PoolGeom g;
  g.N = x.N; g.C = x.C; g.H = x.H; g.W = x.W; g.OH = oh; g.OW = ow;
  g.kh = k[0]; g.kw = k[1]; g.sh = s[0]; g.sw = s[1]; g.ph = p[0]; g.pw = p[1];
  TORCH_CHECK(x.pitch < (1L << 31) && static_cast<long>(x.N) * x.H * x.W * (x.C / 8) < (1L << 31) &&
              static_cast<long>(x.N) * oh * ow * (x.C / 8) < (1L << 31), "pool: tensor too large for 32-bit indexing");
  g.xpitch = static_cast<int>(x.pitch);
  g.ypitch = x.C;
  g.d_c8 = make_fastdiv(x.C / 8);
  g.d_ow = make_fastdiv(static_cast<uint32_t>(ow));
  g.d_oh = make_fastdiv(static_cast<uint32_t>(oh));
  g.d_w = make_fastdiv(x.W);
  g.d_h = make_fastdiv(x.H);
  g.d_sh = make_fastdiv(g.sh);
  g.d_sw = make_fastdiv(g.sw);
  return g;
}

std::tuple<at::Tensor, at::Tensor> pool_fwd(const at::Tensor& x, bool is_max, at::IntArrayRef k, at::IntArrayRef s,
                                            at::IntArrayRef p, int64_t oh, int64_t ow, bool want_idx) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16);
  c10::cuda::CUDAGuard guard(x.device());
  NhwcView xv = nhwc_view(x);
  TORCH_CHECK(xv.C % 8 == 0, "pool: channels must be a multiple of 8");
  TORCH_CHECK(k[0] * k[1] <= 255, "pool: window too large for uint8 tap index");
  at::Tensor y = empty_nhwc(xv.N, xv.C, oh, ow, x.options());
  at::Tensor idx = (is_max && want_idx) ? at::empty({xv.N, oh, ow, xv.C}, x.options().dtype(at::kByte)) : at::Tensor();
  PoolGeom g = make_geom(xv, oh, ow, k, s, p);
  const long total = static_cast<long>(g.N) * g.OH * g.OW * (g.C / 8);
  auto stream = at::cuda::getCurrentCUDAStream();
  auto xp = reinterpret_cast<const __nv_bfloat16*>(x.data_ptr());
  auto yp = reinterpret_cast<__nv_bfloat16*>(y.data_ptr());
  uint8_t* ip = idx.defined() ? idx.data_ptr<uint8_t>() : nullptr;
  const int grid = grid_for(total, 256, 132 * 32);
  const int kt = (g.kh == g.kw && (g.kh == 2 || g.kh == 3)) ? g.kh : 0;
#define PSD_PF(MX, KT) pool_fwd_kernel<MX, KT><<<grid, 256, 0, stream>>>(xp, yp, MX ? ip : nullptr, g, static_cast<uint32_t>(total))
  if (is_max) { if (kt == 3) PSD_PF(true, 3); else if (kt == 2) PSD_PF(true, 2); else PSD_PF(true, 0); }
  else        { if (kt == 3) PSD_PF(false, 3); else if (kt == 2) PSD_PF(false, 2); else PSD_PF(false, 0); }
#undef PSD_PF
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return {y, idx.defined() ? idx : at::empty({0}, x.options().dtype(at::kByte))};
}

at::Tensor pool_bwd(const at::Tensor& dy, const at::Tensor& idx, bool is_max, at::IntArrayRef in_hw, at::IntArrayRef k,
                    at::IntArrayRef s, at::IntArrayRef p) {
  TORCH_CHECK(dy.is_cuda() && dy.scalar_type() == at::kBFloat16);
  c10::cuda::CUDAGuard guard(dy.device());
  NhwcView dv = nhwc_view(dy);
  at::Tensor dx = empty_nhwc(dv.N, dv.C, in_hw[0], in_hw[1], dy.options());
  NhwcView xv = nhwc_view(dx);
  PoolGeom g = make_geom(xv, dv.H, dv.W, k, s, p);
  g.ypitch = static_cast<int>(dv.pitch);
  const long total = static_cast<long>(g.N) * g.H * g.W * (g.C / 8);
  auto stream = at::cuda::getCurrentCUDAStream();
  auto dyp = reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr());
  auto dxp = reinterpret_cast<__nv_bfloat16*>(dx.data_ptr());
  const int grid = grid_for(total, 256, 132 * 32);
  const int ncand = std::max((g.kh + g.sh - 1) / g.sh, (g.kw + g.sw - 1) / g.sw);
  const int nc = ncand <= 3 ? ncand : 0;
  const uint8_t* ip = nullptr;
  if (is_max) {
    TORCH_CHECK(idx.numel() == dy.numel(), "pool_bwd: index tensor missing");
    ip = idx.data_ptr<uint8_t>();
  }
#define PSD_PB(MX, NCV) pool_bwd_kernel<MX, NCV><<<grid, 256, 0, stream>>>(dyp, ip, dxp, g, static_cast<uint32_t>(total))
  if (is_max) { if (nc == 1) PSD_PB(true, 1); else if (nc == 2) PSD_PB(true, 2); else if (nc == 3) PSD_PB(true, 3); else PSD_PB(true, 0); }
  else        { if (nc == 1) PSD_PB(false, 1); else if (nc == 2) PSD_PB(false, 2); else if (nc == 3) PSD_PB(false, 3); else PSD_PB(false, 0); }
#undef PSD_PB
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return dx;
}

}  // namespace psd

TORCH_LIBRARY_FRAGMENT(poseidon, m) {
  m.def("pool_fwd(Tensor x, bool is_max, int[] k, int[] s, int[] p, int oh, int ow, bool want_idx) -> (Tensor, Tensor)",
        &psd::pool_fwd);
  m.def("pool_bwd(Tensor dy, Tensor idx, bool is_max, int[] in_hw, int[] k, int[] s, int[] p) -> Tensor", &psd::pool_bwd);
}
