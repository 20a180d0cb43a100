"""CPU emulation of ``torch.ops.poseidon`` — the same op surface, the same operand layouts, plain PyTorch math.

Why: the sm100 engine is two things — the CUDA kernels in ``csrc/`` and a fair amount of Python around them that decides
operand layouts (ROW / space-to-depth / 8-channel first layers, channel-padded K, (h, w, c) inner-product weights), keeps
bf16 shadows in step with fp32 masters, plans epilogue fusion and routes gradients into the optimizer kernels.  The kernels
can only be tested on an H100; the Python around them is just as easy to break, and with ``POSEIDON_EMULATE=1`` it runs on
any machine: ``sm100.K()`` hands out this module's :class:`EmulatedKernels` instead of the compiled extension, and the
whole engine (``Solver(engine="sm100")``, fusion plan, FusedBackend's single-process path) steps on the CPU.

Every method documents the layout contract of the kernel it stands in for (file:line of the CUDA implementation); the
arithmetic is fp32 with one bf16 rounding at the output, which is also what the kernels do (fp32 accumulation in registers,
bf16 store), so results agree with the GPU to bf16 rounding.  This is a *test double*: it is never selected implicitly,
it is slow.  The multi-GPU peer-memory ops run too: ranks are processes, the symmetric arena is host shared memory
(:class:`EmulatedArena`), the flag protocol is the kernels'.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import reference as R

CL = torch.channels_last
BF16 = torch.bfloat16


def _nhwc(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous(memory_format=CL)


def _storage_order_flat(t: torch.Tensor) -> torch.Tensor:
    """Elements of a dense tensor in memory order."""
    dims = sorted(range(t.dim()), key=lambda d: (t.shape[d] == 1, -t.stride(d)))
    return t.permute(dims).reshape(-1)


E4M3 = torch.float8_e4m3fn
E4M3_MAX = 448.0


def _nan_free_abs(v: torch.Tensor) -> torch.Tensor:
    """|v| with NaN as 0: the kernels' amax uses fmaxf, which skips NaN (an Inf still counts)."""
    a = v.abs()
    return torch.where(torch.isnan(a), torch.zeros_like(a), a)


def e4m3_scale(amax: torch.Tensor) -> torch.Tensor:
    """Just-in-time fp8 scale s = 448 / amax in fp32, at most FLT_MAX, and 1 where amax == 0."""
    amax = amax.float()
    # a true fp32 division, as the kernels do it (torch computes `448 / t` as 448 * reciprocal(t))
    s = torch.where(amax > 0, torch.div(torch.full_like(amax, E4M3_MAX), amax), torch.ones_like(amax))
    return torch.clamp(s, max=torch.finfo(torch.float32).max)


E5M2 = torch.float8_e5m2
E5M2_MAX = 57344.0


def e5m2_scale(amax: torch.Tensor) -> torch.Tensor:
    """Just-in-time e5m2 scale s = 57344 / amax in fp32 (a true division), at most FLT_MAX, and 1 where amax == 0."""
    amax = amax.float()
    s = torch.where(amax > 0, torch.div(torch.full_like(amax, E5M2_MAX), amax), torch.ones_like(amax))
    return torch.clamp(s, max=torch.finfo(torch.float32).max)


def e5m2_quant(v: torch.Tensor, s) -> torch.Tensor:
    """e5m2(v · s) as cvt.rn.satfinite does it: clamp to ±57344 first (torch's cast rounds larger values to inf)."""
    return torch.clamp(v.float() * s, -E5M2_MAX, E5M2_MAX).to(E5M2)


AMAX_HISTORY = 16          # slots of a delayed-scaling amax ring (csrc/ops/fp8_quant.cu kAmaxHistory)


def chwn_images(n: int) -> int:
    """Images per channel row of the fp8 weight gradient's batch-innermost copies: 16, 32, 64 or a multiple of 128."""
    if n <= 64:
        return 16 if n <= 16 else (32 if n <= 32 else 64)
    return (n + 127) // 128 * 128


def e4m3_quant(v: torch.Tensor, s) -> torch.Tensor:
    """e4m3(v · s) as cvt.rn.satfinite does it: clamp to ±448 first (torch's cast gives NaN above 464), NaN stays NaN."""
    return torch.clamp(v.float() * s, -E4M3_MAX, E4M3_MAX).to(E4M3)


def _act(v: torch.Tensor, relu: bool, slope: float) -> torch.Tensor:
    if not relu:
        return v
    return torch.where(v > 0, v, v * slope)


class EmulatedKernels:
    """Drop-in for ``torch.ops.poseidon`` (single-process ops)."""

    emulated = True

    # ------------------------------------------------------------------------------------------ switches
    def set_conv_cluster(self, c):           # csrc/gemm/conv_ops.cu (tuning knobs: no numerical effect)
        return None

    def set_conv_im2col(self, on):
        return None

    def set_conv_mcast(self, c):
        return None

    def set_conv_pair(self, on):
        return None

    def set_bulk_epilogue(self, on):
        return None

    def set_max_stages(self, n):
        return None

    def set_pair_cta(self, on):              # csrc/gemm/gemm_ops.cu (cta_group::2 on/off: no numerical effect)
        return None

    # ------------------------------------------------------------------------------------------ GEMM
    def gemm_bf16(self, a, a_mn, b, b_mn, bias, relu, slope, mask, out, bn):
        """C[M,N] bf16 = act(A·Bᵀ + bias), A = a ([M,K]) or aᵀ, B = b ([N,K]) or bᵀ (csrc/gemm/gemm_ops.cu:173-240)."""
        assert a.dtype == BF16 and b.dtype == BF16
        A = a.t() if a_mn else a
        B = b.t() if b_mn else b
        v = A.float() @ B.float().t()
        if bias is not None:
            v = v + bias.float()
        v = _act(v, relu, slope)
        if mask is not None:
            v = torch.where(mask.float() > 0, v, v * slope)
        if out is None:
            return v.to(BF16)
        out.copy_(v)
        return out

    def gemm_f32(self, a, a_mn, b, b_mn, out, alpha, accumulate, split_k, bn):
        """out[M,N] fp32 (+)= alpha · A·Bᵀ (csrc/gemm/gemm_ops.cu:243-300)."""
        A = a.t() if a_mn else a
        B = b.t() if b_mn else b
        v = (A.float() @ B.float().t()) * alpha
        if accumulate:
            out.add_(v)
        else:
            out.copy_(v)

    # ------------------------------------------------------------------------------------------ convolution
    @staticmethod
    def _w4_tap(wb, cout, r, s, cg, cgk):
        """[Cout, R*S*Cgk] (K ordered (r, s, c), slots >= Cg zero) -> [Cout, Cg, R, S] fp32."""
        cgk = cgk or cg
        return wb.reshape(cout, r, s, cgk)[..., :cg].permute(0, 3, 1, 2).float()

    def conv_fprop(self, x, wb, bias, kernel, stride, pad, groups, mode, OH, OW, relu, slope, out):
        """Implicit-GEMM forward (csrc/gemm/conv_ops.cu:176-247).
        mode 0 (TAP): x logical [N,C,H,W] channels-last; wb [Cout, R*S*Cgk].
        mode 1 (ROW): x is the spatially pre-padded NHWC4 image; wb [Cout, R*Lp], each kernel row = S*4 contiguous
        elements padded to Lp = roundup8(S*4)."""
        r, s = kernel
        cout = wb.shape[0]
        if mode == 1:
            cp = x.shape[1]
            lp = wb.shape[1] // r
            w4 = wb.reshape(cout, r, lp)[:, :, : s * cp].reshape(cout, r, s, cp).permute(0, 3, 1, 2).float()
            y = F.conv2d(x.float(), w4, None, tuple(stride), 0)[:, :, :OH, :OW]
        else:
            cg = x.shape[1] // groups
            cgk = wb.shape[1] // (r * s)
            w4 = self._w4_tap(wb, cout, r, s, cg, cgk)
            y = F.conv2d(x.float(), w4, None, tuple(stride), tuple(pad), 1, groups)
        assert tuple(y.shape[2:]) == (OH, OW), (tuple(y.shape), OH, OW)
        if bias is not None:
            y = y + bias.float().view(1, -1, 1, 1)
        y = _act(y, relu, slope)
        if out is not None:
            out.copy_(y)
            return out
        return _nhwc(y.to(BF16))

    def conv_dgrad(self, dy, wt, kernel, pad, groups, H, W, mask, slope):
        """Stride-1 data gradient from the packed operand wt [groups*Cg, R*S*Cop] (K ordered (r, s, co));
        optional producer-ReLU mask applied in the epilogue (csrc/gemm/conv_ops.cu:250-301)."""
        r, s = kernel
        cout = dy.shape[1]
        cout_g = cout // groups
        cg = wt.shape[0] // groups
        cop = wt.shape[1] // (r * s)
        w = wt.reshape(groups, cg, r, s, cop)[..., :cout_g].float()           # g, ci, r, s, co
        w4 = w.permute(0, 4, 1, 2, 3).reshape(cout, cg, r, s)                  # conv weight [Cout, Cg, R, S]
        # out[t] = sum_j dy[t - j] w[j], t in [0, OH + R - 1);  dx[i] = sum_j dy[i + pad - j] w[j] = out[i + pad], i < H —
        # the output extent is the caller's (the strided data gradient asks for one phase of dX: fewer or more rows than
        # the natural transposed-convolution size, the excess being zero)
        full = F.conv_transpose2d(dy.float(), w4, None, 1, 0, 0, groups)
        full = F.pad(full, (0, max(0, pad[1] + W - full.shape[3]), 0, max(0, pad[0] + H - full.shape[2])))
        dx = full[:, :, pad[0]: pad[0] + H, pad[1]: pad[1] + W]
        if mask is not None:
            dx = torch.where(mask.float() > 0, dx, dx * slope)
        return _nhwc(dx.to(BF16))

    def conv_dgrad_w(self, dy, wb, kernel, pad, groups, H, W, mask, slope):
        """Stride-1 data gradient read from the FPROP operand wb [Cout, R*S*Cg] (no packed copy)
        (csrc/gemm/conv_ops.cu conv_dgrad_w)."""
        r, s = kernel
        cout = wb.shape[0]
        cg = wb.shape[1] // (r * s)
        w4 = wb.float().reshape(cout, r, s, cg).permute(0, 3, 1, 2)             # [Cout, Cg, R, S]
        full = F.conv_transpose2d(dy.float(), w4, None, 1, 0, 0, groups)
        full = F.pad(full, (0, max(0, pad[1] + W - full.shape[3]), 0, max(0, pad[0] + H - full.shape[2])))
        dx = full[:, :, pad[0]: pad[0] + H, pad[1]: pad[1] + W]
        if mask is not None:
            dx = torch.where(mask.float() > 0, dx, dx * slope)
        return _nhwc(dx.to(BF16))

    def conv_wgrad(self, x, dy, dw, kernel, stride, pad, groups, mode, alpha, cgk):
        """dw[Cout, K] fp32 += alpha · (weight gradient in the operand's K order) (csrc/gemm/conv_ops.cu:304-365)."""
        r, s = kernel
        cout = dy.shape[1]
        oh, ow = dy.shape[2:]
        if mode == 1:
            cp = x.shape[1]
            lp = dw.shape[1] // r
            xc = x[:, :, : (oh - 1) * stride[0] + r, : (ow - 1) * stride[1] + s].float()
            g = torch.nn.grad.conv2d_weight(xc, (cout, cp, r, s), dy.float(), tuple(stride), 0)
            g = g.permute(0, 2, 3, 1).reshape(cout, r, s * cp)
            g = F.pad(g, (0, lp - s * cp)).reshape(cout, r * lp)
        else:
            cg = x.shape[1] // groups
            g = torch.nn.grad.conv2d_weight(x.float(), (cout, cg, r, s), dy.float(), tuple(stride), tuple(pad), 1, groups)
            g = g.permute(0, 2, 3, 1).reshape(cout, r * s * cg)
        dw.add_(g, alpha=alpha)

    def conv_pack_dgrad(self, w, Cout, RS, Cg, groups, out, cop):
        """fp32 [Cout][RS][Cg] -> bf16 wt [groups*Cg, RS*Cop], co padded with zeros (csrc/gemm/conv_ops.cu:366-398)."""
        cout_g = Cout // groups
        cop = cop if cop > 0 else cout_g
        t = w.reshape(groups, cout_g, RS, Cg).permute(0, 3, 2, 1)              # g, ci, tap, co
        t = F.pad(t, (0, cop - cout_g)).reshape(groups * Cg, RS * cop)
        if out is None:
            return t.to(BF16).contiguous()
        out.copy_(t.reshape(out.shape))
        return out

    def conv_pack_padded(self, wb, Cout, RS, Cg, Cgk, out):
        """bf16 [Cout][RS][Cg] -> [Cout, RS*Cgk], slots >= Cg zero (csrc/gemm/conv_ops.cu:400-425)."""
        t = F.pad(wb.reshape(Cout, RS, Cg), (0, Cgk - Cg)).reshape(Cout, RS * Cgk)
        if out is None:
            return t.contiguous()
        out.copy_(t)
        return out

    # ------------------------------------------------------------------------------------------ fp8 forward convolution
    def fp8_quant_act(self, x, s_x_out):
        """bf16 NHWC (pitch may exceed C) -> e4m3 [N, C, H, W], a channel slice of a channels-last tensor whose pixel
        pitch is C rounded up to 16; s_x_out <- 1 / s (csrc/ops/fp8_quant.cu fp8_quant_act)."""
        n, c, h, w = x.shape
        v = x.float()
        s = e4m3_scale(_nan_free_abs(v).amax())
        s_x_out.copy_(torch.div(torch.ones_like(s), s).reshape(s_x_out.shape))
        full = torch.zeros((n, (c + 15) // 16 * 16, h, w), dtype=E4M3).contiguous(memory_format=CL)
        full[:, :c].copy_(e4m3_quant(v, s))
        return full[:, :c]

    def fp8_quant_weight(self, w, cgk, s_w_out):
        """fp32 master [Cout, Cg, R, S] -> e4m3 [Cout, R*S*cgk] (slots >= Cg zero), s_w_out[co] <- 1 / s_co
        (csrc/ops/fp8_quant.cu fp8_quant_weight)."""
        cout, cg, r, s_ = w.shape
        rows = w.float().permute(0, 2, 3, 1).reshape(cout, r * s_, cg)
        s = e4m3_scale(_nan_free_abs(rows).reshape(cout, -1).amax(dim=1))
        s_w_out.copy_(torch.div(torch.ones_like(s), s))
        out = torch.zeros((cout, r * s_, cgk), dtype=E4M3)
        out[..., :cg].copy_(e4m3_quant(rows, s.view(cout, 1, 1)))
        return out.reshape(cout, r * s_ * cgk)

    def conv_fprop_fp8(self, x8, w8, s_x, s_w, bias, kernel, stride, pad, groups, OH, OW, relu, slope, out):
        """act(conv(x8, w8) · s_x · s_w[co] + bias[co]) -> bf16 NHWC (csrc/gemm/conv_ops.cu conv_fprop_fp8)."""
        r, s = kernel
        cout = w8.shape[0]
        cg = x8.shape[1] // groups
        w4 = self._w4_tap(w8.float(), cout, r, s, cg, w8.shape[1] // (r * s))
        y = F.conv2d(x8.float(), w4, None, tuple(stride), tuple(pad), 1, groups)
        assert tuple(y.shape[2:]) == (OH, OW), (tuple(y.shape), OH, OW)
        y = y * (s_x.float().reshape(()) * s_w.float()).view(1, -1, 1, 1)
        if bias is not None:
            y = y + bias.float().view(1, -1, 1, 1)
        y = _act(y, relu, slope)
        if out is not None:
            out.copy_(y)
            return out
        return _nhwc(y.to(BF16))

    # ------------------------------------------------------------------------------------------ fp8 data gradient
    def fp8_quant_grad(self, dy, s_out, y, slope):
        """bf16 NHWC dY (pitch may exceed C) -> (e5m2 [N, C, H, W] as a channel slice of a channels-last tensor whose pixel
        pitch is C rounded up to 16, the bf16 dY that was cast); s_out <- 1 / s.  With y, dY is first masked as relu_bwd
        does it (dense result) (csrc/ops/fp8_quant.cu fp8_quant_grad)."""
        src = dy if y is None else _nhwc(torch.where(y.float() > 0, dy.float(), dy.float() * slope).to(BF16))
        n, c, h, w = src.shape
        v = src.float()
        s = e5m2_scale(_nan_free_abs(v).amax())
        s_out.copy_(torch.div(torch.ones_like(s), s).reshape(s_out.shape))
        full = torch.zeros((n, (c + 15) // 16 * 16, h, w), dtype=E5M2).contiguous(memory_format=CL)
        full[:, :c].copy_(e5m2_quant(v, s))
        return full[:, :c], src

    def fp8_quant_weight_dgrad(self, w, groups, cok, s_out):
        """fp32 master [Cout, Cg, R, S] -> e4m3 [groups*Cg, R*S*cok] in conv_pack_dgrad's order (slots >= Cout_g zero),
        s_out[g*Cg + ci] <- 1 / s per input channel (csrc/ops/fp8_quant.cu fp8_quant_weight_dgrad)."""
        cout, cg, r, s_ = w.shape
        cout_g = cout // groups
        rows = w.float().reshape(groups, cout_g, cg, r * s_).permute(0, 2, 3, 1).reshape(groups * cg, r * s_, cout_g)
        s = e4m3_scale(_nan_free_abs(rows).reshape(groups * cg, -1).amax(dim=1))
        s_out.copy_(torch.div(torch.ones_like(s), s))
        out = torch.zeros((groups * cg, r * s_, cok), dtype=E4M3)
        out[..., :cout_g].copy_(e4m3_quant(rows, s.view(-1, 1, 1)))
        return out.reshape(groups * cg, r * s_ * cok)

    # ------------------------------------------------------------------------------------------ fp8 weight gradient
    @staticmethod
    def _chwn(q: torch.Tensor) -> torch.Tensor:
        """[N, C, H, W] fp8 -> the batch-innermost copy [C, H, W, Np], Np = N rounded up to 16, 32, 64 or a multiple of 128,
        pad images zero."""
        n, c, h, w = q.shape
        out = torch.zeros((c, h, w, chwn_images(n)), dtype=q.dtype)
        out[..., :n].copy_(q.permute(1, 2, 3, 0))
        return out

    def fp8_quant_act_t(self, x, s_out):
        """bf16 NHWC (pitch may exceed C) -> e4m3 [C, H, W, Np], the transpose of fp8_quant_act's result;
        s_out <- 1 / s (csrc/ops/fp8_quant.cu fp8_quant_act_t)."""
        return self._chwn(self.fp8_quant_act(x, s_out))

    def fp8_quant_grad_t(self, dy, s_out, y, slope, nhwc):
        """(e5m2 [C, OH, OW, Np], fp8_quant_grad's NHWC copy when nhwc else an empty tensor, the bf16 dY that was
        cast) (csrc/ops/fp8_quant.cu fp8_quant_grad_t)."""
        q, src = self.fp8_quant_grad(dy, s_out, y, slope)
        return self._chwn(q), q if nhwc else torch.empty(0, dtype=E5M2), src

    # ------------------------------------------------------------------------------------------ fp8 delayed scaling
    @staticmethod
    def _delayed_cast(v, s_out, ring, seed, scale_fn, quant_fn):
        """One delayed-scaling call on the fp32 values v (csrc/ops/fp8_quant.cu, "Delayed scaling"): s from the amax of
        the 15 history slots other than the position (seed: from v's own amax, then written into every slot), an infinite
        element cast as NaN, v's amax recorded into the position's slot, the position advanced.  Returns the fp8 values."""
        hist = ring[:AMAX_HISTORY].view(torch.float32)
        pos = int(ring[AMAX_HISTORY])
        amax = _nan_free_abs(v).amax() if v.numel() else torch.zeros(())
        window = amax if seed else torch.cat([hist[:pos], hist[pos + 1:]]).amax()
        s = scale_fn(window)
        s_out.copy_(torch.div(torch.ones_like(s), s).reshape(s_out.shape))
        q = quant_fn(torch.where(torch.isinf(v), torch.full_like(v, float("nan")), v), s)
        if seed:
            hist.fill_(float(amax))
        else:
            hist[pos] = amax
        ring[AMAX_HISTORY] = (pos + 1) % AMAX_HISTORY
        return q

    def _delayed_nhwc(self, v, s_out, ring, seed, dtype, scale_fn, quant_fn):
        n, c, h, w = v.shape
        full = torch.zeros((n, (c + 15) // 16 * 16, h, w), dtype=dtype).contiguous(memory_format=CL)
        full[:, :c].copy_(self._delayed_cast(v, s_out, ring, seed, scale_fn, quant_fn))
        return full[:, :c]

    def fp8_quant_act_delayed(self, x, s_out, ring, seed):
        """fp8_quant_act with delayed scaling: ring int32 [AMAX_HISTORY + 3] (csrc/ops/fp8_quant.cu fp8_quant_act_delayed)."""
        return self._delayed_nhwc(x.float(), s_out, ring, seed, E4M3, e4m3_scale, e4m3_quant)

    def fp8_quant_act_t_delayed(self, x, s_out, ring, seed, nhwc):
        """(the batch-innermost e4m3 copy, the NHWC copy when nhwc else an empty tensor), one scale for both
        (csrc/ops/fp8_quant.cu fp8_quant_act_t_delayed)."""
        q = self.fp8_quant_act_delayed(x, s_out, ring, seed)
        return self._chwn(q), q if nhwc else torch.empty(0, dtype=E4M3)

    def fp8_quant_grad_delayed(self, dy, s_out, ring, seed, y, slope):
        """fp8_quant_grad with delayed scaling (csrc/ops/fp8_quant.cu fp8_quant_grad_delayed)."""
        src = dy if y is None else _nhwc(torch.where(y.float() > 0, dy.float(), dy.float() * slope).to(BF16))
        return self._delayed_nhwc(src.float(), s_out, ring, seed, E5M2, e5m2_scale, e5m2_quant), src

    def fp8_quant_grad_t_delayed(self, dy, s_out, ring, seed, y, slope, nhwc):
        """fp8_quant_grad_t with delayed scaling (csrc/ops/fp8_quant.cu fp8_quant_grad_t_delayed)."""
        q, src = self.fp8_quant_grad_delayed(dy, s_out, ring, seed, y, slope)
        return self._chwn(q), q if nhwc else torch.empty(0, dtype=E5M2), src

    def conv_wgrad_fp8(self, dy8t, x8t, s_dy, s_x, dw, kernel, pad, groups, alpha, cgk):
        """dw[Cout, R*S*Cg] fp32 += alpha · s_dy · s_x · (stride-1 weight gradient of the fp8 copies)
        (csrc/gemm/conv_ops.cu conv_wgrad_fp8)."""
        r, s = kernel
        assert dy8t.shape[3] == x8t.shape[3] == chwn_images(dy8t.shape[3]) and cgk >= x8t.shape[0] // groups and cgk % 64 == 0
        assert tuple(dy8t.shape[1:3]) == (x8t.shape[1] + 2 * pad[0] - r + 1, x8t.shape[2] + 2 * pad[1] - s + 1)
        x = x8t.float().permute(3, 0, 1, 2)
        d = dy8t.float().permute(3, 0, 1, 2)
        cout, cg = d.shape[1], x.shape[1] // groups
        g = torch.nn.grad.conv2d_weight(x, (cout, cg, r, s), d, 1, tuple(pad), 1, groups)
        g = g.permute(0, 2, 3, 1).reshape(cout, r * s * cg)
        dw.add_(g * (s_dy.float().reshape(()) * s_x.float().reshape(())), alpha=alpha)

    def conv_dgrad_fp8(self, dy8, wt8, s_dy, s_wt, kernel, pad, groups, H, W, mask, slope):
        """Stride-1 data gradient conv_transpose(dy8, wt8) · s_dy · s_wt[ci], producer-ReLU mask in the epilogue
        (csrc/gemm/conv_ops.cu conv_dgrad_fp8)."""
        r, s = kernel
        assert tuple(dy8.shape[2:]) == (H + 2 * pad[0] - r + 1, W + 2 * pad[1] - s + 1), (tuple(dy8.shape), H, W)
        cout = dy8.shape[1]
        cout_g = cout // groups
        cg = wt8.shape[0] // groups
        cok = wt8.shape[1] // (r * s)
        w = wt8.float().reshape(groups, cg, r, s, cok)[..., :cout_g]               # g, ci, r, s, co
        w4 = w.permute(0, 4, 1, 2, 3).reshape(cout, cg, r, s)
        full = F.conv_transpose2d(dy8.float(), w4, None, 1, 0, 0, groups)
        dx = full[:, :, pad[0]: pad[0] + H, pad[1]: pad[1] + W]
        dx = dx * (s_dy.float().reshape(()) * s_wt.float()).view(1, -1, 1, 1)
        if mask is not None:
            dx = torch.where(mask.float() > 0, dx, dx * slope)
        return _nhwc(dx.to(BF16))

    # ------------------------------------------------------------------------------------------ elementwise
    def relu_fwd(self, x, slope):
        return _act(x.float(), True, slope).to(BF16)

    def relu_bwd(self, y, dy, slope):
        assert y.stride() == dy.stride(), "relu_bwd: layout mismatch"
        return torch.where(y.float() > 0, dy.float(), dy.float() * slope).to(BF16)

    def relu_bwd_nhwc(self, y, dy, slope):
        """Pitch-aware variant (y / dy may be channel slices of wider NHWC buffers); dense NHWC result."""
        return _nhwc(torch.where(y.float() > 0, dy.float(), dy.float() * slope).to(BF16))

    def dropout_apply(self, x, ratio, seed, seed_dev):
        """The same (seed, iteration, element) -> keep map for forward and backward (csrc/ops/elementwise.cu:178-222);
        the emulation draws the map from a generator keyed the same way instead of the kernel's integer hash."""
        it = int(seed_dev.item()) if seed_dev is not None else 0
        g = torch.Generator().manual_seed((int(seed) ^ (it * 0x9E3779B97F4A7C15)) & 0x7FFFFFFFFFFFFFFF)
        keep = torch.rand(x.numel(), generator=g) > ratio
        flat = _storage_order_flat(x).float() * keep * (1.0 / (1.0 - ratio))
        y = torch.empty_like(x)                                   # dense input: same strides
        torch.as_strided(y, (x.numel(),), (1,)).copy_(flat)       # the map is indexed by memory position, like the kernel's
        return y

    def colsum(self, dy, rows, C, ld, out, alpha, accumulate):
        """out[c] (+)= alpha · Σ_rows dy[row*ld + c] over the tensor's memory (csrc/ops/elementwise.cu:224-268)."""
        v = torch.as_strided(dy, (rows, C), (ld, 1), dy.storage_offset()).float().sum(0) * alpha
        if accumulate:
            out.add_(v)
        else:
            out.copy_(v)

    def transform_nhwc(self, x, h_off, w_off, flip, mean, scale, OH, OW, cp, opad, wextra, hextra, s2d):
        """Crop / mirror / mean / scale / channel-pad / spatial pre-pad (/ space-to-depth by 4) in one pass
        (csrc/ops/elementwise.cu:19-148).  Output: bf16 channels-last [N, cp, OH+2opad+hextra, OW+2opad+wextra],
        or [N, 64, ·/4, ·/4] with channel (y%4)*16 + (x%4)*4 + c when s2d."""
        n, c, h, w = x.shape
        xf = x.float()
        if mean is not None:
            xf = xf - (mean.view(1, c, 1, 1) if mean.numel() == c else mean.view(1, c, h, w))
        outs = []
        for i in range(n):
            ho, wo = int(h_off[i]), int(w_off[i])
            t = xf[i, :, ho: ho + OH, wo: wo + OW]
            if int(flip[i]):
                t = t.flip(-1)
            outs.append(t)
        t = torch.stack(outs) * scale
        t = F.pad(t, (opad, opad + wextra, opad, opad + hextra, 0, cp - c))
        if s2d:
            hq, wq = t.shape[2] // 4, t.shape[3] // 4
            t = t.view(n, cp, hq, 4, wq, 4).permute(0, 2, 4, 3, 5, 1).reshape(n, hq, wq, 64)
            return t.to(BF16).permute(0, 3, 1, 2)
        return _nhwc(t.to(BF16))

    # ------------------------------------------------------------------------------------------ LRN / pooling
    def lrn_fwd(self, x, size, alpha, beta, fuse_relu):
        xf = x.float()
        if fuse_relu:
            xf = xf.clamp_min(0)
        return _nhwc(R.lrn_across(xf, size, alpha, beta).to(BF16))

    def lrn_bwd(self, x, dy, size, alpha, beta, fuse_relu):
        """dx of across-channel LRN; with fuse_relu, of LRN(ReLU(x)) and zero where x is not positive
        (csrc/ops/lrn.cu:140-215)."""
        xr = x.float().clamp_min(0) if fuse_relu else x.float()
        xf = xr.detach().requires_grad_(True)
        with torch.enable_grad():
            y = R.lrn_across(xf, size, alpha, beta)
        (dx,) = torch.autograd.grad(y, xf, dy.float())
        if fuse_relu:
            dx = dx * (x.float() > 0)
        return _nhwc(dx.to(BF16))

    @staticmethod
    def _pool_plane(in_hw, out_hw, k, s, p):
        """Extent of the zero-based plane that holds the image at offset (p_h, p_w) and every window of Caffe's
        ceil-mode pooling: with k < s and no pad, the last window may start past the image."""
        return tuple(max((o - 1) * st + kk, p_ + i) for i, o, kk, st, p_ in zip(in_hw, out_hw, k, s, p))

    def _pool_windows(self, x, k, s, p, oh, ow, fill):
        """(N, C, OH, OW, kh*kw) windows in row-major tap order over the plane, `fill` outside the image; plane extent."""
        n, c, h, w = x.shape
        ph_, pw_ = self._pool_plane((h, w), (oh, ow), k, s, p)
        plane = torch.full((n, c, ph_, pw_), fill, dtype=torch.float32)
        plane[:, :, p[0]: p[0] + h, p[1]: p[1] + w] = x.float()
        cols = plane.as_strided((n, c, oh, ow, k[0], k[1]), (c * ph_ * pw_, ph_ * pw_, s[0] * pw_, s[1], pw_, 1))
        return cols.reshape(n, c, oh, ow, k[0] * k[1]), (ph_, pw_)

    @staticmethod
    def _ave_inv(in_hw, out_hw, k, s, p):
        """[OH, OW] 1 / pool_size, pool_size from the window clipped to H + pad (0 for an empty window)."""
        ext = []
        for i, o, kk, st, p_ in zip(in_hw, out_hw, k, s, p):
            start = torch.arange(o) * st - p_
            ext.append(torch.clamp(start + kk, max=i + p_) - start)
        size = ext[0].view(-1, 1) * ext[1].view(1, -1)
        return torch.where(size > 0, 1.0 / size.clamp_min(1).float(), torch.zeros(()))

    @staticmethod
    def _tap_to_plane(tap, k, s, pw_):
        oh, ow = tap.shape[2:]
        rows = torch.arange(oh).view(1, 1, oh, 1) * s[0] + tap // k[1]
        cols = torch.arange(ow).view(1, 1, 1, ow) * s[1] + tap % k[1]
        return rows * pw_ + cols

    def pool_fwd(self, x, is_max, k, s, p, oh, ow, want_idx):
        """(y, idx) with Caffe's window rules (csrc/ops/pool.cu:28-110): the window is clipped to the image for MAX and
        the sum, to H + pad for the AVE divisor; the first maximum in row-major window order wins; an empty window gives
        -inf (MAX) or 0 (AVE).  The kernel's idx is the in-window tap of the maximum; it is opaque to the caller, so the
        emulation stores the index into the padded plane of _pool_plane instead."""
        h, w = x.shape[2:]
        cols, (_, pw_) = self._pool_windows(x, k, s, p, oh, ow, float("-inf") if is_max else 0.0)
        if is_max:
            y, tap = cols.max(-1)
            return _nhwc(y.to(BF16)), (self._tap_to_plane(tap, k, s, pw_) if want_idx else torch.empty(0, dtype=torch.int64))
        return _nhwc((cols.sum(-1) * self._ave_inv((h, w), (oh, ow), k, s, p)).to(BF16)), torch.empty(0, dtype=torch.int64)

    def pool_bwd(self, dy, idx, is_max, in_hw, k, s, p):
        n, c, oh, ow = dy.shape
        h, w = in_hw
        ph_, pw_ = self._pool_plane((h, w), (oh, ow), k, s, p)
        if is_max:
            plane = torch.zeros(n, c, ph_ * pw_, dtype=torch.float32)
            plane.scatter_add_(2, idx.reshape(n, c, -1), dy.float().reshape(n, c, -1))
        else:
            g = dy.float() * self._ave_inv((h, w), (oh, ow), k, s, p)
            plane = torch.zeros(n, c, ph_, pw_, dtype=torch.float32)
            for i in range(k[0]):
                for j in range(k[1]):
                    plane[:, :, i: i + (oh - 1) * s[0] + 1: s[0], j: j + (ow - 1) * s[1] + 1: s[1]] += g
        dx = plane.view(n, c, ph_, pw_)[:, :, p[0]: p[0] + h, p[1]: p[1] + w]
        return _nhwc(dx.to(BF16))

    # ------------------------------------------------------------------------------------------ layer kernels (round 2)
    @staticmethod
    def _like(ref, v):
        """bf16 result with the strides of ``ref`` (the kernels write storage order)."""
        out = torch.empty_like(ref, dtype=BF16)
        out.copy_(v)
        return out

    def unary_fwd(self, x, op, a, b, c):
        """csrc/ops/neuron.cu: 0 sigmoid, 1 tanh, 2 abs, 3 bnll, 4 power(a; scale b, shift c), 5 threshold(a)."""
        xf = x.float()
        y = [torch.sigmoid, torch.tanh, torch.abs, R.bnll, lambda t: R.power(t, a, b, c), lambda t: (t > a).float()][op](xf)
        return self._like(x, y)

    def unary_bwd(self, saved, dy, op, a, b, c):
        s, g = saved.float(), dy.float()
        if op == 0:
            d = g * s * (1 - s)
        elif op == 1:
            d = g * (1 - s * s)
        elif op == 2:
            d = g * torch.sign(s)
        elif op == 3:
            e = torch.exp(s.clamp_max(50.0))
            d = g * e / (e + 1)
        elif op == 4:
            v = c + b * s
            if a * b == 0:
                d = g * 0.0                   # power_layer.cu:42 (v.pow(a - 1) can be inf where v == 0)
            else:
                d = g * b if a == 1 else (g * 2 * b * v if a == 2 else g * a * b * v.pow(a - 1))
        else:
            d = torch.zeros_like(g)
        return self._like(dy, d)

    def eltwise_fwd(self, xs, op, coeffs, want_mask):
        fs = [x.float() for x in xs]
        mask = torch.empty(0, dtype=torch.uint8)
        if op == 0:
            y = fs[0]
            for t in fs[1:]:
                y = y * t
        elif op == 1:
            cs = coeffs or [1.0] * len(fs)
            y = sum(c * t for c, t in zip(cs, fs))
        else:
            st = torch.stack(fs)
            y, arg = st.max(0)
            if want_mask:
                mask = arg.to(torch.uint8)
        return self._like(xs[0], y), mask

    def eltwise_bwd(self, xs, dy, mask, op, coeffs, need):
        g = dy.float()
        outs = []
        for j in range(len(xs)):
            if not need[j]:
                outs.append(torch.empty(0, dtype=BF16))
                continue
            if op == 0:
                d = g
                for q, x in enumerate(xs):
                    if q != j:
                        d = d * x.float()
            elif op == 1:
                d = g * (coeffs[j] if coeffs else 1.0)
            else:
                d = g * (mask == j)
            outs.append(self._like(dy, d))
        return outs

    def softmax_fwd(self, x):
        return self._like(x, torch.softmax(x.float(), 1))

    def softmax_bwd(self, y, dy):
        yf, g = y.float(), dy.float()
        return self._like(y, yf * (g - (g * yf).sum(1, keepdim=True)))

    def mvn_fwd(self, x, nv, ac):
        xf = x.float()
        n, c = x.shape[:2]
        v = xf.reshape(n, 1, -1) if ac else xf.reshape(n, c, -1)
        mean = v.mean(2)
        var = ((v * v).mean(2) - mean * mean).clamp_min(0)
        inv = 1.0 / (var.sqrt() + 1e-10) if nv else torch.ones_like(mean)
        stats = torch.stack([mean.expand(n, c), inv.expand(n, c)], 2).contiguous()
        y = (xf - stats[:, :, 0].view(n, c, 1, 1)) * stats[:, :, 1].view(n, c, 1, 1)
        return _nhwc(y.to(BF16)), stats

    def mvn_bwd(self, y, dy, stats, nv, ac):
        g, yf = dy.float(), y.float()
        n, c = y.shape[:2]
        dims = (1, 2, 3) if ac else (2, 3)
        d = g - g.mean(dims, keepdim=True)
        if nv:
            d = (d - yf * (g * yf).mean(dims, keepdim=True)) * stats[:, :, 1].view(n, c, 1, 1)
        return _nhwc(d.to(BF16))

    def lrn_within_fwd(self, x, size, alpha, beta):
        return _nhwc(R.lrn_within(x.float(), size, alpha, beta).to(BF16))

    def lrn_within_bwd(self, x, dy, size, alpha, beta):
        xf = x.float().detach().requires_grad_(True)
        with torch.enable_grad():
            y = R.lrn_within(xf, size, alpha, beta)
        (dx,) = torch.autograd.grad(y, xf, dy.float())
        return _nhwc(dx.to(BF16))

    def stochastic_pool_fwd(self, x, k, s, oh, ow, train, seed, iter_dev):
        """(y, idx): idx is opaque to the caller (fed back to pool_bwd), so the emulation stores the plane index like
        its pool_fwd does (csrc/ops/lrn_within.cu: the kernel stores the in-window tap)."""
        cols, (_, pw_) = self._pool_windows(x, k, s, (0, 0), oh, ow, 0.0)
        run = cols.cumsum(-1)
        ssum = run[..., -1]                   # taps outside the image add 0: a pick never lands on one
        if not train:
            y = torch.where(ssum > 0, (cols * cols).sum(-1) / ssum, torch.zeros(()))
            return _nhwc(y.to(BF16)), torch.empty(0, dtype=torch.int64)
        it = int(iter_dev.item()) if iter_dev is not None else 0
        g = torch.Generator().manual_seed((int(seed) ^ (it * 0x9E3779B97F4A7C15)) & 0x7FFFFFFFFFFFFFFF)
        thr = torch.rand(ssum.shape, generator=g) * ssum
        tap = (run < thr.unsqueeze(-1)).sum(-1).clamp_max(cols.shape[-1] - 1)
        y = cols.gather(-1, tap.unsqueeze(-1)).squeeze(-1)
        return _nhwc(y.to(BF16)), self._tap_to_plane(tap, k, s, pw_)

    # ------------------------------------------------------------------------------------------ loss
    def softmax_xent(self, x, label, grad_scale, want_grad, want_prob):
        """(loss[1] fp32, dx like x, prob fp32): mean NLL over rows, dx = (p - onehot)·grad_scale/rows
        (csrc/ops/softmax_xent.cu:28-107)."""
        rows, c = x.shape
        prob = torch.softmax(x.float(), 1)
        lab = label.long().view(-1, 1)
        valid = (lab >= 0) & (lab < c)                 # a row whose label is out of range adds 0 to the loss
        lab = torch.where(valid, lab, torch.zeros_like(lab))
        picked = torch.where(valid, prob.gather(1, lab).clamp_min(torch.finfo(torch.float32).tiny), torch.ones(()))
        loss = (-picked.log().sum() / rows).reshape(1)
        dx = torch.empty(0, dtype=x.dtype)
        if want_grad:
            g = prob.clone()
            g.scatter_add_(1, lab, -valid.float())
            dx = (g * (grad_scale / rows)).to(x.dtype)
        return loss, dx, (prob if want_prob else torch.empty(0))

    # ------------------------------------------------------------------------------------------ optimizer
    def fused_update(self, w, g, h, wb, lr, momentum, decay, rule, l1, delta, gscale, lr_dev, rearm=False):
        """One optimizer step in place on (w, h) + refresh of the bf16 shadow in the master's storage order
        (csrc/comm/fused_update.cu:30-108).  rule 0 SGD, 1 Nesterov, 2 AdaGrad."""
        for t in (g, h):
            assert t.shape == w.shape and all(t.stride(d) == w.stride(d) for d in range(w.dim()) if w.shape[d] > 1), \
                "fused_update: layout mismatch"
        if lr_dev is not None:
            lr = lr * float(lr_dev[0])
        self._step(w, g.float(), h, lr, momentum, decay, rule, l1, delta, gscale)
        if rearm:
            g.zero_()                       # persistent accumulation buffer: left zeroed for the next step's wgrad
        if wb is not None:
            wb.view(-1).copy_(_storage_order_flat(w))

    def fused_update_multi(self, ws, gs, hs, wbs, lrs, decays, rearms, momentum, rule, l1, delta, gscale, lr_dev):
        """Many tensors, one launch (csrc/comm/fused_update.cu: fused_update_multi_kernel): per-tensor lr / decay / re-arm."""
        for w, g, h, wb, lr, decay, rearm in zip(ws, gs, hs, wbs, lrs, decays, rearms):
            self.fused_update(w, g, h, wb if wb.numel() else None, lr, momentum, decay, rule, l1, delta, gscale, lr_dev,
                              bool(rearm))

    # ------------------------------------------------------------------------------------------ multi-rank peer memory
    # The kernels address other ranks' memory by raw pointer (NVLink peer mappings of one symmetric arena per rank).
    # On the CPU the arena is a POSIX shared-memory segment per rank, mapped by every rank (EmulatedArena below); the
    # "pointers" are the addresses of those mappings in this process and resolve through the arena registry.  Ranks are
    # processes, the flag protocol is the kernels' (st.release / spin on ld.acquire become plain stores and polling).
    _K_MAX_RANKS = 8

    @staticmethod
    def _mem(ptr: int, nbytes: int, dtype) -> torch.Tensor:
        for base, size, buf in EmulatedArena.mappings:
            if base <= ptr and ptr + nbytes <= base + size:
                return buf[ptr - base: ptr - base + nbytes].view(dtype)
        raise RuntimeError(f"emulated peer op: address {ptr:#x} (+{nbytes}) is not inside a mapped arena")

    @staticmethod
    def _epoch(epoch: int, epoch_dev) -> int:
        return (int(epoch) + (int(epoch_dev[0]) if epoch_dev is not None else 0)) & 0xFFFFFFFF

    @staticmethod
    def _wait_ge(word: torch.Tensor, value: int, what: str, timeout_s: float = 60.0) -> None:
        import time
        t0 = time.time()
        while (int(word) & 0xFFFFFFFF) < value:
            if time.time() - t0 > timeout_s:
                raise RuntimeError(f"emulated peer op: timed out waiting for {what} >= {value} (have {int(word)})")
            time.sleep(0.0002)

    def _flags(self, ptr: int) -> torch.Tensor:
        return self._mem(ptr, 8 * self._K_MAX_RANKS * 4, torch.int32)            # [slot][rank] u32, 8 slots

    def _peer_barrier(self, flag_ptrs, rank, phase, ep):
        """csrc/comm/fused_update.cu:150-158."""
        world = len(flag_ptrs)
        for t in range(world):
            self._flags(flag_ptrs[t])[phase * self._K_MAX_RANKS + rank] = ep
        mine = self._flags(flag_ptrs[rank])
        for t in range(world):
            self._wait_ge(mine[phase * self._K_MAX_RANKS + t], ep, f"barrier phase {phase} flag of rank {t}")

    @staticmethod
    def _step(w, g, h, lr, momentum, decay, rule, l1, delta, gscale):
        g = g * gscale
        if decay != 0:
            g = g + decay * (torch.sign(w) if l1 else w)
        if rule == 0:
            h.mul_(momentum).add_(g, alpha=lr)
            w.sub_(h)
        elif rule == 1:
            h_old = h.clone()
            h.mul_(momentum).add_(g, alpha=lr)
            w.sub_((1.0 + momentum) * h - momentum * h_old)
        else:
            h.add_(g * g)
            w.sub_(lr * g / (h.sqrt() + delta))

    def allreduce_sgd(self, g_ptrs, w_ptrs, wb_ptrs, flag_ptrs, g_mc, w_mc, h, n, rank, epoch, one_shot, done_counter,
                      lr, momentum, decay, rule, l1, delta, gscale, max_ctas, lr_dev, epoch_dev):
        """All-reduce + optimizer step + weight broadcast in one launch (csrc/comm/fused_update.cu:160-262).
        one-shot: every rank reduces the whole bucket and steps its own copy; two-shot: rank r reduces and steps shard
        r (its slice of the history) and writes the new weights / bf16 shadows into every rank's arena."""
        world = len(g_ptrs)
        ep = self._epoch(epoch, epoch_dev)
        if lr_dev is not None:
            lr = lr * float(lr_dev[0])
        self._peer_barrier(flag_ptrs, rank, 0, ep)
        n4 = n // 4
        lo, hi = 0, n4
        if not one_shot:
            per = (n4 + world - 1) // world
            lo = min(n4, per * rank)
            hi = min(n4, lo + per)
        sl = slice(4 * lo, 4 * hi)
        g = self._mem(g_ptrs[rank], n * 4, torch.float32)[sl].clone()
        for q in range(1, world):
            g += self._mem(g_ptrs[(rank + q) % world], n * 4, torch.float32)[sl]
        w = self._mem(w_ptrs[rank], n * 4, torch.float32)[sl].clone()
        hv = h[:n][sl]
        self._step(w, g, hv, lr, momentum, decay, rule, l1, delta, gscale)
        targets = [rank] if one_shot else [(rank + q) % world for q in range(world)]
        for p in targets:
            self._mem(w_ptrs[p], n * 4, torch.float32)[sl] = w
            if wb_ptrs:
                self._mem(wb_ptrs[p], n * 2, BF16)[sl] = w.to(BF16)
        self._peer_barrier(flag_ptrs, rank, 1, ep)

    def allreduce_sgd_multi(self, base_ptrs, mc_base, flag_ptrs, g_offs, w_offs, wb_offs, hists, ns, one_shots, lrs, decays,
                            rank, epoch, done_counter, momentum, rule, l1, delta, gscale, max_ctas, lr_dev, epoch_dev):
        """One launch per bucket: up to 4 segments behind one barrier pair; the kernel re-arms (zeroes) the gradient
        staging it consumed — the shard owner in every rank's arena for two-shot segments, each rank its own copy after
        the closing barrier for one-shot segments (csrc/comm/fused_update.cu: allreduce_sgd_multi_kernel)."""
        world = len(base_ptrs)
        ep = self._epoch(epoch, epoch_dev)
        lr_glob = float(lr_dev[0]) if lr_dev is not None else 1.0
        self._peer_barrier(flag_ptrs, rank, 0, ep)
        for g_off, w_off, wb_off, h, n, one_shot, lr, decay in zip(g_offs, w_offs, wb_offs, hists, ns, one_shots, lrs, decays):
            n4 = n // 4
            lo, hi = 0, n4
            if not one_shot:
                per = (n4 + world - 1) // world
                lo = min(n4, per * rank)
                hi = min(n4, lo + per)
            sl = slice(4 * lo, 4 * hi)
            g = self._mem(base_ptrs[0] + g_off, n * 4, torch.float32)[sl].clone()
            for q in range(1, world):
                g += self._mem(base_ptrs[q] + g_off, n * 4, torch.float32)[sl]
            if not one_shot:
                for q in range(world):
                    self._mem(base_ptrs[q] + g_off, n * 4, torch.float32)[sl] = 0.0
            w = self._mem(base_ptrs[rank] + w_off, n * 4, torch.float32)[sl].clone()
            self._step(w, g, h[:n][sl], lr * lr_glob, momentum, decay, rule, l1, delta, gscale)
            for p in ([rank] if one_shot else range(world)):
                self._mem(base_ptrs[p] + w_off, n * 4, torch.float32)[sl] = w
                if wb_off >= 0:
                    self._mem(base_ptrs[p] + wb_off, n * 2, BF16)[sl] = w.to(BF16)
        self._peer_barrier(flag_ptrs, rank, 1, ep)
        for g_off, n, one_shot in zip(g_offs, ns, one_shots):
            if one_shot:
                self._mem(base_ptrs[rank] + g_off, n * 4, torch.float32).zero_()

    # ---- bounded staleness on the arena (csrc/comm/fused_update.cu: ssp_delta_kernel / ssp_fold_kernel) ----------------
    _SSP_READY, _SSP_CONSUMED = 5, 6

    def ssp_delta(self, base_ptrs, flag_ptrs, g_offs, w_offs, wb_offs, d_offs, ring_stride, hists, ns, lrs, decays, rank, ring,
                  staleness, done_counter, state, momentum, rule, l1, delta, gscale, max_ctas, lr_dev, clock_dev):
        """Own optimizer step on the local gradient (applied at once), the step itself stored in slot clock % ring of this
        rank's delta ring; then the fold of the peers' deltas is planned: clocks <= clock - staleness are due (waited
        for), anything a peer has published beyond that is taken along."""
        world, KM = len(base_ptrs), self._K_MAX_RANKS
        c = int(clock_dev[0]) & 0xFFFFFFFF
        lr_glob = float(lr_dev[0]) if lr_dev is not None else 1.0
        mine = self._flags(flag_ptrs[rank])
        if c >= ring:
            for q in range(world):
                if q != rank:
                    self._wait_ge(mine[self._SSP_CONSUMED * KM + q], c - ring + 1, f"rank {q} consuming my clock {c - ring}")
        for g_off, w_off, wb_off, d_off, h, n, lr, decay in zip(g_offs, w_offs, wb_offs, d_offs, hists, ns, lrs, decays):
            g = self._mem(base_ptrs[rank] + g_off, n * 4, torch.float32)
            w = self._mem(base_ptrs[rank] + w_off, n * 4, torch.float32)
            w0 = w.clone()
            wn = w.clone()
            self._step(wn, g.clone(), h[:n], lr * lr_glob, momentum, decay, rule, l1, delta, gscale)
            g.zero_()
            w.copy_(wn)
            self._mem(base_ptrs[rank] + wb_off, n * 2, BF16).copy_(wn.to(BF16))
            self._mem(base_ptrs[rank] + d_off + (c % ring) * ring_stride, n * 4, torch.float32).copy_(w0 - wn)
        for q in range(world):
            if q == rank:
                continue
            self._flags(flag_ptrs[q])[self._SSP_READY * KM + rank] = c + 1
            lo = int(state[q])
            must = max(c + 1 - staleness, 0)
            if must > lo:
                self._wait_ge(mine[self._SSP_READY * KM + q], must, f"delta of rank {q} for clock {must - 1}")
            avail = int(mine[self._SSP_READY * KM + q]) & 0xFFFFFFFF
            hi = min(max(avail, lo), lo + ring)
            state[KM + q] = hi
            state[2 * KM] = max(int(state[2 * KM]), max(c + 1 - hi, 0))

    def ssp_fold(self, base_ptrs, flag_ptrs, w_offs, wb_offs, d_offs, ring_stride, ns, rank, ring, done_counter, state, drain,
                 max_ctas):
        """W -= sum of the planned (or, draining, of all published) peer deltas, read from the peers' rings; then the
        producers are told how far their rings have been consumed."""
        world, KM = len(base_ptrs), self._K_MAX_RANKS
        mine = self._flags(flag_ptrs[rank])
        rng = {}
        for q in range(world):
            if q == rank:
                continue
            lo = int(state[q])
            hi = (int(mine[self._SSP_READY * KM + q]) & 0xFFFFFFFF) if drain else int(state[KM + q])
            rng[q] = (lo, max(hi, lo))
        if any(hi > lo for lo, hi in rng.values()):
            for w_off, wb_off, d_off, n in zip(w_offs, wb_offs, d_offs, ns):
                w = self._mem(base_ptrs[rank] + w_off, n * 4, torch.float32)
                acc = torch.zeros(n)
                for q, (lo, hi) in rng.items():
                    for cc in range(lo, hi):
                        acc += self._mem(base_ptrs[q] + d_off + (cc % ring) * ring_stride, n * 4, torch.float32)
                w.sub_(acc)
                self._mem(base_ptrs[rank] + wb_off, n * 2, BF16).copy_(w.to(BF16))
        for q, (lo, hi) in rng.items():
            state[q] = hi
            self._flags(flag_ptrs[q])[self._SSP_CONSUMED * KM + rank] = hi

    def peer_push(self, src, dst_ptrs, dst_mc, flag_ptrs, rank, slot, epoch, signal, done_counter, wait_slot, epoch_dev):
        """Payload into every rank's arena, then (optionally) this rank's epoch flag on every peer
        (csrc/comm/fused_update.cu:264-330)."""
        world = len(dst_ptrs)
        ep = self._epoch(epoch, epoch_dev)
        if wait_slot >= 0:
            mine = self._flags(flag_ptrs[rank])
            for t in range(world):
                self._wait_ge(mine[wait_slot * self._K_MAX_RANKS + t], (ep - 1) & 0xFFFFFFFF, f"consumed flag of rank {t}")
        raw = src.contiguous().view(-1).view(torch.uint8)
        for q in range(world):
            self._mem(dst_ptrs[(rank + q) % world], raw.numel(), torch.uint8).copy_(raw)
        if signal:
            for t in range(world):
                self._flags(flag_ptrs[t])[slot * self._K_MAX_RANKS + rank] = ep

    def peer_signal(self, flag_ptrs, rank, slot, epoch, epoch_dev):
        ep = self._epoch(epoch, epoch_dev)
        for t in range(len(flag_ptrs)):
            self._flags(flag_ptrs[t])[slot * self._K_MAX_RANKS + rank] = ep

    def _sfb_outer(self, u_ptrs, v_ptrs, Mb, N, K, flags, epoch, src_rot, epoch_dev):
        ep = self._epoch(epoch, epoch_dev)
        P = len(u_ptrs)
        g = torch.zeros(N, K)
        for s_ in range(P):
            src = (s_ + src_rot) % P
            if flags is not None:
                self._wait_ge(flags[src], ep, f"factor flag of rank {src}")
            u = self._mem(u_ptrs[src], Mb * N * 2, BF16).view(Mb, N).float()
            v = self._mem(v_ptrs[src], Mb * K * 2, BF16).view(Mb, K).float()
            g += u.t() @ v
        return g

    def sfb_outer_sgd(self, u_ptrs, v_ptrs, Mb, N, K, w, h, wb, alpha, lr, momentum, decay, rule, l1, delta, flags, epoch,
                      src_rot, bn, max_ctas, lr_dev, epoch_dev=None):
        """W -= step(alpha * sum_p U_p^T V_p) with the factors read from this rank's staging slots, gated per source by
        its epoch flag (csrc/gemm/gemm_ops.cu:256-290, umma_gemm.cuh producer loop)."""
        g = self._sfb_outer(u_ptrs, v_ptrs, Mb, N, K, flags, epoch, src_rot, epoch_dev)
        if lr_dev is not None:
            lr = lr * float(lr_dev[0])
        self._step(w, g.view_as(w), h, lr, momentum, decay, rule, l1, delta, alpha)
        if wb is not None:
            wb.view(-1).copy_(_storage_order_flat(w))

    def sfb_outer_f32(self, u_ptrs, v_ptrs, Mb, N, K, out, alpha, flags, epoch, src_rot, bn, max_ctas, epoch_dev=None):
        out.copy_(self._sfb_outer(u_ptrs, v_ptrs, Mb, N, K, flags, epoch, src_rot, epoch_dev) * alpha)


class EmulatedArena:
    """``parallel/fused.py::SymmetricArena`` on host shared memory: one POSIX segment per rank, mapped by every rank.
    ``base_ptrs[p]`` is the address of rank p's segment in THIS process — what the peer-mapped device pointers are on
    the GPU.  No multicast object (``multicast_ptr == 0`` selects the P2P code paths)."""
    mappings = []          # (base address, size, uint8 tensor) of every segment mapped in this process

    def __init__(self, nbytes: int, rank_ctx):
        import os
        from multiprocessing import shared_memory
        self.rank, self.world, self.device = rank_ctx.rank, rank_ctx.world_size, rank_ctx.device
        nbytes = (nbytes + (2 << 20) - 1) // (2 << 20) * (2 << 20)
        job = f"psd{os.environ.get('MASTER_PORT', '0')}_{EmulatedArena._generation(rank_ctx)}" \
              f"_n{getattr(rank_ctx, 'node_id', 0)}"              # emulated "nodes" share one /dev/shm
        name = f"{job}_{self.rank}"
        try:
            self._own = shared_memory.SharedMemory(name=name, create=True, size=nbytes)      # new segments are zero-filled
        except FileExistsError:                                 # left behind by a run that was killed
            stale = shared_memory.SharedMemory(name=name)
            stale.close()
            stale.unlink()
            self._own = shared_memory.SharedMemory(name=name, create=True, size=nbytes)
        rank_ctx.barrier()
        self._segs = [self._own if p == self.rank else shared_memory.SharedMemory(name=f"{job}_{p}")
                      for p in range(self.world)]
        try:                                                    # attaching registers the peer's segment with OUR resource
            from multiprocessing import resource_tracker        # tracker too (Python < 3.13), which then tries to unlink it
            for p, seg in enumerate(self._segs):                # a second time at exit: only the creator cleans up
                if p != self.rank:
                    resource_tracker.unregister(seg._name, "shared_memory")
        except Exception:
            pass
        tensors = [torch.frombuffer(seg.buf, dtype=torch.uint8, count=nbytes) for seg in self._segs]
        self.buf = tensors[self.rank]
        self.base_ptrs = [t.data_ptr() for t in tensors]
        for t in tensors:
            EmulatedArena.mappings.append((t.data_ptr(), nbytes, t))
        self.multicast_ptr = 0
        self.offset = 0
        self.nbytes = nbytes
        rank_ctx.barrier()

    _gen = 0

    @staticmethod
    def _generation(rank_ctx) -> int:
        EmulatedArena._gen += 1            # every rank builds its arenas in the same order
        return EmulatedArena._gen

    def carve(self, nbytes: int) -> int:
        off = self.offset
        self.offset = (off + nbytes + 255) // 256 * 256
        if self.offset > self.nbytes:
            raise RuntimeError("symmetric arena exhausted")
        return off

    def view(self, off: int, shape, dtype) -> torch.Tensor:
        n = 1
        for d in shape:
            n *= d
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        return self.buf[off: off + nbytes].view(dtype).view(*shape)

    def peer_ptrs(self, off: int):
        return [b + off for b in self.base_ptrs]

    def mc_ptr(self, off: int) -> int:
        return 0

    def close(self):
        EmulatedArena.mappings[:] = [m for m in EmulatedArena.mappings if m[0] not in self.base_ptrs]
        self.buf = None
        for seg in self._segs:
            try:
                seg.close()
            except BufferError:
                pass
        try:
            self._own.unlink()
        except FileNotFoundError:
            pass
