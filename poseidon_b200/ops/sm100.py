"""The sm100 engine: every hot op runs a hand-written sm_90a kernel from ``csrc/``.

Conventions
-----------
* activations: bf16, logical NCHW with channels-last (NHWC) memory; channel counts multiples of 8
  (first-layer images are padded to 4 channels and spatially pre-padded by the transform kernel);
* learnable blobs: fp32 master (``nn.Parameter``; conv weights physically [Cout][R][S][Cg]) plus a
  bf16 shadow that the fused optimizer kernels refresh in place;
* backward is explicit (``torch.autograd.Function``) so that weight gradients land where the DWBP /
  SFB engines want them and ReLU masks are applied inside the neighbouring kernels' epilogues.

Nothing here silently falls back to a library kernel for the ops the engine claims (conv, inner product,
LRN, pooling, softmax-loss, dropout, transform): unsupported shapes raise, except where noted as
``torch_engine`` delegation for cold ops (within-channel LRN, stochastic pooling, ...).
"""
from __future__ import annotations

import os
from typing import Optional

import torch

from . import reference as R
from . import torch_engine as TE
from .build import load_extension

_ops = None
_emulate = os.environ.get("POSEIDON_EMULATE", "0") == "1"


def emulating() -> bool:
    """True when the engine runs on ops/emulate.py's CPU stand-ins for the kernels (tests of the Python side only)."""
    return _emulate


def set_emulation(on: bool) -> None:
    """Switch between the compiled kernels and their CPU emulation (never implicit: POSEIDON_EMULATE=1 or this call)."""
    global _emulate, _ops
    if bool(on) != _emulate:
        _emulate, _ops = bool(on), None


def active(device) -> bool:
    """Does the sm100 engine own tensors on this device?  (CUDA always; the CPU only under emulation.)"""
    return torch.device(device).type == "cuda" or _emulate


def _on(x: torch.Tensor) -> bool:
    return x.is_cuda or _emulate


def K():
    """torch.ops.poseidon, loading the in-tree extension on first use (fails loudly if absent)."""
    global _ops
    if _ops is None:
        from .counting import CountingOps
        if _emulate:
            from .emulate import EmulatedKernels
            _ops = CountingOps(EmulatedKernels())
        else:
            load_extension()
            _ops = CountingOps(torch.ops.poseidon)
            # schedule switches (A/B knobs; the defaults are what the kernels ship with)
            env = os.environ
            if "POSEIDON_PAIR_CTA" in env:
                torch.ops.poseidon.set_pair_cta(int(env["POSEIDON_PAIR_CTA"]))
            if "POSEIDON_CONV_PAIR" in env:
                torch.ops.poseidon.set_conv_pair(int(env["POSEIDON_CONV_PAIR"]))
            if "POSEIDON_CONV_MCAST" in env:
                torch.ops.poseidon.set_conv_mcast(int(env["POSEIDON_CONV_MCAST"]))
            if "POSEIDON_CONV_HALO" in env:
                torch.ops.poseidon.set_conv_halo(int(env["POSEIDON_CONV_HALO"]))
            if "POSEIDON_CONV_HALO_FPROP" in env:
                torch.ops.poseidon.set_conv_halo_fprop(int(env["POSEIDON_CONV_HALO_FPROP"]))
            if "POSEIDON_BULK_EPI" in env:
                torch.ops.poseidon.set_bulk_epilogue(int(env["POSEIDON_BULK_EPI"]))
    return _ops


CL = torch.channels_last


def to_nhwc_bf16(x: torch.Tensor) -> torch.Tensor:
    if x.dtype != torch.bfloat16:
        x = x.to(torch.bfloat16)
    if x.dim() == 4 and not (x.stride(1) == 1 or x.shape[1] == 1):
        x = x.contiguous(memory_format=CL)
    elif x.dim() == 4 and x.shape[1] == 1 and not x.is_contiguous(memory_format=CL):
        x = x.contiguous(memory_format=CL)
    return x


def _dense_pitch_ok(x: torch.Tensor) -> bool:
    """NHWC tensor whose only irregularity may be a pixel pitch > C (channel-slice view), starting on a 16-byte boundary
    (the kernels read pixels with 16-byte loads: a slice at a channel offset that is not a multiple of 8 is copied)."""
    if x.dim() != 4 or x.stride(1) != 1 or x.data_ptr() % 16 != 0:
        return False
    n, c, h, w = x.shape
    pitch = x.stride(3) if w > 1 else (x.stride(2) if h > 1 else (x.stride(0) if n > 1 else c))
    return (h == 1 or w == 1 or x.stride(2) == pitch * w) and (n == 1 or x.stride(0) == pitch * w * h) and pitch % 8 == 0


def as_kernel_input(x: torch.Tensor) -> torch.Tensor:
    x = x if x.dtype == torch.bfloat16 else x.to(torch.bfloat16)
    if x.dim() == 4 and _dense_pitch_ok(x):
        return x
    return x.contiguous(memory_format=CL) if x.dim() == 4 else x.contiguous()


def _pad64(c: int) -> int:
    """Per-tap slot count on the im2col-TMA path: c rounded up to a multiple of 64 if that costs <= 34 % extra work."""
    if c % 64 == 0 or c % 8 != 0 or c < 48:
        return c
    p = (c + 63) // 64 * 64
    return p if (p - c) * 100 <= 34 * c else c


FP8_MODES = ("off", "fprop", "fprop+dgrad", "fprop+dgrad+wgrad")


def resolve_fp8(mode: Optional[str] = None) -> str:
    """The engine's fp8 setting: ``mode`` when given, else ``POSEIDON_FP8`` (unset: "off").
    "fprop": eligible convolutions run their forward pass on e4m3 operands (data / weight gradients stay bf16).
    "fprop+dgrad": as "fprop", and eligible stride-1 convolutions also compute their data gradient from e5m2 dY and e4m3
    weights (weight / bias gradients stay bf16 / fp32).
    "fprop+dgrad+wgrad": as "fprop+dgrad", and eligible stride-1 convolutions also compute their weight gradient from
    e5m2 dY and e4m3 X (bias gradients stay fp32 from the bf16 dY)."""
    m = str(mode if mode is not None else os.environ.get("POSEIDON_FP8", "off")).lower()
    if m not in FP8_MODES:
        raise ValueError(f"fp8 must be one of {', '.join(FP8_MODES)}, got '{m}'")
    return m


def fp8_for_engine(engine: str, mode: Optional[str] = None) -> str:
    """The fp8 setting a net built for ``engine`` runs with.  Only the sm100 engine has fp8 kernels: asking another
    engine for fp8 explicitly is an error, and ``POSEIDON_FP8`` does not apply to it."""
    if engine == "sm100":
        return resolve_fp8(mode)
    if mode is not None and resolve_fp8(mode) != "off":
        raise ValueError(f"fp8='{mode}' needs the sm100 engine (engine is '{engine}')")
    return "off"


FP8_SCALINGS = ("current", "delayed")
AMAX_HISTORY = 16                       # slots of a delayed-scaling amax ring (csrc/ops/fp8_quant.cu kAmaxHistory)
_RING_WORDS = AMAX_HISTORY + 3          # + position, CTA ticket, running amax of the call in flight


def resolve_fp8_scaling(scaling: Optional[str] = None, fp8: str = "off") -> str:
    """How the fp8 quantisers of activations and dY choose their per-tensor scale: ``scaling`` when given, else
    ``POSEIDON_FP8_SCALING`` when the fp8 mode ``fp8`` is on (unset, or fp8 "off": "current").
    "current": just in time, from an amax pass over the tensor, then a cast pass.
    "delayed": from the amax history of the tensor's previous quantiser calls in device memory, in one pass (DESIGN §17);
    a tensor that grows past its history's amax saturates.  An explicit "delayed" with fp8 "off" is an error."""
    if scaling is None:
        if fp8 == "off":
            return "current"
        scaling = os.environ.get("POSEIDON_FP8_SCALING", "current")
    m = str(scaling).lower()
    if m not in FP8_SCALINGS:
        raise ValueError(f"fp8_scaling must be one of {', '.join(FP8_SCALINGS)}, got '{m}'")
    if m == "delayed" and fp8 == "off":
        raise ValueError("fp8_scaling='delayed' needs an fp8 mode (fp8 is 'off')")
    return m


def fp8_scaling_for_engine(engine: str, fp8: str, scaling: Optional[str] = None) -> str:
    """The fp8 scaling a net built for ``engine`` with the resolved fp8 mode ``fp8`` runs with.  Asking another engine for
    delayed scaling explicitly is an error, and ``POSEIDON_FP8_SCALING`` does not apply to it."""
    if engine == "sm100":
        return resolve_fp8_scaling(scaling, fp8)
    if scaling is not None:
        m = str(scaling).lower()
        if m not in FP8_SCALINGS:
            raise ValueError(f"fp8_scaling must be one of {', '.join(FP8_SCALINGS)}, got '{m}'")
        if m == "delayed":
            raise ValueError(f"fp8_scaling='{scaling}' needs the sm100 engine (engine is '{engine}')")
    return "current"


def _round128(c: int) -> int:
    return (c + 127) // 128 * 128


# =====================================================================================================
# Convolution
# =====================================================================================================
class ConvState:
    """Per-layer engine state: operand layouts + bf16 shadows, refreshed lazily by weight version."""

    def __init__(self, layer, cin_logical: int, fp8: Optional[str] = None, fp8_scaling: Optional[str] = None):
        self.layer = layer
        self.groups = layer.group
        self.R, self.S = layer.kernel
        self.Cout = layer.num_output
        cg = cin_logical // self.groups
        self.row_mode = cg % 8 != 0
        self.s2d = False
        self.pad8 = False
        self.Coutp = self.Cout             # physical output channels (multiple of 8)
        if (cg % 8 != 0 and cin_logical > 4) or (self.Cout // self.groups) % 8 != 0:
            # Channel counts that are not multiples of 8 (LeNet: 1 -> 20 -> 50): input and output channels are
            # zero-padded to the next multiple of 8 around the kernels (the operand carries zero rows / columns, the
            # output is a channel slice of the padded tensor).  Small legacy nets only — costs extra passes.
            if self.groups != 1:
                raise ValueError(f"sm100 conv '{layer.layer_name}': grouped convolution needs channel counts per "
                                 f"group that are multiples of 8 (got {cg} -> {self.Cout // self.groups})")
            self.row_mode = True           # operand derived lazily from the master; no arena shadow / gradient sink
            self.pad8 = True
            self.Cp = (cin_logical + 7) // 8 * 8
            self.Coutp = (self.Cout + 7) // 8 * 8
            self.Kw = self.R * self.S * self.Cp
        elif self.row_mode:
            if self.groups != 1:
                raise ValueError(f"sm100 conv '{layer.layer_name}': input channels {cin_logical} (group "
                                 f"{self.groups}) must be a multiple of 8 or <= 4 (first layer)")
            self.Cp = 4
            self.L = self.S * self.Cp
            self.Lp = (self.L + 7) // 8 * 8
            self.Kw = self.R * self.Lp
            if (layer.stride[1] * self.Cp) % 8:
                # odd horizontal stride (VGG conv1_1: 3x3/s1): kernel rows would start on 8-byte boundaries, so pad the
                # image to 8 channels instead and run it as an ordinary TAP-mode conv (K = R*S*8)
                self.pad8 = True
                self.Cp = 8
                self.Kw = self.R * self.S * 8
            else:
                self._try_s2d(layer)
        else:
            self.Cp = cin_logical
            self.Kw = self.R * self.S * cg
        self.cg = self.Cp // self.groups
        self.cin_logical = cin_logical
        # Channel-padded K for the TMA im2col path: when C_g is not a multiple of 64 (AlexNet conv2: 48, GoogLeNet:
        # 96 / 112 / 144 / 160 / 480 / 528 ...) the per-tap slot count is rounded up to 64 as long as that wastes at
        # most a third of the MMA work; the TMA zero-fills the extra slots, the weight operand carries zeros there.
        self.cgk = self.cg            # K slots per tap of the fprop / wgrad operand
        self.cok = self.Cout // self.groups      # K slots per tap of the dgrad operand
        # Opt-in (POSEIDON_PAD_K=1): numerically validated (tests/test_zz_padded_channels_gpu.py); its effect on throughput is
        # not measured on H100.
        if not self.row_mode and os.environ.get("POSEIDON_PAD_K", "0") == "1":
            self.cgk = _pad64(self.cg)
            self.cok = _pad64(self.Cout // self.groups)
        # fp8 forward (opt-in): e4m3 operands quantised on every forward from the input and the fp32 master, Cgk8 slots
        # per tap (Cg rounded up to 128: one 128-byte K block); decided once here
        mode = resolve_fp8(fp8)
        self.fp8, self.fp8_reason = False, "fp8 off"
        if mode != "off":
            self.fp8, self.fp8_reason = self._fp8_eligible(layer)
        self.cgk8 = _round128(self.cg) if self.fp8 else 0
        self.s_x: Optional[torch.Tensor] = None       # fp8 dequantisation scales, written by the quantisers every forward
        self.s_w: Optional[torch.Tensor] = None
        # fp8 data gradient (opt-in, decided independently of the forward): e5m2 dY x e4m3 weights quantised on every
        # backward from dY and the fp32 master, Cok8 slots per tap (Cout_g rounded up to 128)
        self.fp8_dgrad, self.fp8_dgrad_reason = False, "fp8 dgrad off"
        if mode in ("fprop+dgrad", "fprop+dgrad+wgrad"):
            self.fp8_dgrad, self.fp8_dgrad_reason = self._fp8_dgrad_eligible(layer)
        self.cok8 = _round128(self.Cout // self.groups) if self.fp8_dgrad else 0
        self.s_dy: Optional[torch.Tensor] = None      # written by the quantisers every backward
        self.s_wt: Optional[torch.Tensor] = None
        # fp8 weight gradient (opt-in, decided independently of the other two): e5m2 dY x e4m3 X in batch-innermost copies
        # quantised on every backward, Cgkw8 column slots per tap (Cg rounded up to 64: one B box per 64 columns)
        self.fp8_wgrad, self.fp8_wgrad_reason = False, "fp8 wgrad off"
        if mode == "fprop+dgrad+wgrad":
            self.fp8_wgrad, self.fp8_wgrad_reason = self._fp8_wgrad_eligible(layer)
        self.cgkw8 = _pad64(self.cg) if self.fp8_wgrad else 0
        self.s_xw: Optional[torch.Tensor] = None      # X's scale for the weight gradient (not the forward's s_x)
        # delayed scaling (opt-in): the activation / dY quantisers of training passes scale from amax histories in device
        # memory, one per scaled tensor ("x": the forward input, "dy", "xw": the weight gradient's X when the forward is
        # bf16), each [int32 ring, seeded?]; never saved, so a resumed run seeds them again
        self.fp8_delayed = resolve_fp8_scaling(fp8_scaling, mode) == "delayed" and \
            (self.fp8 or self.fp8_dgrad or self.fp8_wgrad)
        self.amax_rings: dict = {}
        self.wbp: Optional[torch.Tensor] = None      # channel-padded copy of wb (derived, refreshed when wb changes)
        self.dirty_wbp = True
        self.wb: Optional[torch.Tensor] = None
        self.wt: Optional[torch.Tensor] = None
        self.dirty_wb = True               # bf16 fprop/wgrad operand is stale w.r.t. the fp32 master
        self.dirty_wt = True               # packed dgrad operand is stale
        self.arena_shadow = False          # wb lives in the symmetric arena and is refreshed by the update kernels
        self.need_dgrad = True
        self.consumer_masks = False        # a downstream kernel applies this layer's ReLU mask
        self.mask_input = False            # this layer's dgrad applies the producer's ReLU mask
        w = layer.weight
        if not self.row_mode and not w.data.is_contiguous(memory_format=CL):
            w.data = w.data.contiguous(memory_format=CL)

    def _try_s2d(self, layer):
        """Stride-4 first layers (AlexNet / CaffeNet conv1): space-to-depth by 4 turns the 11x11/s4 convolution over
        4 (padded) channels into a 3x3/s1 convolution over 4*4*4 = 64 channels — a plain TAP-mode implicit GEMM whose
        operand the TMA engine fetches in im2col mode, instead of the cp.async ROW gather.  The data layer's transform
        kernel writes the s2d layout directly."""
        if os.environ.get("POSEIDON_S2D", "1") == "0" or tuple(layer.stride) != (4, 4) or layer.pad[0] != layer.pad[1]:
            return
        in_hw = getattr(layer, "in_hw", None)
        if in_hw is None:
            return
        h, w = in_hw
        p = layer.pad[0]
        hq, wq = -(-(h + 2 * p) // 4), -(-(w + 2 * p) // 4)
        rq, sq = -(-self.R // 4), -(-self.S // 4)
        oh, ow = (h + 2 * p - self.R) // 4 + 1, (w + 2 * p - self.S) // 4 + 1
        if hq - rq + 1 != oh or wq - sq + 1 != ow:
            return
        self.s2d = True
        self.s2d_hw = (hq, wq)
        self.Rq, self.Sq = rq, sq
        self.Kw = rq * sq * 64

    def _fp8_eligible(self, layer):
        """(fp8?, reason): TAP mode, channel counts in multiples of 8, an im2col-TMA geometry, and Cg rounded up to 128
        wasting at most a third of the work (the _pad64 threshold)."""
        if self.row_mode or self.s2d or self.pad8:
            return False, "first-layer layout (ROW / s2d / 8-channel pad)"
        if self.Coutp != self.Cout or self.cg % 8:
            return False, "channel counts are not multiples of 8"
        if self.groups > 1 and self.cg % 16:
            return False, "group slices of the e4m3 input are not 16-byte aligned"
        (sh, sw), (ph, pw) = layer.stride, layer.pad
        if sh > 8 or sw > 8:
            return False, "stride > 8"
        corners = [-ph, -pw]
        in_hw = getattr(layer, "in_hw", None)
        if in_hw is not None:
            h, w = in_hw
            oh, ow = (h + 2 * ph - self.R) // sh + 1, (w + 2 * pw - self.S) // sw + 1
            corners += [(oh - 1) * sh + 1 - ph - h, (ow - 1) * sw + 1 - pw - w]
        if any(not -128 <= v <= 127 for v in corners):
            return False, "im2col corner offsets do not fit a signed byte"
        p = _round128(self.cg)
        if (p - self.cg) * 100 > 34 * self.cg:
            return False, f"Cg {self.cg} -> {p} slots wastes more than a third"
        return True, f"Cg {self.cg} -> {p} slots"

    def _fp8_dgrad_eligible(self, layer):
        """(fp8 data gradient?, reason): a stride-1 TAP-mode layer with channel counts in multiples of 8 (Cout_g in
        multiples of 16 when grouped: the e5m2 group slices of dY start on 16-byte boundaries), mirrored im2col corner
        offsets in a signed byte, and Cout_g rounded up to 128 wasting at most a third of the work.  The producer mask a
        fused ReLU hands to this layer is the producer's dense output, laid out like dX (as conv_dgrad requires)."""
        if self.row_mode or self.s2d or self.pad8:
            return False, "first-layer layout (ROW / s2d / 8-channel pad)"
        if tuple(layer.stride) != (1, 1):
            return False, "strided (bf16 phase decomposition)"
        cout_g = self.Cout // self.groups
        if self.Coutp != self.Cout or self.cg % 8 or cout_g % 8:
            return False, "channel counts are not multiples of 8"
        if self.groups > 1 and cout_g % 16:
            return False, "group slices of the e5m2 dY are not 16-byte aligned"
        if self.R > 15 or self.S > 15:
            return False, "kernel larger than 15"
        (ph, pw) = layer.pad
        # mirrored walk: the box starts at pad - (R - 1) and ends at -pad relative to dY's extent
        if any(not -128 <= v <= 127 for v in (ph - (self.R - 1), pw - (self.S - 1), -ph, -pw)):
            return False, "im2col corner offsets do not fit a signed byte"
        p = _round128(cout_g)
        if (p - cout_g) * 100 > 34 * cout_g:
            return False, f"Cout_g {cout_g} -> {p} slots wastes more than a third"
        return True, f"Cout_g {cout_g} -> {p} slots"

    def _fp8_wgrad_eligible(self, layer):
        """(fp8 weight gradient?, reason): a stride-1 TAP-mode layer with channel counts in multiples of 8 whose Cg is a
        multiple of 64 or rounds up to one wasting at most a third (_pad64): every 64-column chunk of the reduction's
        X side is one tap.  Batch only sets the k-block layout, so it does not enter the rule."""
        if self.row_mode or self.s2d or self.pad8:
            return False, "first-layer layout (ROW / s2d / 8-channel pad)"
        if tuple(layer.stride) != (1, 1):
            return False, "strided"
        cout_g = self.Cout // self.groups
        if self.Coutp != self.Cout or self.cg % 8 or cout_g % 8:
            return False, "channel counts are not multiples of 8"
        if self.R > 15 or self.S > 15:
            return False, "kernel larger than 15"
        if any(p >= k for p, k in zip(layer.pad, (self.R, self.S))):
            return False, "padding not below the kernel extent"
        p = _pad64(self.cg)
        if p % 64:
            return False, f"Cg {self.cg} does not round up to a multiple of 64 within a third"
        return True, f"Cg {self.cg} -> {p} columns per tap"

    # physical [Cout, Kw] fp32 view of the master weight (TAP mode only)
    def w2d(self) -> torch.Tensor:
        w = self.layer.weight.data
        return w.permute(0, 2, 3, 1).reshape(self.Cout, self.Kw)

    def mark_updated(self, keep_wb: bool = False):
        """The fp32 master changed (optimizer step / weight load)."""
        self.dirty_wt = True
        self.dirty_wbp = True
        if not keep_wb and not self.arena_shadow:
            self.dirty_wb = True

    def shadow(self) -> torch.Tensor:
        if self.wb is not None and not self.dirty_wb:
            return self.wb
        w = self.layer.weight
        with torch.no_grad():
            if self.pad8:
                t = torch.nn.functional.pad(w.data.permute(0, 2, 3, 1), (0, self.Cp - self.cin_logical))   # Cout,R,S,Cp
                src = t.reshape(self.Cout, self.Kw)
                if self.Coutp != self.Cout:
                    src = torch.nn.functional.pad(src, (0, 0, 0, self.Coutp - self.Cout))                  # zero rows
            elif self.s2d:
                # W'[co][R'][S'][dy][dx][c] = W[co][c][4R'+dy][4S'+dx]  (zero outside the 11x11 support / c >= C)
                t = torch.nn.functional.pad(w.data, (0, 4 * self.Sq - self.S, 0, 4 * self.Rq - self.R,
                                                     0, self.Cp - self.cin_logical))       # Cout,4,4R',4S'
                t = t.view(self.Cout, self.Cp, self.Rq, 4, self.Sq, 4).permute(0, 2, 4, 3, 5, 1)
                src = t.reshape(self.Cout, self.Kw)
            elif self.row_mode:
                t = w.data.permute(0, 2, 3, 1)                                    # Cout,R,S,C
                t = torch.nn.functional.pad(t, (0, self.Cp - self.cin_logical))  # -> Cp
                t = t.reshape(self.Cout, self.R, self.L)
                src = torch.nn.functional.pad(t, (0, self.Lp - self.L)).reshape(self.Cout, self.Kw)
            else:
                src = self.w2d()
            if self.wb is None:
                self.wb = src.to(torch.bfloat16).contiguous()
            else:
                self.wb.copy_(src)
        self.dirty_wb = False
        return self.wb

    def operand(self) -> torch.Tensor:
        """The bf16 fprop operand the kernels consume: the shadow itself, or its channel-padded copy."""
        wb = self.shadow()
        if self.cgk == self.cg:
            return wb
        if self.wbp is None or self.dirty_wbp:
            self.wbp = K().conv_pack_padded(wb.reshape(-1), self.Cout, self.R * self.S, self.cg, self.cgk, self.wbp)
            self.dirty_wbp = False
        return self.wbp

    def dgrad_pack(self) -> torch.Tensor:
        if self.wt is not None and not self.dirty_wt:
            return self.wt
        if self.pad8:
            with torch.no_grad():
                src = torch.nn.functional.pad(self.layer.weight.data.permute(0, 2, 3, 1), (0, self.Cp - self.cin_logical))
            self.wt = K().conv_pack_dgrad(src.reshape(-1).contiguous(), self.Cout, self.R * self.S, self.Cp, 1, self.wt,
                                          self.Coutp)
            self.dirty_wt = False
            return self.wt
        self.wt = K().conv_pack_dgrad(self.w2d().reshape(-1), self.Cout, self.R * self.S, self.cg, self.groups, self.wt,
                                      self.cok)
        self.dirty_wt = False
        return self.wt

    def grad_from_dw(self, dw: torch.Tensor) -> torch.Tensor:
        """[Cout, Kw] fp32 -> gradient tensor with the master weight's logical shape."""
        if self.pad8:
            return dw[: self.Cout].view(self.Cout, self.R, self.S, self.Cp)[..., : self.cin_logical] \
                .permute(0, 3, 1, 2).contiguous()
        if self.s2d:
            g = dw.view(self.Cout, self.Rq, self.Sq, 4, 4, self.Cp).permute(0, 5, 1, 3, 2, 4)   # co,c,R',dy,S',dx
            g = g.reshape(self.Cout, self.Cp, 4 * self.Rq, 4 * self.Sq)
            return g[:, : self.cin_logical, : self.R, : self.S].contiguous()
        if self.row_mode:
            g = dw.view(self.Cout, self.R, self.Lp)[:, :, : self.L].reshape(self.Cout, self.R, self.S, self.Cp)
            return g[..., : self.cin_logical].permute(0, 3, 1, 2).contiguous()
        return dw.view(self.Cout, self.R, self.S, self.cg).permute(0, 3, 1, 2)   # channels-last strided view


def conv_state(layer, cin_logical, fp8: Optional[str] = None, fp8_scaling: Optional[str] = None) -> ConvState:
    st = getattr(layer, "_sm100", None)
    if st is None:
        st = ConvState(layer, cin_logical, fp8, fp8_scaling)
        layer._sm100 = st
    return st


def prepare_first_layer_input(x: torch.Tensor, st: ConvState, pad, in_hw) -> torch.Tensor:
    """Bring the first-layer input into the padded NHWC4 layout ROW-mode conv consumes: channels padded to
    Cp, spatially pre-padded by the conv's own padding, physical width rounded up to even (16-byte rows).
    The data layers emit this layout straight from the transform kernel; anything else is converted here."""
    h, w = in_hw
    if st.pad8:
        if (x.dtype == torch.bfloat16 and x.dim() == 4 and tuple(x.shape[1:]) == (st.Cp, h, w)
                and x.is_contiguous(memory_format=CL)):
            return x
        if x.shape[1] == st.Cp:
            return as_kernel_input(x)
        t = torch.nn.functional.pad(x.float(), (0, 0, 0, 0, 0, st.Cp - x.shape[1]))
        return t.to(torch.bfloat16).contiguous(memory_format=CL)
    if st.s2d:
        hq, wq = st.s2d_hw
        if (x.dtype == torch.bfloat16 and x.dim() == 4 and tuple(x.shape[1:]) == (64, hq, wq)
                and x.is_contiguous(memory_format=CL)):
            return x
        n, c = x.shape[:2]
        if x.shape[2] != h or x.shape[3] != w:
            raise ValueError(f"first-layer conv: unexpected input shape {tuple(x.shape)} for logical {h}x{w}")
        t = torch.nn.functional.pad(x.float(), (pad[1], 4 * wq - w - pad[1], pad[0], 4 * hq - h - pad[0], 0, st.Cp - c))
        t = t.view(n, st.Cp, hq, 4, wq, 4).permute(0, 2, 4, 3, 5, 1).reshape(n, hq, wq, 64)      # n,Y,X,(dy,dx,c)
        return t.to(torch.bfloat16).permute(0, 3, 1, 2)                                      # logical NCHW, CL memory
    wp = w + 2 * pad[1]
    extra = wp % 2
    if (x.dtype == torch.bfloat16 and x.dim() == 4 and x.shape[1] == st.Cp and x.shape[2] == h + 2 * pad[0]
            and x.shape[3] == wp + extra and x.is_contiguous(memory_format=CL)):
        return x
    n, c = x.shape[:2]
    if x.shape[2] != h or x.shape[3] != w:
        raise ValueError(f"first-layer conv: unexpected input shape {tuple(x.shape)} for logical {h}x{w}")
    t = torch.nn.functional.pad(x.float(), (pad[1], pad[1] + extra, pad[0], pad[0], 0, st.Cp - c))
    return t.to(torch.bfloat16).contiguous(memory_format=CL)


class _ConvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, layer, relu_slope, delayed):
        st: ConvState = layer._sm100
        k = K()
        stride, pad = layer.stride, layer.pad
        if st.pad8:
            h, w = layer.in_hw
            xin = prepare_first_layer_input(x, st, pad, (h, w))
            conv_pad = pad
        elif st.row_mode:
            h, w = layer.in_hw
            xin = prepare_first_layer_input(x, st, pad, (h, w))
            conv_pad = (0, 0)
        else:
            xin = as_kernel_input(x)
            h, w = xin.shape[2], xin.shape[3]
            conv_pad = pad
        oh = (h + 2 * pad[0] - st.R) // stride[0] + 1
        ow = (w + 2 * pad[1] - st.S) // stride[1] + 1
        relu = relu_slope is not None
        x8t = None                  # delayed scaling: the weight gradient's X copy, written by the forward's quantiser
        if st.s2d:
            y = k.conv_fprop(xin, st.shadow(), bias, [st.Rq, st.Sq], [1, 1], [0, 0], 1, 0, oh, ow, relu,
                             float(relu_slope or 0.0), None)
        else:
            if st.Coutp != st.Cout and bias is not None:
                bias = torch.nn.functional.pad(bias.detach(), (0, st.Coutp - st.Cout))
            # zero-copy concat: this layer's output is a channel slice of its consumer CONCAT layer's slab
            slab = getattr(layer, "_concat_slab", None)
            out = None
            if slab is not None and st.Coutp == st.Cout:
                out = slab[0].slab_view(slab[1], xin.shape[0], oh, ow, xin.device)
            if st.fp8:
                y, x8t = _fp8_fprop(k, st, weight, xin, bias, list(stride), list(conv_pad), oh, ow, relu,
                                    float(relu_slope or 0.0), out, delayed)
            else:
                y = k.conv_fprop(xin, st.operand(), bias, [st.R, st.S], list(stride), list(conv_pad), st.groups,
                                 1 if (st.row_mode and not st.pad8) else 0, oh, ow, relu, float(relu_slope or 0.0), out)
            if st.Coutp != st.Cout:
                y = y[:, : st.Cout]            # channel slice of the padded tensor (pixel pitch Coutp)
        ctx.layer, ctx.relu_slope, ctx.conv_pad, ctx.delayed = layer, relu_slope, conv_pad, delayed
        ctx.in_shape, ctx.in_dtype = tuple(x.shape), x.dtype
        ctx.save_for_backward(xin, y if relu else None, x8t)
        return y

    @staticmethod
    def backward(ctx, dy):
        layer = ctx.layer
        st: ConvState = layer._sm100
        k = K()
        xin, y, x8t = ctx.saved_tensors
        if st.Coutp != st.Cout:
            # zero-padded output channels: mask (if any) on the logical slice, then widen dY to the padded layout
            if y is not None and not st.consumer_masks:
                dy = torch.where(y > 0, dy, dy * float(ctx.relu_slope))
            dyp = torch.empty((dy.shape[0], st.Coutp, dy.shape[2], dy.shape[3]), device=dy.device,
                              dtype=torch.bfloat16, memory_format=CL).zero_()
            dyp[:, : st.Cout].copy_(dy)
            dy = dyp
        else:
            dy = as_kernel_input(dy)
            if st.fp8_wgrad and ctx.needs_input_grad[1]:
                # e5m2 dY for the weight gradient (batch-innermost copy, plus the NHWC copy of an fp8 data gradient):
                # one amax pass (ReLU backward fused in as below) and one cast pass, on this stream before the fork
                dy8t, dy8, dy = _fp8_quant_grad_t(k, st, dy, y if not st.consumer_masks else None, ctx.relu_slope,
                                                  st.fp8_dgrad and ctx.needs_input_grad[0], ctx.delayed)
            elif st.fp8_dgrad and ctx.needs_input_grad[0]:
                # e5m2 dY: amax pass (with this layer's ReLU backward fused in when it masks its own gradient; the
                # weight / bias gradients below then read the masked bf16 dY it writes) and cast
                dy8, dy = _fp8_quant_grad(k, st, dy, y if not st.consumer_masks else None, ctx.relu_slope, ctx.delayed)
            elif y is not None and not st.consumer_masks:
                if y.is_contiguous(memory_format=CL) and dy.is_contiguous(memory_format=CL):
                    dy = k.relu_bwd(y, dy, float(ctx.relu_slope))
                else:                       # y and / or dy are channel slices of a concat slab: pitch-aware kernel
                    dy = k.relu_bwd_nhwc(y, dy, float(ctx.relu_slope))
        stride = layer.stride
        dw = db = dx = None
        # The weight / bias gradient and the data gradient of one layer are independent: with a data gradient to compute,
        # the former run on a side stream (forked here, joined before returning), so a layer costs max(dgrad, wgrad)
        # instead of their sum on its lane — small convolutions (GoogLeNet at batch 32) do not fill the chip alone.
        # When the gradient lands in a sink whose owner (the fused backend) waits for it itself, the join is deferred: the
        # weight gradients of all layers queue up on the side stream and fill whatever the main chain (data gradients,
        # pooling / LRN backward) leaves idle; the update / communication launches wait on the recorded events.
        side = done = None
        sink = getattr(layer, "_grad_sink", None) if ctx.needs_input_grad[1] else None
        if dy.is_cuda and ctx.needs_input_grad[0] and ctx.needs_input_grad[1] and _wgrad_lane():
            cur = torch.cuda.current_stream()
            side = _wgrad_stream(cur)
        defer = side is not None and sink is not None and getattr(sink, "defers_wgrad_join", False) and _wgrad_defer()
        # one GPU: nothing touches the bias gradient before the end-of-iteration update (autograd adopts the tensor
        # without a copy, the hook only queues it), so its column-sum kernel can ride the side stream as well
        # several GPUs: the bias gradient lands in its arena segment directly (sink.bias_buffer) and the bucket launch
        # waits for the side stream like it does for the weight gradient
        dbf = None
        if layer.bias_term and ctx.needs_input_grad[2] and sink is not None and st.Coutp == st.Cout and \
                hasattr(sink, "bias_buffer"):
            dbf = sink.bias_buffer(layer, st)
        defer_bias = defer and (dbf is not None or (getattr(sink, "world", 0) == 1 and getattr(sink, "multi_update", False)))
        dw2 = None
        if ctx.needs_input_grad[1]:             # (outputs are allocated on the layer's own stream)
            dw2 = sink.weight_buffer(layer, st) if sink is not None else \
                torch.zeros(st.Coutp, st.Kw, device=dy.device, dtype=torch.float32)
        if layer.bias_term and ctx.needs_input_grad[2] and dbf is None:
            dbf = torch.empty(st.Coutp, device=dy.device, dtype=torch.float32)

        def bias_grad():
            pitch = dy.stride(3) if dy.shape[3] > 1 else (dy.stride(2) if dy.shape[2] > 1 else dy.stride(0))
            k.colsum(dy, dy.shape[0] * dy.shape[2] * dy.shape[3], st.Coutp, pitch, dbf, 1.0, False)
            return dbf[: st.Cout]

        if side is not None:
            fork = torch.cuda.Event()
            fork.record(cur)
            side.wait_event(fork)
            dy.record_stream(side)
            xin.record_stream(side)
            if st.fp8_wgrad and dw2 is not None:
                dy8t.record_stream(side)
                if x8t is not None:
                    x8t.record_stream(side)
            torch.cuda.set_stream(side)
        try:
            if dw2 is not None:
                if st.s2d:
                    k.conv_wgrad(xin, dy, dw2, [st.Rq, st.Sq], [1, 1], [0, 0], 1, 0, 1.0, 0)
                elif st.fp8_wgrad and x8t is not None:
                    # delayed scaling: the forward's quantiser wrote X's copy with the forward's scale
                    k.conv_wgrad_fp8(dy8t, x8t, st.s_dy, st.s_x, dw2, [st.R, st.S], list(ctx.conv_pad), st.groups, 1.0,
                                     st.cgkw8)
                elif st.fp8_wgrad:
                    # e4m3 X (its own scale) and the fp8 GEMM, on the weight-gradient side stream
                    if ctx.delayed:
                        x8t, _ = _delayed_quant(st, "xw", k.fp8_quant_act_t_delayed, xin, st.s_xw, False)
                    else:
                        x8t = k.fp8_quant_act_t(xin, st.s_xw)
                    k.conv_wgrad_fp8(dy8t, x8t, st.s_dy, st.s_xw, dw2, [st.R, st.S], list(ctx.conv_pad), st.groups, 1.0,
                                     st.cgkw8)
                else:
                    k.conv_wgrad(xin, dy, dw2, [st.R, st.S], list(stride), list(ctx.conv_pad), st.groups,
                                 1 if (st.row_mode and not st.pad8) else 0, 1.0, st.cgk if not st.row_mode else 0)
                dw = st.grad_from_dw(dw2)
            if dbf is not None and (not defer or defer_bias):
                db = bias_grad()
        finally:
            if side is not None:
                done = torch.cuda.Event()
                done.record(side)
                torch.cuda.set_stream(cur)
        if dbf is not None and defer and not defer_bias:
            db = bias_grad()                    # (multi-GPU: staged into the arena on this stream by the bucket launch)
        if ctx.needs_input_grad[0]:
            # dX comes back in the layout of the tensor the forward received: the physical s2d / ROW / 8-channel input a
            # data layer handed over as it is, a logical input (deploy `input:`, LeNet conv2) through first_layer_diff
            if st.s2d:
                dx = _s2d_dgrad(k, st, layer, dy)
            elif st.row_mode and not st.pad8:
                dx = _strided_dgrad(k, st, layer, dy, xin, row=True)[:, : st.Cp]
            elif tuple(stride) != (1, 1):
                dx = _strided_dgrad(k, st, layer, dy, xin)
            else:
                mask = xin if st.mask_input else None
                if st.fp8_dgrad:
                    # e4m3 weights from the fp32 master, then the fp8 im2col GEMM (mirrored taps), on this stream
                    wt8 = k.fp8_quant_weight_dgrad(layer.weight.detach(), st.groups, st.cok8, st.s_wt)
                    dx = k.conv_dgrad_fp8(dy8, wt8, st.s_dy, st.s_wt, [st.R, st.S], list(layer.pad), st.groups,
                                          xin.shape[2], xin.shape[3], mask, 0.0)
                elif _dgrad_reads_fprop_weights(st, layer, dy):
                    # no packed [Cin][R][S][Cout] copy and no pack kernel per step: the kernel reads the fprop shadow
                    # through a 3-D tensor map as an MN-major B operand
                    dx = k.conv_dgrad_w(dy, st.shadow(), [st.R, st.S], list(layer.pad), st.groups, xin.shape[2],
                                        xin.shape[3], mask, 0.0)
                else:
                    dx = k.conv_dgrad(dy, st.dgrad_pack(), [st.R, st.S], list(layer.pad), st.groups, xin.shape[2],
                                      xin.shape[3], mask, 0.0)
            if tuple(dx.shape) != ctx.in_shape:
                dx = first_layer_diff(dx, layer, ctx.in_shape, ctx.in_dtype == torch.float32)
        if done is not None:
            if defer:
                _pending_wgrad.setdefault(cur.device.index, []).append(done)
            else:
                cur.wait_event(done)            # join: dw / db are complete for whoever consumes them on this stream
        return dx, dw, db, None, None, None


def _fp8_fprop(k, st: ConvState, weight, xin, bias, stride, pad, oh, ow, relu, slope, out, delayed):
    """e4m3 forward: quantise the fp32 master and the input, then the fp8 im2col GEMM.  All three launches run on every
    forward: under a CUDA graph Python does not run at replay, and the optimizer updates the master inside the graph.
    Returns (y, the weight gradient's X copy written by the same pass under delayed scaling, else None)."""
    w = weight.detach()
    if st.s_x is None:
        st.s_x = torch.ones(1, device=w.device, dtype=torch.float32)
        st.s_w = torch.ones(st.Cout, device=w.device, dtype=torch.float32)
    w8 = k.fp8_quant_weight(w, st.cgk8, st.s_w)
    x8t = None
    if delayed and st.fp8_wgrad:
        x8t, x8 = _delayed_quant(st, "x", k.fp8_quant_act_t_delayed, xin, st.s_x, True)
    elif delayed:
        x8 = _delayed_quant(st, "x", k.fp8_quant_act_delayed, xin, st.s_x)
    else:
        x8 = k.fp8_quant_act(xin, st.s_x)
    y = k.conv_fprop_fp8(x8, w8, st.s_x, st.s_w, None if bias is None else bias.detach(), [st.R, st.S], stride, pad,
                         st.groups, oh, ow, relu, slope, out)
    return y, x8t


def _fp8_quant_grad(k, st: ConvState, dy, y, slope, delayed=False):
    """e5m2 dY for the fp8 data gradient: returns (dy8, the bf16 dY the weight / bias gradients read).  With y (the layer
    masks its own gradient) the amax pass applies the ReLU backward and writes the masked dY, bit-identical to relu_bwd.
    Runs on every backward (graph replays included); the scale tensors are allocated once per layer."""
    if st.s_dy is None:
        st.s_dy = torch.ones(1, device=dy.device, dtype=torch.float32)
        st.s_wt = torch.ones(st.Cp, device=dy.device, dtype=torch.float32)
    if delayed:
        return _delayed_quant(st, "dy", k.fp8_quant_grad_delayed, dy, st.s_dy, y, float(slope or 0.0))
    return k.fp8_quant_grad(dy, st.s_dy, y, float(slope or 0.0))


def _fp8_quant_grad_t(k, st: ConvState, dy, y, slope, nhwc: bool, delayed=False):
    """e5m2 dY for the fp8 weight gradient: returns (dy8t, dy8 for an fp8 data gradient (nhwc) else None, the bf16 dY the
    bias gradient reads), with the scale and mask of _fp8_quant_grad."""
    if st.s_dy is None:
        st.s_dy = torch.ones(1, device=dy.device, dtype=torch.float32)
        st.s_wt = torch.ones(st.Cp, device=dy.device, dtype=torch.float32)
    if st.s_xw is None:
        st.s_xw = torch.ones(1, device=dy.device, dtype=torch.float32)
    if delayed:
        dy8t, dy8, src = _delayed_quant(st, "dy", k.fp8_quant_grad_t_delayed, dy, st.s_dy, y, float(slope or 0.0), nhwc)
    else:
        dy8t, dy8, src = k.fp8_quant_grad_t(dy, st.s_dy, y, float(slope or 0.0), nhwc)
    return dy8t, (dy8 if nhwc else None), src


def _capturing() -> bool:
    """Is the current CUDA stream being captured into a graph?"""
    return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()


def _delayed_quant(st: ConvState, key: str, op, x, s_out, *args):
    """One delayed-scaling quantiser call op(x, s_out, ring, seed, *args) on the amax history ``key`` of this layer.  The
    first call seeds the ring (amax pass, then every slot holds that amax: the just-in-time result).  Seeding happens on
    eager steps: a CUDA graph would replay the seed on every step, so a capture that reaches an unseeded ring fails."""
    entry = st.amax_rings.get(key)
    if entry is None:
        entry = st.amax_rings[key] = [torch.zeros(_RING_WORDS, dtype=torch.int32, device=x.device), False]
    if not entry[1] and _capturing():
        raise RuntimeError(f"sm100 conv '{st.layer.layer_name}': fp8_scaling='delayed' reached the unseeded amax history "
                           f"'{key}' inside a CUDA-graph capture; run an eager training step first")
    out = op(x, s_out, entry[0], not entry[1], *args)
    entry[1] = True
    return out


def reset_amax_histories(net) -> None:
    """Forget the delayed-scaling amax histories of ``net``'s convolutions (a restored run seeds them again)."""
    for layer in net.layers:
        st = getattr(layer, "_sm100", None)
        if isinstance(st, ConvState):
            st.amax_rings.clear()


_DGRAD_PACK = os.environ.get("POSEIDON_DGRAD_PACK", "0") == "1"      # A/B switch: always use the packed dgrad operand


def _wgrad_lane() -> bool:
    """Weight gradients on a side stream next to the data gradient (POSEIDON_WGRAD_LANE=0: same stream)."""
    return os.environ.get("POSEIDON_WGRAD_LANE", "1") == "1"



def _wgrad_defer() -> bool:
    """Join the side streams at the update / communication launches instead of at the end of each layer's backward
    (POSEIDON_WGRAD_DEFER=0: join per layer)."""
    return os.environ.get("POSEIDON_WGRAD_DEFER", "1") == "1"


_wgrad_streams: dict = {}
_pending_wgrad: dict = {}          # device index -> events of weight-gradient kernels not yet joined


def add_pending_wgrad(event, device_index: int) -> None:
    """Register work queued behind a forked weight gradient (its optimizer step) for the same deferred join."""
    _pending_wgrad.setdefault(device_index, []).append(event)


def wait_pending_wgrad(stream=None, clear: bool = False) -> None:
    """Make ``stream`` (default: the current one) wait for every weight-gradient kernel that was forked to a side stream
    and not joined yet.  Called by whoever consumes the gradient sinks: the update launches at the end of the iteration
    (``clear=True``) and the per-bucket communication launches."""
    if not _pending_wgrad:
        return
    s = stream if stream is not None else torch.cuda.current_stream()
    lst = _pending_wgrad.get(s.device.index)
    if lst:
        for ev in lst:
            s.wait_event(ev)
        if clear:
            lst.clear()


def _wgrad_stream(cur: "torch.cuda.Stream") -> "torch.cuda.Stream":
    """The side stream paired with ``cur`` (one per stream a layer can run on: the caller's stream and every lane)."""
    key = (cur.device.index, cur.cuda_stream)
    s = _wgrad_streams.get(key)
    if s is None:
        s = _wgrad_streams[key] = torch.cuda.Stream(device=cur.device)
    return s


def _dgrad_reads_fprop_weights(st: "ConvState", layer, dy: torch.Tensor) -> bool:
    """Geometry the pack-free dgrad kernel covers (csrc/gemm/conv_ops.cu conv_dgrad_w): TAP-mode weights, channel counts
    per group that are multiples of 8 (16-byte TMA strides), im2col-descriptor offsets within a signed byte.  An s2d layer
    is asked about its 3x3 / pad-0 problem over 64 channels."""
    if _DGRAD_PACK or (st.row_mode and not st.s2d) or st.pad8 or st.Coutp != st.Cout:
        return False
    if st.s2d:
        cg, kernel, pad = 64, (st.Rq, st.Sq), (0, 0)
    else:
        cg, kernel, pad = st.cg, (st.R, st.S), layer.pad
    if cg % 8 != 0 or (st.Cout // st.groups) % 8 != 0:
        return False
    if max(kernel[0], kernel[1], pad[0], pad[1]) > 64:
        return False
    pitch = dy.stride(3) if dy.shape[3] > 1 else (dy.stride(2) if dy.shape[2] > 1 else dy.stride(0))
    return dy.stride(1) == 1 and pitch % 8 == 0 and dy.data_ptr() % 16 == 0


def _s2d_dgrad(k, st: "ConvState", layer, dy: torch.Tensor) -> torch.Tensor:
    """Data gradient of a space-to-depth first layer: the stride-1 data gradient of its 3x3 / pad-0 convolution over the
    64 s2d channels, [N, 64, hq, wq] like the s2d input.  The shadow is zero at taps outside the 11x11 support and at the
    padded 4th channel, so the padding lanes receive exact zeros."""
    hq, wq = st.s2d_hw
    dy = as_kernel_input(dy)
    if _dgrad_reads_fprop_weights(st, layer, dy):
        return k.conv_dgrad_w(dy, st.shadow(), [st.Rq, st.Sq], [0, 0], 1, hq, wq, None, 0.0)
    if st.wt is None or st.dirty_wt:
        st.wt = k.conv_pack_dgrad(st.shadow().float().reshape(-1), st.Cout, st.Rq * st.Sq, 64, 1, st.wt, 0)
        st.dirty_wt = False
    return k.conv_dgrad(dy, st.wt, [st.Rq, st.Sq], [0, 0], 1, hq, wq, None, 0.0)


def first_layer_diff(dx: torch.Tensor, layer, shape, out_float: bool = True) -> torch.Tensor:
    """A convolution's data gradient in its physical input layout (s2d, spatially pre-padded ROW, padded channels) ->
    the logical blob's [N, C, H, W], contiguous, fp32 (``out_float``) or bf16.  Exact: a gather."""
    st: ConvState = layer._sm100
    n, c, h, w = shape
    ph, pw = layer.pad if (st.s2d or (st.row_mode and not st.pad8)) else (0, 0)
    return K().first_layer_diff(as_kernel_input(dx), c, h, w, ph, pw, st.s2d, out_float)


def _strided_dgrad(k, st: "ConvState", layer, dy: torch.Tensor, xin: torch.Tensor, row: bool = False) -> torch.Tensor:
    """Data gradient of a strided convolution as sh * sw stride-1 problems (reference: any stride through col2im,
    src/caffe/layers/conv_layer.cu:84-119 + util/im2col.cu:74-113).
    ``row``: a ROW-mode first layer, whose input is spatially pre-padded with 4 channels and which runs with pad 0: the
    problem is posed over the pre-padded extent with pad 0 and the weight zero-padded to 8 input channels (the kernels'
    channel granule); the result is an 8-channel dX over the padded extent.

    Input row ih = a + sh * i' (phase a) only receives taps r = r0 + sh * j with r0 = (a + ph) mod sh, and then
        oh = (ih + ph - r) / sh = i' + q - j,          q = (a + ph - r0) / sh   (an integer >= 0),
    i.e. the pixels of one phase are a stride-1 data gradient over dY with the sub-filter W[:, :, r0::sh, s0::sw] and
    padding (q_h, q_w): the same wgmma dgrad kernel, one launch per phase, each writing one interleaved sub-grid of dX.
    No atomics, no col2im scatter."""
    sh, sw = layer.stride
    ph, pw = (0, 0) if row else layer.pad
    n, _, H, W = xin.shape
    cin = 8 if row else st.Cp
    dx = torch.empty((n, cin, H, W), device=dy.device, dtype=torch.bfloat16, memory_format=CL)
    w4 = layer.weight.data.permute(0, 2, 3, 1)                       # [Cout, R, S, Cg] (physical order of the master)
    if st.pad8 or row:
        w4 = torch.nn.functional.pad(w4, (0, cin - st.cin_logical))
    cg = w4.shape[3]
    packs = getattr(st, "_phase_packs", None)
    if packs is None or st.dirty_wt:
        packs = st._phase_packs = {}
    for a in range(sh):
        r0 = (a + ph) % sh
        qh = (a + ph - r0) // sh
        ha = len(range(a, H, sh))
        for b in range(sw):
            s0 = (b + pw) % sw
            qw = (b + pw - s0) // sw
            wb_ = len(range(b, W, sw))
            if ha == 0 or wb_ == 0:
                continue
            sub = w4[:, r0::sh, s0::sw, :]
            rs, ss = sub.shape[1], sub.shape[2]
            if rs == 0 or ss == 0:
                dx[:, :, a::sh, b::sw] = 0                              # no tap reaches this phase (stride > kernel)
                continue
            key = (a, b)
            if key not in packs:
                packs[key] = k.conv_pack_dgrad(sub.contiguous().reshape(-1), st.Cout, rs * ss, cg, st.groups, None, 0)
            part = k.conv_dgrad(dy, packs[key], [rs, ss], [qh, qw], st.groups, ha, wb_, None, 0.0)
            dx[:, :, a::sh, b::sw] = part
    st.dirty_wt = False
    if st.mask_input:
        dx = k.relu_bwd(xin, dx, 0.0)                                   # the producer's ReLU, fused on the stride-1 path
    return dx


def conv2d(x, w, b, stride, pad, groups, relu_slope=None, layer=None):
    if layer is None or not _on(x):
        return TE.conv2d(x, w, b, stride, pad, groups, relu_slope, layer)
    st = conv_state(layer, w.shape[1] * groups)
    # delayed scaling on training passes only: test-phase forwards (test nets share this layer's state) and forwards
    # without autograd scale just in time and leave the amax histories alone
    delayed = st.fp8_delayed and torch.is_grad_enabled() and layer.ctx.train
    return _ConvFn.apply(x, w, b, layer, relu_slope, delayed)


# =====================================================================================================
# Inner product
# =====================================================================================================
class IPState:
    def __init__(self, layer, bottom_shape):
        self.layer = layer
        self.N, self.K = layer.weight.shape
        self.wb: Optional[torch.Tensor] = None
        self.dirty_wb = True
        self.arena_shadow = False
        self.perm = None
        if len(bottom_shape) == 4 and bottom_shape[2] * bottom_shape[3] > 1:
            # activations are NHWC: store the weight with K ordered (h, w, c) so flatten is free
            c, h, w = bottom_shape[1:]
            self.perm = (c, h, w)
            with torch.no_grad():
                wd = layer.weight.data
                layer.weight.data = wd.view(self.N, c, h, w).permute(0, 2, 3, 1).reshape(self.N, self.K).contiguous()
            layer._k_perm = self.perm
        # K not a multiple of 8 (LeNet ip2: 500): the reduction dimension is zero-padded around the kernels (TMA rows
        # must be 16-byte multiples).  The operand is then derived from the master like a first-layer conv operand.
        self.Kp = (self.K + 7) // 8 * 8
        self.row_mode = self.Kp != self.K      # "derived operand": no arena shadow, no gradient sink, no SFB

    def mark_updated(self, keep_wb: bool = False):
        if not keep_wb and not self.arena_shadow:
            self.dirty_wb = True

    def shadow(self) -> torch.Tensor:
        if self.wb is not None and not self.dirty_wb:
            return self.wb
        w = self.layer.weight
        with torch.no_grad():
            src = w.data if self.Kp == self.K else torch.nn.functional.pad(w.data, (0, self.Kp - self.K))
            if self.wb is None:
                self.wb = src.to(torch.bfloat16)
            else:
                self.wb.copy_(src)
        self.dirty_wb = False
        return self.wb


def _flatten_nhwc(x: torch.Tensor) -> torch.Tensor:
    """(N,C,H,W) channels-last -> (N, H*W*C) bf16 row-major without a copy when dense."""
    x = x if x.dtype == torch.bfloat16 else x.to(torch.bfloat16)
    if x.dim() == 2:
        return x.contiguous()
    if x.shape[2] * x.shape[3] == 1:
        return x.reshape(x.shape[0], -1).contiguous()
    if not x.is_contiguous(memory_format=CL):
        x = x.contiguous(memory_format=CL)
    return x.permute(0, 2, 3, 1).reshape(x.shape[0], -1)


class _IPFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, layer, relu):
        st: IPState = layer._sm100
        k = K()
        x2 = _flatten_nhwc(x)
        if st.Kp != st.K:
            x2 = torch.nn.functional.pad(x2, (0, st.Kp - st.K))
        n_pad = (st.N + 7) // 8 * 8
        if n_pad != st.N:
            out = torch.empty(x2.shape[0], n_pad, device=x.device, dtype=torch.bfloat16)[:, : st.N]
        else:
            out = None
        y = k.gemm_bf16(x2, False, st.shadow(), False, bias, bool(relu), 0.0, None, out, 0)
        ctx.layer, ctx.relu = layer, relu
        ctx.x_shape = tuple(x.shape)
        ctx.save_for_backward(x2, y if relu else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        layer = ctx.layer
        st: IPState = layer._sm100
        k = K()
        x2, y = ctx.saved_tensors
        dy = dy if dy.dtype == torch.bfloat16 else dy.to(torch.bfloat16)
        n_pad = (st.N + 7) // 8 * 8
        if y is not None and n_pad == st.N and dy.is_contiguous() and y.is_contiguous():
            dy = k.relu_bwd(y, dy, 0.0)                     # fused ReLU backward: one pass, dense [M, N] result
        elif dy.stride(1) != 1 or dy.stride(0) % 8 or (y is not None):
            buf = torch.empty(dy.shape[0], n_pad, device=dy.device, dtype=torch.bfloat16)
            if n_pad != st.N:
                buf[:, st.N:].zero_()
            d2 = buf[:, : st.N]
            if y is not None:
                d2.copy_(dy * (y > 0))
            else:
                d2.copy_(dy)
            dy = d2
        dw = db = dx = None
        if ctx.needs_input_grad[0]:
            # dX[M, K] = dY[M, N] · W[N, K]   (W row-major is the MN-major B operand).  Must be issued before the
            # fused SFB kernel below, which rewrites W / its bf16 shadow in place.
            dx2 = k.gemm_bf16(dy, False, st.shadow(), True, None, False, 0.0, None, None, 0)
            if st.Kp != st.K:
                dx2 = dx2[:, : st.K]
            xs = ctx.x_shape
            if len(xs) == 4 and xs[2] * xs[3] > 1:
                dx = dx2.reshape(xs[0], xs[2], xs[3], xs[1]).permute(0, 3, 1, 2)
            else:
                dx = dx2.reshape(xs)
        if layer.bias_term and ctx.needs_input_grad[2]:
            if st.N % 8 == 0 and dy.stride(1) == 1 and dy.stride(0) % 8 == 0:
                db = torch.empty(st.N, device=dy.device, dtype=torch.float32)
                k.colsum(dy, dy.shape[0], st.N, dy.stride(0), db, 1.0, False)
            else:
                db = dy.float().sum(0)
        sfb = getattr(layer, "sfb", None)
        if ctx.needs_input_grad[1]:
            if sfb is not None:
                dw = sfb.exchange_and_update(layer, dy, x2 if st.Kp == st.K else x2[:, : st.K].contiguous())
                # (fused path: returns None, W updated in place)
            else:
                sink = getattr(layer, "_grad_sink", None)
                dw = sink.weight_buffer(layer, st) if sink is not None else \
                    torch.empty(st.N, st.Kp, device=dy.device, dtype=torch.float32)
                # output-bound GEMM (fc6: 151 MB of fp32 for 19 GFLOP): on the weight-gradient side stream when its
                # consumer waits for it itself (see _ConvFn.backward), next to the convolutions' backward
                defer = dy.is_cuda and sink is not None and getattr(sink, "defers_wgrad_join", False) and \
                    _wgrad_lane() and _wgrad_defer() and os.environ.get("POSEIDON_IP_WGRAD_LANE", "1") == "1"
                layer._wgrad_side = None
                if defer:
                    cur = torch.cuda.current_stream()
                    side = _wgrad_stream(cur)
                    layer._wgrad_side = side        # the one-GPU backend steps this weight on the same stream, right away
                    fork = torch.cuda.Event()
                    fork.record(cur)
                    side.wait_event(fork)
                    dy.record_stream(side)
                    x2.record_stream(side)
                    torch.cuda.set_stream(side)
                try:
                    k.gemm_f32(dy, True, x2, True, dw, 1.0, False, 1, 0)
                finally:
                    if defer:
                        done = torch.cuda.Event()
                        done.record(side)
                        torch.cuda.set_stream(cur)
                        _pending_wgrad.setdefault(cur.device.index, []).append(done)
                if st.Kp != st.K:
                    dw = dw[:, : st.K]
        return dx, dw, db, None, None


def inner_product(x, w, b, relu=False, layer=None):
    if layer is None or not _on(x):
        return TE.inner_product(x, w, b, relu, layer)
    if getattr(layer, "_sm100", None) is None:
        layer._sm100 = IPState(layer, tuple(x.shape))
    return _IPFn.apply(x, w, b, layer, relu)


# =====================================================================================================
# LRN / pooling / ReLU / dropout / softmax-loss / concat / transform
# =====================================================================================================
class _LRNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, size, alpha, beta, mask_input):
        x = as_kernel_input(x).contiguous(memory_format=CL)
        ctx.save_for_backward(x)
        ctx.args = (size, alpha, beta, mask_input)
        return K().lrn_fwd(x, size, alpha, beta, False)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        size, alpha, beta, mask_input = ctx.args
        dy = as_kernel_input(dy)
        return K().lrn_bwd(x, dy, size, alpha, beta, bool(mask_input)), None, None, None, None


def lrn_across(x, size, alpha, beta, mask_input=False):
    if not _on(x) or x.shape[1] % 8:
        return R.lrn_across(x, size, alpha, beta)
    return _LRNFn.apply(x, size, alpha, beta, mask_input)


def _cl_dense(x: torch.Tensor) -> bool:
    return x.dim() == 4 and x.is_contiguous(memory_format=CL)


class _LRNWithinFn(torch.autograd.Function):
    """One kernel forward, two backward (the reference composes five layers: lrn_layer.cpp:20-69)."""

    @staticmethod
    def forward(ctx, x, size, alpha, beta):
        x = as_kernel_input(x)
        ctx.save_for_backward(x)
        ctx.args = (size, alpha, beta)
        return K().lrn_within_fwd(x, size, alpha, beta)

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        size, alpha, beta = ctx.args
        return K().lrn_within_bwd(x, as_kernel_input(dy), size, alpha, beta), None, None, None


def lrn_within(x, size, alpha, beta):
    if not _on(x) or x.dim() != 4 or x.shape[1] % 8:
        return R.lrn_within(x, size, alpha, beta)
    return _LRNWithinFn.apply(x, int(size), float(alpha), float(beta))


class _StoPoolFn(torch.autograd.Function):
    """Stochastic pooling, training phase: the sampled tap index is stored in MAX pooling's arg-max format, so the
    backward is pool_bwd's gather (reference: pooling_layer.cu:81-118 forward, :295-330 backward)."""

    @staticmethod
    def forward(ctx, x, kernel, stride, seed):
        x = as_kernel_input(x)
        oh = R.pool_out_size(x.shape[2], kernel[0], stride[0], 0)
        ow = R.pool_out_size(x.shape[3], kernel[1], stride[1], 0)
        y, idx = K().stochastic_pool_fwd(x, list(kernel), list(stride), oh, ow, True, seed, iteration_seed(x.device))
        ctx.save_for_backward(idx)
        ctx.args = (tuple(x.shape[2:]), kernel, stride)
        return y

    @staticmethod
    def backward(ctx, dy):
        (idx,) = ctx.saved_tensors
        in_hw, kernel, stride = ctx.args
        dx = K().pool_bwd(as_kernel_input(dy), idx, True, list(in_hw), list(kernel), list(stride), [0, 0])
        return dx, None, None, None


def stochastic_pool(x, kernel, stride, train: bool, generator=None):
    if not _on(x) or x.dim() != 4 or x.shape[1] % 8 or kernel[0] * kernel[1] > 255:
        return R.stochastic_pool(x, kernel, stride, train, generator)
    if not train:
        x = as_kernel_input(x)
        oh = R.pool_out_size(x.shape[2], kernel[0], stride[0], 0)
        ow = R.pool_out_size(x.shape[3], kernel[1], stride[1], 0)
        return K().stochastic_pool_fwd(x, list(kernel), list(stride), oh, ow, False, 0, None)[0]
    _dropout_counter[0] += 1
    seed = (torch.initial_seed() * 1000003 + _dropout_counter[0] * 7919 + 17) & 0x7FFFFFFFFFFFFFFF
    return _StoPoolFn.apply(x, tuple(kernel), tuple(stride), int(seed))


class _PoolFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, is_max, kernel, stride, pad, mask_input):
        x = as_kernel_input(x)
        oh = R.pool_out_size(x.shape[2], kernel[0], stride[0], pad[0])
        ow = R.pool_out_size(x.shape[3], kernel[1], stride[1], pad[1])
        y, idx = K().pool_fwd(x, is_max, list(kernel), list(stride), list(pad), oh, ow, bool(ctx.needs_input_grad[0]))
        ctx.save_for_backward(idx, y if mask_input else None)
        ctx.args = (is_max, tuple(x.shape[2:]), kernel, stride, pad)
        return y

    @staticmethod
    def backward(ctx, dy):
        idx, y = ctx.saved_tensors
        is_max, in_hw, kernel, stride, pad = ctx.args
        dy = as_kernel_input(dy)
        if y is not None:
            # producer's ReLU mask, evaluated on the (small) pooled tensor: max(ReLU(x)) > 0 <=> the arg-max passed the ReLU
            if dy.is_contiguous(memory_format=CL) and y.is_contiguous(memory_format=CL):
                dy = K().relu_bwd(y, dy, 0.0)
            else:
                dy = K().relu_bwd_nhwc(y, dy, 0.0)
        dx = K().pool_bwd(dy, idx, is_max, list(in_hw), list(kernel), list(stride), list(pad))
        return dx, None, None, None, None, None


def max_pool(x, kernel, stride, pad, return_mask=False, mask_input=False):
    if return_mask or not _on(x) or x.shape[1] % 8:
        return R.max_pool(x, kernel, stride, pad, return_mask)
    return _PoolFn.apply(x, True, tuple(kernel), tuple(stride), tuple(pad), mask_input)


def ave_pool(x, kernel, stride, pad, mask_input=False):
    if not _on(x) or x.shape[1] % 8:
        return R.ave_pool(x, kernel, stride, pad)
    return _PoolFn.apply(x, False, tuple(kernel), tuple(stride), tuple(pad), False)


class _ReLUFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, slope):
        y = K().relu_fwd(x, slope)
        ctx.save_for_backward(y)
        ctx.slope = slope
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        dy = dy if dy.dtype == torch.bfloat16 else dy.to(torch.bfloat16)
        if dy.stride() != y.stride():
            dy = dy.contiguous(memory_format=CL) if y.dim() == 4 and y.is_contiguous(memory_format=CL) else dy.contiguous()
        return K().relu_bwd(y, dy, ctx.slope), None


def relu(x, negative_slope=0.0):
    dense = x.is_contiguous() or (x.dim() == 4 and x.is_contiguous(memory_format=CL))
    if not _on(x) or x.dtype != torch.bfloat16 or x.numel() % 8 or not dense:
        return R.relu(x, negative_slope)
    return _ReLUFn.apply(x, float(negative_slope))


_dropout_counter = [0]
_iter_seed: dict = {}          # device -> int64[1] iteration counter mixed into every dropout mask


def iteration_seed(device) -> torch.Tensor:
    t = _iter_seed.get(device)
    if t is None:
        t = torch.zeros(1, dtype=torch.int64, device=device)
        _iter_seed[device] = t
    return t


def bump_iteration_seed(device):
    """Advance the on-device iteration counter (called once per training step; capturable in a CUDA graph)."""
    iteration_seed(device).add_(1)


class _DropoutFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, ratio, seed):
        ctx.ratio, ctx.seed = ratio, seed
        ctx.seed_t = iteration_seed(x.device)
        return K().dropout_apply(x, ratio, seed, ctx.seed_t)

    @staticmethod
    def backward(ctx, dy):
        dy = dy if dy.dtype == torch.bfloat16 else dy.to(torch.bfloat16)
        dy = dy if (dy.is_contiguous() or (dy.dim() == 4 and dy.is_contiguous(memory_format=CL))) else dy.contiguous()
        return K().dropout_apply(dy, ctx.ratio, ctx.seed, ctx.seed_t), None, None


def dropout(x, ratio, train):
    if not train:
        return x
    dense = x.is_contiguous() or (x.dim() == 4 and x.is_contiguous(memory_format=CL))
    if not _on(x) or x.dtype != torch.bfloat16 or x.numel() % 8 or not dense:
        return R.dropout(x, ratio, train)
    _dropout_counter[0] += 1          # distinct per call site within an iteration (a constant under graph replay)
    seed = (torch.initial_seed() * 1000003 + _dropout_counter[0] * 7919) & 0x7FFFFFFFFFFFFFFF
    return _DropoutFn.apply(x, float(ratio), int(seed))


class _SoftmaxLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, label, want_prob):
        x2 = x.reshape(x.shape[0], -1)
        if x2.stride(1) != 1:
            x2 = x2.contiguous()
        lab = label.reshape(-1).float().contiguous()
        loss, dx, prob = K().softmax_xent(x2, lab, 1.0, True, bool(want_prob))
        ctx.save_for_backward(dx)
        ctx.x_shape = tuple(x.shape)
        ctx.mark_non_differentiable(prob)
        return loss.reshape(()), prob

    @staticmethod
    def backward(ctx, dloss, _dprob):
        (dx,) = ctx.saved_tensors
        g = dx * dloss.to(dx.dtype)
        return g.view(ctx.x_shape), None, None


def softmax_loss(x, label, return_prob=False):
    spatial = x.dim() == 4 and x.shape[2] * x.shape[3] > 1
    if not _on(x) or spatial:
        return R.softmax_loss(x, label, return_prob)
    loss, prob = _SoftmaxLossFn.apply(x, label, return_prob)
    if return_prob:
        return loss, prob.view(x.shape[0], -1, 1, 1)
    return loss


class _SoftmaxFn(torch.autograd.Function):
    """Channel softmax: with NHWC memory every (n, h, w) position is one contiguous row (softmax_layer.cu:14-149)."""

    @staticmethod
    def forward(ctx, x):
        y = K().softmax_fwd(x)
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        dy = dy if dy.dtype == torch.bfloat16 else dy.to(torch.bfloat16)
        dy = as_kernel_input(dy) if dy.dim() == 4 else (dy if dy.stride(1) == 1 else dy.contiguous())
        return K().softmax_bwd(y, dy)


def softmax(x):
    if not _on(x) or x.dtype != torch.bfloat16 or x.dim() not in (2, 4):
        return R.softmax(x)
    if x.dim() == 4:
        x = as_kernel_input(x)
    elif x.stride(1) != 1:
        x = x.contiguous()
    return _SoftmaxFn.apply(x)


# ---- elementwise neurons: Sigmoid / TanH / AbsVal / BNLL / Power / Threshold ------------------------------------------
U_SIGMOID, U_TANH, U_ABSVAL, U_BNLL, U_POWER, U_THRESHOLD = range(6)


def _unary_ok(x: torch.Tensor) -> bool:
    dense = x.is_contiguous() or _cl_dense(x)
    return _on(x) and x.dtype == torch.bfloat16 and dense and x.data_ptr() % 16 == 0


class _UnaryFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, op, a, b, c):
        y = K().unary_fwd(x, op, a, b, c)
        ctx.args = (op, a, b, c)
        ctx.save_for_backward(y if op in (U_SIGMOID, U_TANH) else x)       # what the reference's backward reads
        return y

    @staticmethod
    def backward(ctx, dy):
        (s,) = ctx.saved_tensors
        op, a, b, c = ctx.args
        if op == U_THRESHOLD:
            return None, None, None, None, None
        dy = dy if dy.dtype == torch.bfloat16 else dy.to(torch.bfloat16)
        if dy.stride() != s.stride():
            dy = torch.empty_like(s).copy_(dy)
        return K().unary_bwd(s, dy, op, a, b, c), None, None, None, None


def _unary(x, op, a=0.0, b=0.0, c=0.0, fallback=None):
    if not _unary_ok(x):
        return fallback(x)
    return _UnaryFn.apply(x, op, float(a), float(b), float(c))


def sigmoid(x):
    return _unary(x, U_SIGMOID, fallback=torch.sigmoid)


def tanh(x):
    return _unary(x, U_TANH, fallback=torch.tanh)


def absval(x):
    return _unary(x, U_ABSVAL, fallback=torch.abs)


def bnll(x):
    return _unary(x, U_BNLL, fallback=R.bnll)


def power(x, pw, scale, shift):
    return _unary(x, U_POWER, pw, scale, shift, fallback=lambda t: R.power(t, pw, scale, shift))


def threshold(x, t):
    return _unary(x, U_THRESHOLD, t, fallback=lambda v: (v > t).to(v.dtype))


# ---- Eltwise ---------------------------------------------------------------------------------------------------------
_ELT = {"PROD": 0, "SUM": 1, "MAX": 2}


class _EltwiseFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, op, coeffs, *xs):
        need_grad = any(x.requires_grad for x in xs)
        y, mask = K().eltwise_fwd(list(xs), op, list(coeffs), need_grad)
        ctx.op, ctx.coeffs = op, coeffs
        ctx.save_for_backward(mask, *(xs if op == 0 else xs[:1]))       # PROD reads its bottoms again; SUM / MAX do not
        ctx.n = len(xs)
        return y

    @staticmethod
    def backward(ctx, dy):
        mask, *saved = ctx.saved_tensors
        ref = saved[0]
        dy = dy if dy.dtype == torch.bfloat16 else dy.to(torch.bfloat16)
        if dy.stride() != ref.stride():
            dy = torch.empty_like(ref).copy_(dy)
        xs = saved if ctx.op == 0 else [ref] * ctx.n
        need = [1 if g else 0 for g in ctx.needs_input_grad[2:]]
        outs = K().eltwise_bwd(list(xs), dy, mask, ctx.op, list(ctx.coeffs), need)
        return (None, None) + tuple(o if n else None for o, n in zip(outs, need))


def eltwise(xs, op="SUM", coeffs=None):
    ok = 2 <= len(xs) <= 8 and all(_unary_ok(x) and x.stride() == xs[0].stride() for x in xs) and xs[0].numel() % 8 == 0
    if not ok:
        return R.eltwise(xs, op, coeffs)
    return _EltwiseFn.apply(_ELT[op], tuple(float(c) for c in (coeffs or [])), *xs)


# ---- MVN ---------------------------------------------------------------------------------------------------------------
class _MVNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, nv, ac):
        y, stats = K().mvn_fwd(x, nv, ac)
        ctx.save_for_backward(y, stats)
        ctx.args = (nv, ac)
        return y

    @staticmethod
    def backward(ctx, dy):
        y, stats = ctx.saved_tensors
        nv, ac = ctx.args
        return K().mvn_bwd(y, as_kernel_input(dy), stats, nv, ac), None, None


def mvn(x, normalize_variance=True, across_channels=False):
    if not _on(x) or x.dim() != 4 or x.shape[1] % 8 or x.dtype != torch.bfloat16:
        return R.mvn(x, normalize_variance, across_channels)
    return _MVNFn.apply(as_kernel_input(x), bool(normalize_variance), bool(across_channels))


class _SlabConcatFn(torch.autograd.Function):
    """CONCAT over channels whose bottoms were written by their producers straight into one slab (channel-offset views
    with the slab's pixel pitch): forward is the identity on memory, backward hands out channel slices of dY.
    reference: src/caffe/layers/concat_layer.cu:10-72 copies every bottom (forward) and every slice (backward)."""

    @staticmethod
    def forward(ctx, slab, sizes, *xs):
        ctx.sizes = sizes
        return slab

    @staticmethod
    def backward(ctx, dy):
        return (None, None) + tuple(torch.split(dy, ctx.sizes, dim=1))


def concat(xs, dim, layer=None):
    slab = getattr(layer, "_slab", None) if layer is not None else None
    if slab is not None and dim == 1:
        layer._slab = None                       # the next forward pass allocates a fresh slab
        off, ok = 0, True
        for x in xs:
            ok = ok and x.data_ptr() == slab.data_ptr() + off * slab.element_size() and x.shape[1] + off <= slab.shape[1] \
                and x.shape[0] == slab.shape[0] and tuple(x.shape[2:]) == tuple(slab.shape[2:])
            off += x.shape[1]
        if ok and off == slab.shape[1]:
            if not torch.is_grad_enabled() or not any(x.requires_grad for x in xs):
                return slab
            return _SlabConcatFn.apply(slab, tuple(x.shape[1] for x in xs), *xs)
    return torch.cat([x if x.dtype == xs[0].dtype else x.to(xs[0].dtype) for x in xs], dim=dim)


def transform(transformer, x, out_dtype, first_conv=None):
    """uint8/float NCHW batch -> bf16 NHWC in one kernel (crop / mirror / mean / scale / channel pad)."""
    if not _on(x) or out_dtype != torch.bfloat16:
        return TE.transform(transformer, x, out_dtype)
    n, c, h, w = x.shape
    oh, ow = transformer.out_hw(h, w)
    h_off, w_off, flip = transformer.draw(n, h, w)
    dev = x.device
    mean = None
    if transformer.mean is not None:
        mean = transformer.mean.to(dev).float().contiguous()
    elif transformer.mean_values is not None:
        mv = transformer.mean_values.to(dev).float()
        mean = (mv.expand(c) if mv.numel() == 1 else mv).contiguous()
    cp = 4 if c <= 4 else 8
    if c > 8:
        return TE.transform(transformer, x, out_dtype).contiguous(memory_format=CL)
    if first_conv is None or getattr(first_conv, "_sm100", None) is None or not first_conv._sm100.row_mode:
        # generic consumer: logical (N,C,oh,ow) bf16 channels-last
        return TE.transform(transformer, x, out_dtype).contiguous(memory_format=CL)
    opad = first_conv.pad
    if opad[0] != opad[1]:
        return TE.transform(transformer, x, out_dtype).contiguous(memory_format=CL)
    xin = x if x.dtype in (torch.uint8, torch.float32) else x.float()
    st = first_conv._sm100
    if st.pad8:
        if (oh, ow) != tuple(first_conv.in_hw):
            return TE.transform(transformer, x, out_dtype).contiguous(memory_format=CL)
        return K().transform_nhwc(xin.contiguous(), h_off.to(dev, torch.int32), w_off.to(dev, torch.int32),
                                  flip.to(dev, torch.uint8), mean, float(transformer.scale), oh, ow, 8, 0, 0, 0, False)
    if st.s2d:
        hq, wq = st.s2d_hw
        if cp != 4 or (oh, ow) != tuple(first_conv.in_hw):
            return TE.transform(transformer, x, out_dtype).contiguous(memory_format=CL)
        return K().transform_nhwc(xin.contiguous(), h_off.to(dev, torch.int32), w_off.to(dev, torch.int32),
                                  flip.to(dev, torch.uint8), mean, float(transformer.scale), oh, ow, cp, opad[0],
                                  4 * wq - ow - 2 * opad[1], 4 * hq - oh - 2 * opad[0], True)
    wextra = (ow + 2 * opad[1]) % 2      # even physical width => every image row starts 16-byte aligned
    return K().transform_nhwc(xin.contiguous(), h_off.to(dev, torch.int32), w_off.to(dev, torch.int32),
                              flip.to(dev, torch.uint8), mean, float(transformer.scale), oh, ow, cp, opad[0], wextra,
                              0, False)
