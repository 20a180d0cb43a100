"""bf16 convolution kernels (conv_fprop, conv_dgrad, conv_dgrad_w) against float64 references, on rectangular geometry,
channel slices and every schedule.

Each result is checked element by element against a float64 reference computed on the CPU from the exact bf16 inputs and
the bf16 operand the kernel reads, with the GEMM bound of test_accumulate_gpu.py followed by one bf16 rounding:

    |got - ref| <= C_GEMM * K * u * (|x|·|w| + |b|), then half a bf16 ulp      (K = R·S·C_g fprop, R·S·Cout_g dgrad)

where |x|·|w| is the same convolution on absolute values.  The epilogue (bias, ReLU / leaky ReLU, producer mask) is part of
the reference.

Layouts.  Every input sits in a NaN-filled allocation: dense between NaN guard regions, or as a 16-byte aligned channel
slice of a wider slab whose other channels are NaN.  A read outside the tensor (a neighbour's channels in a concat slab,
the channel-padded K slots the TMA must zero-fill, pixels past the end) turns the result into NaN, which fails the bound.
Outputs are written either to a fresh tensor or into a channel slice of a sentinel-filled slab; the rest of the slab and
the guard bands around it must come back bit for bit (a ragged last N tile that stores past Cout would overwrite the
neighbouring concat branch).

The ops run on ``EmulatedKernels`` (CPU: validates references, bounds and guards without a GPU) and on the sm_90a
extension under every schedule knob.  The schedules do not change the arithmetic's contract, so each must pass the same
bound."""
import functools

import pytest
import torch
import torch.nn.functional as F

from test_accumulate_gpu import C_GEMM, U, _assert_guard, _bf16_bound, _dev, _guarded, _randn, _within

BF16 = torch.bfloat16
CL = torch.channels_last
NAN = float("nan")

# Largest err / bound measured on an H100 80GB HBM3 at a 400 W power limit, over every case and schedule: conv_fprop 0.98,
# conv_dgrad 0.98, conv_dgrad_w 0.98; through the engine 0.91 (forward), 0.94 (data gradient), 0.018 (weight gradient).
# At these reduction lengths the half-ulp bf16 rounding of the output is nearly all of the bound, so a correctly rounded
# result can come close to 1; the fp32 accumulation term (C_GEMM) is a small part of it.  A dropped or misplaced tap, a
# swapped axis or a NaN read from outside the input is off by far more.

# ------------------------------------------------------------------------------------------------------------ schedules
# knob -> value the kernels ship with
KNOB_DEFAULTS = {"set_conv_pair": 1, "set_conv_mcast": 1, "set_conv_im2col": 1, "set_conv_cluster": 1, "set_max_stages": 0}
SCHEDULES = {
    "pair": {},                               # default: CTA pairs on the im2col path when there are >= 2 pixel blocks
    "single": {"set_conv_pair": 0},           # one CTA per tile
    "mcast2": {"set_conv_mcast": 2},          # im2col operand shared by TMA multicast in clusters of 2 / 4
    "mcast4": {"set_conv_mcast": 4},
    "gather": {"set_conv_im2col": 0},         # cp.async gather producer for every geometry (the A/B knob of conv_bench.py)
    "cluster2": {"set_conv_cluster": 2},      # gather path, weight tile multicast to 2 / 4 pixel blocks (phantom blocks
    "cluster4": {"set_conv_cluster": 4},      # when the block count does not divide)
    "stages2": {"set_max_stages": 2},         # ring depth 2
}
NO_IM2COL = ("gather", "cluster2", "cluster4")   # a channel-padded operand needs the TMA im2col path these turn off


@pytest.fixture(params=[pytest.param("emu", id="emu")] +
                [pytest.param(s, id="gpu-" + s, marks=pytest.mark.gpu) for s in SCHEDULES])
def ks(request):
    """(op surface, schedule name): the CPU emulation, or the sm_90a extension with one schedule knob set."""
    if request.param == "emu":
        from poseidon_b200.ops.emulate import EmulatedKernels
        yield EmulatedKernels(), "emu"
        return
    ext = request.getfixturevalue("ext")
    try:
        for knob, v in SCHEDULES[request.param].items():
            getattr(ext, knob)(v)
        yield ext, request.param
    finally:
        for knob, v in KNOB_DEFAULTS.items():
            getattr(ext, knob)(v)


# ------------------------------------------------------------------------------------------------------------ layouts
def _in_slab(t, off, dev):
    """t [N, C, H, W] as channels [off, off + C) of a NaN-filled channels-last slab (pixel pitch C + off + 8 when off > 0,
    else C: dense), at element offset 16 of a NaN-filled allocation with 32 NaN elements behind the slab."""
    n, c, h, w = t.shape
    pitch = c + off + 8 if off else c
    buf = torch.full((16 + n * h * w * pitch + 32,), NAN, dtype=BF16, device=dev)
    slab = torch.as_strided(buf, (n, pitch, h, w), (h * w * pitch, 1, w * pitch, pitch), 16)
    v = slab[:, off: off + c]
    v.copy_(t)
    return v


def _out_slab(n, c, h, w, off, dev):
    """(allocation, view): channels [off, off + C) of a sentinel-filled slab with pixel pitch C + off + 8."""
    pitch = c + off + 8
    buf, slab = _guarded((n, pitch, h, w), (h * w * pitch, 1, w * pitch, pitch), BF16, dev)
    return buf, slab[:, off: off + c]


LAYOUTS = {"dense": 0, "slice8": 8, "slice16": 16}      # channel offset of the input / output slice (0: dense)


def _act(v, relu, slope):
    return torch.where(v > 0, v, v * slope) if relu else v


# ------------------------------------------------------------------------------------------------------------ conv_fprop
# (N, Cin, H, W, Cout, (R, S), (sh, sw), (ph, pw), groups, Cgk, mode): Cgk 0 = dense operand (R·S·C_g columns), else the
# channel-padded operand from conv_pack_padded; mode 1 = ROW (first layer: H x W is the pre-padded NHWC4 image, whose last
# column is the even-width padding the transform writes).  m = pixel blocks of 128 (N·OH·OW / 128, rounded up).
FPROP = [
    ((2, 64, 12, 20, 72, (1, 7), (1, 1), (0, 3), 1, 0, 0), "1x7, pad (0,3), im2col C_g 64, m 4, Cout 72 vs the 64 tile"),
    ((2, 128, 17, 9, 40, (7, 1), (1, 1), (3, 0), 1, 0, 0), "7x1, pad (3,0), m 3, Cout 40 (one ragged 64 tile)"),
    ((1, 64, 15, 22, 200, (3, 5), (1, 2), (1, 2), 1, 0, 0), "3x5, stride (1,2), pad (1,2), batch 1, m 2, Cout 200 vs 256"),
    ((2, 192, 19, 11, 136, (3, 5), (2, 1), (1, 2), 1, 0, 0), "3x5, stride (2,1), C_g 192, m 2, Cout 136 vs 192 / 128"),
    ((3, 24, 1, 37, 104, (1, 3), (1, 1), (0, 1), 1, 0, 0), "H == 1, gather C_g 24 (k-blocks straddle taps), Cout 104"),
    ((2, 40, 23, 1, 48, (3, 1), (1, 1), (1, 0), 1, 0, 0), "W == 1, gather C_g 40 (k-blocks straddle taps), Cout 48"),
    ((2, 8, 13, 21, 24, (5, 3), (2, 1), (2, 1), 1, 0, 0), "C_g 8, stride (2,1), pad (2,1), Cout 24"),
    ((2, 96, 10, 14, 264, (3, 5), (1, 1), (1, 2), 1, 128, 0), "channel-padded 96 -> 128, 3x5, Cout 264 vs 256 (+8)"),
    ((2, 256, 9, 13, 144, (3, 1), (1, 2), (1, 0), 2, 0, 0), "groups 2, C_g 128, Cout_g 72, stride (1,2)"),
    ((2, 80, 11, 16, 208, (3, 3), (1, 1), (1, 1), 2, 0, 0), "groups 2, gather C_g 40, Cout_g 104"),
    ((1, 64, 30, 27, 328, (3, 3), (1, 1), (1, 1), 1, 0, 0), "m 7 (7 % 4 = 3), Cout 328: 256 + 72 / multicast tiles of 96"),
    ((1, 128, 40, 16, 64, (1, 1), (1, 1), (0, 0), 1, 0, 0), "1x1, m 5 (5 % 4 = 1): one phantom-padded cluster"),
    ((2, 64, 24, 10, 96, (7, 1), (2, 1), (3, 0), 1, 0, 0), "7x1, stride (2,1), pad (3,0), m 2, Cout 96"),
    ((6, 128, 16, 13, 160, (1, 7), (1, 2), (0, 3), 1, 0, 0), "1x7, stride (1,2), pad (0,3), m 6 (6 % 4 = 2), Cout 160"),
    ((2, 192, 14, 11, 32, (3, 5), (2, 2), (0, 3), 1, 0, 0), "pad (0,3) with 3x5 / stride 2, Cout 32"),
    ((2, 4, 21, 30, 48, (5, 3), (1, 2), (0, 0), 1, 0, 1), "ROW mode, 5x3, stride (1,2), Cout 48"),
    ((1, 4, 39, 40, 96, (11, 11), (4, 4), (0, 0), 1, 0, 1), "ROW mode, 11x11 / 4 (AlexNet conv1 shape), Cout 96"),
]
FPROP_PARAMS = [pytest.param(c, id=d.split(",")[0].replace(" ", "") + "-" + "x".join(map(str, c[:5]))) for c, d in FPROP]
EPILOGUES = {"plain": (False, None), "bias_relu": (True, 0.0), "bias_leaky": (True, 0.1), "leaky": (False, 0.1)}


def _fprop_out_hw(case):
    n, cin, h, w, cout, (r, s), (sh, sw), (ph, pw), g, cgk, mode = case
    if mode == 1:
        return (h - r) // sh + 1, (w - 1 - s) // sw + 1
    return (h + 2 * ph - r) // sh + 1, (w + 2 * pw - s) // sw + 1


@functools.lru_cache(maxsize=None)
def _fprop_ref(case):
    """(x, wk [Cout, R, S, C_g] bf16, bias fp32, pre-activation conv and |x|·|w| in float64)."""
    n, cin, h, w, cout, (r, s), stride, pad, g, cgk, mode = case
    seed = sum(case[:5]) + 31 * r + s
    x = _randn((n, cin, h, w), seed, dtype=BF16)
    wk = _randn((cout, r, s, cin // g), seed + 1, (r * s * cin // g) ** -0.5, dtype=BF16)
    bias = _randn((cout,), seed + 2, 0.5)
    w4 = wk.double().permute(0, 3, 1, 2)
    oh, ow = _fprop_out_hw(case)
    p = (0, 0) if mode == 1 else pad
    v = F.conv2d(x.double(), w4, None, stride, p, 1, g)[:, :, :oh, :ow]
    mag = F.conv2d(x.double().abs(), w4.abs(), None, stride, p, 1, g)[:, :, :oh, :ow]
    return x, wk, bias, v, mag


def _fprop_operand(k, wk, cgk, mode, dev):
    cout, r, s, cg = wk.shape
    if mode == 1:
        lp = (s * cg + 7) // 8 * 8
        return F.pad(wk.reshape(cout, r, s * cg), (0, lp - s * cg)).reshape(cout, r * lp).contiguous().to(dev)
    wb = wk.reshape(cout, r * s * cg).contiguous().to(dev)
    return k.conv_pack_padded(wb.reshape(-1), cout, r * s, cg, cgk, None) if cgk else wb


@pytest.mark.parametrize("case", FPROP_PARAMS)
@pytest.mark.parametrize("epi", list(EPILOGUES))
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_conv_fprop_contract(ks, case, epi, layout):
    """y = act(conv(x, w) + bias) in TAP mode (dense and channel-padded operand) and ROW mode, from a dense or sliced
    input, into a fresh tensor or a channel slice of a wider slab."""
    k, sched = ks
    n, cin, h, w, cout, kern, stride, pad, g, cgk, mode = case
    if cgk and sched in NO_IM2COL:
        pytest.skip("the channel-padded operand needs the TMA im2col path")
    dev = _dev(k)
    off = LAYOUTS[layout]
    x, wk, bias, v, mag = _fprop_ref(case)
    use_bias, slope = EPILOGUES[epi]
    oh, ow = _fprop_out_hw(case)
    xin = _in_slab(x, 0 if mode == 1 else off, dev)
    buf = out = None
    if off:
        buf, out = _out_slab(n, cout, oh, ow, off, dev)
    got = k.conv_fprop(xin, _fprop_operand(k, wk, cgk, mode, dev), bias.to(dev) if use_bias else None, list(kern),
                       list(stride), list(pad), g, mode, oh, ow, slope is not None, slope or 0.0, out)
    assert tuple(got.shape) == (n, cout, oh, ow)
    b64 = bias.double().view(1, -1, 1, 1) if use_bias else 0.0
    ref = _act(v + b64, slope is not None, slope or 0.0)
    kk = kern[0] * kern[1] * (cin // g)
    _within(got, ref, _bf16_bound(ref, C_GEMM * kk * U * (mag + (b64.abs() if use_bias else 0.0))), f"conv_fprop [{sched}]")
    if off:
        assert got.data_ptr() == out.data_ptr()
        _assert_guard(buf, [out], f"conv_fprop out slab [{sched}]")


# ------------------------------------------------------------------------------------------------------------ data gradient
# (N, Cin, H, W, Cout, (R, S), (ph, pw), groups, Cop, (eh, ew)): dY has the stride-1 extent of a convolution over H x W;
# dX is asked for at (H + eh) x (W + ew) — what the strided data gradient does per phase.  Cop 0 = packed operand with
# Cout_g slots per tap, else Cop slots (zero beyond Cout_g).  The K dimension is (r, s, co): im2col when Cout_g (or Cop) is a
# multiple of 64, else the gather producer; the N dimension is C_g.
DGRAD = [
    ((2, 64, 12, 20, 72, (1, 7), (0, 3), 1, 0, (0, 0)), "1x7, pad (0,3), gather (Cout_g 72), C_g 64"),
    ((2, 64, 12, 20, 72, (1, 7), (0, 3), 1, 128, (0, 0)), "as above, channel-padded operand: 72 -> 128 slots, im2col"),
    ((2, 40, 17, 9, 128, (7, 1), (3, 0), 1, 0, (0, 0)), "7x1, pad (3,0), im2col, C_g 40 (one ragged 64 tile)"),
    ((1, 200, 15, 22, 64, (3, 5), (1, 2), 1, 0, (0, 0)), "3x5, pad (1,2), batch 1, C_g 200 vs 256"),
    ((2, 136, 1, 37, 96, (1, 3), (0, 1), 1, 128, (0, 0)), "H == 1, 96 -> 128 slots, C_g 136"),
    ((2, 48, 23, 1, 24, (3, 1), (1, 0), 1, 0, (0, 0)), "W == 1, gather Cout_g 24 (k-blocks straddle taps)"),
    ((2, 144, 9, 13, 256, (3, 1), (1, 0), 2, 0, (0, 0)), "groups 2, Cout_g 128, C_g 72"),
    ((2, 208, 11, 16, 80, (3, 3), (1, 1), 2, 0, (0, 0)), "groups 2, gather Cout_g 40, C_g 104"),
    ((1, 64, 30, 27, 192, (3, 3), (1, 1), 1, 0, (0, 0)), "m 7, C_g 64, Cout_g 192 (3 k-blocks per tap)"),
    ((3, 128, 16, 13, 64, (1, 1), (0, 0), 1, 0, (0, 0)), "1x1, m 5"),
    ((2, 64, 7, 9, 64, (2, 3), (0, 1), 1, 0, (1, 0)), "phase extent: one row more than the transposed convolution's"),
    ((2, 64, 9, 7, 128, (3, 2), (1, 0), 1, 0, (0, -1)), "phase extent: one column less"),
]
DGRAD_PARAMS = [pytest.param(c, id=d.split(",")[0].replace(" ", "") + "-" + "x".join(map(str, c[:5]))) for c, d in DGRAD]
MASKS = {"nomask": None, "mask": 0.0, "mask_leaky": 0.1}


@functools.lru_cache(maxsize=None)
def _dgrad_ref(case):
    """(dY, wk [Cout, R, S, C_g] bf16, mask, dX and |dY|·|w| in float64 at the requested extent)."""
    n, cin, h, w, cout, (r, s), (ph, pw), g, cop, (eh, ew) = case
    seed = sum(case[:5]) + 31 * r + s + 7
    oh, ow = h + 2 * ph - r + 1, w + 2 * pw - s + 1
    hr, wr = h + eh, w + ew
    dy = _randn((n, cout, oh, ow), seed, dtype=BF16)
    wk = _randn((cout, r, s, cin // g), seed + 1, (r * s * cout // g) ** -0.5, dtype=BF16)
    mask = _randn((n, cin, hr, wr), seed + 2, dtype=BF16).contiguous(memory_format=CL)
    w4 = wk.double().permute(0, 3, 1, 2)

    def tconv(a, b):
        full = F.conv_transpose2d(a, b, None, 1, 0, 0, g)
        full = F.pad(full, (0, max(0, pw + wr - full.shape[3]), 0, max(0, ph + hr - full.shape[2])))
        return full[:, :, ph: ph + hr, pw: pw + wr]
    return dy, wk, mask, tconv(dy.double(), w4), tconv(dy.double().abs(), w4.abs())


@pytest.mark.parametrize("case", DGRAD_PARAMS)
@pytest.mark.parametrize("op", ["conv_dgrad", "conv_dgrad_w"])
@pytest.mark.parametrize("masking", list(MASKS))
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_conv_dgrad_contract(ks, case, op, masking, layout):
    """dX = conv_transpose(dY, w), cropped / zero-extended to the requested extent, then the producer's ReLU mask with
    slope 0 or 0.1 — from the packed operand (conv_pack_dgrad, Cop >= Cout_g) and from the fprop operand (conv_dgrad_w), with
    dY dense or a channel slice of a NaN-filled slab."""
    k, sched = ks
    n, cin, h, w, cout, kern, pad, g, cop, (eh, ew) = case
    if op == "conv_dgrad_w" and (cop or sched == "gather"):
        pytest.skip("conv_dgrad_w reads the fprop operand on the TMA im2col path only (it pads the slots itself)")
    if op == "conv_dgrad" and cop and sched in NO_IM2COL:
        pytest.skip("the channel-padded operand needs the TMA im2col path")
    dev = _dev(k)
    dy, wk, mask, ref, mag = _dgrad_ref(case)
    r, s = kern
    cg = cin // g
    hr, wr = h + eh, w + ew
    slope = MASKS[masking]
    m = None if slope is None else mask.to(dev)
    dyin = _in_slab(dy, LAYOUTS[layout], dev)
    if op == "conv_dgrad":
        wt = k.conv_pack_dgrad(wk.float().reshape(-1).to(dev), cout, r * s, cg, g, None, cop)
        got = k.conv_dgrad(dyin, wt, list(kern), list(pad), g, hr, wr, m, slope or 0.0)
    else:
        got = k.conv_dgrad_w(dyin, wk.reshape(cout, r * s * cg).contiguous().to(dev), list(kern), list(pad), g, hr, wr, m,
                             slope or 0.0)
    assert tuple(got.shape) == (n, cin, hr, wr)
    want = ref if slope is None else torch.where(mask.double() > 0, ref, ref * slope)
    bound = _bf16_bound(want, C_GEMM * r * s * (cout // g) * U * mag)
    _within(got, want, bound, f"{op} [{sched}]")


# ------------------------------------------------------------------------------------------------------------ engine layers
# Rectangular strided layers through sm100.conv2d: forward, and the backward the engine runs for them — the data gradient as
# sh·sw stride-1 phase problems (_strided_dgrad), the weight gradient, the bias gradient.
ENGINE = [
    # (N, Cin, H, W, Cout, kernel, stride, pad, group, relu, mask_input)
    ((2, 64, 15, 12, 96, (3, 1), (1, 2), (1, 0), 1, True, True), "sh != sw; stride 2 > kernel 1 along w: phases with no tap"),
    ((2, 64, 14, 17, 64, (1, 3), (3, 2), (0, 1), 1, False, True), "stride 3 > kernel 1 along h, stride 2 along w"),
    ((2, 128, 13, 11, 144, (3, 5), (2, 1), (1, 2), 2, True, False), "grouped 3x5, stride (2,1), pad (1,2), Cout_g 72"),
    ((1, 40, 9, 16, 48, (5, 3), (2, 3), (2, 1), 1, True, True), "gather C_g 40, 5x3, stride (2,3)"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", [pytest.param(c, id=f"engine{i}") for i, (c, _) in enumerate(ENGINE)])
def test_conv_engine_rect_strided(ext, case):
    from poseidon_b200.ops import sm100
    from test_ops_gpu import _FakeLayer
    n, cin, h, w, cout, kern, stride, pad, g, relu, mask_input = case
    layer = _FakeLayer(cout, cin, kern, stride, pad, g)
    layer.in_hw = (h, w)
    sm100.conv_state(layer, cin).mask_input = mask_input      # this layer's data gradient applies the producer's ReLU
    x = _randn((n, cin, h, w), 41, dtype=BF16).contiguous(memory_format=CL)
    xs = x.cuda().requires_grad_(True)
    y = sm100.conv2d(xs, layer.weight, layer.bias, layer.stride, layer.pad, g, relu_slope=0.0 if relu else None,
                     layer=layer)
    w64 = layer.weight.detach().to(BF16).double().cpu()        # the bf16 shadow / packed operands the kernels read
    b64 = layer.bias.detach().double().cpu()
    x64 = x.double()
    v = F.conv2d(x64, w64, b64, stride, pad, 1, g)
    mag = F.conv2d(x64.abs(), w64.abs(), b64.abs(), stride, pad, 1, g)
    ref = _act(v, relu, 0.0)
    rs = kern[0] * kern[1]
    _within(y, ref, _bf16_bound(ref, C_GEMM * rs * (cin // g) * U * mag), "engine conv forward")

    dy = _randn(tuple(y.shape), 42, dtype=BF16).contiguous(memory_format=CL)
    y.backward(dy.cuda())
    dym = torch.where(y.detach().cpu() > 0, dy, torch.zeros_like(dy)).double() if relu else dy.double()
    dx = torch.nn.grad.conv2d_input(x.shape, w64, dym, stride, pad, 1, g)
    dmag = torch.nn.grad.conv2d_input(x.shape, w64.abs(), dym.abs(), stride, pad, 1, g)
    bound = _bf16_bound(dx, C_GEMM * rs * (cout // g) * U * dmag)
    if mask_input:
        dx = torch.where(x64 > 0, dx, torch.zeros_like(dx))
    _within(xs.grad, dx, bound, "engine conv data gradient")
    red = n * y.shape[2] * y.shape[3]
    dw = torch.nn.grad.conv2d_weight(x64, tuple(w64.shape), dym, stride, pad, 1, g)
    wmag = torch.nn.grad.conv2d_weight(x64.abs(), tuple(w64.shape), dym.abs(), stride, pad, 1, g)
    _within(layer.weight.grad, dw, C_GEMM * red * U * wmag, "engine conv weight gradient")
    _within(layer.bias.grad, dym.sum((0, 2, 3)), C_GEMM * red * U * dym.abs().sum((0, 2, 3)), "engine conv bias gradient")


# ------------------------------------------------------------------------------------------------------------ misaligned slices
def _misaligned(dev, sizes=(4, 8, 12)):
    """The middle part of torch.split(x, [4, 8, 12], 1) on a channels-last x [2, 24, 9, 10]: a SLICE layer's output with
    8 channels, pitch 24, 8 bytes past a 16-byte boundary."""
    x = _randn((2, 24, 9, 10), 51, dtype=BF16).contiguous(memory_format=CL).to(dev)
    return torch.split(x, list(sizes), 1)[1]


def test_as_kernel_input_realigns_misaligned_slice():
    """A channel slice that does not start on a 16-byte boundary is copied to dense channels-last (the kernels read pixels
    with 16-byte loads); an aligned slice is handed over as it is."""
    from poseidon_b200.ops import sm100
    v = _misaligned("cpu")
    assert v.data_ptr() % 16 == 8 and v.stride(3) == 24
    got = sm100.as_kernel_input(v)
    assert got.data_ptr() % 16 == 0 and torch.equal(got, v)
    aligned = _misaligned("cpu", (8, 8, 8))
    assert sm100.as_kernel_input(aligned).data_ptr() == aligned.data_ptr()


@pytest.mark.gpu
def test_engine_misaligned_slice(ext):
    """sm100.conv2d and sm100.max_pool on the misaligned view give the float64 answer."""
    from poseidon_b200.ops import sm100
    from test_ops_gpu import _FakeLayer
    v = _misaligned("cuda")
    assert v.data_ptr() % 16 == 8
    layer = _FakeLayer(16, 8, 3, 1, 1, 1)
    layer.in_hw = (9, 10)
    y = sm100.conv2d(v, layer.weight, layer.bias, layer.stride, layer.pad, 1, relu_slope=None, layer=layer)
    x64 = v.cpu().double()
    w64 = layer.weight.detach().to(BF16).double().cpu()
    b64 = layer.bias.detach().double().cpu()
    ref = F.conv2d(x64, w64, b64, 1, 1)
    mag = F.conv2d(x64.abs(), w64.abs(), b64.abs(), 1, 1)
    _within(y, ref, _bf16_bound(ref, C_GEMM * 72 * U * mag), "conv2d on a misaligned slice")
    from poseidon_b200.ops import reference as R
    p = sm100.max_pool(v, (3, 2), (2, 1), (1, 0))
    assert torch.equal(p.cpu().double(), R.max_pool(x64, (3, 2), (2, 1), (1, 0))), "max_pool on a misaligned slice"


@pytest.mark.gpu
def test_raw_conv_rejects_misaligned_input(ext):
    """The conv ops check the gathered tensor's alignment on the host, before anything is launched."""
    v = _misaligned("cuda")                                     # [2, 8, 9, 10]
    assert v.data_ptr() % 16 == 8
    wb = _randn((16, 72), 52, 0.1, dtype=BF16).cuda()           # fprop operand: 8 -> 16 channels, 3x3
    with pytest.raises(RuntimeError, match="16-byte boundary"):
        ext.conv_fprop(v, wb, None, [3, 3], [1, 1], [1, 1], 1, 0, 9, 10, False, 0.0, None)
    # v as dY of a 16 -> 8 channel convolution
    wt = ext.conv_pack_dgrad(_randn((8 * 9 * 16,), 53, 0.1).cuda(), 8, 9, 16, 1, None, 0)
    with pytest.raises(RuntimeError, match="16-byte boundary"):
        ext.conv_dgrad(v, wt, [3, 3], [1, 1], 1, 9, 10, None, 0.0)
    with pytest.raises(RuntimeError, match="16-byte boundary"):
        ext.conv_dgrad_w(v, _randn((8, 144), 54, 0.1, dtype=BF16).cuda(), [3, 3], [1, 1], 1, 9, 10, None, 0.0)
    dy = _randn((2, 16, 9, 10), 55, dtype=BF16).contiguous(memory_format=CL).cuda()
    dw = torch.zeros(16, 72, device="cuda")
    with pytest.raises(RuntimeError, match="16-byte boundary"):
        ext.conv_wgrad(v, dy, dw, [3, 3], [1, 1], [1, 1], 1, 0, 1.0, 0)
    torch.cuda.synchronize()
    assert not dw.any()
