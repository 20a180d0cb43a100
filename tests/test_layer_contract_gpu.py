"""Layer kernels (pooling, across / within-channel LRN, channel softmax, softmax-loss, MVN, the unary neurons, eltwise,
ReLU, stochastic pooling) against float64 references, on every dispatch path and on channel slices.

Every reference is computed in float64 on the CPU from the exact bf16 inputs, following Caffe's loops
(src/caffe/layers/*.cu in the reference tree; file:line beside each reference), not torch's pooling or LRN.

Bounds.  u = 2^-24 (fp32), h = 2^-8 (half a bf16 ulp, relative).  bf16(e) below is test_accumulate_gpu._bf16_bound:
an fp32 error e, then one rounding to bf16, e + 4u|ref| + h(|ref| + e).
* Bit-exact: MAX pool forward (bf16 compares are exact; an empty window is -inf); MAX pool backward at pixels that are
  the arg-max of at most one window; AbsVal, Threshold and ReLU (slope 0) forward / backward; eltwise MAX forward and
  backward; the stochastic-pool pick.
* MAX pool backward at a pixel that is the arg-max of m > 1 windows: the kernel adds the dy values as packed bf16 pairs,
  so each of the m - 1 additions rounds to bf16.  Documented contract: |got - Σdy| <= m · h · Σ|dy| (m - 1 roundings of a
  partial sum at most Σ|dy|, plus the final half ulp).  A gradient routed to the wrong element is off by a whole dy.
* Sums of n fp32 terms: n·u·Σ|terms| (the usual γ_n bound to first order), plus a few u for the scaling around them.
  - AVE pool forward: bf16((k_h·k_w + 2)·u·Σ|x| / pool_size); backward bf16((⌈k_h/s_h⌉⌈k_w/s_w⌉ + 2)·u·Σ|dy| / pool_size).
  - MVN forward: E[x] and E[x²] carry (n + 2)·u relative error (n = H·W, or C·H·W across channels); var = E[x²] - E[x]²
    cancels, so std carries (n + 4)·u·E[x²] / var and y = (x - mean) / std
        |Δy| <= |y|·((n + 4)·u·E[x²] / var + 4u) + (n + 2)·u·E|x| / std.
    With a mean offset of 32σ, E[x²] / var is about 1000: the bound grows with it, as the kernel's error does.
  - MVN backward: bf16((n + 4)·u · inv·(|dy| + E|dy| + |y|·E|dy·y|)) from the forward's inv = 1 / (std + eps).
  - Stochastic pool, test phase (x >= 0, no cancellation): bf16((2·k_h·k_w + 4)·u·y).
* MUFU terms.  __expf(v) is within (2 + 1.17|v|) ulp, so 4u + 3u·|v| relative; lg2.approx / ex2.approx are within
  2^-22 absolute / relative; __logf is within 2^-21.4 absolute.
  - Softmax: e_i = __expf(x_i - max) carries r_i = (4 + 3|x_i - max|)·u; the sum (order unspecified) (C + 4)·u; so
    |Δy_i| <= bf16(y_i·(r_i + max_j r_j + (C + 4)·u)).  Backward dx = y·(dy - Σ y·dy): bf16((C + 4)·u·|y|·(|dy| + Σ|y·dy|)).
  - Softmax-loss: the same r_i on prob (fp32 output, plus 4u), dx = (p - 1[c = label])·g / rows with the same error
    plus 4u|dx| (bf16 dx: one more bf16 rounding); loss: mean over rows of (r_label + 2^-20), plus (rows + 8)·u·loss.
  - Across-channel LRN: the window sum slides over the 8 channels of a thread, so it is within (2n + 24)·u·S_E, where
    S_E is Σx² over the thread's channels widened by n - 1 on both sides (n = local_size); scale^-β = ex2(-β·lg2 scale):
        rel = (2n + 24)·u·(1 + β·(α/n)·S_E + β·|lg2 scale|) + 2^-21·(1 + β),    |Δy| <= bf16(rel·|y|).
    Backward dx = dy·scale^-β - (2αβ/n)·x·Σ r, r = dy·x·scale^(-β-1): bf16((rel + (2n + 32)·u)·(|dy|·scale^-β +
    (2αβ/n)·|x|·Σ_E |r|)).  With α/n around 0.3 and x ~ N(0, 2²), moving the window by one channel changes outputs by
    tens of bounds.
  - Within-channel LRN: the same form with the k²-term spatial window sum (k = local_size) in place of S_E.
  - Unary neurons: bf16(8u·|y| + (first-order propagation of the 2-ulp libm / MUFU error through the op)); see _unary_ref.
  - Eltwise PROD of n bottoms: bf16((n + 1)·u·|y|); SUM: bf16((n + 2)·u·Σ|c_j·x_j|).

Layouts.  Inputs that a kernel reads with a pixel pitch run dense (in a NaN-guarded allocation) and as a channel slice at
offset 8 and 16 of a NaN-filled slab (test_conv_contract_gpu._in_slab); a read outside the slice turns into NaN and
fails the bound.  Dense-only ops (unary, eltwise, relu_fwd / relu_bwd, dropout_apply) get NaN guard bands directly
behind their last element, which also covers the scalar tail loop.  Outputs must come back dense channels-last (or with
the input's strides for the dense-only ops) with the expected shape.

Every case runs on ``EmulatedKernels`` (CPU) and on the sm_90a extension (``gpu`` mark).  test_dispatch_coverage repeats
the host-side dispatch arithmetic over the case lists and fails if a kernel instantiation is no longer reached."""
import math

import pytest
import torch
import torch.nn.functional as F

from test_accumulate_gpu import U, _bf16_bound, _dev, _randn
from test_conv_contract_gpu import _in_slab

BF16 = torch.bfloat16
F64 = torch.float64
CL = torch.channels_last
NAN = float("nan")
INF = float("inf")
H = 2.0 ** -8

# Largest err / bound measured on an H100 80GB HBM3 at a 400 W power limit, over every case and layout (the module prints
# them with -s): pool_fwd 0.87 (AVE; MAX is exact), pool_bwd 0.996 (AVE; MAX is exact at m <= 1), lrn_fwd 0.99, lrn_bwd 0.97,
# lrn_within_fwd 0.98, lrn_within_bwd 0.97, softmax_fwd 0.99, softmax_bwd 0.97, softmax_xent 0.97, mvn_fwd 0.99,
# mvn_bwd 0.99, sigmoid 0.99, tanh 0.96, bnll 0.99, power 0.996, eltwise_fwd 0.99, eltwise_bwd 0.98, relu (slope 0.1) 0.79,
# stochastic_pool 0.96, through the engine 0.99; AbsVal, Threshold and every exact check 0.  The half-ulp bf16 rounding
# of the output is nearly all of each bound, so a correctly rounded result comes close to 1; the fp32 / MUFU terms are
# a small part.  A shifted window, a misrouted gradient or a NaN read from outside the input is off by far more.

_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    """Prints the largest err / bound per op once the module has run (visible with -s)."""
    yield
    if _WORST:
        print("\nlargest err/bound: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(_WORST.items())))


@pytest.fixture(params=[pytest.param("emu", id="emu"), pytest.param("gpu", id="gpu", marks=pytest.mark.gpu)])
def k(request):
    """The op surface: the CPU emulation or the sm_90a extension."""
    if request.param == "emu":
        from poseidon_b200.ops.emulate import EmulatedKernels
        return EmulatedKernels()
    return request.getfixturevalue("ext")


# ------------------------------------------------------------------------------------------------------------ checks
def _close(got, ref, bound, what):
    """|got - ref| <= bound elementwise; equal values (±inf included) always pass, NaN passes only where ref is NaN."""
    g = got.detach().cpu().double()
    assert g.shape == ref.shape, f"{what}: shape {tuple(g.shape)} != {tuple(ref.shape)}"
    same = (g == ref) | (torch.isnan(g) & torch.isnan(ref))
    err = torch.where(same, torch.zeros_like(g), (g - ref).abs())
    err = torch.where(torch.isnan(err), torch.full_like(err, INF), err)
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound.clamp_min(1e-300))
    r = ratio.max().item() if ratio.numel() else 0.0
    op = what.split(" ")[0]
    _WORST[op] = max(_WORST.get(op, 0.0), r)
    if not r <= 1.0:
        i = int(ratio.reshape(-1).argmax())
        raise AssertionError(f"{what}: err/bound {r:.3g} at {list(torch.unravel_index(torch.tensor(i), g.shape))}: got "
                             f"{g.reshape(-1)[i].item()!r}, ref {ref.reshape(-1)[i].item()!r}, "
                             f"bound {bound.reshape(-1)[i].item():.3g}")


def _exact(got, ref, what):
    _close(got, ref, torch.zeros_like(ref), what)


def _nhwc_out(got, shape, what):
    assert tuple(got.shape) == tuple(shape), f"{what}: shape {tuple(got.shape)} != {tuple(shape)}"
    assert got.is_contiguous(memory_format=CL), f"{what}: result is not dense channels-last"


def _dense_guarded(t, dev, memory_format=torch.contiguous_format):
    """t with the strides of `memory_format`, at the start of an allocation whose 32 elements behind it are NaN."""
    strides = torch.empty(t.shape, device="meta").contiguous(memory_format=memory_format).stride()
    buf = torch.full((t.numel() + 32,), NAN, dtype=t.dtype, device=dev)
    v = torch.as_strided(buf, tuple(t.shape), strides, 0)
    v.copy_(t)
    return v


def _rows_slab(t, off, dev):
    """2-D t [rows, C] as columns [off, off + C) of a NaN-filled [rows, C + off + 8] slab (off 0: dense), at element
    offset 16 of a NaN-filled allocation with 32 NaN elements behind it."""
    rows, c = t.shape
    ld = c + off + 8 if off else c
    buf = torch.full((16 + rows * ld + 32,), NAN, dtype=t.dtype, device=dev)
    v = torch.as_strided(buf, (rows, c), (ld, 1), 16 + off)
    v.copy_(t)
    return v


LAYOUTS = {"dense": 0, "slice8": 8, "slice16": 16}


def _q(t, step):
    """bf16 values on a grid of `step`: pooling / eltwise MAX inputs with many exact ties."""
    return (torch.round(t / step) * step).to(BF16)


# ------------------------------------------------------------------------------------------------------------ pooling
def _out_size(n, k, s, p):
    """pooling_layer.cpp:72-87: ceil mode; with padding, a last window that starts in the padding is dropped."""
    o = -(-(n + 2 * p - k) // s) + 1
    if p > 0 and (o - 1) * s >= n + p:
        o -= 1
    return o


def _plane(x64, k, s, p, oh, ow, fill):
    """x placed at (p_h, p_w) in a plane that holds every window (a ceil-mode window may start past the image), and the
    (tap, rows, cols) slices of the windows' taps in row-major window order."""
    n, c, h, w = x64.shape
    eh, ew = max((oh - 1) * s[0] + k[0], p[0] + h), max((ow - 1) * s[1] + k[1], p[1] + w)
    plane = torch.full((n, c, eh, ew), fill, dtype=F64)
    plane[:, :, p[0]: p[0] + h, p[1]: p[1] + w] = x64
    taps = [(i * k[1] + j, slice(i, i + (oh - 1) * s[0] + 1, s[0]), slice(j, j + (ow - 1) * s[1] + 1, s[1]))
            for i in range(k[0]) for j in range(k[1])]
    return plane, taps


def _ave_inv(hw, ohw, k, s, p):
    """[OH, OW] 1 / pool_size with pool_size from the window clipped to H + pad, not to H (pooling_layer.cu:63-66);
    0 for an empty window (one that starts at or past H + pad)."""
    ext = []
    for n, o, kk, st, pp in zip(hw, ohw, k, s, p):
        start = torch.arange(o, dtype=F64) * st - pp
        ext.append(torch.clamp(start + kk, max=n + pp) - start)
    size = ext[0].view(-1, 1) * ext[1].view(1, -1)
    return torch.where(size > 0, 1.0 / size.clamp_min(1), torch.zeros(()))


def _pool_ref(x, dy, is_max, k, s, p):
    """(y, bound_y, dx, bound_dx).  MAX: pooling_layer.cu:12-47 (window clipped to the image, strict '>' in row-major
    order: the first maximum wins, maxval starts at -FLT_MAX, i.e. -inf in bf16) and :213-256 (dy goes to the recorded
    element).  AVE: pooling_layer.cu:50-78 and :259-293."""
    n, c, h, w = x.shape
    oh, ow = _out_size(h, k[0], s[0], p[0]), _out_size(w, k[1], s[1], p[1])
    dy64 = dy.double()
    crop = (slice(None), slice(None), slice(p[0], p[0] + h), slice(p[1], p[1] + w))
    if is_max:
        plane, taps = _plane(x.double(), k, s, p, oh, ow, -INF)
        y = torch.full((n, c, oh, ow), -INF, dtype=F64)
        arg = torch.full((n, c, oh, ow), -1, dtype=torch.long)
        for t, rs, cs in taps:
            v = plane[:, :, rs, cs]
            better = v > y
            y = torch.where(better, v, y)
            arg = torch.where(better, torch.full_like(arg, t), arg)
        g, m, a = (torch.zeros_like(plane) for _ in range(3))
        for t, rs, cs in taps:
            sel = arg == t
            g[:, :, rs, cs] += torch.where(sel, dy64, 0.0)
            m[:, :, rs, cs] += sel.double()
            a[:, :, rs, cs] += torch.where(sel, dy64.abs(), 0.0)
        dx, m, a = g[crop], m[crop], a[crop]
        return y, torch.zeros_like(y), dx, torch.where(m > 1, m * H * a, torch.zeros_like(a))
    inv = _ave_inv((h, w), (oh, ow), k, s, p)
    plane, taps = _plane(x.double(), k, s, p, oh, ow, 0.0)
    y = sum(plane[:, :, rs, cs] for _, rs, cs in taps) * inv
    mag = sum(plane[:, :, rs, cs].abs() for _, rs, cs in taps) * inv
    g, gm = torch.zeros_like(plane), torch.zeros_like(plane)
    for _, rs, cs in taps:
        g[:, :, rs, cs] += dy64 * inv
        gm[:, :, rs, cs] += dy64.abs() * inv
    nc = -(-k[0] // s[0]) * -(-k[1] // s[1])
    return (y, _bf16_bound(y, (k[0] * k[1] + 2) * U * mag), g[crop], _bf16_bound(g[crop], (nc + 2) * U * gm[crop]))


def _pool_kt(k):                          # pool.cu pool_fwd: compile-time square window 2 / 3, else generic
    return k[0] if k[0] == k[1] and k[0] in (2, 3) else 0


def _pool_nc(k, s):                       # pool.cu pool_bwd: windows per input pixel, unrolled up to 3, else generic
    nc = max(-(-k[0] // s[0]), -(-k[1] // s[1]))
    return nc if nc <= 3 else 0


# (N, C, H, W, kernel, stride, pad)
POOL = [
    ((2, 16, 13, 13, (3, 3), (2, 2), (0, 0)), "AlexNet 3x3/2: KT 3, NC 2"),
    ((2, 16, 12, 12, (2, 2), (2, 2), (0, 0)), "VGG 2x2/2: KT 2, NC 1"),
    ((1, 24, 9, 11, (3, 3), (1, 1), (1, 1)), "3x3/1 pad 1, batch 1: KT 3, NC 3"),
    ((2, 16, 10, 12, (3, 3), (2, 2), (1, 1)), "ceil mode: the last window runs past H + pad (divisor 2, not 1)"),
    ((2, 8, 7, 7, (7, 7), (1, 1), (0, 0)), "GoogLeNet 7x7/1: generic forward, NC 0"),
    ((2, 8, 10, 9, (5, 5), (1, 1), (4, 4)), "5x5/1 pad 4 = k - 1: generic forward, NC 0"),
    ((2, 16, 11, 8, (3, 2), (2, 1), (1, 1)), "rectangular 3x2, stride (2,1): generic forward, NC 2"),
    ((2, 8, 8, 7, (2, 2), (4, 3), (0, 0)), "k < s, pad 0: last row of windows starts at H (empty), KT 2, NC 1"),
    ((1, 8, 5, 5, (1, 1), (3, 3), (0, 0)), "1x1/3: the last windows start past the image, NC 1"),
    ((2, 8, 1, 9, (1, 3), (1, 2), (0, 1)), "H == 1, 1x3 / (1,2) pad (0,1)"),
    ((2, 8, 9, 1, (3, 3), (2, 2), (1, 1)), "W == 1, 3x3/2 pad 1: KT 3"),
    ((1, 8, 6, 6, (5, 5), (2, 2), (2, 2)), "5x5/2 pad 2: NC 3 with the generic forward"),
]
POOL_PARAMS = [pytest.param(c, id="x".join(map(str, c[:4])) + f"-k{c[4][0]}{c[4][1]}s{c[5][0]}{c[5][1]}p{c[6][0]}{c[6][1]}")
               for c, _ in POOL]


@pytest.mark.parametrize("case", POOL_PARAMS)
@pytest.mark.parametrize("op", ["max", "ave"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_pool_contract(k, case, op, layout):
    """pool_fwd / pool_bwd against Caffe's loops: ties, clipped and empty windows, pad = k - 1; x and dy pitched."""
    n, c, h, w, kern, stride, pad = case
    dev, off = _dev(k), LAYOUTS[layout]
    is_max = op == "max"
    oh, ow = _out_size(h, kern[0], stride[0], pad[0]), _out_size(w, kern[1], stride[1], pad[1])
    seed = sum(case[:4]) + 7 * kern[0] + kern[1]
    x = _q(_randn((n, c, h, w), seed, 2.0), 0.5)
    dy = _randn((n, c, oh, ow), seed + 1, dtype=BF16)
    y_ref, y_bound, dx_ref, dx_bound = _pool_ref(x, dy, is_max, kern, stride, pad)
    y, idx = k.pool_fwd(_in_slab(x, off, dev), is_max, list(kern), list(stride), list(pad), oh, ow, True)
    _nhwc_out(y, (n, c, oh, ow), "pool_fwd")
    if is_max:
        _exact(y, y_ref, f"pool_fwd max [{layout}]")
    else:
        _close(y, y_ref, y_bound, f"pool_fwd ave [{layout}]")
    dx = k.pool_bwd(_in_slab(dy, off, dev), idx, is_max, [h, w], list(kern), list(stride), list(pad))
    _nhwc_out(dx, (n, c, h, w), "pool_bwd")
    _close(dx, dx_ref, dx_bound, f"pool_bwd {op} [{layout}]")


# ------------------------------------------------------------------------------------------------------------ LRN across
def _chan_sum(t, lo, hi):
    """out[c] = Σ_{c' = c - lo}^{c + hi} t[c'], zero outside [0, C)."""
    c = t.shape[1]
    tp = F.pad(t, (0, 0, 0, 0, lo, hi))
    return sum(tp[:, i: i + c] for i in range(lo + hi + 1))


def _group_sum(t, widen):
    """out[c] = Σ t over the channels [8·⌊c/8⌋ - widen, 8·⌊c/8⌋ + 7 + widen] of c's thread (zero outside [0, C))."""
    s = _chan_sum(t, widen, widen + 7)
    return s[:, (torch.arange(t.shape[1]) // 8) * 8]


def _lrn_ref(x, dy, size, alpha, beta, relu):
    """lrn_layer.cu:10-53 (LRNFillScale: window [c - pre, c + post], scale = 1 + (α/n)·Σx²), :73-78 (y = x·scale^-β),
    :119-177 (LRNComputeDiff).  fuse_relu: the op applied to ReLU(x), its gradient masked by x > 0."""
    x64 = x.double()
    xr = x64.clamp_min(0) if relu else x64
    pre = (size - 1) // 2
    post = size - 1 - pre
    aon = alpha / size
    sq = xr * xr
    scale = 1 + aon * _chan_sum(sq, pre, post)
    p = scale ** -beta
    y = xr * p
    rel = (2 * size + 24) * U * (1 + beta * aon * _group_sum(sq, size - 1) + beta * scale.log2().abs()) + \
        2.0 ** -21 * (1 + beta)
    dy64 = dy.double()
    r = dy64 * xr * scale ** (-beta - 1)
    ratio = 2 * aon * beta
    dx = dy64 * p - ratio * xr * _chan_sum(r, post, pre)
    mag = dy64.abs() * p + ratio * xr.abs() * _group_sum(r.abs(), size - 1)
    rel_b = rel.amax(1, keepdim=True) + (2 * size + 32) * U
    if relu:
        keep = (x64 > 0).double()
        dx, mag = dx * keep, mag * keep
    return y, _bf16_bound(y, rel * y.abs()), dx, _bf16_bound(dx, rel_b * mag)


def _lrn_smem_pix(c, size, bwd):            # lrn.cu lrn_launch: pixels per CTA of the shared-memory kernel
    return max(1, min(64, (96 * 1024) // ((2 if bwd else 1) * (c + size - 1) * 4)))


# (N, C, H, W, local_size): α = 0.3·local_size (α/n = 0.3), β = 0.75, x ~ N(0, 2²)
LRN = [
    ((2, 8, 3, 5, 1), "PRE 0"),
    ((2, 8, 3, 5, 3), "PRE 1, C 8: no neighbour vectors"),
    ((2, 8, 4, 3, 5), "PRE 2, C 8"),
    ((2, 24, 3, 3, 5), "PRE 2 with both neighbour vectors (AlexNet's local_size)"),
    ((1, 8, 3, 5, 7), "PRE 3, batch 1"),
    ((2, 8, 2, 3, 9), "PRE 4, C 8"),
    ((2, 16, 3, 2, 9), "PRE 4, C 16"),
    ((2, 32, 3, 3, 11), "shared-memory kernel, local_size 11"),
    ((2, 392, 7, 5, 13), "shared-memory kernel, local_size 13: 61 / 30 pixels per CTA, 70 pixels (partial strips)"),
]
LRN_PARAMS = [pytest.param(c, id="x".join(map(str, c[:4])) + f"-n{c[4]}") for c, _ in LRN]


@pytest.mark.parametrize("case", LRN_PARAMS)
@pytest.mark.parametrize("relu", [False, True], ids=["plain", "fuse_relu"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_lrn_across_contract(k, case, relu, layout):
    """lrn_fwd / lrn_bwd on the register kernel (every PRE) and the shared-memory kernel, with and without fuse_relu."""
    n, c, h, w, size = case
    dev, off = _dev(k), LAYOUTS[layout]
    alpha, beta = 0.3 * size, 0.75
    seed = 100 + sum(case)
    x = _randn((n, c, h, w), seed, 2.0, dtype=BF16)
    dy = _randn((n, c, h, w), seed + 1, dtype=BF16)
    y_ref, y_bound, dx_ref, dx_bound = _lrn_ref(x, dy, size, alpha, beta, relu)
    xin = _in_slab(x, off, dev)
    y = k.lrn_fwd(xin, size, alpha, beta, relu)
    _nhwc_out(y, (n, c, h, w), "lrn_fwd")
    _close(y, y_ref, y_bound, f"lrn_fwd [{layout}]")
    dx = k.lrn_bwd(xin, _in_slab(dy, off, dev), size, alpha, beta, relu)
    _nhwc_out(dx, (n, c, h, w), "lrn_bwd")
    _close(dx, dx_ref, dx_bound, f"lrn_bwd [{layout}]")


# ------------------------------------------------------------------------------------------------------------ LRN within
def _spatial_sum(t, size):
    """out[h, w] = Σ over rows [h - pre, h + post] x cols [w - pre, w + post] inside the image."""
    pre = (size - 1) // 2
    post = size - 1 - pre
    hh, ww = t.shape[2:]
    tp = F.pad(t, (pre, post, pre, post))
    return sum(tp[:, :, i: i + hh, j: j + ww] for i in range(size) for j in range(size))


def _lrn_within_ref(x, dy, size, alpha, beta):
    """lrn_layer.cpp:20-69 composes x² -> AVE pool (size, pad pre, stride 1) -> (1 + α·s)^-β -> PROD; the pool's divisor
    is the window clipped to H + pre (pooling_layer.cu:50-78)."""
    x64 = x.double()
    hh, ww = x.shape[2:]
    pre = (size - 1) // 2
    ps = _ave_inv((hh, ww), (hh, ww), (size, size), (1, 1), (pre, pre))          # 1 / pool_size
    sq = x64 * x64
    ssum = _spatial_sum(sq, size)
    scale = 1 + alpha * ssum * ps
    p = scale ** -beta
    y = x64 * p
    kk = size * size
    rel = (kk + 8) * U * (1 + beta * alpha * ssum * ps + beta * scale.log2().abs()) + 2.0 ** -21 * (1 + beta)
    dy64 = dy.double()
    r = dy64 * y / scale * ps
    dx = dy64 * p - 2 * alpha * beta * x64 * _spatial_sum(r, size)
    mag = dy64.abs() * p + 2 * alpha * beta * x64.abs() * _spatial_sum(r.abs(), size)
    rel_b = rel.amax((1, 2, 3), keepdim=True) + (kk + 8) * U
    return y, _bf16_bound(y, rel * y.abs()), dx, _bf16_bound(dx, rel_b * mag)


# (N, C, H, W, local_size), α = 2, β = 0.75
LRN_WITHIN = [
    ((2, 16, 6, 9, 3), "3x3"),
    ((1, 8, 3, 4, 5), "5x5 on 3x4: windows clipped on both sides"),
    ((2, 8, 5, 2, 7), "7x7 on 5x2"),
    ((2, 8, 1, 8, 3), "H == 1"),
]


@pytest.mark.parametrize("case", [pytest.param(c, id="x".join(map(str, c))) for c, _ in LRN_WITHIN])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_lrn_within_contract(k, case, layout):
    n, c, h, w, size = case
    dev, off = _dev(k), LAYOUTS[layout]
    alpha, beta = 2.0, 0.75
    x = _randn((n, c, h, w), 200 + sum(case), dtype=BF16)
    dy = _randn((n, c, h, w), 201 + sum(case), dtype=BF16)
    y_ref, y_bound, dx_ref, dx_bound = _lrn_within_ref(x, dy, size, alpha, beta)
    xin = _in_slab(x, off, dev)
    y = k.lrn_within_fwd(xin, size, alpha, beta)
    _nhwc_out(y, (n, c, h, w), "lrn_within_fwd")
    _close(y, y_ref, y_bound, f"lrn_within_fwd [{layout}]")
    dx = k.lrn_within_bwd(xin, _in_slab(dy, off, dev), size, alpha, beta)
    _nhwc_out(dx, (n, c, h, w), "lrn_within_bwd")
    _close(dx, dx_ref, dx_bound, f"lrn_within_bwd [{layout}]")


# ------------------------------------------------------------------------------------------------------------ softmax
def _softmax_rel(x64, dim):
    c = x64.shape[dim]
    r = (4 + 3 * (x64 - x64.amax(dim, keepdim=True)).abs()) * U
    return r + r.amax(dim, keepdim=True) + (c + 4) * U


def _softmax_ref(x, yin, dy):
    """softmax_layer.cu:14-149 over the channel axis: y = exp(x - max) / Σ; dx = y·(dy - Σ dy·y) from the given y."""
    x64 = x.double()
    y = torch.softmax(x64, 1)
    yb, dy64 = yin.double(), dy.double()
    dx = yb * (dy64 - (yb * dy64).sum(1, keepdim=True))
    mag = yb.abs() * (dy64.abs() + (yb * dy64).abs().sum(1, keepdim=True))
    return y, _bf16_bound(y, _softmax_rel(x64, 1) * y), dx, _bf16_bound(dx, (x.shape[1] + 4) * U * mag)


SOFTMAX_C = [1, 7, 33, 1000, 1024, 1025, 4097]       # <= 1024: one warp per row (softmax_rows_kernel), else softmax_long


@pytest.mark.parametrize("c", SOFTMAX_C)
@pytest.mark.parametrize("dims", [2, 4])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_softmax_contract(k, c, dims, layout):
    dev, off = _dev(k), LAYOUTS[layout]
    shape = (5, c) if dims == 2 else (2, c, 3, 2)
    x = _randn(shape, 300 + c + dims, 3.0, dtype=BF16)
    dy = _randn(shape, 301 + c + dims, dtype=BF16)
    yin = torch.softmax(x.double(), 1).to(BF16)
    y_ref, y_bound, dx_ref, dx_bound = _softmax_ref(x, yin, dy)
    put = (lambda t: _rows_slab(t, off, dev)) if dims == 2 else (lambda t: _in_slab(t, off, dev))
    y = k.softmax_fwd(put(x))
    dx = k.softmax_bwd(put(yin), put(dy))
    for t in (y, dx):
        assert tuple(t.shape) == shape and (t.is_contiguous() if dims == 2 else t.is_contiguous(memory_format=CL))
    _close(y, y_ref, y_bound, f"softmax_fwd [{dims}-D {layout}]")
    _close(dx, dx_ref, dx_bound, f"softmax_bwd [{dims}-D {layout}]")


# (rows, C, dtype, row stride offset, labels out of range)
XENT = [
    ((1, 10, "bf16", 0, False), "rows 1, C < 256"),
    ((1, 300, "fp32", 0, False), "rows 1, C > 256"),
    ((7, 100, "bf16", 0, True), "labels C and -1 add 0"),
    ((7, 100, "fp32", 0, True), "labels C and -1 add 0, fp32"),
    ((5, 1000, "bf16", 24, False), "row stride C + 32"),
    ((4, 257, "fp32", 8, True), "row stride C + 16, fp32"),
    ((3, 4097, "fp32", 0, False), "C 4097"),
]


@pytest.mark.parametrize("case", [pytest.param(c, id=f"{c[0]}x{c[1]}-{c[2]}" + (f"-ld+{c[3] + 8}" if c[3] else "") +
                                               ("-oob" if c[4] else "")) for c, _ in XENT])
def test_softmax_xent_contract(k, case):
    """softmax_xent: prob, loss = mean over rows of -log(max(p[label], FLT_MIN)) (a label out of range adds 0), and
    dx = (p - 1[c = label])·grad_scale / rows (softmax_loss_layer.cpp:38-87)."""
    rows, c, dt, off, oob = case
    dev = _dev(k)
    dtype = BF16 if dt == "bf16" else torch.float32
    x = _randn((rows, c), 400 + rows + c, 3.0, dtype=dtype)
    lab = torch.randint(0, c, (rows,), generator=torch.Generator().manual_seed(c)).float()
    if oob:
        lab[2], lab[5 % rows] = float(c), -1.0
    gs = 0.75
    x64 = x.double()
    p = torch.softmax(x64, 1)
    li = lab.long()
    valid = (li >= 0) & (li < c)
    onehot = F.one_hot(torch.where(valid, li, 0), c).double() * valid.double().view(-1, 1)
    rel = _softmax_rel(x64, 1)
    dx_ref = (p - onehot) * gs / rows
    e_dx = (rel * p * gs / rows + 4 * U * dx_ref.abs())
    picked = p.gather(1, torch.where(valid, li, 0).view(-1, 1)).view(-1).clamp_min(1.17549435e-38)
    row_loss = torch.where(valid, -picked.log(), torch.zeros(()))
    loss_ref = row_loss.sum() / rows
    e_loss = (torch.where(valid, rel.gather(1, torch.where(valid, li, 0).view(-1, 1)).view(-1) + 2.0 ** -20,
                          torch.zeros(())).sum() / rows + (rows + 8) * U * loss_ref)
    xin = _rows_slab(x, off, dev)
    loss, dx, prob = k.softmax_xent(xin, lab.to(dev), gs, True, True)
    assert tuple(dx.shape) == (rows, c) and dx.dtype == dtype and dx.is_contiguous()
    _close(prob, p, rel * p + 4 * U * p, "softmax_xent prob")
    _close(dx, dx_ref, _bf16_bound(dx_ref, e_dx) if dtype == BF16 else e_dx + 4 * U * dx_ref.abs(), "softmax_xent dx")
    _close(loss.reshape(()), loss_ref.reshape(()), e_loss.reshape(()), "softmax_xent loss")


# ------------------------------------------------------------------------------------------------------------ MVN
def _mvn_ref(x, dy, inv_k, nv, ac):
    """mvn_layer.cu:15-135: mean, var = E[x²] - E[x]², y = (x - mean) / (sqrt(var) + 1e-10); backward
    dx = (dy - E[dy] - y·E[dy·y]) · inv (normalize_variance) or dy - E[dy], with the forward's inv = 1 / (std + eps)."""
    x64, dy64 = x.double(), dy.double()
    n, c = x.shape[:2]
    dims = (1, 2, 3) if ac else (2, 3)
    cnt = x[0].numel() if ac else x.shape[2] * x.shape[3]
    mean = x64.mean(dims, keepdim=True)
    ex2 = (x64 * x64).mean(dims, keepdim=True)
    var = (ex2 - mean * mean).clamp_min(0)
    std = var.sqrt()
    inv = 1 / (std + 1e-10) if nv else torch.ones_like(std)
    y = (x64 - mean) * inv
    eabs = x64.abs().mean(dims, keepdim=True)
    if nv:
        e_y = y.abs() * ((cnt + 4) * U * ex2 / var + 4 * U) + (cnt + 2) * U * eabs * inv
    else:
        e_y = (cnt + 2) * U * eabs + 2 * U * y.abs()
    e_inv = inv * ((cnt + 4) * U * ex2 / var + 4 * U) if nv else torch.zeros_like(inv)
    yb = y.to(BF16).double()
    ik = inv_k.double().view(n, c, 1, 1)
    gm = dy64.mean(dims, keepdim=True)
    if nv:
        dx = (dy64 - gm - yb * (dy64 * yb).mean(dims, keepdim=True)) * ik
        mag = ik * (dy64.abs() + dy64.abs().mean(dims, keepdim=True) + yb.abs() * (dy64 * yb).abs().mean(dims, keepdim=True))
    else:
        dx = dy64 - gm
        mag = dy64.abs() + dy64.abs().mean(dims, keepdim=True)
    return (y, _bf16_bound(y, e_y), mean.expand(n, c, 1, 1).reshape(n, c), ((cnt + 2) * U * eabs).expand(n, c, 1, 1).reshape(n, c),
            inv.expand(n, c, 1, 1).reshape(n, c), e_inv.expand(n, c, 1, 1).reshape(n, c), yb, dx,
            _bf16_bound(dx, (cnt + 4) * U * mag))


# (N, C, H, W, mean offset in σ)
MVN = [
    ((2, 24, 5, 7, 0.0), "C 24 (not a multiple of 64)"),
    ((1, 16, 3, 3, 32.0), "H·W 9 < 32, mean offset 32σ"),
    ((2, 264, 2, 3, 4.0), "C 264 > 256 (the finishing kernel's channel loop wraps)"),
    ((2, 72, 11, 13, 8.0), "C 72, H·W 143"),
]


@pytest.mark.parametrize("case", [pytest.param(c, id="x".join(map(str, c[:4])) + f"-off{int(c[4])}") for c, _ in MVN])
@pytest.mark.parametrize("nv", [True, False], ids=["nv", "mean"])
@pytest.mark.parametrize("ac", [False, True], ids=["plane", "across"])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_mvn_contract(k, case, nv, ac, layout):
    n, c, h, w, offset = case
    dev, off = _dev(k), LAYOUTS[layout]
    seed = 500 + sum(case[:4])
    shift = _randn((1, c, 1, 1), seed + 2, offset)
    x = (_randn((n, c, h, w), seed) + shift).to(BF16)
    dy = _randn((n, c, h, w), seed + 1, dtype=BF16)
    y, stats = k.mvn_fwd(_in_slab(x, off, dev), nv, ac)
    _nhwc_out(y, (n, c, h, w), "mvn_fwd")
    stats = stats.cpu()
    y_ref, y_bound, m_ref, m_bound, inv_ref, inv_bound, yb, dx_ref, dx_bound = _mvn_ref(x, dy, stats[:, :, 1], nv, ac)
    _close(y, y_ref, y_bound, f"mvn_fwd [{layout}]")
    _close(stats[:, :, 0], m_ref, m_bound, "mvn_fwd mean")
    _close(stats[:, :, 1], inv_ref, inv_bound, "mvn_fwd inv_std")
    dx = k.mvn_bwd(_in_slab(yb.to(BF16), off, dev), _in_slab(dy, off, dev), stats.to(dev), nv, ac)
    _nhwc_out(dx, (n, c, h, w), "mvn_bwd")
    _close(dx, dx_ref, dx_bound, f"mvn_bwd [{layout}]")


# ------------------------------------------------------------------------------------------------------------ unary
U_OPS = {"sigmoid": 0, "tanh": 1, "absval": 2, "bnll": 3, "power": 4, "threshold": 5}
POWER = [(1.0, 1.5, 0.5), (2.0, -0.75, 0.25), (3.0, 0.5, -0.25), (0.5, 0.5, 1.5), (0.0, 1.0, 0.0), (0.5, 0.0, 0.0)]
# numel % 8 = 0 (channels-last 4-D), 7 and 1 (contiguous): the scalar tail loop runs for the last two
UNARY_SHAPES = {"cl480": ((2, 16, 3, 5), CL), "t231": ((1, 3, 7, 11), torch.contiguous_format),
                "t657": ((1, 1, 9, 73), torch.contiguous_format)}


def _unary_ref(op, x64, s64, dy64, a, b, c):
    """(y, |Δy| bound before the bf16 rounding, dx, bound) — sigmoid_layer.cu, tanh_layer.cu, absval_layer.cu,
    bnll_layer.cu, power_layer.cu (dx = 0·dy when power·scale == 0, :42), threshold_layer.cu.  s is the saved tensor of
    the backward: y for sigmoid / tanh, x otherwise."""
    z = torch.zeros_like(x64)
    if op == "sigmoid":
        y = 1 / (1 + torch.exp(-x64))
        return y, (8 + 3 * x64.abs()) * U * y, dy64 * s64 * (1 - s64), 8 * U * (dy64 * s64).abs() * (1 + s64.abs())
    if op == "tanh":
        y = torch.tanh(x64)
        return y, 8 * U * y.abs(), dy64 * (1 - s64 * s64), 8 * U * dy64.abs() * (1 + s64 * s64)
    if op == "absval":
        return x64.abs(), z, dy64 * torch.sign(s64), z
    if op == "bnll":
        y = torch.where(x64 > 0, x64 + torch.log1p(torch.exp(-x64)), torch.log1p(torch.exp(x64)))
        e = torch.exp(s64.clamp_max(50))
        dx = dy64 * e / (e + 1)
        return y, (8 + 3 * x64.abs()) * U * (y.abs() + 1), dx, (8 + 3 * s64.clamp_max(50).abs()) * U * dx.abs()
    if op == "threshold":
        return (x64 > a).double(), z, z, z
    v = c + b * x64
    dv = 2 * U * (abs(c) + (b * x64).abs())                      # v = c + b·x in fp32 (possibly one fma)
    y = v.pow(a)
    ey = 4 * U * y.abs() + (a * v.pow(a - 1)).abs() * dv if a not in (0.0, 1.0) else 2 * U * y.abs() + (dv if a == 1 else 0)
    sv = c + b * s64
    if a * b == 0:
        return y, ey, dy64 * 0.0, z
    dx = dy64 * a * b * sv.pow(a - 1)
    edx = 8 * U * dx.abs() + (dy64 * a * b * (a - 1) * sv.pow(a - 2)).abs() * 2 * U * (abs(c) + (b * s64).abs()) \
        if a != 1 else 2 * U * dx.abs()
    return y, ey, dx, edx


UNARY_CASES = [(op, None) for op in U_OPS if op != "power"] + [("power", p) for p in POWER]


@pytest.mark.parametrize("case", [pytest.param(c, id=c[0] + ("" if c[1] is None else "-a{}b{}c{}".format(*c[1])))
                                  for c in UNARY_CASES])
@pytest.mark.parametrize("shape", list(UNARY_SHAPES))
def test_unary_contract(k, case, shape):
    """unary_fwd / unary_bwd on the 8-wide body and the scalar tail, NaN guard bands behind the last element; Power at
    a in {1, 2, 3, 0.5, 0} and at scale 0 (where power·scale == 0 the gradient is 0, not 0·inf)."""
    op, pw = case
    dims, fmt = UNARY_SHAPES[shape]
    dev = _dev(k)
    a, b, c = pw if pw is not None else ((0.25, 0.0, 0.0) if op == "threshold" else (0.0, 0.0, 0.0))
    seed = 600 + U_OPS[op] + sum(dims)
    x = _randn(dims, seed, 1.5, dtype=BF16)
    x.view(-1)[::5] = 0.0                                        # zeros: Power's base 0, AbsVal's sign 0
    x.view(-1)[1::11] = a if op == "threshold" else x.view(-1)[1::11]     # x == threshold gives 0
    dy = _randn(dims, seed + 1, dtype=BF16)
    x64 = x.double()
    y64 = _unary_ref(op, x64, x64, x64, a, b, c)[0]
    saved = y64.to(BF16) if op in ("sigmoid", "tanh") else x
    y_ref, e_y, dx_ref, e_dx = _unary_ref(op, x64, saved.double(), dy.double(), a, b, c)
    xin = _dense_guarded(x, dev, fmt)
    y = k.unary_fwd(xin, U_OPS[op], a, b, c)
    assert tuple(y.shape) == dims and y.stride() == xin.stride()
    exact = op in ("absval", "threshold")
    what = f"{op} fwd" + ("" if pw is None else " a={} b={} c={}".format(*pw))
    _close(y, y_ref, torch.zeros_like(y_ref) if exact else _bf16_bound(y_ref, e_y), what)
    dx = k.unary_bwd(_dense_guarded(saved, dev, fmt), _dense_guarded(dy, dev, fmt), U_OPS[op], a, b, c)
    assert tuple(dx.shape) == dims and dx.stride() == xin.stride()
    _close(dx, dx_ref, torch.zeros_like(dx_ref) if exact else _bf16_bound(dx_ref, e_dx), what.replace("fwd", "bwd"))


@pytest.mark.parametrize("slope", [0.0, 0.1])
def test_relu_dropout_contract(k, slope):
    """relu_fwd / relu_bwd (dense, guard bands behind the end), relu_bwd_nhwc (y and dy channel slices), dropout_apply
    (every element is 0 or x / (1 - ratio); guard bands behind the end)."""
    dev = _dev(k)
    x = _randn((2, 16, 3, 5), 700, dtype=BF16)
    x.view(-1)[::7] = 0.0
    dy = _randn((2, 16, 3, 5), 701, dtype=BF16)
    x64, dy64 = x.double(), dy.double()
    y_ref = torch.where(x64 > 0, x64, x64 * slope)
    dx_ref = torch.where(x64 > 0, dy64, dy64 * slope)
    bound = (lambda r: _bf16_bound(r, torch.zeros_like(r))) if slope else torch.zeros_like
    y = k.relu_fwd(_dense_guarded(x, dev, CL), slope)
    assert y.is_contiguous(memory_format=CL)
    _close(y, y_ref, bound(y_ref), "relu_fwd")
    dx = k.relu_bwd(_dense_guarded(x, dev, CL), _dense_guarded(dy, dev, CL), slope)
    _close(dx, dx_ref, bound(dx_ref), "relu_bwd")
    for off in (8, 16):
        dxn = k.relu_bwd_nhwc(_in_slab(x, off, dev), _in_slab(dy, 8 if off == 16 else 16, dev), slope)
        _nhwc_out(dxn, x.shape, "relu_bwd_nhwc")
        _close(dxn, dx_ref, bound(dx_ref), f"relu_bwd_nhwc [slice{off}]")
    got = k.dropout_apply(_dense_guarded(x, dev, CL), 0.5, 1234, None).cpu().double()
    assert got.is_contiguous(memory_format=CL)
    kept = got != 0
    assert torch.equal(got[kept], 2 * x64[kept]), "dropout_apply: a kept element is not x / (1 - ratio)"
    assert 0.3 < kept.double().mean().item() < 0.7


# ------------------------------------------------------------------------------------------------------------ eltwise
ELT = {"prod": 0, "sum": 1, "max": 2}


@pytest.mark.parametrize("op", list(ELT))
@pytest.mark.parametrize("nb", [2, 8])
def test_eltwise_contract(k, op, nb):
    """eltwise_fwd / eltwise_bwd (eltwise_layer.cu:11-90): PROD, SUM with coefficients, MAX with ties (the earlier bottom
    wins, exact); the backward for a subset of the bottoms."""
    dev = _dev(k)
    shape = (2, 16, 3, 5)
    xs = [(_q(_randn(shape, 800 + j, 2.0), 0.5) if op == "max" else _randn(shape, 800 + j, 1.2, dtype=BF16))
          for j in range(nb)]
    dy = _randn(shape, 899, dtype=BF16)
    coeffs = [0.5, -1.25, 2.0, 0.75, -0.5, 1.0, 3.0, -2.0][:nb] if op == "sum" else []
    need = [j % 3 != 1 for j in range(nb)]
    x64 = [x.double() for x in xs]
    dy64 = dy.double()
    if op == "prod":
        y_ref = math.prod(x64)
        e_y = (nb + 1) * U * y_ref.abs()
        dx_ref = [dy64 * math.prod(t for q, t in enumerate(x64) if q != j) for j in range(nb)]
        e_dx = [(nb + 1) * U * d.abs() for d in dx_ref]
    elif op == "sum":
        y_ref = sum(cf * t for cf, t in zip(coeffs, x64))
        e_y = (nb + 2) * U * sum(abs(cf) * t.abs() for cf, t in zip(coeffs, x64))
        dx_ref = [cf * dy64 for cf in coeffs]
        e_dx = [2 * U * d.abs() for d in dx_ref]
    else:
        y_ref, arg = torch.zeros(shape, dtype=F64) - INF, torch.zeros(shape, dtype=torch.long)
        for j, t in enumerate(x64):
            better = t > y_ref
            y_ref, arg = torch.where(better, t, y_ref), torch.where(better, j, arg)
        dx_ref = [torch.where(arg == j, dy64, 0.0) for j in range(nb)]
    ins = [_dense_guarded(x, dev, CL) for x in xs]
    y, mask = k.eltwise_fwd(ins, ELT[op], coeffs, True)
    assert tuple(y.shape) == shape and y.stride() == ins[0].stride()
    _close(y, y_ref, torch.zeros_like(y_ref) if op == "max" else _bf16_bound(y_ref, e_y), f"eltwise_fwd {op}")
    outs = k.eltwise_bwd(ins, _dense_guarded(dy, dev, CL), mask, ELT[op], coeffs, [int(v) for v in need])
    for j, (o, nd) in enumerate(zip(outs, need)):
        if not nd:
            assert o.numel() == 0
            continue
        assert o.stride() == ins[0].stride()
        _close(o, dx_ref[j], torch.zeros_like(dx_ref[j]) if op == "max" else _bf16_bound(dx_ref[j], e_dx[j]),
               f"eltwise_bwd {op} bottom {j}")


# ------------------------------------------------------------------------------------------------------------ stochastic
STO = [((2, 16, 9, 10), (3, 3), (2, 2)), ((1, 8, 8, 8), (2, 2), (2, 2)), ((2, 8, 7, 7), (3, 2), (2, 3))]


@pytest.mark.parametrize("case", [pytest.param(c, id="x".join(map(str, c[0])) + f"-k{c[1][0]}{c[1][1]}s{c[2][0]}{c[2][1]}")
                                  for c in STO])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_stochastic_pool_contract(k, case, layout):
    """Test phase: y = Σx² / Σx over the window clipped to the image (0 for an all-zero window) (pooling_layer.cu:121-150).
    Train phase: the picked value is the window element at the returned tap, and pool_bwd routes dy to exactly that
    element — checked on sets of outputs whose windows do not overlap, one set at a time."""
    (n, c, h, w), kern, stride = case
    dev, off = _dev(k), LAYOUTS[layout]
    oh, ow = _out_size(h, kern[0], stride[0], 0), _out_size(w, kern[1], stride[1], 0)
    x = _randn((n, c, h, w), 900 + h + w, dtype=BF16).clamp_min(0)     # post-ReLU: zeros and all-zero windows
    x[:, :, :2, :2] = 0
    xin = _in_slab(x, off, dev)
    plane, taps = _plane(x.double(), kern, stride, (0, 0), oh, ow, 0.0)
    s1 = sum(plane[:, :, rs, cs] for _, rs, cs in taps)
    s2 = sum(plane[:, :, rs, cs] ** 2 for _, rs, cs in taps)
    ref = torch.where(s1 > 0, s2 / s1.clamp_min(1e-300), torch.zeros(()))
    y, _ = k.stochastic_pool_fwd(xin, list(kern), list(stride), oh, ow, False, 0, None)
    _nhwc_out(y, (n, c, oh, ow), "stochastic_pool_fwd")
    _close(y, ref, _bf16_bound(ref, (2 * kern[0] * kern[1] + 4) * U * ref), f"stochastic_pool test [{layout}]")

    it = torch.tensor([3], dtype=torch.int64, device=dev)
    y, idx = k.stochastic_pool_fwd(xin, list(kern), list(stride), oh, ow, True, 77, it)
    _nhwc_out(y, (n, c, oh, ow), "stochastic_pool_fwd train")
    y64 = y.cpu().double()
    ph, pw = -(-kern[0] // stride[0]), -(-kern[1] // stride[1])        # outputs ph / pw apart have disjoint windows
    for a in range(ph):
        for b in range(pw):
            sel = torch.zeros(n, c, oh, ow, dtype=torch.bool)
            sel[:, :, a::ph, b::pw] = True
            dy = sel.to(BF16).contiguous(memory_format=CL)
            dx = k.pool_bwd(dy.to(dev), idx, True, [h, w], list(kern), list(stride), [0, 0]).cpu().double()
            assert set(dx.unique().tolist()) <= {0.0, 1.0} and dx.sum().item() == sel.sum().item(), \
                "stochastic pool: dy routed outside the picked elements"
            dplane, _ = _plane(dx, kern, stride, (0, 0), oh, ow, 0.0)
            hits = sum(dplane[:, :, rs, cs] for _, rs, cs in taps)
            picked = sum(dplane[:, :, rs, cs] * plane[:, :, rs, cs] for _, rs, cs in taps)
            assert torch.equal(hits[sel], torch.ones(int(sel.sum()), dtype=F64)), "stochastic pool: not one element per window"
            assert torch.equal(picked[sel], y64[sel]), "stochastic pool: picked value is not the element at the tap"


# ------------------------------------------------------------------------------------------------------------ engine
@pytest.fixture(params=[pytest.param("emu", id="emu"), pytest.param("gpu", id="gpu", marks=pytest.mark.gpu)])
def engine(request):
    """sm100 wrappers on the CPU emulation or on the GPU; yields the device."""
    from poseidon_b200.ops import sm100
    if request.param == "gpu":
        request.getfixturevalue("ext")
        yield "cuda"
        return
    prev = sm100.emulating()
    sm100.set_emulation(True)
    try:
        yield "cpu"
    finally:
        sm100.set_emulation(prev)


def _cl_slice(t, off, dev):
    """A channel slice of a zero-filled channels-last slab (what zero-copy concat hands to a consumer's backward)."""
    n, c, h, w = t.shape
    slab = torch.zeros((n, c + off + 8, h, w), dtype=t.dtype, device=dev).contiguous(memory_format=CL)
    v = slab[:, off: off + c]
    v.copy_(t)
    return v


def test_engine_max_pool_mask_input(engine):
    """sm100.max_pool(mask_input=True) with dy a channel slice: the producer's ReLU mask (relu_bwd_nhwc on the pooled
    output), then the gather."""
    from poseidon_b200.ops import sm100
    x = _q(_randn((2, 16, 13, 13), 1001, 2.0), 0.5).clamp_min(0)
    dy = _randn((2, 16, 6, 6), 1002, dtype=BF16)
    xs = x.to(engine).contiguous(memory_format=CL).requires_grad_(True)
    y = sm100.max_pool(xs, (3, 3), (2, 2), (0, 0), mask_input=True)
    y_ref, _, _, _ = _pool_ref(x, dy, True, (3, 3), (2, 2), (0, 0))
    _exact(y, y_ref, "engine max_pool")
    dym = torch.where(y_ref > 0, dy.double(), 0.0).to(BF16)
    _, _, dx_ref, dx_bound = _pool_ref(x, dym, True, (3, 3), (2, 2), (0, 0))
    y.backward(_cl_slice(dy, 8, engine))
    _close(xs.grad, dx_ref, dx_bound, "engine max_pool dx")


def test_engine_lrn_mask_input(engine):
    """sm100.lrn_across(mask_input=True) on post-ReLU x: LRN(x) forward, [x > 0]·∂LRN backward."""
    from poseidon_b200.ops import sm100
    x = _randn((2, 24, 5, 4), 1003, 2.0, dtype=BF16).clamp_min(0)
    dy = _randn((2, 24, 5, 4), 1004, dtype=BF16)
    xs = x.to(engine).contiguous(memory_format=CL).requires_grad_(True)
    y = sm100.lrn_across(xs, 5, 1.5, 0.75, mask_input=True)
    y_ref, y_bound, dx_ref, dx_bound = _lrn_ref(x, dy, 5, 1.5, 0.75, True)
    _close(y, y_ref, y_bound, "engine lrn")
    y.backward(_cl_slice(dy, 16, engine))
    _close(xs.grad, dx_ref, dx_bound, "engine lrn dx")


def test_engine_softmax_mvn_sliced(engine):
    """sm100.softmax and sm100.mvn on a channel slice of a slab, forward and backward."""
    from poseidon_b200.ops import sm100
    x = _randn((2, 40, 3, 4), 1005, 3.0, dtype=BF16)
    dy = _randn((2, 40, 3, 4), 1006, dtype=BF16)
    xs = _cl_slice(x, 8, engine).requires_grad_(True)
    y = sm100.softmax(xs)
    y.backward(_cl_slice(dy, 16, engine))
    y_ref, y_bound, dx_ref, dx_bound = _softmax_ref(x, y.detach().cpu(), dy)
    _close(y, y_ref, y_bound, "engine softmax")
    _close(xs.grad, dx_ref, dx_bound, "engine softmax dx")
    xs = _cl_slice(x, 16, engine).requires_grad_(True)
    y = sm100.mvn(xs, True, False)
    y.backward(_cl_slice(dy, 8, engine))
    x64 = x.double()
    mean, var = x64.mean((2, 3), keepdim=True), x64.var((2, 3), unbiased=False, keepdim=True)
    inv = 1 / (var.sqrt() + 1e-10)
    y_ref = (x64 - mean) * inv
    _close(y, y_ref, _bf16_bound(y_ref, 64 * U * (y_ref.abs() + mean.abs() * inv + 1)), "engine mvn")
    yb, dy64 = y.detach().cpu().double(), dy.double()
    dx_ref = (dy64 - dy64.mean((2, 3), keepdim=True) - yb * (dy64 * yb).mean((2, 3), keepdim=True)) * inv
    mag = inv * (dy64.abs() + dy64.abs().mean((2, 3), keepdim=True) + yb.abs() * (dy64 * yb).abs().mean((2, 3), keepdim=True))
    _close(xs.grad, dx_ref, _bf16_bound(dx_ref, 64 * U * mag), "engine mvn dx")


# ------------------------------------------------------------------------------------------------------------ coverage
def test_dispatch_coverage():
    """Every kernel instantiation is reached by some case: the host dispatch of pool.cu, lrn.cu, softmax_mvn.cu,
    softmax_xent.cu, neuron.cu and lrn_within.cu repeated over the case lists."""
    fwd, bwd = set(), set()
    generic = set()
    for (n, c, h, w, kern, stride, pad), _ in POOL:
        for mx in (True, False):
            fwd.add((mx, _pool_kt(kern)))
            bwd.add((mx, _pool_nc(kern, stride)))
        if _pool_kt(kern) == 0:
            generic.add("rect" if kern[0] != kern[1] else ("square5+" if kern[0] >= 5 else "square"))
    assert fwd == {(m, kt) for m in (True, False) for kt in (2, 3, 0)}, fwd
    assert bwd == {(m, nc) for m in (True, False) for nc in (1, 2, 3, 0)}, bwd
    assert {"rect", "square5+"} <= generic, generic
    geo = [case for case, _ in POOL]
    assert any(c[0] == 1 for c in geo) and any(c[2] == 1 for c in geo) and any(c[3] == 1 for c in geo)
    assert any(c[6][0] == c[4][0] - 1 and c[6][0] > 0 for c in geo), "pad = k - 1"
    assert any((_out_size(c[2], c[4][0], c[5][0], c[6][0]) - 1) * c[5][0] - c[6][0] + c[4][0] > c[2] + c[6][0]
               for c in geo), "a ceil-mode window past H + pad"
    assert any(c[6][0] == 0 and (_out_size(c[2], c[4][0], c[5][0], 0) - 1) * c[5][0] >= c[2] for c in geo), \
        "k < s, pad 0: a window that starts past the image"

    reg, smem = set(), set()
    for (n, c, h, w, size), _ in LRN:
        if size <= 9:
            reg.add(((size - 1) // 2, c))
        else:
            npix = n * h * w
            smem.add((size, all(_lrn_smem_pix(c, size, b) < 64 and npix % _lrn_smem_pix(c, size, b) for b in (0, 1))))
    assert {(p, 8) for p in range(5)} | {(4, 16)} <= reg, reg
    assert {s for s, _ in smem} >= {11, 13} and any(partial for _, partial in smem), smem

    assert {1, 7, 33, 1000, 1024, 1025, 4097} <= set(SOFTMAX_C)
    assert any(c <= 1024 for c in SOFTMAX_C) and any(c > 1024 for c in SOFTMAX_C)
    xent = [case for case, _ in XENT]
    assert {(dt, c > 256) for _, c, dt, _, _ in xent} == {(d, big) for d in ("bf16", "fp32") for big in (False, True)}
    assert any(r == 1 for r, *_ in xent) and any(o for *_, o in xent) and any(o > 0 for _, _, _, o, _ in xent)

    tails = {math.prod(d) % 8 for d, _ in UNARY_SHAPES.values()}
    assert tails == {0, 1, 7}, tails
    assert {op for op, _ in UNARY_CASES} == set(U_OPS)
    assert {a for a, _, _ in POWER} == {1.0, 2.0, 3.0, 0.5, 0.0} and any(b == 0 for _, b, _ in POWER)

    mvn = [case for case, _ in MVN]
    assert any(c[1] % 64 for c in mvn) and any(c[2] * c[3] < 32 for c in mvn) and any(c[1] > 256 for c in mvn)
    assert {s for (_, _, _, _, s), _ in LRN_WITHIN} >= {3, 5, 7}
    assert any(min(h, w) < s for (_, _, h, w, s), _ in LRN_WITHIN)
