"""Accumulation contracts, optimizer steps and bit-for-bit repeatability, against float64 references.

Every op that writes a caller-owned fp32 buffer is checked against a float64 reference computed on the CPU from the same
bf16 / fp32 inputs, with per-element bounds derived from fp32 rounding (u = 2^-24):

* GEMM-shaped ops: |got - ref| <= C_GEMM * K * u * (|alpha| * (|A| |B|^T) + |out0|); bf16 outputs add half a bf16 ulp.
* optimizer steps: |w - w64| <= 16 * u * (|w0| + S), where S is the magnitude of the step's terms evaluated without
  cancellation (S = |w0 - w64| when no term cancels); the same form for the history h.
* shadows, re-armed gradients and untouched guard bands: bit for bit.

Every buffer an op writes in place is an aligned slice (offset a multiple of 8 elements, padded rows where the op takes a
row pitch) of a larger allocation filled with a sentinel: a store past a ragged edge, which in the engine would land in the
next layer's gradient or weights, fails the guard check.

Ops that the CPU emulation implements on local tensors run twice: on ``EmulatedKernels`` (CPU, validates references and
bounds without a GPU) and on ``torch.ops.poseidon`` (GPU).  The sufficient-factor ops resolve raw device pointers and are
GPU-only."""
import functools
import math

import numpy as np
import pytest
import torch

BF16 = torch.bfloat16
CL = torch.channels_last
U = 2.0 ** -24
SENT = 7.0
# GEMM bound constant.  Largest err / bound measured with c = 4 on an H100 80GB HBM3 at 700 W: gemm_f32 0.0016 (shapes
# with N % 4 == 0), conv_wgrad 0.0033 (one-m-block cases), sfb_outer_f32 0.0069, gemm_bf16 0.28 (there the bf16 rounding
# dominates).  Raise c only with a measured figure.
C_GEMM = 4.0
C_UPD = 16.0


# ------------------------------------------------------------------------------------------------------------ fixtures
@pytest.fixture(params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def k(request):
    """The op surface under test: the CPU emulation or the sm_90a extension."""
    if request.param == "emu":
        from poseidon_b200.ops.emulate import EmulatedKernels
        return EmulatedKernels()
    return request.getfixturevalue("ext")


@pytest.fixture(params=[1, 0], ids=["pair", "single"])
def mode(k, request):
    k.set_pair_cta(request.param)
    try:
        yield request.param
    finally:
        k.set_pair_cta(1)



@pytest.fixture(params=[1, 0], ids=["pair", "single"])
def gpu_mode(ext, request):
    ext.set_pair_cta(request.param)
    try:
        yield request.param
    finally:
        ext.set_pair_cta(1)


# ------------------------------------------------------------------------------------------------------------ helpers
def _dev(k):
    return "cpu" if getattr(k, "emulated", False) else "cuda"


def _randn(shape, seed, scale=1.0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=torch.float64) * scale).to(dtype)


def _f32(x):
    return float(np.float32(x))


def _operand(t, dev):
    """A 2-D bf16 operand whose rows start 16-byte aligned (row pitch rounded up to 8 elements, as TMA requires)."""
    rows, cols = t.shape
    p = torch.zeros(rows, (cols + 7) // 8 * 8, dtype=BF16)
    p[:, :cols] = t
    return p.to(dev)[:, :cols]


def _guarded(shape, stride, dtype, dev, fill=None):
    """A strided view at element offset 8 of a sentinel-filled allocation (with room behind it); optionally filled."""
    span = 1 + sum((s - 1) * st for s, st in zip(shape, stride))
    buf = torch.full((8 + span + 24,), SENT, dtype=dtype, device=dev)
    v = torch.as_strided(buf, tuple(shape), tuple(stride), 8)
    if fill is not None:
        v.copy_(fill)
    return buf, v


def _bits(t):
    return t.view({4: torch.int32, 2: torch.int16}[t.element_size()])


def _assert_guard(buf, views, what):
    """Everything in `buf` outside the given views still holds the sentinel, bit for bit."""
    keep = torch.ones(buf.numel(), dtype=torch.bool, device=buf.device)
    idx = torch.arange(buf.numel(), device=buf.device)
    for v in views:
        keep[torch.as_strided(idx, v.shape, v.stride(), v.storage_offset()).reshape(-1)] = False
    sent = _bits(torch.full((1,), SENT, dtype=buf.dtype))[0].item()
    bad = (_bits(buf) != sent) & keep
    assert not bool(bad.any()), f"{what}: guard band overwritten at {bad.nonzero()[:8].view(-1).tolist()}"


def _within(got, ref, bound, what):
    """|got - ref| <= bound elementwise (ref, bound float64 on the CPU)."""
    err = (got.detach().cpu().double() - ref).abs()
    ratio = err / bound.clamp_min(1e-300)
    r = ratio.max().item() if ratio.numel() else 0.0
    if not r <= 1.0:
        i = int(ratio.reshape(-1).argmax())
        raise AssertionError(f"{what}: err/bound {r:.3g} at flat index {i}: got {got.detach().cpu().reshape(-1)[i].item()!r}, "
                             f"ref {ref.reshape(-1)[i].item()!r}, bound {bound.reshape(-1)[i].item():.3g}")


def _bf16_bound(ref, e):
    """fp32 error bound e, then one rounding to bf16 (half an ulp: 2^-8 relative) of a value within e (+ 4u) of ref."""
    e = e + 4 * U * ref.abs()
    return e + 2.0 ** -8 * (ref.abs() + e)


# ------------------------------------------------------------------------------------------------------------ gemm_f32
LAYOUTS = [(False, False), (False, True), (True, True)]


@pytest.mark.parametrize("M,N,K", [(200, 328, 520), (130, 96, 1000), (200, 330, 264)])
@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS, ids=["KxK", "KxMN", "MNxMN"])
@pytest.mark.parametrize("split_k", [1, 2, 3, 7])
@pytest.mark.parametrize("alpha", [1.0, -0.5])
@pytest.mark.parametrize("accumulate", [False, True], ids=["store", "accumulate"])
def test_gemm_f32_contract(k, mode, M, N, K, a_mn, b_mn, split_k, alpha, accumulate):
    """out = (accumulate ? out0 : 0) + alpha * A·Bᵀ for every split_k, into a pre-filled out with row pitch N + 8.
    N = 330 (not a multiple of 4) keeps the plain store off the bulk-store epilogue: the per-lane walk writes the ragged
    right edge next to the guard band."""
    dev = _dev(k)
    A, B = _randn((M, K), 1, dtype=BF16), _randn((N, K), 2, K ** -0.5, dtype=BF16)
    out0 = _randn((M, N), 3)
    a = _operand(A.t() if a_mn else A, dev)
    b = _operand(B.t() if b_mn else B, dev)
    buf, out = _guarded((M, N), (N + 8, 1), torch.float32, dev, out0)
    k.gemm_f32(a, a_mn, b, b_mn, out, alpha, accumulate, split_k, 0)
    A64, B64, o64 = A.double(), B.double(), out0.double()
    ref = alpha * (A64 @ B64.t()) + (o64 if accumulate else 0.0)
    bound = C_GEMM * K * U * (abs(alpha) * (A64.abs() @ B64.abs().t()) + (o64.abs() if accumulate else 0.0))
    _within(out, ref, bound, "gemm_f32")
    _assert_guard(buf, [out], "gemm_f32 out")


# ------------------------------------------------------------------------------------------------------------ gemm_bf16
@pytest.mark.parametrize("M", [32, 200])
@pytest.mark.parametrize("N,ldc", [(1000, 1000), (1002, 1008), (1000, 1002)], ids=["vector", "scalar_n", "scalar_ldc"])
@pytest.mark.parametrize("slope", [0.0, 0.1])
@pytest.mark.parametrize("masked", [False, True], ids=["plain", "mask"])
def test_gemm_bf16_splitk_finish(k, M, N, ldc, slope, masked):
    """Small-M bf16 GEMM (bn = 0, K = 4096): the host splits K over the idle SMs and finishes with splitk_finish_kernel —
    its vector form (N, ldc multiples of 4) and its scalar form — with bias, leaky ReLU and a mask of row pitch ldc."""
    dev = _dev(k)
    K = 4096
    A, B = _randn((M, K), 4, dtype=BF16), _randn((N, K), 5, K ** -0.5, dtype=BF16)
    bias = _randn((N,), 6, 0.5)
    mfull = _randn((M, ldc), 7, dtype=BF16)
    mask = mfull.to(dev)[:, :N] if masked else None
    buf, out = _guarded((M, N), (ldc, 1), BF16, dev)
    k.gemm_bf16(_operand(A, dev), False, _operand(B, dev), False, bias.to(dev), True, slope, mask, out, 0)
    A64, B64 = A.double(), B.double()
    v = A64 @ B64.t() + bias.double()
    ref = torch.where(v > 0, v, v * slope)
    if masked:
        ref = torch.where(mfull[:, :N].double() > 0, ref, ref * slope)
    e = C_GEMM * K * U * (A64.abs() @ B64.abs().t() + bias.double().abs())
    _within(out, ref, _bf16_bound(ref, e), "gemm_bf16 split-K finish")
    _assert_guard(buf, [out], "gemm_bf16 out (padding columns)")


# ------------------------------------------------------------------------------------------------------------ conv_wgrad
# conv_wgrad schedules (set_conv_mcast, set_conv_pair, set_conv_im2col, set_conv_cluster).  The weight gradient's M
# dimension is Cout_g: with one m-block (Cout_g <= 128) every im2col schedule launches the single-CTA kernel, so those cases
# run under the default only.  With two or more m-blocks on the im2col path, "mcast" clusters 2 (3 when the m-blocks divide
# by 3 and BN >= 192) CTAs along Cout that share the im2col tile by multicast; "pair" takes CTA pairs when the m-block count
# is even and BN is 128 or 256; "single" is one CTA per tile.  "gather" builds the im2col operand with the cp.async gather
# producer instead of TMA; "cluster2" / "cluster4" do so in clusters of 2 / 4 CTAs along the K columns that share the dY
# tile by multicast.  A channel-padded reduction needs the im2col path, so its cases skip these three.
SCHED = {"mcast": (2, 1, 1, 1), "pair": (1, 1, 1, 1), "single": (1, 0, 1, 1),          # (mcast, pair, im2col, cluster)
         "gather": (1, 1, 0, 1), "cluster2": (1, 1, 1, 2), "cluster4": (1, 1, 1, 4)}
ALL = ("mcast", "pair", "single")
GATHER = ("gather", "cluster2", "cluster4")
CONV_W = [
    # (N, Cin, H, W, Cout, k, stride, pad, group, cgk), schedules whose kernels differ
    ((2, 40, 9, 9, 72, 3, 1, 1, 1, 0), ("pair",)),        # gather (C_g 40), N·OH·OW = 162: one split, one atomic add each
    ((2, 64, 14, 14, 64, 3, 1, 1, 1, 0), ("pair",)),      # im2col, 392 pixels: one split
    ((2, 64, 28, 28, 64, 3, 2, 1, 1, 0), ("pair",)),      # strided im2col, 392 pixels: one split
    ((2, 256, 14, 14, 128, 3, 1, 1, 2, 0), ("pair",)),    # grouped im2col (C_g 128), one split per group
    ((2, 96, 14, 14, 64, 3, 1, 1, 1, 128), ("pair",)),    # channel-padded reduction (C_g 96 -> 128 k-columns per tap)
    ((4, 64, 28, 28, 128, 3, 1, 1, 1, 0), ("pair",)),     # im2col, 3136 pixels: per-split workspace + ordered reduce
    ((4, 96, 27, 27, 256, 5, 1, 2, 2, 0), ("pair",)),     # grouped gather (C_g 48), 2916 pixels: workspace
    ((2, 96, 28, 28, 128, 3, 1, 1, 1, 128), ("pair",)),   # channel-padded reduction, 1568 pixels: workspace
    ((2, 128, 14, 14, 256, 3, 1, 1, 1, 0), ALL + GATHER), # 2 m-blocks, BN 256, one split: cluster of 2 / pair / single
    ((2, 64, 14, 14, 256, 3, 1, 1, 1, 0), ("mcast", "single") + GATHER),   # 2 m-blocks, BN 192 (no pairs), one split
    ((2, 64, 14, 14, 384, 3, 1, 1, 1, 0), ("mcast", "single") + GATHER),   # 3 m-blocks, BN 192: cluster of 3, one split
    ((4, 128, 28, 28, 256, 3, 1, 1, 1, 0), ALL + GATHER), # 2 m-blocks, 3136 pixels: workspace under every schedule
    ((2, 256, 28, 28, 512, 3, 1, 1, 2, 0), ALL + GATHER), # grouped, Cout_g 256, 1568 pixels: workspace per group
    ((2, 96, 28, 28, 256, 3, 1, 1, 1, 128), ALL),         # channel-padded, 2 m-blocks, workspace
    # rectangular 3x5, stride (2,1), pad (1,2): 2 m-blocks, on the im2col and the gather paths
    ((2, 64, 13, 21, 192, (3, 5), (2, 1), (1, 2), 1, 0), ("pair", "single") + GATHER),
]
CONV_W_PARAMS = [pytest.param(c, sc, id="x".join(map(str, c)) + "-" + sc) for c, scheds in CONV_W for sc in scheds]


def _hw(v):
    """(h, w) of a kernel / stride / pad given as one int or a pair."""
    return tuple(v) if isinstance(v, tuple) else (v, v)


@functools.lru_cache(maxsize=None)
def _conv_case(case):
    n, cin, h, w, cout, kk, stride, pad, group, cgk = case
    (r, s), (sh, sw), (ph, pw) = _hw(kk), _hw(stride), _hw(pad)
    cg = cin // group
    x = _randn((n, cin, h, w), 11, dtype=BF16).contiguous(memory_format=CL)
    oh, ow = (h + 2 * ph - r) // sh + 1, (w + 2 * pw - s) // sw + 1
    dy = _randn((n, cout, oh, ow), 12, dtype=BF16).contiguous(memory_format=CL)

    def wg(a, b):
        g = torch.nn.grad.conv2d_weight(a, (cout, cg, r, s), b, (sh, sw), (ph, pw), 1, group)
        return g.permute(0, 2, 3, 1).reshape(cout, r * s * cg)
    ref = wg(x.double(), dy.double())
    mag = wg(x.double().abs(), dy.double().abs())
    return x, dy, ref, mag, n * oh * ow


@pytest.mark.parametrize("case,sched", CONV_W_PARAMS)
@pytest.mark.parametrize("alpha", [1.0, 0.25])
def test_conv_wgrad_accumulates(k, case, sched, alpha):
    """conv_wgrad adds alpha·dW onto a pre-filled, guard-banded gradient sink (a layer sharing its weight with another
    relies on that) — through one split's atomics and through the workspace + ordered reduce, under the single-CTA,
    CTA-pair, multicast-cluster, gather and gather-cluster schedules."""
    dev = _dev(k)
    mc, pair, im2col, cluster = SCHED[sched]
    n, cin, h, w, cout, kk, stride, pad, group, cgk = case
    x, dy, ref, mag, red = _conv_case(case)
    kernel = _hw(kk)
    kw = kernel[0] * kernel[1] * (cin // group)
    dw0 = _randn((cout, kw), 13, 10.0)
    buf, dw = _guarded((cout, kw), (kw, 1), torch.float32, dev, dw0)
    try:
        k.set_conv_mcast(mc)
        k.set_conv_pair(pair)
        k.set_conv_im2col(im2col)
        k.set_conv_cluster(cluster)
        k.conv_wgrad(x.to(dev), dy.to(dev), dw, list(kernel), list(_hw(stride)), list(_hw(pad)), group, 0, alpha, cgk)
    finally:
        k.set_conv_mcast(1)
        k.set_conv_pair(1)
        k.set_conv_im2col(1)
        k.set_conv_cluster(1)
    want = dw0.double() + alpha * ref
    bound = C_GEMM * red * U * (abs(alpha) * mag + dw0.double().abs())
    _within(dw, want, bound, "conv_wgrad")
    _assert_guard(buf, [dw], "conv_wgrad dw")


# ------------------------------------------------------------------------------------------------------------ colsum
@functools.lru_cache(maxsize=4)
def _int_slab(rows, ld):
    g = torch.Generator().manual_seed(rows * 7 + ld)
    return torch.randint(-8, 9, (rows, ld), generator=g, dtype=torch.int16).to(BF16)


COLSUM = [(r, c) for r in (1, 31, 33, 5000) for c in (8, 96, 1000)] + [(256 * 55 * 55, 96)]


@pytest.mark.parametrize("rows,C", COLSUM, ids=lambda v: str(v))
@pytest.mark.parametrize("alpha", [1.0, 0.5])
@pytest.mark.parametrize("accumulate", [False, True], ids=["store", "accumulate"])
def test_colsum(k, rows, C, alpha, accumulate):
    """Bias gradient: out (+)= alpha · Σ_rows dy, dy a channel slice (offset 8, pitch C + 24) of a wider NHWC slab.
    Integer-valued dy makes every partial sum exact in fp32, so the only rounding is the final add onto out0 and a row
    counted twice or dropped fails at any row count (the last case is AlexNet conv1 at batch 256)."""
    dev = _dev(k)
    ld = C + 24
    slab = _int_slab(rows, ld)
    dy = slab.to(dev)[:, 8: 8 + C]
    out0 = _randn((C,), 14, 100.0)
    buf, out = _guarded((C,), (1,), torch.float32, dev, out0)
    k.colsum(dy, rows, C, ld, out, alpha, accumulate)
    s = slab[:, 8: 8 + C].sum(0, dtype=torch.float64) * alpha
    ref = s + (out0.double() if accumulate else 0.0)
    _within(out, ref, U * ref.abs(), "colsum")
    _assert_guard(buf, [out], "colsum out")


# ------------------------------------------------------------------------------------------------------------ optimizer
def _step64(w, g, h, lr, mom, decay, rule, l1, delta, gscale, gabs=None):
    """One optimizer step in float64 -> (w1, h1, S_w, S_h): S_* is the step's magnitude evaluated on absolute values."""
    gg = g * gscale
    G = (g.abs() if gabs is None else gabs) * gscale
    if decay != 0:
        d = torch.sign(w) if l1 else w
        gg = gg + decay * d
        G = G + decay * d.abs()
    if rule in (0, 1):
        h1 = lr * gg + mom * h
        Sh = lr * G + mom * h.abs()
        if rule == 0:
            step, Sw = h1, Sh
        else:
            step = (1 + mom) * h1 - mom * h
            Sw = (1 + mom) * Sh + mom * h.abs()
    else:
        h1 = h + gg * gg
        Sh = h.abs() + G * G
        den = h1.sqrt() + delta
        step = lr * gg / den
        Sw = lr * G / den
    return w - step, h1, Sw, Sh


def _hyper(rule, decay_kind):
    lr, mom = _f32(0.05), (_f32(0.9) if rule != 2 else 0.0)
    decay = {"none": 0.0, "l2": _f32(0.05), "l1": _f32(0.05)}[decay_kind]
    return lr, mom, decay, decay_kind == "l1", _f32(1e-8), _f32(0.37)


def _w_init(n, seed):
    w = _randn((n,), seed)
    w[::7] = 0.0                                  # exact zeros: sign(0) = 0 under L1 decay
    return w


def _h_init(n, seed, rule):
    return _randn((n,), seed).abs() * 0.01 if rule == 2 else _randn((n,), seed, 0.01)


def _check_step(w, h, w0, g0, h0, hp, rule, lr_eff, what, gabs=None, extra_w=0.0, extra_h=0.0):
    lr, mom, decay, l1, delta, gscale = hp
    w64, h64, Sw, Sh = _step64(w0.double(), g0.double(), h0.double(), lr_eff, mom, decay, rule, l1, delta, gscale, gabs)
    _within(w, w64, C_UPD * U * (w0.double().abs() + Sw) + extra_w, f"{what} w")
    _within(h, h64, C_UPD * U * (h0.double().abs() + Sh) + extra_h, f"{what} h")
    return w64, Sw


def _run_update(k, shape, stride, h_stride, wb_shape, shadow_of, rule, decay_kind, use_lr_dev, rearm, shadow, seed, steps=3):
    dev = _dev(k)
    n = math.prod(shape)
    hp = _hyper(rule, decay_kind)
    lr, mom, decay, l1, delta, gscale = hp
    lr_dev = torch.tensor([0.7], device=dev) if use_lr_dev else None
    lr_eff = lr * _f32(0.7) if use_lr_dev else lr          # the device scalar holds fp32(0.7)
    wbuf, w = _guarded(shape, stride, torch.float32, dev)
    gbuf, g = _guarded(shape, stride, torch.float32, dev)
    hbuf, h = _guarded(shape, h_stride, torch.float32, dev)
    w.copy_(_w_init(n, seed).reshape(shape))
    h.copy_(_h_init(n, seed + 1, rule).reshape(shape))
    wbb = wb = None
    if shadow:
        wbb, wb = _guarded(wb_shape, torch.empty(wb_shape).stride(), BF16, dev)
    for step in range(steps):
        g_in = _randn(shape, seed + 10 + step).to(dev)
        g.copy_(g_in)
        w0, h0 = w.detach().cpu().clone(), h.detach().cpu().clone()
        k.fused_update(w, g, h, wb, lr, mom, decay, rule, l1, delta, gscale, lr_dev, rearm)
        _check_step(w, h, w0, g_in.cpu(), h0, hp, rule, lr_eff, "fused_update")
        if rearm:
            assert torch.equal(g, torch.zeros_like(g)), "re-armed gradient must be all zeros"
        else:
            assert torch.equal(g, g_in), "gradient must be left untouched without re-arm"
        if shadow:
            assert torch.equal(wb, shadow_of(w).to(BF16)), "bf16 shadow must equal the master in storage order"
    _assert_guard(wbuf, [w], "fused_update w")
    _assert_guard(gbuf, [g], "fused_update g")
    _assert_guard(hbuf, [h], "fused_update h")
    if shadow:
        _assert_guard(wbb, [wb], "fused_update wb")


UPD_FLAGS = [(False, False, False), (True, True, True), (True, False, True), (False, True, False)]


@pytest.mark.parametrize("n", [1, 3, 4, 5, 1023, 8195, 3 * 2 ** 20 + 3])
@pytest.mark.parametrize("rule", [0, 1, 2])
@pytest.mark.parametrize("decay_kind", ["none", "l2", "l1"])
@pytest.mark.parametrize("use_lr_dev,rearm,shadow", UPD_FLAGS, ids=["plain", "lrdev-rearm-wb", "lrdev-wb", "rearm"])
def test_fused_update(k, n, rule, decay_kind, use_lr_dev, rearm, shadow):
    """Three consecutive steps (the history carries over) on flat tensors: n % 4 tails, one element, and one tensor larger
    than one pass of the capped grid."""
    _run_update(k, (n,), (1,), (1,), (n,), lambda w: w, rule, decay_kind, use_lr_dev, rearm, shadow, seed=n + rule)


@pytest.mark.parametrize("rule", [0, 1, 2])
@pytest.mark.parametrize("layout", ["nhwc3x3", "1x1_odd_strides"])
def test_fused_update_conv_layouts(k, rule, layout):
    """Conv weights in channels-last form: the shadow [Cout, R·S·Cin] is the master in storage order, bit for bit.
    The 1x1 case gives its size-1 dimensions odd (and, for H, different) strides."""
    if layout == "nhwc3x3":
        co, ci, r = 64, 40, 3
        stride = (r * r * ci, 1, r * ci, ci)
        h_stride = stride
    else:
        co, ci, r = 48, 40, 1
        stride, h_stride = (ci, 1, 7, 3), (ci, 1, 5, 1)
    _run_update(k, (co, ci, r, r), stride, h_stride, (co, r * r * ci),
                lambda w: w.permute(0, 2, 3, 1).reshape(w.shape[0], -1), rule, "l1", True, True, True, seed=rule + 50)


MULTI_SIZES = [1, 3, 4, 8192, 8193, 3 * 8192 + 2, 5, 1000, 7, 64]


@pytest.mark.parametrize("count", [1, 48, 49, 100])
@pytest.mark.parametrize("rule", [0, 1, 2])
def test_fused_update_multi(k, count, rule):
    """Many tensors per launch (48 per launch, so 49 and 100 take several), carved from one arena with 8-element sentinel
    gaps; each tensor has its own lr, decay, re-arm flag and shadow, and is checked against its own reference."""
    dev = _dev(k)
    sizes = [MULTI_SIZES[(i + 5) % len(MULTI_SIZES)] for i in range(count)]
    offs, o = [], 8
    for s in sizes:
        offs.append(o)
        o += (s + 7) // 8 * 8 + 8
    total = o + 16
    bufs = {t: torch.full((total,), SENT, dtype=torch.float32, device=dev) for t in "wgh"}
    wbbuf = torch.full((total,), SENT, dtype=BF16, device=dev)
    ws = [bufs["w"][o: o + s] for o, s in zip(offs, sizes)]
    gs = [bufs["g"][o: o + s] for o, s in zip(offs, sizes)]
    hs = [bufs["h"][o: o + s] for o, s in zip(offs, sizes)]
    has_wb = [i % 3 != 0 for i in range(count)]
    wbs = [wbbuf[o: o + s] if hw else torch.empty(0, dtype=BF16, device=dev) for o, s, hw in zip(offs, sizes, has_wb)]
    lrs = [_f32(0.01 * (1 + i / 7)) for i in range(count)]
    decays = [_f32(0.02 * (i % 4)) for i in range(count)]
    rearms = [i % 2 for i in range(count)]
    l1 = rule == 1
    mom = _f32(0.9) if rule != 2 else 0.0
    delta, gscale = _f32(1e-8), _f32(0.37)
    lr_dev = torch.tensor([0.7], device=dev) if rule != 0 else None
    for i, (w, h, s) in enumerate(zip(ws, hs, sizes)):
        w.copy_(_w_init(s, 100 + i))
        h.copy_(_h_init(s, 200 + i, rule))
    for step in range(2):
        g_in = [_randn((s,), 300 + 17 * step + i) for i, s in enumerate(sizes)]
        for g, gi in zip(gs, g_in):
            g.copy_(gi)
        w0s = [w.cpu().clone() for w in ws]
        h0s = [h.cpu().clone() for h in hs]
        k.fused_update_multi(ws, gs, hs, wbs, lrs, decays, rearms, mom, rule, l1, delta, gscale, lr_dev)
        for i in range(count):
            lr_eff = lrs[i] * (_f32(0.7) if lr_dev is not None else 1.0)
            hp = (lrs[i], mom, decays[i], l1, delta, gscale)
            _check_step(ws[i], hs[i], w0s[i], g_in[i], h0s[i], hp, rule, lr_eff, f"fused_update_multi[{i}]")
            if rearms[i]:
                assert torch.equal(gs[i], torch.zeros_like(gs[i])), f"tensor {i}: gradient not re-armed"
            else:
                assert torch.equal(gs[i].cpu(), g_in[i]), f"tensor {i}: gradient changed without re-arm"
            if has_wb[i]:
                assert torch.equal(wbs[i], ws[i].to(BF16)), f"tensor {i}: shadow differs from master"
    for t, views in (("w", ws), ("g", gs), ("h", hs)):
        _assert_guard(bufs[t], views, f"fused_update_multi {t}")
    _assert_guard(wbbuf, [v for v, hw in zip(wbs, has_wb) if hw], "fused_update_multi wb")


# ------------------------------------------------------------------------------------------------------------ sfb (GPU)
@functools.lru_cache(maxsize=8)
def _sfb_case(P, N, K, Mb):
    us = [_randn((Mb, N), 30 + i, dtype=BF16) for i in range(P)]
    vs = [_randn((Mb, K), 40 + i, dtype=BF16) for i in range(P)]
    g64 = sum(u.double().t() @ v.double() for u, v in zip(us, vs))
    a64 = sum(u.double().abs().t() @ v.double().abs() for u, v in zip(us, vs))
    return us, vs, g64, a64


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 3])
@pytest.mark.parametrize("N", [200, 328])
@pytest.mark.parametrize("K", [520, 1000])
@pytest.mark.parametrize("rule", [0, 1, 2])
def test_sfb_outer_sgd_and_two_pass(ext, gpu_mode, P, N, K, rule):
    """The optimizer step inside the outer-product epilogue (alpha = 1/Mb, L1 decay, device lr, bf16 shadow, guard-banded
    W / H / Wb) at ragged N and K, against float64; and the two-pass form (sfb_outer_f32, then fused_update) against both."""
    Mb = 160
    alpha = 1.0 / Mb
    us, vs, g64, a64 = _sfb_case(P, N, K, Mb)
    ud = [u.cuda() for u in us]
    vd = [v.cuda() for v in vs]
    lr, mom, decay, l1, delta, _ = _hyper(rule, "l1")
    hp = (lr, mom, decay, l1, delta, 1.0)
    lr_dev = torch.tensor([0.7], device="cuda")
    lr_eff = lr * _f32(0.7)
    w0 = _w_init(N * K, 60).reshape(N, K)
    h0 = _h_init(N * K, 61, rule).reshape(N, K)
    sets = []
    for _ in range(2):
        wbuf, w = _guarded((N, K), (K, 1), torch.float32, "cuda", w0)
        hbuf, h = _guarded((N, K), (K, 1), torch.float32, "cuda", h0)
        bbuf, wb = _guarded((N, K), (K, 1), BF16, "cuda")
        sets.append((wbuf, w, hbuf, h, bbuf, wb))
    ptr = lambda ts: [t.data_ptr() for t in ts]       # noqa: E731
    (wbuf, w, hbuf, h, bbuf, wb), (wbuf2, w2, hbuf2, h2, bbuf2, wb2) = sets
    ext.sfb_outer_sgd(ptr(ud), ptr(vd), Mb, N, K, w, h, wb, alpha, lr, mom, decay, rule, l1, delta, None, 0, 0, 0, 0,
                      lr_dev, None)
    gbuf, g = _guarded((N, K), (K, 1), torch.float32, "cuda")
    ext.sfb_outer_f32(ptr(ud), ptr(vd), Mb, N, K, g, alpha, None, 0, 0, 0, 0, None)
    gref = alpha * g64
    eg = C_GEMM * Mb * U * alpha * a64
    _within(g, gref, eg, "sfb_outer_f32")
    _assert_guard(gbuf, [g], "sfb_outer_f32 out")
    ext.fused_update(w2, g, h2, wb2, lr, mom, decay, rule, l1, delta, 1.0, lr_dev, False)
    # the gradient itself carries the GEMM error eg: it moves the step by at most L·eg
    w64, h64, Sw, Sh = _step64(w0.double(), gref, h0.double(), lr_eff, mom, decay, rule, l1, delta, 1.0, alpha * a64)
    if rule == 0:
        lw, lh = lr_eff, lr_eff
    elif rule == 1:
        lw, lh = (1 + mom) * lr_eff, lr_eff
    else:
        lw, lh = 2 * lr_eff / (h64.sqrt() + delta), 2 * gref.abs() + eg
    for what, ww, hh in (("sfb_outer_sgd", w, h), ("sfb two-pass", w2, h2)):
        _within(ww, w64, C_UPD * U * (w0.double().abs() + Sw) + lw * eg, f"{what} w")
        _within(hh, h64, C_UPD * U * (h0.double().abs() + Sh) + lh * eg, f"{what} h")
    # both forms reduce the same accumulators: they agree within the update tolerance alone
    _within(w, w2.cpu().double(), C_UPD * U * (w0.double().abs() + Sw), "sfb fused vs two-pass w")
    assert torch.equal(wb, w.to(BF16)) and torch.equal(wb2, w2.to(BF16)), "bf16 shadow must equal the master"
    for buf, v, nm in ((wbuf, w, "w"), (hbuf, h, "h"), (bbuf, wb, "wb"), (wbuf2, w2, "w2"), (hbuf2, h2, "h2"),
                       (bbuf2, wb2, "wb2")):
        _assert_guard(buf, [v], f"sfb {nm}")


# ------------------------------------------------------------------------------------------------------------ repeatability
# name -> builder(ext): makes that op's inputs once and returns fn() -> output tensors; every call of fn starts from the same
# inputs (accumulation targets restored)
_REPEAT = {}
CU = "cuda"


def _repeatable(name):
    def reg(builder):
        _REPEAT[name] = builder
        return builder
    return reg


@_repeatable("gemm_f32")
def _rep_gemm_f32(ext):
    A, B = _randn((1000, 1024), 1, dtype=BF16).to(CU), _randn((520, 1024), 2, dtype=BF16).to(CU)
    o0 = _randn((1000, 520), 3).to(CU)

    def fn():
        out = o0.clone()
        ext.gemm_f32(A, False, B, False, out, 0.5, True, 3, 0)
        return [out]
    return fn


@_repeatable("gemm_bf16")
def _rep_gemm_bf16(ext):
    A, B = _randn((200, 4096), 4, dtype=BF16).to(CU), _randn((1000, 4096), 5, dtype=BF16).to(CU)
    bias = _randn((1000,), 6).to(CU)
    return lambda: [ext.gemm_bf16(A, False, B, False, bias, True, 0.1, None, None, 0)]


REPEAT_CONV = [(2, 40, 9, 9, 72, 3, 1, 1, 1, 0),       # one split: one atomic add per element
               (4, 64, 28, 28, 128, 3, 1, 1, 1, 0),    # workspace, single CTAs
               (4, 96, 27, 27, 256, 5, 1, 2, 2, 0),    # grouped gather, workspace
               (4, 128, 28, 28, 256, 3, 1, 1, 1, 0)]   # workspace, CTA pairs (default schedule)


def _rep_conv(case):
    def builder(ext):
        n, cin, h, w, cout, kk, st, pd, grp, cgk = case
        x, dy, _, _, _ = _conv_case(case)
        xd, dyd = x.to(CU), dy.to(CU)
        d0 = _randn((cout, kk * kk * cin // grp), 13).to(CU)

        def fn():
            dw = d0.clone()
            ext.conv_wgrad(xd, dyd, dw, [kk, kk], [st, st], [pd, pd], grp, 0, 1.0, cgk)
            return [dw]
        return fn
    return builder


for _case in REPEAT_CONV:
    _REPEAT["conv_wgrad_" + "x".join(map(str, _case))] = _rep_conv(_case)


@_repeatable("colsum")
def _rep_colsum(ext):
    dyc = _randn((256 * 27 * 27, 96), 7, dtype=BF16).to(CU)
    c0 = _randn((96,), 8).to(CU)

    def fn():
        out = c0.clone()
        ext.colsum(dyc, dyc.shape[0], 96, 96, out, 1.0, True)
        return [out]
    return fn


@_repeatable("fused_update")
def _rep_fused_update(ext):
    wu, gu, hu = _randn((8195,), 9).to(CU), _randn((8195,), 10).to(CU), _randn((8195,), 11, 0.01).to(CU)

    def fn():
        w, g, h = wu.clone(), gu.clone(), hu.clone()
        wb = torch.empty(8195, dtype=BF16, device=CU)
        ext.fused_update(w, g, h, wb, 0.05, 0.9, 0.01, 1, False, 1e-8, 0.37, None, True)
        return [w, g, h, wb]
    return fn


@_repeatable("fused_update_multi")
def _rep_fused_update_multi(ext):
    sizes = [MULTI_SIZES[i % len(MULTI_SIZES)] for i in range(49)]
    mw = [_randn((s,), 400 + i).to(CU) for i, s in enumerate(sizes)]
    mg = [_randn((s,), 500 + i).to(CU) for i, s in enumerate(sizes)]

    def fn():
        ws, gs = [t.clone() for t in mw], [t.clone() for t in mg]
        hs = [torch.zeros_like(t) for t in mw]
        wbs = [torch.empty(t.numel(), dtype=BF16, device=CU) for t in mw]
        ext.fused_update_multi(ws, gs, hs, wbs, [0.01 * (i + 1) for i in range(49)], [1e-3] * 49, [i % 2 for i in range(49)],
                               0.9, 0, False, 1e-8, 1.0, None)
        return ws + gs + hs + wbs
    return fn


def _sfb_repeat_inputs():
    us, vs, _, _ = _sfb_case(3, 328, 1000, 160)
    ud, vd = [u.to(CU) for u in us], [v.to(CU) for v in vs]
    return ud, vd, [t.data_ptr() for t in ud], [t.data_ptr() for t in vd]


@_repeatable("sfb_outer_sgd")
def _rep_sfb_outer_sgd(ext):
    ud, vd, up, vp = _sfb_repeat_inputs()
    sw0 = _randn((328, 1000), 12).to(CU)

    def fn():
        _ = (ud, vd)                                    # the factors stay alive while their addresses are in use
        w, h, wb = sw0.clone(), torch.zeros_like(sw0), torch.empty(328, 1000, dtype=BF16, device=CU)
        ext.sfb_outer_sgd(up, vp, 160, 328, 1000, w, h, wb, 1 / 160, 0.05, 0.9, 1e-3, 1, True, 1e-8, None, 0, 0, 0, 0,
                          None, None)
        return [w, h, wb]
    return fn


@_repeatable("sfb_outer_f32")
def _rep_sfb_outer_f32(ext):
    ud, vd, up, vp = _sfb_repeat_inputs()

    def fn():
        _ = (ud, vd)
        out = torch.empty(328, 1000, device=CU)
        ext.sfb_outer_f32(up, vp, 160, 328, 1000, out, 1 / 160, None, 0, 0, 0, 0, None)
        return [out]
    return fn


@_repeatable("softmax_xent")
def _rep_softmax_xent(ext):
    xs = _randn((4096, 1000), 15, 3.0, dtype=BF16).to(CU)
    lab = torch.randint(0, 1000, (4096,), generator=torch.Generator().manual_seed(16)).float().to(CU)
    return lambda: list(ext.softmax_xent(xs, lab, 1.0, True, True))


@pytest.mark.gpu
@pytest.mark.parametrize("op", list(_REPEAT))
def test_op_repeatable(ext, op):
    """The same op on identical inputs gives the same bits: no result depends on which CTA finished first."""
    fn = _REPEAT[op](ext)
    first = [t.clone() for t in fn()]
    second = fn()
    for i, (a, b) in enumerate(zip(first, second)):
        assert torch.equal(a, b), f"{op}: output {i} differs between two identical calls"


def _reset_dropout_streams():
    """Dropout masks are keyed on process-wide counters (call site, device iteration counter): restart them so that two
    runs in one process draw the same masks."""
    from poseidon_b200.ops import sm100
    sm100._dropout_counter[0] = 0
    sm100._iter_seed.clear()


def _blobs(s):
    return {f"{n}.{j}": l.export_blob(j) for n, l in zip(s.net.layer_names, s.net.layers) for j in range(len(l.blobs))}


@pytest.mark.gpu
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "cuda_graph"])
def test_smallnet_step_bit_exact(ext, graph):
    """Four training steps of the small net on the sm100 engine, twice: equal losses and bit-identical blobs."""
    from smallnet import feed, make_data, small_net, small_solver_param
    from poseidon_b200 import get_solver

    def run():
        _reset_dropout_streams()
        s = get_solver(small_solver_param(small_net(batch=16), max_iter=4), engine="sm100")
        x, y = make_data(16 * 4)
        feed(s, x, y)
        if graph:
            s.enable_cuda_graph(warmup=2)
        losses = []
        for _ in range(4):
            s.step(1)
            losses.append(float(s.last_loss))
        torch.cuda.synchronize()
        graphed = getattr(s, "_graph", None) is not None
        out = _blobs(s)
        s.close()
        return losses, out, graphed

    l1, b1, g1 = run()
    l2, b2, g2 = run()
    assert g1 == g2 == graph, "the step was (not) captured as requested"
    assert l1 == l2, (l1, l2)
    for name in b1:
        assert np.array_equal(b1[name], b2[name]), f"{name} differs between two identical runs"


@pytest.mark.gpu
def test_googlenet_step_bit_exact(ext):
    """GoogLeNet at batch 4, two steps, twice (lanes, side-stream weight gradients, zero-copy concat): equal losses and
    bit-identical blobs."""
    from poseidon_b200 import get_solver
    from poseidon_b200.models import zoo

    def run():
        _reset_dropout_streams()
        net = zoo.googlenet(batch=4, test_batch=4)
        sp = zoo.get_solver_param("googlenet", net=net, display=0, snapshot=0, snapshot_after_train=False, test_interval=0,
                                  max_iter=2, random_seed=3)
        sp.clear("test_iter")
        sp.base_lr = 0.0005
        s = get_solver(sp, engine="sm100")
        losses = []
        for _ in range(2):
            s.step(1)
            losses.append(float(s.last_loss))
        torch.cuda.synchronize()
        out = _blobs(s)
        s.close()
        return losses, out

    l1, b1 = run()
    l2, b2 = run()
    assert l1 == l2, (l1, l2)
    diff = [n for n in b1 if not np.array_equal(b1[n], b2[n])]
    assert not diff, f"blobs differ between two identical runs: {diff[:10]}"
