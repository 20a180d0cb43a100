"""CTA-pair kernels (2-CTA clusters sharing the B tile by multicast) vs the single-CTA kernels and the fp32 reference.

Every GEMM-shaped op is run twice — ``set_pair_cta(1)`` (default: two CTAs per B tile, each fetching half of it for both) and
``set_pair_cta(0)`` (one CTA per 128 x BN tile) — on shapes with odd m-block counts (phantom block in the last pair),
ragged edges, split-K, multi-source reductions and the im2col-TMA convolution modes."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rand(shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _close(got, ref, rel=2e-2, what=""):
    err = (got.float() - ref.float()).abs().max().item()
    mag = ref.float().abs().max().item() + 1e-6
    assert err <= rel * mag, f"{what}: max err {err} vs magnitude {mag}"


@pytest.fixture(params=[1, 0], ids=["pair", "single"])
def mode(ext, request):
    ext.set_pair_cta(request.param)
    yield request.param
    ext.set_pair_cta(1)


@pytest.fixture(params=[(2, 1), (4, 1), (1, 1), (1, 0)], ids=["mcast2", "mcast4", "pair", "single"])
def conv_mode(ext, request):
    """Convolution schedules: cluster multicast of the im2col operand (2 or 4 CTAs per cluster, each fetching a slice
    of the shared pixel tile), paired CTAs, plain single-CTA."""
    mc, pair = request.param
    ext.set_conv_mcast(mc)
    ext.set_conv_pair(pair)
    yield request.param
    ext.set_conv_mcast(1)
    ext.set_conv_pair(1)


@pytest.mark.parametrize("M,N,K", [(256, 256, 64), (384, 256, 512), (1000, 320, 200), (4096, 1024, 1024), (640, 96, 576),
                                   (130, 4096, 256)])
@pytest.mark.parametrize("bn", [0, 64, 128, 256])
def test_gemm_kmajor(ext, mode, M, N, K, bn):
    a, b = _rand((M, K), 1.0, 1), _rand((N, K), 0.05, 2)
    bias = torch.randn(N, device="cuda")
    c = ext.gemm_bf16(a, False, b, False, bias, True, 0.0, None, None, bn)
    _close(c, torch.relu(a.float() @ b.float().t() + bias), what="K x K")


@pytest.mark.parametrize("M,N,K", [(256, 9216, 512), (384, 1000, 264), (1024, 256, 4096)])
def test_gemm_kmajor_x_mnmajor(ext, mode, M, N, K):
    dy, w = _rand((M, K), 1.0, 3), _rand((K, N), 0.05, 4)
    mask = _rand((M, N), 1.0, 5)
    c = ext.gemm_bf16(dy, False, w, True, None, False, 0.0, mask, None, 0)
    _close(c, (dy.float() @ w.float()) * (mask.float() > 0), what="K x MN")


@pytest.mark.parametrize("Mb,N,K", [(256, 4096, 1024), (200, 384, 520), (512, 256, 256)])
@pytest.mark.parametrize("split_k", [1, 3])
def test_gemm_mnmajor_f32(ext, mode, Mb, N, K, split_k):
    dy, x = _rand((Mb, N), 1.0, 6), _rand((Mb, K), 1.0, 7)
    out = torch.zeros(N, K, device="cuda")
    ext.gemm_f32(dy, True, x, True, out, 1.0, False, split_k, 0)
    _close(out, dy.float().t() @ x.float(), rel=1e-2, what="MN x MN")


def test_sfb_outer_sgd_multi_source(ext, mode):
    """EPI_SGD epilogue over 3 reduction sources (the SFB reconstruct kernel), N = 384 rows -> 3 m-blocks."""
    Mb, N, K, P = 128, 384, 1024, 3
    us, vs = [_rand((Mb, N), 1.0, 10 + i) for i in range(P)], [_rand((Mb, K), 1.0, 20 + i) for i in range(P)]
    w = torch.randn(N, K, device="cuda")
    h = torch.rand(N, K, device="cuda") * 0.1
    wb = torch.empty(N, K, device="cuda", dtype=torch.bfloat16)
    w_ref, h_ref = w.clone(), h.clone()
    lr, mom, wd = 0.01, 0.9, 5e-4
    ext.sfb_outer_sgd([u.data_ptr() for u in us], [v.data_ptr() for v in vs], Mb, N, K, w, h, wb, 1.0, lr, mom, wd, 0, False,
                      1e-8, None, 0, 1, 0, 0, None, None)
    g = sum(u.float().t() @ v.float() for u, v in zip(us, vs)) + wd * w_ref
    h_ref = lr * g + mom * h_ref
    w_ref = w_ref - h_ref
    _close(w, w_ref, rel=1e-3, what="W")
    _close(h, h_ref, rel=1e-2, what="H")
    _close(wb, w_ref, rel=1e-2, what="Wb")


CONV = [
    # (N, Cin, H, W, Cout, k, stride, pad, group) — all TMA-im2col eligible (C_g % 64 == 0)
    (4, 256, 13, 13, 384, 3, 1, 1, 1),     # AlexNet conv3
    (2, 384, 13, 13, 384, 3, 1, 1, 2),     # conv4 (grouped)
    (2, 384, 13, 13, 256, 3, 1, 1, 2),     # conv5
    (2, 64, 56, 56, 192, 3, 1, 1, 1),      # GoogLeNet conv2/3x3
    (3, 128, 7, 9, 256, 3, 1, 1, 1),       # odd spatial extent: ragged last m-block and a phantom block
    (2, 192, 28, 28, 64, 1, 1, 0, 1),      # 1x1
    (2, 512, 14, 14, 512, 3, 1, 1, 1),     # VGG conv4/5 shape: Cout 512 -> wgrad pairs along Cout
    (2, 64, 28, 28, 96, 3, 1, 1, 1),       # Cout 96: multicast tiles of 64 (+32 valid) / 32 columns
    (2, 128, 14, 14, 48, 1, 1, 0, 1),      # Cout 48: narrowest tiles
    (2, 192, 14, 14, 320, 3, 1, 1, 1),     # Cout 320 -> 2 x 192 / 4 x 96 (phantom columns)
]


@pytest.mark.parametrize("case", CONV)
def test_conv_im2col(ext, conv_mode, case):
    from poseidon_b200.ops import sm100
    from test_ops_gpu import _FakeLayer, _nhwc
    n, cin, h, w, cout, k, stride, pad, group = case
    layer = _FakeLayer(cout, cin, k, stride, pad, group)
    layer.in_hw = (h, w)
    x = _nhwc((n, cin, h, w), 5)
    xs = x.clone().requires_grad_(True)
    y = sm100.conv2d(xs, layer.weight, layer.bias, layer.stride, layer.pad, group, relu_slope=0.0, layer=layer)
    wref = layer.weight.detach().float().contiguous().requires_grad_(True)
    bref = layer.bias.detach().clone().requires_grad_(True)
    xr = x.float().requires_grad_(True)
    yr = torch.relu(torch.nn.functional.conv2d(xr, wref.to(torch.bfloat16).float(), bref, stride, pad, 1, group))
    _close(y, yr, what="conv fprop")
    dy = _nhwc(tuple(yr.shape), 6)
    y.backward(dy)
    yr2 = torch.nn.functional.conv2d(xr, wref, bref, stride, pad, 1, group)
    yr2.backward(dy.float() * (y.detach().float() > 0))
    _close(xs.grad, xr.grad, rel=3e-2, what="conv dgrad")
    _close(layer.weight.grad, wref.grad, rel=3e-2, what="conv wgrad")


DGRAD_W = [
    # (N, Cin, H, W, Cout, k, pad, group): the pack-free data gradient (B = fprop weights through a 3-D map, MN-major)
    (4, 256, 13, 13, 384, 3, 1, 1),        # AlexNet conv3: Cout_g 384 = 6 whole k-blocks per tap
    (2, 384, 13, 13, 256, 3, 1, 2),        # conv5 grouped: Cout_g 128, C_g 192 -> BN 256 with 64 zero-filled columns
    (2, 96, 28, 28, 208, 3, 1, 1),         # Cout_g 208: last k-block of every tap is 16 real + 48 zero-filled rows
    (2, 16, 14, 14, 48, 5, 2, 1),          # GoogLeNet 5x5 reduce: C_g 16 (BN 64, 48 columns out of bounds), Cout_g 48
    (3, 128, 7, 9, 24, 1, 0, 1),           # 1x1, Cout_g 24: a single, mostly empty k-block
    (2, 64, 56, 56, 192, 3, 1, 1),         # many m-blocks: pairs and a full wave
    (2, 40, 9, 9, 72, 3, 1, 1),            # C_g 40, Cout_g 72: neither a multiple of 64
]


@pytest.mark.parametrize("case", DGRAD_W)
@pytest.mark.parametrize("masked", [False, True], ids=["plain", "relu_mask"])
def test_conv_dgrad_from_fprop_weights(ext, conv_mode, case, masked):
    """conv_dgrad_w against the fp32 transposed convolution AND against the packed-operand kernel it replaces."""
    if conv_mode[0] != 1:
        pytest.skip("the multicast schedules do not apply to the data gradient's weight operand")
    from test_ops_gpu import _nhwc
    n, cin, h, w, cout, k, pad, group = case
    cg, cout_g = cin // group, cout // group
    wf = (torch.randn(cout, k, k, cg, generator=torch.Generator().manual_seed(3)) * (cg * k * k) ** -0.5).cuda()
    wb = wf.to(torch.bfloat16).reshape(cout, k * k * cg).contiguous()
    oh, ow = h + 2 * pad - k + 1, w + 2 * pad - k + 1
    dy = _nhwc((n, cout, oh, ow), 11)
    mask = _nhwc((n, cin, h, w), 12) if masked else None
    got = ext.conv_dgrad_w(dy, wb, [k, k], [pad, pad], group, h, w, mask, 0.0)
    w4 = wb.float().reshape(cout, k, k, cg).permute(0, 3, 1, 2).contiguous()
    ref = torch.nn.functional.conv_transpose2d(dy.float(), w4, None, 1, pad, 0, group)
    if masked:
        ref = ref * (mask.float() > 0)
    assert got.shape == ref.shape and got.is_contiguous(memory_format=torch.channels_last)
    _close(got, ref, rel=2e-2, what="dgrad from fprop weights")
    wt = ext.conv_pack_dgrad(wf.reshape(-1), cout, k * k, cg, group, None, 0)
    old = ext.conv_dgrad(dy, wt, [k, k], [pad, pad], group, h, w, mask, 0.0)
    _close(got, old, rel=1e-2, what="pack-free vs packed dgrad")
    assert cout_g % 8 == 0 and cg % 8 == 0


@pytest.mark.parametrize("M,N,K,ldc_pad", [(256, 256, 64, 0), (1000, 328, 200, 0), (130, 96, 256, 8), (4096, 1024, 512, 0),
                                           (515, 40, 128, 24), (384, 200, 192, 0)])
@pytest.mark.parametrize("bn", [0, 64, 128, 256])
def test_bf16_bulk_epilogue_matches_walk(ext, mode, M, N, K, ldc_pad, bn):
    """bf16 outputs through the two-slab bulk-store epilogue (bias + ReLU + mask applied in the lane = row layout) against
    the per-warp walk and the fp32 reference; N a multiple of 8 with ragged last tiles, partial last chunk, padded ldc."""
    a, b = _rand((M, K), 1.0, 1), _rand((N, K), K ** -0.5, 2)
    bias = torch.randn(N, device="cuda")
    ref = torch.nn.functional.leaky_relu(a.float() @ b.float().t() + bias, 0.1)
    outs = []
    for bits in (3, 1):
        ext.set_bulk_epilogue(bits)
        try:
            out = torch.full((M, N + ldc_pad), 7.0, device="cuda", dtype=torch.bfloat16)
            c = out[:, :N]
            ext.gemm_bf16(a, False, b, False, bias, True, 0.1, None, c, bn)
            outs.append(out)
        finally:
            ext.set_bulk_epilogue(1)
    _close(outs[0][:, :N], ref, what="bulk epilogue")
    assert torch.equal(outs[0], outs[1]), "bulk-store and walk epilogues must agree bit for bit (padding untouched)"


def test_pair_gemm_throughput(ext):
    """8192^3 bf16: CTA pairs vs single-CTA vs cuBLAS on the same box (printed; asserts a sanity floor relative to cuBLAS on
    the same card, because the absolute rate of an H100 depends on its power limit)."""
    a, b = _rand((8192, 8192), 1.0, 1), _rand((8192, 8192), 1.0, 2)
    out = torch.empty(8192, 8192, device="cuda", dtype=torch.bfloat16)

    def bench(fn, iters=5):
        for _ in range(2):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return 2 * 8192 ** 3 * iters / (e0.elapsed_time(e1) * 1e-3) / 1e12
    ext.set_pair_cta(1)
    tf2 = bench(lambda: ext.gemm_bf16(a, False, b, False, None, False, 0.0, None, out, 256))
    ext.set_pair_cta(0)
    tf1 = bench(lambda: ext.gemm_bf16(a, False, b, False, None, False, 0.0, None, out, 256))
    ext.set_pair_cta(1)
    tfc = bench(lambda: torch.matmul(a, b.t()))
    print(f"\n8192^3 bf16: pair {tf2:.0f} TFLOP/s, single-CTA {tf1:.0f}, cuBLAS {tfc:.0f}")
    assert tf2 > 0.7 * tfc, (tf2, tfc)
