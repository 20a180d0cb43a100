"""sm_90a layer kernels vs fp32 PyTorch references with Caffe semantics (run on an H100)."""
import pytest
import torch

from poseidon_b200.ops import reference as R

pytestmark = pytest.mark.gpu
CL = torch.channels_last


def _nhwc(shape, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, generator=g, device="cuda") * scale
    return x.to(torch.bfloat16).contiguous(memory_format=CL)


def _close(got, ref, rel=2e-2, what=""):
    err = (got.float() - ref.float()).abs().max().item()
    mag = ref.float().abs().max().item() + 1e-6
    assert err <= rel * mag, f"{what}: max err {err} vs magnitude {mag}"


@pytest.mark.parametrize("shape", [(4, 96, 27, 27), (2, 256, 13, 13), (3, 64, 9, 7), (2, 192, 5, 5)])
def test_lrn_fwd_bwd(ext, shape):
    from poseidon_b200.ops import sm100
    x = _nhwc(shape, 1, 2.0)
    dy = _nhwc(shape, 2)
    xr = x.float().requires_grad_(True)
    yr = R.lrn_across(xr, 5, 1e-1, 0.75)
    yr.backward(dy.float())
    xs = x.clone().requires_grad_(True)
    y = sm100.lrn_across(xs, 5, 1e-1, 0.75)
    y.backward(dy)
    _close(y, yr, what="lrn fwd")
    _close(xs.grad, xr.grad, what="lrn bwd")


@pytest.mark.parametrize("shape,k,s,p", [((4, 96, 55, 55), 3, 2, 0), ((2, 256, 13, 13), 3, 2, 0),
                                          ((2, 64, 28, 28), 3, 1, 1), ((2, 192, 56, 56), 3, 2, 0),
                                          ((2, 128, 14, 14), 5, 3, 0),
                                          ((2, 64, 13, 11), (3, 2), (2, 1), (1, 0)),      # rectangular window / stride / pad
                                          ((3, 96, 9, 16), (2, 3), (1, 2), (0, 1))])
@pytest.mark.parametrize("is_max", [True, False])
def test_pool_fwd_bwd(ext, shape, k, s, p, is_max):
    from poseidon_b200.ops import sm100
    k, s, p = _pair(k), _pair(s), _pair(p)
    x = _nhwc(shape, 3)
    xr = x.float().contiguous().requires_grad_(True)      # oracle on plain NCHW fp32
    fn_r = R.max_pool if is_max else R.ave_pool
    yr = fn_r(xr, k, s, p)
    dy = _nhwc(tuple(yr.shape), 4)
    yr.backward(dy.float().contiguous())
    xs = x.clone().requires_grad_(True)
    fn = sm100.max_pool if is_max else sm100.ave_pool
    y = fn(xs, k, s, p)
    assert tuple(y.shape) == tuple(yr.shape)
    y.backward(dy)
    _close(y, yr, what="pool fwd")
    _close(xs.grad, xr.grad, rel=3e-2, what="pool bwd")


@pytest.mark.parametrize("rows,C", [(256, 1000), (32, 10), (50, 21)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_softmax_xent(ext, rows, C, dtype):
    from poseidon_b200.ops import sm100
    x = (torch.randn(rows, C, device="cuda") * 3).to(dtype)
    label = torch.randint(0, C, (rows,), device="cuda").float()
    xr = x.detach().float().clone().requires_grad_(True)
    lr_ = R.softmax_loss(xr, label)
    (lr_ * 0.3).backward()
    xs = x.detach().clone().requires_grad_(True)
    loss, prob = sm100.softmax_loss(xs.view(rows, C, 1, 1), label, return_prob=True)
    (loss * 0.3).backward()
    assert abs(loss.item() - lr_.item()) < 2e-3 * max(1.0, abs(lr_.item()))
    _close(xs.grad, xr.grad, rel=3e-2, what="xent grad")
    _close(prob.view(rows, C), torch.softmax(x.float(), 1), rel=1e-2, what="prob")


def test_dropout_statistics_and_backward(ext):
    from poseidon_b200.ops import sm100
    x = torch.ones(256, 4096, device="cuda", dtype=torch.bfloat16).requires_grad_(True)
    y = sm100.dropout(x, 0.5, True)
    keep = (y > 0).float().mean().item()
    assert abs(keep - 0.5) < 0.01
    assert torch.all((y == 0) | (y == 2))
    y.backward(torch.ones_like(y))
    assert torch.equal(x.grad, y.detach())          # same mask, same scale
    y2 = sm100.dropout(x, 0.5, True)
    assert not torch.equal(y2, y)                    # fresh mask every call
    sm100.bump_iteration_seed(x.device)              # ... and every iteration (device-side counter)
    from poseidon_b200.ops.sm100 import _DropoutFn
    a = _DropoutFn.apply(x, 0.5, 123)
    sm100.bump_iteration_seed(x.device)
    b = _DropoutFn.apply(x, 0.5, 123)
    assert not torch.equal(a, b)


def test_colsum(ext):
    dy = torch.randn(5000, 96, device="cuda").to(torch.bfloat16)
    out = torch.empty(96, device="cuda")
    ext.colsum(dy, 5000, 96, 96, out, 1.0, False)
    _close(out, dy.float().sum(0), rel=1e-3, what="colsum")


def test_transform_kernel_matches_reference(ext):
    from poseidon_b200 import proto as P
    from poseidon_b200.data.transformer import DataTransformer
    tp = P.TransformationParameter(crop_size=27, mirror=True, scale=0.5)
    tp.mean_value = [104.0, 117.0, 123.0]
    tr = DataTransformer(tp, P.TRAIN, "cuda", seed=3)
    x = torch.randint(0, 256, (8, 3, 32, 32), dtype=torch.uint8, device="cuda")
    draws = tr.draw(8, 32, 32)
    ref = tr(x, torch.float32, draws=draws)
    h_off, w_off, flip = draws
    mean = tr.mean_values.float().cuda()
    out = ext.transform_nhwc(x, h_off.int().cuda(), w_off.int().cuda(), flip.to(torch.uint8).cuda(), mean, 0.5, 27, 27, 4,
                             0, 1, 0, False)
    assert tuple(out.shape) == (8, 4, 27, 28)
    _close(out[:, :3, :, :27], ref, rel=1e-2, what="transform")
    assert out[:, 3].abs().max().item() == 0 and out[:, :, :, 27].abs().max().item() == 0
    # border + space-to-depth output: pad 2 each side, extents rounded up to /4 -> 32x32 -> [8, 64, 8, 8]
    s2d = ext.transform_nhwc(x, h_off.int().cuda(), w_off.int().cuda(), flip.to(torch.uint8).cuda(), mean, 0.5, 27, 27, 4,
                             2, 1, 1, True)
    assert tuple(s2d.shape) == (8, 64, 8, 8)
    full = torch.zeros(8, 4, 32, 32, device="cuda")
    full[:, :3, 2:29, 2:29] = ref
    want = full.view(8, 4, 8, 4, 8, 4).permute(0, 2, 4, 3, 5, 1).reshape(8, 8, 8, 64).permute(0, 3, 1, 2)
    _close(s2d, want, rel=1e-2, what="transform s2d")


# ---------------------------------------------------------------------------------------------------- conv
def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


class _FakeLayer:
    """A conv layer's attributes; kernel, stride and pad take an int or an (h, w) pair."""
    def __init__(self, cout, cin, k, stride, pad, group, bias=True):
        self.layer_name = "conv"
        self.num_output, self.kernel, self.stride, self.pad, self.group = cout, _pair(k), _pair(stride), _pair(pad), group
        self.bias_term = bias
        g = torch.Generator(device="cuda").manual_seed(cout + cin + self.kernel[0] + 16 * (self.kernel[1] - self.kernel[0]))
        self.weight = torch.nn.Parameter(torch.randn(cout, cin // group, *self.kernel, generator=g, device="cuda") * 0.05)
        self.bias = torch.nn.Parameter(torch.randn(cout, generator=g, device="cuda") * 0.1) if bias else None
        self.in_hw = None


CONV_CASES = [
    # (N, Cin, H, W, Cout, k, stride, pad, group)
    (4, 96, 27, 27, 256, 5, 1, 2, 2),      # AlexNet conv2
    (4, 256, 13, 13, 384, 3, 1, 1, 1),     # conv3
    (2, 384, 13, 13, 384, 3, 1, 1, 2),     # conv4
    (2, 192, 28, 28, 16, 1, 1, 0, 1),      # GoogLeNet 5x5_reduce
    (2, 16, 28, 28, 32, 5, 1, 2, 1),       # GoogLeNet 5x5
    (2, 64, 56, 56, 192, 3, 1, 1, 1),      # conv2/3x3
    (3, 24, 7, 9, 40, 3, 1, 1, 1),         # odd sizes
    (2, 96, 28, 28, 128, 3, 1, 1, 1),      # GoogLeNet 3x3 after a 96-channel reduce: channel-padded im2col (96 -> 128)
    (2, 480, 14, 14, 208, 1, 1, 0, 1),     # 1x1 on 480 channels (-> 512), Cout 208 (dgrad slots 208 -> 256)
    (2, 160, 14, 14, 320, 3, 1, 1, 1),     # 160 -> 192
    (2, 64, 28, 28, 128, 3, 2, 1, 1),      # strided convolutions inside a net: dgrad = sh*sw stride-1 phase problems
    (2, 192, 15, 13, 64, 1, 2, 0, 1),
    (2, 64, 14, 14, 64, 5, 2, 2, 1),
    (2, 128, 12, 12, 128, 2, 3, 0, 2),     # stride > kernel (phases without taps), grouped
]


@pytest.mark.parametrize("case", CONV_CASES)
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("pad_k", ["0", "1"])
def test_conv_fwd_bwd(ext, case, relu, pad_k, monkeypatch):
    from poseidon_b200.ops import sm100
    n, cin, h, w, cout, k, stride, pad, group = case
    if pad_k == "1" and sm100._pad64(cin // group) == cin // group and sm100._pad64(cout // group) == cout // group:
        pytest.skip("no channel padding applies to this shape")
    monkeypatch.setenv("POSEIDON_PAD_K", pad_k)       # channel-padded K on the TMA im2col path (read at ConvState creation)
    layer = _FakeLayer(cout, cin, k, stride, pad, group)
    layer.in_hw = (h, w)
    x = _nhwc((n, cin, h, w), 5)
    xs = x.clone().requires_grad_(True)
    y = sm100.conv2d(xs, layer.weight, layer.bias, layer.stride, layer.pad, group, relu_slope=0.0 if relu else None,
                     layer=layer)
    wref = layer.weight.detach().float().contiguous().requires_grad_(True)
    bref = layer.bias.detach().clone().requires_grad_(True)
    xr = x.float().requires_grad_(True)
    yr = torch.nn.functional.conv2d(xr, wref.to(torch.bfloat16).float(), bref, stride, pad, 1, group)
    if relu:
        yr = torch.relu(yr)
    _close(y, yr, what="conv fprop")
    dy = _nhwc(tuple(yr.shape), 6)
    y.backward(dy)
    # oracle backward with the same bf16-rounded output mask
    yr2 = torch.nn.functional.conv2d(xr, wref, bref, stride, pad, 1, group)
    dyr = dy.float() * (y.detach().float() > 0) if relu else dy.float()
    yr2.backward(dyr)
    _close(xs.grad, xr.grad, rel=3e-2, what="conv dgrad")
    _close(layer.weight.grad, wref.grad, rel=3e-2, what="conv wgrad")
    _close(layer.bias.grad, bref.grad, rel=2e-2, what="conv bias grad")


@pytest.mark.parametrize("case", [(4, 3, 227, 227, 96, 11, 4, 0), (2, 3, 224, 224, 64, 7, 2, 3), (2, 1, 30, 30, 24, 5, 2, 0),
                                  (2, 3, 64, 64, 32, 11, 4, 2), (2, 3, 67, 67, 32, 8, 4, 0), (2, 3, 32, 30, 64, 3, 1, 1)])
def test_first_layer_conv_row_mode(ext, case):
    from poseidon_b200.ops import sm100
    n, cin, h, w, cout, k, stride, pad = case
    layer = _FakeLayer(cout, cin, k, stride, pad, 1)
    layer.in_hw = (h, w)
    x = torch.randn(n, cin, h, w, device="cuda").to(torch.bfloat16)
    y = sm100.conv2d(x, layer.weight, layer.bias, layer.stride, layer.pad, 1, relu_slope=0.0, layer=layer)
    wref = layer.weight.detach().clone().requires_grad_(True)
    bref = layer.bias.detach().clone().requires_grad_(True)
    yr = torch.relu(torch.nn.functional.conv2d(x.float(), wref.to(torch.bfloat16).float(), bref, stride, pad))
    assert tuple(y.shape) == tuple(yr.shape)
    _close(y, yr, what="conv1 fprop")
    dy = _nhwc(tuple(yr.shape), 7)
    y.backward(dy)
    yr2 = torch.nn.functional.conv2d(x.float(), wref, bref, stride, pad)
    yr2.backward(dy.float() * (y.detach().float() > 0))
    _close(layer.weight.grad, wref.grad, rel=3e-2, what="conv1 wgrad")
    _close(layer.bias.grad, bref.grad, rel=2e-2, what="conv1 bias grad")


@pytest.mark.parametrize("M,K,N", [(256, 9216, 4096), (64, 1024, 1000), (32, 4096, 1000)])
def test_inner_product_fwd_bwd(ext, M, K, N):
    from poseidon_b200.ops import sm100

    class L:
        layer_name = "fc"
        bias_term = True
        sfb = None
    layer = L()
    g = torch.Generator(device="cuda").manual_seed(11)
    layer.weight = torch.nn.Parameter(torch.randn(N, K, generator=g, device="cuda") * 0.02)
    layer.bias = torch.nn.Parameter(torch.randn(N, generator=g, device="cuda") * 0.1)
    x = (torch.randn(M, K, generator=g, device="cuda")).to(torch.bfloat16)
    xs = x.clone().requires_grad_(True)
    y = sm100.inner_product(xs, layer.weight, layer.bias, relu=True, layer=layer)
    wref = layer.weight.detach().clone().requires_grad_(True)
    bref = layer.bias.detach().clone().requires_grad_(True)
    xr = x.float().requires_grad_(True)
    yr = torch.relu(xr @ wref.to(torch.bfloat16).float().t() + bref)
    _close(y, yr, what="ip fwd")
    dy = torch.randn(M, N, generator=g, device="cuda").to(torch.bfloat16)
    y.backward(dy)
    yr2 = xr @ wref.t() + bref
    yr2.backward(dy.float() * (y.detach().float() > 0))
    _close(xs.grad, xr.grad, rel=3e-2, what="ip dgrad")
    _close(layer.weight.grad, wref.grad, rel=3e-2, what="ip wgrad")
    _close(layer.bias.grad, bref.grad, rel=2e-2, what="ip bias grad")
