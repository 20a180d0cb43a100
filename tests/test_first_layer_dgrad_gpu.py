"""First-layer data gradients on sm_90a (s2d, ROW and 8-channel-pad convolutions) against float64, through the data
layer's physical hand-off and through a logical input; force_backward training steps under CUDA-graph capture; Net.backward
on the CaffeNet deploy net."""
import os

import pytest
import torch

from poseidon_b200 import proto as P

from test_accumulate_gpu import C_GEMM, U, _bf16_bound, _within

BF16, CL = torch.bfloat16, torch.channels_last
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference")

CASES = [
    # (N, C, H, W, Cout, kernel, stride, pad, mode)
    ((2, 3, 227, 227, 96, 11, 4, 0, "s2d"), "AlexNet conv1"),
    ((1, 3, 35, 35, 16, 11, 4, 2, "s2d"), "s2d, batch 1, odd size, pad 2"),
    ((2, 3, 224, 224, 64, 7, 2, 3, "row"), "GoogLeNet conv1"),
    ((1, 3, 33, 31, 16, 5, 2, 0, "row"), "ROW, batch 1, odd sizes, pad 0"),
    ((2, 3, 224, 224, 64, 3, 1, 1, "pad8"), "VGG conv1_1"),
    ((2, 1, 28, 28, 20, 5, 1, 0, "pad8"), "LeNet conv1"),
    ((1, 3, 15, 13, 16, 3, 1, 1, "pad8"), "8-channel pad, batch 1, odd sizes"),
]


def _check_case(sm100, case):
    from test_ops_gpu import _FakeLayer
    n, c, h, w, cout, k, stride, pad, mode = case
    layer = _FakeLayer(cout, c, k, stride, pad, 1)
    layer.in_hw = (h, w)
    st = sm100.conv_state(layer, c)
    assert (st.s2d, st.row_mode and not st.pad8 and not st.s2d, st.pad8) == (mode == "s2d", mode == "row", mode == "pad8")
    g = torch.Generator().manual_seed(n * 1000 + h + w)
    x = torch.randn(n, c, h, w, generator=g).to(BF16).float().cuda()

    xl = x.clone().requires_grad_(True)                       # logical input (a deploy `input:`)
    y = sm100.conv2d(xl, layer.weight, layer.bias, layer.stride, layer.pad, 1, relu_slope=None, layer=layer)
    dy = torch.randn(tuple(y.shape), generator=g).to(BF16)
    y.backward(dy.cuda().contiguous(memory_format=CL))
    logical = xl.grad

    xp = sm100.prepare_first_layer_input(x, st, layer.pad, (h, w)).requires_grad_(True)    # the data layer's hand-off
    y2 = sm100.conv2d(xp, layer.weight, layer.bias, layer.stride, layer.pad, 1, relu_slope=None, layer=layer)
    assert torch.equal(y2.float(), y.float())
    y2.backward(dy.cuda().contiguous(memory_format=CL))
    phys = xp.grad
    assert tuple(phys.shape) == tuple(xp.shape)
    handoff = sm100.first_layer_diff(phys, layer, (n, c, h, w), True)
    torch.cuda.synchronize()

    assert logical.dtype == torch.float32 and tuple(logical.shape) == (n, c, h, w)
    assert torch.equal(handoff, logical), f"{mode}: hand-off and logical paths differ"
    pf = phys.float().cpu()
    if mode == "s2d":
        assert not pf.view(n, 16, 4, *pf.shape[2:])[:, :, c:].any(), "s2d padding channels"
    else:
        assert not pf[:, c:].any(), f"{mode}: padded channels"

    w64 = layer.weight.detach().to(BF16).double().cpu()
    ref = torch.nn.grad.conv2d_input((n, c, h, w), w64, dy.double(), layer.stride, layer.pad)
    mag = torch.nn.grad.conv2d_input((n, c, h, w), w64.abs(), dy.double().abs(), layer.stride, layer.pad)
    _within(logical, ref, _bf16_bound(ref, C_GEMM * k * k * cout * U * mag), f"{mode} first-layer dX {case}")


def _check_round_trip(ext, mode, pad):
    oh, ow, n = 19, 17, 2
    c = 1 if mode == "pad8" else 3
    x = torch.randn(n, c, oh, ow, generator=torch.Generator().manual_seed(pad)).to(BF16).float().cuda()
    zero = torch.zeros(n, dtype=torch.int32, device="cuda")
    flip = torch.zeros(n, dtype=torch.uint8, device="cuda")
    if mode == "s2d":
        hq, wq = -(-(oh + 2 * pad) // 4), -(-(ow + 2 * pad) // 4)
        phys = ext.transform_nhwc(x, zero, zero, flip, None, 1.0, oh, ow, 4, pad, 4 * wq - ow - 2 * pad,
                                  4 * hq - oh - 2 * pad, True)
    elif mode == "row":
        phys = ext.transform_nhwc(x, zero, zero, flip, None, 1.0, oh, ow, 4, pad, (ow + 2 * pad) % 2, 0, False)
    else:
        phys = ext.transform_nhwc(x, zero, zero, flip, None, 1.0, oh, ow, 8, 0, 0, 0, False)
    for out_float in (True, False):
        back = ext.first_layer_diff(phys, c, oh, ow, pad, pad, mode == "s2d", out_float)
        assert back.dtype == (torch.float32 if out_float else BF16) and back.is_contiguous()
        assert torch.equal(back.float(), x), (mode, pad, out_float)


def _check_caffenet_deploy():
    """Net.backward on the CaffeNet deploy net with force_backward: a finite, non-zero diff of the image's shape."""
    from poseidon_b200.layers import NetContext
    from poseidon_b200.net.net import Net
    p = P.read_net(os.path.join(GOLDEN, "models", "bvlc_reference_caffenet", "deploy.prototxt"))
    p.force_backward = True
    net = Net(p, phase=P.TEST, ctx=NetContext(phase=P.TEST, device="cuda", engine="sm100", dtype=BF16))
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():
        for prm in net.params:
            prm.copy_(torch.randn(prm.shape, generator=g) * 0.01)
    for layer in net.layers:
        if getattr(layer, "_sm100", None) is not None and hasattr(layer._sm100, "mark_updated"):
            layer._sm100.mark_updated()
    net.to("cuda")
    n = net.blob_shapes["data"][0]
    x = torch.randn(tuple(net.blob_shapes["data"]), generator=g).cuda() * 50
    net.forward({"data": x})
    onehot = torch.zeros(n, 1000, 1, 1, device="cuda")
    onehot[torch.arange(n), torch.arange(n) * 7] = 1.0
    d = net.backward({"prob": onehot})["data"]
    torch.cuda.synchronize()
    assert d.dtype == torch.float32 and tuple(d.shape) == (n, 3, 227, 227)
    assert torch.isfinite(d).all() and d.abs().max() > 0
    assert net.layer_by_name["conv1"]._sm100.s2d


@pytest.mark.gpu
def test_first_layer_dgrad_matches_float64(ext):
    """dX of the first convolution for every geometry in CASES, from the logical input (first_layer_diff in the
    backward) and from the physical layout a data layer hands over (first_layer_diff after it): both within the bf16
    bound of float64 conv_transpose2d of the bf16 dY and weights, bit-identical to each other, padding lanes of the
    physical dX exactly zero.  Then transform_nhwc followed by first_layer_diff is the identity, bit for bit, and
    Net.backward on the CaffeNet deploy net returns the image diff."""
    from poseidon_b200.ops import sm100
    for case, _ in CASES:
        _check_case(sm100, case)
    for mode, pad in [("s2d", 0), ("s2d", 3), ("row", 1), ("row", 2), ("pad8", 0)]:
        _check_round_trip(ext, mode, pad)
    _check_caffenet_deploy()


def _train(model, batch, force, steps=2):
    """Graph-captured sm100 training of a zoo net; returns (losses, weights)."""
    from poseidon_b200 import get_solver
    from poseidon_b200.models import zoo
    from poseidon_b200.ops import sm100
    # dropout masks come from process-wide counters (the call-site counter behind each layer's seed and the device-side
    # iteration counter): start both runs from the same state
    sm100._dropout_counter[0] = 0
    sm100._iter_seed.clear()
    net = zoo.get_model(model, batch=batch, test_batch=batch)
    net.force_backward = force
    sp = zoo.get_solver_param(model, net=net, display=0, snapshot=0, snapshot_after_train=False, test_interval=0,
                              max_iter=100, random_seed=7)
    sp.clear("test_iter")
    s = get_solver(sp, engine="sm100")
    assert s.net.blob_need_backward["data"] == force
    s.enable_cuda_graph(warmup=2)
    losses = []
    for _ in range(steps):
        s.step(1)
        losses.append(float(s.last_loss))
    torch.cuda.synchronize()
    weights = {f"{n}.{j}": l.export_blob(j) for n, l in zip(s.net.layer_names, s.net.layers) for j in range(len(l.blobs))}
    s.close()
    return losses, weights


@pytest.mark.gpu
def test_force_backward_training_is_bit_identical(ext):
    """The forward is unchanged and the image diff force_backward adds is written and never read: graph-captured
    training steps of an AlexNet (s2d conv1) and a GoogLeNet (ROW conv1) give the same losses and weights, bit for bit,
    with and without it."""
    import numpy as np
    for model, batch in (("alexnet", 8), ("googlenet", 4)):
        off = _train(model, batch, False)
        on = _train(model, batch, True)
        assert on[0] == off[0], (model, on[0], off[0])
        for name, w in off[1].items():
            assert np.array_equal(w, on[1][name]), (model, name)
