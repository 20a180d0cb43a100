"""force_backward and Net.backward: Caffe's blob_need_backward rules, input-blob diffs on both engines (the sm100 engine
emulated on the CPU), and first_layer_diff's inverse of the first-layer layouts the transform op writes."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from poseidon_b200 import proto as P
from poseidon_b200.layers import NetContext
from poseidon_b200.models.zoo import NetBuilder
from poseidon_b200.net.net import Net

from test_accumulate_gpu import C_GEMM, U, _bf16_bound, _within

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference")
BF16 = torch.bfloat16


@pytest.fixture
def emu():
    from poseidon_b200.ops import counting, sm100
    sm100.set_emulation(True)
    counting.reset()
    yield sm100
    sm100.set_emulation(False)


def _net(param, engine="torch", phase=P.TRAIN, force=None):
    param = param.copy()
    if force is not None:
        param.force_backward = force
    ctx = NetContext(phase=phase, engine=engine, dtype=BF16 if engine == "sm100" else torch.float32, seed=5)
    return Net(param, ctx=ctx)


# ------------------------------------------------------------------------------------------------ blob_need_backward
def test_need_backward_lenet():
    """LeNet train: the image and the label need no diff; with force_backward the image does, the label never."""
    p = P.read_net(os.path.join(GOLDEN, "examples", "mnist", "lenet_train_test.prototxt"))
    computed = {b: True for b in ("conv1", "pool1", "conv2", "pool2", "ip1", "ip2", "loss")}
    assert _net(p, force=False).blob_need_backward == {"data": False, "label": False, **computed}
    assert _net(p, force=True).blob_need_backward == {"data": True, "label": False, **computed}


def test_need_backward_caffenet_train_val():
    p = P.read_net(os.path.join(GOLDEN, "models", "bvlc_reference_caffenet", "train_val.prototxt"))
    computed = ["conv1", "pool1", "norm1", "conv2", "pool2", "norm2", "conv3", "conv4", "conv5", "pool5", "fc6", "fc7",
                "fc8", "loss"]
    for force in (False, True):
        net = _net(p, force=force)
        want = {"data": force, "label": False, **{b: True for b in computed}}
        assert net.blob_need_backward == want, force
        assert net._grad_leaves == ({"data"} if force else set())


EUCLID = """
name: "euclid"
input: "x"
input_dim: 2 input_dim: 3 input_dim: 1 input_dim: 1
input: "t"
input_dim: 2 input_dim: 3 input_dim: 1 input_dim: 1
layers { name: "rx" type: RELU bottom: "x" top: "rx" }
layers { name: "st" type: SIGMOID bottom: "t" top: "st" }
layers { name: "loss" type: EUCLIDEAN_LOSS bottom: "rx" bottom: "st" top: "loss" }
"""


def test_need_backward_euclidean_forces_both_bottoms(tmp_path):
    """No parameters anywhere: nothing needs a diff, until force_backward marks both Euclidean bottoms (the loss layer
    allows it on both) and so both net inputs."""
    f = tmp_path / "euclid.prototxt"
    f.write_text(EUCLID)
    p = P.read_net(str(f))
    assert _net(p, force=False).blob_need_backward == dict(x=False, t=False, rx=False, st=False, loss=False)
    net = _net(p, force=True)
    assert net.blob_need_backward == dict(x=True, t=True, rx=True, st=True, loss=False)
    x, t = torch.randn(2, 3, 1, 1, dtype=torch.float64).float(), torch.randn(2, 3, 1, 1).float()
    loss, _ = net.forward({"x": x, "t": t})
    diffs = net.backward()
    x64, t64 = x.double().requires_grad_(True), t.double().requires_grad_(True)
    ref = ((x64.relu() - t64.sigmoid()) ** 2).sum() / (2 * 2)
    ref.backward()
    assert set(diffs) == {"x", "t"}
    torch.testing.assert_close(diffs["x"].double(), x64.grad, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(diffs["t"].double(), t64.grad, rtol=1e-5, atol=1e-6)
    assert not x.requires_grad and not t.requires_grad          # the caller's tensors are not touched


def test_backward_rejects_bad_seeds(tmp_path):
    f = tmp_path / "euclid.prototxt"
    f.write_text(EUCLID)
    net = _net(P.read_net(str(f)), force=True)
    net.forward({"x": torch.randn(2, 3, 1, 1), "t": torch.randn(2, 3, 1, 1)})
    with pytest.raises(ValueError, match="not a blob"):
        net.backward({"nope": torch.zeros(2, 3, 1, 1)})
    with pytest.raises(ValueError, match="shape"):
        net.backward({"rx": torch.zeros(2, 3, 2, 1)})


# ------------------------------------------------------------------------------------------------ engines agree
def _lmdb(tmp_path, channels, hw, n=16, classes=8):
    from poseidon_b200.data.lmdb_writer import write_lmdb
    rng = np.random.RandomState(0)
    recs = []
    for i in range(n):
        dt = P.Datum(channels=channels, height=hw, width=hw, label=int(rng.randint(0, classes)))
        dt.data = rng.randint(0, 256, size=(channels, hw, hw)).astype(np.uint8).tobytes()
        recs.append((b"%08d" % i, dt.SerializeToString()))
    path = str(tmp_path / f"db{channels}_{hw}")
    write_lmdb(path, recs)
    return path


# (name, image channels, stored size, crop, conv1 kernel / stride / pad / outputs, mode the sm100 engine picks)
FIRST_LAYERS = [
    ("lenet", 1, 28, 0, 5, 1, 0, 20, "pad8"),          # LeNet conv1: 1 -> 20 channels (8-channel pad)
    ("s2d", 3, 44, 35, 11, 4, 2, 16, "s2d"),           # AlexNet conv1 geometry: 11x11 / 4, space-to-depth
    ("row", 3, 44, 33, 7, 2, 3, 16, "row"),            # GoogLeNet conv1 geometry: 7x7 / 2 pad 3, ROW gather
]


def _first_layer_net(db, channels, crop, k, stride, pad, nout, deploy_hw=None):
    b = NetBuilder("first")
    if deploy_hw is None:
        b.data(db, 4, crop=crop, mirror=True, mean_values=[100.0] * channels, scale=0.02)
    g = {"type": "gaussian", "std": 0.05}
    b.conv("conv1", "data", nout, k, stride=stride, pad=pad, wf=g, bf={"type": "constant", "value": 0.1})
    if deploy_hw is None:
        b.pool("pool1", "conv1", "MAX", 2, 2)
    b.fc("fc", "pool1" if deploy_hw is None else "conv1", 8, wf=g, bf={"type": "constant", "value": 0.0})
    if deploy_hw is None:
        b.softmax_loss("loss", "fc")
    else:
        b.layer("prob", "SOFTMAX", ("fc",), ("prob",))
        b.net.input.append("data")
        for d in (2, channels, deploy_hw, deploy_hw):
            b.net.input_dim.append(d)
    b.net.force_backward = True
    return b.net


def _bf16_weights(net):
    """Round every parameter to bf16 in place: the torch engine then computes with the operands the kernels read."""
    with torch.no_grad():
        for p in net.params:
            p.copy_(p.to(BF16).float())


def _conv1_dgrad_ref(net, dy):
    """float64 data gradient of conv1 (transposed convolution) and the magnitude for its bound."""
    layer = net.layer_by_name["conv1"]
    w64 = torch.from_numpy(layer.export_blob(0)).double()
    shape = tuple(net.blob_shapes["data"])
    dx = torch.nn.grad.conv2d_input(shape, w64, dy.double(), layer.stride, layer.pad)
    mag = torch.nn.grad.conv2d_input(shape, w64.abs(), dy.double().abs(), layer.stride, layer.pad)
    return dx, C_GEMM * layer.kernel[0] * layer.kernel[1] * layer.num_output * U * mag


@pytest.mark.parametrize("case", FIRST_LAYERS, ids=[c[0] for c in FIRST_LAYERS])
def test_data_diff_engines_agree(emu, tmp_path, case):
    """force_backward: Net.backward seeded at conv1's top returns the image diff through the data layer's hand-off of
    the physical layout (sm100) and the logical blob (torch); both are float32 [N, C, H, W] and agree with each other
    and with float64 within the bf16 bound of a conv data gradient.  The loss-driven backward agrees as well."""
    name, channels, hw, crop, k, stride, pad, nout, mode = case
    db = _lmdb(tmp_path, channels, hw)
    p = _first_layer_net(db, channels, crop, k, stride, pad, nout)
    nets = {e: _net(p, engine=e) for e in ("torch", "sm100")}
    _bf16_weights(nets["torch"])
    nets["sm100"].copy_trained_layers_from(nets["torch"].to_proto())
    st = nets["sm100"].layer_by_name["conv1"]._sm100
    assert (st.s2d, st.row_mode and not st.pad8 and not st.s2d, st.pad8) == (mode == "s2d", mode == "row", mode == "pad8")
    assert nets["sm100"].layers[0].first_conv is nets["sm100"].layer_by_name["conv1"]
    shape = tuple(nets["torch"].blob_shapes["data"])
    dy = (torch.randn(tuple(nets["torch"].blob_shapes["conv1"]), generator=torch.Generator().manual_seed(3))).to(BF16)
    got = {}
    for e, net in nets.items():
        net.forward()
        if e == "sm100":
            assert tuple(net.blobs["data"].shape) != shape         # the data layer handed over the physical layout
        assert net.blobs["data"].requires_grad and not net.blobs["label"].requires_grad
        got[e] = net.backward({"conv1": dy.float() if e == "torch" else dy})["data"]
        assert got[e].dtype == torch.float32 and tuple(got[e].shape) == shape
    ref, e = _conv1_dgrad_ref(nets["torch"], dy)
    bound = _bf16_bound(ref, e)
    _within(got["torch"], ref, bound, f"{name}: torch engine data diff")
    _within(got["sm100"], ref, bound, f"{name}: sm100 engine data diff")
    _within(got["sm100"], got["torch"].double(), 2 * bound, f"{name}: engines")
    # from the loss: bf16 activations upstream of conv1 (and max-pooling choices that may flip with them), so the engines
    # agree in norm only (a sanity check: the seeded comparison above is the exact one)
    for net in nets.values():
        net.forward()
    a, b = (nets[e].backward()["data"] for e in ("torch", "sm100"))
    assert torch.isfinite(b).all() and float(a.norm()) > 0
    assert float((a - b).norm()) <= 0.15 * float(a.norm()), float((a - b).norm() / a.norm())


@pytest.mark.parametrize("case", FIRST_LAYERS, ids=[c[0] for c in FIRST_LAYERS])
def test_deploy_net_prob_seed_matches_float64(emu, case):
    """A deploy net (``input:``, no loss; conv1 -> fc -> softmax, nothing piecewise) with force_backward: Net.backward({"prob": onehot}) returns the input diff, equal
    to float64 autograd through the same (bf16) weights within the bf16 bound of the conv data gradient widened by the
    bf16 roundings of the layers above it."""
    name, channels, hw, crop, k, stride, pad, nout, mode = case
    crop = crop or hw
    p = _first_layer_net(None, channels, crop, k, stride, pad, nout, deploy_hw=crop)
    net = _net(p, engine="sm100", phase=P.TEST)
    ref_net = _net(p, engine="torch", phase=P.TEST)
    _bf16_weights(ref_net)
    net.copy_trained_layers_from(ref_net.to_proto())
    st = net.layer_by_name["conv1"]._sm100
    assert (st.s2d, st.row_mode and not st.pad8 and not st.s2d, st.pad8) == (mode == "s2d", mode == "row", mode == "pad8")
    x = torch.randn(2, channels, crop, crop, generator=torch.Generator().manual_seed(8)).to(BF16).float()
    onehot = torch.zeros(2, 8, 1, 1)
    onehot[0, 3] = onehot[1, 5] = 1.0
    net.forward({"data": x})
    got = net.backward({"prob": onehot})["data"]
    assert got.dtype == torch.float32 and tuple(got.shape) == tuple(x.shape)

    conv, fc = ref_net.layer_by_name["conv1"], ref_net.layer_by_name["fc"]
    w1, b1 = (torch.from_numpy(conv.export_blob(j)).double() for j in (0, 1))
    w2, b2 = (torch.from_numpy(fc.export_blob(j)).double().reshape(8, -1) for j in (0, 1))
    x64 = x.double().requires_grad_(True)
    y1 = F.conv2d(x64, w1, b1.reshape(-1), conv.stride, conv.pad)
    y1.retain_grad()
    prob = torch.softmax(y1.reshape(2, -1) @ w2.t() + b2.reshape(-1), dim=1)
    prob.backward(onehot.double().reshape(2, 8))
    dy = y1.grad
    mag = torch.nn.grad.conv2d_input(tuple(x.shape), w1.abs(), dy.abs(), conv.stride, conv.pad)
    # conv dgrad's bound plus 2^-8 relative per bf16 rounding of the activations / diffs above conv1 (softmax, fc, conv1)
    bound = _bf16_bound(x64.grad, C_GEMM * k * k * nout * U * mag) + 8 * 2.0 ** -8 * mag
    _within(got, x64.grad.detach(), bound, f"{name}: deploy input diff")


# ------------------------------------------------------------------------------------------------ first_layer_diff
@pytest.mark.parametrize("mode,pad", [(m, p) for m in ("s2d", "row") for p in range(4)] + [("pad8", 0)])
@pytest.mark.parametrize("hw", [(13, 13), (9, 14), (16, 11)])
def test_first_layer_diff_inverts_transform(emu, mode, pad, hw):
    """transform_nhwc's s2d / ROW / pad8 layout, then first_layer_diff: the identity, bit for bit (odd sizes, odd widths,
    paddings 0-3), and the float32 and bf16 outputs hold the same values."""
    k = emu.K()
    oh, ow = hw
    c = 1 if mode == "pad8" else 3
    n = 2
    x = torch.randn(n, c, oh, ow, generator=torch.Generator().manual_seed(oh * 31 + ow + pad)).to(BF16).float()
    zero = torch.zeros(n, dtype=torch.int32)
    flip = torch.zeros(n, dtype=torch.uint8)
    if mode == "s2d":
        hq, wq = -(-(oh + 2 * pad) // 4), -(-(ow + 2 * pad) // 4)
        phys = k.transform_nhwc(x, zero, zero, flip, None, 1.0, oh, ow, 4, pad, 4 * wq - ow - 2 * pad,
                                4 * hq - oh - 2 * pad, True)
        assert tuple(phys.shape) == (n, 64, hq, wq)
    elif mode == "row":
        phys = k.transform_nhwc(x, zero, zero, flip, None, 1.0, oh, ow, 4, pad, (ow + 2 * pad) % 2, 0, False)
    else:                                   # (the 8-channel layout carries no spatial padding)
        phys = k.transform_nhwc(x, zero, zero, flip, None, 1.0, oh, ow, 8, 0, 0, 0, False)
    back = k.first_layer_diff(phys, c, oh, ow, pad, pad, mode == "s2d", True)
    assert back.dtype == torch.float32 and back.is_contiguous()
    assert torch.equal(back, x)
    back16 = k.first_layer_diff(phys, c, oh, ow, pad, pad, mode == "s2d", False)
    assert back16.dtype == BF16 and torch.equal(back16.float(), x)


# ------------------------------------------------------------------------------------------------ nothing changes when off
def test_force_backward_off_makes_no_leaves(emu, tmp_path):
    db = _lmdb(tmp_path, 3, 44)
    p = _first_layer_net(db, 3, 35, 11, 4, 2, 16)
    for e in ("torch", "sm100"):
        net = _net(p, engine=e, force=False)
        assert not any(net.blob_need_backward[b] for b in ("data", "label"))
        net.forward()
        assert not net.blobs["data"].requires_grad and not net.blobs["label"].requires_grad
        assert net.backward() == {}
        assert net.layer_by_name["conv1"].weight.grad is not None      # the loss was backpropagated


@pytest.mark.parametrize("engine", ["torch", "sm100"])
def test_solver_trains_force_backward_net(emu, tmp_path, engine):
    """Training a force_backward net computes the image diff and drops it: the losses and weights are those of the same
    net without force_backward, bit for bit."""
    from poseidon_b200 import get_solver
    from smallnet import small_solver_param
    db = _lmdb(tmp_path, 3, 44)
    out = {}
    for force in (False, True):
        p = _first_layer_net(db, 3, 33, 7, 2, 3, 16)
        p.force_backward = force
        sp = small_solver_param(p, max_iter=3)
        sp.solver_mode = "CPU"                 # the emulated engine runs on the CPU on a GPU machine as well
        s = get_solver(sp, engine=engine, dtype=torch.float32 if engine == "torch" else None)
        losses = []
        for _ in range(3):
            s.step(1)
            losses.append(float(s.last_loss))
        out[force] = (losses, {n: l.export_blob(j) for n, l in zip(s.net.layer_names, s.net.layers)
                               for j in range(len(l.blobs))})
        s.close()
    assert out[True][0] == out[False][0]
    for n, w in out[False][1].items():
        assert np.array_equal(w, out[True][1][n]), n
