"""The sm100 engine's Python side, exercised on the CPU.

``ops/emulate.py`` stands in for the CUDA kernels (same op surface, same operand layouts), so everything AROUND the
kernels runs here: operand layouts per first-layer mode, bf16 shadows vs fp32 masters, the epilogue-fusion plan, the
single-process FusedBackend path, (h, w, c) inner-product weights and their checkpoint conversion.  The kernels
themselves are tested on an H100 (tests/test_ops_gpu.py, test_engine_gpu.py)."""
import numpy as np
import pytest
import torch

from smallnet import feed, make_data, small_net, small_solver_param


@pytest.fixture
def emu():
    from poseidon_b200.ops import counting, sm100
    sm100.set_emulation(True)
    counting.reset()
    yield sm100
    sm100.set_emulation(False)


def _run(engine, steps, solver_type="SGD", momentum=0.9, net_fn=None, batch=8, hw=35, classes=16):
    from poseidon_b200 import get_solver
    net = (net_fn or (lambda: small_net(batch=batch, hw=hw, classes=classes)))()
    sp = small_solver_param(net, max_iter=steps, solver_type=solver_type, momentum=momentum)
    s = get_solver(sp, engine=engine, dtype=torch.float32 if engine == "torch" else None)
    x, y = make_data(batch * steps, hw=hw, classes=classes)
    feed(s, x, y)
    losses = []
    for _ in range(steps):
        s.step(1)
        losses.append(float(s.last_loss))
    weights = {f"{n}.{j}": l.export_blob(j) for n, l in zip(s.net.layer_names, s.net.layers)
               for j in range(len(l.blobs))}
    return losses, weights, s


def _close(l_ref, l_sm, w_ref, w_sm, const_bias=()):
    for a, b in zip(l_ref, l_sm):
        assert abs(a - b) < 0.05 * max(1.0, abs(a)), (l_ref, l_sm)
    for name in w_ref:
        d = np.abs(w_ref[name] - w_sm[name]).max()
        init = 0.1 if name in const_bias else 0.0
        mm = np.abs(w_ref[name] - init).max() if name.endswith(".1") else np.abs(w_ref[name]).max()
        assert d <= 0.08 * mm + 3e-4, f"{name}: max diff {d} vs magnitude {mm}"


def test_emulation_is_explicit():
    """Without the switch the engine refuses to run on a CPU (no silent fallback)."""
    from poseidon_b200 import get_solver
    from poseidon_b200.ops import sm100
    assert not sm100.emulating()
    sp = small_solver_param(small_net(batch=4), max_iter=1)
    with pytest.raises(RuntimeError, match="CUDA device"):
        get_solver(sp, engine="sm100")


@pytest.mark.parametrize("solver_type,momentum", [("SGD", 0.9), ("NESTEROV", 0.9), ("ADAGRAD", 0.0)])
def test_engine_matches_fp32_engine(emu, solver_type, momentum):
    steps = 3
    l_ref, w_ref, _ = _run("torch", steps, solver_type, momentum)
    l_sm, w_sm, s = _run("sm100", steps, solver_type, momentum)
    assert type(s.sync.backend).__name__ == "FusedBackend"
    # conv1 (3 input channels, 5x5/s2) runs in ROW mode; ReLUs after conv / IP are folded into epilogues
    st = s.net.layer_by_name["conv1"]._sm100
    assert st.row_mode and not st.s2d and not st.pad8
    assert sum(s.net.skip_layer) >= 4
    if solver_type != "ADAGRAD":     # first AdaGrad steps are ±lr·sign(g): dominated by bf16 sign flips
        _close(l_ref, l_sm, w_ref, w_sm, const_bias=("conv1.1", "conv2.1", "fc4.1"))
    else:
        for a, b in zip(l_ref, l_sm):
            assert abs(a - b) < 0.05 * max(1.0, abs(a))


def _first_layer_net(k, stride, pad, hw, batch=4, classes=8):
    from poseidon_b200.models.zoo import NetBuilder
    b = NetBuilder("firstlayer")
    b.layer("data", "MEMORY_DATA", (), ("data", "label"),
            memory_data_param={"batch_size": batch, "channels": 3, "height": hw, "width": hw})
    g = {"type": "gaussian", "std": 0.05}
    b.conv("conv1", "data", 32, k, stride=stride, pad=pad, wf=g, bf={"type": "constant", "value": 0.1})
    b.relu("relu1", "conv1")
    b.pool("pool1", "conv1", "MAX", 3, 2)
    b.conv("conv2", "pool1", 48, 3, pad=1, wf=g, bf={"type": "constant", "value": 0.0})
    b.relu("relu2", "conv2")
    b.conv("conv3", "conv2", 32, 3, pad=1, group=1, wf=g, bf={"type": "constant", "value": 0.0})
    b.relu("relu3", "conv3")
    b.pool("pool3", "conv3", "AVE", 2, 2)
    b.fc("fc4", "pool3", classes, wf=g, bf={"type": "constant", "value": 0.0})
    b.softmax_loss("loss", "fc4")
    return b.net


@pytest.mark.parametrize("mode,k,stride,pad,hw", [
    ("s2d", 11, 4, 0, 67),      # AlexNet / CaffeNet conv1 -> 3x3/s1 over 64 channels
    ("s2d", 11, 4, 2, 63),      # with padding (the transform / conversion writes it)
    ("pad8", 3, 1, 1, 24),      # VGG conv1_1: image padded to 8 channels, ordinary TAP conv
    ("row", 7, 2, 3, 37),       # GoogLeNet conv1: ROW-mode gather
])
def test_first_layer_modes(emu, mode, k, stride, pad, hw):
    fn = lambda: _first_layer_net(k, stride, pad, hw)   # noqa: E731
    l_ref, w_ref, _ = _run("torch", 2, net_fn=fn, batch=4, hw=hw, classes=8)
    l_sm, w_sm, s = _run("sm100", 2, net_fn=fn, batch=4, hw=hw, classes=8)
    st = s.net.layer_by_name["conv1"]._sm100
    assert {"s2d": st.s2d, "pad8": st.pad8, "row": st.row_mode and not st.s2d and not st.pad8}[mode]
    _close(l_ref, l_sm, w_ref, w_sm, const_bias=("conv1.1",))
    # the master weight keeps the reference's logical shape whatever the operand layout is
    assert tuple(s.net.layer_by_name["conv1"].weight.shape) == (32, 3, k, k)


def test_channel_padded_k(emu, monkeypatch):
    """POSEIDON_PAD_K=1: C_g = 48 is padded to 64 slots per tap in the fprop / wgrad operand and in the dgrad pack."""
    monkeypatch.setenv("POSEIDON_PAD_K", "1")
    fn = lambda: _first_layer_net(7, 2, 3, 37)   # noqa: E731
    l_ref, w_ref, _ = _run("torch", 2, net_fn=fn, batch=4, hw=37, classes=8)
    l_sm, w_sm, s = _run("sm100", 2, net_fn=fn, batch=4, hw=37, classes=8)
    st3 = s.net.layer_by_name["conv3"]._sm100          # 48 input channels
    assert (st3.cg, st3.cgk) == (48, 64)
    assert st3.operand().shape == (32, 9 * 64) and st3.shadow().shape == (32, 9 * 48)
    st2 = s.net.layer_by_name["conv2"]._sm100          # 48 output channels -> dgrad operand padded
    assert st2.cok == 64 and st2.dgrad_pack().shape == (32, 9 * 64)
    _close(l_ref, l_sm, w_ref, w_sm, const_bias=("conv1.1",))


def test_transform_layouts_match_conversion(emu):
    """What the transform op writes for a first layer == what prepare_first_layer_input derives from a plain batch."""
    from poseidon_b200 import proto as P
    from poseidon_b200.data.transformer import DataTransformer
    from poseidon_b200.ops import torch_engine as TE

    class Conv:                      # the attributes ConvState reads
        def __init__(self, k, stride, pad, in_hw):
            self.kernel, self.stride, self.pad, self.group, self.num_output = (k, k), (stride, stride), (pad, pad), 1, 16
            self.layer_name, self.in_hw = "conv1", in_hw
            self.weight = torch.nn.Parameter(torch.randn(16, 3, k, k))

    x = torch.randint(0, 256, (3, 3, 40, 40), dtype=torch.uint8)
    for k, stride, pad, crop in [(11, 4, 2, 35), (3, 1, 1, 32), (7, 2, 3, 33)]:
        tp = P.TransformationParameter(crop_size=crop, mirror=True, scale=0.017, mean_value=[104.0, 117.0, 123.0])
        conv = Conv(k, stride, pad, (crop, crop))
        st = emu.conv_state(conv, 3)
        outs = []
        for fn in (emu.transform, None):
            tr = DataTransformer(tp, P.TRAIN, torch.device("cpu"), seed=3)
            if fn is not None:
                outs.append(fn(tr, x, torch.bfloat16, first_conv=conv))
            else:
                plain = TE.transform(tr, x, torch.float32)
                outs.append(emu.prepare_first_layer_input(plain, st, conv.pad, conv.in_hw))
        a, b = outs
        assert a.shape == b.shape and a.dtype == b.dtype == torch.bfloat16, (k, a.shape, b.shape)
        assert torch.equal(a.float(), b.float()), k
        # the transform's output is accepted as-is (no second conversion pass)
        assert emu.prepare_first_layer_input(a, st, conv.pad, conv.in_hw) is a


def test_shadows_are_not_rederived_every_step(emu):
    """The optimizer op refreshes the bf16 operand next to the fp32 master; the layer state must not convert the
    whole weight again on the next forward (a regression here costs ~7 % of an AlexNet step on the GPU)."""
    from poseidon_b200.ops import counting
    _, _, s = _run("sm100", 2)
    for name in ("conv2", "conv3", "fc4", "fc5"):
        st = s.net.layer_by_name[name]._sm100
        assert st.wb is not None and not st.dirty_wb, name
        master = s.net.layer_by_name[name].weight.data
        flat = master.permute(0, 2, 3, 1).reshape(st.wb.shape) if master.dim() == 4 else master
        assert torch.equal(st.wb.float(), flat.to(torch.bfloat16).float()), name
    counting.reset()
    s.step(1)
    ops = counting.by_op()
    n_params = sum(len(l.blobs) for l in s.net.layers)
    # every blob stepped exactly once: the two IP weights by their own wgrad GEMM + update pair, all other blobs (8 of
    # the 10) by ONE multi-tensor launch at the end of the iteration
    assert ops["fused_update"] == 2 and ops["fused_update_multi"] == 1 and n_params == 10, ops
    assert ops["gemm_f32"] == 2, ops
    assert ops["conv_wgrad"] == 3 and ops["conv_fprop"] == 3, ops
    # both data gradients read the fprop weights in place: no packed transposed copy, no pack launch per step
    assert ops.get("conv_dgrad_w", 0) == 2 and "conv_dgrad" not in ops and "conv_pack_dgrad" not in ops, ops
    assert "relu_fwd" not in ops, ops        # all four ReLUs live in epilogues
    for name in ("conv2", "conv3", "fc4", "fc5"):
        assert not s.net.layer_by_name[name]._sm100.dirty_wb


def test_snapshot_roundtrip_between_engines(emu, tmp_path):
    """Checkpoints are engine-neutral: (h, w, c) inner-product weights and channels-last conv weights are converted at
    the file boundary."""
    from poseidon_b200 import get_solver
    net = small_net(batch=8)
    sp = small_solver_param(net, max_iter=2)
    sp.snapshot_prefix = str(tmp_path / "small")
    s = get_solver(sp, engine="sm100")
    x, y = make_data(32)
    feed(s, x, y)
    s.step(2)
    s.snapshot()
    assert s.net.layer_by_name["fc4"]._sm100.perm is not None
    ref = {n: l.export_blob(0) for n, l in zip(s.net.layer_names, s.net.layers) if len(l.blobs)}
    s2 = get_solver(sp, engine="torch", dtype=torch.float32)
    s2.restore(str(tmp_path / "small_iter_2.solverstate"))
    for n, l in zip(s2.net.layer_names, s2.net.layers):
        if len(l.blobs):
            assert np.allclose(l.export_blob(0), ref[n], atol=1e-6), n
    assert s2.iter == 2
    # and back: the sm100 engine resumes from the fp32 engine's file and both take the same next step
    feed(s2, x, y)
    s2.step(1)
    s2.snapshot()
    s3 = get_solver(sp, engine="sm100")
    s3.restore(str(tmp_path / "small_iter_3.solverstate"))
    for n, l in zip(s3.net.layer_names, s3.net.layers):
        if len(l.blobs):
            assert np.allclose(l.export_blob(0), s2.net.layer_by_name[n].export_blob(0), atol=1e-6), n
    st = s3.net.layer_by_name["conv2"]._sm100
    assert torch.equal(st.shadow().float(), st.w2d().to(torch.bfloat16).float())


def _inception_net(batch=4, hw=20, classes=8):
    from poseidon_b200.models.zoo import NetBuilder
    b = NetBuilder("miniception")
    b.layer("data", "MEMORY_DATA", (), ("data", "label"),
            memory_data_param={"batch_size": batch, "channels": 3, "height": hw, "width": hw})
    g = {"type": "gaussian", "std": 0.08}
    z = {"type": "constant", "value": 0.0}
    b.conv("conv1", "data", 32, 3, stride=2, pad=1, wf=g, bf=z)
    b.relu("relu1", "conv1")
    b.conv("b1", "conv1", 16, 1, wf=g, bf=z)
    b.relu("b1r", "b1")
    b.conv("b2r", "conv1", 16, 1, wf=g, bf=z)
    b.relu("b2rr", "b2r")
    b.conv("b2", "b2r", 24, 3, pad=1, wf=g, bf=z)
    b.relu("b2relu", "b2")
    b.pool("b3p", "conv1", "MAX", 3, 1, pad=1)
    b.conv("b3", "b3p", 8, 1, wf=g, bf=z)
    b.relu("b3r", "b3")
    b.layer("cat", "CONCAT", ("b1", "b2", "b3"), ("cat",))
    b.pool("gap", "cat", "AVE", 10, 1)
    b.dropout("drop", "gap", 0.4)
    b.fc("fc", "gap", classes, wf=g, bf=z)
    b.softmax_loss("loss", "fc")
    return b.net


def test_inception_block_with_concat_and_dropout(emu):
    """Branches, CONCAT, global AVE pooling and dropout: the loss falls and the gradient reaches every branch."""
    from poseidon_b200 import get_solver
    sp = small_solver_param(_inception_net(), base_lr=0.05, max_iter=12)
    s = get_solver(sp, engine="sm100")
    x, y = make_data(4, classes=8, hw=20)
    before = {n: l.export_blob(0).copy() for n, l in zip(s.net.layer_names, s.net.layers) if len(l.blobs)}
    losses = []
    for _ in range(12):
        feed(s, x, y)                  # the same 4 images every step: the net must memorise them
        s.step(1)
        losses.append(float(s.last_loss))
    assert losses[-1] < 0.88 * losses[0] and all(b < a + 0.05 for a, b in zip(losses, losses[1:])), losses
    for n, l in zip(s.net.layer_names, s.net.layers):
        if len(l.blobs):
            assert np.abs(l.export_blob(0) - before[n]).max() > 0, f"{n} never updated"
    # dropout masks differ between iterations (device-resident iteration counter) but repeat within one
    d = emu.dropout(torch.ones(2, 8, 2, 2, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last), 0.5, True)
    emu.bump_iteration_seed(torch.device("cpu"))
    e = emu.dropout(torch.ones(2, 8, 2, 2, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last), 0.5, True)
    assert set(d.float().unique().tolist()) <= {0.0, 2.0} and not torch.equal(d, e)


@pytest.mark.parametrize("name,steps", [("alexnet", 3), ("caffenet", 2), ("googlenet", 3), ("vgg16", 2)])
def test_zoo_models_follow_fp32_engine(emu, name, steps):
    """The reference's ImageNet models, full size (batch 2, synthetic data), dropout neutralised: the sm100 engine's
    loss trajectory (space-to-depth conv1, fused ReLU / LRN masks, CONCAT slices, auxiliary losses) tracks fp32."""
    from poseidon_b200 import get_solver
    from poseidon_b200.models import zoo

    def run(engine):
        nb = 1 if name == "vgg16" else 2                      # (VGG-16 on a CPU: keep it to one image)
        net = getattr(zoo, name)(batch=nb, test_batch=nb)
        for l in net.layers:
            if l.enum_name("type") == "DROPOUT":
                l.dropout_param.dropout_ratio = 1e-7
        sp = zoo.get_solver_param(name, net=net, display=0, snapshot=0, snapshot_after_train=False, test_interval=0,
                                  max_iter=steps, random_seed=3)
        sp.clear("test_iter")
        sp.base_lr = 0.001
        s = get_solver(sp, engine=engine, dtype=torch.float32 if engine == "torch" else None)
        out = []
        for _ in range(steps):
            s.step(1)
            out.append(float(s.last_loss))
        s.close()
        return out, s

    l_sm, s = run("sm100")
    l_ref, _ = run("torch")
    if name == "vgg16":
        assert s.net.layer_by_name["conv1_1"]._sm100.pad8             # 3x3 / s1 first layer: image padded to 8 channels
    elif name != "googlenet":
        assert s.net.layer_by_name["conv1"]._sm100.s2d
    for a, b in zip(l_ref, l_sm):
        assert abs(a - b) < 0.01 * abs(a), (l_ref, l_sm)


def _odd_channel_net(batch=4, hw=12, classes=10):
    """Channel counts that are not multiples of 8 everywhere (LeNet-like 20 / 50, K = 180, N = 30 / 10)."""
    from poseidon_b200.models.zoo import NetBuilder
    b = NetBuilder("oddnet")
    b.layer("data", "MEMORY_DATA", (), ("data", "label"),
            memory_data_param={"batch_size": batch, "channels": 3, "height": hw, "width": hw})
    g = {"type": "gaussian", "std": 0.1}
    c = {"type": "constant", "value": 0.1}
    b.conv("conv1", "data", 20, 5, pad=2, wf=g, bf=c)
    b.relu("relu1", "conv1")
    b.pool("pool1", "conv1", "MAX", 2, 2)
    b.conv("conv2", "pool1", 50, 3, pad=1, wf=g, bf=c)
    b.relu("relu2", "conv2")
    b.conv("conv3", "conv2", 20, 1, wf=g, bf=c)
    b.relu("relu3", "conv3")
    b.pool("pool3", "conv3", "AVE", 2, 2)
    b.fc("ip1", "pool3", 30, wf=g, bf=c)
    b.relu("relu4", "ip1")
    b.fc("ip2", "ip1", classes, wf=g, bf=c)
    b.softmax_loss("loss", "ip2")
    return b.net


def test_channel_counts_not_multiples_of_8(emu):
    """The kernels want channel counts (and inner-product K) in multiples of 8; other nets are zero-padded around them."""
    fn = _odd_channel_net
    l_ref, w_ref, _ = _run("torch", 3, net_fn=fn, batch=4, hw=12, classes=10)
    l_sm, w_sm, s = _run("sm100", 3, net_fn=fn, batch=4, hw=12, classes=10)
    L = s.net.layer_by_name
    st1, st2, st3 = (L[n]._sm100 for n in ("conv1", "conv2", "conv3"))
    assert (st1.Cp, st1.Coutp, st2.Cp, st2.Coutp, st3.Cp, st3.Coutp) == (8, 24, 24, 56, 56, 24)
    assert st2.shadow().shape == (56, 9 * 24) and st2.dgrad_pack().shape == (24, 9 * 56)
    assert not st1.consumer_masks and not st2.consumer_masks          # masks stay with the producer for such layers
    assert (L["ip1"]._sm100.K, L["ip1"]._sm100.Kp) == (180, 184) and L["ip1"]._sm100.shadow().shape == (30, 184)
    assert (L["ip2"]._sm100.K, L["ip2"]._sm100.Kp) == (30, 32)
    assert tuple(s.net.blobs["conv2"].shape) == (4, 50, 6, 6)           # logical shapes are the reference's
    assert tuple(L["conv2"].weight.shape) == (50, 20, 3, 3) and tuple(L["ip1"].weight.shape) == (30, 180)
    _close(l_ref, l_sm, w_ref, w_sm, const_bias=("conv1.1", "conv2.1", "conv3.1", "ip1.1", "ip2.1"))


@pytest.mark.parametrize("name", ["lenet", "cifar10_quick"])
def test_small_zoo_models_follow_fp32_engine(emu, name):
    """examples/mnist and examples/cifar10 of the reference, on the sm100 engine (LeNet: 1 -> 20 -> 50 channels, K = 500)."""
    from poseidon_b200 import get_solver
    from poseidon_b200.models import zoo

    def run(engine):
        net = getattr(zoo, name)(batch=8)
        sp = zoo.get_solver_param(name, net=net, display=0, snapshot=0, snapshot_after_train=False, test_interval=0,
                                  max_iter=4, random_seed=3)
        sp.clear("test_iter")
        s = get_solver(sp, engine=engine, dtype=torch.float32 if engine == "torch" else None)
        out = []
        for _ in range(4):
            s.step(1)
            out.append(float(s.last_loss))
        s.close()
        return out

    l_sm, l_ref = run("sm100"), run("torch")
    for a, b in zip(l_ref, l_sm):
        assert abs(a - b) < 0.02 * max(1.0, abs(a)), (l_ref, l_sm)


def test_train_snapshot_then_extract_features_both_engines(emu, tmp_path):
    """caffe_main train on the sm100 engine -> .caffemodel -> tools.extract_features on either engine: the feature
    databases hold the same logical (C, H, W) datums (LeNet: channel-sliced 20 / 50-channel blobs, K-padded ip2)."""
    from poseidon_b200 import proto as P
    from poseidon_b200.data.db import open_db
    from poseidon_b200.models import zoo
    from poseidon_b200.tools import caffe_main, extract_features
    net_path = tmp_path / "lenet.prototxt"
    P.write_text(str(net_path), zoo.lenet(batch=8, test_batch=8))
    sp = zoo.lenet_solver(net_path=str(net_path), max_iter=3, display=0, test_interval=0, solver_mode="CPU", snapshot=3,
                          snapshot_prefix=str(tmp_path / "lenet"))
    sp.clear("test_iter")
    solver_path = tmp_path / "solver.prototxt"
    P.write_text(str(solver_path), sp)
    assert caffe_main.main(["train", f"--solver={solver_path}", "--engine=sm100"]) == 0
    weights = str(tmp_path / "lenet_iter_3.caffemodel")
    for eng in ("sm100", "torch"):
        extract_features.main([weights, str(net_path), "conv2,ip1", f"{tmp_path}/{eng}_conv2,{tmp_path}/{eng}_ip1", "1",
                               "--gpu", "-1", "--engine", eng])
    for blob, shape in (("conv2", (50, 8, 8)), ("ip1", (500, 1, 1))):
        a, b = open_db(f"{tmp_path}/sm100_{blob}_0_0"), open_db(f"{tmp_path}/torch_{blob}_0_0")
        assert len(a) == len(b) == 8
        for i in range(len(a)):
            da, db = a.datum(i), b.datum(i)
            assert (da.channels, da.height, da.width) == (db.channels, db.height, db.width) == shape
            fa, fb = np.array(da.float_data), np.array(db.float_data)
            assert np.abs(fa - fb).max() <= 0.02 * max(1.0, np.abs(fb).max()), blob


# ---------------------------------------------------------------------------------------------------------------
# The layer catalogue beyond the ImageNet models (siamese / autoencoder style nets) on bf16 activations
def _lt_base(b, batch=4, hw=12):
    b.layer("data", "MEMORY_DATA", (), ("data", "label"), memory_data_param={"batch_size": batch, "channels": 3, "height": hw, "width": hw})
    g = {"type": "gaussian", "std": 0.1}
    b.conv("conv1", "data", 16, 3, pad=1, wf=g, bf={"type": "constant", "value": 0.1})
    return g

def _lt_neurons():
    from poseidon_b200.models.zoo import NetBuilder
    b = NetBuilder("neurons"); g = _lt_base(b)
    x = "conv1"
    for i, (t, kw) in enumerate([("SIGMOID", {}), ("TANH", {}), ("ABSVAL", {}), ("BNLL", {}), ("POWER", {"power_param": {"power": 2.0, "scale": 0.5, "shift": 0.1}})]):
        b.layer(f"n{i}", t, (x,), (f"n{i}",), **kw); x = f"n{i}"
    b.pool("pool", x, "MAX", 2, 2)
    b.fc("fc", "pool", 16, wf=g, bf={"type": "constant", "value": 0.0})
    b.softmax_loss("loss", "fc")
    return b.net

def _lt_eltwise():
    from poseidon_b200.models.zoo import NetBuilder
    b = NetBuilder("elt"); g = _lt_base(b)
    b.layer("slice", "SLICE", ("conv1",), ("s1", "s2"), slice_param={"slice_dim": 1})
    b.layer("sum", "ELTWISE", ("s1", "s2"), ("sum",), eltwise_param={"operation": "SUM"})
    b.layer("mx", "ELTWISE", ("s1", "s2"), ("mx",), eltwise_param={"operation": "MAX"})
    b.layer("pr", "ELTWISE", ("sum", "mx"), ("pr",), eltwise_param={"operation": "PROD"})
    b.layer("cat", "CONCAT", ("pr", "s1"), ("cat",))
    b.layer("mvn", "MVN", ("cat",), ("mvn",))
    b.layer("flat", "FLATTEN", ("mvn",), ("flat",))
    b.fc("fc", "flat", 16, wf=g, bf={"type": "constant", "value": 0.0})
    b.softmax_loss("loss", "fc")
    return b.net

def _lt_losses(kind):
    from poseidon_b200.models.zoo import NetBuilder
    b = NetBuilder(kind); g = _lt_base(b)
    b.pool("pool", "conv1", "AVE", 4, 4)
    if kind == "EUCLIDEAN_LOSS":
        b.fc("fc", "pool", 1, wf=g, bf={"type": "constant", "value": 0.0})
        b.layer("loss", kind, ("fc", "label"), ("loss",))
    elif kind == "SIGMOID_CROSS_ENTROPY_LOSS":
        b.fc("fc", "pool", 1, wf=g, bf={"type": "constant", "value": 0.0})
        b.layer("thr", "THRESHOLD", ("label",), ("lab01",), threshold_param={"threshold": 7.5})
        b.layer("loss", kind, ("fc", "lab01"), ("loss",))
    elif kind == "HINGE_LOSS":
        b.fc("fc", "pool", 16, wf=g, bf={"type": "constant", "value": 0.0})
        b.layer("loss", kind, ("fc", "label"), ("loss",))
    elif kind == "MULTINOMIAL_LOGISTIC_LOSS":
        b.fc("fc", "pool", 16, wf=g, bf={"type": "constant", "value": 0.0})
        b.layer("prob", "SOFTMAX", ("fc",), ("prob",))
        b.layer("loss", kind, ("prob", "label"), ("loss",))
    elif kind == "CONTRASTIVE_LOSS":
        b.fc("fa", "pool", 8, wf=g, bf={"type": "constant", "value": 0.0})
        b.fc("fb", "pool", 8, wf={"type": "gaussian", "std": 0.2}, bf={"type": "constant", "value": 0.0})
        b.layer("thr", "THRESHOLD", ("label",), ("sim",), threshold_param={"threshold": 7.5})
        b.layer("loss", kind, ("fa", "fb", "sim"), ("loss",), contrastive_loss_param={"margin": 1.0})
    return b.net


@pytest.mark.parametrize("case", ["neurons", "eltwise", "EUCLIDEAN_LOSS", "SIGMOID_CROSS_ENTROPY_LOSS", "HINGE_LOSS",
                                  "MULTINOMIAL_LOGISTIC_LOSS", "CONTRASTIVE_LOSS"])
def test_layer_catalogue_on_sm100_engine(emu, case):
    from poseidon_b200 import get_solver
    from poseidon_b200.models.zoo import NetBuilder      # noqa: F401  (used by the builders above)
    fn = {"neurons": _lt_neurons, "eltwise": _lt_eltwise}.get(case, lambda: _lt_losses(case))
    out = {}
    for eng in ("torch", "sm100"):
        sp = small_solver_param(fn(), base_lr=0.01, max_iter=3)
        s = get_solver(sp, engine=eng, dtype=torch.float32 if eng == "torch" else None)
        x, y = make_data(12, hw=12)
        feed(s, x, y)
        out[eng] = []
        for _ in range(3):
            s.step(1)
            out[eng].append(float(s.last_loss))
        s.close()
    for a, b in zip(out["torch"], out["sm100"]):
        assert abs(a - b) <= 0.02 * max(1.0, abs(a)), out


@pytest.mark.parametrize("k,stride,pad,crop,mode", [(11, 4, 2, 35, "s2d"), (3, 1, 1, 32, "pad8"), (7, 2, 3, 33, "row"),
                                                   (5, 2, 0, 33, "row")])
def test_data_layer_hands_first_conv_its_layout(emu, tmp_path, k, stride, pad, crop, mode):
    """LMDB -> (native) batch loader -> transform op (random crop, mirror, mean, scale) writing the first
    convolution's operand layout directly -> conv.  Same crops as the fp32 engine (same seeded draws), same losses."""
    from poseidon_b200 import get_solver, proto as P
    from poseidon_b200.data.lmdb_writer import write_lmdb
    from poseidon_b200.models.zoo import NetBuilder
    rng = np.random.RandomState(0)
    recs = []
    for i in range(40):
        dt = P.Datum(channels=3, height=44, width=44, label=int(rng.randint(0, 8)))
        dt.data = rng.randint(0, 256, size=(3, 44, 44)).astype(np.uint8).tobytes()
        recs.append((b"%08d" % i, dt.SerializeToString()))
    write_lmdb(str(tmp_path / "db"), recs)

    def net():
        b = NetBuilder("d")
        b.data(str(tmp_path / "db"), 8, crop=crop, mirror=True, mean_values=[104, 117, 123], scale=0.02)
        g = {"type": "gaussian", "std": 0.05}
        b.conv("conv1", "data", 16, k, stride=stride, pad=pad, wf=g, bf={"type": "constant", "value": 0.1})
        b.relu("relu1", "conv1")
        b.pool("pool1", "conv1", "MAX", 2, 2)
        b.fc("fc", "pool1", 8, wf=g, bf={"type": "constant", "value": 0.0})
        b.softmax_loss("loss", "fc")
        return b.net

    out = {}
    for eng in ("torch", "sm100"):
        s = get_solver(small_solver_param(net(), base_lr=0.01, max_iter=3), engine=eng,
                       dtype=torch.float32 if eng == "torch" else None)
        out[eng] = []
        for _ in range(3):
            s.step(1)
            out[eng].append(float(s.last_loss))
        if eng == "sm100":
            st = s.net.layer_by_name["conv1"]._sm100
            assert ("s2d" if st.s2d else "pad8" if st.pad8 else "row") == mode
            assert s.net.layers[0].first_conv is s.net.layer_by_name["conv1"]
            from poseidon_b200.ops import counting
            assert counting.by_op().get("transform_nhwc", 0) >= 3
        s.close()
    for a, b in zip(out["torch"], out["sm100"]):
        assert abs(a - b) <= 0.02 * max(1.0, abs(a)), out


@pytest.mark.parametrize("engine", ["torch", "sm100"])
def test_learns_a_separable_task(emu, engine):
    """End-to-end sanity beyond "the loss goes down": a 4-class task (which quadrant holds the bright blob) is learnt to
    > 95 % held-out accuracy in 150 SGD steps by both engines, through the TEST-phase accuracy layer."""
    from poseidon_b200 import get_solver, proto as P
    from poseidon_b200.models.zoo import NetBuilder

    def data(n, seed):
        rng = np.random.RandomState(seed)
        y = rng.randint(0, 4, size=n)
        x = rng.randn(n, 1, 12, 12).astype(np.float32) * 0.3
        for i, c in enumerate(y):
            r0, c0 = (c // 2) * 6, (c % 2) * 6
            x[i, 0, r0 + 1: r0 + 5, c0 + 1: c0 + 5] += 1.5
        return torch.from_numpy(x), torch.from_numpy(y.astype(np.float32))

    b = NetBuilder("quadrants")
    b.layer("data", "MEMORY_DATA", (), ("data", "label"),
            memory_data_param={"batch_size": 32, "channels": 1, "height": 12, "width": 12})
    g = {"type": "xavier"}
    b.conv("conv1", "data", 8, 3, pad=1, wf=g, bf={"type": "constant", "value": 0.0})
    b.relu("relu1", "conv1")
    b.pool("pool1", "conv1", "MAX", 2, 2)
    b.fc("ip1", "pool1", 16, wf=g, bf={"type": "constant", "value": 0.0})
    b.relu("relu2", "ip1")
    b.fc("ip2", "ip1", 4, wf=g, bf={"type": "constant", "value": 0.0})
    b.accuracy("accuracy", "ip2")
    b.softmax_loss("loss", "ip2")
    sp = P.SolverParameter(base_lr=0.05, lr_policy="step", gamma=0.5, stepsize=60, momentum=0.9, weight_decay=1e-4,
                           display=0, max_iter=150, snapshot=0, snapshot_after_train=False, random_seed=5,
                           solver_mode="CPU", test_interval=1000)
    sp.test_iter = [4]
    sp.net_param = b.net
    s = get_solver(sp, engine=engine, dtype=torch.float32 if engine == "torch" else None)
    xtr, ytr = data(32 * 150, 1)
    xte, yte = data(32 * 4, 2)
    feed(s, xtr, ytr)
    for layer in s.test_nets[0].layers:
        if layer.type_name == "MEMORY_DATA":
            layer.reset(xte, yte)
    s.step(150)
    scores = s.test(0) if hasattr(s, "test") else None
    acc = None
    if isinstance(scores, dict):
        acc = scores.get("accuracy")
    if acc is None:                                   # evaluate by hand through the shared-weight test net
        net = s.test_nets[0]
        hits = 0
        with torch.no_grad():
            for _ in range(4):
                _, out = net.forward()
                hits += float(out["accuracy"]) * 32
        acc = hits / 128
    assert acc > 0.95, acc
    s.close()


@pytest.mark.parametrize("k,stride,pad,hw,groups", [(3, 2, 1, (9, 11), 1), (5, 2, 2, (12, 10), 1), (2, 2, 0, (8, 8), 1),
                                                     (1, 2, 0, (7, 9), 1), (3, 3, 1, (10, 10), 2), (7, 2, 3, (14, 14), 1),
                                                     (2, 3, 0, (9, 9), 1)])
def test_strided_conv_data_gradient(emu, k, stride, pad, hw, groups):
    """Strided convolutions inside a net (not only as first layer): the data gradient is assembled from sh * sw stride-1
    phase problems (ops/sm100.py::_strided_dgrad) and equals autograd through F.conv2d, also when the stride exceeds the
    kernel (phases without taps) and with groups."""
    from test_ops_gpu import _FakeLayer
    torch.manual_seed(k * 10 + stride)
    cin, cout = 16, 32
    layer = _FakeLayer.__new__(_FakeLayer)
    layer.layer_name, layer.num_output, layer.kernel, layer.stride, layer.pad = "conv", cout, (k, k), (stride, stride), (pad, pad)
    layer.group, layer.bias_term, layer.in_hw = groups, True, hw
    layer.weight = torch.nn.Parameter(torch.randn(cout, cin // groups, k, k) * 0.1)
    layer.bias = torch.nn.Parameter(torch.randn(cout) * 0.1)
    x = torch.randn(2, cin, *hw).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    xs = x.clone().requires_grad_(True)
    y = emu.conv2d(xs, layer.weight, layer.bias, layer.stride, layer.pad, groups, relu_slope=None, layer=layer)
    xr = x.float().requires_grad_(True)
    wr = layer.weight.detach().to(torch.bfloat16).float().requires_grad_(True)
    yr = torch.nn.functional.conv2d(xr, wr, layer.bias.detach(), stride, pad, 1, groups)
    assert tuple(y.shape) == tuple(yr.shape)
    dy = torch.randn_like(yr).to(torch.bfloat16)
    y.backward(dy.contiguous(memory_format=torch.channels_last))
    yr.backward(dy.float())
    err = (xs.grad.float() - xr.grad).abs().max().item()
    assert err <= 2e-2 * xr.grad.abs().max().item() + 1e-3, err
    werr = (layer.weight.grad.float() - wr.grad).abs().max().item()
    assert werr <= 3e-2 * wr.grad.abs().max().item() + 1e-3, werr
