"""fp8 (e4m3) forward convolutions: the opt-in ``fp8="fprop"`` engine setting.

CPU (no GPU needed): the eligibility rule on the zoo nets, the setting's plumbing through get_solver / CaffeEngine /
caffe_main, an emulated training step against the bf16 emulation, checkpoints, and the SASS of the built extension.
H100: the quantisers bit for bit against the torch reference, conv_fprop_fp8 against a float64 reference of the
dequantised operands, and whole nets (loss tracking, bit-for-bit repeatability, CUDA-graph replay)."""
import hashlib
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from smallnet import feed, make_data, small_solver_param

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "poseidon_b200", "_ext", "poseidon_b200_C.so")
GOLDEN_SASS = os.path.join(ROOT, "tests", "golden", "wgmma_bf16_sass.json")


@pytest.fixture(autouse=True)
def _keep_dropout_counters():
    """Nets built here (the zoo nets have dropout) advance the process-wide counters that key dropout masks: restore them,
    so that the tests after this file draw the masks they would draw without it."""
    from poseidon_b200.ops import sm100
    count, seeds = sm100._dropout_counter[0], {k: (t, t.clone()) for k, t in sm100._iter_seed.items()}
    yield
    sm100._dropout_counter[0] = count
    sm100._iter_seed.clear()
    for k, (t, v) in seeds.items():
        t.copy_(v)
        sm100._iter_seed[k] = t


@pytest.fixture
def emu():
    from poseidon_b200.ops import counting, sm100
    sm100.set_emulation(True)
    counting.reset()
    yield sm100
    sm100.set_emulation(False)


# ------------------------------------------------------------------------------------------------ small nets
def fp8_alex_net(batch=8, classes=16, hw=27):
    """AlexNet-shaped: a ROW-mode first layer and a 64-channel conv stay bf16; conv3 (Cg 128), the grouped conv4
    (Cg 96 -> 128 slots) and the stride-2 conv5 run in fp8."""
    from poseidon_b200.models.zoo import NetBuilder
    b = NetBuilder("fp8alex")
    b.layer("data", "MEMORY_DATA", (), ("data", "label"),
            memory_data_param={"batch_size": batch, "channels": 3, "height": hw, "width": hw})
    g = {"type": "gaussian", "std": 0.05}
    b.conv("conv1", "data", 64, 5, stride=2, wf=g, bf={"type": "constant", "value": 0.1})
    b.relu("relu1", "conv1")
    b.conv("conv2", "conv1", 128, 3, pad=1, wf=g, bf={"type": "constant", "value": 0.1})
    b.relu("relu2", "conv2")
    b.conv("conv3", "conv2", 192, 3, pad=1, wf=g, bf={"type": "constant", "value": 0.0})
    b.relu("relu3", "conv3")
    b.conv("conv4", "conv3", 128, 3, pad=1, group=2, wf=g, bf={"type": "constant", "value": 0.1})
    b.relu("relu4", "conv4")
    b.conv("conv5", "conv4", 128, 3, stride=2, pad=1, wf=g, bf={"type": "constant", "value": 0.0})
    b.relu("relu5", "conv5")
    b.pool("pool5", "conv5", "MAX", 2, 2)
    b.fc("fc6", "pool5", classes, wf=g, bf={"type": "constant", "value": 0.0})
    b.softmax_loss("loss", "fc6")
    return b.net


def fp8_inception_net(batch=8, classes=16, hw=19):
    """GoogLeNet-shaped: branch convolutions write straight into a concat slab (zero-copy), 1x1 and 3x3 fp8 layers."""
    from poseidon_b200.models.zoo import NetBuilder
    b = NetBuilder("fp8incep")
    b.layer("data", "MEMORY_DATA", (), ("data", "label"),
            memory_data_param={"batch_size": batch, "channels": 3, "height": hw, "width": hw})
    g = {"type": "gaussian", "std": 0.05}
    b.conv("conv1", "data", 96, 3, pad=1, wf=g, bf={"type": "constant", "value": 0.1})
    b.relu("relu1", "conv1")
    b.conv("a1x1", "conv1", 64, 1, wf=g, bf={"type": "constant", "value": 0.1})
    b.relu("relu_a", "a1x1")
    b.conv("b1x1", "conv1", 112, 1, wf=g, bf={"type": "constant", "value": 0.1})
    b.relu("relu_b1", "b1x1")
    b.conv("b3x3", "b1x1", 128, 3, pad=1, wf=g, bf={"type": "constant", "value": 0.1})
    b.relu("relu_b3", "b3x3")
    b.layer("cat", "CONCAT", ("a1x1", "b3x3"), ("cat",))
    b.conv("mix", "cat", 128, 1, wf=g, bf={"type": "constant", "value": 0.0})
    b.relu("relu_mix", "mix")
    b.pool("pool", "mix", "AVE", 3, 2)
    b.fc("fc", "pool", classes, wf=g, bf={"type": "constant", "value": 0.0})
    b.softmax_loss("loss", "fc")
    return b.net


FP8_LAYERS = {"alex": {"conv3", "conv4", "conv5"}, "incep": {"b3x3", "mix"}}
NETS = {"alex": (fp8_alex_net, 27), "incep": (fp8_inception_net, 19)}


def _solver_param(net, steps):
    """The small solver, on the CPU when the engine runs on the emulated kernels (also on a machine with a GPU)."""
    from poseidon_b200.ops import sm100
    sp = small_solver_param(net, max_iter=steps)
    if sm100.emulating():
        sp.solver_mode = "CPU"
    return sp


def _run(which, fp8, steps, engine="sm100", graph=False, batch=8, classes=16):
    from poseidon_b200 import get_solver
    fn, hw = NETS[which]
    net = fn(batch=batch, classes=classes, hw=hw)
    sp = _solver_param(net, steps)
    s = get_solver(sp, engine=engine, fp8=fp8, dtype=torch.float32 if engine == "torch" else None)
    x, y = make_data(batch * steps, classes=classes, hw=hw)
    feed(s, x, y)
    losses = []
    if graph:
        s.enable_cuda_graph(warmup=2)
    for _ in range(steps):
        s.step(1)
        losses.append(float(s.last_loss))
    if s.rank_ctx.device.type == "cuda":
        torch.cuda.synchronize()
    weights = {f"{n}.{j}": l.export_blob(j) for n, l in zip(s.net.layer_names, s.net.layers) for j in range(len(l.blobs))}
    return losses, weights, s


# ------------------------------------------------------------------------------------------------ CPU: the plan
def _plan(net_param, emu, fp8="fprop"):
    from poseidon_b200 import proto as P
    from poseidon_b200.layers import NetContext
    from poseidon_b200.net.net import Net
    ctx = NetContext(phase=P.TRAIN, device="cpu", engine="sm100", dtype=torch.bfloat16, fp8=fp8)
    net = Net(net_param, phase=P.TRAIN, ctx=ctx)
    return {n: l._sm100 for n, l in zip(net.layer_names, net.layers) if l.type_name == "CONVOLUTION"}


def test_eligibility_alexnet(emu):
    from poseidon_b200.models import zoo
    st = _plan(zoo.alexnet(batch=2, test_batch=2), emu)
    assert {n for n, s in st.items() if s.fp8} == {"conv3", "conv4", "conv5"}
    assert st["conv1"].s2d and "s2d" in st["conv1"].fp8_reason
    assert st["conv2"].cg == 48 and "third" in st["conv2"].fp8_reason
    assert (st["conv3"].cg, st["conv3"].cgk8) == (256, 256)
    assert (st["conv4"].cg, st["conv4"].cgk8) == (192, 256) and (st["conv5"].cg, st["conv5"].cgk8) == (192, 256)


def test_eligibility_vgg16(emu):
    from poseidon_b200.models import zoo
    st = _plan(zoo.vgg16(batch=1, test_batch=1), emu)
    bf16 = {n for n, s in st.items() if not s.fp8}
    assert bf16 == {"conv1_1", "conv1_2", "conv2_1"}, bf16
    assert st["conv1_1"].pad8
    assert all(s.cin_logical >= 128 for s in st.values() if s.fp8)


def test_eligibility_googlenet(emu):
    from poseidon_b200.models import zoo
    st = _plan(zoo.googlenet(batch=1, test_batch=1), emu)
    fp8_in = {s.cin_logical for s in st.values() if s.fp8}
    bf16_in = {s.cin_logical for s in st.values() if not s.fp8}
    assert fp8_in == {96, 112, 128, 192, 256, 480, 512, 528, 832}, sorted(fp8_in)
    assert bf16_in - {3} == {16, 24, 32, 48, 64, 144, 160}, sorted(bf16_in)
    assert not fp8_in & bf16_in


def test_fp8_off_changes_no_plan(emu):
    from poseidon_b200.models import zoo
    for s in _plan(zoo.alexnet(batch=2, test_batch=2), emu, fp8="off").values():
        assert not s.fp8 and s.cgk8 == 0 and s.fp8_reason == "fp8 off"


def test_plan_logs_one_line_per_conv(emu, caplog):
    import logging
    with caplog.at_level(logging.INFO, logger="poseidon_b200"):
        _plan(fp8_alex_net(batch=2), emu)
    lines = [r.getMessage() for r in caplog.records if r.getMessage().startswith("sm100 plan: conv ")]
    assert len(lines) == 5
    assert "conv3: fp8 (Cg 128 -> 128 slots)" in lines[2] and "conv2: bf16" in lines[1]


# ------------------------------------------------------------------------------------------------ CPU: the setting
def test_setting_resolution(monkeypatch):
    from poseidon_b200.ops import sm100
    monkeypatch.delenv("POSEIDON_FP8", raising=False)
    assert sm100.resolve_fp8() == "off"
    monkeypatch.setenv("POSEIDON_FP8", "fprop")
    assert sm100.resolve_fp8() == "fprop" and sm100.resolve_fp8("off") == "off"
    assert sm100.fp8_for_engine("torch") == "off"           # the env var is an sm100 engine switch
    with pytest.raises(ValueError, match="sm100"):
        sm100.fp8_for_engine("torch", "fprop")
    monkeypatch.setenv("POSEIDON_FP8", "e5m2")
    with pytest.raises(ValueError, match="fp8 must be one of"):
        sm100.resolve_fp8()


def test_get_solver_and_engine_plumbing(emu, monkeypatch):
    monkeypatch.delenv("POSEIDON_FP8", raising=False)
    from poseidon_b200 import get_solver
    from poseidon_b200.engine import CaffeEngine
    sp = _solver_param(fp8_alex_net(batch=2), 1)
    s = get_solver(sp, engine="sm100", fp8="fprop")
    assert s.fp8 == "fprop" and s.net.ctx.fp8 == "fprop"
    assert s.net.layer_by_name["conv3"]._sm100.fp8
    assert all(n.ctx.fp8 == "fprop" for n in getattr(s, "test_nets", []))
    assert get_solver(sp, engine="sm100").fp8 == "off"
    with pytest.raises(ValueError, match="sm100"):
        get_solver(sp, engine="torch", fp8="fprop", dtype=torch.float32)
    eng = CaffeEngine(sp, engine="sm100", fp8="fprop")
    assert eng.build().fp8 == "fprop"
    eng.close()


def test_caffe_main_flag(emu, tmp_path, monkeypatch):
    monkeypatch.delenv("POSEIDON_FP8", raising=False)
    from poseidon_b200 import proto as P
    from poseidon_b200.tools import caffe_main
    assert caffe_main.parse_args(["train", "--solver=s.prototxt", "--fp8", "fprop"]).fp8 == "fprop"
    assert caffe_main.parse_args(["train", "--solver=s.prototxt"]).fp8 is None
    with pytest.raises(SystemExit):
        caffe_main.parse_args(["train", "--fp8", "e5m2"])
    model = tmp_path / "net.prototxt"
    model.write_text(P.to_text(fp8_alex_net(batch=2)) if hasattr(P, "to_text") else str(fp8_alex_net(batch=2)))
    args = caffe_main.parse_args(["test", f"--model={model}", "--engine=sm100", "--fp8=fprop", "--gpu=-1"])
    net, _ = caffe_main._build_net(args, P.TEST)
    assert net.ctx.fp8 == "fprop" and net.layer_by_name["conv3"]._sm100.fp8
    args = caffe_main.parse_args(["test", f"--model={model}", "--engine=torch", "--fp8=fprop", "--gpu=-1"])
    with pytest.raises(ValueError, match="sm100"):
        caffe_main._build_net(args, P.TEST)


# ------------------------------------------------------------------------------------------------ CPU: emulated steps
def test_emulated_step_tracks_bf16(emu):
    """fp8=fprop on the emulated kernels: losses within 5 % (and at least 0.05) of the bf16 emulation over 3 steps."""
    l_bf, w_bf, _ = _run("alex", "off", 3)
    l_f8, w_f8, s = _run("alex", "fprop", 3)
    assert all(s.net.layer_by_name[n]._sm100.fp8 for n in FP8_LAYERS["alex"])
    for a, b in zip(l_bf, l_f8):
        assert abs(a - b) <= 0.05 * max(1.0, abs(a)), (l_bf, l_f8)
    for name in (n for n in w_bf if n.endswith(".0")):          # weights (biases start at constants: tiny values)
        d = np.abs(w_bf[name] - w_f8[name]).max()
        assert d <= 0.05 * np.abs(w_bf[name]).max() + 1e-3, (name, d)


def test_quantiser_emulation_reference():
    """The emulated quantisers: scale = 448 / amax, clamp then cast, NaN stays NaN, all-zero input gives scale 1."""
    from poseidon_b200.ops.emulate import EmulatedKernels
    k = EmulatedKernels()
    x = torch.randn(2, 24, 5, 3).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    x[0, 3, 1, 1] = float("nan")
    s_x = torch.empty(1)
    q = k.fp8_quant_act(x, s_x)
    assert q.dtype == torch.float8_e4m3fn and tuple(q.shape) == (2, 24, 5, 3) and q.stride(3) == 32
    amax = x.float().abs().nan_to_num(0.0).max()
    s = torch.div(torch.tensor(448.0), amax)
    assert torch.equal(s_x, torch.div(torch.tensor(1.0), s).reshape(1))
    assert torch.isnan(q.float()[0, 3, 1, 1]) and int(torch.isnan(q.float()).sum()) == 1
    assert float(q.float().nan_to_num(0.0).abs().max()) == 448.0
    z = torch.zeros(1, 8, 2, 2, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    assert float(k.fp8_quant_act(z, s_x).float().abs().max()) == 0.0 and float(s_x) == 1.0
    w = torch.randn(6, 40, 3, 3).contiguous(memory_format=torch.channels_last)
    s_w = torch.empty(6)
    w8 = k.fp8_quant_weight(w, 128, s_w)
    assert tuple(w8.shape) == (6, 9 * 128)
    assert float(w8.float().reshape(6, 9, 128)[..., 40:].abs().max()) == 0.0
    back = w8.float().reshape(6, 9, 128)[..., :40] * s_w.view(6, 1, 1)
    ref = w.permute(0, 2, 3, 1).reshape(6, 9, 40)
    assert float(((back - ref).abs() / ref.abs().amax(dim=(1, 2), keepdim=True)).max()) <= 2 ** -4


def test_caffemodel_from_fp8_run_resumes_without_fp8(emu, tmp_path):
    """fp8 tensors are derived and never saved: a snapshot written with fp8 on loads and resumes with fp8 off."""
    from poseidon_b200 import get_solver
    net = fp8_alex_net(batch=4)
    sp = _solver_param(net, 2)
    sp.snapshot_prefix = str(tmp_path / "f8")
    s = get_solver(sp, engine="sm100", fp8="fprop")
    x, y = make_data(16, hw=27)
    feed(s, x, y)
    s.step(2)
    s.snapshot()
    ref = {n: l.export_blob(0) for n, l in zip(s.net.layer_names, s.net.layers) if len(l.blobs)}
    s2 = get_solver(sp, engine="sm100", fp8="off")
    s2.restore(str(tmp_path / "f8_iter_2.solverstate"))
    for n, l in zip(s2.net.layer_names, s2.net.layers):
        if len(l.blobs):
            assert np.array_equal(l.export_blob(0), ref[n]), n
    assert not s2.net.layer_by_name["conv3"]._sm100.fp8
    s3 = get_solver(sp, engine="sm100", fp8="off")
    s3.load_weights(str(tmp_path / "f8_iter_2.caffemodel"))
    feed(s2, x, y)
    s2.step(1)
    assert s2.iter == 3 and np.isfinite(float(s2.last_loss))


# ------------------------------------------------------------------------------------------------ CPU: SASS
def _sass_by_function(so):
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True, timeout=600).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None:
            m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(.*?;)", line)
            if m:
                funcs[cur].append(m.group(1).strip())
    return funcs


def _demangle(names):
    tool = shutil.which("cu++filt") or shutil.which("c++filt")
    out = subprocess.run([tool], input="\n".join(names), capture_output=True, text=True, timeout=120).stdout.splitlines()
    return dict(zip(names, out))


@pytest.fixture(scope="module")
def sass():
    if not os.path.exists(SO) or shutil.which("cuobjdump") is None or \
            not (shutil.which("cu++filt") or shutil.which("c++filt")):
        pytest.skip("needs the built extension, cuobjdump and a demangler")
    return _sass_by_function(SO)


def test_fp8_kernels_use_e4m3_wgmma_and_im2col_tma(sass):
    names = _demangle([k for k in sass if "wgmma_fp8_conv_kernel" in k])
    fp8 = {k: "\n".join(sass[k]) for k in names}
    assert len(fp8) == 4, sorted(names[k] for k in fp8)          # BN 64 / 128, single CTA / CTA pair
    for k, text in fp8.items():
        assert re.search(r"QGMMA\.64x(64|128)x32\.F32\.E4M3\.E4M3", text), names[k]     # fp8 wgmma is QGMMA
        assert "UTMALDG.4D.IM2COL" in text, names[k]
        assert not re.search(r"\b(HMMA|HGMMA)", text), names[k]
    assert any("UTMALDG.2D.MULTICAST" in t for t in fp8.values()), "CTA-pair multicast of the fp8 weight tile"


def test_bf16_gemm_instruction_streams_unchanged(sass):
    """Every bf16 wgmma_gemm_kernel instantiation compiles to the instruction stream of the commit before the fp8 kernels
    were added (tests/golden/wgmma_bf16_sass.json: sha256 of each kernel's SASS without addresses / encodings, by
    demangled name).  Two kernels are held to their instruction count only: in the CTA-pair optimizer-step GEMMs
    (EPI_SGD, BN 128 / 256) ptxas swaps two independent SELs and, at BN 128, writes one MOV as IMAD.MOV."""
    reordered = {f"void psd::wgmma_gemm_kernel<(int){bn}, (bool)1, (bool)1, (int)2, (int)0, (int)2>"
                 "(psd::TmapSet, psd::GemmParams, psd::ConvGeom)" for bn in (128, 256)}
    with open(GOLDEN_SASS) as f:
        golden = json.load(f)["kernels"]
    names = _demangle([k for k in sass if "wgmma_gemm_kernel" in k])
    now = {d: sass[k] for k, d in names.items()}
    assert set(now) == set(golden), sorted(set(now) ^ set(golden))[:4]

    def sha(lines):
        return hashlib.sha256("\n".join(lines).encode()).hexdigest()

    changed = [n for n, g in golden.items() if n not in reordered and sha(now[n]) != g["sha256"]]
    assert not changed, changed[:4]
    for n in reordered:
        assert len(now[n]) == golden[n]["instructions"], n


# ================================================================================================ H100
gpu = pytest.mark.gpu


def _nhwc_bf16(n, c, h, w, pitch=None, c_off=0, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    pitch = pitch or c
    base = (torch.randn(n, h, w, pitch, generator=g) * scale).to(torch.bfloat16).cuda()
    return base[..., c_off:c_off + c].permute(0, 3, 1, 2)


def _check_quant_act(ext, x):
    from poseidon_b200.ops.emulate import EmulatedKernels
    s_x = torch.empty(1, device="cuda")
    q = ext.fp8_quant_act(x, s_x)
    s_ref = torch.empty(1)
    q_ref = EmulatedKernels().fp8_quant_act(x.cpu(), s_ref)
    assert q.dtype == torch.float8_e4m3fn and tuple(q.shape) == tuple(x.shape)
    assert q.stride(1) == 1 and q.stride(3) == (x.shape[1] + 15) // 16 * 16
    assert torch.equal(s_x.cpu(), s_ref), (float(s_x), float(s_ref))
    a, b = q.cpu().float(), q_ref.float()
    nan = torch.isnan(b)
    assert torch.equal(torch.isnan(a), nan)
    assert torch.equal(q.cpu().view(torch.uint8)[~nan], q_ref.view(torch.uint8)[~nan])
    return q, s_x


@gpu
@pytest.mark.parametrize("shape,pitch,c_off", [
    ((4, 256, 13, 13), None, 0),        # AlexNet conv3 input
    ((3, 24, 7, 5), None, 0),           # C % 16 == 8: one pad half per pixel
    ((2, 96, 9, 9), 256, 64),           # a channel slice of a concat slab
    ((2, 40, 6, 6), 136, 88),           # pitched, C % 16 == 8
])
def test_quant_act_bitexact(ext, shape, pitch, c_off):
    x = _nhwc_bf16(*shape, pitch=pitch, c_off=c_off, seed=sum(shape))
    q1, s1 = _check_quant_act(ext, x)
    q2, s2 = _check_quant_act(ext, x)
    assert torch.equal(q1.view(torch.uint8), q2.view(torch.uint8)) and torch.equal(s1, s2)


@gpu
def test_quant_act_zero_and_nan(ext):
    z = torch.zeros(2, 32, 4, 4, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    q, s = _check_quant_act(ext, z)
    assert float(s) == 1.0 and int(q.view(torch.uint8).count_nonzero()) == 0
    x = _nhwc_bf16(2, 48, 5, 5, seed=3).clone(memory_format=torch.channels_last)
    x[1, 7, 2, 3] = float("nan")
    q, s = _check_quant_act(ext, x)
    f = q.float()
    assert torch.isnan(f[1, 7, 2, 3]) and int(torch.isnan(f).sum()) == 1
    x[0, 0, 0, 0] = float("inf")
    q, _ = _check_quant_act(ext, x)
    assert torch.isnan(q.float()[0, 0, 0, 0])


@gpu
@pytest.mark.parametrize("cout,cg,k,cgk", [(384, 256, 3, 256), (256, 192, 3, 256), (192, 480, 1, 512), (64, 24, 3, 128)])
def test_quant_weight_bitexact(ext, cout, cg, k, cgk):
    from poseidon_b200.ops.emulate import EmulatedKernels
    g = torch.Generator(device="cpu").manual_seed(cout + cg)
    w = (torch.randn(cout, cg, k, k, generator=g) * 0.03).contiguous(memory_format=torch.channels_last)
    w[1].zero_()
    w[2, 3, 0, 0] = float("nan")
    s_w = torch.empty(cout, device="cuda")
    w8 = ext.fp8_quant_weight(w.cuda(), cgk, s_w)
    s_ref = torch.empty(cout)
    w8_ref = EmulatedKernels().fp8_quant_weight(w, cgk, s_ref)
    assert torch.equal(s_w.cpu(), s_ref) and float(s_ref[1]) == 1.0
    nan = torch.isnan(w8_ref.float())
    assert int(nan.sum()) == 1 and torch.equal(torch.isnan(w8.cpu().float()), nan)
    assert torch.equal(w8.cpu().view(torch.uint8)[~nan], w8_ref.view(torch.uint8)[~nan])
    w8b = ext.fp8_quant_weight(w.cuda(), cgk, s_w)
    assert torch.equal(w8.view(torch.uint8), w8b.view(torch.uint8))


def _ref_conv64(x8, s_x, w8, s_w, bias, cg, k, stride, pad, groups, relu, slope):
    """float64 reference of the dequantised operands: (ref, Σ|a·b| per output) after bias / activation."""
    import torch.nn.functional as F
    cout = w8.shape[0]
    cgk = w8.shape[1] // (k * k)
    xd = x8.cpu().double() * float(s_x)
    wd = w8.cpu().double().reshape(cout, k, k, cgk)[..., :cg].permute(0, 3, 1, 2) * s_w.cpu().double().view(-1, 1, 1, 1)
    pre = F.conv2d(xd, wd, None, stride, pad, 1, groups)
    mag = F.conv2d(xd.abs(), wd.abs(), None, stride, pad, 1, groups)
    if bias is not None:
        pre = pre + bias.cpu().double().view(1, -1, 1, 1)
    ref = torch.where(pre > 0, pre, pre * slope) if relu else pre
    return ref, mag


def _sentinel_out(n, cout, oh, ow, pitch, c_off, guard=4096):
    """Output view (channel slice of a slab) inside a sentinel-filled allocation."""
    buf = torch.full((guard + n * oh * ow * pitch + guard,), -7.25, dtype=torch.bfloat16, device="cuda")
    slab = buf[guard:guard + n * oh * ow * pitch].view(n, oh, ow, pitch)
    return buf, slab[..., c_off:c_off + cout].permute(0, 3, 1, 2)


ACC_RATIOS = {}


@gpu
@pytest.mark.parametrize("pair", [1, 0])
@pytest.mark.parametrize("name,n,cin,h,cout,k,stride,pad,groups,act", [
    ("alex_conv3", 4, 256, 13, 384, 3, 1, 1, 1, "relu"),
    ("alex_conv4", 4, 384, 13, 384, 3, 1, 1, 2, "relu"),      # Cg 192 -> 256 slots
    ("alex_conv5", 3, 384, 13, 256, 3, 1, 1, 2, "leaky"),
    ("vgg_512", 2, 512, 14, 512, 3, 1, 1, 1, "relu"),         # K = 4608
    ("goog_1x1", 5, 480, 14, 192, 1, 1, 0, 1, "none"),        # K = 512
    ("stride2", 3, 128, 15, 128, 3, 2, 1, 1, "relu"),
    ("k128", 2, 128, 9, 64, 1, 1, 0, 1, "none"),              # one K block
])
def test_conv_fprop_fp8(ext, pair, name, n, cin, h, cout, k, stride, pad, groups, act):
    ext.set_conv_pair(pair)
    try:
        cg = cin // groups
        cgk = (cg + 127) // 128 * 128
        oh = (h + 2 * pad - k) // stride + 1
        x = _nhwc_bf16(n, cin, h, h, seed=n * cin + h)
        g = torch.Generator(device="cpu").manual_seed(cout + k)
        w = (torch.randn(cout, cg, k, k, generator=g) * 0.05).contiguous(memory_format=torch.channels_last).cuda()
        bias = (torch.randn(cout, generator=g) * 0.1).cuda()
        s_x, s_w = torch.empty(1, device="cuda"), torch.empty(cout, device="cuda")
        w8 = ext.fp8_quant_weight(w, cgk, s_w)
        x8 = ext.fp8_quant_act(x, s_x)
        relu, slope = act != "none", (0.1 if act == "leaky" else 0.0)
        pitch = cout + 32
        buf, out = _sentinel_out(n, cout, oh, oh, pitch, 16)
        before = buf.clone()
        y = ext.conv_fprop_fp8(x8, w8, s_x, s_w, None if act == "none" else bias, [k, k], [stride, stride], [pad, pad],
                               groups, oh, oh, relu, slope, out)
        torch.cuda.synchronize()
        assert y.data_ptr() == out.data_ptr()
        ref, mag = _ref_conv64(x8, s_x, w8, s_w, None if act == "none" else bias, cg, k, (stride, stride), (pad, pad),
                               groups, relu, slope)
        got = y.cpu().double()
        err = (got - ref).abs()
        # bf16 output rounding (2^-9 relative, with margin) + fp32 accumulation of exact e4m3 products, held to the
        # 2^-10 · Σ|a·b| level: beyond that the accumulator would need per-k-block promotion
        bound = 2.0 ** -8 * ref.abs() + 2.0 ** -10 * mag + 1e-30
        worst = float((err / bound).max())
        excess = ((err - 2.0 ** -9 * ref.abs()).clamp(min=0) / mag.clamp(min=1e-30)).max()
        ACC_RATIOS[(name, pair)] = (cg * k * k, float((err / mag.clamp(min=1e-30)).max()), float(excess), worst)
        print(f"fp8 {name} pair={pair} K={cg * k * k}: max|out-ref|/sum|ab| = {ACC_RATIOS[(name, pair)][1]:.3e}, "
              f"beyond output rounding {float(excess):.3e}, err/bound {worst:.3f}")
        assert worst <= 1.0, (name, worst)
        # the sentinel around and between the written channels comes back bit for bit
        region = torch.zeros_like(buf, dtype=torch.bool)
        idx = torch.arange(n * oh * oh * pitch, device="cuda").view(n, oh, oh, pitch)[..., 16:16 + cout]
        region[4096 + idx.reshape(-1)] = True
        assert torch.equal(buf.view(torch.int16)[~region], before.view(torch.int16)[~region])
        y2 = ext.conv_fprop_fp8(x8, w8, s_x, s_w, None if act == "none" else bias, [k, k], [stride, stride], [pad, pad],
                                groups, oh, oh, relu, slope, None)
        assert torch.equal(y2.float().cpu(), y.float().cpu())          # same bits into a fresh tensor
    finally:
        ext.set_conv_pair(1)


@gpu
def test_conv_fprop_fp8_ragged_m(ext):
    """N*OH*OW = 3*11*11 = 363: the last pixel block is partial."""
    n, cin, h, cout = 3, 128, 11, 96
    x = _nhwc_bf16(n, cin, h, h, seed=9)
    w = (torch.randn(cout, cin, 3, 3) * 0.05).contiguous(memory_format=torch.channels_last).cuda()
    s_x, s_w = torch.empty(1, device="cuda"), torch.empty(cout, device="cuda")
    w8, x8 = ext.fp8_quant_weight(w, 128, s_w), ext.fp8_quant_act(x, s_x)
    y = ext.conv_fprop_fp8(x8, w8, s_x, s_w, None, [3, 3], [1, 1], [1, 1], 1, h, h, False, 0.0, None)
    ref, mag = _ref_conv64(x8, s_x, w8, s_w, None, cin, 3, (1, 1), (1, 1), 1, False, 0.0)
    err = (y.cpu().double() - ref).abs()
    assert float((err / (2.0 ** -8 * ref.abs() + 2.0 ** -10 * mag + 1e-30)).max()) <= 1.0


@gpu
def test_conv_fprop_fp8_rejects_what_it_cannot_run(ext):
    x = _nhwc_bf16(2, 128, 8, 8)
    s_x, s_w = torch.empty(1, device="cuda"), torch.empty(64, device="cuda")
    x8 = ext.fp8_quant_act(x, s_x)
    w = torch.randn(64, 128, 3, 3).contiguous(memory_format=torch.channels_last).cuda()
    w8_64 = ext.fp8_quant_weight(w, 192, s_w)                       # 192 slots: not a multiple of 128
    with pytest.raises(RuntimeError, match="multiple of 128"):
        ext.conv_fprop_fp8(x8, w8_64, s_x, s_w, None, [3, 3], [1, 1], [1, 1], 1, 8, 8, False, 0.0, None)
    w8 = ext.fp8_quant_weight(w, 128, s_w)
    ext.set_conv_mcast(2)
    try:
        with pytest.raises(RuntimeError, match="set_conv_mcast"):
            ext.conv_fprop_fp8(x8, w8, s_x, s_w, None, [3, 3], [1, 1], [1, 1], 1, 8, 8, False, 0.0, None)
    finally:
        ext.set_conv_mcast(1)


@gpu
@pytest.mark.parametrize("which", ["alex", "incep"])
def test_net_tracks_bf16_and_repeats(ext, which):
    """fp8=fprop trains: losses within 5 % of the bf16 engine over 4 steps; two runs give identical bits."""
    l_bf, _, s0 = _run(which, "off", 4)
    s0.close()
    l1, w1, s1 = _run(which, "fprop", 4)
    assert all(s1.net.layer_by_name[n]._sm100.fp8 for n in FP8_LAYERS[which])
    if which == "incep":
        assert getattr(s1.net.layer_by_name["b3x3"], "_concat_slab", None) is not None
    s1.close()
    l2, w2, s2 = _run(which, "fprop", 4)
    s2.close()
    print(f"{which}: bf16 losses {l_bf}, fp8 losses {l1}")
    for a, b in zip(l_bf, l1):
        assert abs(a - b) <= 0.05 * max(1.0, abs(a)), (l_bf, l1)
    assert l1 == l2
    for n in w1:
        assert np.array_equal(w1[n], w2[n]), n


@gpu
def test_graph_replay_requantises_the_updated_master(ext):
    """Under CUDA-graph replay the fp8 weights follow the optimizer: after every replayed step the per-channel scales
    are those of the master as it was before the step (not of the weights at capture time).  Two graph runs give
    identical bits, and the graph run follows the eager one as closely as the bf16 engine's graph test requires."""
    from poseidon_b200 import get_solver
    from poseidon_b200.ops.emulate import EmulatedKernels

    def run(graph):
        net = fp8_alex_net(batch=8)
        sp = small_solver_param(net, max_iter=8)
        s = get_solver(sp, engine="sm100", fp8="fprop")
        x, y = make_data(8 * 8, hw=27)
        feed(s, x, y)
        if graph:
            s.enable_cuda_graph(warmup=2)          # 2 eager + 1 captured step: iteration 3, like 3 eager steps
        layer = s.net.layer_by_name["conv3"]
        scales = []
        while s.iter < 8:
            w_before = layer.weight.detach().float().cpu().contiguous(memory_format=torch.channels_last)
            s.step(1)
            torch.cuda.synchronize()
            ref = torch.empty(w_before.shape[0])
            EmulatedKernels().fp8_quant_weight(w_before, layer._sm100.cgk8, ref)
            scales.append((layer._sm100.s_w.cpu().clone(), ref))
        graphed = getattr(s, "_graph", None) is not None
        out = {n: l.export_blob(0) for n, l in zip(s.net.layer_names, s.net.layers) if len(l.blobs)}
        loss = float(s.last_loss)
        s.close()
        return out, loss, scales, graphed

    w_e, l_e, sc_e, g_e = run(False)
    w_g, l_g, sc_g, g_g = run(True)
    w_g2, l_g2, _, _ = run(True)
    assert not g_e and g_g
    assert len(sc_g) == 5 and len(sc_e) == 8
    for got, ref in sc_g + sc_e:
        assert torch.equal(got, ref)
    assert not torch.equal(sc_g[-1][0], sc_g[-2][0])            # the scales do move from replay to replay
    assert l_g == l_g2 and all(np.array_equal(w_g[n], w_g2[n]) for n in w_g)
    assert abs(l_e - l_g) < 0.05 * max(1.0, abs(l_e)), (l_e, l_g)
    for n in w_e:
        d = np.abs(w_e[n] - w_g[n]).max()
        assert d <= 0.02 * np.abs(w_e[n]).max() + 1e-4, (n, d)
