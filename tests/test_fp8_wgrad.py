"""fp8 weight gradients (e5m2 dY x e4m3 X) for stride-1 convolutions: the opt-in ``fp8="fprop+dgrad+wgrad"`` setting.

CPU (no GPU needed): the eligibility rule on the zoo nets, the "off" / "fprop" / "fprop+dgrad" plans unchanged, the
plan line, the setting's plumbing, an emulated training run against the bf16 emulation, checkpoints, and the SASS of the
built extension.
H100: the batch-innermost quantisers bit for bit against the torch reference, conv_wgrad_fp8 against a float64 reference
of the dequantised operands, and whole nets against fprop+dgrad and bf16 (bit-identical bf16 weight gradients, loss
tracking, repeatability, CUDA-graph replay)."""
import hashlib
import json
import os
import re

import numpy as np
import pytest
import torch

from poseidon_b200.ops.emulate import chwn_images
from smallnet import feed, make_data, small_solver_param
from test_fp8_fprop import (  # noqa: F401  (_keep_dropout_counters: autouse fixture, restores the dropout counters)
    NETS, _demangle, _keep_dropout_counters, _nhwc_bf16, _plan, _run, _solver_param, emu, fp8_alex_net, sass)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_DGRAD_SASS = os.path.join(ROOT, "tests", "golden", "wgmma_fp8_dgrad_sass.json")
MODE = "fprop+dgrad+wgrad"

# layers of the small nets (tests/test_fp8_fprop.py) whose weight gradient runs in fp8
WGRAD_LAYERS = {"alex": {"conv2", "conv3", "conv4"}, "incep": {"a1x1", "b1x1", "b3x3", "mix"}}


# ------------------------------------------------------------------------------------------------ CPU: the plan
def test_wgrad_eligibility_alexnet(emu):
    from poseidon_b200.models import zoo
    st = _plan(zoo.alexnet(batch=2, test_batch=2), emu, fp8=MODE)
    assert {n for n, s in st.items() if s.fp8_wgrad} == {"conv2", "conv3", "conv4", "conv5"}
    assert "first-layer" in st["conv1"].fp8_wgrad_reason
    assert [st[n].cgkw8 for n in ("conv2", "conv3", "conv4", "conv5")] == [64, 256, 192, 192]
    assert st["conv2"].fp8_wgrad_reason == "Cg 48 -> 64 columns per tap"


def test_wgrad_eligibility_vgg16(emu):
    from poseidon_b200.models import zoo
    st = _plan(zoo.vgg16(batch=1, test_batch=1), emu, fp8=MODE)
    assert {n for n, s in st.items() if not s.fp8_wgrad} == {"conv1_1"}
    assert "first-layer" in st["conv1_1"].fp8_wgrad_reason
    assert len([s for s in st.values() if s.fp8_wgrad]) == 12


def test_wgrad_eligibility_googlenet(emu):
    from poseidon_b200.models import zoo
    st = _plan(zoo.googlenet(batch=1, test_batch=1), emu, fp8=MODE)
    s1 = {n: s for n, s in st.items() if tuple(s.layer.stride) == (1, 1) and not s.row_mode}
    assert {s.cg for s in s1.values() if not s.fp8_wgrad} == {16, 24, 32}
    assert all("within a third" in s.fp8_wgrad_reason for s in s1.values() if not s.fp8_wgrad)
    assert all(s.cgkw8 % 64 == 0 and s.cgkw8 >= s.cg for s in s1.values() if s.fp8_wgrad)
    strided = [s for s in st.values() if tuple(s.layer.stride) != (1, 1)]
    assert strided and not any(s.fp8_wgrad for s in strided)
    assert len([s for s in st.values() if s.fp8_wgrad]) == 50 and len(st) == 59


def test_other_modes_plan_no_fp8_wgrad(emu):
    from poseidon_b200.models import zoo
    for mode in ("off", "fprop", "fprop+dgrad"):
        for s in _plan(zoo.alexnet(batch=2, test_batch=2), emu, fp8=mode).values():
            assert not s.fp8_wgrad and s.cgkw8 == 0 and s.fp8_wgrad_reason == "fp8 wgrad off"
    a = _plan(zoo.googlenet(batch=1, test_batch=1), emu, fp8="fprop+dgrad")
    b = _plan(zoo.googlenet(batch=1, test_batch=1), emu, fp8=MODE)

    def key(s):
        return s.fp8, s.fp8_reason, s.cgk8, s.fp8_dgrad, s.fp8_dgrad_reason, s.cok8, s.cgk, s.cok, s.mask_input
    assert {n: key(s) for n, s in a.items()} == {n: key(s) for n, s in b.items()}


def _plan_lines(emu, caplog, mode):
    import logging
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="poseidon_b200"):
        _plan(fp8_alex_net(batch=2), emu, fp8=mode)
    return [r.getMessage() for r in caplog.records if r.getMessage().startswith("sm100 plan: conv ")]


def test_plan_log_gives_the_wgrad_decision(emu, caplog):
    dgrad = _plan_lines(emu, caplog, "fprop+dgrad")
    assert len(dgrad) == 5 and not any("wgrad" in l for l in dgrad)
    wgrad = _plan_lines(emu, caplog, MODE)
    assert len(wgrad) == 5
    for a, b in zip(dgrad, wgrad):
        assert b.startswith(a + "; wgrad "), (a, b)
    assert wgrad[0].endswith("; wgrad bf16 (first-layer layout (ROW / s2d / 8-channel pad))"), wgrad[0]
    assert wgrad[3].endswith("; wgrad fp8 (Cg 96 -> 128 columns per tap)"), wgrad[3]
    assert wgrad[4].endswith("; wgrad bf16 (strided)"), wgrad[4]


# ------------------------------------------------------------------------------------------------ CPU: the setting
def test_setting_resolution(monkeypatch):
    from poseidon_b200.ops import sm100
    monkeypatch.setenv("POSEIDON_FP8", MODE)
    assert sm100.resolve_fp8() == MODE and sm100.resolve_fp8("FPROP+DGRAD+WGRAD") == MODE
    assert sm100.fp8_for_engine("torch") == "off"
    with pytest.raises(ValueError, match="sm100"):
        sm100.fp8_for_engine("torch", MODE)
    for bad in ("wgrad", "fprop+wgrad", "dgrad+wgrad"):
        with pytest.raises(ValueError, match="fp8 must be one of"):
            sm100.resolve_fp8(bad)


def test_get_solver_engine_and_cli_plumbing(emu, tmp_path, monkeypatch):
    monkeypatch.delenv("POSEIDON_FP8", raising=False)
    from poseidon_b200 import get_solver
    from poseidon_b200 import proto as P
    from poseidon_b200.engine import CaffeEngine
    from poseidon_b200.tools import caffe_main
    sp = _solver_param(fp8_alex_net(batch=2), 1)
    s = get_solver(sp, engine="sm100", fp8=MODE)
    assert s.fp8 == MODE and s.net.ctx.fp8 == MODE
    st = s.net.layer_by_name["conv3"]._sm100
    assert st.fp8_wgrad and st.fp8_dgrad and st.fp8
    with pytest.raises(ValueError, match="sm100"):
        get_solver(sp, engine="torch", fp8=MODE, dtype=torch.float32)
    eng = CaffeEngine(sp, engine="sm100", fp8=MODE)
    assert eng.build().fp8 == MODE
    eng.close()
    monkeypatch.setenv("POSEIDON_FP8", MODE)
    assert get_solver(sp, engine="sm100").fp8 == MODE
    monkeypatch.delenv("POSEIDON_FP8")
    assert caffe_main.parse_args(["train", "--solver=s.prototxt", "--fp8", MODE]).fp8 == MODE
    assert MODE in caffe_main.make_parser().format_help().replace("\n", " ").replace("  ", "")
    model = tmp_path / "net.prototxt"
    model.write_text(P.to_text(fp8_alex_net(batch=2)) if hasattr(P, "to_text") else str(fp8_alex_net(batch=2)))
    args = caffe_main.parse_args(["test", f"--model={model}", "--engine=sm100", f"--fp8={MODE}", "--gpu=-1"])
    net, _ = caffe_main._build_net(args, P.TEST)
    assert net.ctx.fp8 == MODE and net.layer_by_name["conv2"]._sm100.fp8_wgrad
    args = caffe_main.parse_args(["test", f"--model={model}", "--engine=torch", f"--fp8={MODE}", "--gpu=-1"])
    with pytest.raises(ValueError, match="sm100"):
        caffe_main._build_net(args, P.TEST)


# ------------------------------------------------------------------------------------------------ CPU: emulation
def test_emulated_step_tracks_bf16(emu):
    """fp8=fprop+dgrad+wgrad on the emulated kernels: losses within 5 % (and at least 0.05) of the bf16 emulation over 3
    steps, and the fp8-wgrad weights move away from the fprop+dgrad ones."""
    l_bf, w_bf, _ = _run("alex", "off", 3)
    l_d, w_d, _ = _run("alex", "fprop+dgrad", 3)
    l_f8, w_f8, s = _run("alex", MODE, 3)
    assert {n for n in WGRAD_LAYERS["alex"] if s.net.layer_by_name[n]._sm100.fp8_wgrad} == WGRAD_LAYERS["alex"]
    for a, b in zip(l_bf, l_f8):
        assert abs(a - b) <= 0.05 * max(1.0, abs(a)), (l_bf, l_f8)
    for name in (n for n in w_bf if n.endswith(".0")):
        d = np.abs(w_bf[name] - w_f8[name]).max()
        assert d <= 0.05 * np.abs(w_bf[name]).max() + 1e-3, (name, d)
    assert not np.array_equal(w_d["conv3.0"], w_f8["conv3.0"])


def test_quantiser_emulation_reference():
    """The emulated batch-innermost copies are the transposes of the NHWC quantisers' results, pad images zero; the dY
    sibling returns fp8_quant_grad's NHWC copy and masked dY; conv_wgrad_fp8 is the dequantised weight gradient."""
    from poseidon_b200.ops.emulate import EmulatedKernels
    k = EmulatedKernels()
    x = torch.randn(5, 24, 4, 3).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    s_a, s_t = torch.empty(1), torch.empty(1)
    q = k.fp8_quant_act(x, s_a)
    qt = k.fp8_quant_act_t(x, s_t)
    assert torch.equal(s_a, s_t) and qt.dtype == torch.float8_e4m3fn and tuple(qt.shape) == (24, 4, 3, 16)
    assert torch.equal(qt[..., :5].view(torch.uint8), q.permute(1, 2, 3, 0).contiguous().view(torch.uint8))
    assert int(qt[..., 5:].view(torch.uint8).count_nonzero()) == 0
    y = torch.randn(5, 24, 4, 3).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    g8, src = k.fp8_quant_grad(x, s_a, y, 0.1)
    gt, g8b, src_b = k.fp8_quant_grad_t(x, s_t, y, 0.1, True)
    assert torch.equal(s_a, s_t) and torch.equal(g8b.view(torch.uint8), g8.view(torch.uint8))
    assert torch.equal(src_b.view(torch.int16), src.view(torch.int16)) and gt.dtype == torch.float8_e5m2
    assert torch.equal(gt[..., :5].view(torch.uint8), g8.permute(1, 2, 3, 0).contiguous().view(torch.uint8))
    assert k.fp8_quant_grad_t(x, s_t, None, 0.0, False)[1].numel() == 0
    # the weight gradient of the dequantised copies, added onto dw with alpha
    xs = torch.empty(1)
    xx = torch.relu(torch.randn(3, 16, 6, 6)).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    dd = torch.randn(3, 8, 6, 6).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    x8t = k.fp8_quant_act_t(xx, xs)
    d8t, _, _ = k.fp8_quant_grad_t(dd, s_t, None, 0.0, False)
    dw = torch.ones(8, 9 * 16)
    k.conv_wgrad_fp8(d8t, x8t, s_t, xs, dw, [3, 3], [1, 1], 1, 0.5, 64)
    xd = x8t.float()[..., :3].permute(3, 0, 1, 2) * float(xs)
    dq = d8t.float()[..., :3].permute(3, 0, 1, 2) * float(s_t)
    ref = torch.nn.grad.conv2d_weight(xd, (8, 16, 3, 3), dq, 1, 1).permute(0, 2, 3, 1).reshape(8, -1)
    assert torch.allclose(dw, 1.0 + 0.5 * ref, rtol=1e-5, atol=1e-5)


def test_caffemodel_from_fp8_wgrad_run_resumes_without_fp8(emu, tmp_path):
    """fp8 tensors are derived and never saved: a snapshot written with fprop+dgrad+wgrad loads and resumes with fp8 off."""
    from poseidon_b200 import get_solver
    net = fp8_alex_net(batch=4)
    sp = _solver_param(net, 2)
    sp.snapshot_prefix = str(tmp_path / "f8w")
    s = get_solver(sp, engine="sm100", fp8=MODE)
    x, y = make_data(16, hw=27)
    feed(s, x, y)
    s.step(2)
    s.snapshot()
    ref = {n: l.export_blob(0) for n, l in zip(s.net.layer_names, s.net.layers) if len(l.blobs)}
    s2 = get_solver(sp, engine="sm100", fp8="off")
    s2.restore(str(tmp_path / "f8w_iter_2.solverstate"))
    for n, l in zip(s2.net.layer_names, s2.net.layers):
        if len(l.blobs):
            assert np.array_equal(l.export_blob(0), ref[n]), n
    assert not s2.net.layer_by_name["conv3"]._sm100.fp8_wgrad
    feed(s2, x, y)
    s2.step(1)
    assert s2.iter == 3 and np.isfinite(float(s2.last_loss))


# ------------------------------------------------------------------------------------------------ CPU: SASS
def test_wgrad_kernels_use_e5m2_wgmma_and_tiled_tma(sass):
    names = _demangle([k for k in sass if "wgmma_fp8_wgrad_kernel" in k])
    fp8 = {k: "\n".join(sass[k]) for k in names}
    assert len(fp8) == 4, sorted(names[k] for k in fp8)          # BN 64 / 128, single CTA / CTA pair
    for k, text in fp8.items():
        assert re.search(r"QGMMA\.64x(64|128)x32\.F32\.E5M2\.E4M3", text), names[k]
        assert "UTMALDG.3D" in text and "IM2COL" not in text, names[k]          # plain tiled boxes
        assert not re.search(r"\b(HMMA|HGMMA)", text), names[k]
        assert not re.search(r"\b(LDL|STL)\b", text), names[k]          # no local-memory spills
    pair = [t for k, t in fp8.items() if "(int)2>" in names[k]]
    assert len(pair) == 2 and all("UTMALDG.3D.MULTICAST" in t for t in pair), "CTA-pair multicast of the X tile"


def test_fp8_dgrad_instruction_streams_unchanged(sass):
    """The four e5m2 x e4m3 dgrad kernels compile to the instruction streams of the commit before the weight-gradient
    kernels were added (tests/golden/wgmma_fp8_dgrad_sass.json: sha256 of each kernel's SASS without addresses /
    encodings).  The bf16 and fprop kernels are held to their goldens by test_fp8_fprop.py / test_fp8_dgrad.py."""
    with open(GOLDEN_DGRAD_SASS) as f:
        golden = json.load(f)["kernels"]
    names = _demangle([k for k in sass if "wgmma_fp8_dgrad_kernel" in k])
    now = {d: sass[k] for k, d in names.items()}
    assert set(now) == set(golden), sorted(set(now) ^ set(golden))
    for n, g in golden.items():
        assert hashlib.sha256("\n".join(now[n]).encode()).hexdigest() == g["sha256"], n
        assert len(now[n]) == g["instructions"], n


# ================================================================================================ H100
gpu = pytest.mark.gpu


def _check_quant_act_t(ext, x):
    from poseidon_b200.ops.emulate import EmulatedKernels
    s = torch.empty(1, device="cuda")
    qt = ext.fp8_quant_act_t(x, s)
    s_ref = torch.empty(1)
    qt_ref = EmulatedKernels().fp8_quant_act_t(x.cpu(), s_ref)
    n = x.shape[0]
    assert qt.dtype == torch.float8_e4m3fn and qt.is_contiguous()
    assert tuple(qt.shape) == (x.shape[1], x.shape[2], x.shape[3], chwn_images(n))
    assert torch.equal(s.cpu(), s_ref), (float(s), float(s_ref))
    nan = torch.isnan(qt_ref.float())
    assert torch.equal(torch.isnan(qt.cpu().float()), nan)
    assert torch.equal(qt.cpu().view(torch.uint8)[~nan], qt_ref.view(torch.uint8)[~nan])
    assert int(qt[..., n:].view(torch.uint8).count_nonzero()) == 0          # pad images
    # bit for bit the transpose of the forward's x8 (same scale rule, same partial maxima)
    s_f = torch.empty(1, device="cuda")
    x8 = ext.fp8_quant_act(x, s_f)
    assert torch.equal(s_f, s)
    assert torch.equal(qt[..., :n].view(torch.uint8), x8.permute(1, 2, 3, 0).contiguous().view(torch.uint8))
    return qt, s


@gpu
@pytest.mark.parametrize("n,c,h,w,pitch,c_off", [
    (8, 96, 5, 6, None, 0),
    (32, 64, 7, 7, None, 0),
    (200, 40, 3, 5, None, 0),          # Np = 256: two image chunks of 128; C % 16 == 8
    (256, 128, 3, 3, None, 0),
    (32, 96, 6, 5, 256, 64),           # a channel slice of a concat slab
    (9, 40, 4, 4, 136, 88),            # pitched, C % 16 == 8, N not a multiple of 16
])
def test_quant_act_t_bitexact(ext, n, c, h, w, pitch, c_off):
    x = _nhwc_bf16(n, c, h, w, pitch=pitch, c_off=c_off, seed=n + c, scale=0.5)
    q1, s1 = _check_quant_act_t(ext, x)
    q2, s2 = _check_quant_act_t(ext, x)
    assert torch.equal(q1.view(torch.uint8), q2.view(torch.uint8)) and torch.equal(s1, s2)


def _check_quant_grad_t(ext, dy, y=None, slope=0.0):
    from poseidon_b200.ops.emulate import EmulatedKernels
    s = torch.empty(1, device="cuda")
    qt, q, src = ext.fp8_quant_grad_t(dy, s, y, slope, True)
    s_ref = torch.empty(1)
    qt_ref, _, src_ref = EmulatedKernels().fp8_quant_grad_t(dy.cpu(), s_ref, None if y is None else y.cpu(), slope, True)
    n = dy.shape[0]
    assert qt.dtype == torch.float8_e5m2 and tuple(qt.shape) == tuple(qt_ref.shape) and qt.is_contiguous()
    assert torch.equal(s.cpu(), s_ref), (float(s), float(s_ref))
    nan = torch.isnan(qt_ref.float())
    assert torch.equal(torch.isnan(qt.cpu().float()), nan)
    assert torch.equal(qt.cpu().view(torch.uint8)[~nan], qt_ref.view(torch.uint8)[~nan])
    assert int(qt[..., n:].view(torch.uint8).count_nonzero()) == 0
    # the NHWC copy and the masked dY are fp8_quant_grad's, bit for bit; without it, no NHWC copy
    s_g = torch.empty(1, device="cuda")
    q_g, src_g = ext.fp8_quant_grad(dy, s_g, y, slope)
    assert torch.equal(s_g, s) and q.stride() == q_g.stride() and tuple(q.shape) == tuple(q_g.shape)
    assert torch.equal(q.view(torch.uint8), q_g.view(torch.uint8))
    pitch8 = q.stride(3)
    if pitch8 != q.shape[1]:                          # the pad channels of the NHWC copy are zero, as fp8_quant_grad's
        whole = torch.as_strided(q, (n, pitch8, q.shape[2], q.shape[3]), q.stride())
        assert int(whole[:, q.shape[1]:].contiguous().view(torch.uint8).count_nonzero()) == 0
    assert torch.equal(src.view(torch.int16), src_g.view(torch.int16))
    if y is None:
        assert src.data_ptr() == dy.data_ptr()
    else:
        assert torch.equal(src.cpu().view(torch.int16), src_ref.view(torch.int16))
    qt2, none, _ = ext.fp8_quant_grad_t(dy, s, y, slope, False)
    assert none.numel() == 0 and torch.equal(qt2.view(torch.uint8), qt.view(torch.uint8))
    return qt, s, src


@gpu
@pytest.mark.parametrize("shape,pitch,c_off", [
    ((8, 384, 13, 13), None, 0),
    ((32, 24, 7, 5), None, 0),          # C % 16 == 8
    ((200, 64, 3, 3), None, 0),
    ((256, 128, 3, 3), None, 0),
    ((32, 96, 9, 9), 256, 64),          # a channel slice of a concat-slab gradient
])
def test_quant_grad_t_bitexact(ext, shape, pitch, c_off):
    dy = _nhwc_bf16(*shape, pitch=pitch, c_off=c_off, seed=sum(shape), scale=1e-3)
    q1, s1, _ = _check_quant_grad_t(ext, dy)
    q2, s2, _ = _check_quant_grad_t(ext, dy)
    assert torch.equal(q1.view(torch.uint8), q2.view(torch.uint8)) and torch.equal(s1, s2)


@gpu
@pytest.mark.parametrize("pitched", [False, True])
@pytest.mark.parametrize("slope", [0.0, 0.1])
def test_quant_grad_t_fused_mask_is_relu_bwd(ext, pitched, slope):
    shape = (8, 48, 7, 7)
    if pitched:
        dy = _nhwc_bf16(*shape, pitch=128, c_off=32, seed=5)
        y = _nhwc_bf16(*shape, pitch=96, c_off=16, seed=6)
        ref = ext.relu_bwd_nhwc(y, dy, slope)
    else:
        dy = _nhwc_bf16(*shape, seed=5)
        y = _nhwc_bf16(*shape, seed=6)
        ref = ext.relu_bwd(y, dy, slope)
    _, _, src = _check_quant_grad_t(ext, dy, y, slope)
    assert torch.equal(src.view(torch.int16), ref.view(torch.int16))


@gpu
def test_quant_t_zero_nan_inf(ext):
    z = torch.zeros(8, 32, 4, 4, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    qt, s, _ = _check_quant_grad_t(ext, z)
    assert float(s) == 1.0 and int(qt.view(torch.uint8).count_nonzero()) == 0
    qt, s = _check_quant_act_t(ext, z)
    assert float(s) == 1.0 and int(qt.view(torch.uint8).count_nonzero()) == 0
    dy = _nhwc_bf16(8, 48, 5, 5, seed=3).clone(memory_format=torch.channels_last)
    dy[1, 7, 2, 3] = float("nan")
    qt, _, _ = _check_quant_grad_t(ext, dy)
    assert torch.isnan(qt.float()[7, 2, 3, 1]) and int(torch.isnan(qt.float()).sum()) == 1
    qt, _ = _check_quant_act_t(ext, dy)
    assert torch.isnan(qt.float()[7, 2, 3, 1]) and int(torch.isnan(qt.float()).sum()) == 1
    dy[0, 0, 0, 0] = float("inf")
    qt, _, _ = _check_quant_grad_t(ext, dy)
    assert torch.isnan(qt.float()[0, 0, 0, 0])
    qt, _ = _check_quant_act_t(ext, dy)
    assert torch.isnan(qt.float()[0, 0, 0, 0])


def _ref_wgrad64(dy8t, s_dy, x8t, s_x, groups, k, pad):
    """float64 reference of the dequantised operands (on the GPU): (ref, Σ|a·b| per weight), [Cout, R*S*Cg]."""
    x = x8t.double().permute(3, 0, 1, 2) * float(s_x)
    d = dy8t.double().permute(3, 0, 1, 2) * float(s_dy)
    cout, cg = d.shape[1], x.shape[1] // groups
    shape = (cout, cg, k, k)
    ref = torch.nn.grad.conv2d_weight(x, shape, d, 1, pad, 1, groups)
    mag = torch.nn.grad.conv2d_weight(x.abs(), shape, d.abs(), 1, pad, 1, groups)
    return (ref.permute(0, 2, 3, 1).reshape(cout, -1).cpu(), mag.permute(0, 2, 3, 1).reshape(cout, -1).cpu())


@gpu
@pytest.mark.parametrize("pair", [1, 0])
@pytest.mark.parametrize("name,n,cin,h,w,cout,k,pad,groups,x_pitch", [
    ("alex_conv2", 16, 96, 27, 27, 256, 5, 2, 2, None),     # groups 2, Cg 48 -> 64 columns per tap
    ("alex_conv3_b256", 256, 256, 13, 13, 384, 3, 1, 1, None),
    ("vgg_conv5_b64", 64, 512, 14, 14, 512, 3, 1, 1, None),
    ("goog_1x1_slab", 32, 192, 14, 14, 64, 1, 0, 1, 480),   # X: a channel slice of a concat slab
    ("ragged", 32, 64, 9, 9, 128, 3, 1, 1, None),           # Np 32 x 4 columns: OW 9 leaves a partial column run
    ("n8", 8, 128, 12, 10, 256, 3, 1, 1, None),             # Np = 16: 8 columns per k block, rectangular
    ("n200", 200, 64, 6, 6, 128, 3, 1, 1, None),            # Np = 256: two image chunks per column
    ("longest_split", 64, 64, 224, 224, 64, 3, 1, 1, None),  # VGG-16 conv1_2 at b=64: ~61 k pixels per split
])
def test_conv_wgrad_fp8(ext, pair, name, n, cin, h, w, cout, k, pad, groups, x_pitch):
    ext.set_conv_pair(pair)
    try:
        cg = cin // groups
        cgk = (cg + 63) // 64 * 64
        oh, ow = h + 2 * pad - k + 1, w + 2 * pad - k + 1
        # X as a ReLU output (non-negative), dY of either sign: the operands of a real weight gradient
        x = _nhwc_bf16(n, cin, h, w, pitch=x_pitch, c_off=16 if x_pitch else 0, seed=n * cin + h).relu_()
        dy = _nhwc_bf16(n, cout, oh, ow, seed=cout + k, scale=1e-2)
        s_dy, s_x = torch.empty(1, device="cuda"), torch.empty(1, device="cuda")
        dy8t, _, _ = ext.fp8_quant_grad_t(dy, s_dy, None, 0.0, False)
        x8t = ext.fp8_quant_act_t(x, s_x)
        base = torch.randn(cout, k * k * cg, generator=torch.Generator().manual_seed(3)).cuda()
        alpha = 0.75
        dw = base.clone()
        ext.conv_wgrad_fp8(dy8t, x8t, s_dy, s_x, dw, [k, k], [pad, pad], groups, alpha, cgk)
        torch.cuda.synchronize()
        ref, mag = _ref_wgrad64(dy8t, s_dy, x8t, s_x, groups, k, pad)
        err = ((dw - base).cpu().double() - alpha * ref).abs()
        # fp32 accumulation of exact fp8 products, and the fp32 add onto dw
        bound = 2.0 ** -10 * alpha * mag + 2.0 ** -22 * base.abs().cpu().double() + 1e-30
        worst = float((err / bound).max())
        np_ = chwn_images(n)
        kb = oh * (-(-ow // (128 // np_)) if np_ < 128 else ow * np_ // 128)
        print(f"fp8 wgrad {name} pair={pair} k-blocks={kb}: err/bound {worst:.3f}, "
              f"max|dw-ref|/sum|ab| = {float((err / (alpha * mag).clamp(min=1e-30)).max()):.3e}")
        assert worst <= 1.0, (name, worst)
        dw2 = base.clone()
        ext.conv_wgrad_fp8(dy8t, x8t, s_dy, s_x, dw2, [k, k], [pad, pad], groups, alpha, cgk)
        assert torch.equal(dw2, dw)
    finally:
        ext.set_conv_pair(1)


@gpu
def test_conv_wgrad_fp8_rejects_what_it_cannot_run(ext):
    x = _nhwc_bf16(16, 64, 8, 8)
    dy = _nhwc_bf16(16, 128, 8, 8)
    s_dy, s_x = torch.empty(1, device="cuda"), torch.empty(1, device="cuda")
    dy8t, _, _ = ext.fp8_quant_grad_t(dy, s_dy, None, 0.0, False)
    x8t = ext.fp8_quant_act_t(x, s_x)
    dw = torch.zeros(128, 9 * 64, device="cuda")
    before = dw.clone()
    with pytest.raises(RuntimeError, match="e5m2"):
        ext.conv_wgrad_fp8(x8t, x8t, s_dy, s_x, dw, [3, 3], [1, 1], 1, 1.0, 64)
    with pytest.raises(RuntimeError, match="e4m3"):
        ext.conv_wgrad_fp8(dy8t, dy8t, s_dy, s_x, dw, [3, 3], [1, 1], 1, 1.0, 64)
    with pytest.raises(RuntimeError, match="stride-1"):                     # 8x8 -> 8x8 is not a 3x3 pad-0 output
        ext.conv_wgrad_fp8(dy8t, x8t, s_dy, s_x, dw, [3, 3], [0, 0], 1, 1.0, 64)
    with pytest.raises(RuntimeError, match="dw shape"):
        ext.conv_wgrad_fp8(dy8t, x8t, s_dy, s_x, torch.zeros(128, 9 * 32, device="cuda"), [3, 3], [1, 1], 1, 1.0, 64)
    with pytest.raises(RuntimeError, match="multiple of 64"):
        ext.conv_wgrad_fp8(dy8t, x8t, s_dy, s_x, dw, [3, 3], [1, 1], 1, 1.0, 96)
    with pytest.raises(RuntimeError, match="fp32 dw"):
        ext.conv_wgrad_fp8(dy8t, x8t, s_dy, s_x, dw.to(torch.bfloat16), [3, 3], [1, 1], 1, 1.0, 64)
    for setter, what in ((ext.set_conv_mcast, "set_conv_mcast"), (ext.set_conv_cluster, "set_conv_cluster")):
        setter(2)
        try:
            with pytest.raises(RuntimeError, match=what):
                ext.conv_wgrad_fp8(dy8t, x8t, s_dy, s_x, dw, [3, 3], [1, 1], 1, 1.0, 64)
        finally:
            setter(1)
    torch.cuda.synchronize()
    assert torch.equal(dw, before)                  # no device work ran


@gpu
@pytest.mark.parametrize("which", ["alex", "incep"])
def test_bf16_weight_gradients_unchanged(ext, which):
    """After one step, every bias and every weight of a layer with a bf16 weight gradient is the same bits under
    fprop+dgrad and fprop+dgrad+wgrad; the fp8-wgrad weights differ."""
    _, w_d, s1 = _run(which, "fprop+dgrad", 1)
    s1.close()
    _, w_w, s2 = _run(which, MODE, 1)
    fp8w = {n for n, l in zip(s2.net.layer_names, s2.net.layers)
            if getattr(l, "_sm100", None) is not None and getattr(l._sm100, "fp8_wgrad", False)}
    s2.close()
    assert fp8w == WGRAD_LAYERS[which]
    for key in w_d:
        layer, j = key.rsplit(".", 1)
        if j == "1" or layer not in fp8w:
            assert np.array_equal(w_d[key], w_w[key]), key
        else:
            assert not np.array_equal(w_d[key], w_w[key]), key


@gpu
@pytest.mark.parametrize("which", ["alex", "incep"])
def test_net_tracks_bf16_and_repeats(ext, which):
    """fp8=fprop+dgrad+wgrad trains: losses within 5 % of the bf16 engine over 4 steps; two runs give identical bits."""
    l_bf, _, s0 = _run(which, "off", 4)
    s0.close()
    l1, w1, s1 = _run(which, MODE, 4)
    s1.close()
    l2, w2, s2 = _run(which, MODE, 4)
    s2.close()
    print(f"{which}: bf16 losses {l_bf}, fp8 {MODE} losses {l1}")
    for a, b in zip(l_bf, l1):
        assert abs(a - b) <= 0.05 * max(1.0, abs(a)), (l_bf, l1)
    assert l1 == l2
    for n in w1:
        assert np.array_equal(w1[n], w2[n]), n


@gpu
@pytest.mark.parametrize("which", ["alex", "incep"])
def test_graph_replay_requantises(ext, which):
    """Under CUDA-graph replay the fp8 weight gradient follows each step's dY and X: the X scale moves from replay to
    replay, two graph runs give identical bits, and they track the eager run."""
    layer_name = "conv3" if which == "alex" else "b3x3"

    def run(graph):
        from poseidon_b200 import get_solver
        fn, hw = NETS[which]
        sp = small_solver_param(fn(batch=8, classes=16, hw=hw), max_iter=6)
        s = get_solver(sp, engine="sm100", fp8=MODE)
        x, y = make_data(8 * 6, classes=16, hw=hw)
        feed(s, x, y)
        if graph:
            s.enable_cuda_graph(warmup=2)
        st = s.net.layer_by_name[layer_name]._sm100
        assert st.fp8_wgrad
        scales = []
        while s.iter < 6:
            s.step(1)
            torch.cuda.synchronize()
            scales.append((float(st.s_xw), float(st.s_dy)))
        graphed = getattr(s, "_graph", None) is not None
        out = {n: l.export_blob(0) for n, l in zip(s.net.layer_names, s.net.layers) if len(l.blobs)}
        loss = float(s.last_loss)
        s.close()
        return out, loss, scales, graphed

    w_e, l_e, sc_e, g_e = run(False)
    w_g, l_g, sc_g, g_g = run(True)
    w_g2, l_g2, sc_g2, _ = run(True)
    assert not g_e and g_g
    assert sc_g[-1] != sc_g[-2] and sc_g == sc_g2                # re-quantised on every replay
    assert l_g == l_g2 and all(np.array_equal(w_g[n], w_g2[n]) for n in w_g)
    assert abs(l_e - l_g) < 0.05 * max(1.0, abs(l_e)), (l_e, l_g)
    for n in w_e:
        d = np.abs(w_e[n] - w_g[n]).max()
        assert d <= 0.02 * np.abs(w_e[n]).max() + 1e-4, (n, d)
