"""fp8 data gradients (e5m2 dY x e4m3 weights) for stride-1 convolutions: the opt-in ``fp8="fprop+dgrad"`` setting.

CPU (no GPU needed): the eligibility rule on the zoo nets, the "off" / "fprop" plans unchanged, the setting's plumbing,
an emulated training run against the bf16 emulation, checkpoints, and the SASS of the built extension.
H100: the quantisers bit for bit against the torch reference, conv_dgrad_fp8 against a float64 reference of the
dequantised operands, weight / bias gradients unchanged, and whole nets (loss tracking, repeatability, CUDA-graph replay)."""
import hashlib
import json
import os
import re

import numpy as np
import pytest
import torch

from smallnet import feed, make_data, small_solver_param
from test_fp8_fprop import (  # noqa: F401  (_keep_dropout_counters: autouse fixture, restores the dropout counters)
    _demangle, _keep_dropout_counters, _nhwc_bf16, _plan, _run, _sass_by_function, _solver_param, emu, fp8_alex_net,
    sass)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_FP8_SASS = os.path.join(ROOT, "tests", "golden", "wgmma_fp8_fprop_sass.json")

# layers of the small nets (tests/test_fp8_fprop.py) whose data gradient runs in fp8
DGRAD_LAYERS = {"alex": {"conv2", "conv3"}, "incep": {"b1x1", "b3x3", "mix"}}


# ------------------------------------------------------------------------------------------------ CPU: the plan
def test_dgrad_eligibility_alexnet(emu):
    from poseidon_b200.models import zoo
    st = _plan(zoo.alexnet(batch=2, test_batch=2), emu, fp8="fprop+dgrad")
    assert {n for n, s in st.items() if s.fp8_dgrad} == {"conv2", "conv3", "conv4", "conv5"}
    assert {n for n, s in st.items() if s.fp8} == {"conv3", "conv4", "conv5"}        # conv2: fp8 dgrad, bf16 fprop
    assert "first-layer" in st["conv1"].fp8_dgrad_reason
    assert [st[n].cok8 for n in ("conv2", "conv3", "conv4", "conv5")] == [128, 384, 256, 128]
    assert st["conv4"].mask_input and st["conv5"].mask_input                          # the mask epilogue
    assert st["conv2"].fp8_dgrad_reason == "Cout_g 128 -> 128 slots"


def test_dgrad_eligibility_vgg16(emu):
    from poseidon_b200.models import zoo
    st = _plan(zoo.vgg16(batch=1, test_batch=1), emu, fp8="fprop+dgrad")
    assert {n for n, s in st.items() if not s.fp8_dgrad} == {"conv1_1", "conv1_2"}
    assert "third" in st["conv1_2"].fp8_dgrad_reason
    assert len([s for s in st.values() if s.fp8_dgrad]) == 11


def test_dgrad_eligibility_googlenet(emu):
    from poseidon_b200.models import zoo
    st = _plan(zoo.googlenet(batch=1, test_batch=1), emu, fp8="fprop+dgrad")
    fp8_out = {s.Cout // s.groups for s in st.values() if s.fp8_dgrad}
    bf16_out = {s.Cout // s.groups for s in st.values() if not s.fp8_dgrad and tuple(s.layer.stride) == (1, 1)}
    assert fp8_out == {96, 112, 128, 192, 208, 224, 256, 288, 320, 384}, sorted(fp8_out)
    assert bf16_out == {16, 24, 32, 48, 64, 144, 160}, sorted(bf16_out)
    assert len([s for s in st.values() if s.fp8_dgrad]) == 32 and len(st) == 59
    assert len([s for s in st.values() if s.fp8_dgrad and s.mask_input]) == 14
    assert all(tuple(s.layer.stride) == (1, 1) and not s.row_mode for s in st.values() if s.fp8_dgrad)


def test_off_and_fprop_plans_unchanged(emu):
    from poseidon_b200.models import zoo
    for mode in ("off", "fprop"):
        for s in _plan(zoo.alexnet(batch=2, test_batch=2), emu, fp8=mode).values():
            assert not s.fp8_dgrad and s.cok8 == 0 and s.fp8_dgrad_reason == "fp8 dgrad off"
    a = _plan(zoo.googlenet(batch=1, test_batch=1), emu, fp8="fprop")
    b = _plan(zoo.googlenet(batch=1, test_batch=1), emu, fp8="fprop+dgrad")
    assert {n: (s.fp8, s.fp8_reason, s.cgk8) for n, s in a.items()} == {n: (s.fp8, s.fp8_reason, s.cgk8) for n, s in b.items()}


def _plan_lines(emu, caplog, mode):
    import logging
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="poseidon_b200"):
        _plan(fp8_alex_net(batch=2), emu, fp8=mode)
    return [r.getMessage() for r in caplog.records if r.getMessage().startswith("sm100 plan: conv ")]


def test_plan_log_gives_the_dgrad_decision(emu, caplog):
    fprop = _plan_lines(emu, caplog, "fprop")
    assert len(fprop) == 5 and not any("dgrad" in l for l in fprop)
    both = _plan_lines(emu, caplog, "fprop+dgrad")
    assert len(both) == 5
    for a, b in zip(fprop, both):
        assert b.startswith(a + "; dgrad "), (a, b)
    assert both[2].endswith("; dgrad fp8 (Cout_g 192 -> 256 slots)"), both[2]
    assert both[4].endswith("; dgrad bf16 (strided (bf16 phase decomposition))"), both[4]


# ------------------------------------------------------------------------------------------------ CPU: the setting
def test_setting_resolution(monkeypatch):
    from poseidon_b200.ops import sm100
    monkeypatch.setenv("POSEIDON_FP8", "fprop+dgrad")
    assert sm100.resolve_fp8() == "fprop+dgrad" and sm100.resolve_fp8("FPROP+DGRAD") == "fprop+dgrad"
    assert sm100.fp8_for_engine("torch") == "off"
    with pytest.raises(ValueError, match="sm100"):
        sm100.fp8_for_engine("torch", "fprop+dgrad")
    for bad in ("e5m2", "dgrad"):
        with pytest.raises(ValueError, match="fp8 must be one of"):
            sm100.resolve_fp8(bad)


def test_get_solver_engine_and_cli_plumbing(emu, tmp_path, monkeypatch):
    monkeypatch.delenv("POSEIDON_FP8", raising=False)
    from poseidon_b200 import get_solver
    from poseidon_b200 import proto as P
    from poseidon_b200.engine import CaffeEngine
    from poseidon_b200.tools import caffe_main
    sp = _solver_param(fp8_alex_net(batch=2), 1)
    s = get_solver(sp, engine="sm100", fp8="fprop+dgrad")
    assert s.fp8 == "fprop+dgrad" and s.net.ctx.fp8 == "fprop+dgrad"
    assert s.net.layer_by_name["conv3"]._sm100.fp8_dgrad and s.net.layer_by_name["conv3"]._sm100.fp8
    with pytest.raises(ValueError, match="sm100"):
        get_solver(sp, engine="torch", fp8="fprop+dgrad", dtype=torch.float32)
    eng = CaffeEngine(sp, engine="sm100", fp8="fprop+dgrad")
    assert eng.build().fp8 == "fprop+dgrad"
    eng.close()
    monkeypatch.setenv("POSEIDON_FP8", "fprop+dgrad")
    assert get_solver(sp, engine="sm100").fp8 == "fprop+dgrad"
    monkeypatch.delenv("POSEIDON_FP8")
    assert caffe_main.parse_args(["train", "--solver=s.prototxt", "--fp8", "fprop+dgrad"]).fp8 == "fprop+dgrad"
    model = tmp_path / "net.prototxt"
    model.write_text(P.to_text(fp8_alex_net(batch=2)) if hasattr(P, "to_text") else str(fp8_alex_net(batch=2)))
    args = caffe_main.parse_args(["test", f"--model={model}", "--engine=sm100", "--fp8=fprop+dgrad", "--gpu=-1"])
    net, _ = caffe_main._build_net(args, P.TEST)
    assert net.ctx.fp8 == "fprop+dgrad" and net.layer_by_name["conv2"]._sm100.fp8_dgrad
    args = caffe_main.parse_args(["test", f"--model={model}", "--engine=torch", "--fp8=fprop+dgrad", "--gpu=-1"])
    with pytest.raises(ValueError, match="sm100"):
        caffe_main._build_net(args, P.TEST)


# ------------------------------------------------------------------------------------------------ CPU: emulation
def test_emulated_step_tracks_bf16(emu):
    """fp8=fprop+dgrad on the emulated kernels: losses within 5 % (and at least 0.05) of the bf16 emulation over 3 steps."""
    l_bf, w_bf, _ = _run("alex", "off", 3)
    l_f8, w_f8, s = _run("alex", "fprop+dgrad", 3)
    assert all(s.net.layer_by_name[n]._sm100.fp8_dgrad for n in DGRAD_LAYERS["alex"])
    for a, b in zip(l_bf, l_f8):
        assert abs(a - b) <= 0.05 * max(1.0, abs(a)), (l_bf, l_f8)
    for name in (n for n in w_bf if n.endswith(".0")):
        d = np.abs(w_bf[name] - w_f8[name]).max()
        assert d <= 0.05 * np.abs(w_bf[name]).max() + 1e-3, (name, d)


def test_quantiser_emulation_reference():
    """The emulated quantisers: scale = 57344 / amax, clamp then cast, NaN stays NaN, zero gives scale 1, the masked dY
    is relu_bwd's; the dgrad weights follow conv_pack_dgrad's order with one scale per input channel."""
    from poseidon_b200.ops.emulate import EmulatedKernels
    k = EmulatedKernels()
    dy = torch.randn(2, 24, 5, 3).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    dy[0, 3, 1, 1] = float("nan")
    s = torch.empty(1)
    q, src = k.fp8_quant_grad(dy, s, None, 0.0)
    assert src is dy and q.dtype == torch.float8_e5m2 and tuple(q.shape) == (2, 24, 5, 3) and q.stride(3) == 32
    amax = dy.float().abs().nan_to_num(0.0).max()
    assert torch.equal(s, torch.div(torch.tensor(1.0), torch.div(torch.tensor(57344.0), amax)).reshape(1))
    assert torch.isnan(q.float()[0, 3, 1, 1]) and int(torch.isnan(q.float()).sum()) == 1
    assert float(q.float().nan_to_num(0.0).abs().max()) == 57344.0
    y = torch.randn(2, 24, 5, 3).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    q, src = k.fp8_quant_grad(dy, s, y, 0.25)
    assert torch.equal(src.view(torch.int16), k.relu_bwd(y, dy, 0.25).view(torch.int16))
    z = torch.zeros(1, 8, 2, 2, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    assert float(k.fp8_quant_grad(z, s, None, 0.0)[0].float().abs().max()) == 0.0 and float(s) == 1.0
    w = torch.randn(12, 40, 3, 3).contiguous(memory_format=torch.channels_last)      # groups 2: Cout_g 6, Cg 40
    s_w = torch.empty(80)
    w8 = k.fp8_quant_weight_dgrad(w, 2, 128, s_w)
    assert tuple(w8.shape) == (80, 9 * 128)
    assert float(w8.float().reshape(80, 9, 128)[..., 6:].abs().max()) == 0.0
    back = w8.float().reshape(80, 9, 128)[..., :6] * s_w.view(80, 1, 1)
    ref = k.conv_pack_dgrad(w.permute(0, 2, 3, 1).reshape(-1), 12, 9, 40, 2, None, 0).float().reshape(80, 9, 6)
    ref32 = w.reshape(2, 6, 40, 9).permute(0, 2, 3, 1).reshape(80, 9, 6)
    assert torch.equal(ref, ref32.to(torch.bfloat16).float())
    assert float(((back - ref32).abs() / ref32.abs().amax(dim=(1, 2), keepdim=True)).max()) <= 2 ** -4


def test_caffemodel_from_fp8_dgrad_run_resumes_without_fp8(emu, tmp_path):
    """fp8 tensors are derived and never saved: a snapshot written with fprop+dgrad loads and resumes with fp8 off."""
    from poseidon_b200 import get_solver
    net = fp8_alex_net(batch=4)
    sp = _solver_param(net, 2)
    sp.snapshot_prefix = str(tmp_path / "f8d")
    s = get_solver(sp, engine="sm100", fp8="fprop+dgrad")
    x, y = make_data(16, hw=27)
    feed(s, x, y)
    s.step(2)
    s.snapshot()
    ref = {n: l.export_blob(0) for n, l in zip(s.net.layer_names, s.net.layers) if len(l.blobs)}
    s2 = get_solver(sp, engine="sm100", fp8="off")
    s2.restore(str(tmp_path / "f8d_iter_2.solverstate"))
    for n, l in zip(s2.net.layer_names, s2.net.layers):
        if len(l.blobs):
            assert np.array_equal(l.export_blob(0), ref[n]), n
    assert not s2.net.layer_by_name["conv3"]._sm100.fp8_dgrad
    feed(s2, x, y)
    s2.step(1)
    assert s2.iter == 3 and np.isfinite(float(s2.last_loss))


# ------------------------------------------------------------------------------------------------ CPU: SASS
def test_dgrad_kernels_use_e5m2_wgmma_and_im2col_tma(sass):
    names = _demangle([k for k in sass if "wgmma_fp8_dgrad_kernel" in k])
    fp8 = {k: "\n".join(sass[k]) for k in names}
    assert len(fp8) == 4, sorted(names[k] for k in fp8)          # BN 64 / 128, single CTA / CTA pair
    for k, text in fp8.items():
        assert re.search(r"QGMMA\.64x(64|128)x32\.F32\.E5M2\.E4M3", text), names[k]
        assert "UTMALDG.4D.IM2COL" in text, names[k]
        assert not re.search(r"\b(HMMA|HGMMA)", text), names[k]
    pair = [t for k, t in fp8.items() if "(int)2>" in names[k]]
    assert len(pair) == 2 and all("UTMALDG.2D.MULTICAST" in t for t in pair), "CTA-pair multicast of the weight tile"


def test_fp8_fprop_instruction_streams_unchanged(sass):
    """The four e4m3 fprop kernels compile to the instruction streams of the commit before the data-gradient kernels were
    added (tests/golden/wgmma_fp8_fprop_sass.json: sha256 of each kernel's SASS without addresses / encodings)."""
    with open(GOLDEN_FP8_SASS) as f:
        golden = json.load(f)["kernels"]
    names = _demangle([k for k in sass if "wgmma_fp8_conv_kernel" in k])
    now = {d: sass[k] for k, d in names.items()}
    assert set(now) == set(golden), sorted(set(now) ^ set(golden))
    for n, g in golden.items():
        assert hashlib.sha256("\n".join(now[n]).encode()).hexdigest() == g["sha256"], n
        assert len(now[n]) == g["instructions"], n


# ================================================================================================ H100
gpu = pytest.mark.gpu


def _check_quant_grad(ext, dy, y=None, slope=0.0):
    from poseidon_b200.ops.emulate import EmulatedKernels
    s = torch.empty(1, device="cuda")
    q, src = ext.fp8_quant_grad(dy, s, y, slope)
    s_ref = torch.empty(1)
    q_ref, src_ref = EmulatedKernels().fp8_quant_grad(dy.cpu(), s_ref, None if y is None else y.cpu(), slope)
    assert q.dtype == torch.float8_e5m2 and tuple(q.shape) == tuple(dy.shape)
    assert q.stride(1) == 1 and q.stride(3) == (dy.shape[1] + 15) // 16 * 16
    assert torch.equal(s.cpu(), s_ref), (float(s), float(s_ref))
    nan = torch.isnan(q_ref.float())
    assert torch.equal(torch.isnan(q.cpu().float()), nan)
    assert torch.equal(q.cpu().view(torch.uint8)[~nan], q_ref.view(torch.uint8)[~nan])
    if y is None:
        assert src.data_ptr() == dy.data_ptr()
    else:
        assert src.is_contiguous(memory_format=torch.channels_last)
        assert torch.equal(src.cpu().view(torch.int16), src_ref.view(torch.int16))
    return q, s, src


@gpu
@pytest.mark.parametrize("shape,pitch,c_off", [
    ((4, 384, 13, 13), None, 0),        # AlexNet conv4 output gradient
    ((3, 24, 7, 5), None, 0),           # C % 16 == 8: one pad half per pixel
    ((2, 96, 9, 9), 256, 64),           # a channel slice of a concat-slab gradient
    ((2, 40, 6, 6), 136, 88),           # pitched, C % 16 == 8
])
def test_quant_grad_bitexact(ext, shape, pitch, c_off):
    dy = _nhwc_bf16(*shape, pitch=pitch, c_off=c_off, seed=sum(shape), scale=1e-3)
    q1, s1, _ = _check_quant_grad(ext, dy)
    q2, s2, _ = _check_quant_grad(ext, dy)
    assert torch.equal(q1.view(torch.uint8), q2.view(torch.uint8)) and torch.equal(s1, s2)


@gpu
@pytest.mark.parametrize("pitched", [False, True])
@pytest.mark.parametrize("slope", [0.0, 0.1])
def test_quant_grad_fused_mask_is_relu_bwd(ext, pitched, slope):
    """The masked dY the amax pass writes is relu_bwd's (dense) / relu_bwd_nhwc's (concat-slab slices), bit for bit."""
    shape = (3, 48, 7, 7)
    if pitched:
        dy = _nhwc_bf16(*shape, pitch=128, c_off=32, seed=5)
        y = _nhwc_bf16(*shape, pitch=96, c_off=16, seed=6)
        ref = ext.relu_bwd_nhwc(y, dy, slope)
    else:
        dy = _nhwc_bf16(*shape, seed=5)
        y = _nhwc_bf16(*shape, seed=6)
        ref = ext.relu_bwd(y, dy, slope)
    q, s, src = _check_quant_grad(ext, dy, y, slope)
    assert torch.equal(src.view(torch.int16), ref.view(torch.int16))
    assert int((src.float() == 0).sum()) > 0 if slope == 0.0 else True


@gpu
def test_quant_grad_zero_nan_inf(ext):
    z = torch.zeros(2, 32, 4, 4, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    q, s, _ = _check_quant_grad(ext, z)
    assert float(s) == 1.0 and int(q.view(torch.uint8).count_nonzero()) == 0
    dy = _nhwc_bf16(2, 48, 5, 5, seed=3).clone(memory_format=torch.channels_last)
    dy[1, 7, 2, 3] = float("nan")
    q, _, _ = _check_quant_grad(ext, dy)
    assert torch.isnan(q.float()[1, 7, 2, 3]) and int(torch.isnan(q.float()).sum()) == 1
    dy[0, 0, 0, 0] = float("inf")
    q, _, _ = _check_quant_grad(ext, dy)
    assert torch.isnan(q.float()[0, 0, 0, 0])


@gpu
@pytest.mark.parametrize("cout,cg,k,groups,cok", [(384, 256, 3, 1, 384), (384, 192, 3, 2, 256), (192, 480, 1, 1, 256),
                                                  (256, 48, 5, 2, 128), (64, 24, 3, 1, 128)])
def test_quant_weight_dgrad_bitexact(ext, cout, cg, k, groups, cok):
    from poseidon_b200.ops.emulate import EmulatedKernels
    g = torch.Generator(device="cpu").manual_seed(cout + cg)
    w = (torch.randn(cout, cg, k, k, generator=g) * 0.03).contiguous(memory_format=torch.channels_last)
    w[:, 1].zero_()                                    # input channel 1 of every group: scale 1
    w[2, 3, 0, 0] = float("nan")
    s = torch.empty(groups * cg, device="cuda")
    w8 = ext.fp8_quant_weight_dgrad(w.cuda(), groups, cok, s)
    s_ref = torch.empty(groups * cg)
    w8_ref = EmulatedKernels().fp8_quant_weight_dgrad(w, groups, cok, s_ref)
    assert torch.equal(s.cpu(), s_ref) and float(s_ref[1]) == 1.0
    nan = torch.isnan(w8_ref.float())
    assert int(nan.sum()) == 1 and torch.equal(torch.isnan(w8.cpu().float()), nan)
    assert torch.equal(w8.cpu().view(torch.uint8)[~nan], w8_ref.view(torch.uint8)[~nan])
    w8b = ext.fp8_quant_weight_dgrad(w.cuda(), groups, cok, s)
    assert torch.equal(w8.view(torch.uint8), w8b.view(torch.uint8))


def _ref_dgrad64(dy8, s_dy, wt8, s_wt, groups, k, pad, H, W, mask):
    """float64 reference of the dequantised operands: (ref, Σ|a·b| per output) after the mask."""
    import torch.nn.functional as F
    cin = wt8.shape[0]
    cg = cin // groups
    cout = dy8.shape[1]
    cout_g = cout // groups
    cok = wt8.shape[1] // (k * k)
    dyd = dy8.cpu().double() * float(s_dy)
    w = wt8.cpu().double().reshape(groups, cg, k, k, cok)[..., :cout_g] * s_wt.cpu().double().view(groups, cg, 1, 1, 1)
    w4 = w.permute(0, 4, 1, 2, 3).reshape(cout, cg, k, k)
    pre = F.conv_transpose2d(dyd, w4, None, 1, 0, 0, groups)[:, :, pad: pad + H, pad: pad + W]
    mag = F.conv_transpose2d(dyd.abs(), w4.abs(), None, 1, 0, 0, groups)[:, :, pad: pad + H, pad: pad + W]
    if mask is not None:
        keep = mask.cpu().double() > 0
        pre, mag = torch.where(keep, pre, pre * 0.0), torch.where(keep, mag, mag * 0.0)
    return pre, mag


SENTINEL = -7.25


@gpu
@pytest.mark.parametrize("pair", [1, 0])
@pytest.mark.parametrize("name,n,cin,h,cout,k,pad,groups,masked,dy_pitch", [
    ("alex_conv2", 4, 96, 27, 256, 5, 2, 2, False, None),     # Cg 48: 48-channel dX slices per group
    ("alex_conv4", 4, 384, 13, 384, 3, 1, 2, True, None),     # Cout_g 192 -> 256 slots, producer mask
    ("vgg_512", 2, 512, 14, 512, 3, 1, 1, True, None),        # K = 4608
    ("goog_1x1", 5, 480, 14, 192, 1, 0, 1, False, 512),       # dY: a channel slice of a concat-slab gradient
    ("ragged", 3, 128, 11, 128, 3, 1, 1, False, None),        # N*H*W = 363: partial last pixel block
])
def test_conv_dgrad_fp8(ext, pair, name, n, cin, h, cout, k, pad, groups, masked, dy_pitch):
    ext.set_conv_pair(pair)
    try:
        cg = cin // groups
        cout_g = cout // groups
        cok = (cout_g + 127) // 128 * 128
        oh = h + 2 * pad - k + 1
        dy = _nhwc_bf16(n, cout, oh, oh, pitch=dy_pitch, c_off=16 if dy_pitch else 0, seed=n * cin + h, scale=1e-2)
        g = torch.Generator(device="cpu").manual_seed(cout + k)
        w = (torch.randn(cout, cg, k, k, generator=g) * 0.05).contiguous(memory_format=torch.channels_last).cuda()
        s_dy, s_wt = torch.empty(1, device="cuda"), torch.empty(cin, device="cuda")
        wt8 = ext.fp8_quant_weight_dgrad(w, groups, cok, s_wt)
        dy8, _ = ext.fp8_quant_grad(dy, s_dy, None, 0.0)
        mask = _nhwc_bf16(n, cin, h, h, seed=77).clone(memory_format=torch.channels_last) if masked else None
        # the caching allocator hands dX the block just filled with the sentinel: every element must be overwritten
        numel = n * cin * h * h
        poison = torch.full((numel,), SENTINEL, dtype=torch.bfloat16, device="cuda")
        poison_ptr = poison.data_ptr()
        del poison
        dx = ext.conv_dgrad_fp8(dy8, wt8, s_dy, s_wt, [k, k], [pad, pad], groups, h, h, mask, 0.0)
        torch.cuda.synchronize()
        assert dx.dtype == torch.bfloat16 and tuple(dx.shape) == (n, cin, h, h)
        assert dx.is_contiguous(memory_format=torch.channels_last)
        if dx.data_ptr() == poison_ptr:
            assert int((dx == SENTINEL).sum()) == 0, "dX elements left unwritten"
        ref, mag = _ref_dgrad64(dy8, s_dy, wt8, s_wt, groups, k, pad, h, h, mask)
        err = (dx.cpu().double() - ref).abs()
        # bf16 output rounding (2^-9 relative, with margin) + fp32 accumulation of exact fp8 products at the 2^-10 level
        bound = 2.0 ** -8 * ref.abs() + 2.0 ** -10 * mag + 1e-30
        worst = float((err / bound).max())
        print(f"fp8 dgrad {name} pair={pair} K={k * k * cok}: err/bound {worst:.3f}, "
              f"max|dx-ref|/sum|ab| = {float((err / mag.clamp(min=1e-30)).max()):.3e}")
        assert worst <= 1.0, (name, worst)
        if mask is not None:
            assert int((dx[mask <= 0] != 0).sum()) == 0
        dx2 = ext.conv_dgrad_fp8(dy8, wt8, s_dy, s_wt, [k, k], [pad, pad], groups, h, h, mask, 0.0)
        assert torch.equal(dx2.view(torch.int16), dx.view(torch.int16))
    finally:
        ext.set_conv_pair(1)


@gpu
def test_conv_dgrad_fp8_rejects_what_it_cannot_run(ext):
    dy = _nhwc_bf16(2, 64, 8, 8)
    s_dy, s_wt = torch.empty(1, device="cuda"), torch.empty(128, device="cuda")
    dy8, _ = ext.fp8_quant_grad(dy, s_dy, None, 0.0)
    w = torch.randn(64, 128, 3, 3).contiguous(memory_format=torch.channels_last).cuda()
    wt8_bad = ext.fp8_quant_weight_dgrad(w, 1, 192, s_wt)                  # 192 slots: not a multiple of 128
    with pytest.raises(RuntimeError, match="multiple of 128"):
        ext.conv_dgrad_fp8(dy8, wt8_bad, s_dy, s_wt, [3, 3], [1, 1], 1, 8, 8, None, 0.0)
    wt8 = ext.fp8_quant_weight_dgrad(w, 1, 128, s_wt)
    with pytest.raises(RuntimeError, match="stride-1"):
        ext.conv_dgrad_fp8(dy8, wt8, s_dy, s_wt, [3, 3], [1, 1], 1, 16, 16, None, 0.0)
    with pytest.raises(RuntimeError, match="e5m2"):
        ext.conv_dgrad_fp8(dy.contiguous(memory_format=torch.channels_last), wt8, s_dy, s_wt, [3, 3], [1, 1], 1, 8, 8,
                           None, 0.0)
    bad_mask = _nhwc_bf16(2, 128, 8, 8, pitch=256)
    with pytest.raises(RuntimeError, match="mask must match"):
        ext.conv_dgrad_fp8(dy8, wt8, s_dy, s_wt, [3, 3], [1, 1], 1, 8, 8, bad_mask, 0.0)
    for setter, what in ((ext.set_conv_mcast, "set_conv_mcast"), (ext.set_conv_cluster, "set_conv_cluster")):
        setter(2)
        try:
            with pytest.raises(RuntimeError, match=what):
                ext.conv_dgrad_fp8(dy8, wt8, s_dy, s_wt, [3, 3], [1, 1], 1, 8, 8, None, 0.0)
        finally:
            setter(1)


# per small net: the topmost fp8-dgrad layer and the learnable layers above it.  Their dY does not depend on any fp8 data
# gradient, so after one step their weights and biases are the same under fprop and fprop+dgrad.  "mix" masks its own dY
# (its consumer is a pooling layer that cannot): the fused mask + amax pass writes the dY its weight gradient reads.
TOP_DGRAD = {"alex": ("conv3", ("conv3", "conv4", "conv5", "fc6"), "conv2"), "incep": ("mix", ("mix", "fc"), "b3x3")}


@gpu
@pytest.mark.parametrize("which", ["alex", "incep"])
def test_weight_and_bias_gradients_unchanged(ext, which):
    top, same, below = TOP_DGRAD[which]
    _, w_f, s1 = _run(which, "fprop", 1)
    s1.close()
    _, w_d, s2 = _run(which, "fprop+dgrad", 1)
    st = s2.net.layer_by_name[top]._sm100
    assert st.fp8_dgrad and (which == "alex" or not st.consumer_masks)
    s2.close()
    for n in same:
        for j in (0, 1):
            assert np.array_equal(w_f[f"{n}.{j}"], w_d[f"{n}.{j}"]), f"{n}.{j}"
    assert not np.array_equal(w_f[f"{below}.0"], w_d[f"{below}.0"])      # the fp8 data gradient does reach below


@gpu
@pytest.mark.parametrize("which", ["alex", "incep"])
def test_net_tracks_bf16_and_repeats(ext, which):
    """fp8=fprop+dgrad trains: losses within 5 % of the bf16 engine over 4 steps; two runs give identical bits."""
    l_bf, _, s0 = _run(which, "off", 4)
    s0.close()
    l1, w1, s1 = _run(which, "fprop+dgrad", 4)
    assert all(s1.net.layer_by_name[n]._sm100.fp8_dgrad for n in DGRAD_LAYERS[which])
    s1.close()
    l2, w2, s2 = _run(which, "fprop+dgrad", 4)
    s2.close()
    print(f"{which}: bf16 losses {l_bf}, fp8 fprop+dgrad losses {l1}")
    for a, b in zip(l_bf, l1):
        assert abs(a - b) <= 0.05 * max(1.0, abs(a)), (l_bf, l1)
    assert l1 == l2
    for n in w1:
        assert np.array_equal(w1[n], w2[n]), n


@gpu
@pytest.mark.parametrize("which", ["alex", "incep"])
def test_graph_replay_requantises_the_updated_master(ext, which):
    """Under CUDA-graph replay the e4m3 dgrad weights follow the optimizer: after every step the per-input-channel scales
    are those of the master as it was before the step.  Two graph runs give identical bits and track the eager run."""
    from poseidon_b200.ops.emulate import EmulatedKernels
    layer_name = "conv3" if which == "alex" else "b3x3"

    def run(graph):
        l, w, s = None, None, None
        from poseidon_b200 import get_solver
        from test_fp8_fprop import NETS
        fn, hw = NETS[which]
        sp = small_solver_param(fn(batch=8, classes=16, hw=hw), max_iter=6)
        s = get_solver(sp, engine="sm100", fp8="fprop+dgrad")
        x, y = make_data(8 * 6, classes=16, hw=hw)
        feed(s, x, y)
        if graph:
            s.enable_cuda_graph(warmup=2)
        layer = s.net.layer_by_name[layer_name]
        st = layer._sm100
        scales = []
        while s.iter < 6:
            w_before = layer.weight.detach().float().cpu().contiguous(memory_format=torch.channels_last)
            s.step(1)
            torch.cuda.synchronize()
            ref = torch.empty(st.Cp)
            EmulatedKernels().fp8_quant_weight_dgrad(w_before, st.groups, st.cok8, ref)
            scales.append((st.s_wt.cpu().clone(), ref))
        graphed = getattr(s, "_graph", None) is not None
        out = {n: l.export_blob(0) for n, l in zip(s.net.layer_names, s.net.layers) if len(l.blobs)}
        loss = float(s.last_loss)
        s.close()
        return out, loss, scales, graphed

    w_e, l_e, sc_e, g_e = run(False)
    w_g, l_g, sc_g, g_g = run(True)
    w_g2, l_g2, _, _ = run(True)
    assert not g_e and g_g
    for got, ref in sc_g + sc_e:
        assert torch.equal(got, ref)
    assert not torch.equal(sc_g[-1][0], sc_g[-2][0])            # the scales do move from replay to replay
    assert l_g == l_g2 and all(np.array_equal(w_g[n], w_g2[n]) for n in w_g)
    assert abs(l_e - l_g) < 0.05 * max(1.0, abs(l_e)), (l_e, l_g)
    for n in w_e:
        d = np.abs(w_e[n] - w_g[n]).max()
        assert d <= 0.02 * np.abs(w_e[n]).max() + 1e-4, (n, d)
