"""Delayed scaling for the fp8 convolutions: the opt-in ``fp8_scaling="delayed"`` setting.

CPU (no GPU needed): how the setting resolves and its plumbing, the plan line, the emulated amax rings (seeding, the
15-slot window, recording, wrap-around), an emulated training run against the bf16 emulation, the quantiser launches per
step, the test-phase rule, the capture guard, and the SASS of the new kernels.
H100: each delayed quantiser's seeding call bit for bit against the just-in-time op, the steady state against a torch
reference (saturation included) on grids of hundreds of CTAs, ring consistency, NaN / Inf / zero inputs, the one-pass
x8 / x8ᵀ pair, and whole nets (loss tracking, repeatability, CUDA-graph replay)."""
import re

import numpy as np
import pytest
import torch

from smallnet import feed, make_data, small_solver_param
from test_fp8_fprop import (  # noqa: F401  (_keep_dropout_counters: autouse fixture, restores the dropout counters)
    NETS, _demangle, _keep_dropout_counters, _nhwc_bf16, _plan, _run, _solver_param, emu, fp8_alex_net, sass)

MODE = "fprop+dgrad+wgrad"
H = 16                     # AMAX_HISTORY
E4M3_MAX, E5M2_MAX = 448.0, 57344.0


def _hist(ring):
    return ring[:H].view(torch.float32)


def _pos(ring):
    return int(ring[H])


def _new_ring(device="cpu"):
    from poseidon_b200.ops import sm100
    return torch.zeros(sm100._RING_WORDS, dtype=torch.int32, device=device)


def _set_ring(ring, values, pos):
    _hist(ring).copy_(torch.tensor(values, dtype=torch.float32))
    ring[H] = pos


# ------------------------------------------------------------------------------------------------ CPU: the setting
def test_setting_resolution(monkeypatch):
    from poseidon_b200.ops import sm100
    monkeypatch.delenv("POSEIDON_FP8_SCALING", raising=False)
    assert sm100.AMAX_HISTORY == H
    assert sm100.resolve_fp8_scaling(None, MODE) == "current" and sm100.resolve_fp8_scaling(None, "off") == "current"
    assert sm100.resolve_fp8_scaling("DELAYED", "fprop") == "delayed"
    monkeypatch.setenv("POSEIDON_FP8_SCALING", "delayed")
    assert sm100.resolve_fp8_scaling(None, "fprop+dgrad") == "delayed"
    assert sm100.resolve_fp8_scaling(None, "off") == "current"          # the variable applies only with fp8 on
    assert sm100.resolve_fp8_scaling("current", MODE) == "current"
    with pytest.raises(ValueError, match="needs an fp8 mode"):
        sm100.resolve_fp8_scaling("delayed", "off")
    assert sm100.fp8_scaling_for_engine("torch", "off") == "current"
    assert sm100.fp8_scaling_for_engine("torch", "off", "current") == "current"
    with pytest.raises(ValueError, match="sm100"):
        sm100.fp8_scaling_for_engine("torch", "off", "delayed")
    for bad in ("late", "jit", "amax"):
        with pytest.raises(ValueError, match="fp8_scaling must be one of"):
            sm100.resolve_fp8_scaling(bad, MODE)
        with pytest.raises(ValueError, match="fp8_scaling must be one of"):
            sm100.fp8_scaling_for_engine("torch", "off", bad)
    monkeypatch.setenv("POSEIDON_FP8_SCALING", "late")
    assert sm100.resolve_fp8_scaling(None, "off") == "current"
    with pytest.raises(ValueError, match="fp8_scaling must be one of"):
        sm100.resolve_fp8_scaling(None, "fprop")


def test_get_solver_engine_and_cli_plumbing(emu, tmp_path, monkeypatch):
    monkeypatch.delenv("POSEIDON_FP8", raising=False)
    monkeypatch.delenv("POSEIDON_FP8_SCALING", raising=False)
    from poseidon_b200 import get_solver
    from poseidon_b200 import proto as P
    from poseidon_b200.engine import CaffeEngine
    from poseidon_b200.tools import caffe_main
    sp = _solver_param(fp8_alex_net(batch=2), 1)
    s = get_solver(sp, engine="sm100", fp8=MODE, fp8_scaling="delayed")
    assert s.fp8_scaling == "delayed" and s.net.ctx.fp8_scaling == "delayed"
    assert all(n.ctx.fp8_scaling == "delayed" for n in getattr(s, "test_nets", []))
    assert s.net.layer_by_name["conv3"]._sm100.fp8_delayed
    assert not s.net.layer_by_name["conv1"]._sm100.fp8_delayed          # no fp8 pass: nothing to scale
    assert get_solver(sp, engine="sm100", fp8=MODE).fp8_scaling == "current"
    assert not get_solver(sp, engine="sm100", fp8=MODE).net.layer_by_name["conv3"]._sm100.fp8_delayed
    with pytest.raises(ValueError, match="needs an fp8 mode"):
        get_solver(sp, engine="sm100", fp8="off", fp8_scaling="delayed")
    with pytest.raises(ValueError, match="sm100"):
        get_solver(sp, engine="torch", fp8_scaling="delayed", dtype=torch.float32)
    eng = CaffeEngine(sp, engine="sm100", fp8=MODE, fp8_scaling="delayed")
    assert eng.build().fp8_scaling == "delayed"
    eng.close()
    monkeypatch.setenv("POSEIDON_FP8", "fprop")
    monkeypatch.setenv("POSEIDON_FP8_SCALING", "delayed")
    assert get_solver(sp, engine="sm100").fp8_scaling == "delayed"
    assert get_solver(sp, engine="sm100", fp8="off").fp8_scaling == "current"
    monkeypatch.delenv("POSEIDON_FP8")
    monkeypatch.delenv("POSEIDON_FP8_SCALING")
    a = caffe_main.parse_args(["train", "--solver=s.prototxt", "--fp8", MODE, "--fp8_scaling", "delayed"])
    assert a.fp8_scaling == "delayed"
    assert caffe_main.parse_args(["train", "--solver=s.prototxt"]).fp8_scaling is None
    with pytest.raises(SystemExit):
        caffe_main.parse_args(["train", "--fp8_scaling", "late"])
    help_text = caffe_main.make_parser().format_help().replace("\n", " ")
    assert "--fp8_scaling {current,delayed}" in help_text and "POSEIDON_FP8_SCALING" in help_text
    model = tmp_path / "net.prototxt"
    model.write_text(P.to_text(fp8_alex_net(batch=2)) if hasattr(P, "to_text") else str(fp8_alex_net(batch=2)))
    args = caffe_main.parse_args(["test", f"--model={model}", "--engine=sm100", f"--fp8={MODE}",
                                  "--fp8_scaling=delayed", "--gpu=-1"])
    net, _ = caffe_main._build_net(args, P.TEST)
    assert net.ctx.fp8_scaling == "delayed" and net.layer_by_name["conv3"]._sm100.fp8_delayed
    args = caffe_main.parse_args(["test", f"--model={model}", "--engine=torch", "--fp8_scaling=delayed", "--gpu=-1"])
    with pytest.raises(ValueError, match="sm100"):
        caffe_main._build_net(args, P.TEST)
    args = caffe_main.parse_args(["test", f"--model={model}", "--engine=sm100", "--fp8_scaling=delayed", "--gpu=-1"])
    with pytest.raises(ValueError, match="needs an fp8 mode"):
        caffe_main._build_net(args, P.TEST)


def _plan_lines(caplog, mode, scaling):
    import logging
    from poseidon_b200 import proto as P
    from poseidon_b200.layers import NetContext
    from poseidon_b200.net.net import Net
    caplog.clear()
    ctx = NetContext(phase=P.TRAIN, device="cpu", engine="sm100", dtype=torch.bfloat16, fp8=mode, fp8_scaling=scaling)
    with caplog.at_level(logging.INFO, logger="poseidon_b200"):
        Net(fp8_alex_net(batch=2), phase=P.TRAIN, ctx=ctx)
    return [r.getMessage() for r in caplog.records if r.getMessage().startswith("sm100 plan: conv ")]


def test_plan_line_gains_the_scaling(emu, caplog, monkeypatch):
    monkeypatch.delenv("POSEIDON_FP8_SCALING", raising=False)
    for mode in ("fprop", "fprop+dgrad", MODE):
        cur = _plan_lines(caplog, mode, None)
        assert len(cur) == 5 and not any("scaling" in l for l in cur)
        assert _plan_lines(caplog, mode, "current") == cur
        delayed = _plan_lines(caplog, mode, "delayed")
        assert delayed == [l + "; scaling delayed" for l in cur]


# ------------------------------------------------------------------------------------------------ CPU: the rings
def test_emulated_rings():
    """Seeding scales like the just-in-time op and fills every slot; a steady-state call scales from the 15 other slots
    (saturating beyond their amax), records its own amax into its slot and advances; the position wraps at 16."""
    from poseidon_b200.ops.emulate import EmulatedKernels
    k = EmulatedKernels()
    x = torch.randn(5, 24, 4, 3).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    amax = float(x.float().abs().max())
    ring, s, s_ref = _new_ring(), torch.empty(1), torch.empty(1)
    q = k.fp8_quant_act_delayed(x, s, ring, True)
    ref = k.fp8_quant_act(x, s_ref)
    assert torch.equal(s, s_ref) and torch.equal(q.view(torch.uint8), ref.view(torch.uint8))
    assert q.stride() == ref.stride()
    assert torch.equal(_hist(ring), torch.full((H,), amax)) and _pos(ring) == 1
    # steady state: window = the 15 slots other than the position; the position's own (larger) value does not count
    vals = [0.5] * H
    vals[3] = 100.0
    vals[7] = 0.25 * amax                   # the window's amax: x is 4x beyond it and saturates
    vals = [min(v, 0.25 * amax) if i != 3 else v for i, v in enumerate(vals)]
    _set_ring(ring, vals, 3)
    q = k.fp8_quant_act_delayed(x, s, ring, False)
    sc = torch.div(torch.tensor(E4M3_MAX), torch.tensor(0.25 * amax, dtype=torch.float32))
    assert torch.equal(s, torch.div(torch.tensor(1.0), sc).reshape(1))
    exp = torch.clamp(x.float() * sc, -E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    assert torch.equal(q.view(torch.uint8), exp.view(torch.uint8))
    assert int((q.float().abs() == E4M3_MAX).sum()) > 0
    assert float(_hist(ring)[3]) == amax and _pos(ring) == 4
    # the dY ops, the batch-innermost copies and the wrap-around
    y = torch.randn(5, 24, 4, 3).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    dring, tring = _new_ring(), _new_ring()
    for i in range(H + 3):
        dy = (x.float() * (i + 1)).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        q8, src = k.fp8_quant_grad_delayed(dy, s, dring, i == 0, y, 0.1)
        qt, q8b, src_t = k.fp8_quant_grad_t_delayed(dy, s_ref, tring, i == 0, y, 0.1, True)
        assert torch.equal(s, s_ref) and torch.equal(q8.view(torch.uint8), q8b.view(torch.uint8))
        assert torch.equal(qt[..., :5].view(torch.uint8), q8.permute(1, 2, 3, 0).contiguous().view(torch.uint8))
        assert torch.equal(src.view(torch.int16), src_t.view(torch.int16))
        assert float(_hist(dring)[i % H]) == float(src.float().abs().max()) and _pos(dring) == (i + 1) % H
    assert torch.equal(dring, tring)
    xt, x8 = k.fp8_quant_act_t_delayed(x, s, _new_ring(), True, True)
    assert torch.equal(xt[..., :5].view(torch.uint8), x8.permute(1, 2, 3, 0).contiguous().view(torch.uint8))
    assert k.fp8_quant_act_t_delayed(x, s, _new_ring(), True, False)[1].numel() == 0


def _quant_counts():
    from poseidon_b200.ops import counting
    return {n: c for n, c in counting.by_op().items() if n.startswith("fp8_quant_")}


def test_emulated_step_tracks_bf16(emu, monkeypatch):
    """Delayed scaling on the emulated kernels: losses within 5 % (and at least 0.05) of the bf16 emulation over 3 steps;
    one quantiser launch per scaled tensor and step, and no X quantiser in the backward of a layer whose forward is fp8."""
    from poseidon_b200.ops import counting
    l_bf, w_bf, _ = _run("alex", "off", 3)
    monkeypatch.setenv("POSEIDON_FP8_SCALING", "delayed")
    counting.reset()
    l_d, w_d, s = _run("alex", MODE, 3)
    for a, b in zip(l_bf, l_d):
        assert abs(a - b) <= 0.05 * max(1.0, abs(a)), (l_bf, l_d)
    for name in (n for n in w_bf if n.endswith(".0")):
        d = np.abs(w_bf[name] - w_d[name]).max()
        assert d <= 0.05 * np.abs(w_bf[name]).max() + 1e-3, (name, d)
    st = {n: s.net.layer_by_name[n]._sm100 for n in ("conv1", "conv2", "conv3", "conv4", "conv5")}
    assert [(st[n].fp8, st[n].fp8_wgrad) for n in st] == \
        [(False, False), (False, True), (True, True), (True, True), (True, False)]
    keys = {n: sorted(st[n].amax_rings) for n in st}
    assert keys == {"conv1": [], "conv2": ["dy", "xw"], "conv3": ["dy", "x"], "conv4": ["dy", "x"], "conv5": ["x"]}
    for n in st:
        for ring, seeded in st[n].amax_rings.values():
            assert seeded and _pos(ring) == 3
    # per step: one x8 + x8t launch each for conv3 / conv4 (fp8 forward and weight gradient), x8t for conv2 in its
    # backward (bf16 forward), x8 for conv5 (strided: fp8 forward only), one dY launch each for conv2-conv4
    assert _quant_counts() == {"fp8_quant_weight": 9, "fp8_quant_weight_dgrad": 6, "fp8_quant_act_t_delayed": 9,
                               "fp8_quant_act_delayed": 3, "fp8_quant_grad_t_delayed": 9}, _quant_counts()


def test_test_phase_forward_leaves_the_rings(emu, monkeypatch):
    """A test net shares the train net's ConvState: its forwards (and any forward without autograd) scale just in time
    and neither read nor advance the training rings."""
    from poseidon_b200 import get_solver
    from poseidon_b200 import proto as P
    from poseidon_b200.net.net import Net
    from poseidon_b200.ops import counting
    sp = _solver_param(fp8_alex_net(batch=4), 2)
    s = get_solver(sp, engine="sm100", fp8=MODE, fp8_scaling="delayed")
    x, y = make_data(8, hw=27)
    feed(s, x, y)
    s.step(2)
    before = {(n, key): t.clone() for n, l in s.net.layer_by_name.items() if getattr(l, "_sm100", None) is not None
              and hasattr(l._sm100, "amax_rings") for key, (t, _) in l._sm100.amax_rings.items()}
    assert len(before) == 7
    tn = Net(fp8_alex_net(batch=4), phase=P.TEST, ctx=s._ctx(P.TEST))
    tn.share_trained_layers_with(s.net)
    assert tn.layer_by_name["conv3"]._sm100 is s.net.layer_by_name["conv3"]._sm100
    for layer in tn.layers:
        if layer.type_name == "MEMORY_DATA":
            layer.reset(x, y)
    counting.reset()
    tn.forward()                             # test phase, autograd on
    with torch.no_grad():
        s.net.forward()                      # training net, no autograd
    assert _quant_counts() == {"fp8_quant_weight": 6, "fp8_quant_act": 6}, _quant_counts()
    for (n, key), t in before.items():
        assert torch.equal(s.net.layer_by_name[n]._sm100.amax_rings[key][0], t), (n, key)


def test_capture_of_an_unseeded_ring_fails(emu, monkeypatch):
    from poseidon_b200 import get_solver
    from poseidon_b200.ops import sm100
    sp = _solver_param(fp8_alex_net(batch=4), 2)
    s = get_solver(sp, engine="sm100", fp8=MODE, fp8_scaling="delayed")
    x, y = make_data(8, hw=27)
    feed(s, x, y)
    monkeypatch.setattr(sm100, "_capturing", lambda: True)
    with pytest.raises(RuntimeError, match="unseeded amax history"):
        s.step(1)
    assert all(not l._sm100.amax_rings.get("x", [None, False])[1] for l in s.net.layers
               if getattr(l, "_sm100", None) is not None and hasattr(l._sm100, "amax_rings"))
    monkeypatch.setattr(sm100, "_capturing", lambda: False)
    s2 = get_solver(sp, engine="sm100", fp8=MODE, fp8_scaling="delayed")
    feed(s2, x, y)
    s2.step(1)                                   # seeded on an eager step: a capture may now reach every ring
    monkeypatch.setattr(sm100, "_capturing", lambda: True)
    s2.step(1)
    assert _pos(s2.net.layer_by_name["conv3"]._sm100.amax_rings["x"][0]) == 2


def test_restore_seeds_again(emu, tmp_path):
    """Histories are not in the snapshot: a restored solver seeds them on its first step."""
    from poseidon_b200 import get_solver
    sp = _solver_param(fp8_alex_net(batch=4), 3)
    sp.snapshot_prefix = str(tmp_path / "dl")
    s = get_solver(sp, engine="sm100", fp8=MODE, fp8_scaling="delayed")
    x, y = make_data(12, hw=27)
    feed(s, x, y)
    s.step(2)
    s.snapshot()
    s.restore(str(tmp_path / "dl_iter_2.solverstate"))
    assert all(not l._sm100.amax_rings for l in s.net.layers if hasattr(getattr(l, "_sm100", None), "amax_rings"))
    s.step(1)
    assert _pos(s.net.layer_by_name["conv3"]._sm100.amax_rings["x"][0]) == 1


# ------------------------------------------------------------------------------------------------ CPU: SASS
def test_delayed_kernels_do_not_spill(sass):
    names = _demangle([k for k in sass if "delayed_kernel" in k])
    assert len(names) == 8, sorted(names.values())          # NHWC / batch-innermost x e4m3 / e5m2 x mask
    for k, d in names.items():
        text = "\n".join(sass[k])
        assert not re.search(r"\b(LDL|STL)\b", text), d


# ================================================================================================ H100
gpu = pytest.mark.gpu

SHAPES = [
    ((8, 96, 5, 6), None, 0),
    ((3, 24, 7, 5), None, 0),              # C % 16 == 8
    ((200, 40, 3, 5), None, 0),            # Np = 256
    ((32, 96, 6, 5), 256, 64),             # a channel slice of a concat slab
    ((9, 40, 4, 4), 136, 88),              # pitched, C % 16 == 8
]


def _same(a, b):
    assert a.dtype == b.dtype and tuple(a.shape) == tuple(b.shape) and a.stride() == b.stride()
    assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def _seeded_ring_ok(ring, amax):
    r = ring.cpu()
    assert torch.equal(_hist(r), torch.full((H,), amax)) and _pos(r) == 1 and int(r[H + 1]) == 0 and int(r[H + 2]) == 0


@gpu
@pytest.mark.parametrize("shape,pitch,c_off", SHAPES)
def test_seeding_matches_current_act(ext, shape, pitch, c_off):
    x = _nhwc_bf16(*shape, pitch=pitch, c_off=c_off, seed=sum(shape), scale=0.5)
    amax = float(x.float().abs().max())
    s_c, s_d = torch.empty(1, device="cuda"), torch.empty(1, device="cuda")
    q_c = ext.fp8_quant_act(x, s_c)
    ring = _new_ring("cuda")
    _same(ext.fp8_quant_act_delayed(x, s_d, ring, True), q_c)
    assert torch.equal(s_c, s_d)
    _seeded_ring_ok(ring, amax)
    qt_c = ext.fp8_quant_act_t(x, s_c)
    for nhwc in (False, True):
        ring = _new_ring("cuda")
        qt, q = ext.fp8_quant_act_t_delayed(x, s_d, ring, True, nhwc)
        _same(qt, qt_c)
        assert torch.equal(s_c, s_d)
        _seeded_ring_ok(ring, amax)
        if nhwc:
            _same(q, q_c)
            pitch8 = q.stride(3)
            if pitch8 != q.shape[1]:             # the pad channels of the NHWC copy are zero, as fp8_quant_act's
                whole = torch.as_strided(q, (q.shape[0], pitch8, q.shape[2], q.shape[3]), q.stride())
                assert int(whole[:, q.shape[1]:].contiguous().view(torch.uint8).count_nonzero()) == 0
        else:
            assert q.numel() == 0


@gpu
@pytest.mark.parametrize("slope", [None, 0.0, 0.1])
@pytest.mark.parametrize("shape,pitch,c_off", SHAPES)
def test_seeding_matches_current_grad(ext, shape, pitch, c_off, slope):
    dy = _nhwc_bf16(*shape, pitch=pitch, c_off=c_off, seed=sum(shape) + 1, scale=1e-3)
    y = None if slope is None else _nhwc_bf16(*shape, pitch=pitch and pitch + 16, c_off=c_off, seed=7)
    sl = slope or 0.0
    s_c, s_d = torch.empty(1, device="cuda"), torch.empty(1, device="cuda")
    q_c, src_c = ext.fp8_quant_grad(dy, s_c, y, sl)
    amax = float(src_c.float().abs().max())
    ring = _new_ring("cuda")
    q, src = ext.fp8_quant_grad_delayed(dy, s_d, ring, True, y, sl)
    _same(q, q_c)
    assert torch.equal(s_c, s_d) and torch.equal(src.view(torch.int16), src_c.view(torch.int16))
    _seeded_ring_ok(ring, amax)
    for nhwc in (False, True):
        qt_c, _, _ = ext.fp8_quant_grad_t(dy, s_c, y, sl, nhwc)
        ring = _new_ring("cuda")
        qt, q, src = ext.fp8_quant_grad_t_delayed(dy, s_d, ring, True, y, sl, nhwc)
        _same(qt, qt_c)
        assert torch.equal(s_c, s_d) and torch.equal(src.view(torch.int16), src_c.view(torch.int16))
        _seeded_ring_ok(ring, amax)
        if nhwc:
            _same(q, q_c)
        if y is None:
            assert src.data_ptr() == dy.data_ptr()


def _steady_cases(ext, x, y=None, slope=0.0, seed=False):
    """{name: (run(ring, s) -> (outputs to compare, the bf16 dY cast), fp8 dtype, MAX)} for every delayed op."""
    def act(ring, s):
        return [ext.fp8_quant_act_delayed(x, s, ring, seed)], x

    def act_t(ring, s):
        qt, q = ext.fp8_quant_act_t_delayed(x, s, ring, seed, True)
        return [q, qt], x

    def grad(ring, s):
        q, src = ext.fp8_quant_grad_delayed(x, s, ring, seed, y, slope)
        return [q], src

    def grad_t(ring, s):
        qt, q, src = ext.fp8_quant_grad_t_delayed(x, s, ring, seed, y, slope, True)
        return [q, qt], src
    return {"act": (act, torch.float8_e4m3fn, E4M3_MAX), "act_t": (act_t, torch.float8_e4m3fn, E4M3_MAX),
            "grad": (grad, torch.float8_e5m2, E5M2_MAX), "grad_t": (grad_t, torch.float8_e5m2, E5M2_MAX)}


def _inv_scale(fmax, window):
    """1 / s as the kernels store it, s = MAX / window (an fp32 division)."""
    return torch.div(torch.tensor(1.0), torch.div(torch.tensor(fmax), torch.tensor(window, dtype=torch.float32))).reshape(1)


def _check_steady(outs, v, window, dtype, fmax, s_out):
    """One scale for the whole tensor: q == fp8(clamp(v * s)), s = MAX / window (an fp32 division)."""
    sc = torch.div(torch.tensor(fmax), torch.tensor(window, dtype=torch.float32))
    assert torch.equal(s_out.cpu(), torch.div(torch.tensor(1.0), sc).reshape(1))
    ref = torch.clamp(v.float().cpu() * sc, -fmax, fmax).to(dtype)
    q = outs[0].cpu()
    assert torch.equal(q.view(torch.uint8), ref.view(torch.uint8))
    if len(outs) > 1:
        n = v.shape[0]
        assert torch.equal(outs[1][..., :n].cpu().view(torch.uint8), q.permute(1, 2, 3, 0).contiguous().view(torch.uint8))
        assert int(outs[1][..., n:].view(torch.uint8).count_nonzero()) == 0


@gpu
@pytest.mark.parametrize("masked", [False, True])
def test_steady_state_matches_reference(ext, masked):
    """A ring set by hand: the window is the 15 slots other than the position (whose larger value must not count); the
    input's amax is 4x the window's, so its large values saturate, and the recorded amax is the true one.  The tensor
    (64 x 256 x 14 x 14) spreads over hundreds of CTAs (784 NHWC, 1568 batch-innermost): one scale for all of them."""
    x = _nhwc_bf16(64, 256, 14, 14, pitch=288, c_off=16, seed=21, scale=0.5)
    y = _nhwc_bf16(64, 256, 14, 14, seed=22) if masked else None
    for name, (run, dtype, fmax) in _steady_cases(ext, x, y, 0.1).items():
        if masked and name.startswith("act"):
            continue
        v = x if y is None or not name.startswith("grad") else ext.relu_bwd_nhwc(y, x, 0.1)
        amax = float(v.float().abs().max())
        window = amax / 4
        vals = [window * (0.25 + 0.05 * i) for i in range(H)]
        vals[9] = window
        vals[5] = 50 * amax                       # the position's own slot: outside the window
        ring = _new_ring("cuda")
        _set_ring(ring, vals, 5)
        s = torch.empty(1, device="cuda")
        outs, src = run(ring, s)
        _check_steady(outs, v, window, dtype, fmax, s)
        assert int((outs[0].float().abs() == fmax).sum()) > 100, name       # saturated
        if y is not None:
            assert torch.equal(src.view(torch.int16), v.contiguous(memory_format=torch.channels_last).view(torch.int16))
        r = ring.cpu()
        assert float(_hist(r)[5]) == amax and _pos(r) == 6 and int(r[H + 1]) == 0 and int(r[H + 2]) == 0, name
        vals[5] = amax
        assert torch.equal(_hist(r), torch.tensor(vals, dtype=torch.float32)), name


@gpu
def test_ring_advances_once_per_call_and_wraps(ext):
    base = _nhwc_bf16(32, 128, 9, 9, seed=4)
    calls = 2 * H + 3
    for name in ("act", "act_t", "grad", "grad_t"):
        ring, s = _new_ring("cuda"), torch.empty(1, device="cuda")
        amaxes = []
        for i in range(calls):
            x = (base.float() * (1 + i % 5)).to(torch.bfloat16)
            _steady_cases(ext, x, seed=i == 0)[name][0](ring, s)
            amaxes.append(float(x.float().abs().max()))
            r = ring.cpu()
            assert _pos(r) == (i + 1) % H and int(r[H + 1]) == 0 and int(r[H + 2]) == 0, (name, i)
            assert float(_hist(r)[i % H]) == amaxes[-1], (name, i)
        h = _hist(ring.cpu())                     # the amaxes of the last 16 calls, each in its slot
        for i in range(calls - H, calls):
            assert float(h[i % H]) == amaxes[i], (name, i)


@gpu
def test_nonfinite_and_zero(ext):
    """NaN stays NaN and is not recorded; +Inf becomes NaN in the call that sees it and is recorded, so the next calls
    scale with 0 (1 / s = inf: the GEMM output turns non-finite) while it is in the window; all-zero inputs scale with 1
    and record 0."""
    x = _nhwc_bf16(8, 48, 5, 5, seed=3).clone(memory_format=torch.channels_last)
    amax = float(x.float().abs().max())
    z = torch.zeros(8, 48, 5, 5, device="cuda", dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    for name in ("act", "act_t", "grad", "grad_t"):
        _, dtype, fmax = _steady_cases(ext, x)[name]
        ring, s = _new_ring("cuda"), torch.empty(1, device="cuda")
        _set_ring(ring, [amax] * H, 0)
        xn = x.clone(memory_format=torch.channels_last)
        xn[1, 7, 2, 3] = float("nan")
        f = _steady_cases(ext, xn)[name][0](ring, s)[0][0].float()
        assert torch.isnan(f[1, 7, 2, 3]) and int(torch.isnan(f).sum()) == 1, name
        assert float(_hist(ring.cpu())[0]) == float(xn.float().nan_to_num(0.0).abs().max()), name
        xi = x.clone(memory_format=torch.channels_last)
        xi[0, 0, 0, 0] = float("inf")
        f = _steady_cases(ext, xi)[name][0](ring, s)[0][0].float()
        assert torch.isnan(f[0, 0, 0, 0]) and int(torch.isnan(f).sum()) == 1, name
        assert torch.equal(s.cpu(), _inv_scale(fmax, amax)), name
        assert float(_hist(ring.cpu())[1]) == float("inf"), name
        for _ in range(H - 1):                   # the Inf slot stays in the window for the next 15 calls
            q = _steady_cases(ext, x)[name][0](ring, s)[0][0]
            assert float(s) == float("inf") and float(q.float().abs().max()) == 0.0, name       # +-0
        q = _steady_cases(ext, x)[name][0](ring, s)[0][0]     # ... and is overwritten by the 16th
        assert torch.equal(s.cpu(), _inv_scale(fmax, amax)), name
        zr = _new_ring("cuda")
        for _ in range(3):
            q = _steady_cases(ext, z)[name][0](zr, s)[0][0]
            assert float(s) == 1.0 and int(q.view(torch.uint8).count_nonzero()) == 0, name
        assert int(zr[:H].count_nonzero()) == 0 and _pos(zr.cpu()) == 3


@gpu
@pytest.mark.parametrize("which", ["alex", "incep"])
def test_net_tracks_bf16_and_repeats(ext, which, monkeypatch):
    """Delayed scaling trains: losses within 5 % of the bf16 engine over 4 steps; two runs give identical bits; the
    rings advanced once per step; the backward ran no X quantiser for layers whose forward is fp8."""
    from poseidon_b200.ops import counting
    l_bf, _, s0 = _run(which, "off", 4)
    s0.close()
    monkeypatch.setenv("POSEIDON_FP8_SCALING", "delayed")
    counting.reset()
    l1, w1, s1 = _run(which, MODE, 4)
    counts = counting.by_op()
    sts = [l._sm100 for l in s1.net.layers if l.type_name == "CONVOLUTION"]
    for st in sts:
        for ring, seeded in st.amax_rings.values():
            assert seeded and _pos(ring.cpu()) == 4
    fwd_t = sum(1 for st in sts if st.fp8 and st.fp8_wgrad)
    bwd_t = sum(1 for st in sts if st.fp8_wgrad and not st.fp8)
    assert counts.get("fp8_quant_act_t_delayed", 0) == 4 * (fwd_t + bwd_t) and fwd_t > 0
    assert "fp8_quant_act_t" not in counts and "fp8_quant_act" not in counts and "fp8_quant_grad_t" not in counts
    s1.close()
    l2, w2, s2 = _run(which, MODE, 4)
    s2.close()
    print(f"{which}: bf16 losses {l_bf}, fp8 {MODE} delayed losses {l1}")
    for a, b in zip(l_bf, l1):
        assert abs(a - b) <= 0.05 * max(1.0, abs(a)), (l_bf, l1)
    assert l1 == l2
    for n in w1:
        assert np.array_equal(w1[n], w2[n]), n


@gpu
@pytest.mark.parametrize("which", ["alex", "incep"])
def test_graph_replay_advances_the_rings(ext, which, monkeypatch):
    """Under CUDA-graph replay the rings advance on every replay; two graph runs give identical bits and track the
    eager run."""
    monkeypatch.setenv("POSEIDON_FP8_SCALING", "delayed")
    layer_name = "conv3" if which == "alex" else "b3x3"

    def run(graph):
        from poseidon_b200 import get_solver
        fn, hw = NETS[which]
        sp = small_solver_param(fn(batch=8, classes=16, hw=hw), max_iter=6)
        s = get_solver(sp, engine="sm100", fp8=MODE)
        assert s.fp8_scaling == "delayed"
        x, y = make_data(8 * 6, classes=16, hw=hw)
        feed(s, x, y)
        if graph:
            s.enable_cuda_graph(warmup=2)
        st = s.net.layer_by_name[layer_name]._sm100
        trace = []
        while s.iter < 6:
            s.step(1)
            torch.cuda.synchronize()
            trace.append(({k: _pos(r.cpu()) for k, (r, _) in st.amax_rings.items()}, float(st.s_x), float(st.s_dy)))
        graphed = getattr(s, "_graph", None) is not None
        out = {n: l.export_blob(0) for n, l in zip(s.net.layer_names, s.net.layers) if len(l.blobs)}
        loss = float(s.last_loss)
        s.close()
        return out, loss, trace, graphed

    w_e, l_e, tr_e, g_e = run(False)
    w_g, l_g, tr_g, g_g = run(True)
    w_g2, l_g2, tr_g2, _ = run(True)
    assert not g_e and g_g
    assert [t[0] for t in tr_g] == [{"x": i, "dy": i} for i in range(4, 7)], tr_g     # 3 eager steps, then replays
    assert [t[0] for t in tr_e] == [{"x": i, "dy": i} for i in range(1, 7)], tr_e
    assert tr_g == tr_g2
    assert l_g == l_g2 and all(np.array_equal(w_g[n], w_g2[n]) for n in w_g)
    assert abs(l_e - l_g) < 0.05 * max(1.0, abs(l_e)), (l_e, l_g)
    for n in w_e:
        d = np.abs(w_e[n] - w_g[n]).max()
        assert d <= 0.02 * np.abs(w_e[n]).max() + 1e-4, (n, d)
