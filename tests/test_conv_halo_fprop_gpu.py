"""The halo-tiled forward (halo_fprop_kernel, csrc/gemm/halo_conv.cuh) behind conv_fprop: bit-identical to the gather
schedule (set_conv_halo_fprop(0)) and within the float64 bound test_conv_contract_gpu.py uses for conv_fprop.

AlexNet conv2 at batch 256 takes the halo forward by default; the small edge geometries run it forced
(set_conv_halo_fprop(2)), since by default problems with fewer than two CTA tiles per SM stay on the gather schedule.
conv_halo_fprop_launches() tells which schedule ran."""
import json
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from test_accumulate_gpu import C_GEMM, U, _bf16_bound, _randn, _within

BF16 = torch.bfloat16
CL = torch.channels_last
SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "poseidon_b200", "_ext", "poseidon_b200_C.so")

# (N, Cin, H, W, Cout, R (= S), (ph, pw), groups)
CASES = [
    pytest.param((2, 96, 27, 27, 256, 5, (2, 2), 2), id="conv2-batch2"),
    pytest.param((2, 16, 13, 11, 64, 3, (1, 1), 1), id="odd-hw-cg16"),
    pytest.param((1, 32, 9, 7, 128, 5, (1, 0), 1), id="pad-below-r-1-cg32"),
    pytest.param((1, 128, 71, 5, 384, 3, (1, 1), 2), id="partial-last-tile-cg64-cout192"),
    pytest.param((2, 48, 5, 9, 64, 5, (0, 1), 1), id="no-pad-h-cg48"),
    pytest.param((3, 16, 36, 100, 128, 3, (1, 1), 1), id="wide-rows-odd-tile-count"),
]
EPILOGUES = [(False, None), (True, 0.0), (True, 0.1)]      # (bias, ReLU slope or None)


def _slab(t, off):
    """t [N, C, H, W] as channels [off, off + C) of a NaN-filled channels-last slab (pixel pitch C + off + 8 when off > 0)."""
    n, c, h, w = t.shape
    if not off:
        return t.contiguous(memory_format=CL).cuda()
    slab = torch.full((n, c + off + 8, h, w), float("nan"), dtype=t.dtype).contiguous(memory_format=CL).cuda()
    v = slab[:, off: off + c]
    v.copy_(t)
    return v


def _fprop(ext, mode, x, wb, bias, k, pad, g, oh, ow, slope, out=None):
    """(y, halo forward launches) of conv_fprop under set_conv_halo_fprop(mode)."""
    ext.set_conv_halo_fprop(mode)
    try:
        n0 = ext.conv_halo_fprop_launches()
        y = ext.conv_fprop(x, wb, bias, [k, k], [1, 1], list(pad), g, 0, oh, ow, slope is not None, slope or 0.0, out)
        return y, ext.conv_halo_fprop_launches() - n0
    finally:
        ext.set_conv_halo_fprop(1)


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous(memory_format=CL).view(torch.int16),
                                              b.contiguous(memory_format=CL).view(torch.int16))


@pytest.mark.gpu
def test_alexnet_conv2_batch256_bit_identical(ext):
    n, cin, h, cout, k, g = 256, 96, 27, 256, 5, 2
    gen = torch.Generator(device="cuda").manual_seed(13)
    x = torch.randn(n, cin, h, h, device="cuda", generator=gen).relu().to(BF16).contiguous(memory_format=CL)
    wb = (torch.randn(cout, k * k * cin // g, device="cuda", generator=gen) * (k * k * cin // g) ** -0.5).to(BF16)
    b = torch.randn(cout, device="cuda", generator=gen) * 0.1
    for has_bias, slope in EPILOGUES + [(True, None), (False, 0.0)]:
        bias = b if has_bias else None
        ref, launched = _fprop(ext, 0, x, wb, bias, k, (2, 2), g, h, h, slope)
        assert launched == 0
        got, launched = _fprop(ext, 1, x, wb, bias, k, (2, 2), g, h, h, slope)
        assert launched == 1, "conv2 did not select the halo forward"
        assert _bits_equal(got, ref), f"halo and gather schedules differ (bias {has_bias}, slope {slope})"


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_halo_fprop_edges(ext, case):
    """Forced halo forward vs the gather schedule, bit for bit, and against float64: bias and ReLU (slope 0 and 0.1) on and
    off, the input dense and as a channel slice of a NaN-filled slab, the output dense and as a pitched slab slice."""
    n, cin, h, w, cout, k, (ph, pw), g = case
    cg = cin // g
    oh, ow = h + 2 * ph - k + 1, w + 2 * pw - k + 1
    seed = n + cin + h + w + cout + k
    x = _randn((n, cin, h, w), seed, dtype=BF16)
    wk = _randn((cout, k, k, cg), seed + 1, (k * k * cg) ** -0.5, dtype=BF16)
    b = _randn((cout,), seed + 2, 0.5).float()
    wbd = wk.reshape(cout, -1).contiguous().cuda()
    w4 = wk.double().permute(0, 3, 1, 2)
    conv64 = F.conv2d(x.double(), w4, None, 1, (ph, pw), 1, g)
    mag = F.conv2d(x.double().abs(), w4.abs(), None, 1, (ph, pw), 1, g)
    if cg % 64 == 0:
        ext.set_conv_im2col(0)                  # otherwise the TMA im2col path runs it, not the gather kernel
    try:
        for off in (0, 24):
            xin = _slab(x, off)
            for has_bias, slope in EPILOGUES:
                bias = b.cuda() if has_bias else None
                out = None
                if off:
                    out = torch.full((n, cout + 40, oh, ow), float("nan"), dtype=BF16,
                                     device="cuda").contiguous(memory_format=CL)[:, 16: 16 + cout]
                got, launched = _fprop(ext, 2, xin, wbd, bias, k, (ph, pw), g, oh, ow, slope, out)
                assert launched == 1, "the forced halo forward did not run"
                ref, launched = _fprop(ext, 0, xin, wbd, bias, k, (ph, pw), g, oh, ow, slope)
                assert launched == 0
                what = f"conv_fprop [halo, input channel offset {off}, bias {has_bias}, slope {slope}]"
                assert _bits_equal(got, ref), f"{what}: halo and gather schedules differ"
                want = conv64 + (b.double().view(1, -1, 1, 1) if has_bias else 0.0)
                e = C_GEMM * k * k * cg * U * mag
                if slope is not None:
                    want = torch.where(want > 0, want, want * slope)
                _within(got, want, _bf16_bound(want, e), what)
    finally:
        ext.set_conv_im2col(1)


STEP = r"""
import hashlib, json
import torch
from poseidon_b200 import get_solver
from poseidon_b200.models import zoo
from poseidon_b200.ops import build
build.load_extension()
k = torch.ops.poseidon
net = zoo.alexnet(batch=32, test_batch=8)
sp = zoo.get_solver_param("alexnet", net=net, display=0, snapshot=0, snapshot_after_train=False, test_interval=0,
                          max_iter=1, random_seed=7)
sp.clear("test_iter")
s = get_solver(sp, engine="sm100")
n0 = k.conv_halo_fprop_launches()
s.step(1)
torch.cuda.synchronize()
out = {"launches": k.conv_halo_fprop_launches() - n0, "loss": float(s.last_loss).hex(),
       "blobs": {f"{nm}.{j}": hashlib.sha256(l.export_blob(j).tobytes()).hexdigest()
                 for nm, l in zip(s.net.layer_names, s.net.layers) for j in range(len(l.blobs))}}
s.close()
print(json.dumps(out))
"""


@pytest.mark.gpu
def test_alexnet_training_step_bit_identical(ext):
    """One sm100 training step of AlexNet (batch 32) with the halo forward forced on and off (POSEIDON_CONV_HALO_FPROP 2 / 0,
    one fresh process each, so that both start from the same seeds): identical loss and blobs."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

    def run(mode):
        env = dict(os.environ, POSEIDON_CONV_HALO_FPROP=str(mode), POSEIDON_SYNTHETIC_DATA="1")
        r = subprocess.run([sys.executable, "-c", STEP], cwd=root, env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        return json.loads(r.stdout.strip().splitlines()[-1])

    off, on = run(0), run(2)
    assert off["launches"] == 0 and on["launches"] >= 1, (off["launches"], on["launches"])
    assert off["loss"] == on["loss"], (float.fromhex(off["loss"]), float.fromhex(on["loss"]))
    assert off["blobs"].keys() == on["blobs"].keys()
    differ = [b for b in off["blobs"] if off["blobs"][b] != on["blobs"][b]]
    assert not differ, differ


def test_halo_fprop_sass():
    """The halo forward is wgmma (m64n64k16) on a TMA-loaded halo with the weight tile multicast to the CTA pair."""
    if not os.path.exists(SO) or shutil.which("cuobjdump") is None:
        pytest.skip("needs the built extension and cuobjdump")
    out = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, timeout=600).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(line)
    kern = [k for k in funcs if "halo_fprop_kernel" in k]
    assert len(kern) == 1, kern
    text = "\n".join(funcs[kern[0]])
    assert "HGMMA.64x64x16.F32.BF16" in text
    assert re.search(r"UTMALDG\.2D\.MULTICAST", text)
    assert "UTMALDG.4D" in text
    assert not re.search(r"\bHMMA\b", text)
