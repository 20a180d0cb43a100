"""The halo-tiled data gradient (csrc/gemm/halo_conv.cuh) behind conv_dgrad_w: bit-identical to the im2col schedule
(set_conv_halo(0)) and within the float64 bound test_conv_contract_gpu.py uses for conv_dgrad_w.

AlexNet conv2 at batch 256 takes the halo schedule by default; the small edge geometries run it forced (set_conv_halo(2)),
since by default problems with fewer than two tiles per SM stay on the im2col schedule.  conv_halo_launches() tells which
schedule ran."""
import pytest
import torch
import torch.nn.functional as F

from test_accumulate_gpu import C_GEMM, U, _bf16_bound, _randn, _within

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
CL = torch.channels_last

# (N, Cin, H, W, Cout, R (= S), (ph, pw), groups, (eh, ew): dX rows / columns beyond the input extent)
CASES = [
    pytest.param((1, 96, 27, 27, 256, 5, (2, 2), 2, (0, 0)), id="conv2-batch1"),
    pytest.param((2, 16, 13, 11, 64, 3, (1, 1), 1, (0, 0)), id="odd-hw-3x3"),
    pytest.param((1, 8, 9, 7, 64, 5, (1, 2), 1, (0, 0)), id="pad-below-r-1"),
    pytest.param((1, 48, 71, 5, 256, 3, (0, 0), 2, (0, 0)), id="partial-last-tile-groups2"),
    pytest.param((2, 64, 5, 9, 128, 5, (0, 1), 1, (2, 1)), id="dx-past-input-extent"),
    pytest.param((3, 32, 36, 100, 64, 3, (1, 1), 1, (0, 0)), id="wide-rows-odd-tile-count"),
]
SLOPES = [None, 0.0, 0.1]          # no mask; the producer's ReLU mask with slope 0 and 0.1


def _slab(t, off):
    """t [N, C, H, W] as channels [off, off + C) of a NaN-filled channels-last slab (pixel pitch C + off + 8 when off > 0)."""
    n, c, h, w = t.shape
    if not off:
        return t.contiguous(memory_format=CL).cuda()
    slab = torch.full((n, c + off + 8, h, w), float("nan"), dtype=t.dtype).contiguous(memory_format=CL).cuda()
    v = slab[:, off: off + c]
    v.copy_(t)
    return v


def _dgrad(ext, mode, dy, wk, kern, pad, g, h, w, mask, slope):
    """(dX, halo kernel launches) of conv_dgrad_w under set_conv_halo(mode)."""
    ext.set_conv_halo(mode)
    try:
        n0 = ext.conv_halo_launches()
        out = ext.conv_dgrad_w(dy, wk, [kern, kern], list(pad), g, h, w, mask, slope)
        return out, ext.conv_halo_launches() - n0
    finally:
        ext.set_conv_halo(1)


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous(memory_format=CL).view(torch.int16),
                                              b.contiguous(memory_format=CL).view(torch.int16))


def test_alexnet_conv2_batch256_bit_identical(ext):
    n, cin, h, cout, k, g = 256, 96, 27, 256, 5, 2
    gen = torch.Generator(device="cuda").manual_seed(11)
    dy = torch.randn(n, cout, h, h, device="cuda", generator=gen).to(BF16).contiguous(memory_format=CL)
    wk = (torch.randn(cout, k * k * cin // g, device="cuda", generator=gen) * (k * k * cout // g) ** -0.5).to(BF16)
    mask = torch.randn(n, cin, h, h, device="cuda", generator=gen).to(BF16).contiguous(memory_format=CL)
    for slope in SLOPES:
        m = None if slope is None else mask
        ref, launched = _dgrad(ext, 0, dy, wk, k, (2, 2), g, h, h, m, slope or 0.0)
        assert launched == 0
        got, launched = _dgrad(ext, 1, dy, wk, k, (2, 2), g, h, h, m, slope or 0.0)
        assert launched == g, "conv2 did not select the halo schedule"
        assert _bits_equal(got, ref), f"halo and im2col schedules differ (slope {slope})"


@pytest.mark.parametrize("case", CASES)
def test_halo_dgrad_edges(ext, case):
    """Forced halo schedule vs the im2col schedule, bit for bit, and against float64: with and without the mask (slope 0 and
    0.1), dY dense and as a channel slice of a NaN-filled slab."""
    n, cin, h, w, cout, k, (ph, pw), g, (eh, ew) = case
    oh, ow = h + 2 * ph - k + 1, w + 2 * pw - k + 1
    hr, wr = h + eh, w + ew
    seed = n + cin + h + w + cout + k
    dy = _randn((n, cout, oh, ow), seed, dtype=BF16)
    wk = _randn((cout, k, k, cin // g), seed + 1, (k * k * cout // g) ** -0.5, dtype=BF16)
    mask = _randn((n, cin, hr, wr), seed + 2, dtype=BF16).contiguous(memory_format=CL)
    wkd = wk.reshape(cout, -1).contiguous().cuda()
    mask_d = mask.cuda()

    w4 = wk.double().permute(0, 3, 1, 2)

    def tconv(a, b):
        full = F.conv_transpose2d(a, b, None, 1, 0, 0, g)
        full = F.pad(full, (0, max(0, pw + wr - full.shape[3]), 0, max(0, ph + hr - full.shape[2])))
        return full[:, :, ph: ph + hr, pw: pw + wr]
    ref64, mag = tconv(dy.double(), w4), tconv(dy.double().abs(), w4.abs())

    for off in (0, 24):
        dyin = _slab(dy, off)
        for slope in SLOPES:
            m = None if slope is None else mask_d
            got, launched = _dgrad(ext, 2, dyin, wkd, k, (ph, pw), g, hr, wr, m, slope or 0.0)
            assert launched == g, "the forced halo schedule did not run"
            ref, _ = _dgrad(ext, 0, dyin, wkd, k, (ph, pw), g, hr, wr, m, slope or 0.0)
            what = f"conv_dgrad_w [halo, dY channel offset {off}, slope {slope}]"
            assert _bits_equal(got, ref), f"{what}: halo and im2col schedules differ"
            want = ref64 if slope is None else torch.where(mask.double() > 0, ref64, ref64 * slope)
            _within(got, want, _bf16_bound(want, C_GEMM * k * k * (cout // g) * U * mag), what)
