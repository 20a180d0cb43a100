"""The CPU emulation of the op surface (ops/emulate.py) against the kernels it stands in for, op by op, same inputs.

The CPU suite trusts the emulator to test the Python side of the engine; this is the check of the emulator itself.
Not compared: dropout (the emulation draws its keep-map from a generator instead of the kernel's integer hash)
and the pooling index tensor (opaque to the caller; only y and dx are contract)."""
import pytest
import torch

pytestmark = [pytest.mark.gpu]

CL = torch.channels_last
BF = torch.bfloat16


@pytest.fixture(scope="module")
def pair(ext):
    from poseidon_b200.ops.emulate import EmulatedKernels
    return EmulatedKernels(), torch.ops.poseidon


def _cu(t):
    if t is None or not torch.is_tensor(t):
        return t
    c = t.cuda()
    if t.dim() == 4 and t.is_contiguous(memory_format=CL) and not t.is_contiguous():
        c = c.contiguous(memory_format=CL)
    return c


def _close(a, b, rel=0.02, what=""):
    a, b = a.float().cpu(), b.float().cpu()
    assert a.shape == b.shape, (what, a.shape, b.shape)
    d = (a - b).abs().max().item()
    m = b.abs().max().item()
    assert d <= rel * m + 1e-3, (what, d, m)


def _nhwc(n, c, h, w, scale=1.0):
    return (torch.randn(n, c, h, w) * scale).to(BF).contiguous(memory_format=CL)


@pytest.mark.parametrize("cin,cout,k,stride,pad,groups,hw", [(16, 32, 3, 1, 1, 1, 9), (32, 64, 5, 1, 2, 2, 12),
                                                             (24, 40, 1, 1, 0, 1, 7), (64, 64, 3, 2, 1, 1, 14)])
def test_conv_tap_mode(pair, cin, cout, k, stride, pad, groups, hw):
    emu, op = pair
    torch.manual_seed(0)
    x = _nhwc(3, cin, hw, hw)
    cg = cin // groups
    w = (torch.randn(cout, k * k * cg) * 0.1).to(BF)
    bias = torch.randn(cout)
    oh = (hw + 2 * pad - k) // stride + 1
    args = ([k, k], [stride, stride], [pad, pad], groups, 0, oh, oh, True, 0.1, None)
    ye = emu.conv_fprop(x, w, bias, *args)
    yg = op.conv_fprop(_cu(x), w.cuda(), bias.cuda(), *args)
    _close(yg, ye, what="fprop")
    dy = _nhwc(3, cout, oh, oh)
    dwe, dwg = torch.zeros(cout, k * k * cg), torch.zeros(cout, k * k * cg, device="cuda")
    emu.conv_wgrad(x, dy, dwe, [k, k], [stride, stride], [pad, pad], groups, 0, 1.0, cg)
    op.conv_wgrad(_cu(x), _cu(dy), dwg, [k, k], [stride, stride], [pad, pad], groups, 0, 1.0, cg)
    _close(dwg, dwe, what="wgrad")
    if stride == 1:
        wf = torch.randn(cout * k * k * cg)
        wte = emu.conv_pack_dgrad(wf, cout, k * k, cg, groups, None, 0)
        wtg = op.conv_pack_dgrad(wf.cuda(), cout, k * k, cg, groups, None, 0)
        _close(wtg, wte, 0.0, "pack_dgrad")
        mask = _nhwc(3, cin, hw, hw)
        dxe = emu.conv_dgrad(dy, wte, [k, k], [pad, pad], groups, hw, hw, mask, 0.0)
        dxg = op.conv_dgrad(_cu(dy), wtg, [k, k], [pad, pad], groups, hw, hw, _cu(mask), 0.0)
        _close(dxg, dxe, what="dgrad")


def test_conv_row_mode_and_padded_operand(pair):
    emu, op = pair
    torch.manual_seed(1)
    x = _nhwc(2, 4, 23, 24)                                   # pre-padded NHWC4 image, even physical width
    r = s = 7
    lp = (s * 4 + 7) // 8 * 8
    w = torch.zeros(32, r, lp)
    w[:, :, : s * 4] = torch.randn(32, r, s * 4) * 0.1
    w = w.reshape(32, r * lp).to(BF)
    oh, ow = (23 - 7) // 2 + 1, (23 - 7) // 2 + 1
    ye = emu.conv_fprop(x, w, None, [r, s], [2, 2], [0, 0], 1, 1, oh, ow, False, 0.0, None)
    yg = op.conv_fprop(_cu(x), w.cuda(), None, [r, s], [2, 2], [0, 0], 1, 1, oh, ow, False, 0.0, None)
    _close(yg, ye, what="row fprop")
    dy = _nhwc(2, 32, oh, ow)
    dwe, dwg = torch.zeros(32, r * lp), torch.zeros(32, r * lp, device="cuda")
    emu.conv_wgrad(x, dy, dwe, [r, s], [2, 2], [0, 0], 1, 1, 1.0, 0)
    op.conv_wgrad(_cu(x), _cu(dy), dwg, [r, s], [2, 2], [0, 0], 1, 1, 1.0, 0)
    _close(dwg, dwe, what="row wgrad")
    wb = (torch.randn(16, 9 * 48) * 0.1).to(BF)
    _close(op.conv_pack_padded(wb.cuda().reshape(-1), 16, 9, 48, 64, None), emu.conv_pack_padded(wb.reshape(-1), 16, 9, 48, 64, None), 0.0)


def test_gemm_lrn_pool_loss_update_transform(pair):
    emu, op = pair
    torch.manual_seed(2)
    a, b = (torch.randn(40, 72) * 0.3).to(BF), (torch.randn(24, 72) * 0.3).to(BF)
    bias = torch.randn(24)
    _close(op.gemm_bf16(a.cuda(), False, b.cuda(), False, bias.cuda(), True, 0.0, None, None, 0),
           emu.gemm_bf16(a, False, b, False, bias, True, 0.0, None, None, 0), what="gemm_bf16")
    oe, og = torch.zeros(72, 72), torch.zeros(72, 72, device="cuda")
    emu.gemm_f32(a, True, a, True, oe, 0.5, False, 1, 0)
    op.gemm_f32(a.cuda(), True, a.cuda(), True, og, 0.5, False, 1, 0)
    _close(og, oe, what="gemm_f32")
    x = _nhwc(2, 32, 9, 9).abs()
    dy = _nhwc(2, 32, 9, 9)
    _close(op.lrn_fwd(_cu(x), 5, 1e-2, 0.75, False), emu.lrn_fwd(x, 5, 1e-2, 0.75, False), what="lrn_fwd")
    _close(op.lrn_bwd(_cu(x), _cu(dy), 5, 1e-2, 0.75, True), emu.lrn_bwd(x, dy, 5, 1e-2, 0.75, True), 0.03, "lrn_bwd")
    for is_max in (True, False):
        ye, ie = emu.pool_fwd(x, is_max, [3, 3], [2, 2], [0, 0], 4, 4, True)
        yg, ig = op.pool_fwd(_cu(x), is_max, [3, 3], [2, 2], [0, 0], 4, 4, True)
        _close(yg, ye, what=f"pool_fwd max={is_max}")
        d = _nhwc(2, 32, 4, 4)
        _close(op.pool_bwd(_cu(d), ig, is_max, [9, 9], [3, 3], [2, 2], [0, 0]),
               emu.pool_bwd(d, ie, is_max, [9, 9], [3, 3], [2, 2], [0, 0]), 0.03, f"pool_bwd max={is_max}")
    logits, lab = (torch.randn(16, 10) * 2).to(BF), torch.randint(0, 10, (16,)).float()
    le, dxe, pe = emu.softmax_xent(logits, lab, 1.0, True, True)
    lg, dxg, pg = op.softmax_xent(logits.cuda(), lab.cuda(), 1.0, True, True)
    _close(lg, le, 0.01, "loss")
    _close(dxg, dxe, 0.02, "dloss")
    _close(pg, pe, 0.01, "prob")
    for rule in (0, 1, 2):
        w, g, h = torch.randn(33, 8), torch.randn(33, 8), torch.rand(33, 8)
        wg, hg, wbg = w.cuda(), h.cuda(), torch.zeros(33, 8, dtype=BF, device="cuda")
        we, he, wbe = w.clone(), h.clone(), torch.zeros(33, 8, dtype=BF)
        lr_dev = torch.tensor([0.5])
        emu.fused_update(we, g, he, wbe, 0.1, 0.9, 0.01, rule, rule == 2, 1e-8, 0.5, lr_dev)
        op.fused_update(wg, g.cuda(), hg, wbg, 0.1, 0.9, 0.01, rule, rule == 2, 1e-8, 0.5, lr_dev.cuda())
        _close(wg, we, 1e-5, f"update rule {rule}")
        _close(hg, he, 1e-5, f"history rule {rule}")
        _close(wbg, wbe, 0.0, f"shadow rule {rule}")
    img = torch.randint(0, 256, (3, 3, 20, 20), dtype=torch.uint8)
    ho, wo, fl = torch.tensor([1, 0, 3], dtype=torch.int32), torch.tensor([2, 4, 0], dtype=torch.int32), \
        torch.tensor([0, 1, 1], dtype=torch.uint8)
    mean = torch.tensor([104.0, 117.0, 123.0])
    for cp, opad, wex, hex_, s2d in ((4, 2, 0, 0, False), (8, 0, 0, 0, False), (4, 0, 0, 0, True)):
        te = emu.transform_nhwc(img, ho, wo, fl, mean, 0.017, 16, 16, cp, opad, wex, hex_, s2d)
        tg = op.transform_nhwc(img.cuda(), ho.cuda(), wo.cuda(), fl.cuda(), mean.cuda(), 0.017, 16, 16, cp, opad, wex, hex_, s2d)
        _close(tg, te, 0.0, f"transform cp={cp} s2d={s2d}")
    dyc = _nhwc(2, 16, 5, 5)
    se, sg = torch.zeros(16), torch.zeros(16, device="cuda")
    emu.colsum(dyc, 50, 16, 16, se, 1.0, False)
    op.colsum(_cu(dyc), 50, 16, 16, sg, 1.0, False)
    _close(sg, se, 1e-3, "colsum")
    y = _nhwc(2, 16, 5, 5)
    _close(op.relu_bwd(_cu(y), _cu(dyc), 0.1), emu.relu_bwd(y, dyc, 0.1), 0.0, "relu_bwd")
