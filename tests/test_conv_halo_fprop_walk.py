"""The index arithmetic of the halo-tiled forward (halo_fprop_kernel, csrc/gemm/halo_conv.cuh), replayed in numpy without a
GPU, and the geometry selection of conv_fprop_halo replayed over the zoo nets.

A tile is T rows of one image's output in a padded-pitch pixel space of row pitch P = OW + S - 1; its input halo is Hb rows
x P columns starting at input (h0 - ph, -pw), zero outside the input; k16 step j covers weight columns [16j, 16j + 16),
i.e. tap j // (Cg/16) and channels 16 (j mod Cg/16) .. + 16, and tap (r, s) of tile row m reads halo pixel m + r*P + s.
Rows with column >= OW, past T or past OH are computed and dropped.  With integer-valued operands every float64 sum is
exact, so the walk must reproduce conv2d exactly."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

M = 64 * (4 + 3)                   # tile rows: 64-row blocks of the two consumer warpgroups (the instantiated kernel)
SMEM = 232448 - 1024 - 8 * 8192 - 2048 - 256     # beside the B ring, the zero block and the barriers: two halos
SMS = 132                          # H100 SXM


def plan(OH, OW, R, S, cg, cout_g):
    """(T, tiles per image, Hb) as halo_fprop_plan picks them, or None where the kernel cannot run."""
    if cg % 16 or cg > 64 or cout_g % 64:
        return None
    P = OW + S - 1
    T = min(OH, M // P)
    if P > 256 or T < 1:
        return None
    tiles = -(-OH // T)
    T = -(-OH // tiles)
    Hb = -(-(M + (R - 1) * P + S - 1) // P)
    HP = -(-(Hb * P) // 8) * 8
    if Hb > 256 or 2 * (cg // 8) * HP * 16 > SMEM:
        return None
    return T, tiles, Hb


def selected(n, cg, cout_g, groups, H, W, R, S, stride, pad):
    """Whether conv_fprop runs this convolution on the halo kernel by default (set_conv_halo_fprop(1))."""
    if tuple(stride) != (1, 1) or cg % 8 or cg % 64 == 0:     # gather path only: not ROW mode, not the TMA im2col path
        return False
    OH, OW = H + 2 * pad[0] - R + 1, W + 2 * pad[1] - S + 1
    pl = plan(OH, OW, R, S, cg, cout_g)
    if pl is None:
        return False
    _, tiles, _ = pl
    return R * S >= 9 and tiles * M * 10 <= 13 * OH * OW and n * tiles * groups * (cout_g // 64) >= 2 * SMS


def halo_walk(x, wb, pad, R, S):
    """y [N, Cout, OH, OW] from x [N, Cg, H, W] and the forward operand wb [Cout, R*S*Cg] (one group) by the kernel's walk."""
    n_img, cg, H, W = x.shape
    cout = wb.shape[0]
    ph, pw = pad
    OH, OW = H + 2 * ph - R + 1, W + 2 * pw - S + 1
    P = OW + S - 1
    T, tiles, Hb = plan(OH, OW, R, S, cg, cout)
    assert T * P <= M
    cpt = cg // 16
    steps = R * S * cpt
    kb_per_tile = -(-steps // 4)
    kpad = np.zeros((cout, 64 * kb_per_tile))     # the weight map's k blocks, zero-filled past K
    kpad[:, : R * S * cg] = wb
    y = np.full((n_img, cout, OH, OW), np.nan)
    # input zero-padded so that every halo row / column index is in range: padded row i + ph is input row i
    rows = (tiles - 1) * T + Hb
    xp = np.zeros((n_img, cg, ph + max(H, rows) + 1, pw + max(W, P) + 1))
    xp[:, :, ph: ph + H, pw: pw + W] = x
    m = np.arange(M)
    tr, col = m // P, m % P
    for t in range(tiles):
        h0 = t * T
        # box origin (h0 - ph, -pw) is padded index (h0, 0)
        halo = xp[:, :, h0: h0 + Hb, 0: P].transpose(0, 2, 3, 1).reshape(n_img, Hb * P, cg)
        zeros = np.zeros((n_img, M, 16))
        acc = np.zeros((n_img, M, cout))
        for j in range(4 * kb_per_tile):          # whole k blocks, in order
            kb, kk = divmod(j, 4)
            b = kpad[:, 64 * kb + 16 * kk: 64 * kb + 16 * kk + 16]          # B slice kk of k block kb
            if j >= steps:                         # past K: zeros x zero-filled B
                assert not b.any()
                acc += zeros @ b.T
                continue
            tap, cp = divmod(j, cpt)
            r, s = divmod(tap, S)
            assert 16 * j == tap * cg + 16 * cp, "a k16 step straddles a tap"
            shift = r * P + s
            assert 0 <= shift and M - 1 + shift < Hb * P, "a read leaves the halo box"
            acc += halo[:, shift: shift + M, 16 * cp: 16 * cp + 16] @ b.T
        live = (col < OW) & (tr < T) & (h0 + tr < OH)
        y[:, :, h0 + tr[live], col[live]] = acc[:, live].transpose(0, 2, 1)
    return y


CASES = [
    # n, cg, cout_g, H, W, R, pad
    (1, 48, 128, 27, 27, 5, (2, 2)),      # AlexNet conv2 geometry, batch 1
    (2, 16, 64, 13, 11, 3, (1, 1)),       # odd H / W
    (1, 32, 64, 9, 7, 5, (1, 0)),         # pad below (R - 1) / 2
    (1, 64, 192, 71, 5, 3, (1, 1)),       # a partial last tile (36 + 35 rows)
    (2, 48, 64, 5, 9, 5, (0, 1)),         # output smaller than the input: no padding along H
    (3, 16, 128, 36, 100, 3, (1, 1)),     # wide rows: 4 rows per tile
]


@pytest.mark.parametrize("case", CASES)
def test_halo_fprop_walk_matches_conv2d(case):
    n, cg, cout, h, w, k, pad = case
    rng = np.random.default_rng(5)
    x = rng.integers(-3, 4, size=(n, cg, h, w)).astype(np.float64)
    wt = rng.integers(-3, 4, size=(cout, cg, k, k)).astype(np.float64)
    wb = wt.transpose(0, 2, 3, 1).reshape(cout, -1)        # [Cout][R][S][Cg]
    got = halo_walk(x, wb, pad, k, k)
    assert not np.isnan(got).any(), "an output pixel was never stored"
    want = F.conv2d(torch.from_numpy(x), torch.from_numpy(wt), None, 1, pad).numpy()
    np.testing.assert_array_equal(got, want)


def test_alexnet_conv2_plan():
    """conv2 (27 x 27 output, 5 x 5, 48 input channels per group): two tiles of 14 + 13 rows, 19 halo rows."""
    assert plan(27, 27, 5, 5, 48, 128) == (14, 2, 19)
    assert selected(256, 48, 128, 2, 27, 27, 5, 5, (1, 1), (2, 2))


def test_zoo_selection_is_the_two_conv2s():
    """Over every convolution of the zoo nets at their default batch, the halo forward is selected for AlexNet's and
    CaffeNet's conv2 and nothing else."""
    from poseidon_b200.layers import NetContext
    from poseidon_b200.models import zoo
    from poseidon_b200.net.net import Net
    from poseidon_b200 import proto as P

    picked = set()
    for name, batch in (("alexnet", 256), ("caffenet", 256), ("googlenet", 32), ("vgg16", 64), ("lenet", 64)):
        hint = (1, 28, 28) if name == "lenet" else (3, 224, 224)
        net = Net(getattr(zoo, name)(batch=2, test_batch=2), phase=P.TRAIN,
                  ctx=NetContext(phase=P.TRAIN, device="cpu", engine="torch", data_shape_hint=hint))
        convs = 0
        for lname, layer in zip(net.layer_names, net.layers):
            if not hasattr(layer, "group") or not hasattr(layer, "in_hw"):
                continue
            convs += 1
            cout, cg, R, S = layer.weight.shape
            h, w = layer.in_hw
            if selected(batch, cg, cout // layer.group, layer.group, h, w, R, S, layer.stride, layer.pad):
                picked.add((name, lname))
        assert convs > 0, name
    assert picked == {("alexnet", "conv2"), ("caffenet", "conv2")}
