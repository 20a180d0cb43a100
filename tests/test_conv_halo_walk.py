"""The index arithmetic of the halo-tiled data gradient (csrc/gemm/halo_conv.cuh), replayed in numpy without a GPU.

A tile is T rows of one image's dX in a padded-pitch pixel space of row pitch P = W + S - 1; its dY halo is Hb rows x P
columns starting at dY (h0 + ph - (R-1), pw - (S-1)), zero outside dY; tap (r, s) of tile row m reads halo pixel
m + (R-1-r)*P + (S-1-s).  Rows with column >= W, past T or past the image are computed and dropped.  With integer-valued
operands every float64 sum is exact, so the walk must reproduce conv_transpose2d's dX exactly."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

SHAPES = [(4, 3), (4, 4)]          # 64-row blocks of the two consumer warpgroups (the instantiated kernels)
HALO_SMEM = 232448 - 1024 - 8 * 8192 - 256


def plan(H, W, R, S, cout_g):
    """Tile rows T, tiles per image, tile rows M and halo rows Hb, as halo_dgrad_plan picks them (None: does not fit)."""
    P = W + S - 1
    best = None
    for nb0, nb1 in SHAPES:
        M = 64 * (nb0 + nb1)
        T = min(H, M // P)
        if T < 1:
            continue
        tiles = -(-H // T)
        T = -(-H // tiles)
        Hb = -(-(M + (R - 1) * P + S - 1) // P)
        HP = -(-(Hb * P) // 8) * 8
        if Hb > 256 or cout_g // 8 * HP * 16 > HALO_SMEM:
            continue
        if best is None or tiles * M < best[1] * best[2]:
            best = (T, tiles, M, Hb)
    return best


def halo_walk(dy, w, pad, H, W):
    """dX [N, Cg, H, W] from dY [N, Cout, OH, OW] and w [Cout, Cg, R, S] (one group) by the kernel's tile walk."""
    n_img, cout, OH, OW = dy.shape
    _, cg, R, S = w.shape
    ph, pw = pad
    P = W + S - 1
    T, tiles, M, Hb = plan(H, W, R, S, cout)
    assert T * P <= M
    dx = np.full((n_img, cg, H, W), np.nan)
    # dY zero-padded so that every halo row / column index is in range: padded row y + oy0 is dY row y
    oy0, ox0 = max(0, (R - 1) - ph), max(0, (S - 1) - pw)
    rows = (tiles - 1) * T + Hb
    dyp = np.zeros((n_img, cout, oy0 + max(OH, rows + ph) + 1, ox0 + max(OW, P + pw) + 1))
    dyp[:, :, oy0: oy0 + OH, ox0: ox0 + OW] = dy
    m = np.arange(M)
    tr, x = m // P, m % P
    for t in range(tiles):
        h0 = t * T
        y0, x0 = h0 + ph - (R - 1) + oy0, pw - (S - 1) + ox0
        halo = dyp[:, :, y0: y0 + Hb, x0: x0 + P].transpose(0, 2, 3, 1).reshape(n_img, Hb * P, cout)
        acc = np.zeros((n_img, M, cg))
        for r in range(R):                           # K order of the kernel: taps, then channels
            for s in range(S):
                shift = (R - 1 - r) * P + (S - 1 - s)
                assert 0 <= shift and M - 1 + shift < Hb * P, "a read leaves the halo box"
                acc += halo[:, shift: shift + M] @ w[:, :, r, s]
        live = (x < W) & (tr < T) & (h0 + tr < H)
        dx[:, :, h0 + tr[live], x[live]] = acc[:, live].transpose(0, 2, 1)
    return dx


def reference(dy, w, pad, H, W):
    full = F.conv_transpose2d(torch.from_numpy(dy), torch.from_numpy(w), None, 1, 0)
    ph, pw = pad
    full = F.pad(full, (0, max(0, pw + W - full.shape[3]), 0, max(0, ph + H - full.shape[2])))
    return full[:, :, ph: ph + H, pw: pw + W].numpy()


CASES = [
    # n, cg, cout, H, W, R, pad, dX rows / columns beyond the convolution's input extent
    (1, 48, 64, 27, 27, 5, (2, 2), (0, 0)),      # AlexNet conv2 geometry, batch 1
    (2, 16, 64, 13, 11, 3, (1, 1), (0, 0)),      # odd H / W
    (1, 8, 64, 9, 7, 5, (1, 2), (0, 0)),         # pad below R - 1
    (1, 24, 128, 71, 5, 3, (0, 0), (0, 0)),      # no padding; a partial last tile (36 + 35 rows)
    (2, 8, 64, 5, 9, 5, (0, 1), (2, 1)),         # dX extended past the input extent: zero-filled dY reads
    (3, 16, 64, 36, 100, 3, (1, 1), (0, 0)),     # wide rows: 4 rows per tile, 27 tiles (odd: the last CTA pair has one)
]


@pytest.mark.parametrize("case", CASES)
def test_halo_walk_matches_conv_transpose(case):
    n, cg, cout, h, w_, k, pad, (eh, ew) = case
    rng = np.random.default_rng(7)
    oh, ow = h + 2 * pad[0] - k + 1, w_ + 2 * pad[1] - k + 1
    dy = rng.integers(-3, 4, size=(n, cout, oh, ow)).astype(np.float64)
    wt = rng.integers(-3, 4, size=(cout, cg, k, k)).astype(np.float64)
    H, W = h + eh, w_ + ew
    got = halo_walk(dy, wt, pad, H, W)
    assert not np.isnan(got).any(), "a dX pixel was never stored"
    np.testing.assert_array_equal(got, reference(dy, wt, pad, H, W))


def test_alexnet_conv2_plan():
    """conv2 (27 x 27, 5 x 5, 128 dY channels per group): two tiles of 14 + 13 rows, 448 rows each, 19 halo rows."""
    assert plan(27, 27, 5, 5, 128) == (14, 2, 448, 19)
