"""wgmma GEMM family vs fp32 PyTorch references (run on an H100)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rand(shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _close(got, ref, rel=2e-2):
    err = (got.float() - ref).abs().max().item()
    mag = ref.abs().max().item() + 1e-6
    assert err <= rel * mag, f"max err {err} vs magnitude {mag}"


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 256, 256), (256, 4096, 9216), (200, 1000, 4096),
                                   (77, 40, 96), (3000, 96, 528)])
@pytest.mark.parametrize("bn", [0, 64, 128, 256])
def test_gemm_tn_bf16(ext, M, N, K, bn):
    a, b = _rand((M, K), 1.0, 1), _rand((N, K), 0.05, 2)
    bias = torch.randn(N, device="cuda")
    c = ext.gemm_bf16(a, False, b, False, bias, True, 0.0, None, None, bn)
    ref = torch.relu(a.float() @ b.float().t() + bias)
    _close(c, ref)


@pytest.mark.parametrize("M,N,K", [(256, 9216, 4096), (256, 4096, 1000), (130, 72, 200)])
def test_gemm_dgrad_kmajor_x_mnmajor(ext, M, N, K):
    # dX[M, N] = dY[M, K] · W[K, N]   (W row-major [K, N] is the MN-major B operand)
    dy, w = _rand((M, K), 1.0, 3), _rand((K, N), 0.05, 4)
    mask = _rand((M, N), 1.0, 5)
    c = ext.gemm_bf16(dy, False, w, True, None, False, 0.0, mask, None, 0)
    ref = (dy.float() @ w.float()) * (mask.float() > 0)
    _close(c, ref)


@pytest.mark.parametrize("Mb,N,K", [(256, 4096, 9216), (256, 1000, 4096), (64, 128, 128), (100, 72, 200)])
@pytest.mark.parametrize("split_k", [1, 3])
def test_gemm_wgrad_mn_mn_f32(ext, Mb, N, K, split_k):
    # dW[N, K] = dYᵀ[N, Mb] · X[Mb, K]
    dy, x = _rand((Mb, N), 1.0, 6), _rand((Mb, K), 1.0, 7)
    out = torch.zeros(N, K, device="cuda")
    ext.gemm_f32(dy, True, x, True, out, 1.0, False, split_k, 0)
    ref = dy.float().t() @ x.float()
    _close(out, ref, rel=1e-2)


@pytest.mark.parametrize("rule", [0, 1, 2])
def test_sfb_outer_sgd_single_source(ext, rule):
    Mb, N, K = 256, 512, 1024
    u, v = _rand((Mb, N), 1.0, 8), _rand((Mb, K), 1.0, 9)
    w = torch.randn(N, K, device="cuda")
    h = torch.rand(N, K, device="cuda") * 0.1
    wb = torch.empty(N, K, device="cuda", dtype=torch.bfloat16)
    w_ref, h_ref = w.clone(), h.clone()
    lr, mom, wd, delta = 0.01, 0.0 if rule == 2 else 0.9, 5e-4, 1e-8
    ext.sfb_outer_sgd([u.data_ptr()], [v.data_ptr()], Mb, N, K, w, h, wb, 1.0 / Mb, lr, mom, wd, rule, False,
                      delta, None, 0, 0, 0, 0, None, None)
    g = (u.float().t() @ v.float()) / Mb + wd * w_ref
    if rule == 0:
        h_ref = lr * g + mom * h_ref
        w_ref = w_ref - h_ref
    elif rule == 1:
        h_old = h_ref.clone()
        h_ref = lr * g + mom * h_ref
        w_ref = w_ref - ((1 + mom) * h_ref - mom * h_old)
    else:
        h_ref = h_ref + g * g
        w_ref = w_ref - lr * g / (h_ref.sqrt() + delta)
    _close(w, w_ref, rel=1e-3)
    _close(h, h_ref, rel=1e-2)
    _close(wb, w_ref, rel=1e-2)


def test_sfb_outer_multi_source_local(ext):
    # several sources that all live on this GPU: checks the source loop / rotation logic
    Mb, N, K, P = 128, 256, 320, 4
    us = [_rand((Mb, N), 1.0, 20 + i) for i in range(P)]
    vs = [_rand((Mb, K), 1.0, 30 + i) for i in range(P)]
    w = torch.zeros(N, K, device="cuda")
    h = torch.zeros(N, K, device="cuda")
    flags = torch.full((P,), 7, dtype=torch.int32, device="cuda")
    ext.sfb_outer_sgd([u.data_ptr() for u in us], [v.data_ptr() for v in vs], Mb, N, K, w, h, None, 1.0, 1.0, 0.0,
                      0.0, 0, False, 1e-8, flags, 4, 2, 0, 0, None, torch.full((1,), 3, device="cuda", dtype=torch.int32))
    ref = sum(u.float().t() @ v.float() for u, v in zip(us, vs))
    _close(-w, ref, rel=1e-2)
