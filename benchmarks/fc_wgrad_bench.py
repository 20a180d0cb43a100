"""Inner-product weight gradient dW[N, K] = dY^T[N, M] · X[M, K] (fp32 output, batch M = 256 rows of reduction):
output-bound — 151 MB of fp32 for AlexNet fc6 against 19 GFLOP.
    python benchmarks/fc_wgrad_bench.py [iters]
"""
import sys
import torch
sys.path.insert(0, ".")
from poseidon_b200.ops import sm100

K = sm100.K()
iters = int(sys.argv[1]) if len(sys.argv) > 1 else 20
for name, (n, k_in) in {"fc6": (4096, 9216), "fc7": (4096, 4096), "fc8": (1000, 4096)}.items():
    dy = torch.randn(256, n, device="cuda").to(torch.bfloat16)
    x = torch.randn(256, k_in, device="cuda").to(torch.bfloat16)
    dw = torch.zeros(n, k_in, device="cuda", dtype=torch.float32)
    for _ in range(3):
        K.gemm_f32(dy, True, x, True, dw, 1.0, False, 1, 0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        K.gemm_f32(dy, True, x, True, dw, 1.0, False, 1, 0)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / iters * 1e3
    mb = n * k_in * 4 / 1e6
    print(f"{name} wgrad {n}x{k_in} (M=256): {us:8.1f} us   output {mb:6.1f} MB -> {mb / us * 1e3:7.0f} GB/s", flush=True)
    ref = dy.float().t() @ x.float()
    err = (dw - ref).abs().max().item() / ref.abs().max().item()
    assert err < 2e-2, err
    if len(sys.argv) > 2:
        break
