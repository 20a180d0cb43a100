"""Plain wgmma GEMM micro-benchmark: TFLOP/s of the four operand-major combinations and tile widths.

Separates "how fast is the TMA/MMA/epilogue core" from "how fast is the conv gather" when reading conv numbers.
    python benchmarks/gemm_bench.py [M N K] [iters]
"""
import sys
import torch
sys.path.insert(0, ".")
from poseidon_b200.ops import sm100

K = sm100.K()
M, N, Kd = (int(v) for v in sys.argv[1:4]) if len(sys.argv) > 3 else (8192, 8192, 8192)
iters = int(sys.argv[4]) if len(sys.argv) > 4 else 5


def bench(fn):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


flops = 2.0 * M * N * Kd
import os
PAIR = int(os.environ.get("PSD_PAIR", "1"))
K.set_pair_cta(PAIR)
print(f"== cta_group::{2 if PAIR else 1} kernels ==", flush=True)
for a_mn in (False, True):
    for b_mn in (False, True):
        if a_mn and not b_mn:
            continue          # MN-major A x K-major B is not instantiated (no layer needs it)
        if a_mn and b_mn:
            # the wgrad combination: fp32 epilogue only
            a = torch.randn(Kd, M, device="cuda").to(torch.bfloat16)
            b = torch.randn(Kd, N, device="cuda").to(torch.bfloat16)
            o32 = torch.empty(M, N, device="cuda", dtype=torch.float32)
            for bn in (256, 128):
                ms = bench(lambda: K.gemm_f32(a, True, b, True, o32, 1.0, False, 1, bn))
                print(f"f32 out   A_MN=1 B_MN=1 BN={bn:3d}: {ms*1e3:9.1f} us  {flops/ms/1e9:7.1f} TFLOP/s", flush=True)
            a = torch.randn(M, Kd, device="cuda").to(torch.bfloat16)
            b = torch.randn(N, Kd, device="cuda").to(torch.bfloat16)
            ms = bench(lambda: K.gemm_f32(a, False, b, False, o32, 1.0, False, 1, 256))
            print(f"f32 out   A_MN=0 B_MN=0 BN=256: {ms*1e3:9.1f} us  {flops/ms/1e9:7.1f} TFLOP/s", flush=True)
            continue
        a = torch.randn((Kd, M) if a_mn else (M, Kd), device="cuda").to(torch.bfloat16)
        b = torch.randn((Kd, N) if b_mn else (N, Kd), device="cuda").to(torch.bfloat16)
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        for bn in (256, 128, 64):
            ms = bench(lambda: K.gemm_bf16(a, a_mn, b, b_mn, None, False, 0.0, None, out, bn))
            print(f"bf16 out  A_MN={int(a_mn)} B_MN={int(b_mn)} BN={bn:3d}: {ms*1e3:9.1f} us  {flops/ms/1e9:7.1f} TFLOP/s", flush=True)
a = torch.randn(M, Kd, device="cuda").to(torch.bfloat16)
bT = torch.randn(N, Kd, device="cuda").to(torch.bfloat16)
ms = bench(lambda: torch.matmul(a, bT.t()))
print(f"cuBLAS bf16 (torch.matmul)          : {ms*1e3:9.1f} us  {flops/ms/1e9:7.1f} TFLOP/s")
# the small-M inner-product shapes of AlexNet (fc6 / fc7 forward), K-major x K-major
for (m, n, k) in ((256, 4096, 9216), (256, 4096, 4096), (256, 1000, 4096)):
    a = torch.randn(m, k, device="cuda").to(torch.bfloat16)
    b = torch.randn(n, k, device="cuda").to(torch.bfloat16)
    out = torch.empty(m, n, device="cuda", dtype=torch.bfloat16)
    for bn in (0, 64, 128):
        ms = bench(lambda: K.gemm_bf16(a, False, b, False, None, False, 0.0, None, out, bn))
        print(f"fc {m}x{n}x{k} BN={bn:3d}: {ms*1e3:8.1f} us  {2.0*m*n*k/ms/1e9:7.1f} TFLOP/s  weight stream {n*k*2/ms/1e6:6.0f} GB/s")
    ms = bench(lambda: torch.matmul(a, b.t()))
    print(f"fc {m}x{n}x{k} cuBLAS: {ms*1e3:8.1f} us")
