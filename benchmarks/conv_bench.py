"""Standalone conv micro-benchmark (AlexNet shapes): CUDA-event timings."""
import sys
import torch
sys.path.insert(0, ".")
sys.path.insert(0, "tests")
from poseidon_b200.ops import sm100
from test_ops_gpu import _FakeLayer, _nhwc

CASES = {
    "conv1": (256, 3, 227, 227, 96, 11, 4, 0, 1),
    "conv2": (256, 96, 27, 27, 256, 5, 1, 2, 2),
    "conv3": (256, 256, 13, 13, 384, 3, 1, 1, 1),
    "conv4": (256, 384, 13, 13, 384, 3, 1, 1, 2),
    "conv5": (256, 384, 13, 13, 256, 3, 1, 1, 2),
    # experiments: same GEMM extent as conv3 (M 43264, N 384, K 2304) with ...
    "conv3_nopad": (256, 256, 15, 15, 384, 3, 1, 0, 1),       # ... no padding: no zero-filled pixels in the im2col boxes
    "conv3_as1x1": (256, 2304, 13, 13, 384, 1, 1, 0, 1),      # ... one tap over 2304 channels: im2col-mode TMA reading a plain [M, K] matrix
}
import os
if os.environ.get('PSD_CONV_IM2COL') == '0':
    os.environ['POSEIDON_PAD_K'] = '0'
    sm100.K().set_conv_im2col(0)
PAIR = int(os.environ.get("PSD_PAIR", "1"))
sm100.K().set_conv_pair(PAIR)
if os.environ.get("PSD_MAX_STAGES"):
    sm100.K().set_max_stages(int(os.environ["PSD_MAX_STAGES"]))
MC = int(os.environ.get("PSD_MCAST", "1"))
sm100.K().set_conv_mcast(MC)
print(f"== cta_group::{2 if PAIR else 1} kernels, im2col multicast cluster {MC} ==", flush=True)
which = sys.argv[1].split(",") if len(sys.argv) > 1 else list(CASES)
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 5
for name in which:
    n, cin, h, w, cout, k, stride, pad, group = CASES[name]
    layer = _FakeLayer(cout, cin, k, stride, pad, group)
    layer.in_hw = (h, w)
    x = (torch.randn(n, cin, h, w, device="cuda").to(torch.bfloat16)) if cin == 3 else _nhwc((n, cin, h, w), 5)
    xs = x.clone().requires_grad_(cin != 3)
    flops = 2.0 * n * cout * (cin // group) * k * k
    def run():
        y = sm100.conv2d(xs, layer.weight, layer.bias, layer.stride, layer.pad, group, relu_slope=0.0, layer=layer)
        return y
    y = run()
    oh, ow = y.shape[2], y.shape[3]
    flops *= oh * ow
    dy = torch.randn_like(y)
    for _ in range(2):
        layer.weight.grad = None
        run().backward(dy)
    torch.cuda.synchronize()
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    tf = tb = 0.0
    for _ in range(iters):
        layer.weight.grad = None
        layer.bias.grad = None
        e[0].record()
        y = run()
        e[1].record()
        y.backward(dy)
        e[2].record()
        torch.cuda.synchronize()
        tf += e[0].elapsed_time(e[1]); tb += e[1].elapsed_time(e[2])
    tf /= iters; tb /= iters
    print(f"{name}: fwd {tf*1e3:8.1f} us ({flops/tf/1e9:7.1f} TFLOPS)   bwd {tb*1e3:8.1f} us ({(2 if cin != 3 else 1)*flops/tb/1e9:7.1f} TFLOPS eq)")
