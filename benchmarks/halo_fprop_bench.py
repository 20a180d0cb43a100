"""conv_fprop on the halo forward vs the gather schedule (set_conv_halo_fprop 1 / 0), alternating in one process, CUDA events.

Layer: AlexNet conv2 at batch 256 with bias and the fused ReLU, as the engine runs it (CaffeNet's conv2 has the same
geometry).  Per schedule: ms per call (median of the rounds), logical TFLOP/s (2·N·OH·OW·Cg·R·S·Cout) and padded TFLOP/s
(the MMA work the tiles issue, zero-filled k tail included), and the byte model: input (A) and weight (B) bytes delivered
from L2 to the SMs per group.  The card's name, power limit and maximum SM clock are printed in the same run.

    python benchmarks/halo_fprop_bench.py [rounds] [calls per round]"""
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from poseidon_b200.ops import build  # noqa: E402
from test_conv_halo_fprop_walk import M, plan  # noqa: E402

# name: (N, Cin, H, W, Cout, R (= S), pad, groups)
LAYERS = {
    "alexnet_conv2": (256, 96, 27, 27, 256, 5, 2, 2),
}


def model(n, cin, h, w, cout, k, pad, g):
    """(logical flops, {schedule: (padded flops, A bytes per group, B bytes per group)})."""
    cg, cout_g = cin // g, cout // g
    oh, ow = h + 2 * pad - k + 1, w + 2 * pad - k + 1
    kb = -(-k * k * cg // 64)                                   # 64-wide k blocks
    logical = 2.0 * n * oh * ow * cg * k * k * cout_g * g
    m_blocks = -(-n * oh * ow // 128)
    bn = 128                                                    # gather kernel tile width (kGatherMaxBN)
    nb = -(-cout_g // bn)
    gather = (2.0 * m_blocks * 128 * nb * bn * kb * 64 * g, m_blocks * nb * kb * 128 * 64 * 2,
              m_blocks * nb * kb * bn * 64 * 2)
    T, tiles, Hb = plan(oh, ow, k, k, cg, cout_g)
    P = ow + k - 1
    ctas = n * tiles * (cout_g // 64)                           # CTA tiles per group
    halo = (2.0 * ctas * M * 64 * kb * 64 * g, ctas * (cg // 8) * Hb * P * 16,
            -(-n * tiles // 2) * (cout_g // 64) * kb * 64 * 64 * 2)   # B: one L2 read per CTA pair (multicast)
    return logical, {0: gather, 1: halo}


def card():
    props = torch.cuda.get_device_properties(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit not available"
    return f"{props.name}, {props.multi_processor_count} SMs, {q}"


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    calls = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    build.load_extension()
    k = torch.ops.poseidon
    print(f"# {card()}; {rounds} alternating rounds of {calls} calls per schedule")
    for name, (n, cin, h, w, cout, ks, pad, g) in LAYERS.items():
        gen = torch.Generator(device="cuda").manual_seed(1)
        oh, ow = h + 2 * pad - ks + 1, w + 2 * pad - ks + 1
        x = torch.randn(n, cin, h, w, device="cuda", generator=gen).relu().to(torch.bfloat16).contiguous(
            memory_format=torch.channels_last)
        wb = (torch.randn(cout, ks * ks * cin // g, device="cuda", generator=gen) * 0.05).to(torch.bfloat16)
        bias = torch.randn(cout, device="cuda", generator=gen) * 0.1

        def run(mode):
            k.set_conv_halo_fprop(mode)
            return k.conv_fprop(x, wb, bias, [ks, ks], [1, 1], [pad, pad], g, 0, oh, ow, True, 0.0, None)

        n0 = k.conv_halo_fprop_launches()
        outs = {m: run(m) for m in (0, 1)}
        torch.cuda.synchronize()
        assert k.conv_halo_fprop_launches() - n0 == 1, "the halo forward was not selected"
        same = torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16))
        times = {0: [], 1: []}
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for _ in range(rounds):
            for mode in (0, 1):
                run(mode)
                ev[0].record()
                for _ in range(calls):
                    run(mode)
                ev[1].record()
                torch.cuda.synchronize()
                times[mode].append(ev[0].elapsed_time(ev[1]) / calls)
        k.set_conv_halo_fprop(1)
        logical, sched = model(n, cin, h, w, cout, ks, pad, g)
        print(f"{name}: N={n} Cin={cin} {h}x{w} Cout={cout} {ks}x{ks} pad={pad} groups={g}; "
              f"halo == gather bit for bit: {same}")
        for mode, label in ((0, "gather"), (1, "halo")):
            ms = statistics.median(times[mode])
            padded, a_b, b_b = sched[mode]
            print(f"  {label:7s} {ms:.4f} ms (min {min(times[mode]):.4f}, max {max(times[mode]):.4f})  "
                  f"logical {logical / ms / 1e9:.0f} TFLOP/s  padded {padded / ms / 1e9:.0f} TFLOP/s  "
                  f"L2->SM per group: A {a_b / 1e9:.3f} GB, B {b_b / 1e9:.3f} GB")


if __name__ == "__main__":
    main()
