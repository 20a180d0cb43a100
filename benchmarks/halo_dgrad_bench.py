"""conv_dgrad_w on the halo schedule vs the im2col schedule (set_conv_halo 1 / 0), alternating in one process, CUDA events.

Layers: AlexNet conv2 at batch 256 (the zoo's one data gradient that selects the halo schedule by default) and VGG-16
conv1_2 at batch 64 (halo schedule forced: 9 k blocks per tile, measured slower, hence excluded by the selection), with the
producer's ReLU mask as the engine runs them.  Per schedule: ms per call (median of the rounds), logical
TFLOP/s (2·N·H·W·Cg·R·S·Cout per layer) and padded TFLOP/s (the MMA work the tiles issue), and the byte model: dY (A) and
weight (B) bytes delivered from L2 to the SMs per group.

    python benchmarks/halo_dgrad_bench.py [rounds] [calls per round]"""
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from poseidon_b200.ops import build  # noqa: E402
from test_conv_halo_walk import plan  # noqa: E402

# name: (N, Cin, H, W, Cout, R (= S), pad, groups, set_conv_halo mode of the halo runs)
LAYERS = {
    "alexnet_conv2": (256, 96, 27, 27, 256, 5, 2, 2, 1),
    "vgg16_conv1_2": (64, 64, 224, 224, 64, 3, 1, 1, 2),
}


def model(n, cin, h, w, cout, k, g):
    """(logical flops, {schedule: (padded flops, A bytes per group, B bytes per group)})."""
    cg, cout_g = cin // g, cout // g
    cok = -(-cout_g // 64) * 64
    kdim = k * k * cok
    logical = 2.0 * n * h * w * cg * k * k * cout_g * g
    m_blocks = -(-n * h * w // 128)
    im2col = (2.0 * m_blocks * 128 * 64 * kdim * g, m_blocks * 128 * kdim * 2, m_blocks * kdim * 64 * 2)
    T, tiles, M, Hb = plan(h, w, k, k, cout_g)
    P = w + k - 1
    ntiles = n * tiles
    halo = (2.0 * ntiles * M * 64 * kdim * g, ntiles * Hb * P * cout_g * 2,
            -(-ntiles // 2) * kdim * 64 * 2)                     # B: one L2 read per CTA pair (multicast)
    return logical, {0: im2col, 1: halo}


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    calls = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    build.load_extension()
    k = torch.ops.poseidon
    props = torch.cuda.get_device_properties(0)
    print(f"# {props.name}, {props.multi_processor_count} SMs; {rounds} alternating rounds of {calls} calls per schedule")
    for name, (n, cin, h, w, cout, ks, pad, g, on) in LAYERS.items():
        gen = torch.Generator(device="cuda").manual_seed(1)
        oh, ow = h + 2 * pad - ks + 1, w + 2 * pad - ks + 1
        dy = torch.randn(n, cout, oh, ow, device="cuda", generator=gen).to(torch.bfloat16).contiguous(
            memory_format=torch.channels_last)
        wb = (torch.randn(cout, ks * ks * cin // g, device="cuda", generator=gen) * 0.05).to(torch.bfloat16)
        mask = torch.randn(n, cin, h, w, device="cuda", generator=gen).to(torch.bfloat16).contiguous(
            memory_format=torch.channels_last)

        def run(mode):
            k.set_conv_halo(on if mode else 0)
            return k.conv_dgrad_w(dy, wb, [ks, ks], [pad, pad], g, h, w, mask, 0.0)

        outs = {m: run(m) for m in (0, 1)}
        torch.cuda.synchronize()
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
        k.set_conv_halo(1)
        logical, sched = model(n, cin, h, w, cout, ks, g)
        print(f"{name}: N={n} Cin={cin} {h}x{w} Cout={cout} {ks}x{ks} pad={pad} groups={g}; halo == im2col bit for bit: {same}")
        for mode, label in ((0, "im2col"), (1, "halo")):
            ms = statistics.median(times[mode])
            padded, a_b, b_b = sched[mode]
            print(f"  {label:7s} {ms:.4f} ms (min {min(times[mode]):.4f}, max {max(times[mode]):.4f})  "
                  f"logical {logical / ms / 1e9:.0f} TFLOP/s  padded {padded / ms / 1e9:.0f} TFLOP/s  "
                  f"L2->SM per group: A {a_b / 1e9:.3f} GB, B {b_b / 1e9:.3f} GB")


if __name__ == "__main__":
    main()
