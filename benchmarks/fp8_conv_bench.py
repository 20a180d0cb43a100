"""Forward time per fp8-eligible convolution: bf16 (conv_fprop) against fp8 (fp8_quant_weight + fp8_quant_act +
conv_fprop_fp8), each with its relative error against an fp32 reference of the same layer.  Then the data gradient per
layer eligible under fp8="fprop+dgrad": bf16 (conv_dgrad_w, the kernel the engine runs for these layers) against fp8
(fp8_quant_weight_dgrad + fp8_quant_grad + conv_dgrad_fp8), without the producer's ReLU mask.  Then the weight gradient
per layer eligible under fp8="fprop+dgrad+wgrad": bf16 conv_wgrad against fp8 (fp8_quant_act_t + fp8_quant_grad_t +
conv_wgrad_fp8), with the reduction length each split of the fp8 GEMM runs (the accumulation-length figure of DESIGN §16).

    python benchmarks/fp8_conv_bench.py [--iters 50] [--json out.json] [--only fprop|dgrad|wgrad]

Layers: the convolutions the engine's plan runs in fp8 for AlexNet at batch 256, VGG-16 at batch 64 and GoogLeNet at
batch 32 (duplicate shapes once).  The quantise launches are reported on their own and inside the fp8 total, since the
just-in-time activation scale costs one extra read of the layer input.  Times are CUDA events over --iters launches after
warm-up; the card's name, power limit and maximum SM clock are printed from the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("POSEIDON_SYNTHETIC_DATA", "1")

NETS = [("alexnet", 256), ("vgg16", 64), ("googlenet", 32)]


def eligible_layers(mode="fprop"):
    """(net, layer, N, Cin, H, W, Cout, k, stride, pad, groups, slots) of every conv the fp8 plan selects: for the forward
    (mode "fprop", slots = Cgk8), the data gradient (mode "fprop+dgrad", slots = Cok8) or the weight gradient (mode
    "fprop+dgrad+wgrad", slots = Cgkw8)."""
    from poseidon_b200 import proto as P
    from poseidon_b200.layers import NetContext
    from poseidon_b200.models import zoo
    from poseidon_b200.net.net import Net
    from poseidon_b200.ops import sm100
    out, seen = [], set()
    sm100.set_emulation(True)          # plan on the CPU: only the layer geometry is needed here
    try:
        for name, batch in NETS:
            ctx = NetContext(phase=P.TRAIN, device="cpu", engine="sm100", dtype=torch.bfloat16, fp8=mode)
            net = Net(getattr(zoo, name)(batch=1, test_batch=1), phase=P.TRAIN, ctx=ctx)
            for i, layer in enumerate(net.layers):
                st = getattr(layer, "_sm100", None)
                pick = {"fprop": "fp8", "fprop+dgrad": "fp8_dgrad", "fprop+dgrad+wgrad": "fp8_wgrad"}[mode]
                if layer.type_name != "CONVOLUTION" or not getattr(st, pick):
                    continue
                _, c, h, w = net.blob_shapes[net.bottom_names[i][0]]
                key = (batch, c, h, w, layer.num_output, layer.kernel, layer.stride, layer.pad, layer.group)
                if key in seen:
                    continue
                seen.add(key)
                out.append((name, net.layer_names[i], batch, c, h, w, layer.num_output, layer.kernel[0], layer.stride[0],
                            layer.pad[0], layer.group,
                            {"fprop": st.cgk8, "fprop+dgrad": st.cok8, "fprop+dgrad+wgrad": st.cgkw8}[mode]))
    finally:
        sm100.set_emulation(False)
    return out


def time_ms(fn, iters):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", default="")
    ap.add_argument("--only", choices=["fprop", "dgrad", "wgrad"], default=None, help="run one section")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "fp8_conv_bench needs a CUDA device"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(f"card: {card[0] if card else 'unknown'}")
    layers = eligible_layers()
    from poseidon_b200.ops.build import load_extension
    load_extension()
    k = torch.ops.poseidon
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    rows = []
    hdr = f"{'net':10s} {'layer':26s} {'shape':28s} {'bf16 ms':>8s} {'qw ms':>7s} {'qx ms':>7s} {'gemm ms':>8s} " \
          f"{'fp8 ms':>8s} {'speedup':>7s} {'err bf16':>9s} {'err fp8':>9s}"
    print(hdr)
    g = torch.Generator(device="cuda").manual_seed(0)
    for net, name, n, c, h, w, cout, ks, s, p, grp, cgk8 in (layers if args.only in (None, "fprop") else []):
        cg = c // grp
        oh, ow = (h + 2 * p - ks) // s + 1, (w + 2 * p - ks) // s + 1
        x = torch.randn(n, c, h, w, device="cuda", generator=g).clamp_(min=0).to(torch.bfloat16) \
            .contiguous(memory_format=torch.channels_last)
        wm = (torch.randn(cout, cg, ks, ks, device="cuda", generator=g) * (2.0 / (cg * ks * ks)) ** 0.5) \
            .contiguous(memory_format=torch.channels_last)
        bias = torch.randn(cout, device="cuda", generator=g) * 0.01
        wb = wm.permute(0, 2, 3, 1).reshape(cout, -1).to(torch.bfloat16).contiguous()
        s_x, s_w = torch.empty(1, device="cuda"), torch.empty(cout, device="cuda")
        args_c = ([ks, ks], [s, s], [p, p], grp)

        def bf16():
            return k.conv_fprop(x, wb, bias, *args_c[:3], grp, 0, oh, ow, True, 0.0, None)

        w8 = k.fp8_quant_weight(wm, cgk8, s_w)
        x8 = k.fp8_quant_act(x, s_x)

        def gemm8():
            return k.conv_fprop_fp8(x8, w8, s_x, s_w, bias, *args_c, oh, ow, True, 0.0, None)

        def fp8():
            w8_ = k.fp8_quant_weight(wm, cgk8, s_w)
            x8_ = k.fp8_quant_act(x, s_x)
            return k.conv_fprop_fp8(x8_, w8_, s_x, s_w, bias, *args_c, oh, ow, True, 0.0, None)

        t_bf = time_ms(bf16, args.iters)
        t_qw = time_ms(lambda: k.fp8_quant_weight(wm, cgk8, s_w), args.iters)
        t_qx = time_ms(lambda: k.fp8_quant_act(x, s_x), args.iters)
        t_g8 = time_ms(gemm8, args.iters)
        t_f8 = time_ms(fp8, args.iters)
        ref = F.relu(F.conv2d(x.float(), wm, bias, s, p, 1, grp))
        nref = ref.norm().item()
        e_bf = (bf16().float() - ref).norm().item() / nref
        e_f8 = (fp8().float() - ref).norm().item() / nref
        shape = f"{n}x{c}x{h}x{w}->{cout} k{ks}s{s}g{grp}"
        print(f"{net:10s} {name:26s} {shape:28s} {t_bf:8.3f} {t_qw:7.3f} {t_qx:7.3f} {t_g8:8.3f} {t_f8:8.3f} "
              f"{t_bf / t_f8:7.2f} {e_bf:9.2e} {e_f8:9.2e}")
        rows.append(dict(net=net, layer=name, shape=shape, bf16_ms=t_bf, quant_w_ms=t_qw, quant_x_ms=t_qx, gemm_fp8_ms=t_g8,
                         fp8_total_ms=t_f8, rel_err_bf16=e_bf, rel_err_fp8=e_f8))
        del x, wm, wb, w8, x8
        torch.cuda.empty_cache()
    for net, _ in NETS:
        sel = [r for r in rows if r["net"] == net]
        if sel:
            tb, tf = sum(r["bf16_ms"] for r in sel), sum(r["fp8_total_ms"] for r in sel)
            print(f"{net}: distinct eligible layers {len(sel)}, bf16 {tb:.3f} ms, fp8 {tf:.3f} ms (x{tb / tf:.2f})")
    drows = dgrad_rows(k, args.iters) if args.only in (None, "dgrad") else []
    wrows = wgrad_rows(k, args.iters) if args.only in (None, "wgrad") else []
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card, layers=rows, dgrad=drows, wgrad=wrows), f, indent=1)


def dgrad_rows(k, iters):
    """Data gradient of every layer the fprop+dgrad plan runs in fp8: bf16 conv_dgrad_w against the three fp8 launches."""
    rows = []
    print(f"\n{'data gradient':10s} {'layer':26s} {'shape':28s} {'bf16 ms':>8s} {'qw ms':>7s} {'qdy ms':>7s} "
          f"{'gemm ms':>8s} {'fp8 ms':>8s} {'speedup':>7s} {'err bf16':>9s} {'err fp8':>9s}")
    g = torch.Generator(device="cuda").manual_seed(1)
    for net, name, n, c, h, w, cout, ks, s, p, grp, cok8 in eligible_layers("fprop+dgrad"):
        cg = c // grp
        oh, ow = h + 2 * p - ks + 1, w + 2 * p - ks + 1
        dy = (torch.randn(n, cout, oh, ow, device="cuda", generator=g) * 1e-3).to(torch.bfloat16) \
            .contiguous(memory_format=torch.channels_last)
        wm = (torch.randn(cout, cg, ks, ks, device="cuda", generator=g) * (2.0 / (cg * ks * ks)) ** 0.5) \
            .contiguous(memory_format=torch.channels_last)
        wb = wm.permute(0, 2, 3, 1).reshape(cout, -1).to(torch.bfloat16).contiguous()
        s_dy, s_wt = torch.empty(1, device="cuda"), torch.empty(c, device="cuda")
        geo = ([ks, ks], [p, p], grp, h, w)

        def bf16():
            return k.conv_dgrad_w(dy, wb, *geo, None, 0.0)

        wt8 = k.fp8_quant_weight_dgrad(wm, grp, cok8, s_wt)
        dy8, _ = k.fp8_quant_grad(dy, s_dy, None, 0.0)

        def fp8():
            wt8_ = k.fp8_quant_weight_dgrad(wm, grp, cok8, s_wt)
            dy8_, _ = k.fp8_quant_grad(dy, s_dy, None, 0.0)
            return k.conv_dgrad_fp8(dy8_, wt8_, s_dy, s_wt, *geo, None, 0.0)

        t_bf = time_ms(bf16, iters)
        t_qw = time_ms(lambda: k.fp8_quant_weight_dgrad(wm, grp, cok8, s_wt), iters)
        t_qd = time_ms(lambda: k.fp8_quant_grad(dy, s_dy, None, 0.0), iters)
        t_g8 = time_ms(lambda: k.conv_dgrad_fp8(dy8, wt8, s_dy, s_wt, *geo, None, 0.0), iters)
        t_f8 = time_ms(fp8, iters)
        ref = torch.nn.grad.conv2d_input((n, c, h, w), wm, dy.float(), 1, p, 1, grp)
        nref = ref.norm().item()
        e_bf = (bf16().float() - ref).norm().item() / nref
        e_f8 = (fp8().float() - ref).norm().item() / nref
        shape = f"{n}x{cout}x{oh}x{ow}->{c} k{ks}g{grp}"
        print(f"{net:10s} {name:26s} {shape:28s} {t_bf:8.3f} {t_qw:7.3f} {t_qd:7.3f} {t_g8:8.3f} {t_f8:8.3f} "
              f"{t_bf / t_f8:7.2f} {e_bf:9.2e} {e_f8:9.2e}")
        rows.append(dict(net=net, layer=name, shape=shape, bf16_ms=t_bf, quant_w_ms=t_qw, quant_dy_ms=t_qd,
                         gemm_fp8_ms=t_g8, fp8_total_ms=t_f8, rel_err_bf16=e_bf, rel_err_fp8=e_f8))
        del dy, wm, wb, wt8, dy8
        torch.cuda.empty_cache()
    for net, _ in NETS:
        sel = [r for r in rows if r["net"] == net]
        if sel:
            tb, tf = sum(r["bf16_ms"] for r in sel), sum(r["fp8_total_ms"] for r in sel)
            print(f"{net} data gradient: distinct eligible layers {len(sel)}, bf16 {tb:.3f} ms, fp8 {tf:.3f} ms "
                  f"(x{tb / tf:.2f})")
    return rows


def wgrad_split_length(n, oh, ow, cout_g, cols, sms):
    """Pixels one split of conv_wgrad_fp8 reduces over (its k blocks x 128): the op's tile-width and split-K rules
    (csrc/gemm/conv_ops.cu conv_wgrad_fp8)."""
    from poseidon_b200.ops.emulate import chwn_images
    np_ = chwn_images(n)
    wr, nch = (128 // np_, 1) if np_ < 128 else (1, np_ // 128)
    kb = oh * -(-ow // wr) * nch
    bn = 128 if -(-cols // 128) * 128 * 8 <= cols * 9 else 64
    tiles = -(-cout_g // 128) * -(-cols // bn)
    split = min(max(1, -(-2 * sms // tiles)), max(1, kb // 8))
    return -(-kb // split) * 128


def wgrad_rows(k, iters):
    """Weight gradient of every layer the fprop+dgrad+wgrad plan runs in fp8: bf16 conv_wgrad against the three fp8
    launches, with the relative error of both against fp32 and the fp8 GEMM's reduction length per split."""
    rows = []
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"\n{'weight gradient':10s} {'layer':26s} {'shape':28s} {'bf16 ms':>8s} {'qx ms':>7s} {'qdy ms':>7s} "
          f"{'gemm ms':>8s} {'fp8 ms':>8s} {'speedup':>7s} {'err bf16':>9s} {'err fp8':>9s} {'split px':>8s}")
    g = torch.Generator(device="cuda").manual_seed(2)
    for net, name, n, c, h, w, cout, ks, s, p, grp, cgkw8 in eligible_layers("fprop+dgrad+wgrad"):
        cg = c // grp
        oh, ow = h + 2 * p - ks + 1, w + 2 * p - ks + 1
        x = torch.randn(n, c, h, w, device="cuda", generator=g).clamp_(min=0).to(torch.bfloat16) \
            .contiguous(memory_format=torch.channels_last)
        dy = (torch.randn(n, cout, oh, ow, device="cuda", generator=g) * 1e-3).to(torch.bfloat16) \
            .contiguous(memory_format=torch.channels_last)
        dw = torch.zeros(cout, ks * ks * cg, device="cuda")
        s_dy, s_x = torch.empty(1, device="cuda"), torch.empty(1, device="cuda")

        def bf16():
            dw.zero_()
            k.conv_wgrad(x, dy, dw, [ks, ks], [1, 1], [p, p], grp, 0, 1.0, cg)

        dy8t, _, _ = k.fp8_quant_grad_t(dy, s_dy, None, 0.0, False)
        x8t = k.fp8_quant_act_t(x, s_x)

        def fp8():
            dw.zero_()
            d_, _, _ = k.fp8_quant_grad_t(dy, s_dy, None, 0.0, False)
            x_ = k.fp8_quant_act_t(x, s_x)
            k.conv_wgrad_fp8(d_, x_, s_dy, s_x, dw, [ks, ks], [p, p], grp, 1.0, cgkw8)

        t_bf = time_ms(bf16, iters)
        t_qx = time_ms(lambda: k.fp8_quant_act_t(x, s_x), iters)
        t_qd = time_ms(lambda: k.fp8_quant_grad_t(dy, s_dy, None, 0.0, False), iters)
        t_g8 = time_ms(lambda: k.conv_wgrad_fp8(dy8t, x8t, s_dy, s_x, dw, [ks, ks], [p, p], grp, 1.0, cgkw8), iters)
        t_f8 = time_ms(fp8, iters)
        ref = torch.nn.grad.conv2d_weight(x.float(), (cout, cg, ks, ks), dy.float(), 1, p, 1, grp)
        ref = ref.permute(0, 2, 3, 1).reshape(cout, -1)
        nref = ref.norm().item()
        bf16()
        e_bf = (dw - ref).norm().item() / nref
        fp8()
        e_f8 = (dw - ref).norm().item() / nref
        split_px = wgrad_split_length(n, oh, ow, cout // grp, ks * ks * cgkw8, sms)
        shape = f"{n}x{c}x{h}x{w}->{cout} k{ks}g{grp}"
        print(f"{net:10s} {name:26s} {shape:28s} {t_bf:8.3f} {t_qx:7.3f} {t_qd:7.3f} {t_g8:8.3f} {t_f8:8.3f} "
              f"{t_bf / t_f8:7.2f} {e_bf:9.2e} {e_f8:9.2e} {split_px:8d}")
        rows.append(dict(net=net, layer=name, shape=shape, bf16_ms=t_bf, quant_x_ms=t_qx, quant_dy_ms=t_qd,
                         gemm_fp8_ms=t_g8, fp8_total_ms=t_f8, rel_err_bf16=e_bf, rel_err_fp8=e_f8,
                         split_pixels=split_px))
        del x, dy, dw, dy8t, x8t
        torch.cuda.empty_cache()
    for net, _ in NETS:
        sel = [r for r in rows if r["net"] == net]
        if sel:
            tb, tf = sum(r["bf16_ms"] for r in sel), sum(r["fp8_total_ms"] for r in sel)
            tg = sum(r["gemm_fp8_ms"] for r in sel)
            print(f"{net} weight gradient: distinct eligible layers {len(sel)}, bf16 {tb:.3f} ms, fp8 {tf:.3f} ms "
                  f"(x{tb / tf:.2f}; GEMM alone {tg:.3f} ms), longest split {max(r['split_pixels'] for r in sel)} px")
    return rows


if __name__ == "__main__":
    main()
