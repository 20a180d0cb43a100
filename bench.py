#!/usr/bin/env python
"""Headline benchmark: training throughput (images/sec, whole job) of the flagship models.

Contract (see the task statement): ``python bench.py --gpus N --steps K --warmup W`` — for N > 1 it is
launched under ``torch.distributed.run`` (one rank per GPU, NCCL for bootstrap only).  Prints ONE JSON
line on rank 0.  ``--impl reference`` reports why the unmodified reference cannot run here.

What is timed
-------------
* ``value``      : K optimizer steps (forward + backward + DWBP/SFB communication + weight update) with the
                   input batch already resident on the device (the data layer's transform kernel still runs);
                   CUDA events on the compute stream, barrier + synchronize on both sides, max over ranks.
* ``e2e.value``  : the same K steps through the public API (``Solver.step``) with, every step, the raw uint8
                   batch copied host->device from pinned memory and the loss read back device->host.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

BASELINE_IMG_S_PER_GPU = 133.0   # BASELINE.md §1: derived 1.07 k img/s on 8 x K20 (AlexNet) — the only citeable figure


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--model", default="alexnet", choices=["alexnet", "caffenet", "googlenet", "vgg16", "lenet"])
    ap.add_argument("--allow-cpu", action="store_true",
                    help="self-test of the harness on a box without a GPU (wall-clock timed, torch engine; NOT a benchmark)")
    ap.add_argument("--engine", default="sm100", choices=["sm100", "torch"])
    ap.add_argument("--comm", default="auto")
    ap.add_argument("--batch", type=int, default=0, help="per-GPU batch (default: the reference prototxt's)")
    ap.add_argument("--svb", type=int, default=1)
    ap.add_argument("--sfb-mode", default="auto")
    ap.add_argument("--staleness", type=int, default=0)
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--graph", type=int, default=-1, help="CUDA-graph the step (default: on for the sm100 engine)")
    ap.add_argument("--vendor-dtype", default="bf16", choices=["bf16", "fp32"])
    ap.add_argument("--no-exposed-comm", action="store_true",
                    help="skip the compute-only arm (N > 1) that exposed_comm_ms is measured against")
    ap.add_argument("--require-nvls", action="store_true", help="fail if the arena has no NVLS multicast mapping")
    ap.add_argument("--dump-outputs", default="", metavar="DIR",
                    help="after the timed steps, write what the last timed step computed (loss, every learnable blob) "
                         "as DIR/<name>.npy; blobs over the budget are a fixed seeded sample")
    ap.add_argument("--kernel-list", default="", help="write a per-kernel time table (CUPTI via torch.profiler, a few EAGER "
                    "steps on every rank, rank r -> FILE.r) — works for multi-rank runs, where ncu cannot be used")
    return ap.parse_args()


class ClockSampler:
    """Samples SM clocks / throttle reasons with nvidia-smi while the timed region runs."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.idx = gpu_index
        self.samples = []
        self.proc = None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "100", "-i", str(self.idx)], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.samples.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], None, set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for s in self.samples:
            f = [x.strip() for x in s.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1]))
                mx = float(f[2])
            except ValueError:
                continue
            for name, v in zip(names, f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": mx, "reasons": sorted(reasons),
                "samples": len(sm)}


def reference_unavailable():
    why = ("petuum/poseidon cannot be built offline: needs the un-vendored petuum/third_party bundle (zmq, glog, gflags, "
           "leveldb, lmdb, hdf5, opencv, protobuf-dev), cuDNN R2/R3 APIs removed since cuDNN 8, and sm_20..sm_50 "
           "gencodes rejected by nvcc 12.9; the reference tree has no setup.py/pyproject to install it with (see DESIGN.md)")
    print(json.dumps({"impl": "reference", "unavailable": why}))


def measure_compute_only(args, rc):
    """The same per-GPU step with communication removed: every rank trains its own replica (world-size-1 context, local
    fused update) at the same time as its peers, so power and clocks match the N-GPU run.  exposed_comm_ms is the N-GPU
    step time minus this one."""
    from poseidon_b200.parallel.context import RankContext
    solo = RankContext(0, 1, rc.local_rank, rc.device)
    solver = build_solver(args, solo, device_resident=True)
    if args.engine == "sm100" or args.graph == 1:
        solver.enable_cuda_graph(warmup=2)
    for _ in range(max(3, args.warmup)):
        solver.step(1)
    ms, _ = timed_steps(solver, rc, args.steps, read_loss=False)      # rc: barrier + max over the REAL ranks
    solver.close()
    return ms / args.steps


def dump_kernel_list(args, rc, path):
    """Kernel names / counts / device time of 3 eager training steps of THIS rank (comm-stream kernels included)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    solver = build_solver(args, rc, device_resident=True)
    for _ in range(4):
        solver.step(1)
    solver.sync.wait_all()
    torch.cuda.synchronize(rc.device)
    rc.barrier()
    steps = 3
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            solver.step(1)
        solver.sync.wait_all()
        torch.cuda.synchronize(rc.device)
    rows = sorted(prof.key_averages(), key=lambda e: -e.device_time_total)
    cp = solver.sync.backend.comm_profile() if hasattr(solver.sync.backend, "comm_profile") else {}
    with open(f"{path}.{rc.rank}", "w") as f:
        f.write(f"# {args.model} rank {rc.rank}/{rc.world_size}, {steps} eager steps, CUPTI kernel times (torch.profiler)\n")
        f.write(f"# comm profile per step: {json.dumps(cp)}\n")
        f.write(f"{'us/step':>10s} {'calls/step':>10s} {'avg us':>9s}  kernel\n")
        for e in rows:
            if e.device_time_total <= 0:
                continue
            f.write(f"{e.device_time_total / steps:10.1f} {e.count / steps:10.1f} "
                    f"{e.device_time_total / max(e.count, 1):9.1f}  {e.key[:150]}\n")
    solver.close()


DUMP_BUDGET_BYTES = 64 << 20


def dump_outputs(solver, out_dir):
    """What a caller of the timed step gets back from its last step: the loss and the updated learnable blobs (Caffe
    layout, float32, as a snapshot writes them).  A blob larger than its share of the 64 MB budget is replaced by a
    sample at fixed indices (seeded by the blob's name, so two builds sample the same elements); the indices are
    written beside it as <name>.idx.npy."""
    import re
    import zlib
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    blobs = [(f"{lname}.{j}", layer, j) for lname, layer in zip(solver.net.layer_names, solver.net.layers)
             for j in range(len(layer.blobs))]
    cap = max(1, (DUMP_BUDGET_BYTES - 4096) // 12 // max(1, len(blobs)))     # 4 B value + 8 B index per sampled element
    np.save(os.path.join(out_dir, "loss.npy"), np.asarray([float(solver.last_loss)], dtype=np.float64))
    for name, layer, j in blobs:
        a = np.ascontiguousarray(layer.export_blob(j), dtype=np.float32).reshape(-1)
        fn = re.sub(r"[^A-Za-z0-9_.-]", "_", name)
        if a.size > cap:
            idx = np.sort(np.random.default_rng(zlib.crc32(name.encode())).choice(a.size, cap, replace=False))
            np.save(os.path.join(out_dir, fn + ".idx.npy"), idx.astype(np.int64))
            a = a[idx]
        np.save(os.path.join(out_dir, fn + ".npy"), a)


def build_solver(args, rank_ctx, device_resident: bool):
    import torch
    from poseidon_b200 import get_solver
    from poseidon_b200.models import zoo
    kw = {}
    if args.batch:
        kw["batch"] = args.batch
    net = zoo.get_model(args.model, **kw)
    sp = zoo.get_solver_param(args.model, net=net, display=0, snapshot=0, snapshot_after_train=False,
                              test_interval=0, max_iter=10 ** 9, random_seed=1234)
    sp.clear("test_iter")
    dtype = None
    if args.engine == "torch":
        dtype = torch.bfloat16 if args.vendor_dtype == "bf16" else torch.float32
    solver = get_solver(sp, rank_ctx=rank_ctx, engine=args.engine, comm=args.comm, svb=bool(args.svb),
                        sfb_mode=args.sfb_mode, staleness=args.staleness, dtype=dtype)
    for dl in solver.net.data_layers():
        dl.device_resident = device_resident
    return solver


def timed_steps(solver, rank_ctx, steps, read_loss: bool):
    import torch
    dev = rank_ctx.device
    rank_ctx.barrier()
    cuda = dev.type == "cuda"
    if cuda:
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    else:
        t0 = time.perf_counter()      # --allow-cpu self-test only
    last = None
    pending = None
    for _ in range(steps):
        solver.step(1)
        if read_loss:
            # device -> host read of EVERY step's loss: the copy into pinned memory is issued now and consumed one step
            # later, so the host never waits for a step to drain before launching the next one
            h = solver.read_loss_async()
            if pending is not None:
                last = pending.value()
            pending = h
    if pending is not None:
        last = pending.value()
    solver.sync.wait_all()
    if cuda:
        e1.record()
        torch.cuda.synchronize(dev)
        rank_ctx.barrier()
        ms = e0.elapsed_time(e1)
    else:
        rank_ctx.barrier()
        ms = (time.perf_counter() - t0) * 1e3
    return rank_ctx.max_over_ranks(ms), last


def measure_e2e(args, solver, rc, batch, world):
    """The same K steps through the public API with, every step, the raw uint8 batch copied host->device from pinned
    memory (prefetch thread + copy stream) and the step's loss copied device->host."""
    for dl in solver.net.data_layers():
        dl.device_resident = False
    for _ in range(max(3, args.warmup)):
        solver.step(1)
        float(solver.last_loss)
    ms2, _ = timed_steps(solver, rc, args.steps, read_loss=True)
    h2d = sum(getattr(dl.prefetch, "h2d_bytes", 0) for dl in solver.net.data_layers() if getattr(dl, "prefetch", None))
    return {"value": batch * world * args.steps / (ms2 / 1e3), "unit": "images/sec", "ms_per_step": ms2 / args.steps,
            "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": 4,
            "d2h": "loss of every step copied to pinned memory (async), read one step later"}


def main():
    args = parse_args()
    os.environ.setdefault("POSEIDON_SYNTHETIC_DATA", "1")     # the benchmark runs on stand-in data by contract (no datasets)
    if args.impl == "reference":
        reference_unavailable()
        return 0
    import torch
    from poseidon_b200 import init_rank_context
    from poseidon_b200.ops import sm100 as _sm  # noqa: F401
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.gpus != world and world == 1 and args.gpus > 1:
        # convenience: re-launch ourselves under torchrun
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={args.gpus}",
               "--master-addr", "127.0.0.1", "--master-port", str(29500 + os.getpid() % 1000), __file__] + sys.argv[1:]
        return subprocess.call(cmd)
    if args.require_nvls:
        os.environ["POSEIDON_REQUIRE_NVLS"] = "1"
    if args.engine == "torch" and "--svb" not in " ".join(sys.argv):
        args.svb = 0          # vendor baseline: dense NCCL all-reduce (DDP-style), no sufficient factors
    rc = init_rank_context("cpu" if (args.allow_cpu and not torch.cuda.is_available()) else None)
    if rc.device.type != "cuda":
        if not args.allow_cpu:
            print(json.dumps({"error": "bench.py needs a CUDA device"}))
            return 1
        from poseidon_b200.ops import sm100 as _sm100
        if not (args.engine == "sm100" and _sm100.emulating()):     # POSEIDON_EMULATE=1: the sm100 control flow on CPU stand-ins
            args.engine = "torch"
        args.graph = 0
    torch.backends.cudnn.benchmark = True
    if args.engine == "torch":
        torch.backends.cuda.matmul.allow_tf32 = args.vendor_dtype != "fp32"
        torch.backends.cudnn.allow_tf32 = args.vendor_dtype != "fp32"

    from poseidon_b200.ops import counting
    # ---------------- device-resident-input measurement (kernel + comm + update time)
    solver = build_solver(args, rc, device_resident=True)
    batch = solver.net.blob_shapes[solver.net.top_names[0][0]][0]
    # CUDA-graph the step: sm100 engine on one GPU, or on several with the fused NVLink backend (device-side epochs)
    use_graph = (args.graph == 1) or (args.graph < 0 and args.engine == "sm100" and
                                       (world == 1 or solver.comm_name == "fused"))
    if rc.device.type != "cuda":
        use_graph = False
    if use_graph and args.engine == "torch" and world > 1:
        # capturing NCCL collectives has hung (both ranks stuck inside the capture until the timeout) — the multi-GPU
        # vendor arm runs eager
        if rc.is_root:
            print("[bench] vendor arm on >1 GPU: NCCL capture is unreliable here, running eager", file=sys.stderr)
        use_graph = False
    if use_graph:
        try:
            solver.enable_cuda_graph(warmup=2)
        except Exception as exc:              # deterministic across ranks; the eager path is always available
            if rc.is_root:
                print(f"[bench] CUDA-graph capture failed ({type(exc).__name__}: {exc}); running eager", file=sys.stderr)
            use_graph = False
    for _ in range(args.warmup):
        solver.step(1)
    solver.sync.wait_all()
    sampler = ClockSampler(rc.device.index if rc.device.type == "cuda" else 0)
    if rc.is_root:
        sampler.start()
    counting.reset()
    ms, _ = timed_steps(solver, rc, args.steps, read_loss=False)
    if args.dump_outputs and rc.is_root:
        dump_outputs(solver, args.dump_outputs)
    launches = counting.total() + (args.steps * getattr(solver, 'graph_launches', 0) if use_graph else 0)
    clocks = sampler.stop() if rc.is_root else None
    value = batch * world * args.steps / (ms / 1e3)
    wire = solver.sync.backend.bytes_on_wire() if hasattr(solver.sync.backend, "bytes_on_wire") else {}
    sfb_layers = getattr(getattr(solver.sync.backend, "sfb_stats", None), "layers", {})
    comm_profile = solver.sync.backend.comm_profile() if hasattr(solver.sync.backend, "comm_profile") else {}
    # ---------------- end-to-end through the public API: pinned H2D of every batch + D2H of every loss
    e2e = None
    if not args.no_e2e:
        try:
            e2e = measure_e2e(args, solver, rc, batch, world)
        except Exception as exc:      # never lose the device-timed result to a failure of the end-to-end leg
            e2e = {"error": f"{type(exc).__name__}: {exc}"}
    solver.close()
    # ---------------- exposed communication time: N-GPU step minus the same step with communication removed
    exposed = None
    if world > 1 and not args.no_exposed_comm and rc.device.type == "cuda":
        try:
            ms_solo = measure_compute_only(args, rc)
            exposed = {"exposed_comm_ms": ms / args.steps - ms_solo, "compute_only_ms_per_step": ms_solo,
                       "how": "same step, every rank on its own replica (world-size-1 context, local fused update), all "
                              "ranks running concurrently; device-timed, max over ranks"}
        except Exception as exc:
            exposed = {"error": f"{type(exc).__name__}: {exc}"}
    if args.kernel_list and rc.device.type == "cuda":
        try:
            dump_kernel_list(args, rc, args.kernel_list)
        except Exception as exc:
            print(f"[bench] kernel list failed: {type(exc).__name__}: {exc}", file=sys.stderr)
    if rc.is_root:
        shape = solver.net.blob_shapes[solver.net.top_names[0][0]]
        out = {
            "metric": f"{args.model}_train_images_per_sec", "value": value, "unit": "images/sec", "n_gpus": world,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": value / (BASELINE_IMG_S_PER_GPU * world) if args.model == "alexnet" else None,
            "dtype": "fp32" if rc.device.type != "cuda" else
                     ("bf16" if (args.engine == "sm100" or args.vendor_dtype == "bf16") else "fp32"),
            "data": "synthetic (random uint8 images, random-init weights)",
            "config": {"model": args.model, "global_batch": batch * world, "per_gpu_batch": batch,
                       "input": list(shape[1:]), "seq_len": None,
                       "parallelism": f"dp{world}" + ("+dwbp" if world > 1 else "") +
                                      ("+sfb" if any(v == "sfb" for v in sfb_layers.values()) and world > 1 else ""),
                       "engine": args.engine, "comm": solver.comm_name, "cuda_graph": bool(use_graph),
                       "solver": "SGD momentum 0.9 wd 5e-4 (reference solver.prototxt)",
                       "l2": "per-step working set (weights+history+grads+activations) >> 50 MB L2; "
                             "inputs rotate over 4 batches",
                       "sfb_layers": sfb_layers, "wire_bytes_total": wire,
                       "baseline_ref": "133 img/s per K20 derived in BASELINE.md §1 (reference publishes no img/s)"},
            "clocks": clocks, "gpu_launches": launches,
            "impl": "ours" if args.engine == "sm100" else
                    "vendor_baseline (cuDNN/cuBLAS via PyTorch + NCCL; constructed, NOT the reference)",
            "sfb_layers": sfb_layers, "wire_bytes": comm_profile, "multimem": comm_profile.get("multimem"),
        }
        if exposed is not None:
            out["exposed_comm_ms"] = exposed.get("exposed_comm_ms")
            out["exposed_comm"] = exposed
        if e2e is not None:
            out["e2e"] = e2e
        print(json.dumps(out))
    rc.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
