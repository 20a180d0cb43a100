"""``caffe_main`` — the Poseidon command line, flag-for-flag.

    python -m poseidon_b200.tools.caffe_main train --solver=solver.prototxt [--gpu=0,1] [--snapshot=...]
        [--weights=...] [--svb=true] [--table_staleness=1] [--net_outputs=prefix] ...
    python -m poseidon_b200.tools.caffe_main test  --model=net.prototxt --weights=x.caffemodel --iterations=50
    python -m poseidon_b200.tools.caffe_main time  --model=net.prototxt --iterations=50
    python -m poseidon_b200.tools.caffe_main device_query [--gpu=0]

One process per GPU: with ``--gpu=0,1,..`` on a single host the tool re-launches itself under
``torch.distributed.run``; across hosts use torchrun (or ``--hostfile/--client_id``, Poseidon style).
Bösen-only tuning flags are accepted for script compatibility and ignored with a note.
``test`` and ``time`` are compiled out of the reference (``#if 0``); they work here.

reference: tools/caffe_main.cpp:24-46 (flags), :100-185 (train), :188-329 (test/time, disabled), :331-350 (main);
ps/src/petuum_ps_common/include/system_gflags.cpp:6-45, table_gflags.cpp:7-23 (PS flags).
"""
from __future__ import annotations

import argparse
import logging
import os
import subprocess
import sys
import time

log = logging.getLogger("poseidon_b200")

# PS / Bösen flags kept for command-line compatibility (value type only matters for parsing)
_PS_FLAGS = [
    "stats_path", "num_clients", "num_comm_channels_per_client", "init_thread_access_table", "num_table_threads",
    "consistency_model", "client_bandwidth_mbps", "server_bandwidth_mbps", "bg_idle_milli", "thread_oplog_batch_size",
    "row_candidate_factor", "server_idle_milli", "update_sort_policy", "snapshot_clock", "resume_clock", "snapshot_dir",
    "resume_dir", "numa_opt", "numa_index", "numa_policy", "naive_table_oplog_meta", "suppression_on", "use_approx_sort",
    "num_zmq_threads", "row_type", "row_oplog_type", "oplog_dense_serialized", "oplog_type", "append_only_oplog_type",
    "append_only_buffer_capacity", "append_only_buffer_pool_size", "bg_apply_append_oplog_freq", "process_storage_type",
    "no_oplog_replay", "server_push_row_upper_bound", "client_send_oplog_upper_bound", "server_table_logic",
    "version_maintain", "num_rows_per_table", "svb_timeout_ms",
]


def _bool(v):
    return str(v).lower() in ("1", "true", "yes", "on")


def make_parser():
    ap = argparse.ArgumentParser(prog="caffe_main", description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("command", choices=["train", "test", "time", "device_query"])
    ap.add_argument("--solver", default="")
    ap.add_argument("--model", default="")
    ap.add_argument("--gpu", default="", help="comma separated device ids (overrides solver device_id)")
    ap.add_argument("--snapshot", default="", help="resume from <prefix>_iter_N.solverstate")
    ap.add_argument("--weights", default="", help="finetune from a .caffemodel")
    ap.add_argument("--net_outputs", default="", help="prefix of the .netoutputs CSV")
    ap.add_argument("--iterations", type=int, default=50)
    ap.add_argument("--svb", default="false")
    ap.add_argument("--table_staleness", type=int, default=0)
    ap.add_argument("--hostfile", default="")
    ap.add_argument("--client_id", type=int, default=None)
    # framework-specific
    ap.add_argument("--engine", default="auto", choices=["auto", "sm100", "torch"])
    ap.add_argument("--comm", default="auto", choices=["auto", "fused", "nccl", "gloo", "ssp", "ssp_aggr", "local"])
    ap.add_argument("--aggr_fraction", type=float, default=0.1,
                    help="SSPAggr: fraction of the pending update sent per clock (the rest waits, bounded by --table_staleness)")
    ap.add_argument("--wire_dtype", default="", choices=["", "fp32", "bf16"],
                    help="gradients on the network as bf16 (= --row_oplog_type=3, the reference's DenseFloat16 oplogs)")
    ap.add_argument("--sfb_mode", default="auto", choices=["auto", "all", "none"])
    ap.add_argument("--grad_reduce", default="sum", choices=["sum", "mean"])
    ap.add_argument("--synthetic_shape", default="", help="CxHxW of stand-in data when a DB is absent")
    ap.add_argument("--cuda_graph", default="auto", choices=["auto", "0", "1"],
                    help="replay the training step as one CUDA graph (auto: sm100 engine with the fused backend)")
    ap.add_argument("--fp8", default=None, choices=["off", "fprop", "fprop+dgrad", "fprop+dgrad+wgrad"],
                    help="sm100 engine: run eligible convolution forward passes on fp8 (e4m3) operands; fprop+dgrad: "
                         "also eligible stride-1 data gradients (e5m2 dY x e4m3 weights); fprop+dgrad+wgrad: also "
                         "eligible stride-1 weight gradients (e5m2 dY x e4m3 X) (default: POSEIDON_FP8, else off)")
    ap.add_argument("--fp8_scaling", default=None, choices=["current", "delayed"],
                    help="with an fp8 mode on: current scales activations and dY just in time (an amax pass, then a "
                         "cast); delayed scales them from the amax history of their last 16 training steps in one pass, "
                         "saturating values beyond it (default: POSEIDON_FP8_SCALING, else current)")
    ap.add_argument("--stats_json", default="")
    ap.add_argument("--log_level", default="INFO")
    for f in _PS_FLAGS:
        ap.add_argument("--" + f, default=None, help=argparse.SUPPRESS)
    return ap


def parse_args(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    # gflags accepts "-flag=value" and "--flag=value"
    argv = [("-" + a if a.startswith("-") and not a.startswith("--") and len(a) > 2 else a) for a in argv]
    args = make_parser().parse_args(argv)
    # --consistency_model keeps its meaning: SSP / SSPPush -> bounded staleness (BSP at staleness 0), SSPAggr -> budgeted,
    # magnitude-prioritised updates
    cm = (getattr(args, "consistency_model", None) or "").lower()
    if args.comm == "auto" and cm == "sspaggr":
        args.comm = "ssp_aggr"
    elif args.comm == "auto" and cm == "ssp" and args.table_staleness > 0:
        args.comm = "ssp"
    ignored = [f for f in _PS_FLAGS if getattr(args, f) is not None and
               f not in ("stats_path", "num_rows_per_table", "consistency_model", "row_oplog_type")]
    args.ignored_ps_flags = ignored
    return args


def _maybe_relaunch(args) -> int:
    """--gpu=0,1,.. on one host => one process per GPU under torch.distributed.run."""
    ids = [g for g in args.gpu.split(",") if g.strip() != ""]
    if len(ids) <= 1 or "WORLD_SIZE" in os.environ:
        return -1
    env = dict(os.environ, CUDA_VISIBLE_DEVICES=",".join(ids))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={len(ids)}",
           "--master-addr", "127.0.0.1", "--master-port", str(29400 + os.getpid() % 500),
           "-m", "poseidon_b200.tools.caffe_main"] + sys.argv[1:]
    return subprocess.call(cmd, env=env)


def _setup_logging(level, rank):
    logging.basicConfig(level=getattr(logging, level.upper(), logging.INFO) if rank == 0 else logging.WARNING,
                        format="I%(asctime)s %(message)s", datefmt="%m%d %H:%M:%S")


def _engine(args, device):
    if args.engine != "auto":
        return args.engine
    return "sm100" if device.type == "cuda" else "torch"


def cmd_train(args) -> int:
    import torch
    from .. import proto as P
    from ..parallel.context import init_rank_context
    from ..solver.solver import get_solver
    from ..utils.stats import STATS
    if not args.solver:
        raise SystemExit("Need a solver definition to train.")
    if args.snapshot and args.weights:
        raise SystemExit("Give a snapshot to resume training or weights to finetune but not both.")
    rc_code = _maybe_relaunch(args)
    if rc_code >= 0:
        return rc_code
    sp = P.read_solver(args.solver)
    cpu_mode = sp.enum_name("solver_mode") == "CPU"
    device = "cpu" if cpu_mode else None
    if args.gpu and "WORLD_SIZE" not in os.environ and not cpu_mode:
        device = f"cuda:{args.gpu.split(',')[0]}"
    rc = init_rank_context(device, args.hostfile or None, args.client_id)
    _setup_logging(args.log_level, rc.rank)
    if args.ignored_ps_flags and rc.is_root:
        log.info("ignoring parameter-server-only flags (no PS in this framework): %s", ", ".join(args.ignored_ps_flags))
    hint = tuple(int(x) for x in args.synthetic_shape.lower().split("x")) if args.synthetic_shape else None
    solver = get_solver(sp, rank_ctx=rc, engine=_engine(args, rc.device), comm=args.comm,
                        staleness=args.table_staleness, svb=_bool(args.svb), grad_reduce=args.grad_reduce,
                        model_dir=os.path.dirname(os.path.abspath(args.solver)), data_shape_hint=hint,
                        sfb_mode=args.sfb_mode, aggr_fraction=args.aggr_fraction,
                        wire_dtype=args.wire_dtype or ("bf16" if str(args.row_oplog_type) == "3" else None),
                        fp8=args.fp8, fp8_scaling=args.fp8_scaling)
    if args.cuda_graph != "auto":
        solver.use_cuda_graph = args.cuda_graph == "1"
    if rc.is_root:
        log.info("Starting Optimization (world_size=%d, engine=%s, comm=%s, svb=%s, staleness=%d)",
                 rc.world_size, solver.engine, solver.comm_name, _bool(args.svb), args.table_staleness)
    if args.weights:
        log.info("Finetuning from %s", args.weights)
        solver.load_weights(args.weights)
    solver.solve(args.snapshot or None)
    if args.net_outputs:
        solver.print_net_outputs(args.net_outputs + ".netoutputs")
    if args.stats_path or args.stats_json:
        STATS.set("bytes_on_wire", solver.sync.backend.bytes_on_wire())
        if args.stats_path:
            STATS.dump_yaml(f"{args.stats_path}.{rc.rank}")
        if args.stats_json:
            import json
            with open(f"{args.stats_json}.{rc.rank}", "w") as f:
                json.dump(STATS.as_dict(), f)
    solver.close()
    rc.shutdown()
    return 0


def _build_net(args, phase):
    import torch
    from .. import proto as P
    from ..layers import NetContext
    from ..net.net import Net
    from ..ops.sm100 import fp8_for_engine, fp8_scaling_for_engine
    dev = torch.device(f"cuda:{args.gpu.split(',')[0] or 0}" if (torch.cuda.is_available() and args.gpu != "-1") else "cpu")
    if dev.type == "cuda":
        torch.cuda.set_device(dev)
    engine = _engine(args, dev)
    fp8 = fp8_for_engine(engine, args.fp8)
    ctx = NetContext(phase=phase, device=dev, engine=engine,
                     dtype=torch.bfloat16 if engine == "sm100" else torch.float32,
                     model_dir=os.path.dirname(os.path.abspath(args.model)), fp8=fp8,
                     fp8_scaling=fp8_scaling_for_engine(engine, fp8, args.fp8_scaling))
    if args.synthetic_shape:
        ctx.data_shape_hint = tuple(int(x) for x in args.synthetic_shape.lower().split("x"))
    net = Net(P.read_net(args.model), phase=phase, ctx=ctx)
    net.to(dev)
    return net, dev


def cmd_test(args) -> int:
    """Score a model: average every net output over --iterations batches.
    reference: tools/caffe_main.cpp:188-252 (compiled out there)."""
    import torch
    from .. import proto as P
    _setup_logging(args.log_level, 0)
    if not args.model or not args.weights:
        raise SystemExit("Need a model definition and model weights to score.")
    net, dev = _build_net(args, P.TEST)
    net.copy_trained_layers_from(args.weights)
    log.info("Running for %d iterations.", args.iterations)
    sums, loss_sum = {}, 0.0
    with torch.no_grad():
        for i in range(args.iterations):
            loss, outs = net.forward()
            loss_sum += float(loss) if loss is not None else 0.0
            for name, o in outs.items():
                for k, v in enumerate(o.float().reshape(-1).tolist()):
                    sums[(name, k)] = sums.get((name, k), 0.0) + v
                    log.info("Batch %d, %s = %g", i, name, v)
    log.info("Loss: %g", loss_sum / args.iterations)
    for (name, k), v in sums.items():
        log.info("%s = %g", name, v / args.iterations)
    return 0


def cmd_time(args) -> int:
    """Per-layer forward/backward timing (device timed). reference: tools/caffe_main.cpp:255-328 (compiled out)."""
    import torch
    from .. import proto as P
    from ..utils.timer import Timer
    _setup_logging(args.log_level, 0)
    if not args.model:
        raise SystemExit("Need a model definition to time.")
    # per-layer times only mean something when layers run one after the other: no branch lanes, no side streams
    os.environ["POSEIDON_LANES"] = "1"
    os.environ["POSEIDON_WGRAD_LANE"] = "0"
    net, dev = _build_net(args, P.TRAIN)
    log.info("Performing Forward + Backward warm-up")
    loss, _ = net.forward()
    if loss is not None and loss.requires_grad:
        loss.backward()
    net.zero_grad_()
    n = len(net.layers)
    fwd = [0.0] * n
    bwd = [0.0] * n
    total_f = total_b = 0.0
    hooks = []
    timers = [Timer(dev) for _ in range(n)]
    cuda = dev.type == "cuda"
    marks = []                    # (layer index | -1 for "backward finished", timestamp or CUDA event) in firing order

    def mark(i):
        if cuda:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            marks.append((i, ev))
        else:
            marks.append((i, time.perf_counter()))

    def after_forward(i, outs):
        timers[i].stop()
        # Backward of layer i starts when the gradient of its output is complete and ends when the next such
        # gradient (an earlier layer's output) is: autograd runs the graph in reverse topological order.
        for o in (outs if isinstance(outs, (tuple, list)) else (outs,)):
            if torch.is_tensor(o) and o.requires_grad:
                o.register_hook(lambda g, i=i: mark(i))
                break

    for i, layer in enumerate(net.layers):
        hooks.append(layer.register_forward_pre_hook(lambda m, a, i=i: timers[i].start()))
        hooks.append(layer.register_forward_hook(lambda m, a, o, i=i: after_forward(i, o)))
    for _ in range(args.iterations):
        tf = Timer(dev)
        tf.start()
        loss, _ = net.forward()
        total_f += tf.milliseconds()
        for i in range(n):
            fwd[i] += timers[i].milliseconds()
        tb = Timer(dev)
        tb.start()
        del marks[:]
        if loss is not None and loss.requires_grad:
            loss.backward()
        mark(-1)
        total_b += tb.milliseconds()
        for (i, t0), (_, t1) in zip(marks, marks[1:]):
            if i >= 0:
                bwd[i] += t0.elapsed_time(t1) if cuda else (t1 - t0) * 1e3
        net.zero_grad_()
    for h in hooks:
        h.remove()
    for i, name in enumerate(net.layer_names):
        log.info("%-28s forward: %.4f ms.", name, fwd[i] / args.iterations)
    for i in range(n - 1, -1, -1):
        log.info("%-28s backward: %.4f ms.", net.layer_names[i], bwd[i] / args.iterations)
    log.info("Average Forward pass: %.4f ms.", total_f / args.iterations)
    log.info("Average Backward pass: %.4f ms.", total_b / args.iterations)
    log.info("Average Forward-Backward: %.4f ms.", (total_f + total_b) / args.iterations)
    return 0


def cmd_device_query(args) -> int:
    """reference: tools/caffe_main.cpp:80-97, src/caffe/common.cpp:165-183 (DeviceQuery)."""
    import torch
    _setup_logging(args.log_level, 0)
    if not torch.cuda.is_available():
        log.info("No CUDA device visible (CPU mode).")
        return 0
    ids = [int(g) for g in args.gpu.split(",") if g.strip() != ""] or list(range(torch.cuda.device_count()))
    for i in ids:
        p = torch.cuda.get_device_properties(i)
        log.info("Device id:                     %d", i)
        log.info("Name:                          %s", p.name)
        log.info("Major revision number:         %d", p.major)
        log.info("Minor revision number:         %d", p.minor)
        log.info("Total global memory:           %d", p.total_memory)
        log.info("Number of multiprocessors:     %d", p.multi_processor_count)
        log.info("Shared memory per SM (opt-in): %d", getattr(p, "shared_memory_per_block_optin", 0))
        log.info("L2 cache size:                 %d", getattr(p, "L2_cache_size", 0))
    return 0


def main(argv=None) -> int:
    args = parse_args(argv)
    return {"train": cmd_train, "test": cmd_test, "time": cmd_time, "device_query": cmd_device_query}[args.command](args)


if __name__ == "__main__":
    sys.exit(main())
