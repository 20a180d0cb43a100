"""Solver family: SGD / Nesterov / AdaGrad with Caffe's exact semantics, distributed test,
snapshot / restore in the .caffemodel / .solverstate wire formats, and the net-outputs table.

reference: src/caffe/solver.cpp:42-63 (Init), :66-231 (InitTrainNet/InitTestNets), :246-402
(Solve), :405-451 (ForwardBackward), :543-628 (TestAll/Test), :632-696 (Snapshot/Restore),
:699-756 (PrintNetOutputs), :767-790 (GetLearningRate), :815-892 (SGD), :1013-1120
(Nesterov), :1240-1364 (AdaGrad); include/caffe/solver.hpp:186-205 (GetSolver).
"""
from __future__ import annotations

import logging
import math
import os
import time
from typing import Dict, List, Optional

import numpy as np
import torch

from .. import proto as P
from ..layers import NetContext, set_filler_seed
from ..net.net import Net
from ..parallel.context import RankContext
from ..parallel.gradsync import (ADAGRAD, NESTEROV, SGD, GradSync, Hyper, LocalBackend,
                                 SSPAggrBackend, SSPBackend, TorchDistBackend)
from ..utils import fault, trace
from ..utils.stats import STATS
from .lr_policy import learning_rate

log = logging.getLogger("poseidon_b200")

_NUM_FIXED_COLS = 3   # iter, time, loss — reference: include/caffe/common.hpp:65-70


class LossHandle:
    """Deferred read of a scalar device tensor (see :meth:`Solver.read_loss_async`)."""

    def __init__(self, t):
        self._t = t
        self._host = None
        self._ev = None
        if t is not None and t.is_cuda:
            try:
                self._host = torch.empty((), dtype=torch.float32, pin_memory=True)
                self._host.copy_(t.detach().float().reshape(()), non_blocking=True)
                self._ev = torch.cuda.Event()
                self._ev.record()
            except RuntimeError:
                self._host = None           # fall back to a synchronous read

    def value(self) -> float:
        if self._t is None:
            return float("nan")
        if self._host is None:
            return float(self._t)
        self._ev.synchronize()
        return float(self._host)


class OutputTable:
    """The "net outputs" table: every worker adds its row entries, rows are summed across
    workers (one tiny all-reduce per display point) and divided by #workers when printed.
    reference: src/caffe/caffe_engine.cpp:190-225, solver.cpp:336-369,596-610,699-756."""

    def __init__(self, names: List[str], rank_ctx: RankContext):
        self.names = names
        self.rank_ctx = rank_ctx
        self.rows: List[np.ndarray] = []

    def add_row(self, it: int, t: float, loss: float, values: List[float]):
        row = np.zeros(_NUM_FIXED_COLS + len(values), dtype=np.float64)
        if self.rank_ctx.is_root:
            row[0], row[1] = it, t
        row[2] = loss
        row[3:] = values
        if self.rank_ctx.distributed:
            tt = torch.from_numpy(row).to(self.rank_ctx.device)
            self.rank_ctx.all_reduce_(tt)
            row = tt.cpu().numpy()
        self.rows.append(row)

    def write(self, f, world: int):
        f.write("Iteration,time,loss," + "".join(n + "," for n in self.names) + "\n")
        for r in self.rows:
            vals = [r[0], r[1]] + [x / world for x in r[2:]]
            f.write(",".join("%g" % v for v in vals) + ",\n")


class Solver:
    solver_type = SGD

    def __init__(self, param, rank_ctx: Optional[RankContext] = None, engine: str = "torch",
                 comm: str = "auto", staleness: int = 0, svb: bool = False, grad_reduce: str = "sum",
                 dtype=None, model_dir: Optional[str] = None, data_shape_hint=None,
                 snapshot_dir: Optional[str] = None, sfb_mode: str = "auto", aggr_fraction: float = 0.1,
                 wire_dtype: Optional[str] = None, fp8: Optional[str] = None, fp8_scaling: Optional[str] = None):
        if isinstance(param, str):
            model_dir = model_dir or os.path.dirname(os.path.abspath(param))
            param = P.read_solver(param)
        self.param = param
        self.model_dir = model_dir
        if rank_ctx is None:
            use_cuda = torch.cuda.is_available() and param.enum_name("solver_mode") != "CPU"
            if use_cuda:
                ids = [int(x) for x in str(param.device_id or "0").split(",") if x.strip() != ""]
                rank_ctx = RankContext(device=f"cuda:{ids[0] if ids else 0}")
                torch.cuda.set_device(rank_ctx.device)
            else:
                rank_ctx = RankContext()
        self.rank_ctx = rank_ctx
        self.engine = engine
        from ..ops.sm100 import fp8_for_engine, fp8_scaling_for_engine
        self.fp8 = fp8_for_engine(engine, fp8)     # "fprop" / "fprop+dgrad" / "fprop+dgrad+wgrad" (ops/sm100.py)
        self.fp8_scaling = fp8_scaling_for_engine(engine, self.fp8, fp8_scaling)      # "current" / "delayed"
        self.staleness = int(staleness)
        self.aggr_fraction = float(aggr_fraction)
        # gradients on the network as bf16 (the reference's DenseFloat16 row oplogs: fp16 on the wire, fp32 at rest);
        # applies to the library all-reduce and to the fused engine's inter-node hop, never to NVLink traffic
        self.wire_dtype = (wire_dtype or os.environ.get("POSEIDON_WIRE_DTYPE", "fp32")).lower()
        if self.wire_dtype not in ("fp32", "bf16"):
            raise ValueError(f"wire_dtype must be fp32 or bf16, got '{self.wire_dtype}'")
        self.svb = bool(svb)
        self.iter = 0
        self.display_counter = 0
        self.test_counter = 0
        self.t0 = time.time()
        self.data_shape_hint = data_shape_hint
        self.snapshot_dir = snapshot_dir
        if dtype is None:
            dtype = torch.bfloat16 if engine == "sm100" else torch.float32
        self.dtype = dtype
        if param.random_seed is not None and param.random_seed >= 0:
            torch.manual_seed(int(param.random_seed))
            set_filler_seed(int(param.random_seed))
        self._init_train_net()
        self._init_test_nets()
        if self.solver_type == ADAGRAD and (param.momentum or 0) != 0:
            raise ValueError("Momentum cannot be used with AdaGrad.")
        self.hyper = Hyper(self.solver_type, float(param.momentum or 0.0), float(param.weight_decay or 0.0),
                           (param.regularization_type or "L2") == "L1", float(param.delta))
        if param.regularization_type not in (None, "L1", "L2"):
            raise ValueError(f"Unknown regularization type: {param.regularization_type}")
        self._sync_initial_weights()
        self.sync = self._make_sync(comm, grad_reduce, sfb_mode)
        trace.annotate_net(self.net)                 # NVTX ranges per layer when POSEIDON_NVTX=1
        self.last_loss = None

    # ---- net construction ------------------------------------------------------------------
    def _ctx(self, phase):
        dev = self.rank_ctx.device
        if self.param.enum_name("solver_mode") == "CPU" and dev.type != "cpu":
            dev = torch.device("cpu")
        seed = int(self.param.random_seed) if (self.param.random_seed or -1) >= 0 else None
        ctx = NetContext(phase=phase, device=dev, engine=self.engine, dtype=self.dtype,
                         rank=self.rank_ctx.rank, world_size=self.rank_ctx.world_size,
                         seed=None if seed is None else seed + self.rank_ctx.rank,
                         data_shape_hint=self.data_shape_hint, model_dir=self.model_dir, fp8=self.fp8,
                         fp8_scaling=self.fp8_scaling)
        return ctx

    def _resolve(self, path):
        """Net files named by the solver: CAFFE_ROOT placeholder, model directory, its ancestors, working directory."""
        from ..utils.paths import resolve
        return resolve(path, self.model_dir, basename_fallback=True)

    def _init_train_net(self):
        sp = self.param
        n = sum([sp.has("net"), sp.has("net_param"), sp.has("train_net"), sp.has("train_net_param")])
        if n == 0:
            raise ValueError("SolverParameter must specify a train net.")
        if n > 1:
            raise ValueError("SolverParameter must not contain more than one train net specifier.")
        if sp.has("train_net_param"):
            netp = sp.train_net_param.copy()
        elif sp.has("train_net"):
            netp = P.read_net(self._resolve(sp.train_net))
        elif sp.has("net_param"):
            netp = sp.net_param.copy()
        else:
            netp = P.read_net(self._resolve(sp.net))
        state = P.NetState(phase=P.TRAIN)
        if netp.has("state"):
            state.MergeFrom(netp.state)
        if sp.has("train_state"):
            state.MergeFrom(sp.train_state)
        state.phase = P.TRAIN
        netp.state = state
        self.net = Net(netp, ctx=self._ctx(P.TRAIN))
        self.net.to(self.net.ctx.device)
        self.device = self.net.ctx.device

    def _init_test_nets(self):
        sp = self.param
        has_net_param, has_net_file = sp.has("net_param"), sp.has("net")
        n_generic = int(has_net_param) + int(has_net_file)
        n_tnp, n_tnf = len(sp.test_net_param), len(sp.test_net)
        n_iter = len(sp.test_iter)
        n_inst = n_tnp + n_tnf
        if n_generic > 1:
            raise ValueError("Both net_param and net_file may not be specified.")
        if n_inst:
            if n_inst != n_iter:
                raise ValueError("test_iter must be specified for each test network.")
        elif n_generic and n_iter == 0:
            self.test_nets = []
            return
        n_all = n_inst + (n_iter - n_inst if n_generic else 0)
        if n_all != n_iter:
            raise ValueError("test_iter must be specified for each test network.")
        if n_all and not sp.test_interval:
            raise ValueError("test_interval must be positive when test nets are given")
        sources = []
        for np_ in sp.test_net_param:
            sources.append(np_.copy())
        for f in sp.test_net:
            sources.append(P.read_net(self._resolve(f)))
        remaining = n_iter - n_inst
        for _ in range(remaining):
            sources.append(sp.net_param.copy() if has_net_param else P.read_net(self._resolve(sp.net)))
        if len(sp.test_state) not in (0, n_all):
            raise ValueError("test_state must be unspecified or specified once per test net.")
        self.test_nets = []
        for i, netp in enumerate(sources):
            state = P.NetState(phase=P.TEST)
            if netp.has("state"):
                state.MergeFrom(netp.state)
            if len(sp.test_state):
                state.MergeFrom(sp.test_state[i])
            state.phase = P.TEST
            netp.state = state
            tn = Net(netp, ctx=self._ctx(P.TEST))
            tn.to(self.device)
            tn.share_trained_layers_with(self.net)
            self.test_nets.append(tn)

    def _sync_initial_weights(self):
        """Rank 0's fillers define the model; everyone else receives a broadcast (the
        reference's client0/thread0 FillPSTable + initial SyncWithPS:
        include/caffe/layer.hpp:464-497, src/caffe/solver.cpp:304-306)."""
        if self.rank_ctx.distributed:
            for p in self.net.params:
                self.rank_ctx.broadcast_(p.data, 0)

    def _make_sync(self, comm, grad_reduce, sfb_mode):
        rc = self.rank_ctx
        local_world = int(os.environ.get("LOCAL_WORLD_SIZE", rc.world_size))
        if comm == "auto":
            if not rc.distributed:
                comm = "local"
            elif self.staleness > 0 and not (self.engine == "sm100" and 1 < local_world == rc.world_size):
                comm = "ssp"                     # library bounded staleness (torch engine / multi-node jobs)
            elif self.engine == "sm100":
                # NVLink arena per node (+ a library all-reduce across nodes); one GPU per node has no NVLink peer
                comm = "fused" if int(os.environ.get("LOCAL_WORLD_SIZE", rc.world_size)) > 1 else "nccl"
            else:
                comm = "nccl"
        self.comm_name = comm
        if self.engine == "sm100" and comm in ("fused", "local"):
            from ..ops import sm100
            if not sm100.active(self.device):
                raise RuntimeError("the sm100 engine needs a CUDA device (H100)")
            from ..parallel.fused import FusedBackend
            self.comm_name = "fused"
            backend = FusedBackend(self.svb, sfb_mode, grad_reduce, staleness=self.staleness)
            backend.wire_bf16 = self.wire_dtype == "bf16"
            return GradSync(self.net, rc, self.hyper, backend)
        if comm == "local":
            backend = LocalBackend()
        elif comm in ("nccl", "gloo", "torchdist"):
            backend = TorchDistBackend(grad_reduce)
        elif comm == "ssp":
            backend = SSPBackend(self.staleness)
        elif comm == "ssp_aggr":
            backend = SSPAggrBackend(self.staleness, self.aggr_fraction)
        else:
            raise ValueError(f"unknown comm backend '{comm}' for engine '{self.engine}'")
        backend.wire_bf16 = self.wire_dtype == "bf16"
        sync = GradSync(self.net, rc, self.hyper, backend)
        if self.svb and rc.distributed:
            from ..parallel.sfb import enable_sfb
            enable_sfb(self.net, sync, rc, sfb_mode)
        return sync

    # ---- training loop -------------------------------------------------------------------------
    def elapsed(self):
        return time.time() - self.t0

    def step(self, iters: int = 1):
        """Run ``iters`` training iterations (no test / snapshot scheduling)."""
        for _ in range(iters):
            self._train_iteration()

    # ---- CUDA-graph execution: the whole step (forward, backward, DWBP hooks, fused updates) is one graph ----
    GRAPH_WARMUP = 2

    def _graph_wanted(self) -> bool:
        """``solve()`` (i.e. ``caffe_main train`` and ``CaffeEngine.start``) replays the training step as one CUDA graph
        whenever that is possible: sm100 engine on a GPU with the fused backend (one GPU, or many with BSP).  The library
        backends can be graphed on request (``use_cuda_graph=True`` / POSEIDON_CUDA_GRAPH=1).  Eager otherwise."""
        mode = getattr(self, "use_cuda_graph", None)
        env = os.environ.get("POSEIDON_CUDA_GRAPH", "")
        if env in ("0", "1"):
            mode = env == "1"
        if mode is False or self.device.type != "cuda" or bool(self.param.debug_info):
            return False
        name = type(self.sync.backend).__name__
        if name == "FusedBackend":
            from ..ops import sm100
            return not sm100.emulating()
        return bool(mode) and name in ("LocalBackend", "TorchDistBackend")

    def _graph_window_ok(self, max_iter: int) -> bool:
        """Capturing runs GRAPH_WARMUP eager iterations plus the captured one inside ``enable_cuda_graph``: start only
        where none of them is a snapshot / test boundary and the captured one is not a display iteration."""
        sp, w = self.param, self.GRAPH_WARMUP
        if self.iter + w + 1 > max_iter:
            return False
        for interval in (int(sp.snapshot or 0), int(sp.test_interval or 0)):
            if interval and (self.iter + w) // interval != self.iter // interval:
                return False
        return not (sp.display and (self.iter + w) % int(sp.display) == 0)

    def _try_enable_graph(self) -> bool:
        try:
            self.enable_cuda_graph(warmup=self.GRAPH_WARMUP)
            if self.rank_ctx.is_root:
                log.info("Training step captured as one CUDA graph (%d kernels of this framework per replay)",
                         getattr(self, "graph_launches", 0))
            return True
        except Exception as exc:          # deterministic across ranks (same net, same backend): everyone falls back together
            self._graph = None
            log.warning("CUDA-graph capture failed (%s: %s); continuing with eager launches", type(exc).__name__, exc)
            return False

    def read_loss_async(self):
        """Start a device->host copy of the latest step's loss into page-locked memory and return a handle whose
        ``.value()`` blocks only on that copy.  Reading the handle one step later keeps the copy off the critical
        path (``float(solver.last_loss)`` instead stalls the host until the whole step has drained, which opens a
        launch bubble before the next step)."""
        return LossHandle(self.last_loss)

    def enable_cuda_graph(self, warmup: int = 3):
        """Capture forward+backward+update of everything after the data layers into a CUDA graph and replay it
        every iteration (launch-bound nets such as GoogLeNet at batch 32).  The data layers stay eager and feed
        static input tensors; the learning rate and the dropout iteration counter live in device memory so replays
        see fresh values, and so does the fused NVLink backend's epoch counter (multi-GPU replays stay in lock step
        through the in-kernel flag protocol)."""
        fused_comm = type(self.sync.backend).__name__ == "FusedBackend"
        library = type(self.sync.backend).__name__ in ("LocalBackend", "TorchDistBackend")
        if self.device.type != "cuda":
            raise RuntimeError("CUDA-graph steps need a CUDA device")
        if not fused_comm and not library:
            raise RuntimeError("CUDA-graph steps need the fused NVLink backend (device-side epochs) or the all-reduce "
                               "library backend; the bounded-staleness library backends schedule on the host")
        if library:
            # the constructed vendor baseline (any engine): per-bucket all-reduce from the hooks + one foreach SGD step,
            # learning rate in device memory
            self.sync.backend.enable_deferred_step(self.device)
        from ..ops import sm100
        net = self.net
        k = net.num_leading_data_layers()
        # PyTorch's whole-network capture recipe: warm up on the side stream the capture will use, so that the
        # autograd accumulators and the caching allocator are bound to it (not to the legacy default stream)
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup)):
                self._train_iteration()
            self._g_inputs = {n: t.clone() for n, t in net.forward_data().items()}
        side.synchronize()
        torch.cuda.synchronize(self.device)
        if self.rank_ctx.distributed:
            # the captured step must be self-contained: it forks the comm stream at its first bucket and joins it at
            # the end, so it may not wait on events recorded by the eager warm-up steps
            self.rank_ctx.barrier()
            for b in self.sync.buckets:
                b.event = None
                b.sfb_event = None
            for h in getattr(self.sync.backend, "sfb_layers", {}).values():
                h.event = None
        self._g_first = k
        self.sync.begin_iteration(learning_rate(self.param, self.iter))
        if self.rank_ctx.distributed and library:
            for b in self.sync.buckets:
                b.event = None
        graph = torch.cuda.CUDAGraph()
        from ..ops import counting
        n0 = counting.total()
        with torch.cuda.stream(side):
            with torch.cuda.graph(graph, stream=side):
                sm100.bump_iteration_seed(self.device)
                loss, outs = net.forward(self._g_inputs, start=k)
                loss.backward()
                self.sync.finish_iteration()
        torch.cuda.current_stream().wait_stream(side)
        if self.rank_ctx.distributed:
            for b in self.sync.buckets:      # events recorded during capture are graph-internal: never wait on them eagerly
                b.event = None
                b.sfb_event = None
            for h in getattr(self.sync.backend, "sfb_layers", {}).values():
                h.event = None
        graph.replay()       # capture only records: run the captured step once on the batch that was staged for it
        self.graph_launches = counting.total() - n0          # kernels of ours inside one replay
        self._graph, self._g_loss, self._g_outs = graph, loss.detach(), {n: o.detach() for n, o in outs.items()}
        self.iter += 1           # the capture pass executed one real step
        return graph

    def _graph_iteration(self):
        sp = self.param
        display = bool(sp.display) and self.iter % sp.display == 0
        lr = learning_rate(sp, self.iter)
        fresh = self.net.forward_data()
        for n, t in fresh.items():
            self._g_inputs[n].copy_(t, non_blocking=True)
        if hasattr(self.sync.backend, "set_lr"):
            self.sync.backend.set_lr(lr)
        self._graph.replay()
        self.last_loss = self._g_loss
        if display:
            self._display(self._g_loss, self._g_outs, lr)
        self.iter += 1
        STATS.count("iterations")

    def _train_iteration(self):
        fault.maybe_inject(self.rank_ctx.rank, self.iter)
        if getattr(self, "_graph", None) is not None:
            return self._graph_iteration()
        sp = self.param
        display = bool(sp.display) and self.iter % sp.display == 0
        self.net.debug_info = display and bool(sp.debug_info)
        lr = learning_rate(sp, self.iter)
        self.sync.begin_iteration(lr)
        if self.engine == "sm100":
            from ..ops import sm100
            if sm100.active(self.device):
                sm100.bump_iteration_seed(self.device)
        with STATS.timer("forward_backward"):
            loss, outputs = self.net.forward()
            if loss is not None and loss.requires_grad:
                loss.backward()
        self.sync.finish_iteration()
        if self.net.debug_info:
            self.net.backward_debug()
        self.last_loss = None if loss is None else loss.detach()
        if display:
            self._display(loss, outputs, lr)
        self.iter += 1
        STATS.count("iterations")

    def _display(self, loss, outputs, lr):
        lossv = float(loss.detach().float().cpu()) if loss is not None else 0.0
        t = self.elapsed()
        root = self.rank_ctx.is_root
        if root:
            log.info("Iteration %d, loss: %g, time: %g", self.iter, lossv, t)
            log.info("Iteration %d, lr = %g", self.iter, lr)
        names, vals = [], []
        idx = 0
        lw = self._output_loss_weights(self.net)
        for name in self.net.output_names:
            o = outputs.get(name)
            if o is None:
                continue
            flat = o.detach().float().reshape(-1).cpu().tolist()
            w = lw.get(name, 0.0)
            for v in flat:
                if root:
                    msg = f" (* {w:g} = {w * v:g} loss)" if w else ""
                    log.info("    Train net output #%d: %s = %g%s", idx, name, v, msg)
                names.append(name)
                vals.append(v * (w if w else 1.0))
                idx += 1
        if not hasattr(self, "train_table"):
            self.train_table = OutputTable(names, self.rank_ctx)
        self.train_table.add_row(self.iter, t, lossv, vals)
        self.display_counter += 1
        self._emit_metrics(lossv, lr, dict(zip(names, vals)))

    # ---- JSONL metrics (SURVEY §5.5): one line per display point, throughput timed on the device ----------------------
    def _emit_metrics(self, lossv, lr, outputs):
        path = os.environ.get("POSEIDON_METRICS_JSONL") or getattr(self, "metrics_path", None)
        if not path:
            return
        now_iter = self.iter
        cuda = self.device.type == "cuda"
        if cuda:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
        else:
            ev = time.time()
        prev = getattr(self, "_metrics_prev", None)
        self._metrics_prev = (now_iter, ev)
        rec = {"iter": now_iter, "loss": lossv, "lr": lr, "rank": self.rank_ctx.rank, "world_size": self.rank_ctx.world_size,
               "outputs": outputs}
        if prev is not None and now_iter > prev[0]:
            if cuda:
                ev.synchronize()
                dt = prev[1].elapsed_time(ev) / 1e3
            else:
                dt = ev - prev[1]
            batch = self.net.blob_shapes[self.net.top_names[0][0]][0] if self.net.top_names and self.net.top_names[0] else 0
            if dt > 0:
                rec["images_per_sec_per_rank"] = batch * (now_iter - prev[0]) / dt
                rec["ms_per_iter"] = 1e3 * dt / (now_iter - prev[0])
        wire = getattr(self.sync.backend, "bytes_on_wire", None)
        if wire is not None:
            rec["bytes_on_wire"] = wire()
        if self.rank_ctx.is_root:
            os.makedirs(os.path.dirname(os.path.abspath(path)) or ".", exist_ok=True)
            import json
            with open(path, "a") as f:
                f.write(json.dumps(rec) + "\n")

    @staticmethod
    def _output_loss_weights(net) -> Dict[str, float]:
        out = {}
        for tn, lw in zip(net.top_names, net.loss_weights):
            for t, w in zip(tn, lw):
                out[t] = w
        return out

    def solve(self, resume_file: Optional[str] = None):
        sp = self.param
        if self.rank_ctx.is_root:
            log.info("Solving %s", self.net.name)
        if resume_file:
            self.restore(resume_file)
        self.rank_ctx.barrier()
        self.t0 = time.time()
        max_iter = int(sp.max_iter or 0)
        want_graph = self._graph_wanted()
        while self.iter < max_iter:
            if sp.snapshot and self.iter > int(getattr(self, "_start_iter", 0)) and self.iter % sp.snapshot == 0:
                self.snapshot()
            if sp.test_interval and self.iter % sp.test_interval == 0 and \
                    (self.iter > 0 or sp.test_initialization):
                self.test_all()
            if want_graph and getattr(self, "_graph", None) is None and self._graph_window_ok(max_iter):
                want_graph = self._try_enable_graph()          # runs GRAPH_WARMUP + 1 real iterations
                continue
            self._train_iteration()
        self.sync.wait_all()
        if hasattr(self.sync.backend, "drain"):
            self.sync.backend.drain()
        if sp.snapshot_after_train:
            self.snapshot()
        if sp.display and max_iter % sp.display == 0:
            with torch.no_grad():
                loss, _ = self.net.forward()
            if self.rank_ctx.is_root and loss is not None:
                log.info("Iteration %d, loss = %g", self.iter, float(loss))
        if sp.test_interval and max_iter % sp.test_interval == 0:
            self.test_all()
        self.rank_ctx.barrier()
        if self.rank_ctx.is_root:
            log.info("Optimization Done.")

    # ---- evaluation -------------------------------------------------------------------------------
    def test_all(self):
        for i in range(len(self.test_nets)):
            self.test(i)

    def test(self, test_net_id: int = 0):
        """Each worker runs ceil((test_iter / num_clients) / num_threads) batches of its own
        shard; scores are summed over workers and divided by #workers when printed.
        reference: src/caffe/solver.cpp:552-628."""
        sp = self.param
        net = self.test_nets[test_net_id]
        self.sync.wait_all()
        if hasattr(self.sync.backend, "drain"):
            self.sync.backend.drain()          # evaluate the table all workers agree on (see snapshot())
        world = self.rank_ctx.world_size
        n_iters = max(1, int(math.ceil(float(sp.test_iter[test_net_id]) / world)))
        scores: List[float] = []
        names: List[str] = []
        loss_sum = 0.0
        with torch.no_grad():
            for i in range(n_iters):
                loss, outputs = net.forward()
                if sp.test_compute_loss and loss is not None:
                    loss_sum += float(loss)
                k = 0
                for name in net.output_names:
                    o = outputs.get(name)
                    if o is None:
                        continue
                    for v in o.detach().float().reshape(-1).cpu().tolist():
                        if i == 0:
                            scores.append(v)
                            names.append(name)
                        else:
                            scores[k] += v
                        k += 1
        root = self.rank_ctx.is_root
        if root:
            log.info("Iteration %d, Testing net (#%d)", self.iter, test_net_id)
        mean = [s / n_iters for s in scores]
        lossv = loss_sum / n_iters if sp.test_compute_loss else 0.0
        if not hasattr(self, "test_tables"):
            self.test_tables = {}
        tab = self.test_tables.setdefault(test_net_id, OutputTable(names, self.rank_ctx))
        tab.add_row(self.iter, self.elapsed(), lossv, mean)
        row = tab.rows[-1]
        if root:
            if sp.test_compute_loss:
                log.info("Test loss: %g", row[2] / world)
            lw = self._output_loss_weights(net)
            for i, name in enumerate(names):
                v = row[3 + i] / world
                w = lw.get(name, 0.0)
                msg = f" (* {w:g} = {w * v:g} loss)" if w else ""
                log.info("    Test net output #%d: %s = %g%s", i, name, v, msg)
        self.test_counter += 1
        return {n: row[3 + i] / world for i, n in enumerate(names)}

    def print_net_outputs(self, filename: str):
        """reference: src/caffe/solver.cpp:699-756 (CSV, values averaged over workers)."""
        if not self.rank_ctx.is_root:
            return
        os.makedirs(os.path.dirname(os.path.abspath(filename)) or ".", exist_ok=True)
        with open(filename, "w") as f:
            if self.param.display and hasattr(self, "train_table"):
                self.train_table.write(f, self.rank_ctx.world_size)
                f.write("\n")
            if self.param.test_interval:
                for i in sorted(getattr(self, "test_tables", {})):
                    self.test_tables[i].write(f, self.rank_ctx.world_size)
                    f.write("\n")

    # ---- snapshot / restore ---------------------------------------------------------------------------
    def _snapshot_prefix(self):
        from ..utils.paths import expand_placeholder
        prefix = expand_placeholder(self.param.snapshot_prefix or "snapshot", self.model_dir, must_exist=False)
        if self.snapshot_dir:
            prefix = os.path.join(self.snapshot_dir, os.path.basename(prefix))
        d = os.path.dirname(prefix)
        if d:
            os.makedirs(d, exist_ok=True)
        return prefix

    def snapshot(self):
        """``<prefix>_iter_N.caffemodel`` by rank 0 and ``<prefix>_iter_N.solverstate[.<rank>]``.
        Optimizer state is replicated in the synchronous modes (single rank-0 file); under SSP
        momentum is per-worker and every rank writes its own suffixed file like the reference.
        reference: src/caffe/solver.cpp:632-667, 990-997."""
        self.sync.wait_all()
        if hasattr(self.sync.backend, "drain"):
            # bounded-staleness backends: fold in the peers' in-flight deltas / flush unsent residuals first, so that the
            # rank-0 .caffemodel is the table every worker agrees on (a collective: every rank snapshots at the same iter)
            self.sync.backend.drain()
        if self.device.type == "cuda":
            torch.cuda.synchronize(self.device)
        base = f"{self._snapshot_prefix()}_iter_{self.iter}"
        model_file = base + ".caffemodel"
        state_file = base + ".solverstate"
        # per-worker momentum in the asynchronous modes (library ssp / ssp_aggr, or the fused engine's SSP kernels)
        per_rank = self.comm_name in ("ssp", "ssp_aggr") or getattr(self.sync.backend, "per_worker_state", False)
        if hasattr(self.sync.backend, "gather_history"):
            # a collective (two-shot buckets keep the optimizer history sharded by rank): EVERY rank takes part, not
            # only the one that writes the file
            self.sync.backend.gather_history()
        if self.rank_ctx.is_root:
            netp = self.net.to_proto(bool(self.param.snapshot_diff))
            log.info("Snapshotting to %s", model_file)
            P.write_binary(model_file, netp)
        if self.rank_ctx.is_root or per_rank:
            st = P.SolverState(iter=self.iter, learned_net=model_file)
            for h, (layer, j) in zip(self.sync.history_tensors(), self.net.param_owner):
                st.history.append(P.array_to_blob(layer.export_blob(j, h)))
            fn = state_file + (f".{self.rank_ctx.rank}.0" if per_rank else "")
            log.info("Snapshotting solver state to %s", fn)
            P.write_binary(fn, st)
        self.rank_ctx.barrier()
        return model_file, state_file

    def restore(self, state_file: str):
        """reference: src/caffe/solver.cpp:670-696 (per-worker suffix, falling back to the
        unsuffixed / worker-0 file), 1000-1010."""
        cands = [f"{state_file}.{self.rank_ctx.rank}.0", state_file, f"{state_file}.0.0"]
        fn = next((c for c in cands if os.path.exists(c)), None)
        if fn is None:
            raise FileNotFoundError(state_file)
        st = P.read_binary(fn, P.SolverState)
        if st.has("learned_net"):
            path = st.learned_net
            if not os.path.exists(path):
                path = os.path.join(os.path.dirname(os.path.abspath(fn)), os.path.basename(path))
            if self.rank_ctx.is_root:
                self.net.copy_trained_layers_from(path)
            self._sync_initial_weights()
            if hasattr(self.sync, "weights_changed"):
                self.sync.weights_changed()
        self.iter = int(st.iter)
        self._start_iter = self.iter
        hs = self.sync.history_tensors()
        if len(st.history) != len(hs):
            raise ValueError("Incorrect length of history blobs.")
        for b, h, (layer, j) in zip(st.history, hs, self.net.param_owner):
            layer.import_blob(j, np.asarray(b.data, dtype=np.float32), tensor=h)
        if self.fp8_scaling == "delayed":
            from ..ops import sm100
            sm100.reset_amax_histories(self.net)      # not in the snapshot: the resumed run seeds them on its first step
        if self.rank_ctx.is_root:
            log.info("Restored solver state from %s (iter %d)", fn, self.iter)

    def load_weights(self, model_file: str):
        """Finetune: rank 0 loads a .caffemodel, everyone receives it.
        reference: src/caffe/caffe_engine.cpp:277-282, blob.cpp:403-411."""
        if self.rank_ctx.is_root:
            self.net.copy_trained_layers_from(model_file)
        self._sync_initial_weights()
        if hasattr(self.sync, "weights_changed"):
            self.sync.weights_changed()

    def close(self):
        self.net.close()
        for t in self.test_nets:
            t.close()
        if hasattr(self.sync.backend, "close"):
            self.sync.backend.close()


class SGDSolver(Solver):
    solver_type = SGD


class NesterovSolver(Solver):
    solver_type = NESTEROV


class AdaGradSolver(Solver):
    solver_type = ADAGRAD


def get_solver(param, *args, **kw) -> Solver:
    """reference: include/caffe/solver.hpp:186-205 (GetSolver factory)."""
    if isinstance(param, str):
        kw.setdefault("model_dir", os.path.dirname(os.path.abspath(param)))
        param = P.read_solver(param)
    t = param.enum_name("solver_type")
    cls = {"SGD": SGDSolver, "NESTEROV": NesterovSolver, "ADAGRAD": AdaGradSolver}.get(t)
    if cls is None:
        raise ValueError(f"Unknown SolverType: {t}")
    return cls(param, *args, **kw)
