"""CaffeEngine — the process-level runtime object of the reference, re-thought for one-process-per-GPU.

The reference's ``CaffeEngine`` (src/caffe/caffe_engine.cpp:79-305) does three jobs:

1. a *pre-pass* over the train / test nets that counts and creates the parameter-server tables (two per
   CONV / INNER_PRODUCT layer, one "net outputs" table per net);
2. ``Start()``: per worker thread — register with the PS, bind the GPU, build the solver, then
   ``Solve`` / resume from a snapshot / fine-tune from weights, barrier, dump ``.netoutputs``;
3. ``StartExtractingFeature()``: the same bring-up for the distributed feature extractor.

Here a "worker thread" is a rank (one process per GPU), the "tables" are the buckets of the gradient-sync
backend (symmetric-memory arena segments for the fused NVLink engine), and bring-up is
``init_rank_context`` + ``get_solver``.  The pre-pass survives as :meth:`plan`, which reports exactly what
the reference would have created tables for — and what this framework communicates instead (dense
all-reduce+SGD kernel vs. sufficient-factor push per layer).
"""
from __future__ import annotations

import dataclasses
import logging
import os
from typing import Dict, List, Optional

from . import proto as P

log = logging.getLogger("poseidon_b200")


@dataclasses.dataclass
class TablePlan:
    """One parameter blob that the reference would bind to a PS table."""
    layer: str
    blob: int                 # 0 weight, 1 bias
    count: int
    global_id: int
    route: str                # "dense" | "sfb" | "local"


class CaffeEngine:
    def __init__(self, solver_param, rank_ctx=None, *, engine: str = "auto", comm: str = "auto", svb: bool = True,
                 staleness: int = 0, grad_reduce: str = "sum", sfb_mode: str = "auto", model_dir: Optional[str] = None,
                 data_shape_hint=None, aggr_fraction: float = 0.1, wire_dtype: Optional[str] = None,
                 fp8: Optional[str] = None, fp8_scaling: Optional[str] = None):
        if isinstance(solver_param, str):
            model_dir = model_dir or os.path.dirname(os.path.abspath(solver_param))
            solver_param = P.read_solver(solver_param)
        self.solver_param = solver_param
        self.rank_ctx = rank_ctx
        self.opts = dict(engine=engine, comm=comm, svb=svb, staleness=staleness, grad_reduce=grad_reduce,
                         sfb_mode=sfb_mode, model_dir=model_dir, data_shape_hint=data_shape_hint,
                         aggr_fraction=aggr_fraction, wire_dtype=wire_dtype, fp8=fp8, fp8_scaling=fp8_scaling)
        self.solver = None

    # ---------------------------------------------------------------------------------- bring-up
    def _ensure_rank(self):
        if self.rank_ctx is None:
            from .parallel.context import init_rank_context
            cpu = self.solver_param.enum_name("solver_mode") == "CPU"
            self.rank_ctx = init_rank_context("cpu" if cpu else None)
        return self.rank_ctx

    def build(self):
        """Create nets + solver + communication backend on this rank (``CaffeEngine::Start`` up to Solve)."""
        if self.solver is None:
            from .solver.solver import get_solver
            rc = self._ensure_rank()
            o = dict(self.opts)
            eng = o.pop("engine")
            if eng == "auto":
                eng = "sm100" if rc.device.type == "cuda" else "torch"
            self.solver = get_solver(self.solver_param, rank_ctx=rc, engine=eng, **o)
        return self.solver

    # ---------------------------------------------------------------------------------- pre-pass
    def plan(self) -> List[TablePlan]:
        """What the reference's InitPSForTrainNet would create (caffe_engine.cpp:79-128), annotated with the
        route each blob takes here."""
        solver = self.build()
        backend = solver.sync.backend
        sfb_layers: Dict[str, str] = dict(getattr(getattr(backend, "sfb_stats", None), "layers", {}) or {})
        out: List[TablePlan] = []
        gid = 0
        for layer in solver.net.layers:
            for j, p in enumerate(layer.blobs):
                route = "local" if solver.rank_ctx.world_size == 1 else "dense"
                if j == 0 and sfb_layers.get(layer.layer_name) == "sfb" and solver.rank_ctx.world_size > 1:
                    route = "sfb"
                out.append(TablePlan(layer.layer_name, j, p.numel(), gid, route))
                gid += 1
        return out

    # ---------------------------------------------------------------------------------- Start()
    def start(self, snapshot: Optional[str] = None, weights: Optional[str] = None, net_outputs: Optional[str] = None):
        """Solve (optionally resuming / fine-tuning), barrier, dump net outputs. reference: caffe_engine.cpp:251-293."""
        if snapshot and weights:
            raise ValueError("give a snapshot to resume training or weights to finetune, not both")
        solver = self.build()
        if weights:
            solver.load_weights(weights)
        solver.solve(snapshot or None)
        solver.rank_ctx.barrier()
        if net_outputs:
            solver.print_net_outputs(net_outputs + ".netoutputs")
        return solver

    def start_extracting_feature(self, weights: str, model: str, blobs: List[str], dbs: List[str], num_mini_batches: int):
        """reference: caffe_engine.cpp:296-305 -> FeatureExtractor::ExtractFeatures."""
        from .tools import extract_features
        return extract_features.main([weights, model, ",".join(blobs), ",".join(dbs), str(num_mini_batches)])

    def close(self):
        if self.solver is not None:
            self.solver.close()
            self.solver = None
