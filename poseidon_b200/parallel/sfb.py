"""Sufficient-factor broadcasting (SFB / "SVB") for fully-connected layers.

For an InnerProduct weight W (N×K) the dense gradient of a batch of M samples is
ΔW = uᵀ·v with u = ∂L/∂y (M×N) and v = x (M×K).  Instead of all-reducing the N×K matrix,
every rank broadcasts its (u, v) and reconstructs ΔW_total = Σ_p u_pᵀ v_p = U_allᵀ·V_all
locally — one GEMM over the gathered P·M rows, then ONE optimizer step (the mathematically
clean version; the reference re-applies momentum/decay once per received factor, SURVEY S6).

This file holds the library-based implementation (``all_gather`` + cuBLAS GEMM) used by the
baseline engine and by the CPU/gloo tests, plus the cost-model hybrid chooser that decides
per layer between SFB and dense all-reduce (absent from the reference, which applies SFB to
every IP weight whenever ``--svb`` is on: tools/caffe_main.cpp:149-151, solver.cpp:434-436).
The fused NVLink-multicast + wgmma kernel version lives in ``fused.py`` / ``csrc/comm``.

reference: src/caffe/solver.cpp:477-531 (ThreadSyncWithSVB), src/caffe/svb_worker.cpp:125-167,
src/caffe/layers/inner_product_layer.cu:55-64 (ComputeGradientFromSV_gpu),
include/caffe/sufficient_vector.hpp:17-50.
"""
from __future__ import annotations

import logging
from typing import Dict

import torch
import torch.distributed as dist

log = logging.getLogger("poseidon_b200")


def sfb_wins(M: int, N: int, K: int, P: int) -> bool:
    """Per-GPU ingress bytes: SFB (P−1)·M·(N+K) vs two-shot dense all-reduce (1+1/P)·N·K."""
    return (P - 1) * M * (N + K) < (1.0 + 1.0 / P) * N * K


def sfb_bytes(M: int, N: int, K: int, P: int, elem: int = 4) -> Dict[str, int]:
    return {
        "sfb_egress": M * (N + K) * elem,
        "sfb_ingress": (P - 1) * M * (N + K) * elem,
        "dense_each_way": int((1.0 + 1.0 / P) * N * K * elem),
    }


class SufficientVector:
    """(u, v) factor pair of one layer with SVProto (de)serialisation — the unit the reference ships between
    machines (include/caffe/sufficient_vector.hpp:17-50, src/caffe/proto/caffe.proto:6-10)."""

    def __init__(self, a: torch.Tensor, b: torch.Tensor, layer_id: int = 0):
        self.a, self.b, self.layer_id = a, b, layer_id

    def to_proto(self):
        from .. import proto as P
        m = P.SVProto(layer_id=self.layer_id)
        m.a = self.a.detach().float().reshape(-1).cpu().numpy()
        m.b = self.b.detach().float().reshape(-1).cpu().numpy()
        return m

    @classmethod
    def from_proto(cls, m, a_shape, b_shape, device="cpu"):
        import numpy as np
        a = torch.from_numpy(np.asarray(m.a, dtype=np.float32).reshape(a_shape).copy()).to(device)
        b = torch.from_numpy(np.asarray(m.b, dtype=np.float32).reshape(b_shape).copy()).to(device)
        return cls(a, b, int(m.layer_id or 0))

    def gradient(self) -> torch.Tensor:
        """ΔW = aᵀ·b  (reference: inner_product_layer.cu:55-64 ComputeGradientFromSV_gpu)."""
        return self.a.t() @ self.b


class SufficientVectorQueue:
    """FIFO whose head is retired only after ``max_read_count`` readers have fetched it — the host-side queue of
    the reference (include/caffe/sufficient_vector_queue.hpp:17-35).  The fused engine replaces it with the
    double-buffered slot ring in the symmetric arena; this class serves the library path and tools."""

    def __init__(self, max_read_count: int):
        import threading
        self.max_read_count = max_read_count
        self.q = []
        self.read_count = 0
        self.lock = threading.Lock()

    def add(self, sv: SufficientVector):
        with self.lock:
            self.q.append(sv)

    def get(self):
        """Non-blocking: returns the head (shared) or None; the head is popped after max_read_count reads."""
        with self.lock:
            if not self.q:
                return None
            sv = self.q[0]
            self.read_count += 1
            if self.read_count >= self.max_read_count:
                self.q.pop(0)
                self.read_count = 0
            return sv

    def __len__(self):
        with self.lock:
            return len(self.q)


class SFBStats:
    def __init__(self):
        self.sfb_bytes = 0
        self.dense_equiv_bytes = 0
        self.layers: Dict[str, str] = {}


class _SFBLinear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, relu, world, layer_name, stats):
        x2 = x.reshape(x.shape[0], -1)
        y = torch.nn.functional.linear(x2, w.to(x2.dtype), None if b is None else b.to(x2.dtype))
        if relu:
            y = torch.relu(y)
        ctx.save_for_backward(x2, w, y if relu else None)
        ctx.relu, ctx.has_bias, ctx.world = relu, b is not None, world
        ctx.x_shape, ctx.stats = x.shape, stats
        return y

    @staticmethod
    def backward(ctx, dy):
        x2, w, y = ctx.saved_tensors
        if ctx.relu:
            dy = dy * (y > 0).to(dy.dtype)
        dy = dy.contiguous()
        dx = (dy @ w.to(dy.dtype)).reshape(ctx.x_shape) if ctx.needs_input_grad[0] else None
        db = dy.sum(0).to(torch.float32) if ctx.has_bias else None
        # --- sufficient-factor exchange: all-gather u and v, reconstruct the global ΔW ---
        P = ctx.world
        M, N = dy.shape
        K = x2.shape[1]
        fac = torch.cat([dy.reshape(-1), x2.reshape(-1).to(dy.dtype)])
        gathered = torch.empty(P * fac.numel(), dtype=fac.dtype, device=fac.device)
        dist.all_gather_into_tensor(gathered, fac)
        gathered = gathered.view(P, fac.numel())
        U = gathered[:, : M * N].reshape(P * M, N)
        V = gathered[:, M * N:].reshape(P * M, K)
        dw = (U.t() @ V).to(torch.float32)
        st = ctx.stats
        st.sfb_bytes += fac.numel() * fac.element_size()
        st.dense_equiv_bytes += N * K * 4
        return dx, dw, db, None, None, None, None


class SFBHandle:
    """Attached to an InnerProduct layer as ``layer.sfb``; the op engines route the layer's
    forward through it so that backward exchanges factors instead of a dense gradient."""

    def __init__(self, world: int, stats: SFBStats):
        self.world, self.stats = world, stats

    def apply(self, layer, x, w, b, relu):
        return _SFBLinear.apply(x, w, b, relu, self.world, layer.layer_name, self.stats)

    def exchange_and_update(self, layer, dy: torch.Tensor, x2: torch.Tensor):
        """Entry point of the sm100 engine's inner-product backward (ops/sm100.py::_IPFn) when the communication
        backend is a library one (NCCL / gloo: multi-node jobs): all-gather the bf16 factors u = dY [M,N], v = X [M,K],
        rebuild the global ΔW = Σ_p u_pᵀ v_p with our GEMM kernel and hand it to the optimizer as an already-global
        gradient (same contract as ``_SFBLinear.backward``; the fused NVLink engine has its own handle, FusedSFB)."""
        P = self.world
        M, N = dy.shape
        K = x2.shape[1]
        fac = torch.cat([dy.reshape(-1), x2.reshape(-1)])
        gathered = torch.empty(P * fac.numel(), dtype=fac.dtype, device=fac.device)
        dist.all_gather_into_tensor(gathered, fac)
        gathered = gathered.view(P, fac.numel())
        U = gathered[:, : M * N].reshape(P * M, N)
        V = gathered[:, M * N:].reshape(P * M, K)
        if N % 8 == 0 and K % 8 == 0 and U.dtype == torch.bfloat16:
            from ..ops import sm100
            dw = torch.empty(N, K, device=dy.device, dtype=torch.float32)
            sm100.K().gemm_f32(U, True, V, True, dw, 1.0, False, 1, 0)
        else:
            dw = U.float().t() @ V.float()
        self.stats.sfb_bytes += fac.numel() * fac.element_size()
        self.stats.dense_equiv_bytes += N * K * 4
        return dw


def enable_sfb(net, sync, rank_ctx, mode: str = "auto") -> SFBStats:
    """Mark IP weights for SFB. ``mode``: "all" (reference behaviour), "auto" (cost model),
    "none".  SFB weights carry an already-global gradient, so the dense backend must skip
    their all-reduce (bias still goes dense, as in the reference: solver.cpp:441-443)."""
    stats = SFBStats()
    if mode == "none" or not rank_ctx.distributed:
        return stats
    P = rank_ctx.world_size
    for li, (name, layer) in enumerate(zip(net.layer_names, net.layers)):
        if layer.type_name != "INNER_PRODUCT" or not layer.weight.requires_grad:
            continue
        N, K = layer.weight.shape
        M = net.blob_shapes[net.bottom_names[li][0]][0]
        use = mode == "all" or sfb_wins(M, N, K, P)
        stats.layers[name] = "sfb" if use else "dense"
        if use:
            layer.sfb = SFBHandle(P, stats)
            layer.weight._grad_is_global = True
            b = sync.bucket_of.get(id(layer.weight))
            if b is not None:
                b.mode = "sfb"
        if rank_ctx.is_root:
            by = sfb_bytes(M, N, K, P)
            log.info("SFB chooser: layer %s (M=%d N=%d K=%d P=%d): %s  [sfb ingress %.1f MB vs dense %.1f MB]",
                     name, M, N, K, P, stats.layers[name], by["sfb_ingress"] / 1e6, by["dense_each_way"] / 1e6)
    sync.sfb_stats = stats
    return stats
