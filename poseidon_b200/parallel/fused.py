"""The product's communication backend: fused NVLink kernels, no NCCL on the hot path.

* ``SymmetricArena`` — one symmetric-memory allocation per rank (CUDA VMM, peer-mapped on every rank
  and bound to an NVLS multicast object; handles come from ``torch.distributed._symmetric_memory``,
  which is bootstrap plumbing only).  It holds, at identical offsets on every rank: the gradient
  staging buffer G, the fp32 master weights W, the bf16 shadow weights Wb, the sufficient-factor
  staging slots (u, v per SFB layer and rank; single-buffered, guarded by "consumed" flags), the bounded-staleness
  delta rings (SSP mode) and the epoch-flag blocks.
  This replaces the Bösen PS tables + process/thread caches (reference: src/caffe/blob.cpp:58-83,
  ps/src/petuum_ps/client/client_table.cpp:26-158, ps/src/petuum_ps/server/server_table.cpp).
* ``FusedBackend`` — per-bucket ``allreduce_sgd`` kernel (two-shot, history sharded across ranks;
  one-shot for small buckets) launched from the DWBP hooks on a high-priority stream.
* ``FusedSFB`` — sufficient-factor broadcasting: every rank PUSHES its u, v into slot `rank` of every peer's arena
  (one NVSwitch-multicast store stream) and raises a release flag; ONE wgmma kernel then walks the P local slots as
  P reduction sources (waiting on slot p's flag right before its first TMA load) and accumulates Σ_p u_pᵀ v_p in registers
  with the optimizer step fused into its epilogue — no dense ΔW ever exists, locally or on the wire.  With one rank it
  degenerates to the fused wgrad+update kernel.

reference: src/caffe/solver.cpp:455-531 (ThreadSyncWithPS / ThreadSyncWithSVB),
src/caffe/svb_worker.cpp:19-179, ps/src/petuum_ps/thread/ssp_push_bg_worker.cpp:12-68.
"""
from __future__ import annotations

import logging
import os
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from ..ops import sm100
from .gradsync import Backend, Bucket
from .sfb import SFBStats, sfb_bytes, sfb_wins

log = logging.getLogger("poseidon_b200")

K_MAX_RANKS = 8
_ALIGN = 256          # bytes; every arena segment starts on this boundary


def _round_up(x, a):
    return (x + a - 1) // a * a


class _NoCuda:
    """Stand-ins for the CUDA stream API when the engine runs on the CPU emulation of the kernels (ops/emulate.py,
    tests only): everything is synchronous there, so streams and events degenerate to no-ops."""

    class Stream:
        def __init__(self, *a, **k):
            pass

        def wait_stream(self, s):
            pass

    class Event:
        def __init__(self, *a, **k):
            pass

        def record(self, s=None):
            pass

    @staticmethod
    def current_stream(device=None):
        return _NoCuda.Stream()

    @staticmethod
    def stream(s):
        import contextlib
        return contextlib.nullcontext()

    @staticmethod
    def synchronize(device=None):
        pass

    @staticmethod
    def is_current_stream_capturing():
        return False


def _record_stream(t: torch.Tensor, s) -> None:
    if t.is_cuda:
        t.record_stream(s)


class SymmetricArena:
    def __init__(self, nbytes: int, rank_ctx):
        import torch.distributed._symmetric_memory as symm
        self.rank, self.world = rank_ctx.rank, rank_ctx.world_size
        self.device = rank_ctx.device
        nbytes = _round_up(nbytes, 2 << 20)
        group = getattr(rank_ctx, "group", None) or dist.group.WORLD      # the node-local group on multi-node jobs
        group_name = group.group_name
        try:
            symm.enable_symm_mem_for_group(group_name)      # required on some builds, deprecated no-op on others
        except Exception:
            pass
        self.buf = symm.empty(nbytes, dtype=torch.uint8, device=self.device)
        self.hdl = symm.rendezvous(self.buf, group_name)
        self.buf.zero_()
        self.base_ptrs = [int(p) for p in self.hdl.buffer_ptrs]
        mc = getattr(self.hdl, "multicast_ptr", 0) or 0
        self.multicast_ptr = int(mc)
        self.offset = 0
        self.nbytes = nbytes
        # Which branch the comm kernels will take is decided here and nowhere else: a non-zero multicast pointer means
        # multimem.ld_reduce / multimem.st through the NVSwitch (NVLS); zero means per-peer P2P loads / stores.
        if self.rank == 0:
            log.info("symmetric arena: %d MiB per rank, %d ranks, NVLS multicast %s", nbytes >> 20, self.world,
                     f"mapped at {self.multicast_ptr:#x}" if self.multicast_ptr else "UNAVAILABLE (P2P loads/stores)")
        if os.environ.get("POSEIDON_REQUIRE_NVLS", "0") == "1" and not self.multicast_ptr:
            raise RuntimeError("POSEIDON_REQUIRE_NVLS=1 but the symmetric-memory rendezvous returned no multicast mapping")
        torch.cuda.synchronize(self.device)
        rank_ctx.barrier()

    def carve(self, nbytes: int) -> int:
        off = self.offset
        self.offset = _round_up(off + nbytes, _ALIGN)
        if self.offset > self.nbytes:
            raise RuntimeError("symmetric arena exhausted")
        return off

    def view(self, off: int, shape, dtype) -> torch.Tensor:
        n = 1
        for s in shape:
            n *= s
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        return self.buf[off:off + nbytes].view(dtype).view(*shape)

    def peer_ptrs(self, off: int) -> List[int]:
        return [b + off for b in self.base_ptrs]

    def mc_ptr(self, off: int) -> int:
        return self.multicast_ptr + off if self.multicast_ptr else 0


class _Seg:
    __slots__ = ("param", "numel", "g_off", "w_off", "wb_off", "hist", "d_off")


class _NodeContext:
    """The ranks of one node as seen by the arena: local rank / world, the node's process group, a group barrier."""
    distributed = True

    def __init__(self, rank: int, world_size: int, device, group, node_id: int):
        self.rank, self.world_size, self.device, self.group, self.node_id = rank, world_size, device, group, node_id

    def barrier(self):
        if self.device.type == "cuda":
            dist.barrier(group=self.group, device_ids=[self.device.index])
        else:
            dist.barrier(group=self.group)


class FusedBackend(Backend):
    manages_operands = True        # its kernels rewrite the bf16 operands next to the fp32 masters
    name = "fused"

    def __init__(self, svb: bool = False, sfb_mode: str = "auto", grad_reduce: str = "sum",
                 one_shot_bytes: int = 256 * 1024, use_multimem: bool = True, staleness: int = 0):
        self.svb, self.sfb_mode, self.reduce = svb, sfb_mode, grad_reduce
        # staleness > 0: bounded-staleness (SSP) async SGD on the same arena — per-worker deltas in a ring of s + 1 slots,
        # folded by the peers at most s clocks late (ssp_delta / ssp_fold kernels); no SFB, no sharded history
        self.staleness = int(staleness)
        self.ssp = self.staleness > 0 or os.environ.get("POSEIDON_FUSED_SSP", "0") == "1"
        self.per_worker_state = False
        # buckets up to this size are reduced whole by every rank (one launch latency); larger ones are sharded
        self.one_shot_bytes = int(os.environ.get("POSEIDON_ONE_SHOT_BYTES", one_shot_bytes))
        self.use_multimem = use_multimem and os.environ.get("POSEIDON_MULTIMEM", "1") != "0"
        # SFB reconstruct: optimizer step fused into the outer-product kernel's epilogue (1), or the two-pass form
        # "P-source outer product -> fp32 buffer (bulk row stores), then the streaming update kernel" (0)
        # The two-pass form is the default: the update kernel streams W / H as one linear pass, the epilogue touches them
        # tile by tile.
        self.fuse_sfb_sgd = os.environ.get("POSEIDON_SFB_FUSED_SGD", "0") == "1"
        self.arena: Optional[SymmetricArena] = None
        self.epoch = 0
        self.dense_bytes = 0
        self.sfb_stats = SFBStats()
        self.launches = 0

    # ------------------------------------------------------------------------------ setup
    def setup(self, sync):
        super().setup(sync)
        rc = sync.rank_ctx
        self.device = rc.device
        # Topology.  The NVLink arena spans ONE node: `world` / `rank` below are node-local (they address arena slots and
        # shards); `gworld` is the size of the whole job.  Across nodes every rank first all-reduces its gradient with
        # the ranks of equal local index on the other nodes (library collective over the network), then the node-local
        # kernel reduces over NVLink, steps and broadcasts: sum_r sum_n g[n][r] is the global sum on every node.
        self.gworld, self.grank = rc.world_size, rc.rank
        lw = int(os.environ.get("LOCAL_WORLD_SIZE", self.gworld)) if rc.distributed else 1
        if lw <= 0 or self.gworld % lw:
            lw = self.gworld
        self.nnodes = self.gworld // lw
        self.node, self.cross_group = rc, None
        self.world, self.rank = self.gworld, self.grank
        self.inter_node_bytes = 0
        if self.nnodes > 1:
            if lw == 1:
                raise RuntimeError("the fused NVLink backend needs more than one GPU per node; use --comm nccl")
            node_id = self.grank // lw
            self.world, self.rank = lw, self.grank % lw
            # every rank creates every group, in the same order
            node_groups = [dist.new_group(list(range(n * lw, (n + 1) * lw))) for n in range(self.nnodes)]
            cross_groups = [dist.new_group([n * lw + r for n in range(self.nnodes)]) for r in range(lw)]
            self.node = _NodeContext(self.rank, lw, rc.device, node_groups[node_id], node_id)
            self.cross_group = cross_groups[self.rank]
        self.cu = torch.cuda if self.device.type == "cuda" else _NoCuda
        self.uses_comm_stream = self.world > 1 and self.device.type == "cuda"
        self.stream = self.cu.Stream(device=self.device, priority=-1) if self.world > 1 else None
        self.k = sm100.K()
        net = sync.net
        # engine state for every learnable layer must exist before we re-home weights
        self._ensure_layer_states(net)
        self.sfb_layers: Dict[int, "FusedSFB"] = {}
        self._choose_sfb(net, sync)
        if self.world > 1:
            self._build_arena(net, sync)
        if self.world == 1:
            for layer in net.layers:
                st = getattr(layer, "_sm100", None)
                if isinstance(st, sm100.ConvState) and not st.row_mode and layer.weight.requires_grad:
                    layer._grad_sink = self
        self.multi_update = self.world == 1 and os.environ.get("POSEIDON_MULTI_UPDATE", "1") != "0"
        # (off by default)
        self._early_ip_update = os.environ.get("POSEIDON_EARLY_IP_UPDATE", "0") == "1"
        self._deferred = []
        self.per_worker_state = self.ssp and self.world > 1
        self.done_counter = torch.zeros(4, dtype=torch.int32, device=self.device)
        self.lr_t = torch.zeros(1, dtype=torch.float32, device=self.device)     # global lr, read by the kernels
        self.epoch_t = torch.zeros(1, dtype=torch.int32, device=self.device)    # step counter, read by the comm kernels

    def _ensure_layer_states(self, net):
        for li, layer in enumerate(net.layers):
            if layer.type_name == "CONVOLUTION" and getattr(layer, "_sm100", None) is None:
                cin = net.blob_shapes[net.bottom_names[li][0]][1]
                sm100.conv_state(layer, cin)
            elif layer.type_name == "INNER_PRODUCT" and getattr(layer, "_sm100", None) is None:
                layer._sm100 = sm100.IPState(layer, tuple(net.blob_shapes[net.bottom_names[li][0]]))

    def _choose_sfb(self, net, sync):
        """Per-layer SFB-vs-dense decision.  world==1: every IP weight takes the fused wgrad+update kernel
        (same kernel, one source).  world>1 with --svb: cost model (auto) or every IP layer (all)."""
        P = self.world
        for li, (name, layer) in enumerate(zip(net.layer_names, net.layers)):
            if layer.type_name != "INNER_PRODUCT" or not layer.weight.requires_grad:
                continue
            N, Kd = layer.weight.shape
            M = net.blob_shapes[net.bottom_names[li][0]][0]
            ok_shape = (N % 8 == 0 and Kd % 8 == 0)
            if P == 1:
                use = ok_shape
            elif not self.svb or self.sfb_mode == "none" or self.nnodes > 1 or self.ssp:
                use = False                   # (across nodes the factors would have to travel the network too: dense;
                                              #  under SSP every worker steps on its own gradient: nothing to reconstruct)
            else:
                use = ok_shape and (self.sfb_mode == "all" or sfb_wins(M, N, Kd, P))
            self.sfb_stats.layers[name] = "sfb" if use else "dense"
            if P > 1 and sync.rank_ctx.is_root:
                by = sfb_bytes(M, N, Kd, P, 2)
                log.info("SFB chooser: %s (M=%d N=%d K=%d P=%d) -> %s  [sfb ingress %.1f MB vs dense %.1f MB]",
                         name, M, N, Kd, P, self.sfb_stats.layers[name], by["sfb_ingress"] / 1e6,
                         by["dense_each_way"] * 2 / 1e6)
            if use:
                h = FusedSFB(self, layer, li, M, N, Kd)
                layer.sfb = h
                self.sfb_layers[li] = h
                b = sync.bucket_of.get(id(layer.weight))
                if b is not None:
                    b.mode = "sfb"
                    h.bucket = b
                    h.param_idx = [id(q) for q in b.params].index(id(layer.weight))
                    b.self_updating.add(id(layer.weight))

    def _build_arena(self, net, sync):
        segs: List[_Seg] = []
        total = 0
        n_flag_blocks = len(sync.buckets) + len(self.sfb_layers) + 4
        ring = self.staleness + 1 if self.ssp else 0
        for b in sync.buckets:
            for p in b.params:
                n4 = _round_up(p.numel(), 4)
                total += _round_up(n4 * 4, _ALIGN) * (2 + ring) + _round_up(n4 * 2, _ALIGN)
        for h in self.sfb_layers.values():
            total += h.arena_bytes(self.world)
        total += n_flag_blocks * _ALIGN * 2 + (1 << 20)
        if self.device.type == "cuda":
            self.arena = SymmetricArena(total, self.node)
        else:
            from ..ops.emulate import EmulatedArena          # host shared memory standing in for NVLink peer memory
            self.arena = EmulatedArena(total, self.node)
        ar = self.arena
        self.flag_off = ar.carve(n_flag_blocks * _ALIGN)
        self._next_flag = 0
        self.seg_of: Dict[int, _Seg] = {}
        for b in sync.buckets:
            b.flag_off = self._alloc_flag_block()
            b.segs = []
            for pi, (p, hist) in enumerate(zip(b.params, b.history)):
                s = _Seg()
                s.param, s.numel = p, _round_up(p.numel(), 4)
                s.g_off = ar.carve(s.numel * 4)
                s.w_off = ar.carve(s.numel * 4)
                s.wb_off = ar.carve(s.numel * 2)
                s.hist = hist
                # re-home the fp32 master into the arena, keeping shape/strides
                wflat = ar.view(s.w_off, (s.numel,), torch.float32)
                src = p.data
                if not _is_dense(src):
                    raise RuntimeError("parameters must be dense")
                wflat[: src.numel()].copy_(_storage_order_flat(src))
                p.data = torch.as_strided(wflat, src.shape, src.stride())
                # history must share the master's storage order
                hflat = torch.zeros(s.numel, dtype=torch.float32, device=self.device)
                hflat[: hist.numel()].copy_(_storage_order_flat(hist))
                s.hist = hflat
                b.history[pi] = torch.as_strided(hflat, src.shape, src.stride())
                self.seg_of[id(p)] = s
                b.segs.append(s)
                self._bind_shadow(p, s)
            if self.ssp:
                # delta ring of the bucket: `ring` slots, each holding the bucket's segments back to back
                b.ring_stride = sum(_round_up(sg.numel * 4, _ALIGN) for sg in b.segs)
                base = ar.carve(b.ring_stride * ring)
                off = 0
                for sg in b.segs:
                    sg.d_off = base + off
                    off += _round_up(sg.numel * 4, _ALIGN)
                b.ssp_state = torch.zeros(2 * K_MAX_RANKS + 1, dtype=torch.int32, device=self.device)
        for h in self.sfb_layers.values():
            h.alloc(ar, self._alloc_flag_block())
        for layer in net.layers:
            st = getattr(layer, "_sm100", None)
            if st is not None and not getattr(st, "row_mode", False) and id(layer.weight) in self.seg_of:
                layer._grad_sink = self
        self.cu.synchronize(self.device)
        self.node.barrier()
        self.refresh_shadows()

    def weight_buffer(self, layer, st) -> torch.Tensor:
        """Gradient sink: the layer's wgrad kernel accumulates straight into the symmetric G arena (the segment
        is zeroed by the previous step's all-reduce launch).  One GPU: a persistent per-layer fp32 buffer that the
        update kernel re-arms (zeroes) after reading — no torch.zeros per layer and step."""
        if self.world == 1:
            shape = (st.Coutp, st.Kw) if isinstance(st, sm100.ConvState) else (st.N, st.Kp)
            buf = getattr(st, "_gsink", None)
            if buf is None or tuple(buf.shape) != shape:
                buf = st._gsink = torch.zeros(shape, device=self.device, dtype=torch.float32)
            elif getattr(st, "_gsink_dirty", False):
                buf.zero_()                 # the last hand-out was not consumed by a re-arming update (shared weights, ...)
            st._gsink_dirty = True
            return buf
        seg = self.seg_of[id(layer.weight)]
        shape = (st.Cout, st.Kw) if isinstance(st, sm100.ConvState) else (st.N, st.K)
        return self.arena.view(seg.g_off, (seg.numel,), torch.float32)[: layer.weight.numel()].view(*shape)

    def bias_buffer(self, layer, st) -> Optional[torch.Tensor]:
        """Bias-gradient sink (multi-GPU): the column-sum kernel writes straight into the bias segment of the G arena, so
        the bucket launch has nothing to stage (one copy and its launch per layer and step less)."""
        if self.world == 1 or getattr(layer, "bias", None) is None:
            return None
        seg = self.seg_of.get(id(layer.bias))
        if seg is None:
            return None
        return self.arena.view(seg.g_off, (seg.numel,), torch.float32)[: layer.bias.numel()]

    def _alloc_flag_block(self) -> int:
        off = self.flag_off + self._next_flag * _ALIGN
        self._next_flag += 1
        return off

    def _bind_shadow(self, p, seg):
        """Point the layer's bf16 operand at the arena shadow so the update kernels refresh it in place."""
        layer = self._layer_of(p)
        st = getattr(layer, "_sm100", None)
        if st is None or p is not layer.weight:
            return
        if getattr(st, "row_mode", False):
            return                                  # derived operand (first-layer / channel-padded layouts): refreshed lazily
        shape = (st.Cout, st.Kw) if isinstance(st, sm100.ConvState) else (st.N, st.K)
        st.wb = self.arena.view(seg.wb_off, (seg.numel,), torch.bfloat16)[: p.numel()].view(*shape)
        st.arena_shadow = True

    def _layer_of(self, p):
        b = self.sync.bucket_of[id(p)]
        return b.layer

    def refresh_shadows(self):
        """fp32 master -> bf16 operands for every layer (after init / weight load)."""
        for layer in self.sync.net.layers:
            st = getattr(layer, "_sm100", None)
            if st is None:
                continue
            st.mark_updated()
            if getattr(st, "arena_shadow", False):
                with torch.no_grad():
                    st.wb.copy_(_storage_order_flat(layer.weight.data).view(st.wb.shape))
                st.dirty_wb = False

    # ------------------------------------------------------------------------------ per-bucket launch
    def set_lr(self, lr: float):
        """The global learning rate is a device scalar so that captured CUDA graphs see per-step changes."""
        self.lr_t.fill_(float(lr))

    def _hyper_args(self, lm, dm):
        hy = self.sync.hyper
        ws = self.gworld
        decay = hy.weight_decay * dm * (ws if self.reduce == "sum" else 1.0)
        gscale = 1.0 if self.reduce == "sum" else 1.0 / ws
        # lr here is only the per-blob multiplier; the kernels multiply by lr_t[0]
        return (lm, hy.momentum, decay, hy.solver_type, hy.l1, hy.delta, gscale)

    defers_wgrad_join = True        # ops/sm100.py: convolution weight gradients may still be running on a side stream

    def launch(self, bucket: Bucket):
        st = getattr(bucket.layer, "_sm100", None)
        if self.world == 1:
            if not self.multi_update:
                sm100.wait_pending_wgrad()          # per-tensor updates read the sinks on this stream right now
            fresh = self._launch_local(bucket)
        else:
            self._launch_peer(bucket)
            fresh = False                           # arena shadows are refreshed by the kernels (arena_shadow flag)
        if st is not None:
            # the update kernels already rewrote the bf16 operand next to the fp32 master: do not re-derive it
            st.mark_updated(keep_wb=fresh)

    def _launch_local(self, bucket) -> bool:
        """Steps the bucket's parameters; returns True when the layer's bf16 weight operand is still in sync.
        One GPU has nothing to overlap the update with, so (default) the steps of all buckets are deferred to ONE
        multi-tensor launch at the end of the iteration (`fused_update_multi`, POSEIDON_MULTI_UPDATE=0 restores one
        launch per tensor)."""
        st = getattr(bucket.layer, "_sm100", None)
        fresh = st is not None and not st.dirty_wb
        if self.multi_update:
            for p, h, lm, dm in zip(bucket.params, bucket.history, bucket.lr_mult, bucket.decay_mult):
                if p.grad is None:
                    continue
                wb = None
                if st is not None and p is bucket.layer.weight and st.wb is not None and not getattr(st, "row_mode", False):
                    wb = st.wb
                g = p.grad
                if not _same_order(g, p.data):
                    g = torch.empty_like(p.data).copy_(g)
                lr, mom, decay, rule, l1, delta, gscale = self._hyper_args(lm, dm)
                gs = getattr(st, "_gsink", None) if p is getattr(bucket.layer, "weight", None) else None
                rearm = gs is not None and g.data_ptr() == gs.data_ptr()
                side = getattr(bucket.layer, "_wgrad_side", None) if p is getattr(bucket.layer, "weight", None) else None
                if side is not None and rearm and self._early_ip_update:
                    # inner-product weight whose gradient GEMM was forked to the side stream (ops/sm100.py): its HBM-bound
                    # optimizer step follows on that stream at once and fills the tails of the convolution backward
                    # kernels, instead of running alone at the end of the step.  (The layer's data gradient, which reads
                    # the bf16 operand this step rewrites, completed before the fork.)
                    bucket.layer._wgrad_side = None
                    with self.cu.stream(side):
                        self.k.fused_update(p.data, g, h, wb, lr, mom, decay, rule, l1, delta, gscale, self.lr_t, True)
                        ev = torch.cuda.Event()
                        ev.record(side)
                    sm100.add_pending_wgrad(ev, side.device.index)
                    st._gsink_dirty = False
                    self.launches += 1
                    if p is getattr(bucket.layer, "weight", None):
                        fresh = wb is not None
                    continue
                self._deferred.append((p.data, g, h, wb, lr, decay, rearm, st if rearm else None))
                if p is getattr(bucket.layer, "weight", None):
                    fresh = wb is not None
            return fresh
        for p, h, lm, dm in zip(bucket.params, bucket.history, bucket.lr_mult, bucket.decay_mult):
            if p.grad is None:
                continue                            # weight already stepped inside the fused SFB/wgrad kernel
            wb = None
            if st is not None and p is bucket.layer.weight and st.wb is not None and not getattr(st, "row_mode", False):
                wb = st.wb
            g = p.grad
            if not _same_order(g, p.data):
                g = torch.empty_like(p.data).copy_(g)
            lr, mom, decay, rule, l1, delta, gscale = self._hyper_args(lm, dm)
            gs = getattr(st, "_gsink", None) if p is getattr(bucket.layer, "weight", None) else None
            rearm = gs is not None and g.data_ptr() == gs.data_ptr()      # the persistent sink: leave it zeroed
            self.k.fused_update(p.data, g, h, wb, lr, mom, decay, rule, l1, delta, gscale, self.lr_t, rearm)
            if rearm:
                st._gsink_dirty = False
            self.launches += 1
            if p is getattr(bucket.layer, "weight", None):
                fresh = wb is not None
        return fresh

    def _launch_peer(self, bucket):
        ar = self.arena
        cur = self.cu.current_stream()
        # stage gradients that were not produced directly inside the arena (biases, first-layer weights)
        for p, seg in zip(bucket.params, bucket.segs):
            if p.grad is None:
                continue
            gview = torch.as_strided(ar.view(seg.g_off, (seg.numel,), torch.float32), p.shape, p.data.stride())
            if p.grad.data_ptr() != gview.data_ptr():
                gview.copy_(p.grad)
        self.stream.wait_stream(cur)
        sm100.wait_pending_wgrad(self.stream)       # weight gradients forked to side streams (no-op on the CPU emulation)
        self.epoch_of_bucket = self.epoch + 1
        with self.cu.stream(self.stream):
            live = [(p, seg, lm, dm) for p, seg, lm, dm in zip(bucket.params, bucket.segs, bucket.lr_mult, bucket.decay_mult)
                    if p.grad is not None]
            if live and self.ssp:
                self._launch_ssp(bucket, live)
            elif live:
                use_mc = self.use_multimem and ar.multicast_ptr != 0
                g_offs, w_offs, wb_offs, hists, ns, ones, lrs, decays = [], [], [], [], [], [], [], []
                hy = None
                for p, seg, lm, dm in live:
                    n = seg.numel
                    one_shot = n * 4 <= self.one_shot_bytes
                    lr, mom, decay, rule, l1, delta, gscale = hy = self._hyper_args(lm, dm)
                    if self.cross_group is not None:
                        self._inter_node_reduce(ar.view(seg.g_off, (n,), torch.float32), n, one_shot)
                    g_offs.append(seg.g_off); w_offs.append(seg.w_off); wb_offs.append(seg.wb_off)
                    hists.append(seg.hist); ns.append(n); ones.append(1 if one_shot else 0)
                    lrs.append(lr); decays.append(decay)
                    self.dense_bytes += n * 4
                _, mom, _, rule, l1, delta, gscale = hy
                # ONE launch per bucket (weight + bias behind one barrier pair); the kernel also re-arms (zeroes) the
                # gradient staging it consumed, so no memset launch follows
                self.k.allreduce_sgd_multi(ar.base_ptrs, ar.multicast_ptr if use_mc else 0, ar.peer_ptrs(bucket.flag_off),
                                           g_offs, w_offs, wb_offs, hists, ns, ones, lrs, decays, self.rank, 1,
                                           self.done_counter, mom, rule, l1, delta, gscale, 64, self.lr_t, self.epoch_t)
                self.launches += 1
            if bucket.event is None:
                bucket.event = self.cu.Event()
            bucket.event.record(self.stream)

    def _launch_ssp(self, bucket, live):
        """Bounded staleness on the arena (csrc/comm/fused_update.cu: ssp_delta / ssp_fold): own step now, the peers'
        deltas folded at most `staleness` clocks late, exactly once, read over NVLink from their rings."""
        ar, hy = self.arena, self.sync.hyper
        if self.cross_group is not None:
            raise RuntimeError("fused SSP spans one NVLink node; use --comm ssp across nodes")
        g_offs = [seg.g_off for _, seg, _, _ in live]
        w_offs = [seg.w_off for _, seg, _, _ in live]
        wb_offs = [seg.wb_off for _, seg, _, _ in live]
        d_offs = [seg.d_off for _, seg, _, _ in live]
        ns = [seg.numel for _, seg, _, _ in live]
        hists = [seg.hist for _, seg, _, _ in live]
        lrs = [lm for _, _, lm, _ in live]
        # every worker steps on ITS gradient with the plain decay; the sum of the P deltas is what BSP-sum applies at once
        decays = [hy.weight_decay * dm for _, _, _, dm in live]
        flags = ar.peer_ptrs(bucket.flag_off)
        ring = self.staleness + 1
        self.k.ssp_delta(ar.base_ptrs, flags, g_offs, w_offs, wb_offs, d_offs, bucket.ring_stride, hists, ns, lrs, decays,
                         self.rank, ring, self.staleness, self.done_counter, bucket.ssp_state, hy.momentum, hy.solver_type,
                         hy.l1, hy.delta, 1.0, 0, self.lr_t, self.epoch_t)
        self.k.ssp_fold(ar.base_ptrs, flags, w_offs, wb_offs, d_offs, bucket.ring_stride, ns, self.rank, ring,
                        self.done_counter, bucket.ssp_state, False, 0)
        self.launches += 2
        self.ssp_delta_bytes = getattr(self, "ssp_delta_bytes", 0) + sum(ns) * 4

    def drain(self):
        """Fold every delta that is still in flight (end of training, before a snapshot or a test pass): afterwards all
        replicas hold the same table.  A collective: every rank calls it at the same iteration."""
        if not self.ssp or self.world == 1:
            return
        self.cu.synchronize(self.device)
        self.node.barrier()                        # every rank has published its last clock
        ar = self.arena
        with self.cu.stream(self.stream):
            for b in self.sync.buckets:
                segs = getattr(b, "segs", [])
                if not segs:
                    continue
                self.k.ssp_fold(ar.base_ptrs, ar.peer_ptrs(b.flag_off), [sg.w_off for sg in segs], [sg.wb_off for sg in segs],
                                [sg.d_off for sg in segs], b.ring_stride, [sg.numel for sg in segs], self.rank,
                                self.staleness + 1, self.done_counter, b.ssp_state, True, 0)
        self.cu.synchronize(self.device)
        self.node.barrier()                        # nobody publishes again before everyone has drained

    @property
    def max_observed_lag(self) -> int:
        """Largest number of a peer's clocks that were still unfolded right after a fold was planned (<= staleness)."""
        if not self.ssp:
            return 0
        return max([int(b.ssp_state[2 * K_MAX_RANKS].item()) for b in self.sync.buckets if hasattr(b, "ssp_state")] + [0])

    def _network_all_reduce(self, t: torch.Tensor) -> torch.Tensor:
        """Sum ``t`` over the ranks of equal local index on all nodes; bf16 on the wire if asked for."""
        if getattr(self, "wire_bf16", False):
            wire = t.to(torch.bfloat16)
            dist.all_reduce(wire, group=self.cross_group)
            self.inter_node_bytes += wire.numel() * 2
            return wire.float()
        dist.all_reduce(t, group=self.cross_group)
        self.inter_node_bytes += t.numel() * 4
        return t

    def _inter_node_reduce(self, gseg: torch.Tensor, n: int, one_shot: bool):
        """Multi-node jobs, in front of the node-local kernel (same stream).  Small (one-shot) buckets: all-reduce the
        whole segment across nodes.  Sharded (two-shot) buckets: reduce-scatter inside the node first, so that only
        this rank's shard — 1 / (GPUs per node) of the bucket — crosses the network; the global shard sum is then put
        back into this rank's segment with the rest zeroed, and the unchanged kernel (which sums shard r over the local
        ranks, steps it and broadcasts it) produces the global result."""
        if one_shot:
            gseg.copy_(self._network_all_reduce(gseg))
            return
        W = self.world
        per = ((n // 4 + W - 1) // W) * 4                       # the kernel's shard size (in floats)
        lo = min(n, per * self.rank)
        hi = min(n, lo + per)
        if self.device.type == "cuda":
            buf = torch.zeros(per * W, dtype=torch.float32, device=self.device)
            buf[:n].copy_(gseg)
            shard = torch.empty(per, dtype=torch.float32, device=self.device)
            dist.reduce_scatter_tensor(shard, buf, group=self.node.group)
            shard = shard[: hi - lo]
        else:                                                    # gloo has no reduce-scatter
            full = gseg.clone()
            dist.all_reduce(full, group=self.node.group)
            shard = full[lo:hi].clone()
        if hi > lo:
            shard = self._network_all_reduce(shard)
        gseg.zero_()
        gseg[lo:hi].copy_(shard)

    def _flush_deferred(self):
        if not self._deferred:
            return
        hy = self.sync.hyper
        d = self._deferred
        self._deferred = []
        empty = torch.empty(0, dtype=torch.bfloat16, device=self.device)
        self.k.fused_update_multi([e[0] for e in d], [e[1] for e in d], [e[2] for e in d],
                                  [e[3] if e[3] is not None else empty for e in d], [e[4] for e in d], [e[5] for e in d],
                                  [1 if e[6] else 0 for e in d], hy.momentum, hy.solver_type, hy.l1, hy.delta,
                                  1.0 if self.reduce == "sum" else 1.0 / self.gworld, self.lr_t)
        for e in d:
            if e[7] is not None:
                e[7]._gsink_dirty = False
        self.launches += (len(d) + 47) // 48

    def finish_iteration(self):
        """Close the step: the device-resident epoch counter (read by every comm kernel of this step as
        ``epoch_t + 1``) is bumped on the comm stream, i.e. after all of them in stream order.  Keeping it on the
        device is what lets a captured CUDA graph of the whole step be replayed."""
        self.epoch += 1
        sm100.wait_pending_wgrad(clear=True)        # every side stream joins the caller's stream (capture-safe)
        if self.world == 1:
            self._flush_deferred()
        if self.world > 1:
            cur = self.cu.current_stream()
            self.stream.wait_stream(cur)
            with self.cu.stream(self.stream):
                self.epoch_t.add_(1)
            if self.cu.is_current_stream_capturing():
                cur.wait_stream(self.stream)           # a capture must end with every forked stream joined

    def close(self):
        """Release host-side resources of the arena (the emulated shared-memory segments; the CUDA arena lives as long
        as its tensors)."""
        ar = self.arena
        if ar is not None and hasattr(ar, "close"):
            self.arena = None
            ar.close()

    def comm_profile(self) -> Dict:
        """Static description of one step's communication (valid under CUDA-graph replay, where the Python-side byte
        counters stand still): per rank, bytes of dense gradients entering the in-kernel all-reduce, bytes of sufficient
        factors published, and the dense bytes those SFB layers would have cost; plus which NVLink path the kernels use."""
        dense = sfb = sfb_equiv = 0
        if self.world > 1:
            for b in self.sync.buckets:
                for p, seg in zip(b.params, getattr(b, "segs", [])):
                    if id(p) in b.self_updating:
                        continue
                    dense += seg.numel * 4
            for h in self.sfb_layers.values():
                sfb += h.M * (h.N + h.K) * 2
                sfb_equiv += h.N * h.K * 4
        mc = bool(self.arena is not None and getattr(self.arena, "multicast_ptr", 0) and self.use_multimem)
        return {"dense_allreduce_bytes_per_step": dense, "sfb_factor_bytes_per_step": sfb,
                "sfb_dense_equiv_bytes_per_step": sfb_equiv, "multimem": mc,
                "nvlink_path": ("nvls_multicast" if mc else "p2p") if self.world > 1 else "none"}

    def bytes_on_wire(self):
        return {"dense_allreduce_bytes": self.dense_bytes, "inter_node_allreduce_bytes": self.inter_node_bytes,
                "ssp_delta_bytes": getattr(self, "ssp_delta_bytes", 0), "sfb_bytes": self.sfb_stats.sfb_bytes,
                "sfb_dense_equiv_bytes": self.sfb_stats.dense_equiv_bytes}

    # optimizer-state plumbing for snapshots: history of a two-shot bucket is sharded by rank
    def gather_history(self):
        if self.world == 1 or self.ssp:            # SSP: momentum is per worker and never sharded
            return
        for b in self.sync.buckets:
            for seg in getattr(b, "segs", []):
                n = seg.numel
                if n * 4 <= self.one_shot_bytes:
                    continue
                per = ((n // 4 + self.world - 1) // self.world) * 4
                padded = torch.zeros(per * self.world, dtype=torch.float32, device=self.device)
                lo = min(n, per * self.rank)
                hi = min(n, lo + per)
                mine = torch.zeros(per, dtype=torch.float32, device=self.device)
                mine[: hi - lo] = seg.hist[lo:hi]
                dist.all_gather_into_tensor(padded, mine, group=getattr(self.node, "group", None))
                seg.hist.copy_(padded[:n])


def _is_dense(t: torch.Tensor) -> bool:
    """Non-overlapping and dense: some permutation of the dims is contiguous."""
    dims = sorted((st, n) for n, st in zip(t.shape, t.stride()) if n > 1)
    expect = 1
    for st, n in dims:
        if st != expect:
            return False
        expect *= n
    return True


def _same_order(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.shape == b.shape and all(sa == sb for n, sa, sb in zip(a.shape, a.stride(), b.stride()) if n > 1)


def _storage_order_flat(t: torch.Tensor) -> torch.Tensor:
    """1-D view of a dense tensor in storage order."""
    return t.as_strided((t.numel(),), (1,))


class FusedSFB:
    """Per-layer sufficient-factor exchange + fused outer-product/optimizer kernel.

    Staging layout inside every rank's arena (single-buffered; a rank may only overwrite a peer's slot after that peer
    raised its *consumed* flag for the previous step):  U[P][M][N], V[P][M][K] bf16.  Rank r
    *pushes* its factors into slot r of every rank (one NVSwitch-multicast store stream, or P2P stores),
    raises its epoch flag on every peer, and the wgmma kernel walks the P slots as P reduction sources,
    waiting on slot p's flag right before its first TMA load of that slot — so the outer product of the
    factors that have already landed overlaps the arrival of the rest.  All ranks reduce in the same slot
    order, so replicas stay bit-identical."""

    def __init__(self, backend: FusedBackend, layer, layer_idx, M, N, Kd):
        self.be, self.layer, self.layer_idx = backend, layer, layer_idx
        self.M, self.N, self.K = M, N, Kd
        self.bucket = None
        self.param_idx = 0
        self.u_off = self.v_off = None
        self.flag_off = None
        self.local_flags = None
        self.event = None

    def arena_bytes(self, world):
        return 2 * world * (_round_up(self.M * self.N * 2, _ALIGN) + _round_up(self.M * self.K * 2, _ALIGN))

    def alloc(self, arena: SymmetricArena, flag_off: int):
        P = arena.world
        self.u_slot = _round_up(self.M * self.N * 2, _ALIGN)
        self.v_slot = _round_up(self.M * self.K * 2, _ALIGN)
        self.u_off = [arena.carve(P * self.u_slot) for _ in range(2)]
        self.v_off = [arena.carve(P * self.v_slot) for _ in range(2)]
        self.flag_off = flag_off
        # flag block: [slot][rank] u32; slots 2/3 = SFB parity 0/1 (slots 0/1 belong to the all-reduce barriers)
        self.local_flags = [arena.view(flag_off + (2 + par) * K_MAX_RANKS * 4, (K_MAX_RANKS,), torch.int32)
                            for par in range(2)]

    def exchange_and_update(self, layer, dy: torch.Tensor, x2: torch.Tensor):
        """Called from the IP backward with u = dY [M,N] and v = X [M,K] (bf16).  Steps W, H and the bf16
        shadow in place; returns None (no dense gradient exists, locally or on the wire)."""
        be = self.be
        k = be.k
        b = self.bucket
        st = layer._sm100
        lm, dm = b.lr_mult[self.param_idx], b.decay_mult[self.param_idx]
        lr, mom, decay, rule, l1, delta, gscale = be._hyper_args(lm, dm)
        w = layer.weight.data
        h = b.history[self.param_idx]
        if st.wb is None or st.dirty_wb:
            st.shadow()
        dy = dy.contiguous()
        x2 = x2.contiguous()
        M = dy.shape[0]
        if be.world == 1:
            if getattr(be, "fuse_local_sgd", False):
                k.sfb_outer_sgd([dy.data_ptr()], [x2.data_ptr()], M, self.N, self.K, w, h, st.wb, gscale, lr, mom, decay,
                                rule, l1, delta, None, 0, 0, 0, 0, be.lr_t)
                be.launches += 1
            else:
                # Single GPU: the optimizer epilogue has only the 8 epilogue warps' loads in flight (64 KB/SM) and
                # measured 2.4 TB/s, while the wgrad GEMM -> fp32 buffer followed by the streaming update kernel
                # runs at 5.3 TB/s: 213 us vs 279 us for fc6 (benchmarks/sgd_bench.py).  Use the faster pair.
                g = getattr(self, "_gbuf", None)
                if g is None:
                    g = self._gbuf = torch.empty(self.N, self.K, device=w.device, dtype=torch.float32)
                k.gemm_f32(dy, True, x2, True, g, 1.0, False, 1, 0)
                k.fused_update(w, g, h, st.wb, lr, mom, decay, rule, l1, delta, gscale, be.lr_t)
                be.launches += 2
            st.mark_updated(keep_wb=True)
            be.sfb_stats.dense_equiv_bytes += self.N * self.K * 4
            return None
        ar = be.arena
        P = be.world
        par = 0                      # single-buffered slots: peers acknowledge consumption on flag slot 4
        cur = be.cu.current_stream()
        be.stream.wait_stream(cur)
        with be.cu.stream(be.stream):
            _record_stream(dy, be.stream)
            _record_stream(x2, be.stream)
            mc = be.use_multimem and ar.multicast_ptr != 0
            u_dst = self.u_off[par] + be.rank * self.u_slot
            v_dst = self.v_off[par] + be.rank * self.v_slot
            flags = ar.peer_ptrs(self.flag_off)
            k.peer_push(dy, ar.peer_ptrs(u_dst), ar.mc_ptr(u_dst) if mc else 0, flags, be.rank,
                        2 + par, 1, False, be.done_counter[1:2], 4, be.epoch_t)
            k.peer_push(x2, ar.peer_ptrs(v_dst), ar.mc_ptr(v_dst) if mc else 0, flags, be.rank,
                        2 + par, 1, True, be.done_counter[1:2], -1, be.epoch_t)
            base = ar.base_ptrs[be.rank]
            u_ptrs = [base + self.u_off[par] + p * self.u_slot for p in range(P)]
            v_ptrs = [base + self.v_off[par] + p * self.v_slot for p in range(P)]
            if getattr(be, "fuse_sfb_sgd", True):
                k.sfb_outer_sgd(u_ptrs, v_ptrs, M, self.N, self.K, w, h, st.wb, gscale, lr, mom, decay, rule, l1, delta,
                                self.local_flags[par], 1, 0, 0, 0, be.lr_t, be.epoch_t)
                be.launches += 4
            else:
                # two-pass variant: P-source outer product into a local fp32 buffer + streaming update (measured
                # slower than the fused epilogue when it shares the GPU with the backward pass: 129 k vs 132 k img/s)
                g = getattr(self, "_gbuf", None)
                if g is None:
                    g = self._gbuf = torch.empty(self.N, self.K, device=w.device, dtype=torch.float32)
                _record_stream(g, be.stream)
                k.sfb_outer_f32(u_ptrs, v_ptrs, M, self.N, self.K, g, 1.0, self.local_flags[par], 1, 0, 0, 0, be.epoch_t)
                k.fused_update(w, g, h, st.wb, lr, mom, decay, rule, l1, delta, gscale, be.lr_t)
                be.launches += 5
            k.peer_signal(flags, be.rank, 4, 1, be.epoch_t)      # "I have consumed every slot of this step"
            if self.event is None:
                self.event = be.cu.Event()
            self.event.record(be.stream)
        st.mark_updated(keep_wb=True)
        be.sfb_stats.sfb_bytes += M * (self.N + self.K) * 2
        be.sfb_stats.dense_equiv_bytes += self.N * self.K * 4
        self.bucket.sfb_event = self.event      # the layer's next forward also waits for this kernel
        return None
