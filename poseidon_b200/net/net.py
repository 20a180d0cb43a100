"""Net: builds an executable layer graph from a Caffe ``NetParameter``.

Differences from the reference's design (deliberate — this is not a port):
  * blobs are plain ``torch.Tensor``s flowing through a name→tensor dict; fan-out needs no
    Split layers (autograd accumulates), in-place layers simply rebind the name;
  * backward is autograd, so "layer i's Backward finished" events — the trigger points of
    distributed wait-free backprop — are per-parameter post-accumulate-grad hooks;
  * learnable blobs are fp32 ``nn.Parameter``s that the parallel engine re-homes into one
    flat symmetric-memory arena (the PS-table replacement).

reference: src/caffe/net.cpp:39-249 (Init), :366-468 (FilterNet/StateMeetsRule), :473-615
(AppendTop/Bottom/Param), :709-784 (Forward/Backward), :855-950 (Share/CopyTrainedLayers),
:953-971 (ToProto).
"""
from __future__ import annotations

import logging
from collections import OrderedDict
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn as nn

from .. import proto as P
from ..layers import NetContext, create_layer

log = logging.getLogger("poseidon_b200")


def state_meets_rule(state, rule, layer_name: str) -> bool:
    """reference: src/caffe/net.cpp:410-468."""
    if rule.has("phase") and rule.phase != state.phase:
        return False
    if rule.has("min_level") and state.level < rule.min_level:
        return False
    if rule.has("max_level") and state.level > rule.max_level:
        return False
    stages = set(state.stage)
    for s in rule.stage:
        if s not in stages:
            return False
    for s in rule.not_stage:
        if s in stages:
            return False
    return True


def filter_net(param, state=None):
    """Drop layers whose include/exclude rules do not match the net state.
    reference: src/caffe/net.cpp:366-407."""
    state = state if state is not None else param.state
    out = param.copy()
    out.clear("layers")
    for lp in param.layers:
        if len(lp.include) and len(lp.exclude):
            raise ValueError(f"layer {lp.name}: specify either include rules or exclude rules; not both.")
        included = len(lp.include) == 0
        for r in lp.exclude:
            if included and state_meets_rule(state, r, lp.name):
                included = False
        for r in lp.include:
            if not included and state_meets_rule(state, r, lp.name):
                included = True
        if included:
            out.layers.append(lp.copy())
    return out


class Net(nn.Module):
    def __init__(self, param, phase: Optional[int] = None, ctx: Optional[NetContext] = None,
                 level: int = 0, stages: Optional[List[str]] = None):
        super().__init__()
        if isinstance(param, str):
            import os
            model_dir = os.path.dirname(os.path.abspath(param))
            param = P.read_net(param)
        else:
            model_dir = None
        self.ctx = ctx if ctx is not None else NetContext()
        if model_dir and self.ctx.model_dir is None:
            self.ctx.model_dir = model_dir
        state = param.state.copy() if param.has("state") else P.NetState()
        if phase is not None:
            state.phase = phase
        elif not param.has("state"):
            state.phase = self.ctx.phase
        if level:
            state.level = level
        if stages:
            state.stage = list(stages)
        self.state = state
        self.ctx.phase = state.phase
        self.phase = state.phase
        self.param_def = filter_net(param, state)
        self.name = self.param_def.name or ""
        self._build()

    # ------------------------------------------------------------------------------------
    def _build(self):
        pd = self.param_def
        self.layers = nn.ModuleList()
        self.layer_names: List[str] = []
        self.bottom_names: List[List[str]] = []
        self.top_names: List[List[str]] = []
        self.blob_shapes: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
        self.loss_weights: List[List[float]] = []
        available = set()
        # net-level inputs
        self.input_names = list(pd.input)
        dims = list(pd.input_dim)
        if len(dims) != 4 * len(self.input_names):
            raise ValueError("Incorrect input blob dimension specifications.")
        for i, name in enumerate(self.input_names):
            self.blob_shapes[name] = tuple(dims[4 * i:4 * i + 4])
            available.add(name)
        consumed = set()
        # param bookkeeping
        self.params: List[nn.Parameter] = []
        self.params_lr: List[float] = []
        self.params_weight_decay: List[float] = []
        self.param_display_names: List[str] = []
        self.param_layer_idx: List[int] = []
        self.param_is_owner: List[bool] = []
        self.param_owner: List[tuple] = []     # (layer, blob index) owning each entry of self.params
        named: Dict[str, int] = {}
        for li, lp in enumerate(pd.layers):
            layer = create_layer(lp, self.ctx)
            bnames, tnames = list(lp.bottom), list(lp.top)
            layer.n_bottoms, layer.n_tops = len(bnames), len(tnames)
            layer.check_blob_counts(len(bnames), len(tnames))
            for b in bnames:
                if b not in available:
                    raise ValueError(f"Unknown blob input {b} (at index {bnames.index(b)}) to layer {lp.name}")
                consumed.add(b)
            bshapes = [self.blob_shapes[b] for b in bnames]
            tshapes = layer.setup(bshapes)[: len(tnames)]
            if len(tshapes) < len(tnames):
                raise ValueError(f"layer {lp.name} declares {len(tnames)} tops but produces {len(tshapes)}")
            for t, s in zip(tnames, tshapes):
                if t in available and t not in bnames:
                    raise ValueError(f"Duplicate blobs produced by multiple sources: {t}")
                self.blob_shapes[t] = tuple(s)
                available.add(t)
            # loss weights (default 1 on the first top of loss layers)
            lw = [float(x) for x in lp.loss_weight]
            if lw and len(lw) != len(tnames):
                raise ValueError(f"loss_weight must be unspecified or specified once per top blob (layer {lp.name})")
            if not lw:
                lw = [1.0 if (layer.is_loss and i == 0) else 0.0 for i in range(len(tnames))]
            self.loss_weights.append(lw)
            # params: lr / decay multipliers and sharing by name
            nb = len(layer.blobs)
            lrs = [float(x) for x in lp.blobs_lr]
            wds = [float(x) for x in lp.weight_decay]
            if lrs and len(lrs) != nb:
                raise ValueError(f"layer {lp.name}: blobs_lr count must match number of blobs")
            if wds and len(wds) != nb:
                raise ValueError(f"layer {lp.name}: weight_decay count must match number of blobs")
            pnames = list(lp.param)
            if pnames and len(pnames) != nb:
                raise ValueError(f"layer {lp.name}: param names must match number of blobs")
            for j in range(nb):
                pname = pnames[j] if pnames else ""
                attr = layer.blob_names[j]
                p = getattr(layer, attr)
                lr = lrs[j] if lrs else 1.0
                wd = wds[j] if wds else 1.0
                if pname and pname in named:
                    owner = self.params[named[pname]]
                    strict = not (len(lp.blob_share_mode) > j and lp.blob_share_mode[j] == 1)
                    if strict and tuple(owner.shape) != tuple(p.shape):
                        raise ValueError(f"Shared parameter blobs must have the same shape ({pname})")
                    if owner.numel() != p.numel():
                        raise ValueError(f"Shared parameter blobs must have the same count ({pname})")
                    setattr(layer, attr, owner)
                    continue
                if lr == 0.0:
                    p.requires_grad_(False)
                idx = len(self.params)
                self.param_owner.append((layer, j))
                self.params.append(p)
                self.params_lr.append(lr)
                self.params_weight_decay.append(wd)
                self.param_display_names.append(pname or f"{lp.name}.{attr}")
                self.param_layer_idx.append(li)
                if pname:
                    named[pname] = idx
            self.layers.append(layer)
            self.layer_names.append(lp.name or f"layer{li}")
            self.bottom_names.append(bnames)
            self.top_names.append(tnames)
        # outputs = produced but never consumed, in production order
        produced = []
        for tn in self.top_names:
            for t in tn:
                if t not in produced:
                    produced.append(t)
        used = set(b for bn in self.bottom_names for b in bn)
        # an in-place top is still "consumed" only by its own layer
        self.output_names = [t for t in produced if not self._consumed_later(t)]
        del used
        self.layer_by_name = {n: l for n, l in zip(self.layer_names, self.layers)}
        self.blobs: Dict[str, torch.Tensor] = {}
        self.force_backward = bool(pd.force_backward)
        self._plan_backward()
        self._loss = None
        self.debug_info = False
        self.skip_layer = [False] * len(self.layers)
        if self.ctx.engine == "sm100":
            from ..ops import sm100
            if sm100.active(self.ctx.device):
                from .fusion import plan_sm100
                plan_sm100(self)
        from .lanes import default_lanes, plan_lanes
        plan_lanes(self, default_lanes(self.ctx))

    def _plan_backward(self):
        """``blob_need_backward``: which blobs get a diff, by the reference's rules (src/caffe/net.cpp:80-220).  A layer
        needs backward when it has a parameter with a non-zero learning rate (every parameter counts when blobs_lr is
        not given) or a bottom that needs backward; then all its tops do.  force_backward then marks every bottom a
        layer allows (Layer.allow_force_backward: not a loss layer's label).  Net inputs and data-layer tops that end up
        needing backward, labels excepted, become autograd leaves in forward() (only with force_backward)."""
        need: Dict[str, bool] = {n: False for n in self.input_names}
        for li, (lp, layer) in enumerate(zip(self.param_def.layers, self.layers)):
            bnames = self.bottom_names[li]
            lrs = [float(x) for x in lp.blobs_lr]
            layer_needs = any(need[b] for b in bnames) or (any(lr > 0 for lr in lrs) if lrs else bool(layer.blob_names))
            for t in self.top_names[li]:
                need[t] = layer_needs or (t in bnames and need[t])      # an in-place top keeps its own flag
        if self.force_backward:
            for li, layer in enumerate(self.layers):
                for j, b in enumerate(self.bottom_names[li]):
                    if layer.allow_force_backward(j):
                        need[b] = True
        self.blob_need_backward: Dict[str, bool] = need
        leaves = []
        if self.force_backward:
            leaves = [n for n in self.input_names if need[n]]
            for li, layer in enumerate(self.layers):
                if getattr(layer, "is_data", False):
                    leaves += [t for j, t in enumerate(self.top_names[li]) if need[t] and j not in layer.label_tops]
        self._grad_leaves = set(leaves)

    @staticmethod
    def _leaf(t: torch.Tensor) -> torch.Tensor:
        return t.detach().requires_grad_(True) if t.is_floating_point() else t

    def _data_outs(self, i: int, outs):
        """A data layer's tops, the ones force_backward wants a diff of as autograd leaves."""
        if not self._grad_leaves or not getattr(self.layers[i], "is_data", False):
            return outs
        return tuple(self._leaf(o) if t in self._grad_leaves else o for t, o in zip(self.top_names[i], outs))

    def _consumed_later(self, blob: str) -> bool:
        last_prod = max(i for i, tn in enumerate(self.top_names) if blob in tn)
        for i in range(last_prod + 1, len(self.layers)):
            if blob in self.bottom_names[i]:
                return True
        return False

    # ------------------------------------------------------------------------------------
    def forward(self, inputs: Optional[Dict[str, torch.Tensor]] = None, start: int = 0,
                end: Optional[int] = None, keep_blobs: bool = True):
        """Run layers [start, end]; returns (loss, {output blob name: tensor}).
        reference: src/caffe/net.cpp:709-750 (ForwardFromTo / ForwardPrefilled)."""
        blobs = dict(self.blobs) if (start > 0 and self.blobs) else {}
        if inputs:
            blobs.update(inputs)
        for n in self.input_names:
            if n not in blobs:
                raise ValueError(f"missing net input '{n}'")
        for n in self._grad_leaves:           # (force_backward) every pass starts from fresh leaves
            if n in blobs:
                blobs[n] = self._leaf(blobs[n])
        end = len(self.layers) - 1 if end is None else end
        loss = None
        lanes = self._lane_runner(start, end)
        if lanes is not None:
            loss = self._forward_lanes(lanes, blobs, start, end)
            start = end + 1
        for i in range(start, end + 1):
            if self.skip_layer[i]:
                continue                      # fused into the producer's epilogue (in-place layer: blob unchanged)
            layer = self.layers[i]
            ins = [blobs[b] for b in self.bottom_names[i]]
            outs = self._data_outs(i, layer(*ins))
            for t, o, w in zip(self.top_names[i], outs, self.loss_weights[i]):
                blobs[t] = o
                if w != 0.0:
                    term = o.float().sum() * w if o.numel() > 1 else o.float().reshape(()) * w
                    loss = term if loss is None else loss + term
            if self.debug_info:
                self._forward_debug(i, outs)
        self.blobs = blobs if keep_blobs else {}
        self._loss = loss if keep_blobs else None
        outputs = {n: blobs[n] for n in self.output_names if n in blobs}
        return loss, outputs

    def _forward_lanes(self, lanes, blobs, start: int, end: int):
        """Branch-parallel pass (net/lanes.py): every layer runs on its lane's stream, which first waits for bottoms
        produced on other lanes; loss terms are summed on the caller's stream after all lanes have joined it."""
        terms = []
        cur_lane = 0
        try:
            for i in range(start, end + 1):
                if self.skip_layer[i]:
                    continue
                lane = self.lane[i]
                if lane != cur_lane:          # (switching only on a change: the context manager costs ~10 us per layer)
                    torch.cuda.set_stream(lanes.streams[lane])
                    cur_lane = lane
                lanes.before(i)
                outs = self._data_outs(i, self.layers[i](*[blobs[b] for b in self.bottom_names[i]]))
                for t, o, w in zip(self.top_names[i], outs, self.loss_weights[i]):
                    blobs[t] = o
                    if w != 0.0:
                        terms.append((o.float().sum() * w if o.numel() > 1 else o.float().reshape(()) * w, lane))
                lanes.after(i, outs)
        finally:
            torch.cuda.set_stream(lanes.cur)
        lanes.finish()                        # every lane has joined the caller's stream
        loss = None
        for term, lane in terms:
            if lane != 0:
                term.record_stream(lanes.cur)
            loss = term if loss is None else loss + term
        return loss

    def _lane_runner(self, start: int, end: int):
        """Stream bookkeeping of a branch-parallel pass, or None (CPU nets, single-lane plans, passes that stop early)."""
        if getattr(self, "n_lanes", 1) <= 1 or self.debug_info or end != len(self.layers) - 1:
            return None
        if self.ctx.device is None or torch.device(self.ctx.device).type != "cuda":
            return None
        r = getattr(self, "_lanes", None)
        if r is None:
            from .lanes import LaneRunner
            r = self._lanes = LaneRunner(self)
        r.begin(start)
        return r

    def _forward_debug(self, i, outs):
        """reference: src/caffe/net.cpp:787-812 (ForwardDebugInfo: mean |x| per top/param)."""
        for t, o in zip(self.top_names[i], outs):
            log.info("    [Forward] Layer %s, top blob %s data: %g", self.layer_names[i], t,
                     float(o.detach().float().abs().mean()))
        for j, p in enumerate(self.layers[i].blobs):
            log.info("    [Forward] Layer %s, param blob %d data: %g", self.layer_names[i], j,
                     float(p.detach().abs().mean()))

    def backward_debug(self):
        """reference: src/caffe/net.cpp:814-852 (BackwardDebugInfo / UpdateDebugInfo)."""
        for i, layer in enumerate(self.layers):
            for j, p in enumerate(layer.blobs):
                if p.grad is not None:
                    log.info("    [Backward] Layer %s, param blob %d diff: %g", self.layer_names[i], j,
                             float(p.grad.abs().mean()))

    def forward_backward(self, inputs=None):
        loss, outputs = self.forward(inputs)
        if loss is not None and loss.requires_grad:
            loss.backward()
            if self.ctx.engine == "sm100":
                from ..ops import sm100
                sm100.wait_pending_wgrad(clear=True)     # weight gradients forked to side streams join here
        return loss, outputs

    def backward(self, top_diffs: Optional[Dict[str, torch.Tensor]] = None) -> Dict[str, torch.Tensor]:
        """Backpropagate through the last forward pass: from ``top_diffs`` (blob name -> diff of that blob) when given,
        else from the loss.  Parameter gradients accumulate into ``p.grad`` as in forward_backward().  Returns the diff
        of every net input and data-layer top that needs backward (``blob_need_backward``; with force_backward off,
        none), as float32 in the blob's logical NCHW shape whatever layout the engine ran it in.
        reference: src/caffe/net.cpp:752-784 (Backward), python/caffe/pycaffe.py (net.backward(**diffs))."""
        if not self.blobs:
            raise RuntimeError("Net.backward() needs a forward pass that kept its blobs")
        roots, seeds = [], []
        for name, g in (top_diffs or {}).items():
            t = self.blobs.get(name)
            if t is None:
                raise ValueError(f"'{name}' is not a blob of the last forward pass")
            g = torch.as_tensor(g)
            shapes = (tuple(t.shape), tuple(self.blob_shapes.get(name, t.shape)))
            if tuple(g.shape) not in shapes or g.numel() != t.numel():
                raise ValueError(f"diff for '{name}' has shape {tuple(g.shape)}; the blob has shape {shapes[1]}")
            if t.requires_grad:
                roots.append(t)
                seeds.append(g.detach().to(device=t.device, dtype=t.dtype).reshape(t.shape))
        if not top_diffs and self._loss is not None and self._loss.requires_grad:
            roots.append(self._loss)
            seeds.append(torch.ones_like(self._loss))
        leaves = {n: self.blobs[n] for n in sorted(self._grad_leaves) if n in self.blobs and self.blobs[n].requires_grad}
        for t in leaves.values():
            t.grad = None
        if roots:
            torch.autograd.backward(roots, seeds)
            if self.ctx.engine == "sm100":
                from ..ops import sm100
                sm100.wait_pending_wgrad(clear=True)     # weight gradients forked to side streams join here
        return {n: self._logical_diff(n, t) for n, t in leaves.items()}

    def _logical_diff(self, name: str, leaf: torch.Tensor) -> torch.Tensor:
        """The diff of a net input / data-layer top as float32 in the blob's logical shape.  On the sm100 engine a data
        layer may have handed its first convolution the physical s2d / ROW / 8-channel layout: first_layer_diff maps
        that convolution's data gradient back."""
        g = leaf.grad
        logical = tuple(self.blob_shapes[name]) if name not in self.input_names else tuple(leaf.shape)
        if g is None:
            return torch.zeros(logical, dtype=torch.float32, device=leaf.device)
        if tuple(g.shape) == logical:
            return g.detach().float()
        conv = None
        for i, layer in enumerate(self.layers):
            if getattr(layer, "is_data", False) and self.top_names[i][:1] == [name]:
                conv = getattr(layer, "first_conv", None)
        if conv is None:
            raise RuntimeError(f"blob '{name}': diff of shape {tuple(g.shape)} for a blob of shape {logical}")
        from ..ops import sm100
        return sm100.first_layer_diff(g.detach(), conv, logical, True)

    def zero_grad_(self):
        for p in self.params:
            p.grad = None

    def data_layers(self):
        return [l for l in self.layers if getattr(l, "is_data", False)]

    def num_leading_data_layers(self) -> int:
        n = 0
        for l in self.layers:
            if not getattr(l, "is_data", False):
                break
            n += 1
        return n

    def forward_data(self) -> Dict[str, torch.Tensor]:
        """Run only the leading data layers; returns their top blobs."""
        out = {}
        for i in range(self.num_leading_data_layers()):
            for t, o in zip(self.top_names[i], self.layers[i]()):
                out[t] = o
        return out

    def close(self):
        for l in self.layers:
            if hasattr(l, "close"):
                l.close()

    # ---- weights in / out -------------------------------------------------------------------
    def share_trained_layers_with(self, other: "Net"):
        """Test nets alias the train net's parameters (no copy).
        reference: src/caffe/net.cpp:855-883."""
        for name, layer in zip(self.layer_names, self.layers):
            src = other.layer_by_name.get(name)
            if src is None or not layer.blob_names:
                continue
            if len(src.blob_names) != len(layer.blob_names):
                raise ValueError(f"Incompatible number of blobs for layer {name}")
            for a_dst, a_src in zip(layer.blob_names, src.blob_names):
                ps, pd_ = getattr(src, a_src), getattr(layer, a_dst)
                if ps.numel() != pd_.numel():
                    raise ValueError(f"Cannot share layer {name}: shape mismatch")
                setattr(layer, a_dst, ps)
            if getattr(src, "_sm100", None) is not None:
                layer._sm100 = src._sm100            # one set of bf16 operands per weight
                if hasattr(src, "_k_perm"):
                    layer._k_perm = src._k_perm
        self._reindex_params()

    def _reindex_params(self):
        seen, out = {}, []
        for li, layer in enumerate(self.layers):
            for a in layer.blob_names:
                p = getattr(layer, a)
                if id(p) not in seen:
                    seen[id(p)] = True
                    out.append(p)
        self.params = out

    def copy_trained_layers_from(self, src) -> List[str]:
        """Load weights by layer name from a NetParameter or a .caffemodel path.
        reference: src/caffe/net.cpp:908-950 (shape-checked, unknown layers ignored)."""
        if isinstance(src, str):
            src = P.read_net(src)
        loaded = []
        for slp in src.layers:
            layer = self.layer_by_name.get(slp.name)
            if layer is None:
                log.info("Ignoring source layer %s", slp.name)
                continue
            if not len(slp.blobs):
                continue
            if len(slp.blobs) != len(layer.blobs):
                raise ValueError(f"Incompatible number of blobs for layer {slp.name}")
            for j, (blob, p) in enumerate(zip(slp.blobs, layer.blobs)):
                want = layer.caffe_blob_shape(j)
                got = (blob.num, blob.channels, blob.height, blob.width)
                if got != want:
                    raise ValueError(f"layer {slp.name} blob {j}: shape mismatch {got} vs {want}")
                layer.import_blob(j, np.asarray(blob.data, dtype=np.float32))
            st = getattr(layer, "_sm100", None)
            if st is not None:
                st.mark_updated()
            loaded.append(slp.name)
        return loaded

    def to_proto(self, write_diff: bool = False):
        """NetParameter with every layer's current blobs. reference: src/caffe/net.cpp:953-971,
        layer.hpp:571-578, blob.cpp:429-448."""
        out = P.NetParameter()
        if self.name:
            out.name = self.name
        out.input = list(self.param_def.input)
        out.input_dim = list(self.param_def.input_dim)
        for lp, layer in zip(self.param_def.layers, self.layers):
            nl = lp.copy()
            nl.clear("blobs")
            for j, p in enumerate(layer.blobs):
                diff = layer.export_blob(j, p.grad) if (write_diff and p.grad is not None) else None
                nl.blobs.append(P.array_to_blob(layer.export_blob(j), diff=diff))
            out.layers.append(nl)
        return out

    def num_params(self) -> int:
        return sum(p.numel() for p in self.params)
