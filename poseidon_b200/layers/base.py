"""Layer base class, registry and fillers.

A layer is a ``torch.nn.Module`` built from a Caffe ``LayerParameter``.  ``setup`` receives
the bottom shapes (NCHW tuples), creates parameters and returns the top shapes;
``forward`` maps bottom tensors to a tuple of top tensors.  Backward is autograd (custom
CUDA ops are ``torch.autograd.Function``s), which is what lets the solver hang the
DWBP communication off per-parameter gradient hooks.

reference: include/caffe/layer.hpp:61-168 (SetUp/Reshape/Forward/Backward contract),
src/caffe/layer_factory.cpp:177-261 (type -> class switch), include/caffe/filler.hpp.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from .. import proto as P

Shape = Tuple[int, ...]
LAYER_REGISTRY: Dict[str, type] = {}


def register(*type_names):
    def deco(cls):
        for t in type_names:
            LAYER_REGISTRY[t] = cls
        cls.type_names = type_names
        return cls
    return deco


class NetContext:
    """Everything a layer may need to know about where it runs."""

    def __init__(self, phase=P.TRAIN, device="cpu", engine="torch", dtype=torch.float32,
                 rank=0, world_size=1, seed=None, data_shape_hint=None, model_dir=None,
                 channels_last=False, fp8=None, fp8_scaling=None):
        self.phase = phase
        self.device = torch.device(device)
        self.engine = engine            # "torch" (cpu / vendor libs) | "sm100" (our kernels)
        self.dtype = dtype              # activation dtype
        self.rank = rank
        self.world_size = world_size
        self.seed = seed
        self.data_shape_hint = data_shape_hint
        self.model_dir = model_dir
        self.channels_last = channels_last
        self.fp8 = fp8                  # sm100 engine: an ops/sm100.py FP8_MODES value (None: POSEIDON_FP8)
        self.fp8_scaling = fp8_scaling  # an ops/sm100.py FP8_SCALINGS value (None: POSEIDON_FP8_SCALING when fp8 is on)

    @property
    def train(self):
        return self.phase == P.TRAIN


class ParamSpec:
    def __init__(self, name, lr_mult=1.0, decay_mult=1.0, share_name=None):
        self.name, self.lr_mult, self.decay_mult = name, lr_mult, decay_mult
        self.share_name = share_name


class Layer(nn.Module):
    type_names: Sequence[str] = ()
    exact_bottoms: Optional[int] = None
    min_bottoms: Optional[int] = None
    exact_tops: Optional[int] = None
    min_tops: Optional[int] = None
    max_tops: Optional[int] = None
    is_loss = False
    is_data = False
    label_tops: Sequence[int] = ()     # data layers: tops that carry labels (never made differentiable by force_backward)

    def __init__(self, lp, ctx: NetContext):
        super().__init__()
        self.lp = lp
        self.ctx = ctx
        self.layer_name = lp.name or ""
        self.type_name = P.LayerTypeName.get(lp.type, "NONE")
        self.blob_names: List[str] = []   # attribute names of learnable blobs, in order

    # -- contract -------------------------------------------------------------------
    def setup(self, bottom_shapes: List[Shape]) -> List[Shape]:
        raise NotImplementedError

    def check_blob_counts(self, n_bottom: int, n_top: int):
        n = self.layer_name
        if self.exact_bottoms is not None and n_bottom != self.exact_bottoms:
            raise ValueError(f"{self.type_name} layer '{n}' takes {self.exact_bottoms} bottom blob(s), got {n_bottom}")
        if self.min_bottoms is not None and n_bottom < self.min_bottoms:
            raise ValueError(f"{self.type_name} layer '{n}' takes at least {self.min_bottoms} bottom blob(s)")
        if self.exact_tops is not None and n_top != self.exact_tops:
            raise ValueError(f"{self.type_name} layer '{n}' produces {self.exact_tops} top blob(s), got {n_top}")
        if self.min_tops is not None and n_top < self.min_tops:
            raise ValueError(f"{self.type_name} layer '{n}' produces at least {self.min_tops} top blob(s)")
        if self.max_tops is not None and n_top > self.max_tops:
            raise ValueError(f"{self.type_name} layer '{n}' produces at most {self.max_tops} top blob(s)")

    def allow_force_backward(self, bottom: int) -> bool:
        """May a net's force_backward ask this layer for the diff of bottom ``bottom``?
        reference: include/caffe/layer.hpp:296-298 (and the loss layers' overrides)."""
        return True

    def add_blob(self, attr: str, shape: Shape, filler=None) -> nn.Parameter:
        t = torch.empty(shape, dtype=torch.float32)
        fill(t, filler)
        p = nn.Parameter(t)
        setattr(self, attr, p)
        self.blob_names.append(attr)
        return p

    @property
    def blobs(self) -> List[nn.Parameter]:
        return [getattr(self, a) for a in self.blob_names]

    def caffe_blob_shape(self, idx: int) -> Shape:
        """4-D shape used when this blob is written to a .caffemodel."""
        s = tuple(self.blobs[idx].shape)
        return (1,) * (4 - len(s)) + s

    # ---- checkpoint views: engines may store a blob in a permuted physical order -------------------
    def export_blob(self, idx: int, tensor=None):
        """Blob ``idx`` (or a same-shaped companion tensor such as its momentum history) as a numpy array in
        Caffe's canonical element order and 4-D shape."""
        t = (self.blobs[idx] if tensor is None else tensor).detach().float()
        perm = getattr(self, "_k_perm", None)
        if perm is not None and idx == 0:
            c, h, w = perm
            t = t.reshape(t.shape[0], h, w, c).permute(0, 3, 1, 2)
        shape = getattr(self, "_caffe_shapes", {}).get(idx) or self.caffe_blob_shape(idx)
        return t.cpu().contiguous().numpy().reshape(shape)

    def import_blob(self, idx: int, array, tensor=None):
        """Inverse of :meth:`export_blob` (in-place copy into the blob / companion tensor)."""
        dst = self.blobs[idx] if tensor is None else tensor
        src = torch.from_numpy(array.copy()).float()
        perm = getattr(self, "_k_perm", None)
        with torch.no_grad():
            if perm is not None and idx == 0:
                c, h, w = perm
                n = dst.shape[0]
                src = src.reshape(n, c, h, w).permute(0, 2, 3, 1).reshape(n, -1)
            dst.copy_(src.reshape(dst.shape).to(dst.device))

    def extra_repr(self):
        return f"name={self.layer_name!r}, type={self.type_name}"


# ---------------------------------------------------------------------------------------
# Fillers — reference: include/caffe/filler.hpp:35-80 (constant/uniform), :84-134
# (gaussian + sparse), :138-204 (positive_unitball), :210-275 (xavier: fan_in = count/num)
# ---------------------------------------------------------------------------------------
_FILL_GEN: Optional[torch.Generator] = None


def set_filler_seed(seed: Optional[int]):
    global _FILL_GEN
    if seed is None or seed < 0:
        _FILL_GEN = None
    else:
        _FILL_GEN = torch.Generator()
        _FILL_GEN.manual_seed(int(seed))


def _caffe_num(t: torch.Tensor) -> int:
    """`num` of the Caffe blob holding this tensor: blobs are 4-D, lower-rank tensors are left-padded with ones."""
    return t.shape[0] if t.dim() == 4 else 1


def fill(t: torch.Tensor, filler=None) -> torch.Tensor:
    typ = filler.type if filler is not None else "constant"
    g = _FILL_GEN
    with torch.no_grad():
        if typ == "constant":
            t.fill_(filler.value if filler is not None else 0.0)
        elif typ == "uniform":
            t.uniform_(filler.min, filler.max, generator=g)
        elif typ == "gaussian":
            t.normal_(filler.mean, filler.std, generator=g)
            if filler.sparse >= 0:
                # each output unit keeps on average `sparse` non-zero inputs
                num_outputs = t.shape[0] if t.dim() > 1 else 1
                # Caffe uses blob->height() for IP weights (1,1,N,K) => N; num for conv.
                non_zero_p = float(filler.sparse) / float(num_outputs)
                mask = torch.bernoulli(torch.full_like(t, non_zero_p), generator=g)
                t.mul_(mask)
        elif typ == "positive_unitball":
            # the reference normalises each of the blob's `num` slices (filler.hpp:138-204); an inner-product weight is
            # the 4-D blob (1, 1, N, K), i.e. ONE slice of N*K elements
            t.uniform_(0, 1, generator=g)
            flat = t.view(_caffe_num(t), -1)
            flat.div_(flat.sum(dim=1, keepdim=True))
        elif typ == "xavier":
            # fan_in = count / num of the 4-D blob (filler.hpp:210-275): Cin*kh*kw for a convolution, but N*K for an
            # inner-product weight (blob (1,1,N,K)) and N for its bias — kept for parity with nets tuned on the reference
            # (GoogLeNet's classifiers), although it is not the layer's true fan-in
            fan_in = t.numel() // _caffe_num(t)
            scale = math.sqrt(3.0 / fan_in)
            t.uniform_(-scale, scale, generator=g)
        else:
            raise ValueError(f"unknown filler type '{typ}'")
    return t


def hw_param(msg, base: str, h_name: str, w_name: str, default=None):
    """Resolve Caffe's (x | x_h, x_w) parameter triplets, e.g. kernel_size/kernel_h/kernel_w."""
    if msg.has(h_name) or msg.has(w_name):
        h, w = getattr(msg, h_name), getattr(msg, w_name)
        if msg.has(base) and base not in ("pad", "stride"):
            raise ValueError(f"specify either {base} or {h_name}/{w_name}, not both")
        return int(h or 0), int(w or 0)
    v = getattr(msg, base)
    if v is None:
        v = default
    if v is None:
        raise ValueError(f"missing {base}")
    return int(v), int(v)
