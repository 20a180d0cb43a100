"""Data layers: Data, ImageData, WindowData, HDF5Data/Output, MemoryData, DummyData.

reference: include/caffe/data_layers.hpp:32 (BaseData), :73 (BasePrefetching), :103 (Data),
:146 (DummyData), :182 (HDF5Data), :226 (HDF5Output), :270 (ImageData), :299 (MemoryData),
:341 (WindowData).
"""
from __future__ import annotations

import logging
import os
from typing import List, Optional

import numpy as np
import torch

from .. import ops
from ..data.db import RecordReader, open_db, shard_indices
from ..data.source import DBSource, Prefetcher, SyntheticSource
from ..data.transformer import DataTransformer
from .base import Layer, fill, register

log = logging.getLogger("poseidon_b200")


def _resolve(ctx, path):
    from ..utils.paths import resolve
    return resolve(path, ctx.model_dir)


def synthetic_allowed(ctx) -> bool:
    """Stand-in data is an explicit request, never a silent fallback: ``--synthetic_shape`` / ``data_shape_hint=`` or
    ``POSEIDON_SYNTHETIC_DATA=1`` (set by bench.py, smoke() and the test-suite).  Otherwise an unopenable source is
    fatal, like the reference's LOG(FATAL) (src/caffe/layers/data_layer.cpp:118-141)."""
    return ctx.data_shape_hint is not None or os.environ.get("POSEIDON_SYNTHETIC_DATA", "0") == "1"


def _no_source(ctx, layer_name, what):
    if not synthetic_allowed(ctx):
        raise IOError(f"data layer '{layer_name}': {what}. Refusing to train on synthetic data; pass "
                      "--synthetic_shape CxHxW (or set POSEIDON_SYNTHETIC_DATA=1) to request stand-in data explicitly")
    if ctx.rank == 0:
        log.warning("data layer '%s': %s -> synthetic data (explicitly allowed)", layer_name, what)


def _guess_shape(ctx, source: str, crop: int):
    """Shape of synthetic stand-in data when the named DB is not present on this box."""
    if ctx.data_shape_hint is not None:
        return tuple(ctx.data_shape_hint), 1000
    s = (source or "").lower()
    if "mnist" in s:
        return (1, 28, 28), 10
    if "cifar" in s:
        return (3, 32, 32), 10
    if crop:
        full = 256 if crop in (224, 227) else crop
        return (3, full, full), 1000
    return (3, 256, 256), 1000


class BasePrefetchingDataLayer(Layer):
    """Source → prefetch thread → (H2D on copy stream) → transform on device.
    reference: src/caffe/layers/base_data_layer.cpp:57-104."""
    exact_bottoms = 0
    min_tops = 1
    max_tops = 2
    is_data = True
    label_tops = (1,)

    def make_source(self):
        raise NotImplementedError

    def setup(self, bottom_shapes):
        self.transformer = DataTransformer(self.lp.transform_param, self.ctx.phase, self.ctx.device,
                                           seed=self.ctx.seed, model_dir=self.ctx.model_dir,
                                           allow_missing_mean=synthetic_allowed(self.ctx))
        self.source = self.make_source()
        x, y = self.source.next_batch()
        self._first = (x, y)
        n, c, h, w = x.shape
        oh, ow = self.transformer.out_hw(h, w)
        self.prefetch: Optional[Prefetcher] = None
        self.label_shape = (n,) + tuple(y.shape[1:]) if y.dim() > 1 else (n, 1, 1, 1)
        return [(n, c, oh, ow), self.label_shape]

    device_resident = False   # benchmarking: rotate over batches already staged on the device (no H2D)

    def _resident_batch(self):
        pool = getattr(self, "_resident_pool", None)
        if pool is None:
            dev = self.ctx.device
            pool = []
            for _ in range(4):
                x, y = self.source.next_batch()
                pool.append((x.to(dev), y.to(dev)))
            self._resident_pool, self._resident_i = pool, 0
        b = self._resident_pool[self._resident_i % len(self._resident_pool)]
        self._resident_i += 1
        return b

    def next_raw(self):
        if self.device_resident:
            self._first = None
            return self._resident_batch()
        if self._first is not None:
            x, y = self._first
            self._first = None
            dev = self.ctx.device
            if dev.type == "cuda":
                x, y = x.pin_memory().to(dev, non_blocking=True), y.pin_memory().to(dev, non_blocking=True)
            return x, y
        if self.prefetch is None:
            self.prefetch = Prefetcher(self.source, self.ctx.device)
        return self.prefetch.next()

    def forward(self):
        x, y = self.next_raw()
        k = ops.get(self.ctx)
        data = k.transform(self.transformer, x, self.ctx.dtype, first_conv=getattr(self, 'first_conv', None))
        if self.n_tops == 1:
            return (data,)
        return data, y.reshape(self.label_shape)

    def close(self):
        if self.prefetch is not None:
            self.prefetch.close()
        if hasattr(self.source, "close"):
            self.source.close()


@register("DATA")
class DataLayer(BasePrefetchingDataLayer):
    """Record-DB data layer with the reference's worker sharding; falls back to synthetic
    data of the right shape when the DB is absent (no datasets on the benchmark box).
    reference: src/caffe/layers/data_layer.cpp:102-259."""

    def make_source(self):
        dp = self.lp.data_param
        batch = int(dp.batch_size)
        src = _resolve(self.ctx, dp.source)
        shared = bool(dp.shared_file_system)
        nthreads = getattr(self.ctx, "threads_per_client", 1)
        client = self.ctx.rank // nthreads
        thread = self.ctx.rank % nthreads
        nclients = max(1, self.ctx.world_size // nthreads)
        path = src if shared or nclients == 1 else f"{src}_{client}"
        try:
            reader = open_db(path, dp.enum_name("backend"))
        except (IOError, OSError) as e:
            _no_source(self.ctx, self.layer_name, f"cannot open {path}: {e}")
            shape, ncls = _guess_shape(self.ctx, src, int(self.lp.transform_param.crop_size))
            return SyntheticSource(batch, shape, ncls, seed=1234 + self.ctx.rank)
        off, stride = shard_indices(len(reader), shared, nclients, client, nthreads, thread)
        from ..data.lmdb_reader import LMDBFile
        from ..data.native import NativeRecordDB
        if isinstance(reader, (RecordReader, LMDBFile, NativeRecordDB)) and \
                os.environ.get("POSEIDON_NATIVE_LOADER", "1") != "0":
            # C++ record loader: thread-pool Datum decode straight into pinned batch buffers
            from ..data import native
            if native.available():
                pdb = reader.path
                reader.close()
                return native.NativeDBSource(pdb, batch, off, stride, int(dp.rand_skip), self.ctx.seed)
        return DBSource(reader, batch, off, stride, int(dp.rand_skip), self.ctx.seed)


@register("IMAGE_DATA")
class ImageDataLayer(BasePrefetchingDataLayer):
    """List-file ("path label" per line) image source, optional resize + shuffle, sharded
    across workers. reference: src/caffe/layers/image_data_layer.cpp:24-102."""

    def make_source(self):
        ip = self.lp.image_data_param
        batch = int(ip.batch_size)
        src = _resolve(self.ctx, ip.source)
        if not src or not os.path.exists(src):
            shape, ncls = _guess_shape(self.ctx, src, int(self.lp.transform_param.crop_size))
            if ip.new_height and ip.new_width:
                shape = (3, int(ip.new_height), int(ip.new_width))
            _no_source(self.ctx, self.layer_name, f"image list {src!r} missing")
            return SyntheticSource(batch, shape, ncls, seed=4321 + self.ctx.rank)
        from ..data.images import ImageListSource
        nthreads = getattr(self.ctx, "threads_per_client", 1)
        nclients = max(1, self.ctx.world_size // nthreads)
        off, stride = shard_indices(0, bool(ip.shared_file_system), nclients, self.ctx.rank // nthreads,
                                    nthreads, self.ctx.rank % nthreads)
        return ImageListSource(src, batch, int(ip.new_height), int(ip.new_width), bool(ip.shuffle),
                               int(ip.rand_skip), off, stride, self.ctx.seed)


@register("WINDOW_DATA")
class WindowDataLayer(BasePrefetchingDataLayer):
    """R-CNN window sampling (fg/bg by overlap threshold, context padding, warp).
    reference: src/caffe/layers/window_data_layer.cpp:51-112 (window file), :170-390 (sampling)."""

    def make_source(self):
        wp = self.lp.window_data_param
        src = _resolve(self.ctx, wp.source)
        crop = int(self.lp.transform_param.crop_size)
        if not src or not os.path.exists(src):
            _no_source(self.ctx, self.layer_name, f"window file {src!r} missing")
            return SyntheticSource(int(wp.batch_size), (3, crop or 227, crop or 227), 21, seed=99 + self.ctx.rank)
        from ..data.images import WindowSource
        return WindowSource(src, int(wp.batch_size), crop, float(wp.fg_threshold), float(wp.bg_threshold),
                            float(wp.fg_fraction), int(wp.context_pad), wp.crop_mode,
                            mirror=bool(self.lp.transform_param.mirror), seed=self.ctx.seed)

    def setup(self, bottom_shapes):
        shapes = super().setup(bottom_shapes)
        # windows are already cropped/warped to crop_size by the source
        self.transformer.crop = 0
        n, c = shapes[0][:2]
        x = self._first[0]
        return [(n, c, x.shape[2], x.shape[3]), shapes[1]]


@register("HDF5_DATA")
class HDF5DataLayer(Layer):
    """Reads the "data" / "label" datasets of every file listed in ``source`` into memory, file after file (HDF5 through
    the built-in reader data/hdf5.py — contiguous or chunked / gzip / shuffle datasets of the classic file format —
    and ``.npz`` archives).  reference: src/caffe/layers/hdf5_data_layer.cpp:38-108, src/caffe/util/io.cpp
    (hdf5_load_nd_dataset: float / double data of at most 4 dimensions)."""
    exact_bottoms = 0
    exact_tops = 2
    is_data = True
    label_tops = (1,)

    def _load(self, path):
        if path.endswith(".npz") or path.endswith(".npy"):
            z = np.load(path)
            return z["data"].astype(np.float32), z["label"].astype(np.float32)
        from ..data import hdf5
        with hdf5.File(path) as f:
            for name in ("data", "label"):
                if name not in f:
                    raise IOError(f"{path}: dataset '{name}' not found (have: {', '.join(f.keys()) or 'none'})")
            d, l = f["data"], f["label"]
        if d.ndim > 4 or d.ndim < 1:
            raise ValueError(f"{path}: 'data' must have 1..4 dimensions, has {d.ndim}")
        if d.shape[0] != l.shape[0]:
            raise ValueError(f"{path}: 'data' has {d.shape[0]} rows but 'label' has {l.shape[0]}")
        return d.astype(np.float32), l.astype(np.float32)

    def setup(self, bottom_shapes):
        hp = self.lp.hdf5_data_param
        src = _resolve(self.ctx, hp.source)
        self.batch = int(hp.batch_size)
        with open(src) as f:
            self.files = [_resolve(self.ctx, l.strip()) for l in f if l.strip()]
        if not self.files:
            raise ValueError("HDF5 source list is empty")
        self.file_idx, self.row = 0, 0
        self.data, self.label = self._load(self.files[0])
        d = self.data.reshape(self.data.shape[0], *((1,) * (4 - self.data.ndim)), *self.data.shape[1:]) \
            if self.data.ndim < 4 else self.data
        self.data = d
        lab = self.label.reshape(self.label.shape[0], -1)
        self.label = lab
        return [(self.batch,) + tuple(d.shape[1:]), (self.batch, lab.shape[1], 1, 1)]

    def forward(self):
        xs, ys = [], []
        for _ in range(self.batch):
            if self.row == self.data.shape[0]:
                if len(self.files) > 1:
                    self.file_idx = (self.file_idx + 1) % len(self.files)
                    d, l = self._load(self.files[self.file_idx])
                    self.data = d.reshape(d.shape[0], *((1,) * (4 - d.ndim)), *d.shape[1:]) if d.ndim < 4 else d
                    self.label = l.reshape(l.shape[0], -1)
                self.row = 0
            xs.append(self.data[self.row])
            ys.append(self.label[self.row])
            self.row += 1
        dev = self.ctx.device
        x = torch.from_numpy(np.stack(xs)).to(dev).to(self.ctx.dtype)
        y = torch.from_numpy(np.stack(ys)).to(dev).reshape(self.batch, -1, 1, 1)
        return x, y


@register("HDF5_OUTPUT")
class HDF5OutputLayer(Layer):
    """Writes the (data, label) bottoms seen so far to ``file_name`` as the float datasets "data" / "label" of an HDF5
    file (built-in writer; an ``.npz`` name selects a numpy archive instead).
    reference: src/caffe/layers/hdf5_output_layer.cpp:17-68."""
    exact_bottoms = 2
    exact_tops = 0

    def setup(self, bottom_shapes):
        self.file_name = self.lp.hdf5_output_param.file_name
        self.saved = []
        return []

    def forward(self, data, label):
        self.saved.append((data.detach().float().cpu().numpy(), label.detach().float().cpu().numpy()))
        d = np.concatenate([s[0] for s in self.saved])
        l = np.concatenate([s[1] for s in self.saved])
        if self.file_name.endswith(".npz"):
            np.savez(self.file_name, data=d, label=l)
        else:
            from ..data import hdf5
            hdf5.save(self.file_name, {"data": d.astype(np.float32), "label": l.astype(np.float32)})
        return ()


@register("MEMORY_DATA")
class MemoryDataLayer(Layer):
    """Zero-copy batches from user memory: ``reset(data, labels)`` then forward advances by
    batch_size. reference: src/caffe/layers/memory_data_layer.cpp:34-73."""
    exact_bottoms = 0
    exact_tops = 2
    is_data = True
    label_tops = (1,)

    def setup(self, bottom_shapes):
        mp = self.lp.memory_data_param
        self.batch = int(mp.batch_size)
        self.shape = (int(mp.channels), int(mp.height), int(mp.width))
        self.data = self.labels = None
        self.pos = 0
        return [(self.batch,) + self.shape, (self.batch, 1, 1, 1)]

    def reset(self, data, labels):
        data = torch.as_tensor(data)
        labels = torch.as_tensor(labels).float()
        if data.shape[0] % self.batch:
            raise ValueError("The number of added datum must be a multiple of the batch size.")
        self.data = data.reshape(data.shape[0], *self.shape).to(self.ctx.device)
        self.labels = labels.reshape(-1).to(self.ctx.device)
        self.pos = 0

    Reset = reset

    def forward(self):
        if self.data is None:
            raise RuntimeError("MemoryDataLayer needs to be initialized by calling reset")
        s = slice(self.pos, self.pos + self.batch)
        x = self.data[s].to(self.ctx.dtype)
        y = self.labels[s].reshape(self.batch, 1, 1, 1)
        self.pos = (self.pos + self.batch) % self.data.shape[0]
        return x, y


@register("DUMMY_DATA")
class DummyDataLayer(Layer):
    """N filler-generated tops; constant fillers are filled once, others refilled every
    forward — generated directly on the device.
    reference: src/caffe/layers/dummy_data_layer.cpp:10-98."""
    exact_bottoms = 0
    min_tops = 1
    is_data = True

    def setup(self, bottom_shapes):
        p = self.lp.dummy_data_param
        nt = self.n_tops

        def dim(lst, i):
            lst = list(lst)
            if len(lst) not in (1, nt):
                raise ValueError("Must specify either a single (1) or one per top blob")
            return int(lst[0] if len(lst) == 1 else lst[i])

        self.shapes = [(dim(p.num, i), dim(p.channels, i), dim(p.height, i), dim(p.width, i))
                       for i in range(nt)]
        nf = len(p.data_filler)
        if nf not in (0, 1, nt):
            raise ValueError("Number of data fillers must be 0, 1 or equal to the number of tops")
        self.fillers = [None if nf == 0 else p.data_filler[0 if nf == 1 else i] for i in range(nt)]
        self.cache: List[Optional[torch.Tensor]] = [None] * nt
        return list(self.shapes)

    def forward(self):
        outs = []
        for i, (shape, f) in enumerate(zip(self.shapes, self.fillers)):
            const = f is None or f.type == "constant"
            if self.cache[i] is None or not const:
                t = torch.empty(shape, dtype=torch.float32)
                fill(t, f)
                self.cache[i] = t.to(self.ctx.device)
            t = self.cache[i]
            outs.append(t)
        return tuple(outs)
