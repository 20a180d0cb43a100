"""Branch-parallel execution: independent branches of the layer graph run on separate CUDA streams ("lanes").

GoogLeNet's inception modules fan one blob out to four branches of small convolutions (at batch 32 a 14x14 stage has
49 m-blocks, a 7x7 stage 13 — a fraction of the 132 SMs), plus two auxiliary classifier heads hanging off the trunk.
Run back to back every one of those kernels leaves most of the chip idle; on separate streams the branches overlap, and
the whole-step CUDA graph records them as parallel branches.  The reference executes layers strictly in sequence
(src/caffe/net.cpp:709-750 ForwardFromTo; :752-784 BackwardFromTo) — one kernel at a time on one stream.

Plan (static, per net): walking the layers in order, the k-th consumer of a producer's outputs runs on lane
``(lane(producer) + k) mod L`` — the first consumer continues on the producer's lane, further consumers fork.  A layer
with several bottoms (CONCAT, losses) sits on the lane given by its first bottom and waits for the others.

Execution: lane 0 is the caller's current stream.  A layer whose bottom was produced on another lane waits on that
producer's event; outputs read on another lane are registered with the caching allocator (``record_stream``) so their
memory is not recycled while the other lane still reads it.  All lanes fork from the caller's stream at the start of a
forward pass and join it at the end.  Backward needs nothing here: autograd runs every node on the stream its forward
ran on and synchronises across streams itself, so the backward of the branches overlaps the same way.
"""
from __future__ import annotations

import logging
import os
from typing import List

import torch

log = logging.getLogger("poseidon_b200")


def default_lanes(ctx) -> int:
    env = os.environ.get("POSEIDON_LANES")
    if env is not None:
        return max(1, int(env))
    # the vendor-library arm keeps the reference's one-kernel-at-a-time schedule.  8: GoogLeNet 3.25 ms with 4 lanes,
    # 3.17 ms with 8 (an inception output has up to 5 readers, and every lane has its own weight-gradient side stream)
    return 8 if getattr(ctx, "engine", "") == "sm100" else 1


def plan_lanes(net, n_lanes: int) -> None:
    """Sets net.lane (per layer), net.lane_wait (per layer: producer layer indices on other lanes), net.lane_share (per
    layer: for each top, the other lanes that read it) and net.n_lanes (1 = feature off)."""
    n = len(net.layers)
    net.n_lanes = 1
    net.lane = [0] * n
    net.lane_wait = [[] for _ in range(n)]
    net.lane_share = [[[] for _ in net.top_names[i]] for i in range(n)]
    if n_lanes <= 1:
        return
    skip = getattr(net, "skip_layer", [False] * n)
    producer = {}                        # blob name -> layer index of its current version
    slots = [0] * n                      # consumers seen so far per producer
    lane: List[int] = [0] * n
    for i in range(n):
        if skip[i]:
            continue                     # fused away: the blob keeps its producer
        prods = []
        for b in net.bottom_names[i]:
            p = producer.get(b)
            if p is not None and p not in prods:
                prods.append(p)
        if prods:
            p0 = prods[0]
            lane[i] = (lane[p0] + slots[p0]) % n_lanes
            for p in prods:
                slots[p] += 1
        for p in prods:
            if lane[p] != lane[i]:
                net.lane_wait[i].append(p)
                for k, t in enumerate(net.top_names[p]):
                    if t in net.bottom_names[i] and lane[i] not in net.lane_share[p][k]:
                        net.lane_share[p][k].append(lane[i])
        for t in net.top_names[i]:
            producer[t] = i
    used = sorted(set(lane[i] for i in range(n) if not skip[i]))
    if len(used) <= 1:
        return
    net.n_lanes = n_lanes
    net.lane = lane
    if net.ctx.rank == 0:
        forks = sum(1 for i in range(n) if net.lane_wait[i])
        log.info("lane plan: %d layers on %d streams (%s), %d cross-stream edges", n - sum(skip), len(used),
                 ", ".join(f"lane {u}: {sum(1 for i in range(n) if lane[i] == u and not skip[i])}" for u in used), forks)


class LaneRunner:
    """Per-forward-pass stream bookkeeping (streams and events are created once per net and reused)."""

    def __init__(self, net):
        self.net = net
        self.side = None
        self.events = {}

    def begin(self, start: int = 0):
        net = self.net
        self.first = start               # blobs of earlier layers come from the caller (prefilled inputs): no event
        self.cur = torch.cuda.current_stream()
        if self.side is None or self.side[0].device != self.cur.device:
            self.side = [torch.cuda.Stream(device=self.cur.device) for _ in range(net.n_lanes - 1)]
            self.start = torch.cuda.Event()
            self.join = [torch.cuda.Event() for _ in self.side]
            self.events = {}
        self.streams = [self.cur] + self.side
        self.start.record(self.cur)
        for s in self.side:
            s.wait_event(self.start)     # fork: everything the caller queued so far (inputs, weight updates) is visible

    def stream_of(self, i):
        return self.streams[self.net.lane[i]]

    def before(self, i):
        s = self.streams[self.net.lane[i]]
        for p in self.net.lane_wait[i]:
            if p >= self.first:
                s.wait_event(self.events[p])

    def after(self, i, outs):
        net = self.net
        shared = False
        for k, o in enumerate(outs[: len(net.lane_share[i])]):
            for l in net.lane_share[i][k]:
                shared = True
                if isinstance(o, torch.Tensor) and o.is_cuda:
                    o.record_stream(self.streams[l])
        if shared:
            ev = self.events.get(i)
            if ev is None:
                ev = self.events[i] = torch.cuda.Event()
            ev.record(self.streams[net.lane[i]])

    def finish(self):
        for s, ev in zip(self.side, self.join):
            ev.record(s)
            self.cur.wait_event(ev)
