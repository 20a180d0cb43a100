"""Rank / device context: the replacement for Poseidon's hostfile + client_id + thread-per-GPU
topology (one process per GPU, ``torchrun`` environment, ``torch.distributed`` for bootstrap).

reference: src/caffe/common.cpp:126-221 (Caffe singleton: device list, thread→device map,
per-device handles, cluster seed), ps/src/petuum_ps/thread/context.hpp:69-467
(GlobalContext: client/thread id arithmetic), ps/src/petuum_ps_common/util/utils.cpp:15-35
(hostfile parser).
"""
from __future__ import annotations

import datetime
import logging
import os
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist

log = logging.getLogger("poseidon_b200")


class RankContext:
    def __init__(self, rank=0, world_size=1, local_rank=0, device="cpu", backend=None):
        self.rank, self.world_size, self.local_rank = rank, world_size, local_rank
        self.device = torch.device(device)
        self.backend = backend

    @property
    def is_root(self):
        return self.rank == 0

    @property
    def distributed(self):
        return self.world_size > 1

    def barrier(self):
        if self.distributed:
            if self.device.type == "cuda":
                dist.barrier(device_ids=[self.device.index])
            else:
                dist.barrier()

    def broadcast_(self, t: torch.Tensor, src=0):
        if self.distributed:
            dist.broadcast(t, src)
        return t

    def all_reduce_(self, t: torch.Tensor):
        if self.distributed:
            dist.all_reduce(t)
        return t

    def max_over_ranks(self, value: float) -> float:
        if not self.distributed:
            return value
        t = torch.tensor([value], dtype=torch.float64, device=self.device)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def shutdown(self):
        if self.distributed and dist.is_initialized():
            dist.destroy_process_group()


def parse_hostfile(path: str) -> List[Tuple[int, str, int]]:
    """Lines of ``<id> <ip> <port>``; '#' comments allowed.
    reference: ps/src/petuum_ps_common/util/utils.cpp:15-35, machinefiles/localserver."""
    out = []
    with open(path) as f:
        for line in f:
            line = line.split("#", 1)[0].strip()
            if not line:
                continue
            i, ip, port = line.split()[:3]
            out.append((int(i), ip, int(port)))
    return sorted(out)


def init_rank_context(device: Optional[str] = None, hostfile: Optional[str] = None,
                      client_id: Optional[int] = None, timeout_s: int = 600) -> RankContext:
    """Build the rank context from the torchrun env (RANK/LOCAL_RANK/WORLD_SIZE/MASTER_*) or,
    Poseidon-style, from ``--hostfile`` + ``--client_id`` (host 0 becomes the rendezvous)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if hostfile and "WORLD_SIZE" not in os.environ:
        hosts = parse_hostfile(hostfile)
        if len(hosts) > 1:
            if client_id is None:
                raise ValueError("--client_id is required with a multi-host hostfile")
            world, rank = len(hosts), int(client_id)
            os.environ.setdefault("MASTER_ADDR", hosts[0][1])
            os.environ.setdefault("MASTER_PORT", str(hosts[0][2]))
            local_rank = sum(1 for (i, ip, _) in hosts if ip == hosts[rank][1] and i < rank)
            # node layout for the NVLink arena (parallel/fused.py): lines of one host must be contiguous and every host
            # must list the same number of processes — what torchrun's node-major rank order guarantees
            ips = [ip for (_, ip, _) in hosts]
            per_host = ips.count(ips[rank])
            blocks_ok = all(ips[i] == ips[i - i % per_host] for i in range(world)) and world % per_host == 0 and \
                len(set(ips)) * per_host == world
            if blocks_ok:
                os.environ.setdefault("LOCAL_WORLD_SIZE", str(per_host))
                os.environ.setdefault("LOCAL_RANK", str(local_rank))
            elif len(set(ips)) > 1:
                raise ValueError("hostfile: list the processes of each host on consecutive lines, the same number per "
                                 "host (needed to form the per-node NVLink groups)")
    use_cuda = torch.cuda.is_available() and (device is None or str(device).startswith("cuda"))
    if use_cuda:
        if device is not None and ":" in str(device) and world == 1:
            dev = torch.device(device)
        else:
            dev = torch.device("cuda", local_rank % torch.cuda.device_count())
        torch.cuda.set_device(dev)
        # NumaMgr's role (ps/src/petuum_ps/thread/numa_mgr.hpp:28-203): the per-GPU process — and with it the first-touch
        # placement of its pinned input buffers — stays on the CPUs of the GPU's NUMA node, so the per-step H2D copies do
        # not cross sockets.  POSEIDON_NUMA=off (default, like the reference's optional NumaMgr) | center | even;
        # its effect is not measured on H100.
        policy = os.environ.get("POSEIDON_NUMA", "off")
        if policy != "off":
            from ..utils.affinity import pin_to_gpu_numa
            cpus = pin_to_gpu_numa(dev.index if dev.index is not None else 0, policy, local_rank,
                                   int(os.environ.get("LOCAL_WORLD_SIZE", str(world))))
            log.debug("rank %d: pinned to %d CPUs (%s)", rank, len(cpus), policy)
    else:
        dev = torch.device("cpu")
    backend = None
    if world > 1:
        backend = "nccl" if dev.type == "cuda" else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if not dist.is_initialized():
            kw = dict(backend=backend, rank=rank, world_size=world,
                      timeout=datetime.timedelta(seconds=timeout_s))
            if dev.type == "cuda":
                kw["device_id"] = dev
            dist.init_process_group(**kw)
    return RankContext(rank, world, local_rank, dev, backend)
