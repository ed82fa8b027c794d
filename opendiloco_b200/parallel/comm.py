"""Process topology and collectives.

One process per GPU, ``torch.distributed`` (NCCL over NVLink / NVSwitch; gloo on CPU) for the plumbing.  The job is
a grid ``galaxy_size x gpus_per_worker``:

    rank = world_rank * gpus_per_worker + local_rank
    inner group  = the ranks of one DiLoCo worker   (gradient reduce / ZeRO sharding every step)
    outer group  = same local_rank across workers   (pseudo-gradient all-reduce every H steps)

which is the reference's "galaxy" of workers (train_fsdp.py:91-92,151-156) collapsed onto one NCCL world instead of
one torchrun + hivemind swarm per worker (SURVEY.md §1 process topology, §5.8).  Workers may also be launched as
separate ``torchrun`` jobs that rendezvous on one TCP store (``--hv.initial-peers tcp://host:port``), mirroring
run_training.sh.

Every collective here is issued ONCE on a flat buffer (the reference issues one per parameter tensor:
train_diloco_torch.py:255,345; train_fsdp.py:410-413).
"""
from __future__ import annotations

import datetime
import os
from dataclasses import dataclass

import torch
import torch.distributed as dist

TIMEOUT_NCCL_MINUTES = int(os.environ.get("TIMEOUT_NCCL_MINUTES", 120))  # reference: train_fsdp.py:64


def default_backend() -> str:
    return "nccl" if torch.cuda.is_available() else "gloo"


def init_distributed(backend: str | None = None, init_method: str | None = None, rank: int | None = None,
                     world_size: int | None = None) -> None:
    """Idempotent process-group bring-up from the torchrun environment (reference: ddp_setup, train_fsdp.py:70-72)."""
    if dist.is_initialized():
        return
    backend = backend or default_backend()
    local_rank = int(os.environ.get("LOCAL_RANK", 0))
    kwargs: dict = dict(backend=backend, timeout=datetime.timedelta(minutes=TIMEOUT_NCCL_MINUTES))
    if backend == "nccl":
        torch.cuda.set_device(local_rank)
        kwargs["device_id"] = torch.device("cuda", local_rank)
    if init_method is not None and init_method.startswith("tcp://"):
        # Workers launched as SEPARATE torchrun jobs (run_training.sh) meet on one address.  The store is created here and
        # not by init_process_group: under torchrun ``TORCHELASTIC_USE_AGENT_STORE`` makes torch's tcp:// handler connect
        # to the address as a client on EVERY rank (it assumes the elastic agent hosts it), so nobody would ever listen.
        host, port = init_method[len("tcp://"):].rsplit(":", 1)
        store = dist.TCPStore(host, int(port), world_size, is_master=(rank == 0),
                              timeout=datetime.timedelta(minutes=TIMEOUT_NCCL_MINUTES), wait_for_workers=False)
        kwargs.update(store=store, rank=rank, world_size=world_size)
    elif init_method is not None:
        kwargs.update(init_method=init_method, rank=rank, world_size=world_size)
    elif "RANK" not in os.environ:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29512")
        kwargs.update(rank=0, world_size=1)
    dist.init_process_group(**kwargs)


def shutdown_distributed() -> None:
    if dist.is_initialized():
        dist.destroy_process_group()


@dataclass
class Topology:
    rank: int
    world_size: int
    local_rank: int                 # rank inside the DiLoCo worker
    gpus_per_worker: int
    world_rank: int                 # index of this DiLoCo worker
    galaxy_size: int                # number of DiLoCo workers
    inner_group: dist.ProcessGroup | None
    outer_group: dist.ProcessGroup | None

    @property
    def is_worker_leader(self) -> bool:
        return self.local_rank == 0


def build_topology(galaxy_size: int | None = None, gpus_per_worker: int | None = None) -> Topology:
    """Carve the default world into (workers x gpus-per-worker).  Groups are created collectively by every rank."""
    if not dist.is_initialized():
        return Topology(0, 1, 0, 1, 0, 1, None, None)
    world, rank = dist.get_world_size(), dist.get_rank()
    if galaxy_size is None and gpus_per_worker is None:
        galaxy_size, gpus_per_worker = world, 1
    elif galaxy_size is None:
        galaxy_size = world // gpus_per_worker
    elif gpus_per_worker is None:
        gpus_per_worker = world // galaxy_size
    assert galaxy_size * gpus_per_worker == world, (galaxy_size, gpus_per_worker, world)
    wr, lr = divmod(rank, gpus_per_worker)
    inner = outer = None
    if gpus_per_worker > 1:
        for w in range(galaxy_size):
            g = dist.new_group(list(range(w * gpus_per_worker, (w + 1) * gpus_per_worker)))
            if w == wr:
                inner = g
    if galaxy_size > 1:
        if gpus_per_worker == 1:
            outer = dist.group.WORLD
        else:
            for l in range(gpus_per_worker):
                g = dist.new_group(list(range(l, world, gpus_per_worker)))
                if l == lr:
                    outer = g
    return Topology(rank, world, lr, gpus_per_worker, wr, galaxy_size, inner, outer)


def group_size(group) -> int:
    if group is None or not dist.is_initialized():
        return 1
    return dist.get_world_size(group)


def all_reduce_avg_(buf: torch.Tensor, group) -> torch.Tensor:
    """In-place mean over the group on ONE flat buffer.  NCCL has a native AVG; gloo gets SUM + scale."""
    n = group_size(group)
    if n == 1:
        return buf
    if buf.is_cuda:
        dist.all_reduce(buf, op=dist.ReduceOp.AVG, group=group)
    else:
        work = buf if buf.dtype in (torch.float32, torch.float64) else buf.float()
        dist.all_reduce(work, op=dist.ReduceOp.SUM, group=group)
        work.div_(n)
        if work is not buf:
            buf.copy_(work)
    return buf


def _global_rank(group, r: int) -> int:
    return r if (group is None or group is dist.group.WORLD) else dist.get_global_rank(group, r)


def p2p_all_reduce_mean_(buf: torch.Tensor, members: list[int], group) -> torch.Tensor:
    """In-place mean of ONE flat buffer over a SUBSET of the group (``members`` = sorted ranks inside ``group``), built
    from point-to-point transfers only, so ranks outside the subset do not have to take part - the elastic (NO_WAIT)
    outer round.  Butterfly: member j owns slice j; everybody sends slice j to its owner, the owner averages and sends
    the result back to everybody (2 * (k-1)/k of the vector per member, like a reduce-scatter + all-gather)."""
    k = len(members)
    if k <= 1:
        return buf
    me = dist.get_rank(group)
    idx = members.index(me)
    flat = buf.view(-1)
    n = flat.numel()
    per = -(-n // k)
    per += (-per) % 8                                    # keep slices 8-element aligned
    bounds = [(min(j * per, n), min((j + 1) * per, n)) for j in range(k)]
    lo, hi = bounds[idx]
    mine = flat[lo:hi]
    # phase 1: my slice of everybody's vector comes to me
    inbox = [torch.empty_like(mine) for _ in range(k - 1)]
    ops, slot = [], 0
    for j, r in enumerate(members):
        if j == idx:
            continue
        a, b = bounds[j]
        if b > a:
            ops.append(dist.P2POp(dist.isend, flat[a:b], _global_rank(group, r), group))
        if hi > lo:
            ops.append(dist.P2POp(dist.irecv, inbox[slot], _global_rank(group, r), group))
        slot += 1
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    if hi > lo:
        acc = mine.float() if mine.dtype not in (torch.float32, torch.float64) else mine
        for t in inbox:
            acc += t.to(acc.dtype)
        acc /= k
        if acc is not mine:
            mine.copy_(acc)
    # phase 2: averaged slices go back out
    ops = []
    for j, r in enumerate(members):
        if j == idx:
            continue
        a, b = bounds[j]
        if hi > lo:
            ops.append(dist.P2POp(dist.isend, mine, _global_rank(group, r), group))
        if b > a:
            ops.append(dist.P2POp(dist.irecv, flat[a:b], _global_rank(group, r), group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    return buf


def p2p_send_(bufs: list[torch.Tensor], dst_rank_in_group: int, group) -> None:
    for req in dist.batch_isend_irecv([dist.P2POp(dist.isend, b, _global_rank(group, dst_rank_in_group), group) for b in bufs]):
        req.wait()


def p2p_recv_(bufs: list[torch.Tensor], src_rank_in_group: int, group) -> None:
    for req in dist.batch_isend_irecv([dist.P2POp(dist.irecv, b, _global_rank(group, src_rank_in_group), group) for b in bufs]):
        req.wait()


def all_reduce_sum_(buf: torch.Tensor, group) -> torch.Tensor:
    if group_size(group) > 1:
        dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)
    return buf


def broadcast_(buf: torch.Tensor, src_rank_in_group: int, group) -> torch.Tensor:
    """Flat broadcast (reference N1/N6: one broadcast per tensor, train_diloco_torch.py:253-255, train_fsdp.py:410-413)."""
    if group_size(group) > 1:
        src = dist.get_global_rank(group, src_rank_in_group) if group is not dist.group.WORLD else src_rank_in_group
        dist.broadcast(buf, src=src, group=group)
    return buf


def barrier(group=None) -> None:
    if dist.is_initialized() and dist.get_world_size() > 1:
        if torch.cuda.is_available() and dist.get_backend() == "nccl":
            dist.barrier(group=group, device_ids=[torch.cuda.current_device()])
        else:
            dist.barrier(group=group)
