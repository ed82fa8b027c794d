"""Swarm membership for DiLoCo workers on one NVLink domain.

The reference discovers peers through hivemind's Kademlia DHT + a Go libp2p daemon and tracks training progress in DHT
records (SURVEY.md E11/E12, hivemind_diloco.py:174-282).  On a single 8-GPU box the workers are ranks of one NCCL
world, so "the DHT" reduces to (a) the outer process group and (b) the c10d key-value store that already backs the
rendezvous — used here for arrival handshakes, straggler time-outs and drop detection.

``DHT`` keeps the constructor surface of ``hivemind.DHT`` that the reference touches (train_fsdp.py:205-212,
tests/test_diloco_hivemind.py:42-50) so calling code ports 1:1.
"""
from __future__ import annotations

import contextlib
import os
import threading
import time
from dataclasses import dataclass

import torch.distributed as dist

from . import comm


def get_dht_time() -> float:
    """Swarm clock.  One box => one clock domain; kept as a function for API parity (hivemind.utils.get_dht_time)."""
    return time.time()


class DHT:
    """Handle on the group of DiLoCo workers this process averages with."""

    def __init__(self, start: bool = True, initial_peers=None, host_maddrs=None, announce_maddrs=None,
                 group: dist.ProcessGroup | None = None, await_ready: bool = True, **_ignored):
        self.initial_peers = [initial_peers] if isinstance(initial_peers, str) else (initial_peers or [])
        self.host_maddrs, self.announce_maddrs = host_maddrs, announce_maddrs
        if group is None and dist.is_initialized() and dist.get_world_size() > 1:
            group = dist.group.WORLD
        self.group = group
        self._alive = bool(start)
        # Optional native membership board (csrc/host/rendezvous.cc): an ``odb://host:port`` entry in ``initial_peers`` (or
        # ODB_BOARD) makes progress records, arrival handshakes and liveness go through it instead of the c10d store -
        # it outlives / spans torchrun jobs and is visible to launchers and monitors.
        self.board = None
        board_addr = next((p for p in self.initial_peers if str(p).startswith("odb://")), os.environ.get("ODB_BOARD"))
        if start and board_addr:
            from . import rendezvous as rdv

            hp = rdv.parse_address(str(board_addr))
            if hp is None:
                raise ValueError(f"bad board address {board_addr!r} (expected odb://host:port)")
            self.board = rdv.RendezvousClient(hp[0], hp[1], peer_id=self.peer_id)
            self.board.start_heartbeat(ttl=float(os.environ.get("ODB_PEER_TTL", 120.0)))

    # -- membership
    @property
    def num_peers(self) -> int:
        return comm.group_size(self.group)

    @property
    def rank_in_group(self) -> int:
        return dist.get_rank(self.group) if self.group is not None else 0

    @property
    def peer_id(self) -> str:
        return f"worker-{self.rank_in_group}"

    def peer_ids(self) -> list[str]:
        return [f"worker-{r}" for r in range(self.num_peers)]

    def alive_peers(self) -> list[str]:
        """Peers with a live heartbeat on the board (all peers of the group when no board is attached)."""
        return sorted(self.board.alive_peers()) if self.board is not None else self.peer_ids()

    def store(self):
        if self.board is not None:
            return self.board.as_store()
        if not dist.is_initialized():
            return None
        try:
            return dist.distributed_c10d._get_default_store()
        except Exception:
            return None

    # -- hivemind.DHT surface
    def get_visible_maddrs(self) -> list[str]:
        addr = os.environ.get("MASTER_ADDR", "127.0.0.1")
        port = os.environ.get("MASTER_PORT", "0")
        return [f"/ip4/{addr}/tcp/{port}/p2p/{self.peer_id}"]

    def wait_until_ready(self, timeout: float | None = None) -> None:
        return None

    def is_alive(self) -> bool:
        return self._alive

    def shutdown(self) -> None:
        self._alive = False
        if self.board is not None:
            self.board.close()
            self.board = None


def log_visible_maddrs(maddrs, only_p2p: bool = False) -> None:
    from ..utils.logger import get_logger

    get_logger().info(f"Running a DHT instance. To connect other peers, use: --hv.initial-peers {' '.join(maddrs)}")


class PerformanceEMA:
    """Exponential moving average of samples/second (hivemind.utils.PerformanceEMA)."""

    def __init__(self, alpha: float = 0.1, eps: float = 1e-20):
        self.alpha, self.eps = alpha, eps
        self.samples_per_second = eps
        self.ema_seconds_per_sample = 0.0
        self.num_updates = 0
        self.timestamp = time.perf_counter()
        self.paused = False

    def update(self, task_size: float, interval: float | None = None) -> float:
        now = time.perf_counter()
        if interval is None:
            interval = max(0.0, now - self.timestamp)
        self.timestamp = now
        if task_size <= 0:
            return self.samples_per_second
        self.ema_seconds_per_sample = self.alpha * interval / task_size + (1 - self.alpha) * self.ema_seconds_per_sample
        self.num_updates += 1
        adjusted = self.ema_seconds_per_sample / (1 - (1 - self.alpha) ** self.num_updates)
        self.samples_per_second = 1.0 / max(adjusted, self.eps)
        return self.samples_per_second

    def reset_timer(self) -> None:
        self.timestamp = time.perf_counter()

    @contextlib.contextmanager
    def pause(self):
        self.paused = True
        try:
            yield
        finally:
            self.paused = False
            self.reset_timer()


@dataclass
class LocalTrainingProgress:
    peer_id: str
    epoch: int = 0
    samples_accumulated: int = 0
    samples_per_second: float = 0.0
    time: float = 0.0
    client_mode: bool = False


@dataclass
class GlobalTrainingProgress:
    epoch: int = 0
    samples_accumulated: int = 0
    target_batch_size: int = 0
    num_peers: int = 0
    num_clients: int = 0
    eta_next_epoch: float = 0.0
    next_fetch_time: float = 0.0


class StepControl:
    """Handle on a scheduled averaging round (subset of hivemind.averaging.control.StepControl used by the reference:
    hivemind_diloco.py:154-156,641,667-668,731-735)."""

    def __init__(self, scheduled_time: float | None = None, weight: float | None = None):
        self.scheduled_time = scheduled_time if scheduled_time is not None else get_dht_time()
        self.weight = weight
        self.stage = "LOOKING_FOR_GROUP"
        self._trigger = threading.Event()
        self._done = threading.Event()
        self._cancelled = False
        self._result = None
        self._exc: BaseException | None = None

    @property
    def triggered(self) -> bool:
        return self._trigger.is_set()

    def allow_allreduce(self) -> None:
        self._trigger.set()

    def done(self) -> bool:
        return self._done.is_set()

    def cancel(self) -> bool:
        if self._done.is_set():
            return False
        self._cancelled = True
        self.stage = "FINISHED"
        self._done.set()
        return True

    def cancelled(self) -> bool:
        return self._cancelled

    def set_result(self, result) -> None:
        self._result = result
        self.stage = "FINISHED"
        self._done.set()

    def set_exception(self, exc: BaseException) -> None:
        self._exc = exc
        self.stage = "FINISHED"
        self._done.set()

    def result(self, timeout: float | None = None):
        if not self._done.wait(timeout):
            raise TimeoutError("averaging round did not finish in time")
        if self._exc is not None:
            raise self._exc
        return self._result
