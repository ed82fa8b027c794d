"""Host side of the fused outer step (``csrc/outer_comm.cu``): NVLink symmetric-memory windows + launch.

``torch.distributed._symmetric_memory`` is used purely as plumbing: it allocates the same-sized window on every rank of
the outer group, exchanges the handles, maps every peer's window into this process (P2P over NVLink) and - when the
fabric supports NVLS - binds them to one multicast address.  The kernel that touches those pointers is ours.
"""
from __future__ import annotations

import ctypes
import os

import torch
import torch.distributed as dist

from .. import _lib
from ..utils.logger import get_logger

c_void_p, c_int, c_ll, c_float, c_uint = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float, ctypes.c_uint
_lib.register_optional("odb_fused_outer_step", [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                c_int, c_int, c_ll, c_float, c_float, c_int, c_uint, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p])
_lib.register_optional("odb_fused_outer_pipelined", [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                                    c_ll, c_float, c_float, c_int, c_uint, c_uint, c_int, c_int, c_int, c_void_p,
                                                    c_void_p, c_void_p])
_lib.register_optional("odb_fused_outer_sharded", [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_ll,
                                                  c_float, c_float, c_int, c_uint, c_uint, c_int, c_int, c_void_p, c_void_p,
                                                  c_void_p, c_void_p, c_void_p])
_lib.register_optional("odb_outer_set_timeout_ms", [c_int])
_lib.register_optional("odb_fused_outer_subset", [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                                 c_int, c_int, c_ll, c_float, c_float, c_int, c_uint, c_int, c_void_p, c_void_p])
logger = get_logger()
MAX_CHUNKS, MAX_PEERS = 64, 16
FLAG_WORDS = 2 * MAX_CHUNKS * MAX_PEERS     # pipelined kernel: ready[chunk][peer] | done[chunk][peer]; phase-sequential kernel uses the first 32


class FusedOuterStep:
    """pseudo-gradient -> (bf16 cast) -> NVLink all-reduce -> Nesterov -> theta_local/shadow write-back: one launch."""

    def __init__(self, opt, group, delta_bf16: bool):
        import torch.distributed._symmetric_memory as symm_mem

        sa = opt.state_averager
        self.opt, self.sa, self.group = opt, sa, group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.n = sa.theta_outer.numel()
        assert self.n % (8 * self.world) == 0
        dev = sa.theta_outer.device
        self.delta_bf16 = delta_bf16
        dt = torch.bfloat16 if delta_bf16 else torch.float32
        self.window = symm_mem.empty(self.n, dtype=dt, device=dev)
        self.flags = symm_mem.empty(FLAG_WORDS, dtype=torch.int32, device=dev)
        self.flags.zero_()
        gname = group.group_name
        try:
            if hasattr(symm_mem, "is_symm_mem_enabled_for_group") and not symm_mem.is_symm_mem_enabled_for_group(gname):
                symm_mem.enable_symm_mem_for_group(gname)
        except Exception:
            pass
        self.h_win = symm_mem.rendezvous(self.window, gname)
        self.h_flag = symm_mem.rendezvous(self.flags, gname)
        self.mc_ptr = int(getattr(self.h_win, "multicast_ptr", 0) or 0)
        if os.environ.get("ODB_FUSED_OUTER_NO_MULTIMEM"):
            self.mc_ptr = 0
        PtrArr = c_void_p * self.world
        self._win_ptrs = PtrArr(*[int(p) for p in self.h_win.buffer_ptrs])
        self._flag_ptrs = PtrArr(*[int(p) for p in self.h_flag.buffer_ptrs])
        self.timeout_flag = torch.zeros(1, dtype=torch.int32, device=dev)
        # ODB_OUTER_STAMPS=1: block 0 records globaltimer at the phase boundaries (phase profile of the fused kernel)
        self.stamps = torch.zeros(8, dtype=torch.int64, device=dev) if os.environ.get("ODB_OUTER_STAMPS") else None
        self.seq = 0
        self.launch_idx = 0
        self.counters = torch.zeros(2 * MAX_CHUNKS, dtype=torch.int32, device=dev)
        self.nchunk = int(os.environ.get("ODB_OUTER_CHUNKS", 16))
        while self.n % (8 * self.world * self.nchunk):
            self.nchunk //= 2
        self.pipelined = bool(self.mc_ptr) and self.nchunk >= 2 and os.environ.get("ODB_OUTER_PIPELINED", "1") != "0" \
            and _lib.has_symbol("odb_fused_outer_pipelined")
        # bounded cross-GPU waits: a missing peer raises the flag after this long (the host then raises, see poll_timeout)
        if _lib.has_symbol("odb_outer_set_timeout_ms"):
            lib = _lib.cuda_lib()
            lib.odb_outer_set_timeout_ms(int(float(os.environ.get("ODB_OUTER_TIMEOUT_S", 20.0)) * 1e3))
        self._tf_host = torch.zeros(1, dtype=torch.int32, pin_memory=True)
        self._tf_event: torch.cuda.Event | None = None
        self.fingerprint: torch.Tensor | None = None
        # ---- sharded in-place form (fp32 transport): the master weights themselves live in a symmetric window
        self.sharded = False
        self._side = None                 # side stream of the background momentum re-replication
        self._regather_pending = False
        want_sharded = (not delta_bf16 and bool(self.mc_ptr) and os.environ.get("ODB_OUTER_SHARDED", "1") != "0"
                        and _lib.has_symbol("odb_fused_outer_sharded") and sa.theta_outer.dtype == torch.float32)
        if want_sharded:
            try:
                self._init_sharded(symm_mem, gname)
            except Exception as e:        # keep the replicated-update kernel
                logger.warning(f"sharded outer step unavailable ({type(e).__name__}: {e}); using the replicated-update kernel")
                self.sharded = False
        torch.cuda.synchronize(dev)
        self.h_flag.barrier()
        mode = "sharded in-place x" + str(self.nchunk_sh) if self.sharded else \
            ("pipelined x" + str(self.nchunk) if self.pipelined else "phase-sequential")
        logger.info(f"fused outer step: {self.world} ranks, window {self.n * self.window.element_size() / 1e6:.0f} MB "
                    f"{'bf16' if delta_bf16 else 'fp32'}, multimem={'yes' if self.mc_ptr else 'no (P2P loads/stores)'}, {mode}")

    def _init_sharded(self, symm_mem, gname: str) -> None:
        """Re-home the fp32 master weights into a symmetric allocation (so the switch can reduce / multicast them in
        place) and set up the sharded kernel's bookkeeping."""
        sa, fv = self.sa, self.sa.fv
        dev = sa.theta_outer.device
        nch = int(os.environ.get("ODB_OUTER_CHUNKS", 16))
        while nch > 1 and self.n % (4 * self.world * nch):
            nch //= 2
        if self.n % (4 * self.world * nch):
            raise ValueError("parameter vector not divisible into slabs")
        master = symm_mem.empty(fv.flat.numel(), dtype=torch.float32, device=dev)
        h = symm_mem.rendezvous(master, gname)
        mc = int(getattr(h, "multicast_ptr", 0) or 0)
        if not mc:
            raise RuntimeError("no multicast address for the master-weight window")
        fv.rehome(master)
        self.master, self.h_master = master, h
        lo = fv.lo
        sa.theta_local = fv.own(fv.flat)
        self.opt.diloco_grad_averager._flat = (sa.theta_outer, sa.delta, sa.theta_local)
        self._theta_mc = mc + lo * 4
        self.nchunk_sh = nch
        self.counters_sh = torch.zeros(2 * MAX_CHUNKS, dtype=torch.int32, device=dev)
        self.launch_idx_sh = 0
        self.fingerprint = torch.zeros(1, dtype=torch.int64, device=dev)
        self.slab = self.n // self.world
        self._side = torch.cuda.Stream(device=dev)
        self.sharded = True

    @classmethod
    def try_create(cls, opt, compression=None):
        dht = opt.dht
        if dht is None or dht.group is None or not torch.cuda.is_available():
            return None
        if dist.get_backend(dht.group) != "nccl" or not _lib.has_symbol("odb_fused_outer_step"):
            return None
        sa = opt.state_averager
        g = sa._sgd_hparams()
        if g is None or g.get("momentum", 0) == 0 or sa.theta_outer.device != sa.theta_local.device:
            return None
        bf16 = compression is not None and getattr(compression, "name", "") == "bf16"
        try:
            return cls(opt, dht.group, bf16)
        except Exception as e:  # symmetric memory unavailable (no P2P, driver too old, ...): NCCL path is used instead
            logger.warning(f"fused outer step unavailable ({type(e).__name__}: {e}); using flat NCCL all-reduce + fused Nesterov")
            return None

    def _seq_for(self, epoch: int | None) -> int:
        """Sequence number of the cross-GPU flags of this round.  Derived from the OUTER EPOCH, not from a per-process launch
        counter: the members of a round are at the same epoch by construction, whereas launch counts diverge as soon as a
        worker sits out a partial round.  8 numbers per epoch: full round {0, 1}, partial rounds {2, 3}."""
        if epoch is None:
            self.seq += 8
            return self.seq
        self.seq = max(self.seq, 8 * (int(epoch) + 1))
        return 8 * (int(epoch) + 1)

    @torch.no_grad()
    def outer_step_subset(self, members: list[int], epoch: int | None = None) -> None:
        """Partial round: pseudo-gradient mean over ``members`` only (peer loads / stores on the symmetric window with a
        member list - absent workers are neither waited for nor read), Nesterov on this rank's full outer state."""
        sa = self.sa
        g = sa._sgd_hparams()
        self.wait_momentum()
        arr = (c_int * len(members))(*members)
        rc = _lib.cuda_lib().odb_fused_outer_subset(
            sa.theta_outer.data_ptr(), sa.momentum_buffer.data_ptr(), sa.theta_local.data_ptr(),
            sa.shadow_local.data_ptr() if sa.shadow_local is not None else None, self.window.data_ptr(), self._win_ptrs,
            self._flag_ptrs, arr, len(members), self.rank, self.world, self.n, float(g["lr"]), float(g["momentum"]),
            int(bool(g.get("nesterov", False))), self._seq_for(epoch) + 2, int(self.delta_bf16), self.timeout_flag.data_ptr(),
            _lib.stream_ptr(sa.theta_outer))
        _lib.check(rc, "fused_outer_subset")
        _lib.count_launch()
        self._arm_timeout_probe()
        sa.fv.gather_compute_weights()

    @torch.no_grad()
    def outer_step(self, epoch: int | None = None, replicated: bool = False) -> None:
        """One full round.  ``replicated``: every rank applies the mean pseudo-gradient to ITS OWN theta_outer / momentum
        (pipelined or phase-sequential kernel) - the form a drifted swarm needs, because a state-averaging round follows and
        must see each worker's own update (hivemind semantics); the sharded form would hand everybody the slab owner's
        state instead."""
        sa = self.sa
        g = sa._sgd_hparams()
        lib = _lib.cuda_lib()
        seq = self._seq_for(epoch)
        if replicated:
            self.wait_momentum()
        if self.sharded and not replicated:
            self.wait_momentum()            # the previous background all-gather reads the slab this launch rewrites
            self.launch_idx_sh += 1
            self.fingerprint.zero_()
            rc = lib.odb_fused_outer_sharded(
                sa.theta_outer.data_ptr(), sa.momentum_buffer.data_ptr(), sa.theta_local.data_ptr(),
                sa.shadow_local.data_ptr() if sa.shadow_local is not None else None, self._theta_mc, self._flag_ptrs,
                self.rank, self.world, self.n, float(g["lr"]), float(g["momentum"]), int(bool(g.get("nesterov", False))),
                seq, self.launch_idx_sh, self.nchunk_sh, int(os.environ.get("ODB_OUTER_COMM_CTAS", 0)),
                self.counters_sh.data_ptr(), self.timeout_flag.data_ptr(), self.fingerprint.data_ptr(),
                self.stamps.data_ptr() if self.stamps is not None else None, _lib.stream_ptr(sa.theta_outer))
            _lib.check(rc, "fused_outer_sharded")
            _lib.count_launch()
            self._arm_timeout_probe()
            self._regather_pending = True
            sa.fv.gather_compute_weights()
            return
        if self.pipelined:
            self.launch_idx += 1
            rc = lib.odb_fused_outer_pipelined(
                sa.theta_outer.data_ptr(), sa.momentum_buffer.data_ptr(), sa.theta_local.data_ptr(),
                sa.shadow_local.data_ptr() if sa.shadow_local is not None else None, self.window.data_ptr(), self.mc_ptr,
                self._flag_ptrs, self.rank, self.world, self.n, float(g["lr"]), float(g["momentum"]),
                int(bool(g.get("nesterov", False))), seq, self.launch_idx, self.nchunk,
                int(os.environ.get("ODB_OUTER_COMM_CTAS", 0)), int(self.delta_bf16), self.counters.data_ptr(),
                self.timeout_flag.data_ptr(), _lib.stream_ptr(sa.theta_outer))
            _lib.check(rc, "fused_outer_pipelined")
            _lib.count_launch()
            self._arm_timeout_probe()
            sa.fv.gather_compute_weights()
            return
        rc = lib.odb_fused_outer_step(
            sa.theta_outer.data_ptr(), sa.momentum_buffer.data_ptr(), sa.theta_local.data_ptr(),
            sa.shadow_local.data_ptr() if sa.shadow_local is not None else None, self.window.data_ptr(),
            self.mc_ptr if self.mc_ptr else None, self._win_ptrs, self._flag_ptrs, self.rank, self.world, self.n,
            float(g["lr"]), float(g["momentum"]), int(bool(g.get("nesterov", False))), seq, int(self.delta_bf16),
            self.timeout_flag.data_ptr(), int(os.environ.get("ODB_OUTER_P1_CTAS", 0)), int(os.environ.get("ODB_OUTER_MM_WEAK", 1)),
            self.stamps.data_ptr() if self.stamps is not None else None, _lib.stream_ptr(sa.theta_outer))
        _lib.check(rc, "fused_outer_step")
        _lib.count_launch()
        self._arm_timeout_probe()
        sa.fv.gather_compute_weights()

    # ------------------------------------------------------------------ background re-replication of the momentum
    def start_momentum_regather(self) -> None:
        """Sharded form only: every owner publishes its momentum slab to the peers with ONE all-gather on a side stream,
        overlapped with the next inner steps (the critical path of the outer step never touches foreign momentum)."""
        if not (self.sharded and self._regather_pending):
            return
        self._regather_pending = False
        buf = self.sa.momentum_buffer
        cur = torch.cuda.current_stream(buf.device)
        self._side.wait_stream(cur)
        with torch.cuda.stream(self._side):
            dist.all_gather_into_tensor(buf, buf[self.rank * self.slab:(self.rank + 1) * self.slab], group=self.group)

    def wait_momentum(self) -> None:
        """Make the current stream see the fully replicated momentum (no-op unless a re-gather is in flight)."""
        if self._side is not None:
            if self._regather_pending:
                self.start_momentum_regather()
            torch.cuda.current_stream(self.sa.momentum_buffer.device).wait_stream(self._side)

    # ------------------------------------------------------------------ time-out reporting
    def _arm_timeout_probe(self) -> None:
        self._tf_host.copy_(self.timeout_flag, non_blocking=True)
        if self._tf_event is None:
            self._tf_event = torch.cuda.Event()
        self._tf_event.record()

    def poll_timeout(self, block: bool = False) -> None:
        """Raise if the last fused round gave up waiting for a peer (the kernel then left theta / momentum untouched, but
        the swarm is out of step: the caller must not train on).  Non-blocking unless ``block``."""
        ev = self._tf_event
        if ev is None:
            return
        if block:
            ev.synchronize()
        elif not ev.query():
            return
        self._tf_event = None
        if int(self._tf_host[0]) != 0:
            raise RuntimeError("fused outer step: a peer did not reach the NVLink barrier within ODB_OUTER_TIMEOUT_S "
                               "(worker lost?); the outer update was NOT applied - restart from the last checkpoint or "
                               "run with --hv.fused-collective false")

    def phase_times_us(self) -> dict | None:
        if self.stamps is None:
            return None
        t = self.stamps.cpu().tolist()
        if self.sharded:
            return {"entry_barrier": (t[1] - t[0]) / 1e3, "owner_ctas(reduce+update+multicast)": (t[2] - t[1]) / 1e3,
                    "post_cta_end_after_owner_end": (t[3] - t[2]) / 1e3, "total(block0 start -> post end)": (t[3] - t[0]) / 1e3}
        return {"phase0_delta": (t[1] - t[0]) / 1e3, "barrier0": (t[2] - t[1]) / 1e3, "phase1_reduce_bcast": (t[3] - t[2]) / 1e3,
                "barrier1": (t[4] - t[3]) / 1e3, "phase2_nesterov(block0)": (t[5] - t[4]) / 1e3}

    def check_timeout(self) -> bool:
        return bool(self.timeout_flag.item())

    def close(self) -> None:
        self.window = self.flags = None


def try_make_fused_outer(opt, compression=None):
    """Return a FusedOuterStep bound to ``opt``, or None when the fused path is unavailable (no CUDA / NCCL group, library
    built without the kernels, symmetric memory not supported): the caller then uses the flat NCCL transport."""
    return FusedOuterStep.try_create(opt, compression)
