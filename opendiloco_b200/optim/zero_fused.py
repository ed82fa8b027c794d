"""Host side of the fused ZeRO step (``csrc/zero_comm.cu``): the optimizer step of a sharded DiLoCo worker as one kernel.

The fp32 gradient arena and the bf16 compute-weight arena are re-homed into NVLink symmetric-memory windows of the
worker's inner group (``torch.distributed._symmetric_memory`` is plumbing only: allocation, handle exchange, peer mapping,
multicast binding).  The kernel then does reduce-scatter (``multimem.ld_reduce``), global-norm clip, AdamW on the rank's
slab and the all-gather of the new bf16 weights (``multimem.st``) in a single launch - no ``ncclDevKernel_ReduceScatter`` /
``AllGather`` is left in a training step (reference call sites: FSDP SHARD_GRAD_OP, train_fsdp.py:239-245,395,403).
"""
from __future__ import annotations

import ctypes
import os

import torch
import torch.distributed as dist

from .. import _lib
from ..utils.logger import get_logger

c_void_p, c_int, c_ll, c_uint = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_uint
_lib.register_optional("odb_zero_fused_step", [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                              c_int, c_int, c_ll, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                              c_uint, c_void_p, c_void_p])
_lib.register_optional("odb_zero_set_timeout_ms", [c_int])
logger = get_logger()
MAX_PEERS = 16


class FusedZeroStep:
    def __init__(self, opt):
        import torch.distributed._symmetric_memory as symm_mem

        fv, group = opt.fv, opt.dp_group
        self.opt, self.group = opt, group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        n = fv.flat.numel()
        if n % (8 * self.world):
            raise ValueError("flat buffer not divisible into 8-element aligned slabs")
        dev = fv.flat.device
        gname = group.group_name
        try:
            if hasattr(symm_mem, "is_symm_mem_enabled_for_group") and not symm_mem.is_symm_mem_enabled_for_group(gname):
                symm_mem.enable_symm_mem_for_group(gname)
        except Exception:
            pass
        grad = symm_mem.empty(n, dtype=torch.float32, device=dev)
        h_grad = symm_mem.rendezvous(grad, gname)
        grad_mc = int(getattr(h_grad, "multicast_ptr", 0) or 0)
        if not grad_mc:
            raise RuntimeError("no multicast address for the gradient window (NVLS unavailable)")
        self.shadow_mode, self._shadow_ptr = 0, None
        shadow = h_shadow = None
        if fv.param_sharded:
            self.shadow_mode = 2                                     # FULL_SHARD: bf16 shard stays local
        elif fv.shadow is not None and fv.shadow.dtype == torch.bfloat16:
            shadow = symm_mem.empty(n, dtype=torch.bfloat16, device=dev)
            h_shadow = symm_mem.rendezvous(shadow, gname)
            mc = int(getattr(h_shadow, "multicast_ptr", 0) or 0)
            if not mc:
                raise RuntimeError("no multicast address for the compute-weight window")
            self.shadow_mode, self._shadow_ptr = 1, mc
        flags = symm_mem.empty(3 * MAX_PEERS, dtype=torch.int32, device=dev)
        xchg = symm_mem.empty(2 * MAX_PEERS, dtype=torch.float32, device=dev)
        flags.zero_()
        xchg.zero_()
        h_flags, h_xchg = symm_mem.rendezvous(flags, gname), symm_mem.rendezvous(xchg, gname)
        # ---- nothing failed: re-home the arenas
        fv.rehome_grad(grad)
        if shadow is not None:
            fv.rehome_shadow(shadow)
        self.grad, self.h_grad, self.grad_mc = grad, h_grad, grad_mc
        self.shadow, self.h_shadow = shadow, h_shadow
        self.flags, self.xchg, self.h_flags, self.h_xchg = flags, xchg, h_flags, h_xchg
        PtrArr = c_void_p * self.world
        self._flag_ptrs = PtrArr(*[int(p) for p in h_flags.buffer_ptrs])
        self._xchg_ptrs = PtrArr(*[int(p) for p in h_xchg.buffer_ptrs])
        self.n = n
        self.partials = torch.zeros(2048, dtype=torch.float32, device=dev)
        self.bcast = torch.zeros(2, dtype=torch.float32, device=dev)
        self.timeout_flag = torch.zeros(1, dtype=torch.int32, device=dev)
        self._tf_host = torch.zeros(1, dtype=torch.int32, pin_memory=True)
        self._tf_event = None
        self.seq = 1
        lib = _lib.cuda_lib()
        if _lib.has_symbol("odb_zero_set_timeout_ms"):
            lib.odb_zero_set_timeout_ms(int(float(os.environ.get("ODB_OUTER_TIMEOUT_S", 20.0)) * 1e3))
        torch.cuda.synchronize(dev)
        h_flags.barrier()
        logger.info(f"fused ZeRO step: {self.world} GPUs per worker, gradient window {n * 4 / 1e6:.0f} MB fp32, compute weights "
                    f"{['fp32 (gathered by NCCL)', 'bf16 multicast', 'bf16 local shard (FULL_SHARD)'][self.shadow_mode]}")

    @classmethod
    def try_create(cls, opt):
        fv = opt.fv
        if (opt.dp_group is None or not fv.sharded or not fv.flat.is_cuda or os.environ.get("ODB_ZERO_FUSED", "1") == "0"
                or dist.get_backend(opt.dp_group) != "nccl" or not _lib.has_symbol("odb_zero_fused_step")):
            return None
        try:
            return cls(opt)
        except Exception as e:      # symmetric memory / multicast unavailable: NCCL reduce-scatter + kernel + all-gather
            logger.warning(f"fused ZeRO step unavailable ({type(e).__name__}: {e}); using NCCL reduce-scatter / all-gather")
            return None

    @torch.no_grad()
    def step(self, hp: torch.Tensor, check_inf: bool, found_inf: torch.Tensor, skipped: torch.Tensor, stats: torch.Tensor) -> None:
        opt, fv = self.opt, self.opt.fv
        self.poll_timeout(block=False)
        if self.shadow_mode == 1:
            sh = self._shadow_ptr
        elif self.shadow_mode == 2:
            sh = fv.own_shadow().data_ptr()
        else:
            sh = None
        found_inf.zero_()
        rc = _lib.cuda_lib().odb_zero_fused_step(
            fv.own(fv.flat).data_ptr(), opt.exp_avg.data_ptr(), opt.exp_avg_sq.data_ptr(), fv.grad.data_ptr(), self.grad_mc, sh,
            self.shadow_mode, self._flag_ptrs, self._xchg_ptrs, self.rank, self.world, self.n, hp.data_ptr(),
            self.partials.data_ptr(), self.bcast.data_ptr(), int(check_inf), found_inf.data_ptr(), skipped.data_ptr(),
            stats.data_ptr(), self.seq, self.timeout_flag.data_ptr(), _lib.stream_ptr(fv.flat))
        _lib.check(rc, "zero_fused_step")
        _lib.count_launch()
        self.seq += 1
        self._tf_host.copy_(self.timeout_flag, non_blocking=True)
        if self._tf_event is None:
            self._tf_event = torch.cuda.Event()
        self._tf_event.record()
        if self.shadow_mode == 0:
            fv.gather_compute_weights()

    def poll_timeout(self, block: bool = False) -> None:
        ev = self._tf_event
        if ev is None:
            return
        if block:
            ev.synchronize()
        elif not ev.query():
            return
        self._tf_event = None
        if int(self._tf_host[0]) != 0:
            raise RuntimeError("fused ZeRO step: a GPU of this worker did not reach the NVLink barrier in time; the update was "
                               "not applied (set ODB_ZERO_FUSED=0 to use the NCCL path)")
