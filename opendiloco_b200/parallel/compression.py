"""Pseudo-gradient compression codecs + the compressed "butterfly" all-reduce.

The reference offers hivemind's codecs through ``--hv.hivemind-compression`` (train_fsdp.py:87,299; utils.py:83-121):
fp16, scaled-fp16, uniform8bit, quantile8bit, blockwise8bit.  hivemind's all-reduce splits the vector across peers,
each part is compressed, streamed to its owner, averaged there in fp32, compressed again and streamed back
(SURVEY.md E9/E10).  ``Codec.all_reduce_mean_`` is that algorithm on NVLink:

    all_to_all(compressed parts)  ->  owner dequantises + averages N parts in fp32  ->  compress  ->  all_gather

so the wire carries 2 or 1 bytes per element instead of 4, and the averaging itself stays fp32.  8-bit quantisation /
dequantisation run as CUDA kernels (``csrc/quant.cu``); CPU tensors use the equivalent torch ops (gloo path, tests).
"""
from __future__ import annotations

import ctypes

import torch
import torch.distributed as dist

from .. import _lib

c_void_p, c_int, c_ll, c_float = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float
for _name, _sig in {
    "odb_quant_blockwise8": [c_void_p, c_void_p, c_void_p, c_ll, c_void_p],
    "odb_dequant_blockwise8": [c_void_p, c_void_p, c_void_p, c_ll, c_float, c_int, c_void_p],
    "odb_quant_affine8": [c_void_p, c_void_p, c_ll, c_void_p, c_void_p],
    "odb_quant_bucket8": [c_void_p, c_void_p, c_ll, c_void_p, c_void_p],
    "odb_bucket_stats": [c_void_p, c_void_p, c_ll, c_void_p, c_void_p, c_void_p],
    "odb_dequant_lookup8": [c_void_p, c_void_p, c_void_p, c_ll, c_float, c_int, c_void_p],
}.items():
    _lib.register_optional(_name, _sig)

QBLOCK = 4096
FP16_MAX = 65504.0


def _call(name: str, *args) -> None:
    _lib.check(getattr(_lib.cuda_lib(), name)(*args), name)
    _lib.count_launch()


class Codec:
    """compress(x fp32 [n]) -> (payload tensor, meta fp32 tensor) ; decompress_into(payload, meta, out, alpha, accumulate)."""

    name = "none"
    is_identity = True
    payload_dtype = torch.float32
    meta_len = 0          # fp32 metadata elements per compressed part

    def meta_size(self, n: int) -> int:
        return self.meta_len

    def compress(self, x: torch.Tensor):
        return x, x.new_empty(0)

    def decompress_into(self, payload, meta, out, alpha: float = 1.0, accumulate: bool = False) -> None:
        if accumulate:
            out.add_(payload.to(torch.float32), alpha=alpha)
        else:
            out.copy_(payload)
            if alpha != 1.0:
                out.mul_(alpha)

    # ------------------------------------------------------------------------------------------ butterfly all-reduce
    @torch.no_grad()
    def all_reduce_mean_(self, flat: torch.Tensor, group) -> torch.Tensor:
        """In-place mean of ``flat`` (fp32, 1-D) across ``group`` with compressed transport."""
        N = dist.get_world_size(group)
        if N == 1:
            return flat
        n = flat.numel()
        part = (n + N - 1) // N
        part = (part + QBLOCK - 1) // QBLOCK * QBLOCK
        padded = flat if part * N == n else torch.cat([flat, flat.new_zeros(part * N - n)])
        msz = self.meta_size(part)
        send_p = torch.empty(N * part, dtype=self.payload_dtype, device=flat.device)
        send_m = torch.empty(N * max(msz, 1), dtype=torch.float32, device=flat.device)
        for r in range(N):
            p, m = self.compress(padded[r * part:(r + 1) * part])
            send_p[r * part:(r + 1) * part].copy_(p.reshape(-1))
            if msz:
                send_m[r * msz:(r + 1) * msz].copy_(m)
        recv_p, recv_m = torch.empty_like(send_p), torch.empty_like(send_m)
        dist.all_to_all_single(_as_wire(recv_p), _as_wire(send_p), group=group)
        dist.all_to_all_single(recv_m, send_m, group=group)
        mine = torch.zeros(part, dtype=torch.float32, device=flat.device)
        for r in range(N):
            self.decompress_into(recv_p[r * part:(r + 1) * part], recv_m[r * msz:(r + 1) * msz] if msz else recv_m[:0], mine,
                                 alpha=1.0 / N, accumulate=r > 0)
        p, m = self.compress(mine)
        all_p = torch.empty(N * part, dtype=self.payload_dtype, device=flat.device)
        all_m = torch.empty(N * max(msz, 1), dtype=torch.float32, device=flat.device)
        dist.all_gather_into_tensor(_as_wire(all_p), _as_wire(p.reshape(-1).contiguous()), group=group)
        dist.all_gather_into_tensor(all_m, m if msz else all_m.new_zeros(1), group=group)
        for r in range(N):
            lo, hi = r * part, min((r + 1) * part, n)
            if lo >= n:
                break
            tmp = padded[lo:lo + part]
            self.decompress_into(all_p[r * part:(r + 1) * part], all_m[r * msz:(r + 1) * msz] if msz else all_m[:0], tmp)
            if padded is not flat:
                flat[lo:hi].copy_(tmp[:hi - lo])
        return flat


def _as_wire(t: torch.Tensor) -> torch.Tensor:
    """int8 payloads travel as uint8 (collectives on every backend accept it)."""
    return t.view(torch.uint8) if t.dtype == torch.int8 else t


class NoCompression(Codec):
    pass


class Float16Compression(Codec):
    """Clamp to the fp16 range and cast (hivemind Float16Compression)."""

    name, is_identity, payload_dtype = "fp16", False, torch.float16

    def compress(self, x):
        return x.clamp(-FP16_MAX, FP16_MAX).to(torch.float16), x.new_empty(0)

    def decompress_into(self, payload, meta, out, alpha=1.0, accumulate=False):
        if accumulate:
            out.add_(payload.to(torch.float32), alpha=alpha)
        else:
            out.copy_(payload.to(torch.float32))
            if alpha != 1.0:
                out.mul_(alpha)


class BFloat16Compression(Float16Compression):
    """fp32 -> bf16 cast: the precision BASELINE.json names for the fused outer kernel; fusable into it."""

    name, payload_dtype, fusable = "bf16", torch.bfloat16, True

    def compress(self, x):
        return x.to(torch.bfloat16), x.new_empty(0)


class ScaledFloat16Compression(Codec):
    """Per-block (4096) mean/std normalisation, then fp16 (hivemind ScaledFloat16Compression, row-wise there)."""

    name, is_identity, payload_dtype = "scaled-fp16", False, torch.float16

    def meta_size(self, n):
        return 2 * (n // QBLOCK)

    def compress(self, x):
        v = x.view(-1, QBLOCK)
        mean = v.mean(dim=1, keepdim=True)
        std = (v - mean).pow(2).mean(dim=1, keepdim=True).sqrt().clamp_min(1e-12)
        q = ((v - mean) / std).clamp(-FP16_MAX, FP16_MAX).to(torch.float16)
        return q.reshape(-1), torch.cat([mean.reshape(-1), std.reshape(-1)])

    def decompress_into(self, payload, meta, out, alpha=1.0, accumulate=False):
        nb = payload.numel() // QBLOCK
        mean, std = meta[:nb, None], meta[nb:2 * nb, None]
        val = (payload.view(nb, QBLOCK).to(torch.float32) * std + mean).reshape(-1)
        out.add_(val, alpha=alpha) if accumulate else out.copy_(val * alpha if alpha != 1.0 else val)


class _Lookup8(Codec):
    """uint8 codes + a 256-entry code book of bucket means."""

    is_identity, payload_dtype, meta_len = False, torch.uint8, 256

    def _codes(self, x) -> torch.Tensor:
        raise NotImplementedError

    def compress(self, x):
        x = x.contiguous()
        q = self._codes(x)
        sums = torch.zeros(256, dtype=torch.float32, device=x.device)
        cnts = torch.zeros(256, dtype=torch.int32, device=x.device)          # exact past 2^24 members per bucket
        if x.is_cuda:
            _call("odb_bucket_stats", x.data_ptr(), q.data_ptr(), x.numel(), sums.data_ptr(), cnts.data_ptr(), _lib.stream_ptr(x))
        else:
            qi = q.long()
            sums.index_add_(0, qi, x)
            cnts.index_add_(0, qi, torch.ones_like(qi, dtype=torch.int32))
        return q, sums / cnts.clamp_min(1.0)

    def decompress_into(self, payload, meta, out, alpha=1.0, accumulate=False):
        if out.is_cuda:
            _call("odb_dequant_lookup8", payload.data_ptr(), meta.data_ptr(), out.data_ptr(), out.numel(), float(alpha),
                  int(accumulate), _lib.stream_ptr(out))
        else:
            val = meta[payload.long()] * alpha
            out.add_(val) if accumulate else out.copy_(val)


class Uniform8BitQuantization(_Lookup8):
    """256 uniform buckets over +-6 sigma around the mean (hivemind Uniform8BitQuantization: RANGE_IN_SIGMAS = 6)."""

    name = "uniform8bit"
    RANGE_IN_SIGMAS = 6

    def _codes(self, x):
        mean = x.mean()
        std = (x - mean).pow(2).mean().sqrt()
        scale = self.RANGE_IN_SIGMAS * std / 256
        q = torch.empty(x.numel(), dtype=torch.uint8, device=x.device)
        if x.is_cuda:
            ms = torch.stack([mean, scale]).to(torch.float32)
            _call("odb_quant_affine8", x.data_ptr(), q.data_ptr(), x.numel(), ms.data_ptr(), _lib.stream_ptr(x))
        else:
            inv = 1.0 / scale if float(scale) > 0 else 0.0
            q.copy_((torch.round((x - mean) * inv) + 128).clamp(0, 255).to(torch.uint8))
        return q


class Quantile8BitQuantization(_Lookup8):
    """256 equal-mass buckets; borders = quantiles of a strided sample (hivemind Quantile8BitQuantization)."""

    name = "quantile8bit"
    SAMPLE = 1 << 20

    def _codes(self, x):
        n = x.numel()
        sample = x[:: max(1, n // self.SAMPLE)].float()
        probs = torch.linspace(0, 1, 257, device=x.device, dtype=torch.float32)[1:-1]
        srt = sample.sort().values
        idx = (probs * (srt.numel() - 1)).round().long()
        borders = srt[idx].contiguous()
        q = torch.empty(n, dtype=torch.uint8, device=x.device)
        if x.is_cuda:
            _call("odb_quant_bucket8", x.data_ptr(), q.data_ptr(), n, borders.data_ptr(), _lib.stream_ptr(x))
        else:
            q.copy_(torch.bucketize(x, borders, right=True).to(torch.uint8))
        return q


class BlockwiseQuantization(Codec):
    """8-bit block-wise absmax quantisation, block 4096 (hivemind BlockwiseQuantization -> bitsandbytes)."""

    name, is_identity, payload_dtype = "blockwise8bit", False, torch.int8

    def meta_size(self, n):
        return n // QBLOCK

    @staticmethod
    def _check_blocks(n: int) -> None:
        # one absmax per whole block: a partial block would have no slot for its scale
        if n % QBLOCK:
            raise ValueError(f"blockwise8bit works on whole {QBLOCK}-element blocks; got {n} elements")

    def compress(self, x):
        x = x.contiguous()
        n = x.numel()
        self._check_blocks(n)
        q = torch.empty(n, dtype=torch.int8, device=x.device)
        absmax = torch.empty(n // QBLOCK, dtype=torch.float32, device=x.device)
        if x.is_cuda:
            _call("odb_quant_blockwise8", x.data_ptr(), q.data_ptr(), absmax.data_ptr(), n, _lib.stream_ptr(x))
        else:
            v = x.view(-1, QBLOCK)
            absmax.copy_(v.abs().amax(dim=1))
            inv = torch.where(absmax > 0, 127.0 / absmax, torch.zeros_like(absmax))
            q.copy_(torch.round(v * inv[:, None]).to(torch.int8).reshape(-1))
        return q, absmax

    def decompress_into(self, payload, meta, out, alpha=1.0, accumulate=False):
        payload = payload.view(torch.int8)
        self._check_blocks(out.numel())
        if out.is_cuda:
            _call("odb_dequant_blockwise8", payload.data_ptr(), meta.data_ptr(), out.data_ptr(), out.numel(), float(alpha),
                  int(accumulate), _lib.stream_ptr(out))
        else:
            val = (payload.view(-1, QBLOCK).float() * (meta[:, None] * (alpha / 127.0))).reshape(-1)
            out.add_(val) if accumulate else out.copy_(val)


_CODECS = {
    None: NoCompression, "none": NoCompression, "fp16": Float16Compression, "bf16": BFloat16Compression,
    "scaled-fp16": ScaledFloat16Compression, "uniform8bit": Uniform8BitQuantization,
    "quantile8bit": Quantile8BitQuantization, "blockwise8bit": BlockwiseQuantization,
}


def get_compression(name: str | None) -> Codec:
    if name not in _CODECS:
        raise ValueError(f"Invalid hivemind_compression: {name}")
    return _CODECS[name]()


def get_compression_kwargs(hivemind_compression: str | None) -> dict:
    """kwargs for DiLoCoOptimizer from the ``--hv.hivemind-compression`` flag (reference utils.py:83-121)."""
    return {"grad_compression": get_compression(hivemind_compression),
            "state_averaging_compression": get_compression(hivemind_compression)}
