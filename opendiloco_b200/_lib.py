"""ctypes loader for the in-tree native libraries (``_C/libodb200.so`` CUDA kernels, ``_C/libodbhost.so`` host runtime).

The CUDA library is *required* whenever a CUDA device is present: there is no silent eager fallback for CUDA tensors
(``cuda_lib()`` raises).  CPU tensors take the pure-PyTorch reference path that lives next to every op (used by the CPU
test-suite and by the CPU/gloo configuration of BASELINE.json).
"""
from __future__ import annotations

import ctypes
import os
import threading
from pathlib import Path

import torch

_HERE = Path(__file__).resolve().parent
_CUDA_SO = _HERE / "_C" / "libodb200.so"
_HOST_SO = _HERE / "_C" / "libodbhost.so"

_lock = threading.Lock()
_cuda: ctypes.CDLL | None = None
_host: ctypes.CDLL | None = None

c_void_p, c_int, c_ll, c_float = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float

# name -> argtypes ; every function returns int (0 ok / cudaError / negative usage error) unless noted
_CUDA_SIGS: dict[str, list] = {
    "odb_embedding_fwd": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p],
    "odb_embedding_bwd": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p],
    "odb_rmsnorm_fwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p],
    "odb_rmsnorm_bwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p],
    "odb_rope": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p],
    "odb_swiglu_fwd": [c_void_p, c_void_p, c_ll, c_int, c_void_p],
    "odb_swiglu_bwd": [c_void_p, c_void_p, c_void_p, c_ll, c_int, c_void_p],
    "odb_cast_f32_bf16": [c_void_p, c_void_p, c_ll, c_void_p],
    "odb_add_bf16": [c_void_p, c_void_p, c_void_p, c_ll, c_void_p],
    "odb_ce_fwd_bwd": [c_void_p, c_void_p, c_int, c_int, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "odb_ce_fwd": [c_void_p, c_void_p, c_int, c_int, c_ll, c_void_p, c_void_p],
    "odb_grad_sqnorm": [c_void_p, c_ll, c_void_p, c_void_p, c_void_p],
    "odb_adamw_step": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_void_p, c_int, c_void_p,
                       c_void_p, c_void_p, c_int, c_void_p],
    "odb_pseudo_grad": [c_void_p, c_void_p, c_void_p, c_ll, c_int, c_void_p],
    "odb_nesterov_outer": [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_ll, c_float, c_float, c_int,
                           c_float, c_void_p],
}

# optional symbols: present once the corresponding .cu exists; looked up lazily
_OPTIONAL_SIGS: dict[str, list] = {}


def register_optional(name: str, argtypes: list) -> None:
    _OPTIONAL_SIGS[name] = argtypes
    if _cuda is not None and hasattr(_cuda, name):     # library already loaded: bind the prototype now
        fn = getattr(_cuda, name)
        fn.argtypes = argtypes
        fn.restype = c_int


class NativeLibraryMissing(RuntimeError):
    pass


def cuda_lib_path() -> Path:
    return _CUDA_SO


def host_lib_path() -> Path:
    return _HOST_SO


def cuda_lib() -> ctypes.CDLL:
    """Load (once) and return the CUDA kernel library; raise loudly if it is not built."""
    global _cuda
    if _cuda is not None:
        return _cuda
    with _lock:
        if _cuda is not None:
            return _cuda
        if not _CUDA_SO.exists():
            raise NativeLibraryMissing(
                f"{_CUDA_SO} is missing: run `python -m opendiloco_b200.build` (or __graft_entry__.build()). "
                "opendiloco_b200 has no eager fallback for CUDA tensors."
            )
        lib = ctypes.CDLL(str(_CUDA_SO), mode=os.RTLD_NOW | os.RTLD_LOCAL)
        for name, sig in _CUDA_SIGS.items():
            fn = getattr(lib, name)
            fn.argtypes = sig
            fn.restype = c_int
        for name, sig in _OPTIONAL_SIGS.items():
            if hasattr(lib, name):
                fn = getattr(lib, name)
                fn.argtypes = sig
                fn.restype = c_int
        _cuda = lib
        return lib


def has_symbol(name: str) -> bool:
    try:
        return hasattr(cuda_lib(), name)
    except NativeLibraryMissing:
        return False


def host_lib() -> ctypes.CDLL | None:
    global _host
    if _host is not None:
        return _host
    with _lock:
        if _host is None and _HOST_SO.exists():
            _host = ctypes.CDLL(str(_HOST_SO), mode=os.RTLD_NOW | os.RTLD_LOCAL)
        return _host


def stream_ptr(t: torch.Tensor | None = None) -> int:
    """Raw cudaStream_t of torch's current stream on the tensor's device."""
    dev = t.device if t is not None else None
    return torch.cuda.current_stream(dev).cuda_stream


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"opendiloco_b200 native call {what} failed with code {rc}")


_launch_count = 0


def count_launch(n: int = 1) -> None:
    """Book-keeping for bench.py's ``gpu_launches`` (kernels of OURS launched)."""
    global _launch_count
    _launch_count += n


def launch_count() -> int:
    return _launch_count


def reset_launch_count() -> None:
    global _launch_count
    _launch_count = 0
