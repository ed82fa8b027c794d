"""In-tree build of the sm_90a native libraries.

    python -m opendiloco_b200.build            # build everything that is stale
    python -m opendiloco_b200.build --force    # rebuild

Two shared objects are produced next to this file (git-ignored build products):

  * ``_C/libodb200.so``   - every CUDA kernel (nvcc, ``-gencode arch=compute_90a,code=sm_90a -lineinfo``),
                            plain C ABI, loaded with ctypes (raw device pointers + stream handles, no pybind).
  * ``_C/libodbhost.so``  - host runtime in C++17 (safetensors reader, synthetic-token prefetcher, TCP rendezvous).

nvcc cross-compiles without a GPU, so the libraries can be built on a machine without one (``__graft_entry__.build``).
"""
from __future__ import annotations

import argparse
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
OUT = HERE / "_C"
OBJ = OUT / "obj"

NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CXX = os.environ.get("CXX") or shutil.which("g++") or "g++"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "--expt-extended-lambda",
    "-Xcompiler", "-fPIC,-fvisibility=hidden",
    "-Xptxas", "-v",
    "--threads", "2",
]


def _site_packages() -> Path:
    import sysconfig

    return Path(sysconfig.get_paths()["purelib"])


def cutlass_include_dirs() -> list[str]:
    """CUTLASS/CuTe header trees vendored in the image (used with -I by kernels that want CuTe helpers)."""
    sp = _site_packages()
    cands = [sp / "flashinfer/data/cutlass/include", sp / "tilelang/3rdparty/cutlass/include"]
    return [str(c) for c in cands if c.is_dir()][:1]


def nccl_dirs() -> tuple[str | None, str | None]:
    sp = _site_packages() / "nvidia" / "nccl"
    inc, lib = sp / "include", sp / "lib"
    return (str(inc) if inc.is_dir() else None, str(lib) if lib.is_dir() else None)


def _digest(paths: list[Path], extra: str) -> str:
    h = hashlib.sha256(extra.encode())
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    return h.hexdigest()


def _run(cmd: list[str], log: Path | None = None) -> None:
    res = subprocess.run(cmd, capture_output=True, text=True)
    if log is not None:
        log.write_text("$ " + " ".join(cmd) + "\n" + res.stdout + res.stderr)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError(f"build step failed: {' '.join(cmd[:6])} ...")


def build_cuda(force: bool = False, verbose: bool = False) -> Path:
    OUT.mkdir(exist_ok=True)
    OBJ.mkdir(exist_ok=True)
    target = OUT / "libodb200.so"
    cu = sorted(CSRC.glob("*.cu"))
    headers = sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h"))
    hdr_digest = _digest(headers, " ".join(NVCC_FLAGS))
    incs = [f"-I{CSRC}"] + [f"-I{d}" for d in cutlass_include_dirs()]
    nccl_inc, _ = nccl_dirs()
    if nccl_inc:
        incs.append(f"-I{nccl_inc}")

    def compile_one(src: Path) -> tuple[Path, bool]:
        obj = OBJ / (src.stem + ".o")
        stamp = OBJ / (src.stem + ".stamp")
        dig = _digest([src], hdr_digest)
        if not force and obj.exists() and stamp.exists() and stamp.read_text() == dig:
            return obj, False
        _run([NVCC, *NVCC_FLAGS, *incs, "-c", str(src), "-o", str(obj)], log=OBJ / (src.stem + ".log"))
        stamp.write_text(dig)
        return obj, True

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(cu)))) as ex:
        results = list(ex.map(compile_one, cu))
    objs = [o for o, _ in results]
    if force or any(c for _, c in results) or not target.exists():
        _run([NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(target), *map(str, objs),
              "-Xcompiler", "-fPIC", "-cudart", "static", "-ldl", "-lpthread"])
    if verbose:
        for src in cu:
            log = OBJ / (src.stem + ".log")
            if log.exists():
                sys.stdout.write(log.read_text())
    return target


def build_host(force: bool = False) -> Path:
    OUT.mkdir(exist_ok=True)
    OBJ.mkdir(exist_ok=True)
    target = OUT / "libodbhost.so"
    srcs = sorted((CSRC / "host").glob("*.cc"))
    if not srcs:
        return target
    dig = _digest(srcs + sorted((CSRC / "host").glob("*.h")), CXX)
    stamp = OBJ / "host.stamp"
    if not force and target.exists() and stamp.exists() and stamp.read_text() == dig:
        return target
    _run([CXX, "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-pthread", "-o", str(target),
          *map(str, srcs)])
    stamp.write_text(dig)
    return target


def build_all(force: bool = False, verbose: bool = False) -> dict[str, Path]:
    host = build_host(force)          # first: it needs only g++, so it survives on machines without nvcc (CPU CI)
    return {"cuda": build_cuda(force, verbose), "host": host}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true", help="print ptxas -v output (registers / spills / smem)")
    ap.add_argument("--host-only", action="store_true", help="build libodbhost.so only (no CUDA toolkit needed)")
    a = ap.parse_args()
    built = {"host": build_host(a.force)} if a.host_only else build_all(a.force, a.verbose)
    for k, v in built.items():
        print(f"{k}: {v} ({v.stat().st_size if v.exists() else 0} bytes)")
