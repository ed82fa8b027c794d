"""Compare the machine code of two builds of a CUDA object, kernel by kernel.

    python profiles/sass_compare.py OLD.o NEW.o [--rename REGEX REPLACEMENT ...]

Both objects are dumped with ``cuobjdump -sass``; kernel names are demangled with ``cu++filt`` and the optional
``--rename`` rules (Python regular expressions) are applied to the OLD names, so that a kernel whose template list
changed can be matched with its counterpart.  Branch labels are renumbered per kernel.  Prints every kernel that is only
in one of the two objects or whose instructions (text and encoding) differ, and exits non-zero if there is any.

Example: the GEMM family lost its cluster-size template argument (always 1) between two commits:

    python profiles/sass_compare.py old/gemm_sm90.o new/gemm_sm90.o \\
        --rename 'gemm_kernel<(.*), \\(int\\)1, (\\(int\\)\\d)>' 'gemm_kernel<\\1, \\2>'
"""
from __future__ import annotations

import argparse
import re
import shutil
import subprocess
import sys


def _tool(name: str) -> str:
    return shutil.which(name) or f"/usr/local/cuda/bin/{name}"


def kernels(obj: str) -> dict[str, list[str]]:
    sass = subprocess.run([_tool("cuobjdump"), "-sass", obj], check=True, capture_output=True, text=True).stdout
    out: dict[str, list[str]] = {}
    body: list[str] | None = None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            body = out.setdefault(m.group(1), [])
        elif body is not None and re.match(r"\s*/\*[0-9a-f]{4,}\*/|\s*/\* 0x", line):
            body.append(re.sub(r"^\s*/\*[0-9a-f]+\*/", "", line).strip())      # drop the address column
    demangled = subprocess.run([_tool("cu++filt")], input="\n".join(out), check=True, capture_output=True,
                               text=True).stdout.splitlines()
    return {d: _renumber_labels(out[m]) for m, d in zip(out, demangled)}


def _renumber_labels(body: list[str]) -> list[str]:
    seen: dict[str, str] = {}
    return [re.sub(r"\.L_x_\d+", lambda m: seen.setdefault(m.group(0), f".L{len(seen)}"), line) for line in body]


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("old")
    ap.add_argument("new")
    ap.add_argument("--rename", nargs=2, action="append", default=[], metavar=("REGEX", "REPLACEMENT"))
    args = ap.parse_args()
    old, new = kernels(args.old), kernels(args.new)
    for pat, rep in args.rename:
        old = {re.sub(pat, rep, k): v for k, v in old.items()}
    bad = 0
    for name in sorted(old.keys() | new.keys()):
        if name not in new or name not in old:
            print(f"only in {'old' if name in old else 'new'}: {name}")
            bad += 1
        elif old[name] != new[name]:
            diff = sum(a != b for a, b in zip(old[name], new[name])) + abs(len(old[name]) - len(new[name]))
            print(f"differs ({diff} of {len(old[name])} lines): {name}")
            bad += 1
    print(f"{len(old)} old, {len(new)} new kernels, {bad} not identical")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
