"""In-tree build of libmerlot_b200.so with plain nvcc for sm_90a (no torch extension machinery).

`python -m merlot_b200.build` compiles every csrc/*.cu to an object (in parallel, only when stale) and links
merlot_b200/libmerlot_b200.so.  Objects and the .so are build products and stay out of git.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
OBJ = HERE / "csrc" / "build"
LIB = HERE / "libmerlot_b200.so"

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-I", str(HERE.parent / "include"),
]


def _digest(src: Path) -> str:
    h = hashlib.sha1()
    for f in sorted(list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh")) + [src, HERE.parent / "include" / "merlot_b200.h"]):
        h.update(f.read_bytes())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(src: Path, verbose: bool) -> Path:
    obj = OBJ / (src.stem + ".o")
    stamp = OBJ / (src.stem + ".sha1")
    dig = _digest(src)
    if obj.exists() and stamp.exists() and stamp.read_text() == dig:
        return obj
    cmd = [NVCC, *FLAGS, "-c", str(src), "-o", str(obj)]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
    if verbose and r.stderr:
        print(r.stderr)
    stamp.write_text(dig)
    return obj


def build(verbose: bool = False, force: bool = False) -> Path:
    OBJ.mkdir(parents=True, exist_ok=True)
    if force:
        for f in OBJ.glob("*.sha1"):
            f.unlink()
    srcs = sorted(CSRC.glob("*.cu"))
    if not srcs:
        raise RuntimeError("no CUDA sources found")
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), srcs))
    newest = max(o.stat().st_mtime for o in objs)
    if (not LIB.exists()) or LIB.stat().st_mtime < newest or force:
        cmd = [NVCC, "-shared", "-o", str(LIB), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a",
               "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    p = build(verbose="-v" in sys.argv, force="-f" in sys.argv)
    print(p)
