"""Builds libhumanrf_b200.so (sm_90a) in-tree with nvcc.  No torch involvement: the library is
a plain C-ABI shared object (include/humanrf_b200.h).  Every .cu is compiled to its own object file (in parallel,
re-done only when that file, a header or the flags change), then linked."""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libhumanrf_b200.so"
STAMP = PKG / ".libhumanrf_b200.stamp"
OBJ = PKG / "build"
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _sources():
    return sorted(CSRC.glob("*.cu"))


def _headers():
    return sorted(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "humanrf_b200.h"]


def _digest(files) -> str:
    h = hashlib.sha256()
    for f in files:
        h.update(f.name.encode())
        h.update(f.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def nvcc_path() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _compile_one(src: Path, force: bool):
    obj, stamp = OBJ / (src.stem + ".o"), OBJ / (src.stem + ".stamp")
    dig = _digest([src] + _headers())
    if not force and obj.exists() and stamp.exists() and stamp.read_text().strip() == dig:
        log = OBJ / (src.stem + ".log")
        return 0, log.read_text() if log.exists() else ""
    res = subprocess.run([nvcc_path(), *NVCC_FLAGS, "-c", "-o", str(obj), str(src)], capture_output=True, text=True)
    log = res.stdout + res.stderr
    (OBJ / (src.stem + ".log")).write_text(log)
    if res.returncode == 0:
        stamp.write_text(dig)
    return res.returncode, log


def build_library(force: bool = False, verbose: bool = False) -> Path:
    dig = _digest(_sources() + _headers())
    if not force and LIB.exists() and STAMP.exists() and STAMP.read_text().strip() == dig:
        return LIB
    OBJ.mkdir(exist_ok=True)
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(len(srcs), os.cpu_count() or 4)) as ex:
        results = list(ex.map(lambda s: _compile_one(s, force), srcs))
    log = "".join(f"==== {s.name}\n{l}" for s, (_, l) in zip(srcs, results))
    (PKG / "build.log").write_text(log)
    if any(rc != 0 for rc, _ in results):
        sys.stderr.write(log)
        raise RuntimeError("nvcc failed building libhumanrf_b200.so (see humanrf_b200/build.log)")
    tmp = LIB.with_suffix(".so.tmp")      # linked beside, then renamed: a reader never sees a half-written library
    res = subprocess.run([nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC", "-o", str(tmp),
                          *[str(OBJ / (s.stem + ".o")) for s in srcs]], capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("link of libhumanrf_b200.so failed")
    os.replace(tmp, LIB)
    if verbose:
        print(log)
    STAMP.write_text(dig)
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
