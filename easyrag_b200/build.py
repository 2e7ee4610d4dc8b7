"""Builds the CUDA extension in-tree: easyrag_b200/_lib/libeasyrag_b200.so (sm_90a only).

``python -m easyrag_b200.build`` or ``__graft_entry__.build()``.  nvcc cross-compiles
without a GPU; the .so is git-ignored but travels to the GPU box with the tree.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
OUT_DIR = PKG / "_lib"
LIB = OUT_DIR / "libeasyrag_b200.so"
STAMP = OUT_DIR / "build.stamp"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--cudart", "static",
    "-Xptxas", "-v",
]


def _sources():
    return sorted(CSRC.glob("*.cu")) + sorted((CSRC / "encoder").glob("*.cu"))


def _digest() -> str:
    h = hashlib.sha256()
    files = _sources() + sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h")) \
        + sorted((CSRC / "encoder").glob("*.cuh")) + [PKG.parent / "include" / "easyrag_b200.h", Path(__file__)]
    for f in files:
        h.update(f.name.encode())
        h.update(f.read_bytes())
    return h.hexdigest()


def nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def build(force: bool = False, verbose: bool = False) -> Path:
    OUT_DIR.mkdir(exist_ok=True)
    extra = os.environ.get("EZR_NVCC_DEFS", "").split()       # e.g. "-DEZR_BM25_RANGE=4096" for tuning experiments
    if extra:
        return _build_variant(extra, verbose)
    digest = _digest()
    if not force and LIB.exists() and STAMP.exists() and STAMP.read_text().strip() == digest:
        return LIB
    objs = []
    procs = []
    for src in _sources():
        obj = OUT_DIR / (src.stem + ".o")
        cmd = [nvcc(), *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    failed = False
    for src, obj, pr in procs:
        out, _ = pr.communicate()
        log.append(f"==== {src.name}\n{out}")
        if pr.returncode != 0:
            failed = True
        objs.append(str(obj))
    (OUT_DIR / "build.log").write_text("\n".join(log))
    if failed:
        sys.stderr.write("\n".join(log))
        raise RuntimeError("nvcc failed; see easyrag_b200/_lib/build.log")
    if verbose:
        print("\n".join(log))
    link = [nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "--cudart", "static",
            "-Xcompiler", "-fPIC", "-o", str(LIB), *objs]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    STAMP.write_text(digest)
    return LIB


def _build_variant(extra, verbose):
    """Tuning builds: compile with extra -D flags into _lib/variant_<tag>/ (select with EASYRAG_B200_LIB)."""
    tag = hashlib.sha256(" ".join(extra).encode()).hexdigest()[:8]
    vdir = OUT_DIR / f"variant_{tag}"
    vdir.mkdir(exist_ok=True)
    lib = vdir / "libeasyrag_b200.so"
    cmd = [nvcc(), *[f for f in NVCC_FLAGS if f not in ("-Xptxas", "-v")], *extra, "-shared", "-o", str(lib),
           *[str(x) for x in _sources()]]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("variant build failed")
    return lib


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
