"""In-tree build of the sm_90a CUDA extension (`metamorph_b200/_C.so`).

nvcc cross-compiles without a GPU; the resulting shared library exports a plain C ABI
(see include/metamorph_b200.h) and is loaded with ctypes by `metamorph_b200._lib`.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
BUILD = PKG.parent / "build" / "obj"
SO = PKG / "_C.so"

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]   # H100 (Hopper): wgmma / setmaxnreg need the "a" target
NVCC_FLAGS = [
    *ARCH,
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "--expt-relaxed-constexpr",
]
# No --use_fast_math: fast intrinsics (__expf, ex2.approx) are used explicitly where they are safe.


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _digest(src: Path, flags) -> str:
    h = hashlib.sha256()
    h.update(" ".join(flags).encode())
    h.update(src.read_bytes())
    for hdr in sorted(CSRC.glob("*.cuh")):
        h.update(hdr.read_bytes())
    return h.hexdigest()[:16]


def _compile_one(src: Path, verbose: bool) -> Path:
    flags = list(NVCC_FLAGS)
    obj = BUILD / f"{src.stem}.{_digest(src, flags)}.o"
    if obj.exists():
        return obj
    for old in BUILD.glob(f"{src.stem}.*.o"):
        old.unlink()
    cmd = [_nvcc(), *flags, "-Xptxas", "-v", "-c", str(src), "-o", str(obj)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{res.stdout}\n{res.stderr}")
    (BUILD / f"{src.stem}.ptxas.log").write_text(res.stderr)
    if verbose:
        print(f"[build] compiled {src.name}", flush=True)
    return obj


def build(verbose: bool = True, force: bool = False) -> Path:
    """Compile every csrc/*.cu for sm_90a and link metamorph_b200/_C.so."""
    BUILD.mkdir(parents=True, exist_ok=True)
    srcs = sorted(CSRC.glob("*.cu"))
    if force:
        for o in BUILD.glob("*.o"):
            o.unlink()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile_one(s, verbose), srcs))
    stamp = BUILD / "link.stamp"
    sig = " ".join(o.name for o in objs)
    if SO.exists() and stamp.exists() and stamp.read_text() == sig and not force:
        return SO
    cmd = [_nvcc(), "-shared", *ARCH, "-o", str(SO),
           *map(str, objs), "-cudart", "static"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    stamp.write_text(sig)
    if verbose:
        print(f"[build] linked {SO}", flush=True)
    return SO


if __name__ == "__main__":
    build(verbose=True, force="--force" in sys.argv)
