"""Build the C-ABI CUDA library (``libplip_b200.so``) in-tree with nvcc for sm_90a.

Usage: ``python -m plip_b200.build [--force] [--verbose]``.  The library has no torch / python
dependency; it is loaded with ctypes (``plip_b200._lib``).  Objects are compiled in parallel and
cached by source hash under ``plip_b200/csrc/_build``.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
OBJ_DIR = CSRC / "_build"
LIB_PATH = PKG_DIR / "libplip_b200.so"
INCLUDE = PKG_DIR.parent / "include"

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]

NVCC_FLAGS = [
    *GENCODE,
    "-O3", "-std=c++17", "-lineinfo",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
    "-Xcompiler", "-fvisibility=hidden",
    "-Xptxas", "-v",
]


NVCC_FLAGS += os.environ.get("PLIP_EXTRA_NVCC_FLAGS", "").split()   # extra defines for an A/B build


def _nvcc() -> str:
    cand = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(cand).exists():
        raise RuntimeError("nvcc not found; set NVCC=/path/to/nvcc")
    return cand


def _sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _hash(src: Path) -> str:
    h = hashlib.sha256()
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(src.read_bytes())
    for hdr in sorted(list(CSRC.glob("*.cuh")) + list(INCLUDE.glob("*.h"))):
        h.update(hdr.read_bytes())
    return h.hexdigest()[:16]


def _compile_one(src: Path, verbose: bool) -> tuple[Path, str]:
    obj = OBJ_DIR / f"{src.stem}.{_hash(src)}.o"
    log = ""
    if not obj.exists():
        for old in OBJ_DIR.glob(f"{src.stem}.*.o"):
            old.unlink()
        cmd = [_nvcc(), *NVCC_FLAGS, "-I", str(INCLUDE), "-I", str(CSRC), "-c", str(src), "-o", str(obj)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        log = res.stdout + res.stderr
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{log}")
        (OBJ_DIR / f"{src.stem}.ptxas.log").write_text(log)
    return obj, log


def build(force: bool = False, verbose: bool = False) -> Path:
    OBJ_DIR.mkdir(parents=True, exist_ok=True)
    if force:
        for o in OBJ_DIR.glob("*.o"):
            o.unlink()
    srcs = _sources()
    if not srcs:
        raise RuntimeError(f"no CUDA sources under {CSRC}")
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile_one(s, verbose), srcs))
    objs = [o for o, _ in results]
    if verbose:
        for _, log in results:
            if log:
                print(log)
    stamp = OBJ_DIR / "link.stamp"
    want = " ".join(o.name for o in objs)
    if force or not LIB_PATH.exists() or not stamp.exists() or stamp.read_text() != want:
        cmd = [_nvcc(), "-shared", *GENCODE,
               "-o", str(LIB_PATH), *map(str, objs), "-cudart", "static", "-lpthread", "-ldl", "-lrt"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"link failed:\n{res.stdout}{res.stderr}")
        stamp.write_text(want)
    return LIB_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(p)
