"""Builds libalm_b200.so (hand-written sm_90a CUDA + C ABI) in-tree with nvcc.

`python -m audiolm_pytorch_b200.build` or `__graft_entry__.build()`.  nvcc cross-compiles for
sm_90a (H100) without a GPU; the resulting .so is git-ignored and must be built on every checkout.
"""
from __future__ import annotations

import hashlib
import os
import re
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
OBJ_DIR = PKG_DIR / "_build"
LIB_PATH = PKG_DIR / "libalm_b200.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
    *os.environ.get("ALM_EXTRA_NVCC_FLAGS", "").split(),
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; libalm_b200.so cannot be built")


def _digest(path: Path, headers: list[Path]) -> str:
    h = hashlib.sha256()
    h.update(" ".join(NVCC_FLAGS).encode())
    for p in [path, *headers]:
        h.update(p.read_bytes())
    return h.hexdigest()[:16]


def _wgmma_serialised(ptxas_log: str) -> list[str]:
    """Kernels for which ptxas reports C7510 (wgmma.mma_async serialised by a call in the wgmma pipeline)."""
    found = []
    for line in ptxas_log.splitlines():
        if "C7510" in line:
            m = re.search(r"in the function '([^']+)'", line)
            found.append(m.group(1) if m else line.strip())
    return found


def sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def build(force: bool = False, verbose: bool = False) -> Path:
    nvcc = _nvcc()
    OBJ_DIR.mkdir(exist_ok=True)
    headers = sorted(CSRC.glob("*.cuh")) + sorted((PKG_DIR.parent / "include").glob("*.h"))
    jobs = []
    objs = []
    for src in sources():
        tag = _digest(src, headers)
        obj = OBJ_DIR / f"{src.stem}.{tag}.o"
        objs.append(obj)
        if force or not obj.exists():
            for stale in OBJ_DIR.glob(f"{src.stem}.*.o"):
                stale.unlink()
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = OBJ_DIR / f"{src.stem}.ptxas.log"
        log.write_text(r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        serialised = _wgmma_serialised(r.stderr)
        if serialised:
            obj.unlink()
            raise RuntimeError(
                f"{src.name}: ptxas serialises wgmma (C7510) in {', '.join(serialised)}; a function call (printf, a "
                f"non-inlined helper) inside a wgmma kernel costs every mma_async a wait. See {log}.")
        if verbose:
            print(f"[build] {src.name} ok", file=sys.stderr)
        return obj

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    if jobs or force or not LIB_PATH.exists():
        cmd = [nvcc, "-shared", "-o", str(LIB_PATH), *map(str, objs), "-cudart", "static", "-Xcompiler", "-fPIC"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose=True)
    print(p)
