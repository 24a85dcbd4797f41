"""In-tree build of libance_b200.so (sm_90a only) and of the CPU oracle library.

nvcc cross-compiles without a GPU, so this runs in the CPU-only build container; the resulting
``ance_b200/lib/*.so`` files are git-ignored but travel to the GPU box with the snapshot.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "ance_b200" / "csrc"
LIBDIR = ROOT / "ance_b200" / "lib"
OBJDIR = ROOT / "build" / "obj"
LIB = LIBDIR / "libance_b200.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3,-pthread",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libance_b200.so cannot be built (there is no CPU fallback)")


def _sources():
    return sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cpp")))


def _headers():
    return sorted(list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + list((ROOT / "include").glob("*.h")))


def _stale(target: Path, deps) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(d.stat().st_mtime > t for d in deps)


def build_cuda(force: bool = False, verbose: bool = False) -> Path:
    """Serialised across processes by an flock on build/.lock: when the .so is missing every rank of a torchrun job
    lands here at once, and they must not write the same object / .so.tmp files concurrently.  The first one builds,
    the others find the library up to date when they get the lock."""
    import fcntl
    LIBDIR.mkdir(parents=True, exist_ok=True)
    OBJDIR.mkdir(parents=True, exist_ok=True)
    with open(OBJDIR.parent / ".lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            return _build_cuda_locked(force, verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_cuda_locked(force: bool, verbose: bool) -> Path:
    srcs, hdrs = _sources(), _headers()
    if not force and not _stale(LIB, srcs + hdrs + [Path(__file__)]):
        return LIB
    nvcc = _nvcc()

    def compile_one(src: Path) -> Path:
        obj = OBJDIR / (src.stem + ".o")
        if force or _stale(obj, [src] + hdrs + [Path(__file__)]):
            cmd = [nvcc, *NVCC_FLAGS, "-x", "cu", "-c", str(src), "-o", str(obj)]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
            if verbose:
                sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    tmp = LIB.with_suffix(".so.tmp")
    cmd = [nvcc, "-shared", "-o", str(tmp), *map(str, objs), "-gencode", "arch=compute_90a,code=sm_90a",
           "-Xcompiler", "-pthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    os.replace(tmp, LIB)
    return LIB


def build_oracle(force: bool = False) -> Path | None:
    """Compile oracle/'s C restatement (test infrastructure only — never loaded by the product)."""
    odir = ROOT / "oracle"
    src = odir / "flat_ip_oracle.c"
    if not src.exists():
        return None
    out = odir / "_build" / "liboracle.so"
    out.parent.mkdir(parents=True, exist_ok=True)
    if force or _stale(out, [src]):
        cmd = ["gcc", "-O3", "-mavx2", "-mfma", "-fopenmp", "-shared", "-fPIC", "-o", str(out), str(src), "-lm"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"gcc failed for oracle:\n{r.stdout}\n{r.stderr}")
    return out


if __name__ == "__main__":
    print(build_cuda(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_oracle(force="--force" in sys.argv))
