"""In-tree build of the native runtime (`libdmnist_sm90a.so`).

Every CUDA source is compiled for sm_90a (H100) only
(`-gencode arch=compute_90a,code=sm_90a -lineinfo`); nvcc cross-compiles without a GPU, so this
runs on a machine without one. The shared object lands next to this file, so a built tree can be
copied to a GPU machine as it is (a JIT cache under ~/.cache would not travel with it).

    python -m dist_mnist_b200._build [--force] [--verbose]
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
BUILD_DIR = PKG_DIR.parent / "build" / "native"
LIB_NAME = "libdmnist_sm90a.so"
LIB_PATH = PKG_DIR / LIB_NAME

CUDA_SOURCES = ["gemm_sm90.cu", "head_sm90.cu", "ps_apply_sm90.cu", "p2p_sm90.cu", "fused_step_sm90.cu",
                "clip_sm90.cu", "nvls_sm90.cu", "executor.cu", "fused_exec.cu", "api.cu"]
CXX_SOURCES = ["host_runtime.cpp", "loader_api.cpp"]
HEADERS = ["common.cuh", "protocol.h", "fused.h", "loader.h", "trace.h", "lr_schedule.h", "grad_clip.cuh",
           "activation.cuh", "loss.cuh"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-diag-suppress", "550",
]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-Wall"]


def _cuda_home() -> Path:
    for cand in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if cand and (Path(cand) / "bin" / "nvcc").exists():
            return Path(cand)
    nvcc = shutil.which("nvcc")
    if nvcc:
        return Path(nvcc).resolve().parent.parent
    raise RuntimeError("nvcc not found (set CUDA_HOME)")


def _stale(target: Path, deps: list[Path]) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(d.stat().st_mtime > t for d in deps)


def _run(cmd: list[str], verbose: bool) -> None:
    if verbose:
        print(" ".join(cmd), flush=True)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"command failed ({res.returncode}): {' '.join(cmd)}\n{res.stdout}\n{res.stderr}")
    if verbose and (res.stdout or res.stderr):
        print(res.stdout, res.stderr, flush=True)


HASH_PATH = PKG_DIR / (LIB_NAME + ".srchash")


def source_hash() -> str:
    """Content hash of every source, header and the build recipe (mtimes do not survive repo snapshots)."""
    import hashlib

    h = hashlib.sha256()
    for name in sorted(CUDA_SOURCES + CXX_SOURCES + HEADERS):
        h.update(name.encode())
        h.update((CSRC / name).read_bytes())
    h.update(" ".join(NVCC_FLAGS + CXX_FLAGS).encode())
    return h.hexdigest()


def is_current() -> bool:
    return LIB_PATH.exists() and HASH_PATH.exists() and HASH_PATH.read_text().strip() == source_hash()


def build_if_stale(verbose: bool = False) -> Path:
    """Rebuild only when the sources changed since the shared object was produced (cross-process safe)."""
    if is_current():
        return LIB_PATH
    import fcntl

    BUILD_DIR.mkdir(parents=True, exist_ok=True)
    with open(BUILD_DIR / ".lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not is_current():
                build(force=True, verbose=verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB_PATH


def build(force: bool = False, verbose: bool = False, ptxas_info: bool = False) -> Path:
    """Compile (if stale) and return the path of the shared object."""
    cuda = _cuda_home()
    nvcc = str(cuda / "bin" / "nvcc")
    BUILD_DIR.mkdir(parents=True, exist_ok=True)
    headers = [CSRC / h for h in HEADERS]
    jobs = []
    objs: list[Path] = []
    for src in CUDA_SOURCES:
        s = CSRC / src
        o = BUILD_DIR / (s.stem + ".o")
        objs.append(o)
        if force or _stale(o, [s, *headers, Path(__file__)]):
            flags = list(NVCC_FLAGS) + (["-Xptxas", "-v"] if ptxas_info else [])
            jobs.append([nvcc, *flags, "-I", str(CSRC), "-c", str(s), "-o", str(o)])
    for src in CXX_SOURCES:
        s = CSRC / src
        o = BUILD_DIR / (s.stem + ".o")
        objs.append(o)
        if force or _stale(o, [s, *headers, Path(__file__)]):
            jobs.append(["g++", *CXX_FLAGS, "-I", str(CSRC), "-I", str(cuda / "include"), "-c", str(s), "-o", str(o)])
    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            list(ex.map(lambda c: _run(c, verbose or ptxas_info), jobs))
    if force or jobs or _stale(LIB_PATH, objs):
        tmp = LIB_PATH.with_suffix(".so.tmp")
        _run(
            [nvcc, "-shared", "-cudart", "shared", "-o", str(tmp), *map(str, objs),
             "-Xlinker", f"-rpath={cuda / 'lib64'}", "-lpthread", "-lrt"],
            verbose,
        )
        os.replace(tmp, LIB_PATH)
    HASH_PATH.write_text(source_hash() + "\n")
    return LIB_PATH


def main(argv: list[str]) -> int:
    force = "--force" in argv
    verbose = "--verbose" in argv
    path = build(force=force, verbose=verbose, ptxas_info="--ptxas-info" in argv)
    print(f"built {path} ({path.stat().st_size} bytes)")
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
