"""Build libu2b200.so (the sm_90a kernels + C ABI) in-tree with nvcc.

No JIT cache, no torch extension machinery: plain ``nvcc -c`` per translation unit (in parallel)
and one ``nvcc -shared`` link, output next to this file so it travels with the source tree.
nvcc cross-compiles without a GPU.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
REPO = PKG_DIR.parent
CSRC = PKG_DIR / "csrc"
LIB_PATH = PKG_DIR / "libu2b200.so"
BUILD_DIR = REPO / "build" / "obj"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "--expt-relaxed-constexpr",
    f"-I{REPO / 'include'}", f"-I{CSRC}",
] + [f"-D{d}" for d in os.environ.get("U2_NVCC_DEFINES", "").split() if d]


def _nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libu2b200.so")
    return nvcc


def _newest_header_mtime() -> float:
    hs = list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh")) + list((REPO / "include").glob("*.h"))
    return max((h.stat().st_mtime for h in hs), default=0.0)


def _compile_one(nvcc: str, src: Path, obj: Path, verbose: bool) -> str:
    cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
    return r.stderr


def build(force: bool = False, verbose: bool = False) -> Path:
    nvcc = _nvcc()
    BUILD_DIR.mkdir(parents=True, exist_ok=True)
    srcs = sorted(CSRC.glob("*.cu"))
    if not srcs:
        raise RuntimeError(f"no .cu sources under {CSRC}")
    hdr_m = _newest_header_mtime()
    jobs = []
    objs = []
    for s in srcs:
        o = BUILD_DIR / (s.stem + ".o")
        objs.append(o)
        if force or not o.exists() or o.stat().st_mtime < max(s.stat().st_mtime, hdr_m):
            jobs.append((s, o))
    if jobs:
        with cf.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            futs = [ex.submit(_compile_one, nvcc, s, o, verbose) for s, o in jobs]
            for f in futs:
                log = f.result()
                if verbose and log:
                    print(log, file=sys.stderr)
    need_link = force or bool(jobs) or not LIB_PATH.exists() or any(
        o.stat().st_mtime > LIB_PATH.stat().st_mtime for o in objs)
    if need_link:
        cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static",
               "-o", str(LIB_PATH), *map(str, objs)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
