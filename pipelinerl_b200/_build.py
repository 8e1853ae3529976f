"""In-tree build of libprl.so (hand-written sm_90a CUDA behind the C ABI in include/prl.h).

nvcc cross-compiles for sm_90a without a GPU.  The .so is written next to the
package (pipelinerl_b200/_lib/libprl.so) so that it travels to the GPU box with
the repository snapshot; it is git-ignored, never pip-installed.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
REPO_ROOT = PKG_DIR.parent
CSRC = PKG_DIR / "csrc"
LIB_DIR = PKG_DIR / "_lib"
OBJ_DIR = LIB_DIR / "obj"
LIB_PATH = LIB_DIR / "libprl.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC,-O3,-Wall,-Wno-unused-function",
    "-Xptxas", "-v",
    "-I", str(REPO_ROOT / "include"),
]


def _nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: libprl.so cannot be built")
    return nvcc


def _sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _digest(src: Path) -> str:
    h = hashlib.sha256()
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(src.read_bytes())
    for hdr in sorted(list(CSRC.glob("*.cuh")) + list((REPO_ROOT / "include").glob("*.h"))):
        h.update(hdr.read_bytes())
    return h.hexdigest()


def _compile_one(src: Path, verbose: bool) -> tuple[Path, bool]:
    obj = OBJ_DIR / (src.stem + ".o")
    stamp = OBJ_DIR / (src.stem + ".sha")
    dig = _digest(src)
    if obj.exists() and stamp.exists() and stamp.read_text() == dig:
        return obj, False
    cmd = [_nvcc(), *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = OBJ_DIR / (src.stem + ".ptxas.log")
    log.write_text(res.stdout + res.stderr)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError(f"nvcc failed on {src.name}")
    if verbose:
        print(f"[prl build] compiled {src.name}")
    stamp.write_text(dig)
    return obj, True


def build(force: bool = False, verbose: bool = True) -> Path:
    """Compile every csrc/*.cu for sm_90a and link pipelinerl_b200/_lib/libprl.so."""
    OBJ_DIR.mkdir(parents=True, exist_ok=True)
    if force:
        for f in OBJ_DIR.glob("*.sha"):
            f.unlink()
    srcs = _sources()
    if not srcs:
        raise RuntimeError("no CUDA sources found")
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile_one(s, verbose), srcs))
    objs = [o for o, _ in results]
    changed = any(c for _, c in results) or not LIB_PATH.exists()
    if changed:
        tmp = LIB_DIR / "libprl.so.tmp"
        cmd = [_nvcc(), "-shared", "-o", str(tmp), *map(str, objs),
               "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            sys.stderr.write(res.stdout + res.stderr)
            raise RuntimeError("link of libprl.so failed")
        os.replace(tmp, LIB_PATH)
        if verbose:
            print(f"[prl build] linked {LIB_PATH}")
    return LIB_PATH


if __name__ == "__main__":
    build(force="--force" in sys.argv)
