"""In-tree build of the C-ABI library (nvcc, sm_90a only).

`python -m unispeech_b200.build` compiles every `csrc/*.cu` into `unispeech_b200/lib/libunispeech_b200.so`.
nvcc cross-compiles without a GPU.
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
LIBDIR = PKG / "lib"
BUILD = PKG.parent / "build"
LIB = LIBDIR / "libunispeech_b200.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    cand = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return cand if os.path.exists(cand) else "nvcc"


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    srcs = sorted(CSRC.glob("*.cu"))
    hdrs = sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h")) + sorted((PKG.parent / "include").glob("*.h"))
    stamp = LIBDIR / ".build_digest"
    dig = _digest(srcs + hdrs)
    if not force and LIB.exists() and stamp.exists() and stamp.read_text() == dig:
        return LIB
    LIBDIR.mkdir(exist_ok=True)
    BUILD.mkdir(exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src: Path) -> Path:
        obj = BUILD / (src.stem + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
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
    tmp = BUILD / (LIB.name + ".tmp")  # linked aside and renamed: a reader (or a repo snapshot) never sees a half-written library
    cmd = [nvcc, "-shared", "-o", str(tmp), *map(str, objs), "-cudart", "static"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    os.replace(tmp, LIB)
    stamp.write_text(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
