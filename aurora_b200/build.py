"""In-tree build of libaurora_b200.so (sm_90a only; nvcc cross-compiles without a GPU).

``python -m aurora_b200.build`` or ``aurora_b200.build.build_native()``.  The .so lands
next to this file, so the package imports straight from the source tree.
"""

from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libaurora_b200.so")
SOURCES = ["capi.cu", "kernels_simt.cu", "simtopk_tc.cu", "encoder.cu", "encoder_simt.cu", "gemm_tc.cu", "attn_tc.cu", "keyword.cu", "kw_text.cu", "hybrid.cu", "listsearch.cu", "filter.cu", "tokenizer.cpp", "host_merge.cpp"]
HEADERS = ["internal.h", "ptx.cuh", "unicode_tables.inc", os.path.join("..", "..", "include", "aurora_b200.h")]

PROFILE = bool(int(os.environ.get("AUR_TC_PROFILE", "0")))   # bring-up timers in the tensor-core similarity kernel
EXTRA_DEFS = os.environ.get("AUR_EXTRA_DEFS", "").split()     # extra -D flags for an A/B build

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O2,-Wall,-Wno-unused-function",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: aurora_b200 needs the CUDA toolkit to build its sm_90a library")


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build_native(force: bool = False, verbose: bool = False, out: str = "", tag: str = "") -> str:
    """out / tag: A/B builds (``AUR_EXTRA_DEFS=... python -m aurora_b200.build --out lib_b.so --tag b``) land beside
    the product library and are selected at run time with AURORA_B200_LIB."""
    lib = os.path.join(HERE, out) if out else LIB
    if not out and not force and not _stale():
        return LIB
    nvcc = _nvcc()
    objs = []
    for src in SOURCES:
        obj = os.path.join(CSRC, os.path.splitext(src)[0] + (f".{tag}" if tag else "") + ".o")
        cmd = [nvcc, *NVCC_FLAGS, *(["-DAUR_TC_PROFILE"] if PROFILE else []), *EXTRA_DEFS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd), flush=True)
        subprocess.run(cmd, check=True)
        objs.append(obj)
    cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", *objs, "-o", lib, "-cudart", "static"]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.run(cmd, check=True)
    return lib


if __name__ == "__main__":
    def _opt(name):
        return sys.argv[sys.argv.index(name) + 1] if name in sys.argv else ""
    print(build_native(force="--force" in sys.argv, verbose="-v" in sys.argv, out=_opt("--out"), tag=_opt("--tag")))
