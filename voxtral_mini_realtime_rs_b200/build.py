"""In-tree build of libvoxtral_b200.so (sm_90a only: H100; nvcc cross-compiles without a GPU).

    python -m voxtral_mini_realtime_rs_b200.build [--force]

Objects are cached under csrc/build/ by source mtime; the shared library lands next to this
file, so the package imports from the source tree (both are git-ignored).
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "build")
LIB = os.path.join(HERE, "libvoxtral_b200.so")

CU_SOURCES = ["kernels.cu", "matvec_tc.cu", "decode_attn.cu", "decode_mega.cu", "enc_attn_tc.cu", "gemm_tc5.cu", "model.cu", "stream.cu", "capi.cu"]
CXX_SOURCES = ["gguf.cpp", "audio_host.cpp", "tokenizer.cpp"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=default"]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-Wall"]
# extra nvcc flags for instrumented builds (e.g. VOX_NVCC_EXTRA="-DVOX_MEGA_WARP_TRACE"); rebuild with force=True
NVCC_FLAGS += os.environ.get("VOX_NVCC_EXTRA", "").split()


def _nvcc() -> str:
    for c in ("/usr/local/cuda/bin/nvcc", "nvcc"):
        if os.path.isabs(c) and os.path.exists(c):
            return c
    return "nvcc"


def _deps(src: str):
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    hdrs.append(os.path.join(HERE, "..", "include", "voxtral.h"))
    return [src] + hdrs


def _stale(out: str, deps) -> bool:
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(d) > t for d in deps)


def _compile(src_name: str, force: bool) -> str:
    src = os.path.join(CSRC, src_name)
    obj = os.path.join(OBJ, src_name + ".o")
    if force or _stale(obj, _deps(src)):
        if src_name.endswith(".cu"):
            cmd = [_nvcc()] + NVCC_FLAGS + ["-c", src, "-o", obj]
        else:
            cmd = ["g++"] + CXX_FLAGS + ["-I/usr/local/cuda/include", "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"compile failed: {' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    return obj


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    names = CU_SOURCES + CXX_SOURCES
    with ThreadPoolExecutor(max_workers=min(len(names), os.cpu_count() or 4)) as ex:
        objs = list(ex.map(lambda n: _compile(n, force), names))
    if force or _stale(LIB, objs):
        cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ARCH + ["-lcudart_static", "-ldl", "-lrt", "-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed: {' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
    if verbose:
        print("built", LIB)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
