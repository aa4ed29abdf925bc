"""In-tree build of libwkb200.so (nvcc, sm_90a only) and of the test-only C oracles.

`python -m whisperkit_b200.build` or `__graft_entry__.build()`.  nvcc cross-compiles without a GPU.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
BUILD = os.path.join(PKG, "_build")
LIB = os.path.join(PKG, "libwkb200.so")
SOURCES = ["gemm_wgmma.cu", "attention_wgmma.cu", "mel.cu", "encoder_ops.cu", "decoder_ops.cu", "cross_attention_mq.cu", "align_pass.cu", "engine.cu", "session.cu", "longform.cu", "wordtiming.cu", "tokenizer.cu", "writers.cu", "comm.cu", "audio.cu", "flac.cu", "streaming.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "--use_fast_math=false",
]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(p.encode())
            h.update(f.read())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "wkb200.h")]
    stamp = os.path.join(BUILD, "stamp")
    dig = _digest(deps)
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    nvcc = _nvcc()
    flags = [f for f in NVCC_FLAGS if not f.startswith("--use_fast_math")]

    def compile_one(src):
        obj = os.path.join(BUILD, src.replace(".cu", ".o"))
        cmd = [nvcc, *flags, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [nvcc, "-shared", "-o", LIB, *objs, "-lcudart", "-lz", "-ldl", "-Xlinker", "-rpath=$ORIGIN"]
    # cudart is linked dynamically: torch ships the same major runtime; curand device headers are header-only
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


def build_hostcheck() -> str:
    """CPU replay library of the mel kernel's task functions (test infrastructure)."""
    src = os.path.join(ROOT, "tests", "hostcheck", "mel_hostcheck.cpp")
    out = os.path.join(ROOT, "tests", "hostcheck", "libmel_hostcheck.so")
    deps = [src, os.path.join(CSRC, "mel_core.cuh"), os.path.join(CSRC, "mel_tables.h")]
    if os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps):
        return out
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"hostcheck build failed:\n{r.stderr}")
    return out


def build_flac_hostcheck(sanitize: bool = False, out_dir: str | None = None) -> str:
    """CPU build of csrc/flac_core.cuh (test infrastructure): libflac_hostcheck.so for ctypes, or with sanitize=True an executable built
    with -fsanitize=address,undefined (written to out_dir) that decodes the files named on its command line."""
    src = os.path.join(ROOT, "tests", "hostcheck", "flac_hostcheck.cpp")
    deps = [src, os.path.join(CSRC, "flac_core.cuh")]
    if sanitize:
        out = os.path.join(out_dir or BUILD, "flac_hostcheck_asan")
        cmd = ["g++", "-O1", "-g", "-std=c++17", "-DFLAC_HOSTCHECK_MAIN", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
               "-o", out, src]
    else:
        out = os.path.join(out_dir or os.path.join(ROOT, "tests", "hostcheck"), "libflac_hostcheck.so")
        cmd = ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src]
    if os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps):
        return out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"flac hostcheck build failed:\n{r.stderr}")
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_hostcheck())
    print(build_flac_hostcheck())
