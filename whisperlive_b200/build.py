"""Build whisperlive_b200/libwlb200.so (sm_90a only) with nvcc.  In-tree so the .so travels to
the GPU box with the repository snapshot.  `python -m whisperlive_b200.build [--force] [--verbose]`"""
from __future__ import annotations

import concurrent.futures as cf
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libwlb200.so")
SOURCES = ["gemm.cu", "dec_gemm.cu", "wgemm.cu", "mel.cu", "elementwise.cu", "attention.cu", "flash_attn.cu", "search.cu", "prefill.cu", "misc.cu", "vad.cu", "spk.cu", "mt.cu", "engine.cu", "vad_engine.cu", "spk_engine.cu", "hooks.cu", "mt_engine.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "--expt-relaxed-constexpr",
         "-Xcompiler", "-fPIC"]


def _deps():
    files = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "wlb200.h")]
    return max(os.path.getmtime(f) for f in files)


def build(force: bool = False, verbose: bool = False, timeline: bool = False) -> str:
    """timeline=True (or WLB200_TL_BUILD=1) compiles the in-graph timeline stamps in (tools/timeline.py): a profiling
    build, never the shipped one."""
    timeline = timeline or bool(os.environ.get("WLB200_TL_BUILD"))
    if not force and not timeline and os.path.exists(OUT) and os.path.getmtime(OUT) >= _deps():
        return OUT
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    extra = ["-Xptxas", "-v"] if verbose else []
    if timeline:
        extra.append("-DWLB200_TL=1")

    def compile_one(src):
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [NVCC, *FLAGS, *extra, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with cf.ThreadPoolExecutor(max_workers=8) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [NVCC, "-shared", "-o", OUT, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv, timeline="--timeline" in sys.argv))
