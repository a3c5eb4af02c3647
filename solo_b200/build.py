"""Build libsolo_b200.so (sm_90a, H100) in-tree with nvcc.  No JIT cache, no arch fall-backs."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRCS = [os.path.join(HERE, "csrc", f) for f in ("solo_b200.cu", "sb_analysis.cu")]
OUT = os.path.join(HERE, "libsolo_b200.so")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-fmad=false",            # decoder float path and the three IEEE ops of the encoder must not be contracted
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-shared", "-t", "2",
]


def sources():
    d = os.path.join(HERE, "csrc")
    return [os.path.join(d, f) for f in sorted(os.listdir(d)) if f.endswith((".cu", ".cuh", ".inc"))] + [
        os.path.join(os.path.dirname(HERE), "include", f) for f in ("solo_b200.h", "AGR_JC1_SDK_API.h")] + [
        os.path.abspath(__file__)]     # the flags live here: a library built with other flags (another arch) is stale


def up_to_date():
    if not os.path.exists(OUT):
        return False
    t = os.path.getmtime(OUT)
    return all(os.path.getmtime(s) <= t for s in sources())


def build(force=False, verbose=True, extra=(), out=None):
    """extra: additional nvcc flags (e.g. -DSB_ANALYSIS_WARP=1); out: build a variant somewhere else."""
    if not force and not extra and not out and up_to_date():
        return OUT
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: libsolo_b200.so cannot be built (there is no CPU fallback)")
    cmd = [nvcc] + NVCC_FLAGS + list(extra) + SRCS + ["-o", out or OUT]
    if verbose:
        print("[solo_b200] " + " ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd)
    return out or OUT


if __name__ == "__main__":
    ex = [a for a in sys.argv[1:] if a.startswith("-D")]
    o = [a[2:] for a in sys.argv[1:] if a.startswith("-o")]
    build(force="--force" in sys.argv, extra=ex, out=(o[0] if o else None))
