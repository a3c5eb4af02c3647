"""Build tests/_gpu_ops/libsb_gpu_ops.so: the single-routine harness (ops.cu) with the library's own nvcc flags, so the
routines under test compile exactly as they do in libsolo_b200.so.  Test infrastructure only."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from solo_b200 import build as sb_build  # noqa: E402

SRC = os.path.join(HERE, "ops.cu")
OUT_DIR = os.path.join(ROOT, "tests", "_gpu_ops")
OUT = os.path.join(OUT_DIR, "libsb_gpu_ops.so")


def up_to_date():
    if not os.path.exists(OUT):
        return False
    t = os.path.getmtime(OUT)
    return all(os.path.getmtime(s) <= t for s in sb_build.sources() + [SRC, os.path.abspath(__file__)])


def build(force=False, verbose=True):
    if not force and up_to_date():
        return OUT
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: the routine harness cannot be built")
    os.makedirs(OUT_DIR, exist_ok=True)
    cmd = [nvcc] + sb_build.NVCC_FLAGS + ["-I", os.path.join(ROOT, "solo_b200", "csrc"), SRC, "-o", OUT]
    if verbose:
        print("[gpu_ops] " + " ".join(cmd), file=sys.stderr)
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv)
