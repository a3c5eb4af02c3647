"""Build the host (g++) compilation of the per-stream kernel source -- CPU test infrastructure only."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from solo_b200 import build as sb_build  # noqa: E402

OUT_DIR = os.path.join(ROOT, "tests", "_hostsim")
OUT = os.path.join(OUT_DIR, "libsb_hostsim.so")
SRC = os.path.join(HERE, "hostsim.cpp")


def build(force=False, emu=False):
    """emu=True: the cooperative (32 threads per stream) build of the analysis stage, libsb_hostsim_emu.so;
    emu="gw16": the same with the quantiser code in its two-lane-groups-per-warp packing, libsb_hostsim_emu16.so."""
    if emu == "gw16":
        return _build(os.path.join(OUT_DIR, "libsb_hostsim_emu16.so"), ["-DSB_EMU", "-DSB_EMU_GW16"], force)
    if emu:
        return _build(os.path.join(OUT_DIR, "libsb_hostsim_emu.so"), ["-DSB_EMU"], force)
    return _build(OUT, [], force)


def _build(OUT, extra, force):
    os.makedirs(OUT_DIR, exist_ok=True)
    deps = sb_build.sources() + [SRC, os.path.abspath(__file__)]     # the flags live here: a flag change rebuilds
    if not force and os.path.exists(OUT) and all(os.path.getmtime(d) <= os.path.getmtime(OUT) for d in deps):
        return OUT
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-w"] + extra + [SRC, "-o", OUT])
    return OUT


if __name__ == "__main__":
    print(build(force=True))
