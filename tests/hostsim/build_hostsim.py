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
SRCS = [os.path.join(HERE, "hostsim.cpp"), os.path.join(HERE, "server.cpp")]   # the codec; the mixer and both queues


LIB_FLAGS = ["-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-w"]


def build(force=False, emu=False):
    """emu=True: the cooperative (32 threads per stream) build of the analysis stage, libsb_hostsim_emu.so;
    emu="gw16": the same with the quantiser code in its two-lane-groups-per-warp packing, libsb_hostsim_emu16.so."""
    if emu == "gw16":
        return _build("libsb_hostsim_emu16.so", SRCS, LIB_FLAGS + ["-DSB_EMU", "-DSB_EMU_GW16"], force)
    if emu:
        return _build("libsb_hostsim_emu.so", SRCS, LIB_FLAGS + ["-DSB_EMU"], force)
    return _build("libsb_hostsim.so", SRCS, LIB_FLAGS, force)


def build_fuzzer(force=False):
    """The malformed-packet fuzzer (fuzz_dec.cpp) under AddressSanitizer and UBSan, tests/_hostsim/fuzz_dec."""
    return _build("fuzz_dec", [os.path.join(HERE, "fuzz_dec.cpp")],
                  ["-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-w"], force)


def _build(name, srcs, flags, force):
    os.makedirs(OUT_DIR, exist_ok=True)
    out = os.path.join(OUT_DIR, name)
    deps = sb_build.sources() + srcs + [os.path.abspath(__file__)]     # the flags live here: a flag change rebuilds
    if not force and os.path.exists(out) and all(os.path.getmtime(d) <= os.path.getmtime(out) for d in deps):
        return out
    subprocess.check_call(["g++"] + flags + srcs + ["-o", out])
    return out


if __name__ == "__main__":
    print(build(force=True))
