"""The host model with run-time encoder control: enc_control.cpp (hostsim.cpp + hs_enc_set_control) compiled by g++ into
tests/_hostsim/ on first use, with the flags of build_hostsim.  TEST INFRASTRUCTURE ONLY."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import build_hostsim, sim

SRC = os.path.join(build_hostsim.HERE, "enc_control.cpp")
_libs = {}


def build(emu=False):
    out = os.path.join(build_hostsim.OUT_DIR, "libsb_hostsim_control%s.so" % ("_emu" if emu else ""))
    csrc = os.path.join(build_hostsim.ROOT, "solo_b200", "csrc")
    deps = [SRC, build_hostsim.SRC] + [os.path.join(csrc, f) for f in os.listdir(csrc)]
    if not (os.path.exists(out) and all(os.path.getmtime(d) <= os.path.getmtime(out) for d in deps)):
        os.makedirs(build_hostsim.OUT_DIR, exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-w"] + (["-DSB_EMU"] if emu else [])
                              + [SRC, "-o", out])
    return out


def lib(emu=False):
    if emu not in _libs:
        L = C.CDLL(build(emu))
        L.hs_enc_create3.restype = C.c_void_p
        L.hs_enc_create3.argtypes = [C.c_int] * 5
        L.hs_enc_encode.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.hs_enc_destroy.argtypes = [C.c_void_p]
        L.hs_enc_set_control.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        if emu:
            L.hs_set_emu_nsq.argtypes = [C.c_int]
        _libs[emu] = L
    return _libs[emu]


class SimEncoder(sim.SimEncoder):
    """sim.SimEncoder on the build above, plus set_control.  emu=True: the analysis stage in its cooperative form on 32
    emulated lanes."""

    def __init__(self, rate=13600, dtx=0, use_md_index=0, cap=1024, emu=False, framesize_ms=40, joint_hb=0):
        self.L = lib(bool(emu))
        self.emu_nsq = False
        self.h = self.L.hs_enc_create3(rate, dtx, use_md_index, framesize_ms, joint_hb)
        self.samples = 16 * framesize_ms
        self.cap = cap
        self.out = np.zeros(cap, np.uint8)
        self.nb = np.zeros(6, np.int16)

    def set_control(self, rate=None, dtx=None, loss=None):
        """Rate (b/s), DTX and expected loss (%) from the next packet on, through enc_set_control; None = unchanged."""
        self.L.hs_enc_set_control(self.h, *(-1 if v is None else int(v) for v in (rate, dtx, loss)))
