"""ctypes driver of tests/_hostsim/libsb_hostsim_core.so: the core-output decoder of 32 kHz streams (dec_core.cpp, the
body of sb_decode_kernel<16, true> compiled by g++).

TEST INFRASTRUCTURE ONLY, like sim.py, whose SimDecoder this mirrors."""
import ctypes as C
import os

import numpy as np

from . import build_hostsim
from .sim import ARITH

SRC = os.path.join(build_hostsim.HERE, "dec_core.cpp")
_lib = None


def build(force=False):
    """tests/_hostsim/libsb_hostsim_core.so, with the flags of the host model's other builds."""
    return build_hostsim._build("libsb_hostsim_core.so", [SRC], build_hostsim.LIB_FLAGS, force)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.hs_dec_core_create.restype = C.c_void_p
        L.hs_dec_core_create.argtypes = [C.c_int] * 4
        L.hs_dec_core_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        L.hs_dec_core_destroy.argtypes = [C.c_void_p]
        _lib = L
    return _lib


class SimCoreDecoder:
    """One 32 kHz stream decoded to its 16 kHz core: rows of 16 * framesize_ms samples.  Same call shapes as
    sim.SimDecoder."""

    def __init__(self, use_md_index=0, framesize_ms=40, joint_hb=0, arith="flp"):
        self.L = lib()
        self.h = self.L.hs_dec_core_create(use_md_index, framesize_ms, joint_hb, ARITH[arith])
        assert self.h
        self.pcm = np.zeros(16 * framesize_ms, np.int16)
        self.fl = np.zeros(1, np.uint8)
        self.flags = 0      # the activity flags of the last packet: bit f VAD flag, bit 2 + f concealed; 0 if rejected

    def decode(self, payload, nbytes, lostflag):
        buf = np.zeros(max(len(payload), 1), np.uint8)
        buf[:len(payload)] = np.frombuffer(payload, np.uint8)
        nb = np.array([nbytes[0], nbytes[1]], np.int16)
        r = self.L.hs_dec_core_decode(self.h, self.pcm.ctypes.data, buf.ctypes.data, len(buf), nb.ctypes.data, int(lostflag),
                                      self.fl.ctypes.data)
        self.flags = int(self.fl[0])
        return self.pcm.copy(), r

    def close(self):
        if self.h:
            self.L.hs_dec_core_destroy(self.h)
            self.h = None
