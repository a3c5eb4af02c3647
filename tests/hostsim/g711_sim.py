"""ctypes driver of tests/_hostsim/libsb_g711.so: the G.711 gateway's per-stream code (solo_b200/csrc/sb_g711.cuh)
compiled by g++ (g711_model.cpp).

TEST INFRASTRUCTURE ONLY: it lets the CPU-only container check the gateway's arithmetic against the reference and the
GPU tests check the kernels against it; the product (libsolo_b200.so) never links or loads it.  Same call shapes as
solo_b200.G711Gateway."""
import ctypes as C
import os

import numpy as np

from . import build_hostsim

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "g711_model.cpp")
_lib = None


def build(force=False):
    """tests/_hostsim/libsb_g711.so, with the flags of the codec's host build; rebuilt when a source is newer."""
    return build_hostsim._build("libsb_g711.so", [SRC], build_hostsim.LIB_FLAGS, force)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        vp, ci = C.c_void_p, C.c_int
        L.g711_model_reset.argtypes = [vp, vp, ci, vp, ci]
        L.g711_model_uplink.argtypes = [vp, ci, ci] + [vp] * 6
        L.g711_model_downlink.argtypes = [vp, ci, ci, vp, vp, vp]
        L.g711_model_compress.argtypes = [ci, vp, ci, vp]
        L.g711_model_expand.argtypes = [ci, vp, ci, vp]
        _lib = L
    return _lib


def g711_compress(law, x):
    """g711_compress over int16 x under law 0 (mu-law) / 1 (A-law) -> uint8 codes."""
    x = np.ascontiguousarray(x, np.int16)
    c = np.zeros(x.shape, np.uint8)
    lib().g711_model_compress(int(law), x.ctypes.data, x.size, c.ctypes.data)
    return c


def g711_expand(law, c):
    """g711_expand over uint8 codes -> int16."""
    c = np.ascontiguousarray(c, np.uint8)
    x = np.zeros(c.shape, np.int16)
    lib().g711_model_expand(int(law), c.ctypes.data, c.size, x.ctypes.data)
    return x


class SimG711:
    """A G.711 gateway of n streams (solo_b200_g711) in the device layout of G711State, advanced by the host build of
    sb_g711.cuh."""

    def __init__(self, n, framesize_ms=40, law=0):
        self.L, self.n, self.nf, self.law = lib(), int(n), framesize_ms // 20, int(law)
        self.spp8, self.spp16 = 160 * self.nf, 320 * self.nf
        self.st = np.zeros(self.n * self.L.g711_model_state_bytes(), np.uint8)
        self.L.g711_model_reset(self.st.ctypes.data, None, self.n, None, self.law)
        self.sa_Q8 = np.zeros((self.n, self.nf), np.int32)     # each frame's speech activity in the last uplink
        self.low = np.zeros((self.n, self.spp8), np.int16)     # the low band of the last downlink, before companding

    def uplink(self, payload, lost=None):
        """payload uint8 [n, spp8], lost int32 [n] or None -> (pcm int16 [n, spp16], level uint8 [n], flags uint8 [n])."""
        g = np.ascontiguousarray(payload, np.uint8)
        assert g.shape == (self.n, self.spp8)
        lo = None if lost is None else np.ascontiguousarray(lost, np.int32)
        pcm = np.zeros((self.n, self.spp16), np.int16)
        level, flags = np.zeros(self.n, np.uint8), np.zeros(self.n, np.uint8)
        self.L.g711_model_uplink(self.st.ctypes.data, self.n, self.nf, g.ctypes.data, None if lo is None else lo.ctypes.data,
                                 pcm.ctypes.data, level.ctypes.data, flags.ctypes.data, self.sa_Q8.ctypes.data)
        return pcm, level, flags

    def downlink(self, pcm):
        """pcm int16 [n, spp16] -> payload uint8 [n, spp8]."""
        x = np.ascontiguousarray(pcm, np.int16)
        assert x.shape == (self.n, self.spp16)
        out = np.zeros((self.n, self.spp8), np.uint8)
        self.L.g711_model_downlink(self.st.ctypes.data, self.n, self.nf, x.ctypes.data, self.low.ctypes.data, out.ctypes.data)
        return out

    def reset(self, streams, law=None):
        s = np.ascontiguousarray(streams, np.int32)
        lw = None if law is None else np.ascontiguousarray(np.broadcast_to(law, s.shape), np.int32)
        self.L.g711_model_reset(self.st.ctypes.data, s.ctypes.data, len(s), None if lw is None else lw.ctypes.data, self.law)


if __name__ == "__main__":
    print(build(force=True))
