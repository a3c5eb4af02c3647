"""ctypes driver of tests/_hostsim/librx_timing.so: the receive queue's timing rules (solo_b200/csrc/sb_rx.cuh) compiled by
g++ from tests/hostsim/rx_timing.cpp.

TEST INFRASTRUCTURE ONLY: the CPU tests check it against a direct statement of RFC 3550, the GPU tests check the kernels
against it bit for bit; the product (libsolo_b200.so) never links or loads it."""
import ctypes as C
import os

import numpy as np

from . import build_hostsim

SRC = os.path.join(build_hostsim.HERE, "rx_timing.cpp")


def build(force=False):
    """tests/_hostsim/librx_timing.so, rebuilt when the kernel source or rx_timing.cpp is newer."""
    return build_hostsim._build("librx_timing.so", SRC, build_hostsim.LIB_FLAGS, force)


_rx = None


def rx_lib():
    """tests/_hostsim/librx_timing.so, loaded once."""
    global _rx
    if _rx is None:
        L = C.CDLL(build())
        L.rx_model_timing.argtypes = [C.c_int, C.c_int, C.c_uint32] + [C.c_void_p] * 12 + [C.c_int, C.c_int64]
        _rx = L
    return _rx


class SimRxTiming:
    """The timing state of a timed receive queue of n streams (solo_b200_rx_enable_timing), advanced by rx_model_timing:
    the kernels' per-arrival rules of sb_rx.cuh applied in array order."""

    def __init__(self, n, desc_cap, ts_per_index):
        self.L, self.n, self.desc_cap, self.ts = rx_lib(), int(n), int(desc_cap), int(ts_per_index)
        self.transit = np.zeros(n, np.uint32)
        self.jitter = np.zeros(n, np.uint32)          # 1/16 units, as the device keeps it
        self.highest = np.zeros(n, np.uint64)
        self.received = np.zeros(n, np.uint32)
        self.margin = np.zeros((n, 8), np.uint32)

    def insert(self, last, stream, index, desc, off, lens, arrival, payload_bytes):
        """One timed insert's timing, with `last` the queue's last played indices (uint32 [n]) at the call."""
        a = [np.ascontiguousarray(x, t) for x, t in ((last, np.uint32), (stream, np.int32), (index, np.uint32),
                                                     (desc, np.uint8), (off, np.int32), (lens, np.int32),
                                                     (arrival, np.uint32))]
        assert a[0].shape == (self.n,)
        self.L.rx_model_timing(self.n, self.desc_cap, self.ts, a[0].ctypes.data, self.transit.ctypes.data,
                               self.jitter.ctypes.data, self.highest.ctypes.data, self.received.ctypes.data,
                               self.margin.ctypes.data, *(x.ctypes.data for x in a[1:]), len(a[1]), int(payload_bytes))

    def reset(self, streams):
        for x in (self.transit, self.jitter, self.highest, self.received, self.margin):
            x[np.asarray(streams, np.int64)] = 0

    def read(self):
        """(jitter >> 4, highest, received, margin), as solo_b200_rx_timing reports them."""
        return self.jitter >> 4, self.highest.copy(), self.received.copy(), self.margin.copy()
