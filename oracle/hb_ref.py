"""ctypes binding of _ref/libjc1_fix_hb.so (hb_ref.c): the reference's high-band frame analysis AGR_Bwe_encode_frame_FIX,
frame by frame from a freshly initialised encoder, with what its linker taps recorded.

TEST INFRASTRUCTURE ONLY.  FRAME_REC mirrors HbFrameRec of hb_ref.c; the constructor compares its size with the library's."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_ref", "libjc1_fix_hb.so")
ORDER, FMAX, BUF = 8, 320, 2 * 320 + 40
# settings of hbref_run: 40 ms packets, 20 ms packets, joint mode 1
SETTINGS = {"40ms": 0, "20ms": 1, "joint": 2}

FRAME_REC = np.dtype([
    ("nlsf_in", "<i4", ORDER), ("nlsf_q", "<i4", ORDER), ("lsp_idx", "<i4"),
    ("n_quant", "<i4"), ("n_nlsf2a", "<i4"), ("n_filter", "<i4"),
    ("coef", "<i2", (4, ORDER)), ("exc", "<i2", FMAX), ("x_hb_buf", "<i2", BUF), ("prev_nlsfq", "<i4", ORDER)], align=True)


def available():
    return os.path.exists(LIB)


class RefHb:
    def __init__(self, path=LIB):
        if not os.path.exists(path):
            raise FileNotFoundError(path + " missing: run `make -C oracle` (needs the reference sources)")
        self.L = L = C.CDLL(path, mode=os.RTLD_LOCAL if hasattr(os, "RTLD_LOCAL") else 0)
        L.hbref_sizes.argtypes = [C.c_void_p]
        L.hbref_frame_size.argtypes = [C.c_int]
        L.hbref_run.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        s = np.zeros(1, np.int32)
        L.hbref_sizes(s.ctypes.data_as(C.c_void_p))
        assert int(s[0]) == FRAME_REC.itemsize, "hb_ref.c record is %d bytes, oracle/hb_ref.py %d" % (int(s[0]), FRAME_REC.itemsize)

    def frame_size(self, setting):
        F = self.L.hbref_frame_size(SETTINGS[setting])
        assert F > 0
        return F

    def run(self, setting, high):
        """high [nfr, F] int16, the high band from a freshly initialised encoder on -> records [nfr] (FRAME_REC)."""
        high = np.ascontiguousarray(high, np.int16)
        rec = np.zeros(len(high), FRAME_REC)
        F = self.L.hbref_run(SETTINGS[setting], len(high), high.ctypes.data, rec.ctypes.data)
        assert F == high.shape[1], (F, high.shape)
        return rec
