"""ctypes binding of _ref/libjc1_fix_nsq.so (nsq_ref.c): the reference's quantiser SKP_Silk_NSQ_del_dec one frame at a time.

TEST INFRASTRUCTURE ONLY.  The numpy dtypes below mirror nsq_io.h, the frame / state layout shared with the host model and
the GPU harness; check_sizes() compares them with the sizes a library was compiled with."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(_HERE, "_ref")
LIB = os.path.join(REF_DIR, "libjc1_fix_nsq.so")
COV_DIR = os.path.join(REF_DIR, "cov")
COV_LIB = os.path.join(COV_DIR, "libjc1_fix_nsq.so")
FRAME = 160

FRAME_IN = np.dtype([
    ("sigtype", "<i4"), ("QuantOffsetType", "<i4"), ("Seed", "<i4"), ("NLSFInterpCoef_Q2", "<i4"),
    ("pitchL", "<i4", 4), ("Gains_Q16", "<i4", 4),
    ("DeltaGains_Q16", "<i4"), ("Lambda_Q10", "<i4"), ("LTP_scale_Q14", "<i4"),
    ("LF_shp_Q14", "<i4", 4), ("Tilt_Q14", "<i4", 4), ("HarmShapeGain_Q14", "<i4", 4),
    ("PredCoef_Q12", "<i2", (2, 10)), ("LTPCoef_Q14", "<i2", 20), ("AR2_Q13", "<i2", 64), ("x", "<i2", FRAME)])
FRAME_OUT = np.dtype([("q_md", "i1", (2, FRAME)), ("r16", "<i2", FRAME), ("Seed", "<i4")])
STATE = np.dtype([
    ("xq", "<i2", FRAME), ("sLTP_shp_Q10", "<i4", FRAME), ("sLPC_Q14", "<i4", 32), ("sAR2_Q14", "<i4", 16),
    ("sLF_AR_shp_Q12", "<i4"), ("lagPrev", "<i4"), ("prev_inv_gain_Q16", "<i4")])


def check_sizes(L):
    s = np.zeros(3, np.int32)
    L.nsq_io_sizes(s.ctypes.data_as(C.c_void_p))
    want = (FRAME_IN.itemsize, FRAME_OUT.itemsize, STATE.itemsize)
    assert tuple(int(v) for v in s) == want, "nsq_io.h layout %s differs from oracle/nsq_ref.py %s" % (tuple(s), want)


def available():
    return os.path.exists(LIB)


class RefNsq:
    def __init__(self, path=LIB):
        if not os.path.exists(path):
            raise FileNotFoundError(path + " missing: run `make -C oracle` (needs the reference sources)")
        self.L = L = C.CDLL(path, mode=os.RTLD_LOCAL if hasattr(os, "RTLD_LOCAL") else 0)
        L.nsq_io_sizes.argtypes = [C.c_void_p]
        L.nsqref_reset_state.argtypes = [C.c_void_p]
        L.nsqref_run.argtypes = [C.c_int] + [C.c_void_p] * 4
        check_sizes(L)

    def reset_state(self):
        """The three quantiser states (centre, description 1, description 2) of a freshly initialised encoder."""
        st = np.zeros(3, STATE)
        assert self.L.nsqref_reset_state(st.ctypes.data) == 0
        return st

    def run(self, st0, frames):
        """Frames [nfr] (FRAME_IN) from the states st0 [3]: (out [nfr] FRAME_OUT, states after every frame [nfr, 3])."""
        st0 = np.ascontiguousarray(st0, STATE)
        frames = np.ascontiguousarray(frames, FRAME_IN)
        assert st0.shape == (3,)
        out = np.zeros(len(frames), FRAME_OUT)
        st = np.zeros((len(frames), 3), STATE)
        assert self.L.nsqref_run(len(frames), st0.ctypes.data, frames.ctypes.data, out.ctypes.data, st.ctypes.data) == 0
        return out, st


def read_anchors():
    """{name: (source file, line)} written by oracle/Makefile next to the coverage build."""
    res = {}
    with open(os.path.join(COV_DIR, "anchors.txt")) as f:
        for row in f:
            name, src, line = row.split()
            res[name] = (src, int(line))
    return res
