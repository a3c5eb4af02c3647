"""ctypes binding of _ref/libjc1_fix_enc.so (enc_ref.c): whole packets through the reference encoder with what its linker
taps recorded of the voice-activity detector and the high-band gain stage, packet by packet.

TEST INFRASTRUCTURE ONLY.  PACKET_REC mirrors EncPacketRec of enc_ref.c; the constructor compares its size with the
library's."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "_ref", "libjc1_fix_enc.so")
FR, NV, HB_SF, MAXB = 160, 28, 80, 1024

PACKET_REC = np.dtype([
    ("low", "<i2", (2, FR)), ("vad_before", "<i4", (2, NV)), ("vad_after", "<i4", (2, NV)),
    ("sa_Q8", "<i4", 2), ("snr_Q7", "<i4", 2), ("quality_Q15", "<i4", (2, 4)), ("tilt_Q15", "<i4", 2),
    ("res_Q10", "<i4", (2, FR)), ("hb_lsp_idx", "<i4", 2), ("hb_exc", "<i2", (2, 4, HB_SF)),
    ("hb_gain", "<i4", (2, 4)), ("hb_gain_idx", "<i4", (2, 4)),
    ("n_vad", "<i4"), ("n_res", "<i4"), ("n_lsp", "<i4"), ("n_gain", "<i4"),
    ("ret", "<i4"), ("nbytes", "<i4", 2), ("no_speech_counter", "<i4"), ("in_dtx", "<i4"),
    ("payload", "u1", MAXB)], align=True)


def available():
    return os.path.exists(LIB)


class RefEnc:
    def __init__(self, path=LIB):
        if not os.path.exists(path):
            raise FileNotFoundError(path + " missing: run `make -C oracle` (needs the reference sources)")
        self.L = L = C.CDLL(path, mode=os.RTLD_LOCAL if hasattr(os, "RTLD_LOCAL") else 0)
        L.encref_sizes.argtypes = [C.c_void_p]
        L.encref_run.argtypes = [C.c_int] * 7 + [C.c_void_p, C.c_void_p]
        s = np.zeros(1, np.int32)
        L.encref_sizes(s.ctypes.data_as(C.c_void_p))
        assert int(s[0]) == PACKET_REC.itemsize, "enc_ref.c record is %d bytes, oracle/enc_ref.py %d" % (int(s[0]), PACKET_REC.itemsize)

    def run(self, pcm, rate=13600, dtx=0, framesize_ms=40, joint=0, mdi=0, loss=0):
        """pcm [npk, 16 * framesize_ms] int16 from a freshly initialised encoder on -> records [npk] (PACKET_REC)."""
        pcm = np.ascontiguousarray(pcm, np.int16)
        assert pcm.shape[1] == 16 * framesize_ms, pcm.shape
        rec = np.zeros(len(pcm), PACKET_REC)
        r = self.L.encref_run(rate, dtx, framesize_ms, joint, mdi, loss, len(pcm), pcm.ctypes.data, rec.ctypes.data)
        assert r == 0, "the reference refused the settings"
        return rec
