"""ctypes binding of the UNMODIFIED reference codec built by oracle/Makefile into oracle/_ref/.

TEST INFRASTRUCTURE ONLY.  Only tests/ and __graft_entry__.smoke() import this module (bench.py runs the
reference's own executable).  Nothing under solo_b200/ does.

API bound: JC1_SDK_SRC_{ARM,FLP}/interface/AGR_JC1_SDK_API.h:33-64 (six functions).
Internal reference functions (exported by the .so because they are non-static C) are reachable
through ``RefLib.lib`` for unit-level parity tests of individual primitives.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(_HERE, "_ref")


class EncCtrl(C.Structure):
    # AGR_JC1_SDK_API.h:11-21
    _fields_ = [(n, C.c_int32) for n in ("mode", "targetRate_bps", "samplerate", "dtx_enable",
                                         "framesize_ms", "joint_enable", "joint_mode", "useMDIndex")]


class DecCtrl(C.Structure):
    # AGR_JC1_SDK_API.h:23-31
    _fields_ = [(n, C.c_int32) for n in ("packetLoss_perc", "samplerate", "framesize_ms",
                                         "joint_enable", "joint_mode", "useMDIndex")]


class SilkEncControl(C.Structure):
    # SKP_SILK_SDK_EncControlStruct (interface/SKP_Silk_control.h:41-69): nine ints
    _fields_ = [(n, C.c_int32) for n in ("API_sampleRate", "maxInternalSampleRate", "packetSize", "bitRate", "packetLossPercentage",
                                         "complexity", "useInBandFEC", "useDTX", "useMDIndex")]


class SateEncHead(C.Structure):
    # the leading fields of SATEEncCtl (libBWE/AGR_BWE_structs.h:61-67): SILK state, high-band state, SILK control
    _fields_ = [("stEnc", C.c_void_p), ("stHBEnc", C.c_void_p), ("encControl", SilkEncControl)]


def available():
    return all(os.path.exists(os.path.join(REF_DIR, f)) for f in ("libjc1_fix.so", "libjc1_flp.so"))


def lowband_available():
    """The decoders with a tap on their low band (oracle/lowband.mk) are built."""
    return all(os.path.exists(os.path.join(REF_DIR, "libjc1_%s_lowband.so" % k)) for k in ("flp", "fix"))


class RefLib:
    def __init__(self, kind="fix"):
        path = os.path.join(REF_DIR, "libjc1_%s.so" % kind)
        if not os.path.exists(path):
            raise FileNotFoundError(path + " missing: run `make -C oracle` (needs /root/reference)")
        self.lib = L = C.CDLL(path, mode=os.RTLD_LOCAL if hasattr(os, "RTLD_LOCAL") else 0)
        L.AGR_Sate_Encoder_Init.restype = C.c_void_p
        L.AGR_Sate_Encoder_Init.argtypes = [C.POINTER(EncCtrl)]
        L.AGR_Sate_Encoder_Encode.restype = C.c_int32
        L.AGR_Sate_Encoder_Encode.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
        L.AGR_Sate_Encoder_Uninit.argtypes = [C.c_void_p]
        L.AGR_Sate_Decoder_Init.restype = C.c_void_p
        L.AGR_Sate_Decoder_Init.argtypes = [C.POINTER(DecCtrl)]
        L.AGR_Sate_Decoder_Decode.restype = C.c_int32
        L.AGR_Sate_Decoder_Decode.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32]
        L.AGR_Sate_Decoder_Uninit.argtypes = [C.c_void_p]


_libs = {}


def lib(kind):
    if kind not in _libs:
        _libs[kind] = RefLib(kind)
    return _libs[kind]


class RefEncoder:
    """One reference encoder handle (kind = 'fix' | 'flp') at the API sample rate `samplerate` (16000 or 32000)."""

    def __init__(self, kind="fix", rate=13600, dtx=0, use_md_index=0, framesize_ms=40, joint_hb=0, samplerate=16000):
        self.kind = kind
        self.L = lib(kind).lib
        self.samples = samplerate // 1000 * framesize_ms
        self.ctrl = EncCtrl(2, rate, samplerate, dtx, framesize_ms, 1 if joint_hb else 0, 1 if joint_hb else 0, use_md_index)
        self.h = self.L.AGR_Sate_Encoder_Init(C.byref(self.ctrl))
        self._bits = (C.c_uint8 * 1024)()
        self._nb = (C.c_int16 * 6)()

    def encode(self, pcm_packet):
        pcm = np.ascontiguousarray(pcm_packet, dtype=np.int16)
        assert pcm.size == self.samples
        C.memset(self._nb, 0, 12)
        n = self.L.AGR_Sate_Encoder_Encode(self.h, pcm.ctypes.data, self._bits, 1024, self._nb)
        return bytes(self._bits[:max(n, 0)]), (int(self._nb[0]), int(self._nb[1])), n

    def head(self):
        return C.cast(C.c_void_p(self.h), C.POINTER(SateEncHead)).contents

    def set_control(self, rate=None, dtx=None, loss=None):
        """From the next packet on: target rate (b/s, less 1600 -- or 800 with joint mode 1 -- as Init computes bitRate,
        AGR_BWE_SDK_API.c:118), useDTX, packetLossPercentage.  None leaves a field as it is.

        The SDK sets these three once, in AGR_Sate_Encoder_Init (AGR_BWE_SDK_API.c:38-119), but its SILK core re-reads them
        from the handle's encControl at the start of every packet (SKP_Silk_enc_API.c:161-191), so writing them into a live
        handle the way Init does makes the reference follow a settings schedule.  The handle description above
        (SateEncHead) has only been checked against the FIX library, by tests/test_enc_control.py; the FLP build keeps its
        own SILK structures, so an "flp" handle is refused rather than written through an unchecked layout."""
        if self.kind != "fix":
            raise ValueError("set_control: only the FIX library's handle layout is known")
        c = self.head().encControl
        if rate is not None:
            c.bitRate = int(rate) - (800 if self.ctrl.joint_enable and self.ctrl.joint_mode == 1 else 1600)
        if dtx is not None:
            c.useDTX = int(dtx)
        if loss is not None:
            c.packetLossPercentage = int(loss)

    def close(self):
        if self.h:
            self.L.AGR_Sate_Encoder_Uninit(self.h)
            self.h = None

    __del__ = close


class RefDecoder:
    """One reference decoder handle (kind = 'flp' is the PCM parity target, 'fix' the fixed-point build) at the API sample
    rate `samplerate` (16000 or 32000).

    out_samplerate = 16000 for a 32 kHz stream: the same decoder in the build with a tap on its low band (oracle/lowband.mk).
    decode() then returns the int16 low band the packet handed to the synthesis filter bank (AGR_Sate_qmf_synth's first
    argument, 16 * framesize_ms samples), or an empty row when the filter bank did not run (a rejected packet); `full` keeps
    that call's full-band PCM.  The tap records one low band per library, so decode calls into one tapped library must not
    overlap."""

    def __init__(self, kind="flp", use_md_index=0, framesize_ms=40, joint_hb=0, samplerate=16000, out_samplerate=None):
        out_samplerate = samplerate if out_samplerate is None else out_samplerate
        self.tapped = (samplerate, out_samplerate) == (32000, 16000)
        if out_samplerate != samplerate and not self.tapped:
            raise ValueError("no decoder of %d Hz streams with %d Hz output" % (samplerate, out_samplerate))
        self.L = lib(kind + "_lowband" if self.tapped else kind).lib
        self.ns_want = samplerate // 1000 * framesize_ms
        self.samples = out_samplerate // 1000 * framesize_ms
        self.ctrl = DecCtrl(0, samplerate, framesize_ms, 1 if joint_hb else 0, 1 if joint_hb else 0, use_md_index)
        self.h = self.L.AGR_Sate_Decoder_Init(C.byref(self.ctrl))
        self._out = np.zeros(samplerate // 1000 * 60, dtype=np.int16)
        self._ns = C.c_int16(0)
        if self.tapped:
            self.L.lowband_take.argtypes = [C.c_void_p, C.c_int]
            self._low = np.zeros(self.samples, np.int16)
            self.L.lowband_take(self._low.ctypes.data, self._low.size)

    def decode(self, payload, nbytes, lostflag):
        """payload/nbytes pre-trimmed by the caller as dec_main.c:245-307 does; returns (PCM, return value)."""
        buf = (C.c_uint8 * 1024)(*payload) if payload else (C.c_uint8 * 1024)()
        nb = (C.c_int16 * 6)(int(nbytes[0]), int(nbytes[1]))
        ret = self.L.AGR_Sate_Decoder_Decode(self.h, self._out.ctypes.data, C.byref(self._ns), buf, nb, int(lostflag))
        assert ret != 0 or self._ns.value == self.ns_want, (self._ns.value, self.ns_want)
        if not self.tapped:
            return self._out[:self.samples].copy(), ret
        self.full = self._out[:self.ns_want].copy()
        n = self.L.lowband_take(self._low.ctypes.data, self._low.size)
        assert n in (0, self.samples), n
        return self._low[:n].copy(), ret

    def close(self):
        if self.h:
            self.L.AGR_Sate_Decoder_Uninit(self.h)
            self.h = None

    __del__ = close
