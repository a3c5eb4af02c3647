"""ctypes driver of tests/_hostsim/libsb_hostsim.so: the per-stream kernel source (solo_b200/csrc/*.cuh) compiled by g++.

TEST INFRASTRUCTURE ONLY.  It exists so that the CPU-only container can check the kernel arithmetic bit for bit; the
product (libsolo_b200.so) never links or loads it.  Same call shapes as oracle/ref.py so tests can swap the two."""
import ctypes as C

import numpy as np

from . import build_hostsim

_libs = {}
ARITH = {"flp": 0, "fix": 1}   # sb::DEC_FLP / sb::DEC_FIX
EMU = False   # set tests.hostsim.sim.EMU = True (or use emu=True) to drive the 32-thread cooperative build


def lib(emu=None):
    emu = EMU if emu is None else emu
    if emu not in _libs:
        L = C.CDLL(build_hostsim.build(emu=emu))
        L.hs_enc_create3.restype = C.c_void_p
        L.hs_enc_create3.argtypes = [C.c_int] * 5
        L.hs_dec_create.restype = C.c_void_p
        L.hs_dec_create.argtypes = [C.c_int] * 5
        L.hs_enc_encode.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.hs_enc_destroy.argtypes = [C.c_void_p]
        L.hs_enc_set_control.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.hs_enc_flags.argtypes = [C.c_void_p]
        L.hs_dec_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        L.hs_dec_destroy.argtypes = [C.c_void_p]
        L.nsq_io_sizes.argtypes = [C.c_void_p]
        L.hs_enc_capture.argtypes = [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
        L.hs_nsq_run.argtypes = [C.c_int] * 4 + [C.c_void_p] * 4
        L.hs_level.argtypes = [C.c_longlong, C.c_int]
        L.hs_row_level.argtypes = [C.c_void_p, C.c_int]
        if emu:
            L.hs_set_emu_nsq.argtypes = [C.c_int]
            L.hs_enc_encode_pair.argtypes = [C.c_void_p] * 6 + [C.c_int] + [C.c_void_p] * 3
        _libs[emu] = L
    return _libs[emu]


class SimEncoder:
    def __init__(self, rate=13600, dtx=0, use_md_index=0, cap=1024, emu=None, framesize_ms=40, joint_hb=0, emu_nsq=False):
        """emu_nsq (emu build only): the quantiser stage runs the device kernel's code (sb_nsq_warp.cuh) on emulated lanes too."""
        self.L = lib(emu)
        self.emu_nsq = bool(emu_nsq)
        assert not self.emu_nsq or self.L.hs_is_emu() == 1
        self.h = self.L.hs_enc_create3(rate, dtx, use_md_index, framesize_ms, joint_hb)
        self.samples = 16 * framesize_ms
        self.cap = cap
        self.out = np.zeros(cap, np.uint8)
        self.nb = np.zeros(6, np.int16)

    def encode(self, pcm640):
        x = np.ascontiguousarray(pcm640, np.int16)
        assert x.size == self.samples
        if self.L.hs_is_emu() == 1:
            self.L.hs_set_emu_nsq(1 if self.emu_nsq else 0)
        n = self.L.hs_enc_encode(self.h, x.ctypes.data, self.out.ctypes.data, self.cap, self.nb.ctypes.data)
        return bytes(self.out[:max(n, 0)]), (int(self.nb[0]), int(self.nb[1])), n

    def capture(self, pcm640):
        """Encode one packet and return what its quantiser stage received: the frames (oracle.nsq_ref.FRAME_IN, one per
        frame of the packet) and the three quantiser states before it ran (oracle.nsq_ref.STATE, centre first)."""
        from oracle import nsq_ref
        x = np.ascontiguousarray(pcm640, np.int16)
        assert x.size == self.samples
        fr = np.zeros(self.samples // 320, nsq_ref.FRAME_IN)
        st = np.zeros(3, nsq_ref.STATE)
        if self.L.hs_is_emu() == 1:
            self.L.hs_set_emu_nsq(0)
        n = self.L.hs_enc_capture(self.h, x.ctypes.data, fr.ctypes.data, st.ctypes.data, self.out.ctypes.data, self.cap,
                                  self.nb.ctypes.data)
        assert n >= 0
        return fr, st

    @property
    def flags(self):
        """The activity kernel's flags of the last packet: bit f = frame f's coded VAD flag, 0 for a DTX-dropped packet."""
        return self.L.hs_enc_flags(self.h)

    def set_control(self, rate=None, dtx=None, loss=None):
        """Rate (b/s), DTX and expected loss (%) from the next packet on, through enc_set_control; None = unchanged."""
        self.L.hs_enc_set_control(self.h, *(-1 if v is None else int(v) for v in (rate, dtx, loss)))

    def close(self):
        if self.h:
            self.L.hs_enc_destroy(self.h)
            self.h = None


def encode_pair(ea, eb, pcm_a, pcm_b):
    """Two encoders of the emu="gw16" build through ONE emulated quantiser warp (a lane group each).  Returns the two
    (payload, (n0, n1), n) results."""
    xa, xb = np.ascontiguousarray(pcm_a, np.int16), np.ascontiguousarray(pcm_b, np.int16)
    ret = np.zeros(2, np.int32)
    r = ea.L.hs_enc_encode_pair(ea.h, eb.h, xa.ctypes.data, xb.ctypes.data, ea.out.ctypes.data, eb.out.ctypes.data, ea.cap,
                                ea.nb.ctypes.data, eb.nb.ctypes.data, ret.ctypes.data)
    assert r == 0
    return tuple((bytes(e.out[:max(int(n), 0)]), (int(e.nb[0]), int(e.nb[1])), int(n)) for e, n in ((ea, ret[0]), (eb, ret[1])))


def nsq_run(st0, frames, nf, emu=None):
    """The quantiser stage alone over n cases: st0 [n, 3] (oracle.nsq_ref.STATE), frames [n, npk * nf] (FRAME_IN).
    emu=None: the scalar model; emu="gw16" (or True): the kernel's device code on emulated warps of that build.
    Returns (out [n, npk * nf] FRAME_OUT, states after every packet [n, npk, 3] STATE)."""
    from oracle import nsq_ref
    L = lib(emu if emu else False)
    nsq_ref.check_sizes(L)
    st0 = np.ascontiguousarray(st0, nsq_ref.STATE)
    frames = np.ascontiguousarray(frames, nsq_ref.FRAME_IN)
    n, nfr = frames.shape
    assert st0.shape == (n, 3) and nfr % nf == 0
    out = np.zeros((n, nfr), nsq_ref.FRAME_OUT)
    st = np.zeros((n, nfr // nf, 3), nsq_ref.STATE)
    r = L.hs_nsq_run(1 if emu else 0, n, nfr // nf, nf, st0.ctypes.data, frames.ctypes.data, out.ctypes.data, st.ctypes.data)
    assert r == 0, r
    return out, st


def level(E, n):
    """RFC 6464 level of a row of n samples whose sum of squares is E (sb_activity.cuh)."""
    return lib().hs_level(int(E), n)


def row_level(x):
    """The activity kernel's level of one int16 row."""
    x = np.ascontiguousarray(x, np.int16)
    return lib().hs_row_level(x.ctypes.data, x.size)


class SimDecoder:
    def __init__(self, use_md_index=0, framesize_ms=40, joint_hb=0, arith="flp", samplerate=16000):
        """arith "flp" / "fix": the reference's float or fixed-point build; samplerate 16000 or 32000 (16 kHz SILK core)."""
        self.L = lib()
        self.h = self.L.hs_dec_create(use_md_index, framesize_ms, joint_hb, ARITH[arith], samplerate)
        assert self.h, samplerate
        self.pcm = np.zeros(samplerate // 1000 * framesize_ms, np.int16)
        self.fl = np.zeros(1, np.uint8)
        self.flags = 0      # the activity flags of the last packet: bit f VAD flag, bit 2 + f concealed; 0 if rejected

    def decode(self, payload, nbytes, lostflag):
        buf = np.zeros(max(len(payload), 1), np.uint8)
        buf[:len(payload)] = np.frombuffer(payload, np.uint8)
        nb = np.array([nbytes[0], nbytes[1]], np.int16)
        r = self.L.hs_dec_decode(self.h, self.pcm.ctypes.data, buf.ctypes.data, len(buf), nb.ctypes.data, int(lostflag),
                                 self.fl.ctypes.data)
        self.flags = int(self.fl[0])
        return self.pcm.copy(), r

    def close(self):
        if self.h:
            self.L.hs_dec_destroy(self.h)
            self.h = None
