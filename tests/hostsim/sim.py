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
        L.hs_dec_create.argtypes = [C.c_int] * 6
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
        vp, ci = C.c_void_p, C.c_int
        L.mix_model.argtypes = [vp, vp, ci, ci] + [vp] * 4 + [ci, ci, vp]
        L.rx_model_insert.argtypes = [ci, ci, ci] + [vp] * 13 + [ci, vp, C.c_int64]
        L.rx_model_pull.argtypes = [ci, ci, ci] + [vp] * 6 + [vp, ci, vp, vp]
        L.rx_model_merge.argtypes = [ci, ci, vp, vp]
        L.rx_model_timing.argtypes = [ci, ci, C.c_uint32] + [vp] * 12 + [ci, C.c_int64]
        L.tx_model_pack.argtypes = [ci, vp, ci, vp] + [vp] * 9
        L.tx_model_pack.restype = ci
        L.tx_model_contributors.argtypes = [vp, vp, ci, ci, vp, vp, ci, vp, vp]
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
    def __init__(self, use_md_index=0, framesize_ms=40, joint_hb=0, arith="flp", samplerate=16000, out_samplerate=None):
        """arith "flp" / "fix": the reference's float or fixed-point build; samplerate 16000 or 32000 (16 kHz SILK core);
        out_samplerate the stream's rate (the default) or, for a 32 kHz stream, 16000: rows of its 16 kHz core."""
        out_samplerate = samplerate if out_samplerate is None else out_samplerate
        self.L = lib()
        self.h = self.L.hs_dec_create(use_md_index, framesize_ms, joint_hb, ARITH[arith], samplerate, out_samplerate)
        if not self.h:
            raise ValueError("no decoder of %d Hz streams with %d Hz output" % (samplerate, out_samplerate))
        self.pcm = np.zeros(out_samplerate // 1000 * framesize_ms, np.int16)
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


# ---- the server side: mixer, receive queue, send queue (server.cpp) -----------------------------------------------------
M32 = 1 << 32


def _ptrs(*arrays):
    return [x.ctypes.data for x in arrays]


def mix_model(pcm, level, flags, room_start, members, k, out):
    """The two mix kernels over rows pcm int16 [n, spp] into out (rows of streams in no room are left as they are).
    Returns (out, talkers int32 [rooms, k])."""
    R = len(room_start) - 1
    talkers = np.full((R, k), 12345, np.int32)
    n, spp = pcm.shape
    lib().mix_model(*_ptrs(pcm, out), spp, n, *_ptrs(level, flags, room_start, members), R, k, talkers.ctypes.data)
    return out, talkers


def contributors(room_start, members, k, talkers, level, n):
    """sb_mix_contributors_kernel's lists: (csrc int32 [n, k], csrc_level uint8 [n, k])."""
    csrc, lvl = np.zeros((n, k), np.int32), np.zeros((n, k), np.uint8)
    rs, mb, tk, lv = (np.ascontiguousarray(x, t) for x, t in ((room_start, np.int32), (members, np.int32),
                                                                 (talkers, np.int32), (level, np.uint8)))
    lib().tx_model_contributors(*_ptrs(rs, mb), len(rs) - 1, k, *_ptrs(tk, lv), n, *_ptrs(csrc, lvl))
    return csrc, lvl


def merge(n1, n2):
    """The shared merge rule of descriptions of n1 / n2 bytes (0 = missing): (row length, nbytes int16 [2], lostflag)."""
    nb, lf = np.zeros(2, np.int16), np.zeros(1, np.int32)
    row = lib().rx_model_merge(n1, n2, *_ptrs(nb, lf))
    return row, nb, int(lf[0])


class SimRx:
    """A receive queue of n streams (solo_b200_rx) in the device layout of solo_b200.cu's RxDev, and of RxTiming once
    timing is enabled, advanced by the host build of sb_rx.cuh.  Same call shapes as solo_b200.RxQueue."""

    def __init__(self, n, depth, desc_cap):
        self.L, self.n, self.depth, self.desc_cap = lib(), n, depth, desc_cap
        self.last = np.full(n, M32 - 1, np.uint32)
        self.idx = np.zeros(n * depth, np.uint32)
        self.len = np.zeros(n * depth * 2, np.uint16)
        self.elect = np.zeros(n * depth * 2, np.uint64)
        self.rep = np.full(n * depth, 0xFFFFFFFF, np.uint32)
        self.cnt = np.zeros((n, 8), np.uint32)
        self.bad = np.zeros(1, np.uint64)
        self.store = np.zeros(n * depth * 2 * desc_cap + 16, np.uint8)
        self.ts = None

    def enable_timing(self, ts_per_index):
        self.ts = int(ts_per_index)
        self.transit = np.zeros(self.n, np.uint32)
        self.jitter = np.zeros(self.n, np.uint32)          # 1/16 units, as the device keeps it
        self.highest = np.zeros(self.n, np.uint64)
        self.received = np.zeros(self.n, np.uint32)
        self.margin = np.zeros((self.n, 8), np.uint32)

    def insert(self, stream, index, desc, off, lens, payload, arrival=None):
        """arrival (receive times) makes it a timed insert, which needs enable_timing first."""
        a = [np.ascontiguousarray(x, t) for x, t in ((stream, np.int32), (index, np.uint32), (desc, np.uint8),
                                                     (off, np.int32), (lens, np.int32), (payload, np.uint8))]
        na, pay = len(a[0]), a[5]
        self.L.rx_model_insert(self.n, self.depth, self.desc_cap, *_ptrs(self.last, self.idx, self.len, self.elect, self.rep,
                                                                         self.cnt, self.bad, self.store),
                               *_ptrs(*a[:5]), na, pay.ctypes.data, pay.size)
        if arrival is not None:     # as rx_insert_timed_launch: the insert passes, then the timing of the same arrays
            assert self.ts is not None, "timing is not enabled"
            ar = np.ascontiguousarray(arrival, np.uint32)
            assert ar.shape == (na,)
            self.L.rx_model_timing(self.n, self.desc_cap, self.ts, *_ptrs(self.last, self.transit, self.jitter, self.highest,
                                                                          self.received, self.margin),
                                   *_ptrs(*a[:5], ar), na, pay.size)

    def pull(self, play=None, cap=None):
        """-> (bits uint8 [n, cap], nbytes int16 [n, 2], lostflag int32 [n]); cap defaults to 2 * desc_cap."""
        cap = 2 * self.desc_cap if cap is None else cap
        bits = np.zeros((self.n, cap), np.uint8)
        nb = np.zeros((self.n, 2), np.int16)
        lf = np.zeros(self.n, np.int32)
        p = np.ascontiguousarray(play, np.uint32) if play is not None else None
        self.L.rx_model_pull(self.n, self.depth, self.desc_cap, *_ptrs(self.last, self.idx, self.len, self.cnt, self.store),
                             p.ctypes.data if p is not None else None, bits.ctypes.data, cap, *_ptrs(nb, lf))
        return bits, nb, lf

    def reset(self, streams, start):
        """As solo_b200_rx_reset: the listed streams play start[i] next, with empty slots, zero counters and, on a timed
        queue, cleared timing."""
        for s, t in zip(streams, start):
            self.last[s] = (int(t) - 1) % M32
            self.cnt[s] = 0
            self.len[s * 2 * self.depth:(s + 1) * 2 * self.depth] = 0
        if self.ts is not None:
            for x in (self.transit, self.jitter, self.highest, self.received, self.margin):
                x[np.asarray(streams, np.int64)] = 0

    def stats(self):
        """(counters uint32 [n, 8], arrivals for streams outside [0, n))."""
        return self.cnt.copy(), int(self.bad[0])

    def timing(self):
        """(jitter >> 4, highest, received, margin), as solo_b200_rx_timing reports them."""
        return self.jitter >> 4, self.highest.copy(), self.received.copy(), self.margin.copy()


class SimTx:
    """A send queue of n streams (solo_b200_tx) in the device layout of solo_b200.cu's TxDev, advanced by the host build
    of sb_tx.cuh."""

    def __init__(self, n):
        self.L, self.n = lib(), n
        self.next = np.zeros(n, np.uint32)
        self.cnt = np.zeros((n, 4), np.uint32)

    def pack(self, bits, nbytes):
        """-> (payload bytes, [(stream, index, desc, off, len)])."""
        bits = np.ascontiguousarray(bits, np.uint8)
        nbytes = np.ascontiguousarray(nbytes, np.int16)
        e = 2 * self.n
        payload = np.zeros(self.n * bits.shape[1], np.uint8)
        ent = [np.zeros(e, t) for t in (np.int32, np.uint32, np.uint8, np.int32, np.int32)]
        total = C.c_int64()
        c = self.L.tx_model_pack(self.n, bits.ctypes.data, bits.shape[1], *_ptrs(nbytes, self.next, self.cnt, payload, *ent),
                                 C.byref(total))
        return bytes(payload[:total.value]), list(zip(*(x[:c].tolist() for x in ent)))

    def reset(self, streams, start):
        for s, t in zip(streams, start):
            self.next[s] = int(t) % M32
            self.cnt[s] = 0

    def stats(self):
        return self.cnt.copy()
