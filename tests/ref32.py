"""The reference codec (oracle/_ref, through oracle.ref's bindings) at the 32 kHz API, and the 32 kHz test signals.

TEST INFRASTRUCTURE ONLY.  oracle.ref's handles are made for 16 kHz streams; these are the same six functions with
samplerate = 32000, so that a packet carries 40 ms (or 20 ms) of 32 kHz PCM: 1280 (640) samples."""
import ctypes as C

import numpy as np

from oracle import ref


class Ref32Encoder:
    """One reference encoder handle at 32 kHz (kind = 'fix' is the bitstream parity target)."""

    def __init__(self, kind="fix", rate=24000, dtx=0, use_md_index=0, framesize_ms=40, joint_hb=0):
        self.L = ref.lib(kind).lib
        self.samples = 32 * framesize_ms
        j = 1 if joint_hb else 0
        self.ctrl = ref.EncCtrl(2, rate, 32000, dtx, framesize_ms, j, j, use_md_index)
        self.h = self.L.AGR_Sate_Encoder_Init(C.byref(self.ctrl))
        self._bits = (C.c_uint8 * 1024)()
        self._nb = (C.c_int16 * 6)()

    def encode(self, pcm):
        x = np.ascontiguousarray(pcm, dtype=np.int16)
        assert x.size == self.samples
        C.memset(self._nb, 0, 12)
        n = self.L.AGR_Sate_Encoder_Encode(self.h, x.ctypes.data, self._bits, 1024, self._nb)
        return bytes(self._bits[:max(n, 0)]), (int(self._nb[0]), int(self._nb[1])), n

    def head(self):
        return C.cast(C.c_void_p(self.h), C.POINTER(ref.SateEncHead)).contents

    def set_rate(self, rate):
        """User rate from the next packet on, as Init computes the core's (AGR_BWE_SDK_API.c:118); FIX handles only (the
        handle layout oracle.ref.SateEncHead describes)."""
        c = self.head().encControl
        c.bitRate = int(rate) - (800 if self.ctrl.joint_enable else 1600)

    def close(self):
        if self.h:
            self.L.AGR_Sate_Encoder_Uninit(self.h)
            self.h = None

    __del__ = close


class Ref32Decoder:
    """One reference decoder handle at 32 kHz (kind = 'flp': the float build, 'fix': the fixed-point build)."""

    def __init__(self, kind="flp", use_md_index=0, framesize_ms=40, joint_hb=0):
        self.L = ref.lib(kind).lib
        self.samples = 32 * framesize_ms
        j = 1 if joint_hb else 0
        self.ctrl = ref.DecCtrl(0, 32000, framesize_ms, j, j, use_md_index)
        self.h = self.L.AGR_Sate_Decoder_Init(C.byref(self.ctrl))
        self._out = np.zeros(1920, dtype=np.int16)
        self._ns = C.c_int16(0)

    def decode(self, payload, nbytes, lostflag):
        """payload / nbytes pre-trimmed by the caller as dec_main.c:245-307 does; returns (PCM, return value)."""
        buf = (C.c_uint8 * 1024)(*payload) if payload else (C.c_uint8 * 1024)()
        nb = (C.c_int16 * 6)(int(nbytes[0]), int(nbytes[1]))
        ret = self.L.AGR_Sate_Decoder_Decode(self.h, self._out.ctypes.data, C.byref(self._ns), buf, nb, int(lostflag))
        assert ret != 0 or self._ns.value == self.samples, (self._ns.value, self.samples)
        return self._out[:self.samples].copy(), ret

    def close(self):
        if self.h:
            self.L.AGR_Sate_Decoder_Uninit(self.h)
            self.h = None

    __del__ = close


def upsample2(clip):
    """The clip at 32 kHz by an integer-exact rule: every 16 kHz sample x[n] is followed by the rounded-down mean of x[n]
    and x[n + 1] (the last one by itself).  No content above 8 kHz beyond the rule's images."""
    x = clip.astype(np.int32)
    nxt = np.concatenate([x[1:], x[-1:]])
    y = np.empty(2 * len(x), np.int32)
    y[0::2] = x
    y[1::2] = (x + nxt) >> 1
    return y.astype(np.int16)


def with_high_band(clip, seed=32):
    """upsample2(clip) plus seeded white noise of standard deviation 400 (content across 0-16 kHz, so that the 8-16 kHz
    band carries a signal), clipped to int16."""
    rng = np.random.Generator(np.random.PCG64(seed))
    y = upsample2(clip).astype(np.float64) + rng.normal(0.0, 400.0, 2 * len(clip))
    return np.clip(np.round(y), -32768, 32767).astype(np.int16)


def chirp(n_samples, amp=8000):
    """A linear chirp from 100 Hz to 15 kHz over n_samples at 32 kHz."""
    t = np.arange(n_samples) / 32000.0
    T = n_samples / 32000.0
    ph = 2 * np.pi * (100.0 * t + (15000.0 - 100.0) * t * t / (2 * T))
    return np.round(amp * np.sin(ph)).astype(np.int16)
