"""Activity reports on the CPU: the RFC 6464 level function and the per-frame VAD / concealment flags, through the host build
of their source (tests/hostsim/activity.cpp: sb_activity.cuh with the encoder and decoder it reports on, compiled by g++).

The level is checked at every threshold and against a floating-point restatement; the encoder's flags against the flags
the decoder parses from the same payloads (and, through golden.npz's byte-identical reference payloads, against the
reference encoder's VAD); the decoder's flags under the reference driver's 50 % loss process at 16 and 32 kHz."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.golden import make_golden_32k as mk
from tests.util import GOLDEN, load_clip, load_golden, loss_flags, receive, signal_classes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "activity.cpp")
ROWS = (320, 640, 1280)
ARITH = {"flp": 0, "fix": 1}                    # sb::DEC_FLP / sb::DEC_FIX
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_level_tables  # noqa: E402


def load_lib(out):
    """Compile tests/hostsim/activity.cpp to `out` and load it."""
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-w", SRC, "-o", out])
    lib = C.CDLL(out)
    lib.act_level.argtypes = [C.c_longlong, C.c_int]
    lib.act_row_level.argtypes = [C.c_void_p, C.c_int]
    lib.act_enc_create.restype = C.c_void_p
    lib.act_enc_create.argtypes = [C.c_int] * 5
    lib.act_enc_encode.argtypes = [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 2
    lib.act_enc_destroy.argtypes = [C.c_void_p]
    lib.act_dec_create.restype = C.c_void_p
    lib.act_dec_create.argtypes = [C.c_int] * 5
    lib.act_dec_decode.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    lib.act_dec_destroy.argtypes = [C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def L(tmp_path_factory):
    return load_lib(str(tmp_path_factory.mktemp("activity") / "libactivity.so"))


def row_level(L, x):
    x = np.ascontiguousarray(x, np.int16)
    return L.act_row_level(x.ctypes.data, x.size)


def float_level(E, n):
    """clamp(round(10 log10(n 2^30 / E)), 0, 127) in float64 (127 for E = 0)."""
    E = np.asarray(E, np.float64)
    with np.errstate(divide="ignore"):
        v = np.where(E > 0, 10.0 * np.log10(n * 2.0 ** 30 / np.maximum(E, 1)), 1e9)
    return np.clip(np.round(v), 0, 127).astype(np.int64)


class Encoder:
    def __init__(self, L, rate=13600, dtx=0, use_md_index=0, framesize_ms=40, joint_hb=0):
        self.L, self.samples = L, 16 * framesize_ms
        self.h = L.act_enc_create(rate, dtx, use_md_index, framesize_ms, joint_hb)
        self.out, self.nb, self.fl = np.zeros(1024, np.uint8), np.zeros(2, np.int16), np.zeros(1, np.uint8)

    def encode(self, pcm):
        x = np.ascontiguousarray(pcm, np.int16)
        n = self.L.act_enc_encode(self.h, x.ctypes.data, self.out.ctypes.data, 1024, self.nb.ctypes.data, self.fl.ctypes.data)
        return bytes(self.out[:max(n, 0)]), (int(self.nb[0]), int(self.nb[1])), int(self.fl[0])

    def close(self):
        self.L.act_enc_destroy(self.h)


class Decoder:
    def __init__(self, L, use_md_index=0, framesize_ms=40, joint_hb=0, arith="flp", samplerate=16000):
        self.L, self.sr = L, samplerate
        self.h = L.act_dec_create(use_md_index, framesize_ms, joint_hb, ARITH[arith], samplerate)
        self.pcm, self.fl = np.zeros(samplerate // 1000 * framesize_ms, np.int16), np.zeros(1, np.uint8)

    def decode(self, payload, nbytes, lostflag):
        buf = np.zeros(max(len(payload), 1), np.uint8)
        buf[:len(payload)] = np.frombuffer(payload, np.uint8)
        nb = np.array(nbytes, np.int16)
        r = self.L.act_dec_decode(self.h, self.sr, self.pcm.ctypes.data, buf.ctypes.data, len(buf), nb.ctypes.data, int(lostflag),
                                  self.fl.ctypes.data)
        return self.pcm.copy(), r, int(self.fl[0])

    def close(self):
        self.L.act_dec_destroy(self.h)


# ---- level ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", ROWS)
def test_level_at_every_threshold(L, n):
    """At T_n[k] - 1, T_n[k] and T_n[k] + 1 for every k: the level is the number of thresholds above E."""
    T = np.array(gen_level_tables.thresholds(n), np.int64)
    for t in T:
        for E in (t - 1, t, t + 1):
            if E >= 0:
                assert L.act_level(int(E), n) == int((E < T).sum()), (n, int(E))
    assert L.act_level(0, n) == 127 and L.act_level(n << 30, n) == 0


@pytest.mark.parametrize("n", ROWS)
def test_level_against_float_restatement(L, n):
    """Random rows over the whole dynamic range: equal to round(10 log10(n 2^30 / E)) wherever E is not within 1e-9
    (relative) of a real threshold n 2^30 10^(-(k + 0.5) / 10)."""
    rng = np.random.Generator(np.random.PCG64(n))
    t_real = n * 2.0 ** 30 * 10.0 ** (-(np.arange(127) + 0.5) / 10)
    checked = 0
    for i in range(600):
        amp = 10.0 ** rng.uniform(-0.5, 4.6)
        x = np.clip(np.round(rng.normal(0, amp, n)), -32768, 32767).astype(np.int16)
        E = int((x.astype(np.int64) ** 2).sum())
        if E and np.min(np.abs(E - t_real) / t_real) < 1e-9:
            continue
        assert row_level(L, x) == int(float_level(E, n)), (n, i, E)
        checked += 1
    assert checked > 590


def test_level_of_edge_rows(L):
    """Zeros 127, a +-32767 square 0, a full-scale sine 3, single-LSB noise as the float restatement (and near 115 - 10 log10
    of its density)."""
    rng = np.random.Generator(np.random.PCG64(3))
    for n in ROWS:
        t = np.arange(n)
        assert row_level(L, np.zeros(n, np.int16)) == 127
        assert row_level(L, np.where(t % 2 == 0, 32767, -32767)) == 0
        assert row_level(L, np.full(n, -32768)) == 0
        assert row_level(L, np.round(32767 * np.sin(2 * np.pi * 1000 * t / 16000 + 0.3))) == 3
        for p in (1.0, 0.5, 0.1, 1.0 / n):
            x = (rng.random(n) < p) * rng.choice([-1, 1], n)
            if not x.any():
                x[0] = 1
            E = int((x ** 2).sum())
            assert row_level(L, x) == int(float_level(E, n)), (n, p)
        one = np.zeros(n, np.int16)
        one[7] = 1
        assert row_level(L, one) == int(float_level(1, n)) == int(round(10 * np.log10(n * 2.0 ** 30)))


def test_committed_tables_are_the_generators():
    """solo_b200/csrc/sb_level_tables.inc is what tools/gen_level_tables.py writes (exact decimal arithmetic)."""
    with open(gen_level_tables.OUT) as f:
        assert f.read() == gen_level_tables.text()
    for n in ROWS:
        T = gen_level_tables.thresholds(n)
        t_real = n * 2.0 ** 30 * 10.0 ** (-(np.arange(127) + 0.5) / 10)
        assert np.all(np.abs(np.array(T, np.float64) - np.ceil(t_real)) <= np.maximum(1, 1e-12 * t_real))


# ---- encoder flags ----------------------------------------------------------------------------------------------------
MODES = {"40ms": dict(framesize_ms=40), "20ms": dict(framesize_ms=20), "joint": dict(framesize_ms=40, joint_hb=1)}


def inputs():
    """(name, int16 16 kHz signal, encoder kwargs): the clip, the eight signal classes and a DTX stream fading to silence."""
    clip = load_clip()
    out = [("clip", clip[:640 * 120], {})]
    sc = signal_classes(clip, 8, 30)
    for k in range(8):
        out.append(("class%d" % k, sc[:, k, :].reshape(-1), {}))
    t = np.arange(640 * 90)
    fade = (clip[:t.size] * np.clip(1.0 - t / (0.5 * t.size), 0, 1)).astype(np.int16)
    out.append(("dtx_fade", fade, dict(dtx=1)))
    return out


def encode_with_flags(L, x, **kw):
    e = Encoder(L, **kw)
    k = e.samples
    pk = [e.encode(x[i * k:(i + 1) * k]) for i in range(len(x) // k)]
    e.close()
    return pk


@pytest.mark.parametrize("mode", sorted(MODES))
def test_encoder_flags_are_what_the_decoder_parses(L, mode):
    """For every packet of every input: the encoder's flags equal the VAD flags the decoder parses from its payload; a
    DTX-dropped packet (nothing sent) reports 0.  20 ms packets never set bit 1."""
    cfg = MODES[mode]
    nf = cfg["framesize_ms"] // 20
    seen, dropped = set(), 0
    for name, x, kw in inputs():
        pk = encode_with_flags(L, x, **cfg, **kw)
        d = Decoder(L, **cfg)
        for p, (b, nb, fl) in enumerate(pk):
            assert fl & ~((1 << nf) - 1) == 0, (mode, name, p, fl)
            y, r, dfl = d.decode(*receive(b, nb, 4))
            assert r == 0
            if nb[0] <= 0:
                assert fl == 0 and dfl == (0xC if nf == 2 else 0x4), (mode, name, p)
                dropped += 1
            else:
                assert dfl == fl, (mode, name, p, fl, dfl)
            seen.add(fl)
        d.close()
    assert {0, (1 << nf) - 1} <= seen and dropped > 0, (seen, dropped)


def test_encoder_flags_match_the_reference_payloads(L):
    """golden.npz holds the reference encoder's payloads of the clip (rate 13 600, 40 ms), byte-identical to the host
    model's: the VAD flags parsed from them are the host encoder's flags, packet by packet."""
    g = load_golden()
    clip = load_clip()
    pk = encode_with_flags(L, clip, rate=13600)
    assert len(pk) == g["fix_nbytes"].shape[0]
    d = Decoder(L)
    for p, (b, nb, fl) in enumerate(pk):
        n0 = int(g["fix_nbytes"][p, 0])
        assert nb == tuple(int(v) for v in g["fix_nbytes"][p]) and b[:n0] == bytes(g["fix_bits"][p, :n0]), p
        y, r, dfl = d.decode(bytes(g["fix_bits"][p, :n0]), tuple(int(v) for v in g["fix_nbytes"][p]), 4)
        assert r == 0 and dfl == fl, (p, fl, dfl)
    d.close()


# ---- decoder flags under loss -----------------------------------------------------------------------------------------
def streams_16k(L):
    """(mode, packets, decoder kwargs) of the clip at 16 kHz, encoded by the host model."""
    clip = load_clip()[:640 * 80]
    return [(m, [(b, nb) for b, nb, fl in encode_with_flags(L, clip, rate=13600, **cfg)], cfg) for m, cfg in MODES.items()]


def streams_32k():
    f = np.load(os.path.join(GOLDEN, "golden_32k.npz"))
    return [(s, mk.packets(f, s), mk.STREAMS[s][1]) for s in ("hb40", "hb20", "joint")]


def check_loss(L, pk, cfg, samplerate, arith, seed, lead=0):
    """One stream under the 50 % loss process of `seed`, its first `lead` packets lost (loss before any good frame)."""
    nf = cfg["framesize_ms"] // 20
    conc = 0xC if nf == 2 else 0x4
    ref = Decoder(L, arith=arith, samplerate=samplerate, **cfg)
    parsed = [ref.decode(*receive(b, nb, 4))[2] for b, nb in pk]
    ref.close()
    flags = [1] * lead + loss_flags(len(pk), 50, seed=seed)[lead:]
    d = Decoder(L, arith=arith, samplerate=samplerate, **cfg)
    n_lost = 0
    for p, (b, nb) in enumerate(pk):
        pb, pnb, fl = receive(b, nb, flags[p])
        y, r, dfl = d.decode(pb, pnb, fl)
        assert r == 0
        if fl == 1:
            assert dfl == conc, (p, dfl)
            n_lost += 1
        else:
            assert dfl == parsed[p] and dfl & conc == 0, (p, fl, dfl, parsed[p])
    d.close()
    assert n_lost > 0 and any(parsed)


@pytest.mark.parametrize("arith", ["flp", "fix"])
def test_decoder_flags_under_loss_16k(L, arith):
    """The reference driver's 50 % loss process: the concealed bits are the frames of lost packets (lostflag 1, from the
    first packets on in the second run), the VAD bits of received frames those parsed from the same payloads loss-free."""
    for mode, pk, cfg in streams_16k(L):
        if arith == "fix" and cfg["framesize_ms"] == 20:
            continue
        check_loss(L, pk, cfg, 16000, arith, 1)
        check_loss(L, pk, cfg, 16000, arith, 4, lead=3)


@pytest.mark.parametrize("arith", ["flp", "fix"])
def test_decoder_flags_under_loss_32k(L, arith):
    """The same for golden_32k.npz's 32 kHz streams (16 kHz SILK core)."""
    for s, pk, cfg in streams_32k():
        if arith == "fix" and cfg["framesize_ms"] == 20:
            continue
        check_loss(L, pk, cfg, 32000, arith, 1)
        check_loss(L, pk, cfg, 32000, arith, 4, lead=3)


def test_rejected_packet_reports_no_flags(L):
    """A packet the decoder rejects (bad lostflag, 16 kHz-stream packets to a 32 kHz decoder) gives flags 0."""
    g = load_golden()
    n0 = int(g["fix_nbytes"][0, 0])
    d = Decoder(L, samplerate=32000)
    y, r, fl = d.decode(bytes(g["fix_bits"][0, :n0]), tuple(int(v) for v in g["fix_nbytes"][0]), 4)
    assert r < 0 and fl == 0
    y, r, fl = d.decode(bytes(16), (16, 8), 7)
    assert r < 0 and fl == 0
    d.close()
