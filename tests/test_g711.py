"""The G.711 gateway's arithmetic on the host (tests/hostsim, the host build of solo_b200/csrc/sb_g711.cuh): companding
against a transcription of the G.711 segment rule (and Python's audioop where it exists), the filter banks against the
reference's fixed-point AGR_Sate_qmf_decomp / AGR_Sate_qmf_synth, and the voice activity against the codec's VAD stage."""
import ctypes as C
import warnings

import numpy as np
import pytest

from tests.hostsim import g711_sim, sim
from tests.util import load_clip

LAWS = (0, 1)       # mu-law (PCMU), A-law (PCMA)


# ---- the segment rule of G.711 (the classic Sun / CCITT g711.c), transcribed in numpy ----------------------------------
def ref_compress(law, x):
    x = np.asarray(x, np.int32)
    if law == 1:
        v = x >> 3
        mask = np.where(v >= 0, 0xD5, 0x55)
        v = np.where(v >= 0, v, -v - 1)
        seg = np.searchsorted(np.array([(0x20 << s) - 1 for s in range(8)]), v, side="left")
        q = np.where(seg < 2, v >> 1, v >> np.maximum(seg, 1)) & 0xF
        return (((seg << 4) | q) ^ mask).astype(np.uint8)
    v = x >> 2
    mask = np.where(v < 0, 0x7F, 0xFF)
    v = np.minimum(np.abs(v), 8159) + 33
    seg = np.searchsorted(np.array([(0x40 << s) - 1 for s in range(8)]), v, side="left")
    code = np.where(seg >= 8, 0x7F ^ mask, ((np.minimum(seg, 7) << 4) | ((v >> (np.minimum(seg, 7) + 1)) & 0xF)) ^ mask)
    return code.astype(np.uint8)


def ref_expand(law, c):
    c = np.asarray(c, np.int32)
    if law == 1:
        a = c ^ 0x55
        seg = (a & 0x70) >> 4
        t = ((a & 0xF) << 4) + np.where(seg == 0, 8, 0x108)
        t = np.where(seg > 1, t << np.maximum(seg - 1, 0), t)
        return np.where(a & 0x80, t, -t).astype(np.int16)
    u = ~c & 0xFF
    t = (((u & 0xF) << 3) + 0x84) << ((u & 0x70) >> 4)
    return np.where(u & 0x80, 0x84 - t, t - 0x84).astype(np.int16)


def _audioop():
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            import audioop
        except ImportError:
            return None
    return audioop


ALL_X = np.arange(-32768, 32768, dtype=np.int32).astype(np.int16)
ALL_C = np.arange(256, dtype=np.uint8)


@pytest.mark.parametrize("law", LAWS)
def test_companding_matches_segment_rule(law):
    assert np.array_equal(g711_sim.g711_compress(law, ALL_X), ref_compress(law, ALL_X))
    assert np.array_equal(g711_sim.g711_expand(law, ALL_C), ref_expand(law, ALL_C))
    au = _audioop()
    if au is not None:
        comp, exp = (au.lin2ulaw, au.ulaw2lin) if law == 0 else (au.lin2alaw, au.alaw2lin)
        assert np.array_equal(g711_sim.g711_compress(law, ALL_X), np.frombuffer(comp(ALL_X.astype("<i2").tobytes(), 2), np.uint8))
        assert np.array_equal(g711_sim.g711_expand(law, ALL_C), np.frombuffer(exp(ALL_C.tobytes(), 2), "<i2"))
    back = g711_sim.g711_compress(law, g711_sim.g711_expand(law, ALL_C))
    bad = np.nonzero(back != ALL_C)[0].tolist()
    assert bad == ([0x7F] if law == 0 else []), bad      # mu-law's negative zero expands to 0, which compresses to 0xFF


def test_companding_fixed_points():
    # ends of the scale and the codes of zero
    assert g711_sim.g711_compress(0, [0, -1, 32767, -32768]).tolist() == [0xFF, 0x7E, 0x80, 0x00]
    assert g711_sim.g711_compress(1, [0, -1, 32767, -32768]).tolist() == [0xD5, 0x55, 0xAA, 0x2A]
    assert g711_sim.g711_expand(0, [0x00, 0x80, 0xFF, 0x7F]).tolist() == [-32124, 32124, 0, 0]
    assert g711_sim.g711_expand(1, [0x2A, 0xAA, 0xD5, 0x55]).tolist() == [-32256, 32256, 8, -8]


# ---- signals ------------------------------------------------------------------------------------------------------------
def signals16(n_packets, spp16, seed=3):
    """int16 [rows, n_packets * spp16]: speech, sines across 0-8 kHz (the QMF transition band at 4 kHz included), a
    full-scale square and silence."""
    clip = load_clip().astype(np.int64)
    T = n_packets * spp16
    t = np.arange(T)
    rows = [np.resize(clip, T)]
    for f in (300.0, 1000.0, 3400.0, 3900.0, 4000.0, 4100.0, 6000.0):
        rows.append(np.round(20000 * np.sin(2 * np.pi * f * t / 16000)))
    rows.append(np.where((t // 20) % 2, 32767, -32768))
    rows.append(np.zeros(T))
    return np.clip(np.stack(rows), -32768, 32767).astype(np.int16)


def payloads(n_packets, spp8, seed=4):
    """uint8 [rows, n_packets * spp8]: compressed speech and tones at 8 kHz, random bytes, the codes of silence."""
    rng = np.random.Generator(np.random.PCG64(seed))
    x16 = signals16(n_packets, 2 * spp8)
    x8 = x16[:, ::2]
    rows = [ref_compress(0, x8[0]), ref_compress(1, x8[0]), ref_compress(0, x8[3]), ref_compress(1, x8[8]),
            rng.integers(0, 256, x8.shape[1]), np.full(x8.shape[1], 0xFF), np.full(x8.shape[1], 0xD5)]
    return np.stack(rows).astype(np.uint8)


# ---- the filter banks against the reference ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref():
    from tests.test_gpu_bands import Ref
    return Ref()


@pytest.mark.parametrize("fs", (40, 20))
def test_downlink_low_band_matches_reference(ref, fs):
    spp16, npk = 16 * fs, 12
    x = signals16(npk, spp16)
    for law in LAWS:
        g = g711_sim.SimG711(len(x), fs, law)
        mems = [np.zeros(64, np.int16) for _ in x]
        for p in range(npk):
            rows = x[:, p * spp16:(p + 1) * spp16]
            codes = g.downlink(rows)
            for s in range(len(x)):
                lo, _ = ref.decomp(rows[s], mems[s])
                assert np.array_equal(g.low[s], lo), ("law", law, "row", s, "packet", p)
                assert np.array_equal(codes[s], ref_compress(law, lo))


@pytest.mark.parametrize("fs", (40, 20))
def test_uplink_row_matches_reference(ref, fs):
    spp8, npk = 8 * fs, 12
    pay = payloads(npk, spp8)
    rng = np.random.Generator(np.random.PCG64(7))
    for law in LAWS:
        g = g711_sim.SimG711(len(pay), fs, law)
        mems = [(np.zeros(64, np.int16), np.zeros(64, np.int16)) for _ in pay]
        for p in range(npk):
            lost = rng.integers(0, 1 << (fs // 20), len(pay)).astype(np.int32) if p % 3 == 2 else None
            rows = pay[:, p * spp8:(p + 1) * spp8]
            pcm, level, flags = g.uplink(rows, lost)
            for s in range(len(pay)):
                x8 = ref_expand(law, rows[s])
                for f in range(fs // 20):
                    if lost is not None and (lost[s] >> f) & 1:
                        x8[160 * f:160 * (f + 1)] = 0
                want, _ = ref.synth(True, x8, np.zeros(spp8, np.float32), *mems[s])
                assert np.array_equal(pcm[s], want), ("law", law, "row", s, "packet", p)
                assert level[s] == sim.row_level(want)


# ---- voice activity ------------------------------------------------------------------------------------------------------
def vad_init_io():
    """The detector's state after vad_init, in oracle/vad_io.h's 28 words."""
    nl_bias = [50, 25, 16, 12]
    nl = [100 * b for b in nl_bias]
    return np.array([0] * 6 + [0] * 4 + [100 * 256] * 4 + nl + [0x7FFFFFFF // v for v in nl] + nl_bias + [15, 0], np.int32)


@pytest.mark.parametrize("fs", (40, 20))
def test_uplink_vad_is_the_codec_vad(fs):
    L = sim.lib()
    L.hs_vad_packet.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    nf, spp8, npk = fs // 20, 8 * fs, 60
    pay = payloads(npk, spp8)
    law = np.arange(len(pay)) % 2
    g = g711_sim.SimG711(len(pay), fs, 0)
    g.reset(np.arange(len(pay)), law)
    st = [vad_init_io() for _ in pay]
    rng = np.random.Generator(np.random.PCG64(11))
    seen = set()
    for p in range(npk):
        lost = (rng.random((len(pay), nf)) < 0.15).astype(np.int32) @ (1 << np.arange(nf)).astype(np.int32)
        rows = pay[:, p * spp8:(p + 1) * spp8]
        _, _, flags = g.uplink(rows, lost.astype(np.int32))
        for s in range(len(pay)):
            x8 = ref_expand(int(law[s]), rows[s])
            want = 0
            out = np.zeros(12, np.int32)
            for f in range(nf):
                if (lost[s] >> f) & 1:
                    x8[160 * f:160 * (f + 1)] = 0
            x8 = np.ascontiguousarray(x8)
            L.hs_vad_packet(st[s].ctypes.data, nf, x8.ctypes.data, out.ctypes.data)
            for f in range(nf):
                sa = int(out[6 * f])
                assert g.sa_Q8[s, f] == sa, ("row", s, "packet", p, "frame", f)
                lf = (lost[s] >> f) & 1
                want |= (4 << f) if lf else ((1 << f) if sa >= 26 else 0)
                seen.add((lf, sa >= 26))
            assert flags[s] == want, ("row", s, "packet", p)
    assert {(0, False), (0, True)} <= seen and any(lf for lf, _ in seen)
