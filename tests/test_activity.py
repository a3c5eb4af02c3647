"""Activity reports on the CPU: the RFC 6464 level function and the per-frame VAD / concealment flags, through the host build
of their source (sb_activity.cuh with the encoder and decoder it reports on, in tests/hostsim).

The level is checked at every threshold and against a floating-point restatement; the encoder's flags against the flags
the decoder parses from the same payloads (and, through golden.npz's byte-identical reference payloads, against the
reference encoder's VAD); the decoder's flags under the reference driver's 50 % loss process at 16 and 32 kHz."""
import os
import sys

import numpy as np
import pytest

from tests.golden import make_golden_32k as mk
from tests.parity import sim  # noqa: F401  (fixture)
from tests.util import GOLDEN, load_clip, load_golden, loss_flags, receive, signal_classes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS = (320, 640, 1280)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_level_tables  # noqa: E402


def float_level(E, n):
    """clamp(round(10 log10(n 2^30 / E)), 0, 127) in float64 (127 for E = 0)."""
    E = np.asarray(E, np.float64)
    with np.errstate(divide="ignore"):
        v = np.where(E > 0, 10.0 * np.log10(n * 2.0 ** 30 / np.maximum(E, 1)), 1e9)
    return np.clip(np.round(v), 0, 127).astype(np.int64)


# ---- level ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", ROWS)
def test_level_at_every_threshold(sim, n):
    """At T_n[k] - 1, T_n[k] and T_n[k] + 1 for every k: the level is the number of thresholds above E."""
    T = np.array(gen_level_tables.thresholds(n), np.int64)
    for t in T:
        for E in (t - 1, t, t + 1):
            if E >= 0:
                assert sim.level(E, n) == int((E < T).sum()), (n, int(E))
    assert sim.level(0, n) == 127 and sim.level(n << 30, n) == 0


@pytest.mark.parametrize("n", ROWS)
def test_level_against_float_restatement(sim, n):
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
        assert sim.row_level(x) == int(float_level(E, n)), (n, i, E)
        checked += 1
    assert checked > 590


def test_level_of_edge_rows(sim):
    """Zeros 127, a +-32767 square 0, a full-scale sine 3, single-LSB noise as the float restatement (and near 115 - 10 log10
    of its density)."""
    rng = np.random.Generator(np.random.PCG64(3))
    for n in ROWS:
        t = np.arange(n)
        assert sim.row_level(np.zeros(n, np.int16)) == 127
        assert sim.row_level(np.where(t % 2 == 0, 32767, -32767)) == 0
        assert sim.row_level(np.full(n, -32768)) == 0
        assert sim.row_level(np.round(32767 * np.sin(2 * np.pi * 1000 * t / 16000 + 0.3))) == 3
        for p in (1.0, 0.5, 0.1, 1.0 / n):
            x = (rng.random(n) < p) * rng.choice([-1, 1], n)
            if not x.any():
                x[0] = 1
            E = int((x ** 2).sum())
            assert sim.row_level(x) == int(float_level(E, n)), (n, p)
        one = np.zeros(n, np.int16)
        one[7] = 1
        assert sim.row_level(one) == int(float_level(1, n)) == int(round(10 * np.log10(n * 2.0 ** 30)))


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


def encode_with_flags(sim, x, **kw):
    """[(payload, (n0, n1), flags)] of the host encoder over x."""
    e = sim.SimEncoder(**kw)
    k = e.samples
    pk = []
    for i in range(len(x) // k):
        b, nb, _ = e.encode(x[i * k:(i + 1) * k])
        pk.append((b, nb, e.flags))
    e.close()
    return pk


@pytest.mark.parametrize("mode", sorted(MODES))
def test_encoder_flags_are_what_the_decoder_parses(sim, mode):
    """For every packet of every input: the encoder's flags equal the VAD flags the decoder parses from its payload; a
    DTX-dropped packet (nothing sent) reports 0.  20 ms packets never set bit 1."""
    cfg = MODES[mode]
    nf = cfg["framesize_ms"] // 20
    seen, dropped = set(), 0
    for name, x, kw in inputs():
        pk = encode_with_flags(sim, x, **cfg, **kw)
        d = sim.SimDecoder(**cfg)
        for p, (b, nb, fl) in enumerate(pk):
            assert fl & ~((1 << nf) - 1) == 0, (mode, name, p, fl)
            y, r = d.decode(*receive(b, nb, 4))
            dfl = d.flags
            assert r == 0
            if nb[0] <= 0:
                assert fl == 0 and dfl == (0xC if nf == 2 else 0x4), (mode, name, p)
                dropped += 1
            else:
                assert dfl == fl, (mode, name, p, fl, dfl)
            seen.add(fl)
        d.close()
    assert {0, (1 << nf) - 1} <= seen and dropped > 0, (seen, dropped)


def test_encoder_flags_match_the_reference_payloads(sim):
    """golden.npz holds the reference encoder's payloads of the clip (rate 13 600, 40 ms), byte-identical to the host
    model's: the VAD flags parsed from them are the host encoder's flags, packet by packet."""
    g = load_golden()
    clip = load_clip()
    pk = encode_with_flags(sim, clip, rate=13600)
    assert len(pk) == g["fix_nbytes"].shape[0]
    d = sim.SimDecoder()
    for p, (b, nb, fl) in enumerate(pk):
        n0 = int(g["fix_nbytes"][p, 0])
        assert nb == tuple(int(v) for v in g["fix_nbytes"][p]) and b[:n0] == bytes(g["fix_bits"][p, :n0]), p
        y, r = d.decode(bytes(g["fix_bits"][p, :n0]), tuple(int(v) for v in g["fix_nbytes"][p]), 4)
        assert r == 0 and d.flags == fl, (p, fl, d.flags)
    d.close()


# ---- decoder flags under loss -----------------------------------------------------------------------------------------
def streams_16k(sim):
    """(mode, packets, decoder kwargs) of the clip at 16 kHz, encoded by the host model."""
    clip = load_clip()[:640 * 80]
    return [(m, [(b, nb) for b, nb, fl in encode_with_flags(sim, clip, rate=13600, **cfg)], cfg) for m, cfg in MODES.items()]


def streams_32k():
    f = np.load(os.path.join(GOLDEN, "golden_32k.npz"))
    return [(s, mk.packets(f, s), mk.STREAMS[s][1]) for s in ("hb40", "hb20", "joint")]


def check_loss(sim, pk, cfg, samplerate, arith, seed, lead=0):
    """One stream under the 50 % loss process of `seed`, its first `lead` packets lost (loss before any good frame)."""
    nf = cfg["framesize_ms"] // 20
    conc = 0xC if nf == 2 else 0x4
    ref = sim.SimDecoder(arith=arith, samplerate=samplerate, **cfg)
    parsed = []
    for b, nb in pk:
        ref.decode(*receive(b, nb, 4))
        parsed.append(ref.flags)
    ref.close()
    flags = [1] * lead + loss_flags(len(pk), 50, seed=seed)[lead:]
    d = sim.SimDecoder(arith=arith, samplerate=samplerate, **cfg)
    n_lost = 0
    for p, (b, nb) in enumerate(pk):
        pb, pnb, fl = receive(b, nb, flags[p])
        y, r = d.decode(pb, pnb, fl)
        dfl = d.flags
        assert r == 0
        if fl == 1:
            assert dfl == conc, (p, dfl)
            n_lost += 1
        else:
            assert dfl == parsed[p] and dfl & conc == 0, (p, fl, dfl, parsed[p])
    d.close()
    assert n_lost > 0 and any(parsed)


@pytest.mark.parametrize("arith", ["flp", "fix"])
def test_decoder_flags_under_loss_16k(sim, arith):
    """The reference driver's 50 % loss process: the concealed bits are the frames of lost packets (lostflag 1, from the
    first packets on in the second run), the VAD bits of received frames those parsed from the same payloads loss-free."""
    for mode, pk, cfg in streams_16k(sim):
        if arith == "fix" and cfg["framesize_ms"] == 20:
            continue
        check_loss(sim, pk, cfg, 16000, arith, 1)
        check_loss(sim, pk, cfg, 16000, arith, 4, lead=3)


@pytest.mark.parametrize("arith", ["flp", "fix"])
def test_decoder_flags_under_loss_32k(sim, arith):
    """The same for golden_32k.npz's 32 kHz streams (16 kHz SILK core)."""
    for s, pk, cfg in streams_32k():
        if arith == "fix" and cfg["framesize_ms"] == 20:
            continue
        check_loss(sim, pk, cfg, 32000, arith, 1)
        check_loss(sim, pk, cfg, 32000, arith, 4, lead=3)


def test_rejected_packet_reports_no_flags(sim):
    """A packet the decoder rejects (bad lostflag, 16 kHz-stream packets to a 32 kHz decoder) gives flags 0."""
    g = load_golden()
    n0 = int(g["fix_nbytes"][0, 0])
    d = sim.SimDecoder(samplerate=32000)
    y, r = d.decode(bytes(g["fix_bits"][0, :n0]), tuple(int(v) for v in g["fix_nbytes"][0]), 4)
    assert r < 0 and d.flags == 0
    y, r = d.decode(bytes(16), (16, 8), 7)
    assert r < 0 and d.flags == 0
    d.close()
