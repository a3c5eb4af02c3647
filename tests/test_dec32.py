"""32 kHz streams (the reference's 32 kHz API: 16 kHz SILK core, 8-16 kHz high band) through the decoder on the CPU: the host
build of the kernel source (tests/hostsim, the DecState32 instantiation of sb_dec.cuh) against the reference's float and
fixed-point decoders, at 0 LSB.

tests/golden/golden_32k.npz pins the reference's PCM of 32 kHz bitstreams by per-packet md5 (tests/golden/make_golden_32k.py);
where oracle/_ref is built, the fixture is re-derived from it and the host model runs in lockstep with both reference
decoders over inputs the fixture does not cover."""
import hashlib

import numpy as np
import pytest

from tests.core32 import LOCKSTEP, LOCKSTEP_IDS, flags_for, signals32
from tests.golden import make_golden_32k as mk
from tests.parity import ref, sim  # noqa: F401  (fixtures)
from tests.util import fuzz_decoder, load_clip, load_golden, receive, with_high_band

CASES = mk.decode_cases()


@pytest.mark.parametrize("key,stream,kind,rule", CASES, ids=[c[0] for c in CASES])
def test_host_model_matches_fixture(sim, key, stream, kind, rule):
    """Every pinned 32 kHz decode, in the arithmetic of the reference build that made it: per-packet md5 equal (0 LSB)."""
    f = mk.load()
    d = sim.SimDecoder(arith=kind, samplerate=32000, **mk.STREAMS[stream][1])
    rows = mk.decode(d, mk.packets(f, stream), mk.flags_of(f, stream, rule))
    assert all(len(y) == 32 * mk.STREAMS[stream][1]["framesize_ms"] for y in rows)
    got = mk.packet_md5(rows)
    bad = np.nonzero((got != f[key + "_packet_md5"]).any(axis=1))[0]
    assert bad.size == 0, ("first packet whose PCM differs from the reference's (0 LSB bar)", key, int(bad[0]))
    assert hashlib.md5(np.concatenate(rows).tobytes()).hexdigest() == str(f[key + "_md5"])


def test_fixture_rederived_from_oracle(ref):
    """The committed fixture is what the reference libraries produce now (inputs, payloads, both decoders' PCM)."""
    f, want = mk.fixture(), mk.load()
    assert sorted(f) == sorted(want.files)
    for k in f:
        assert np.array_equal(np.asarray(f[k]), want[k]), k


def test_other_core_rate_is_that_streams_error(sim):
    """A frame whose sampling-rate index is not the decoder's core rate is a rejected packet (-12), as a corrupted one: 16 kHz
    streams' packets (8 kHz core) to a 32 kHz decoder and 32 kHz streams' packets to a 16 kHz decoder.  The decoder stays
    usable: a good packet after the rejected ones decodes as it does on a fresh decoder."""
    g, f = load_golden(), mk.load()
    pk32 = mk.packets(f, "hb40")
    for arith in ("flp", "fix"):
        d = sim.SimDecoder(arith=arith, samplerate=32000)
        for i in range(3):
            n0 = int(g["fix_nbytes"][i, 0])
            y, r = d.decode(bytes(g["fix_bits"][i, :n0]), tuple(int(v) for v in g["fix_nbytes"][i]), 4)
            assert r == -12, (arith, i, r)
        d16 = sim.SimDecoder(arith=arith)
        for i in range(3):
            y, r = d16.decode(pk32[i][0], pk32[i][1], 4)
            assert r == -12, (arith, i, r)
        d16.close()
        fresh = sim.SimDecoder(arith=arith, samplerate=32000)
        ya, ra = d.decode(pk32[0][0], pk32[0][1], 4)
        yb, rb = fresh.decode(pk32[0][0], pk32[0][1], 4)
        assert ra == rb == 0 and np.array_equal(ya, yb)
        d.close(), fresh.close()


def test_low_rate_handset_stream_is_rejected_not_misdecoded(ref, sim):
    """A reference 32 kHz encoder below the 16 kHz-core range (12 kb/s) codes a lower core; every such packet is -12 here."""
    x = with_high_band(load_clip()[:640 * 10])
    e = ref.RefEncoder("fix", rate=12000, samplerate=32000)
    d = sim.SimDecoder(samplerate=32000)
    for p in range(10):
        b, nb, n = e.encode(x[p * 1280:(p + 1) * 1280])
        assert d.decode(*receive(b, nb, 4))[1] == -12
    e.close(), d.close()


@pytest.mark.parametrize("cfg,rate,mdi,dtx,loss", LOCKSTEP, ids=LOCKSTEP_IDS)
def test_lockstep_with_reference_decoders(ref, sim, cfg, rate, mdi, dtx, loss):
    """Reference FIX encoder at 32 kHz -> (receiver under the loss process) -> host model and the reference decoders, float
    and (40 ms packets, joint mode 1) fixed point, over eight signal classes: every packet's PCM identical (0 LSB)."""
    n = 24 if cfg["framesize_ms"] == 40 else 40
    kinds = ["flp"] + (["fix"] if cfg["framesize_ms"] == 40 else [])
    for s, (name, x) in enumerate(signals32(n)):
        e = ref.RefEncoder("fix", rate=rate, dtx=dtx, use_md_index=mdi, samplerate=32000, **cfg)
        k = e.samples
        pk = [e.encode(x[p * k:(p + 1) * k]) for p in range(n)]
        e.close()
        fl = flags_for(loss, n, s)
        for kind in kinds:
            dr = ref.RefDecoder(kind, use_md_index=mdi, samplerate=32000, **cfg)
            ds = sim.SimDecoder(use_md_index=mdi, arith=kind, samplerate=32000, **cfg)
            for p, (b, nb, _) in enumerate(pk):
                rx = receive(b, nb, fl[p])
                (ya, ra), (yb, rb) = dr.decode(*rx), ds.decode(*rx)
                assert ra == rb == 0, (name, kind, p, ra, rb)
                assert np.array_equal(ya, yb), (name, kind, p, "PCM differs (0 LSB bar)", int(np.abs(ya.astype(int) - yb).max()))
            dr.close(), ds.close()


def test_32k_decoder_survives_malformed_packets_under_asan(tmp_path):
    """The ASan / UBSan fuzzer of tests/hostsim/fuzz_dec.cpp with the fixture's 32 kHz packets as its corpus: bit flips,
    garbage, lying lengths, short rows and invalid flags into the 32 kHz decoders of both arithmetics (float 40 ms, 20 ms
    and joint mode 1; fixed point 40 ms and joint mode 1).  Every mode both decodes and rejects some of them."""
    f = mk.load()
    corpus = tmp_path / "corpus32.bit"
    with open(corpus, "wb") as out:
        for s in mk.STREAMS:
            for b, nb in mk.packets(f, s):
                out.write(np.array(nb, np.int16).tobytes() + (b if nb[0] > 0 else b""))
    counts = fuzz_decoder(1500, 11, corpus)
    assert sorted(counts) == ["32k fix 40ms", "32k fix joint", "32k flp 20ms", "32k flp 40ms", "32k flp joint"], counts
    assert all(ok > 0 and bad > 0 and ok + bad == 1500 for ok, bad in counts.values()), counts
