"""Core output of 32 kHz streams on the CPU: the host model's core-output decoder (tests/hostsim, dec_packet<16, true> of
sb_dec.cuh) against the low band the reference's decoders hand to their synthesis filter bank, at 0 LSB.

The reference is tapped, not changed: oracle/lowband.mk links its untouched sources with -Wl,--wrap=AGR_Sate_qmf_synth, and
oracle.ref.RefDecoder(..., samplerate=32000, out_samplerate=16000) returns what the wrapper recorded (the float build's
`lowout`, the fixed-point build's `OutLow`)."""
import numpy as np
import pytest

from tests.core32 import (CORE, LOCKSTEP, LOCKSTEP_IDS, MODE_IDS, MODES, flags_for, malformed_sequence, mixed_loss,  # noqa: F401
                          signals32, stream_of, tap)  # (tap: fixture)
from tests.golden import make_golden_32k as mk
from tests.parity import ref, sim  # noqa: F401  (fixtures)
from tests.util import load_clip, load_golden, receive, upsample2


def core_lockstep(ref, sim, kind, cfg, pk, flags, tag=()):
    """The tapped reference decoder and the host model's core output over what the receiver makes of the packets pk under
    flags: both return 0, and every row equals the reference's low band (0 LSB).  Returns the number of rows compared."""
    dr = ref.RefDecoder(kind, **CORE, **cfg)
    ds = sim.SimDecoder(arith=kind, **CORE, **cfg)
    assert ds.pcm.size == 16 * cfg["framesize_ms"]
    for p, ((b, nb), fl) in enumerate(zip(pk, flags)):
        x = receive(b, nb, fl)
        (low, ra), (y, rb) = dr.decode(*x), ds.decode(*x)
        assert ra == rb == 0, (kind, p, ra, rb) + tuple(tag)
        assert low.size == y.size and np.array_equal(y, low), \
            (kind, p, "core row differs from the reference's low band (0 LSB bar)", int(np.abs(y.astype(int) - low).max())) + tuple(tag)
    dr.close(), ds.close()
    return len(pk)


CASES = mk.decode_cases()


@pytest.mark.parametrize("key,stream,kind,rule", CASES, ids=[c[0] for c in CASES])
def test_tap_leaves_the_reference_pcm_alone(ref, tap, key, stream, kind, rule):
    """The tapped library decodes every pinned 32 kHz decode exactly as the untapped one (the fixture's per-packet md5),
    and records a low band of 16 * framesize_ms samples for every packet."""
    f = mk.load()
    d = ref.RefDecoder(kind, **CORE, **mk.STREAMS[stream][1])
    lows = []

    class Recording:
        def decode(self, *a):
            low, r = d.decode(*a)
            lows.append(low)
            return d.full, r

        def close(self):
            d.close()
    rows = mk.decode(Recording(), mk.packets(f, stream), mk.flags_of(f, stream, rule))
    assert (mk.packet_md5(rows) == f[key + "_packet_md5"]).all()
    assert all(x.size == 16 * mk.STREAMS[stream][1]["framesize_ms"] for x in lows)


@pytest.mark.parametrize("key,stream,kind,rule", CASES, ids=[c[0] for c in CASES])
def test_core_rows_equal_the_reference_low_band(ref, sim, tap, key, stream, kind, rule):
    """Every stream of golden_32k.npz under each of its pinned lostflag sequences, in the arithmetic of that decode."""
    f = mk.load()
    pk, flags = mk.packets(f, stream), mk.flags_of(f, stream, rule)
    assert core_lockstep(ref, sim, kind, mk.STREAMS[stream][1], pk, flags, (key,)) == len(pk)


@pytest.mark.parametrize("name,cfg,kind", MODES, ids=MODE_IDS)
def test_core_rows_under_mixed_loss(ref, sim, tap, name, cfg, kind):
    """Every fixture stream of the configuration under its own mixed loss process over lostflags 1 / 2 / 3 / 4."""
    f = mk.load()
    streams = [s for s in mk.STREAMS if mk.STREAMS[s][1] == cfg]
    assert streams
    for i, s in enumerate(streams):
        pk = mk.packets(f, s)
        fl = mixed_loss(len(pk), seed=40 + i)
        assert {1, 2, 3, 4} <= set(fl)
        core_lockstep(ref, sim, kind, cfg, pk, fl, (s,))


@pytest.mark.parametrize("name,cfg,kind", MODES, ids=MODE_IDS)
def test_core_rows_with_dtx(ref, sim, tap, name, cfg, kind):
    """The reference FIX encoder at 32 kHz with DTX on speech fading to silence (DTX packets are concealed as lost, comfort
    noise follows), clean and under the mixed loss process."""
    clip = load_clip()
    n = 30 if cfg["framesize_ms"] == 40 else 50
    k = 32 * cfg["framesize_ms"]
    L = n * k
    t = np.arange(L)
    x = (upsample2(clip)[:L] * np.clip(1.0 - t / (0.5 * L), 0, 1)).astype(np.int16)
    e = ref.RefEncoder("fix", rate=24000, dtx=1, samplerate=32000, **cfg)
    pk = [e.encode(x[p * k:(p + 1) * k])[:2] for p in range(n)]
    e.close()
    assert sum(nb[0] <= 0 for _, nb in pk) >= 3, "the signal must produce DTX packets"
    core_lockstep(ref, sim, kind, cfg, pk, [4] * n, ("dtx",))
    core_lockstep(ref, sim, kind, cfg, pk, mixed_loss(n, seed=77), ("dtx", "loss"))


@pytest.mark.parametrize("cfg,rate,mdi,dtx,loss", LOCKSTEP, ids=LOCKSTEP_IDS)
def test_core_rows_over_signal_classes(ref, sim, tap, cfg, rate, mdi, dtx, loss):
    """The full-band lockstep's matrix (tests/test_dec32.py) at core output: the reference FIX encoder at 32 kHz over the
    eight signal classes at the row's rate, use_md_index and DTX, under its loss process; float rows for every
    configuration, fixed-point rows for 40 ms packets and joint mode 1."""
    n = 24 if cfg["framesize_ms"] == 40 else 40
    kinds = ["flp"] + (["fix"] if cfg["framesize_ms"] == 40 else [])
    for s, (name, x) in enumerate(signals32(n)):
        e = ref.RefEncoder("fix", rate=rate, dtx=dtx, use_md_index=mdi, samplerate=32000, **cfg)
        k = e.samples
        pk = [e.encode(x[p * k:(p + 1) * k])[:2] for p in range(n)]
        e.close()
        for kind in kinds:
            core_lockstep(ref, sim, kind, dict(cfg, use_md_index=mdi), pk, flags_for(loss, n, s), (name,))


@pytest.mark.parametrize("name,cfg,kind", MODES, ids=MODE_IDS)
def test_return_codes_equal_the_full_band_decoders(ref, sim, name, cfg, kind):
    """Damaged and other-core packets between good ones: the core-output host model returns exactly what the full-band
    one returns for every packet (-12 for the other cores), and both reject some and decode some."""
    f, g = mk.load(), load_golden()
    stream = stream_of(cfg)
    seq = malformed_sequence(f, g, stream, 40, seed=5)
    core = sim.SimDecoder(arith=kind, **CORE, **cfg)
    full = sim.SimDecoder(arith=kind, samplerate=32000, **cfg)
    rets = []
    for p, (b, nb, fl) in enumerate(seq):
        ya, ra = core.decode(b, nb, fl)
        yb, rb = full.decode(b, nb, fl)
        assert ra == rb, (p, ra, rb)
        rets.append(ra)
    assert 0 in rets and -12 in rets and any(r < 0 and r != -12 for r in rets), rets
    core.close(), full.close()
