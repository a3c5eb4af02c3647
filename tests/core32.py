"""What the 32 kHz decoder tests share (tests/test_dec32*.py on the CPU, tests/test_gpu_dec32*.py on the GPU): the decoder
configurations, the skip check for the reference with its low band tapped, the signal classes and lockstep matrix beyond
the fixture, and the loss and damage processes."""
import numpy as np
import pytest

from tests.golden import make_golden_32k as mk
from tests.util import chirp, load_clip, loss_flags, loss_with_bursts, receive, upsample2, with_high_band

# (configuration, arithmetics): every configuration of the 32 kHz decoder in each arithmetic that has it
CONFIGS = [("40ms", dict(framesize_ms=40), ("flp", "fix")), ("20ms", dict(framesize_ms=20), ("flp",)),
           ("joint", dict(framesize_ms=40, joint_hb=1), ("flp", "fix"))]
MODES = [(name, cfg, kind) for name, cfg, kinds in CONFIGS for kind in kinds]
MODE_IDS = ["%s-%s" % (kind, name) for name, cfg, kind in MODES]
# the decoder keyword arguments of core output: oracle.ref.RefDecoder (the tapped reference), sim.SimDecoder, DecoderBatch
CORE = dict(samplerate=32000, out_samplerate=16000)


def stream_of(cfg):
    """The last golden_32k.npz stream of a configuration."""
    return [s for s in mk.STREAMS if mk.STREAMS[s][1] == cfg][-1]


@pytest.fixture(scope="module")
def tap(ref):
    """Skips where oracle/_ref's tap libraries are not built."""
    if not ref.lowband_available():
        pytest.skip("oracle/_ref's low-band tap libraries not built (make -C oracle -f lowband.mk)")


def mixed_loss(n, seed):
    """A per-packet loss process over all four lostflags (both, MD1 only, MD2 + high band only, none), in runs, so that
    concealment, recovery and single-description decoding follow each other."""
    rng = np.random.Generator(np.random.PCG64(seed))
    out, fl = [], 4
    for _ in range(n):
        if rng.random() < 0.35:
            fl = int(rng.choice([1, 2, 3, 4], p=[0.4, 0.2, 0.2, 0.2]))
        out.append(fl)
    return out


def malformed_sequence(f, g, stream, n, seed):
    """(payload, nbytes, lostflag) of n packets of a fixture stream of which about half are damaged: random bytes, a
    16 kHz stream's packet (8 kHz core), a 32 kHz stream's packet at 12 kb/s (a lower core), lying lengths or an invalid
    lostflag."""
    from oracle.ref import RefEncoder
    rng = np.random.Generator(np.random.PCG64(seed))
    e = RefEncoder("fix", rate=12000, samplerate=32000, **mk.STREAMS[stream][1])
    k = e.samples
    x = with_high_band(load_clip()[:k // 2 * n])
    low_core = [e.encode(x[p * k:(p + 1) * k])[:2] for p in range(n)]
    e.close()
    pk = mk.packets(f, stream)
    out = []
    for p in range(n):
        b, nb, fl = receive(*pk[p], 4)
        kind = int(rng.integers(0, 10))
        if kind == 0:
            b = rng.integers(0, 256, max(len(b), 8), dtype=np.uint8).tobytes()
        elif kind == 1:
            n0 = int(g["fix_nbytes"][p, 0])
            b, nb = bytes(g["fix_bits"][p, :n0]), tuple(int(v) for v in g["fix_nbytes"][p])
        elif kind == 2:
            b, nb, fl = receive(*low_core[p], 4)
        elif kind == 3:
            nb = (int(rng.integers(-5, 400)), int(rng.integers(-5, 400)))
        elif kind == 4:
            fl = int(rng.integers(-3, 9))
        out.append((b, nb, fl))
    return out


def signals32(n_packets, seed=11):
    """(name, int16 32 kHz signal) classes beyond the fixture: speech with noise, zeros, DC, full-scale square, a chirp over
    the whole band, loud noise, 2 kHz sine, speech fading to silence (for DTX)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    clip = load_clip()
    L = 1280 * n_packets
    t = np.arange(L)
    sp = with_high_band(clip)[:L]
    fade = (upsample2(clip)[:L] * np.clip(1.0 - t / (0.6 * L), 0, 1)).astype(np.int16)
    return [
        ("speech_hb", sp),
        ("zeros", np.zeros(L, np.int16)),
        ("dc", np.full(L, 1000, np.int16)),
        ("square", np.where((t // 40) % 2 == 0, 32767, -32767).astype(np.int16)),
        ("chirp", chirp(L)),
        ("noise20000", np.clip(rng.normal(0, 20000, L), -32768, 32767).astype(np.int16)),
        ("sine2k", (8000 * np.sin(2 * np.pi * 2000 * t / 32000)).astype(np.int16)),
        ("fade", fade),
    ]


LOCKSTEP = [
    # (configuration, rate, use_md_index, dtx, loss process)
    (dict(framesize_ms=40), 15600, 0, 0, "none"),
    (dict(framesize_ms=40), 32000, 1, 1, "bursts"),
    (dict(framesize_ms=40), 64000, 0, 0, "first"),
    (dict(framesize_ms=20), 24000, 1, 0, "bursts"),
    (dict(framesize_ms=20), 15600, 0, 1, "first"),
    (dict(framesize_ms=40, joint_hb=1), 14800, 0, 0, "bursts"),
    (dict(framesize_ms=40, joint_hb=1), 40000, 1, 1, "first"),
]
LOCKSTEP_IDS = ["%s-%d-mdi%d-dtx%d-%s" % ("joint" if c.get("joint_hb") else "%dms" % c["framesize_ms"], r, m, d, l)
                for c, r, m, d, l in LOCKSTEP]


def flags_for(kind, n, s):
    """The lostflags of n packets under loss process `kind` ("none", "first" or "bursts"), seeded by s."""
    if kind == "none":
        return [4] * n
    if kind == "first":        # loss from the very first packet (a lost burst before anything was decoded), then 30 %
        fl = loss_flags(n, 30, seed=7 + s)
        return [1] * 4 + fl[4:]
    # row 1: loss_with_bursts leaves every fifth row loss-free, row 0 among them
    return [int(v) for v in loss_with_bursts(n, 2, seed=20 + s)[1]]
