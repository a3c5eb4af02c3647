"""What the core-output tests of 32 kHz streams share (tests/test_dec32_core.py on the CPU, tests/test_gpu_dec32_core.py on
the GPU): the decoder configurations, the reference with its low band tapped, and the loss and damage processes."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import ref
from tests.ref32 import Ref32Decoder
from tests.util import load_clip, receive

# (configuration, arithmetics): every configuration of the 32 kHz decoder in each arithmetic that has it
CONFIGS = [("40ms", dict(framesize_ms=40), ("flp", "fix")), ("20ms", dict(framesize_ms=20), ("flp",)),
           ("joint", dict(framesize_ms=40, joint_hb=1), ("flp", "fix"))]
MODES = [(name, cfg, kind) for name, cfg, kinds in CONFIGS for kind in kinds]
MODE_IDS = ["%s-%s" % (kind, name) for name, cfg, kind in MODES]


def stream_of(cfg):
    """The last golden_32k.npz stream of a configuration."""
    from tests.golden import make_golden_32k as mk
    return [s for s in mk.STREAMS if mk.STREAMS[s][1] == cfg][-1]


class Ref32LowbandDecoder(Ref32Decoder):
    """A 32 kHz reference decoder of the build with the low-band tap (oracle/lowband.mk, kind = 'flp' or 'fix'): decode()
    returns the full-band PCM and the return value as Ref32Decoder's, and leaves in `low` the int16 low band that packet
    handed to the synthesis filter bank (AGR_Sate_qmf_synth's first argument, 16 * framesize_ms samples), or None when the
    filter bank did not run (a rejected packet).  The tap records one low band per library, so decode calls of the same
    kind must not overlap."""

    def __init__(self, kind="flp", use_md_index=0, framesize_ms=40, joint_hb=0):
        super().__init__(kind + "_lowband", use_md_index=use_md_index, framesize_ms=framesize_ms, joint_hb=joint_hb)
        self.L.lowband_take.argtypes = [C.c_void_p, C.c_int]
        self._low = np.zeros(640, np.int16)
        self.L.lowband_take(self._low.ctypes.data, self._low.size)
        self.low = None

    def decode(self, payload, nbytes, lostflag):
        pcm, ret = super().decode(payload, nbytes, lostflag)
        n = self.L.lowband_take(self._low.ctypes.data, self._low.size)
        assert n in (0, self.samples // 2), n
        self.low = self._low[:n].copy() if n else None
        return pcm, ret


def lowband_available():
    return all(os.path.exists(os.path.join(ref.REF_DIR, "libjc1_%s_lowband.so" % k)) for k in ("flp", "fix"))


@pytest.fixture(scope="module")
def tap(ref):
    """The tapped reference decoder class; skips where oracle/_ref's tap libraries are not built."""
    if not lowband_available():
        pytest.skip("oracle/_ref's low-band tap libraries not built (make -C oracle -f lowband.mk)")
    return Ref32LowbandDecoder


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
    from tests.ref32 import Ref32Encoder, with_high_band
    rng = np.random.Generator(np.random.PCG64(seed))
    from tests.golden import make_golden_32k as mk
    cfg = mk.STREAMS[stream][1]
    e = Ref32Encoder("fix", rate=12000, **cfg)
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
