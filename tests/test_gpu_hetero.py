"""Batched parity with *different* signal classes in neighbouring streams (SURVEY.md 8(d) ii/iii): the warps of a block, the
two lane groups of a quantiser warp and the 64 threads of an entropy-coding / decoder block then take different paths
(voiced / unvoiced, different decision delays, rewhitening, DTX-like silence, clipping) at the same time.
Every row is compared with the unmodified reference run per stream: payload bytes + length fields against libjc1_fix.so,
decoded PCM under a per-stream 50 % loss process against libjc1_flp.so fed the same payloads and flags.
Tolerances: payloads bit-exact; PCM 0 LSB (the north star allows +-1)."""
import numpy as np
import pytest

from tests.parity import DevicePath, RefRows, ref, sb  # noqa: F401  (fixtures)
from tests.util import load_clip, loss_flags, signal_classes, speech_replay

pytestmark = pytest.mark.gpu


def run_against_reference(sb, ref, x, rate, loss_perc=50):
    """x: [T, N, 640].  GPU batch vs one reference encoder + decoder per row; the batch decoder gets what the receiver makes
    of the reference's payloads."""
    T, N, _ = x.shape
    cap = 1024 if rate > 40000 else 256
    eb, db = sb.EncoderBatch(N, rate=rate), sb.DecoderBatch(N)
    rr = RefRows(ref, range(N), decode="ref", rate=rate)
    flags = np.array([loss_flags(T, loss_perc, seed=1 + s) for s in range(N)], np.int32)
    flags[::5] = 4           # every fifth row loss-free
    for p in range(T):
        bits, nb = eb.encode(x[p], cap=cap)
        tb, tnb, tf = rr.step(x[p], bits, nb, flags[:, p])
        pcm, ret = db.decode(tb, tnb, tf)
        assert (ret == 0).all()
        rr.check_pcm(pcm)
    rr.close()
    eb.close(); db.close()


def test_neighbouring_streams_of_eight_signal_classes_match_the_reference(sb, ref):
    x = signal_classes(load_clip(), 256, 40)
    run_against_reference(sb, ref, x, rate=13600)


@pytest.mark.parametrize("rate", [6000, 24000, 100000])
def test_signal_classes_at_other_rates(sb, ref, rate):
    x = signal_classes(load_clip(), 64, 20, seed=rate)
    run_against_reference(sb, ref, x, rate=rate)


def test_full_batch_sample_of_1024_streams_25_packets(sb, ref):
    """BASELINE configs 3 + 5 at full size (65 536 streams, per-stream loss process, trimming on the device): 1 024 streams
    spread over the batch x 25 packets against the reference (SURVEY.md 8(d) config 4 wording)."""
    N, T, cap = 65536, 25, 128
    clip = load_clip()
    sample = sorted(set(list(range(0, N, 64))))[:1024]
    flags = np.full((N, T), 4, np.int32)
    for s in sample:
        flags[s] = loss_flags(T, 50, seed=1 + s)
    rng = np.random.Generator(np.random.PCG64(11))
    other = rng.integers(1, 5, size=(N, T)).astype(np.int32)
    mask = np.ones(N, bool); mask[sample] = False
    flags[mask] = other[mask]
    eb, db = sb.EncoderBatch(N), sb.DecoderBatch(N)
    dp, rr = DevicePath(sb, eb, db, cap=cap), RefRows(ref, sample, decode="ref", rate=13600)
    for p in range(T):
        xh = speech_replay(clip, N, 1, first_packet=p)[0]
        dp.encode(xh)
        dp.decode(flags[:, p])
        bits, nb, pcm = dp.rows(sample)
        rr.step(xh[sample], bits, nb, flags[sample, p])
        rr.check_pcm(pcm)
    rr.close()
    eb.close(); db.close()
