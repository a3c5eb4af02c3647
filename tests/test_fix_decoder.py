"""The decoder's fixed-point arithmetic (SOLO_B200_DEC_FIX) on the CPU: the host model of the kernel source against the
reference's fixed-point build (JC1_SDK_SRC_ARM), at 0 LSB.

The reference ships a float and a fixed-point build whose decoded PCM differs in the high-band synthesis and the synthesis
filter bank.  tests/golden/golden_fixdec.npz pins the fixed-point build's PCM of the clip's bitstreams by per-packet md5
(made by tests/golden/make_golden_fixdec.py); where oracle/_ref is built, the fixture is re-derived from it and the host
model runs in lockstep with the fixed-point decoder on inputs the fixture does not cover.  The decoder's fuzzer
(tests/test_fuzz_decoder.py) covers the fixed-point arithmetic on malformed packets."""
import hashlib
import os

import numpy as np
import pytest

from tests.golden.make_golden_32k import packet_md5
from tests.parity import lockstep, ref, sim  # noqa: F401  (fixtures)
from tests.util import GOLDEN, load_clip, load_golden, loss_flags, loss_with_bursts, signal_classes, synth_inputs, trim_payload

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI_MD5 = "149ad62fe193f19d6c80aacc7336ebce"    # the reference CLI's fixed-point decode of the clip at loss 0 (SURVEY.md 7.2)


def load_fixdec():
    return np.load(os.path.join(GOLDEN, "golden_fixdec.npz"))


def fixture_case(case):
    """(packets [(payload, (n0, n1))], lostflags, decoder kwargs, fixture key) of one fixture stream."""
    g, f = load_golden(), load_fixdec()
    if case.startswith("joint"):
        bits, nbytes, kw = f["joint_bits"], f["joint_nbytes"], dict(joint_hb=1)
    else:
        bits, nbytes, kw = g["fix_bits"], g["fix_nbytes"], {}
    pk = [(bytes(bits[i, :int(nbytes[i, 0])]), tuple(int(v) for v in nbytes[i])) for i in range(len(nbytes))]
    flags = {"mode4": [4] * len(pk), "mode2": [2] * len(pk), "mode3": [3] * len(pk), "loss50": [int(v) for v in g["loss50_flags"]],
             "joint_mode4": [4] * len(pk), "joint_loss30": [int(v) for v in f["joint_loss30_flags"]]}[case]
    key = ("joint_pcm_" + case[6:]) if case.startswith("joint") else "fix_pcm_" + case
    return pk, flags, kw, key


def decode_all(dec, pk, flags):
    """Per-packet PCM of one decoder over a packet sequence (every return value 0); closes the decoder."""
    out = []
    for (b, nb), fl in zip(pk, flags):
        pb, pnb = trim_payload(b, nb, fl)
        x, r = dec.decode(pb, pnb, fl)
        assert r == 0
        out.append(x)
    dec.close()
    return out


CASES = ["mode4", "mode2", "mode3", "loss50", "joint_mode4", "joint_loss30"]


@pytest.mark.parametrize("case", CASES)
def test_host_model_matches_fixture(sim, case):
    pk, flags, kw, key = fixture_case(case)
    rows = decode_all(sim.SimDecoder(arith="fix", **kw), pk, flags)
    f = load_fixdec()
    got = packet_md5(rows)
    bad = np.nonzero((got != f[key + "_packet_md5"]).any(axis=1))[0]
    assert bad.size == 0, (case, "first packet that differs", int(bad[0]) if bad.size else None)
    md5 = hashlib.md5(np.concatenate(rows).tobytes()).hexdigest()
    assert md5 == str(f[key + "_md5"])
    if case == "mode4":
        assert md5 == CLI_MD5


def test_fixture_differs_from_the_float_build():
    """The two builds really decode differently, so the tests above could not pass on the float arithmetic."""
    g, f = load_golden(), load_fixdec()
    flp = packet_md5(g["flp_pcm_mode4"].reshape(-1, 640))
    assert (flp != f["fix_pcm_mode4_packet_md5"]).any(axis=1).sum() > 150


def test_float_arithmetic_of_the_same_build_matches_golden(sim):
    """The same host build with arith = flp reproduces the float build's golden PCM: the mode switch is what differs."""
    pk, flags, kw, _ = fixture_case("mode4")
    rows = decode_all(sim.SimDecoder(arith="flp", **kw), pk, flags)
    assert np.array_equal(np.concatenate(rows), load_golden()["flp_pcm_mode4"])


def test_fixture_matches_oracle(ref):
    """golden_fixdec.npz re-derived from the fixed-point library of oracle/_ref: fixture and oracle cannot drift apart."""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    try:
        import make_golden_fixdec
    finally:
        sys.path.pop(0)
    want = make_golden_fixdec.fixture()
    f = load_fixdec()
    assert sorted(want) == sorted(f.files)
    for k in want:
        assert np.array_equal(np.asarray(want[k]), f[k]), k


@pytest.fixture(scope="module")
def fix_pairs(ref, sim):
    def make(**cfg):
        """(FIX encoder, FIX decoder) of the reference and (encoder, fixed-point decoder) of the host model."""
        dcfg = {k: v for k, v in cfg.items() if k not in ("rate", "dtx")}
        return (ref.RefEncoder("fix", **cfg), ref.RefDecoder("fix", **dcfg)), (sim.SimEncoder(**cfg), sim.SimDecoder(arith="fix", **dcfg))
    return make


def test_signal_classes_match_reference(fix_pairs):
    """Speech, noise, silence, DC, full-scale square, sine and clipped speech: the saturation paths of the integer high-band
    filter (ADD_SAT32, LSHIFT_SAT32, SAT16) and of the filter bank (SATURATE32 to +-32767), with 30 % loss."""
    x = signal_classes(load_clip(), 8, 25)
    for s in range(8):
        lockstep(*fix_pairs(), x[:, s], loss_flags(25, 30, seed=11 + s), tag=("class", s))


@pytest.mark.parametrize("name", ["rate6000", "rate24000", "rate100000", "clip4x", "noise20000", "zeros", "dc1000", "square100", "mdi"])
def test_synthetic_inputs_match_reference(fix_pairs, name):
    """Rates 6 / 24 / 100 kb/s, the MD index flag and the synthetic signals, loss-free for 20 packets, then under loss."""
    _, x, kw = next(c for c in synth_inputs(load_clip()) if c[0] == name)
    P = min(len(x) // 640, 45)
    flags = [4] * 20 + loss_flags(P - 20, 40, seed=3)
    lockstep(*fix_pairs(**kw), x[:P * 640].reshape(P, 640), flags, tag=(name,))


def test_loss_bursts_and_loss_from_the_first_packet(fix_pairs):
    """The driver's 20 % process with a burst of 10-14 lost packets per stream, and streams whose first packets are lost
    (concealment from the initial state, then the first good high band)."""
    clip = load_clip()
    T = 40
    flags = loss_with_bursts(T, 4)
    for s in range(4):
        x = clip[(s * 7919 * 640) % (len(clip) - T * 640):][:T * 640].reshape(T, 640)
        lockstep(*fix_pairs(), x, [int(v) for v in flags[s]], tag=("bursts", s))
    for first in ([1, 1, 4], [1, 2, 3], [2, 4], [3, 1, 4], [1] * 6 + [3]):
        fl = first + loss_flags(T - len(first), 20, seed=len(first))
        lockstep(*fix_pairs(), clip[:T * 640].reshape(T, 640), fl, tag=("first", tuple(first)))


def test_joint_mode1_matches_reference(fix_pairs):
    clip = load_clip()
    for rate, dtx, mdi in ((13600, 0, 0), (8000, 0, 1), (24000, 1, 0)):
        lockstep(*fix_pairs(rate=rate, dtx=dtx, use_md_index=mdi, joint_hb=1), clip[:640 * 60].reshape(60, 640),
                 loss_flags(60, 30, seed=9), tag=("joint", rate))

