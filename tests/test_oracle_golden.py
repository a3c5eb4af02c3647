"""The oracle (the UNMODIFIED reference compiled into oracle/_ref by `make -C oracle`) against the committed golden
fixtures.  This is what pins parity: tests/golden/golden.npz was produced by tests/golden/make_golden.py from the same
libraries, and the md5 values recorded in SURVEY.md 7.2 for the reference CLI agree with it.  If the fixtures and the
oracle ever disagree (different compiler, different flags) every other parity statement is void, so check it first.
Skipped where oracle/_ref is not built (it needs /root/reference; the GPU box receives the prebuilt libraries)."""
import hashlib

import numpy as np
import pytest

from tests.parity import ref  # noqa: F401  (fixture)
from tests.util import bitfile, encode_signal, load_clip, load_golden, synth_inputs, trim_payload


@pytest.fixture(scope="module")
def clip_packets(ref):
    return encode_signal(ref.RefEncoder("fix", rate=13600), load_clip())


def test_fix_encoder_reproduces_golden_bitstream(clip_packets):
    g = load_golden()
    assert len(clip_packets) == g["fix_nbytes"].shape[0] == 191
    assert hashlib.md5(bitfile(clip_packets)).hexdigest() == str(g["fix_bitfile_md5"])
    for i, (b, nb, n) in enumerate(clip_packets):
        assert nb == tuple(g["fix_nbytes"][i]) and n == nb[0]
        assert b == bytes(g["fix_bits"][i, :n])


@pytest.mark.parametrize("mode", [4, 2, 3, "loss50"])
def test_flp_decoder_reproduces_golden_pcm(ref, clip_packets, mode):
    g = load_golden()
    flags = list(g["loss50_flags"]) if mode == "loss50" else [mode] * len(clip_packets)
    key = "flp_pcm_loss50" if mode == "loss50" else "flp_pcm_mode%d" % mode
    d = ref.RefDecoder("flp")
    out = []
    for (b, nb, n), f in zip(clip_packets, flags):
        pb, pnb = trim_payload(b, nb, int(f))
        x, r = d.decode(pb, pnb, int(f))
        assert r == 0
        out.append(x)
    d.close()
    pcm = np.concatenate(out)
    assert hashlib.md5(pcm.tobytes()).hexdigest() == str(g[key + "_md5"])
    assert np.array_equal(pcm, g[key])


def test_fix_encoder_reproduces_synthetic_hashes(ref):
    g = load_golden()
    for name, x, kw in synth_inputs(load_clip()):
        assert hashlib.md5(bitfile(encode_signal(ref.RefEncoder("fix", **kw), x))).hexdigest() == str(g["synth_" + name]), name


def test_loss_process_matches_fixture():
    """tests/util.loss_flags restates the reference driver's loss process (dec_main.c:24,227-307)."""
    from tests.util import loss_flags
    g = load_golden()
    assert loss_flags(len(g["loss50_flags"]), 50, seed=1) == [int(v) for v in g["loss50_flags"]]
    assert set(loss_flags(400, 0)) == {4} and set(loss_flags(400, 100)) == {1}


def test_flp_encoder_leg_of_config0(ref):
    """BASELINE configs[0] runs the FLP tree's own CLI: FLP encode -> FLP decode of the reference clip.  The product's
    bitstream target is the FIX encoder, but the oracle build is pinned on this leg too: the FLP encoder's .bit file has the
    md5 SURVEY.md 7.2 recorded for the reference CLI (it moves under FMA contraction, which is why oracle/Makefile builds with
    -ffp-contract=off), and the FLP decoder decodes it without error."""
    pk = encode_signal(ref.RefEncoder("flp", rate=13600), load_clip())
    bf = bitfile(pk)
    assert len(bf) == 16545 and hashlib.md5(bf).hexdigest() == "26da320f33e8d8f9f0043df37765533c"
    d = ref.RefDecoder("flp")
    for b, nb, n in pk:
        x, r = d.decode(b, nb, 4)
        assert r == 0 and x.shape == (640,)
    d.close()
