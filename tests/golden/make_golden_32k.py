#!/usr/bin/env python3
"""Regenerate tests/golden/golden_32k.npz: the reference's 32 kHz streams (API samplerate 32000, 16 kHz SILK core) and what
its two decoders make of them -- the parity target of the 32 kHz decoder.  Needs oracle/_ref (`make -C oracle`).

    python tests/golden/make_golden_32k.py

Inputs, made from speech_clip.npz by fixed rules (tests/util.py):
  up   upsample2(clip): every 16 kHz sample followed by floor((x[n] + x[n+1]) / 2) -- integer-exact
  hb   with_high_band(clip): up plus white noise (sigma 400, PCG64 seed 32), so that 8-16 kHz carries a signal
Streams (FIX encoder at 32 kHz; user rates inside the range that keeps the 16 kHz core, see INTEGRATION.md):
  up40    up, 40 ms packets, 16 000 b/s, the first 60 packets
  hb40    hb, 40 ms packets, 24 000 b/s, the first 100 packets
  hb20    hb, 20 ms packets, 24 000 b/s, the first 120 packets
  joint   hb, joint mode 1, 16 000 b/s, the first 100 packets
Per stream: <s>_bits (all payloads back to back) and <s>_nbytes [packets, 2] (the encoder's length fields).
Loss processes: <s>_loss_flags, the reference driver's at 50 % (30 % for joint, as golden_fixdec.npz), seed 3.
PCM, pinned by md5 of every packet's int16 PCM (<k>_packet_md5 [packets, 16]) and of the whole stream (<k>_md5):
  flp_<s>_mode4 for every stream; flp_hb40_mode2 / _mode3; flp_<s>_loss for hb40, hb20, joint
  fix_<s>_mode4 and fix_<s>_loss for hb40 and joint (the fixed-point decoder has no 20 ms mode)
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.ref import RefDecoder, RefEncoder  # noqa: E402
from tests.util import loss_flags, trim_payload, upsample2, with_high_band  # noqa: E402

OUT = os.path.join(HERE, "golden_32k.npz")
# name: (input, encoder / decoder configuration, rate, packets, loss percentage of the lossy decode or None)
STREAMS = {
    "up40": ("up", dict(framesize_ms=40), 16000, 60, None),
    "hb40": ("hb", dict(framesize_ms=40), 24000, 100, 50),
    "hb20": ("hb", dict(framesize_ms=20), 24000, 120, 50),
    "joint": ("hb", dict(framesize_ms=40, joint_hb=1), 16000, 100, 30),
}


def inputs():
    clip = np.load(os.path.join(HERE, "speech_clip.npz"))["pcm"]
    return {"up": upsample2(clip), "hb": with_high_band(clip)}


def load():
    """The committed fixture."""
    return np.load(OUT)


def packet_md5(pcm_rows):
    """uint8 [packets, 16]: md5 of each packet's int16 PCM."""
    return np.array([np.frombuffer(hashlib.md5(np.ascontiguousarray(x, np.int16).tobytes()).digest(), np.uint8) for x in pcm_rows])


def packets(f, s):
    """[(payload, (n0, n1))] of stream s of a fixture."""
    nb, bits = f[s + "_nbytes"], bytes(f[s + "_bits"])
    out, o = [], 0
    for n0, n1 in nb:
        n = max(int(n0), 0)
        out.append((bits[o:o + n], (int(n0), int(n1))))
        o += n
    return out


def decode_cases():
    """(PCM key, stream, decoder kind, lostflags rule) of every pinned decode: rule 'mode<k>' or 'loss'."""
    out = [("flp_%s_mode4" % s, s, "flp", "mode4") for s in STREAMS]
    out += [("flp_hb40_mode2", "hb40", "flp", "mode2"), ("flp_hb40_mode3", "hb40", "flp", "mode3")]
    out += [("flp_%s_loss" % s, s, "flp", "loss") for s in ("hb40", "hb20", "joint")]
    out += [("fix_%s_%s" % (s, m), s, "fix", m) for s in ("hb40", "joint") for m in ("mode4", "loss")]
    return out


def flags_of(f, s, rule):
    n = len(f[s + "_nbytes"])
    return [int(v) for v in f[s + "_loss_flags"]] if rule == "loss" else [int(rule[4:])] * n


def decode(dec, pk, flags):
    """Per-packet PCM of one decoder over a stream (a DTX packet is concealed as lost); every return value must be 0."""
    out = []
    for (b, nb), fl in zip(pk, flags):
        if nb[0] <= 0:
            pb, pnb, fl = bytes(16), (16, 8), 1
        else:
            pb, pnb = trim_payload(b, nb, fl)
        y, r = dec.decode(pb, pnb, fl)
        assert r == 0, r
        out.append(y)
    dec.close()
    return out


def fixture():
    """The contents of golden_32k.npz (tests/test_dec32.py re-derives it from the oracle where that is built)."""
    x = inputs()
    f = {}
    for s, (src, cfg, rate, n, loss) in STREAMS.items():
        e = RefEncoder("fix", rate=rate, samplerate=32000, **cfg)
        pk = [e.encode(x[src][p * e.samples:(p + 1) * e.samples]) for p in range(n)]
        e.close()
        f[s + "_bits"] = np.frombuffer(b"".join(b for b, _, _ in pk), np.uint8)
        f[s + "_nbytes"] = np.array([nb for _, nb, _ in pk], np.int16)
        f[s + "_loss_flags"] = np.array(loss_flags(n, loss if loss else 50, seed=3), np.int32)
    for key, s, kind, rule in decode_cases():
        rows = decode(RefDecoder(kind, samplerate=32000, **STREAMS[s][1]), packets(f, s), flags_of(f, s, rule))
        f[key + "_md5"] = hashlib.md5(np.concatenate(rows).tobytes()).hexdigest()
        f[key + "_packet_md5"] = packet_md5(rows)
    return f


def main():
    f = fixture()
    np.savez_compressed(OUT, **f)
    for k in sorted(f):
        if isinstance(f[k], str):
            print(k, f[k])
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
