#!/usr/bin/env python3
"""Regenerate tests/golden/golden_fixdec.npz: what the reference's fixed-point decoder (oracle/_ref/libjc1_fix.so, built by
`make -C oracle`) makes of the clip's bitstreams -- the parity target of the decoder's fixed-point mode.

    python tests/golden/make_golden_fixdec.py

The PCM itself is not stored (six streams of 191 x 640 samples would be megabytes); each stream is pinned by the md5 of
every packet's PCM and of the whole stream, which is as strict as the samples (the bar is 0 LSB) and names the first
packet that differs.
  fix_pcm_{mode4,mode2,mode3,loss50}_{md5,packet_md5}
        golden.npz's 40 ms FIX bitstream of the clip under lostflag 4 / 2 / 3 and golden.npz's loss50_flags; mode4's md5 is
        the one SURVEY.md 7.2 records for the reference CLI (149ad62f...)
  joint_bits / joint_nbytes            the FIX encoder's joint-mode-1 payloads of the clip (13.6 kb/s)
  joint_loss30_flags                   the driver's loss process at 30 %, seed 2
  joint_pcm_{mode4,loss30}_{md5,packet_md5}   their FIX decoder PCM, loss-free and under joint_loss30_flags
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import ref  # noqa: E402
from tests.util import encode_signal, loss_flags, trim_payload  # noqa: E402

OUT = os.path.join(HERE, "golden_fixdec.npz")


def packet_md5(pcm_rows):
    """uint8 [packets, 16]: md5 of each packet's int16 PCM."""
    return np.array([np.frombuffer(hashlib.md5(np.ascontiguousarray(x, np.int16).tobytes()).digest(), np.uint8) for x in pcm_rows])


def decode_fix(pk, flags, **cfg):
    """Per-packet PCM of the FIX decoder for packets [(payload, (n0, n1))] under lostflags."""
    d = ref.RefDecoder("fix", **cfg)
    out = []
    for (b, nb), f in zip(pk, flags):
        pb, pnb = trim_payload(b, nb, f)
        x, r = d.decode(pb, pnb, f)
        assert r == 0
        out.append(x)
    d.close()
    return out


def fixture():
    """The contents of golden_fixdec.npz (also used by tests/test_fix_decoder.py to re-derive it from the oracle)."""
    g = np.load(os.path.join(HERE, "golden.npz"))
    clip = np.load(os.path.join(HERE, "speech_clip.npz"))["pcm"]
    pk = [(bytes(g["fix_bits"][i, :int(g["fix_nbytes"][i, 0])]), tuple(int(v) for v in g["fix_nbytes"][i]))
          for i in range(len(g["fix_nbytes"]))]
    streams = {"fix_pcm_mode%d" % m: decode_fix(pk, [m] * len(pk)) for m in (4, 2, 3)}
    streams["fix_pcm_loss50"] = decode_fix(pk, [int(v) for v in g["loss50_flags"]])
    f = {}
    jp = encode_signal(ref.RefEncoder("fix", rate=13600, joint_hb=1), clip)
    f["joint_bits"] = np.zeros((len(jp), 128), np.uint8)
    f["joint_nbytes"] = np.zeros((len(jp), 2), np.int16)
    for i, (b, nb, n) in enumerate(jp):
        f["joint_bits"][i, :len(b)] = np.frombuffer(b, np.uint8)
        f["joint_nbytes"][i] = nb
    jpk = [(b, nb) for b, nb, n in jp]
    f["joint_loss30_flags"] = np.array(loss_flags(len(jpk), 30, seed=2), np.int32)
    streams["joint_pcm_mode4"] = decode_fix(jpk, [4] * len(jpk), joint_hb=1)
    streams["joint_pcm_loss30"] = decode_fix(jpk, [int(v) for v in f["joint_loss30_flags"]], joint_hb=1)
    for k, rows in streams.items():
        f[k + "_md5"] = hashlib.md5(np.concatenate(rows).tobytes()).hexdigest()
        f[k + "_packet_md5"] = packet_md5(rows)
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
