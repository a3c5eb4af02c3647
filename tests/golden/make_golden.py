#!/usr/bin/env python3
"""Regenerate the golden fixtures from the UNMODIFIED reference (oracle/_ref, built by `make -C oracle`).

Run in the build container only (needs /root/reference for the input clip):
    python tests/golden/make_golden.py
Writes:
  speech_clip.npz   the reference's own 16 kHz test clip (JC1_SDK_SRC_ARM/bin/Ch_f1_raw.pcm, 122 421 samples) --
                    an input vector, stored compressed; the reference ships no expected outputs (SURVEY.md 4)
  golden.npz        outputs of the reference on that clip and on synthetic inputs:
                      fix_bits / fix_nbytes   FIX encoder payloads + {n0, n1} per packet, rate 13600 (config 1 / 2 target)
                      flp_pcm_mode{4,2,3}     FLP decoder PCM of those payloads (both / MD1 only / MD2+HB only)
                      flp_pcm_loss50, loss50_flags   FLP decoder PCM under the dec_main.c:229-241 loss process (seed 1)
                      md5 strings of the FIX bit file and of every PCM (cross-checks SURVEY.md 7.2)
                      synth_*                 md5 of FIX payload streams for synthetic inputs / other rates
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref  # noqa: E402
from tests.util import bitfile, encode_signal, loss_flags, synth_inputs, trim_payload  # noqa: E402

CLIP = "/root/reference/JC1_SDK_SRC_ARM/bin/Ch_f1_raw.pcm"
HERE = os.path.dirname(os.path.abspath(__file__))


def decode_stream(pk, flags, mdi=0):
    d = ref.RefDecoder("flp", use_md_index=mdi)
    out = []
    for (b, nb, n), f in zip(pk, flags):
        pb, pnb = trim_payload(b, nb, f)
        x, r = d.decode(pb, pnb, f)
        out.append(x)
    d.close()
    return np.concatenate(out)


def main():
    clip = np.fromfile(CLIP, dtype=np.int16)
    np.savez_compressed(os.path.join(HERE, "speech_clip.npz"), pcm=clip)
    g = {}
    pk = encode_signal(ref.RefEncoder("fix", rate=13600), clip)
    cap = 128
    bits = np.zeros((len(pk), cap), np.uint8)
    nbytes = np.zeros((len(pk), 2), np.int16)
    for i, (b, nb, n) in enumerate(pk):
        bits[i, :len(b)] = np.frombuffer(b, np.uint8)
        nbytes[i] = nb
    g["fix_bits"] = bits
    g["fix_nbytes"] = nbytes
    g["fix_bitfile_md5"] = hashlib.md5(bitfile(pk)).hexdigest()
    for mode in (4, 2, 3):
        pcm = decode_stream(pk, [mode] * len(pk))
        g["flp_pcm_mode%d" % mode] = pcm
        g["flp_pcm_mode%d_md5" % mode] = hashlib.md5(pcm.tobytes()).hexdigest()
    flags = loss_flags(len(pk), 50, seed=1)
    g["loss50_flags"] = np.array(flags, np.int32)
    pcm = decode_stream(pk, flags)
    g["flp_pcm_loss50"] = pcm
    g["flp_pcm_loss50_md5"] = hashlib.md5(pcm.tobytes()).hexdigest()
    # synthetic inputs: md5 of the FIX payload stream
    for name, x, kw in synth_inputs(clip):
        p = encode_signal(ref.RefEncoder("fix", **kw), x)
        g["synth_" + name] = hashlib.md5(bitfile(p)).hexdigest()
    np.savez_compressed(os.path.join(HERE, "golden.npz"), **g)
    for k in sorted(g):
        if isinstance(g[k], str):
            print(k, g[k])
    print("packets", len(pk), "mean bytes", float(nbytes[:, 0].mean()))


if __name__ == "__main__":
    main()
