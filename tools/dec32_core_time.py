#!/usr/bin/env python3
"""Decoder time per packet wave of 32 kHz streams decoded to their 16 kHz core (core output), beside full-band 32 kHz and
16 kHz decoding on the same card: decode_device of a 32 kHz core-output batch, a 32 kHz full-band batch and a 16 kHz batch
of `streams` streams, all float mode, alternated in one run and timed with CUDA events.

    python tools/dec32_core_time.py [--streams 65536] [--reps 20] [--warmup 3]

The 32 kHz batches decode one 40 ms packet of golden_32k.npz's hb40 stream (24 kb/s, lostflag 4) in every row, the 16 kHz
batch a wave of speech-replay packets (13.6 kb/s); each batch decodes its wave `reps` times after `warmup` untimed waves.
Core output skips the high band and the synthesis launch; the script checks that every row of every timed wave returned 0
and counts the kernel launches of one wave of each batch.  Prints one JSON line with the card's name and power limit beside
the numbers."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.dec32_time import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import numpy as np
    import torch
    import solo_b200
    from tests.golden import make_golden_32k as mk
    from tests.util import GOLDEN, load_clip, speech_replay
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the decoder has no CPU implementation to time")
    N, cap, dev = a.streams, 256, torch.device("cuda", 0)
    stream = torch.cuda.current_stream()
    # 16 kHz wave: speech replay through the batched encoder
    x = torch.from_numpy(speech_replay(load_clip(), N, 1, first_packet=7)[0]).to(dev)
    bits16 = torch.zeros((N, cap), dtype=torch.uint8, device=dev)
    nb16 = torch.zeros((N, 2), dtype=torch.int16, device=dev)
    enc = solo_b200.EncoderBatch(N, rate=13600)
    enc.encode_device(x.data_ptr(), bits16.data_ptr(), cap, nb16.data_ptr(), stream.cuda_stream)
    torch.cuda.synchronize()
    enc.close()
    # 32 kHz wave: one fixture packet in every row
    f = np.load(os.path.join(GOLDEN, "golden_32k.npz"))
    b, nb = mk.packets(f, "hb40")[7]
    row = np.zeros(cap, np.uint8)
    row[:len(b)] = np.frombuffer(b, np.uint8)
    bits32 = torch.from_numpy(row).to(dev).expand(N, cap).contiguous()
    nb32 = torch.tensor(nb, dtype=torch.int16, device=dev).expand(N, 2).contiguous()
    flags = torch.full((N,), 4, dtype=torch.int32, device=dev)
    ret = torch.zeros(N, dtype=torch.int32, device=dev)
    pcm = torch.zeros((N, 1280), dtype=torch.int16, device=dev)
    dec = {"32k_core": solo_b200.DecoderBatch(N, samplerate=32000, out_samplerate=16000),
           "32k_full": solo_b200.DecoderBatch(N, samplerate=32000), "16k": solo_b200.DecoderBatch(N)}
    inp = {"32k_core": (bits32, nb32), "32k_full": (bits32, nb32), "16k": (bits16, nb16)}

    def wave(m):
        bb, nn = inp[m]
        dec[m].decode_device(pcm.data_ptr(), bb.data_ptr(), cap, nn.data_ptr(), flags.data_ptr(), ret.data_ptr(), stream.cuda_stream)

    launches = {}
    for m in dec:
        k0 = solo_b200.kernel_launches()
        wave(m)
        launches[m] = solo_b200.kernel_launches() - k0
    for _ in range(a.warmup):
        for m in dec:
            wave(m)
    torch.cuda.synchronize()
    ms = {m: [] for m in dec}
    for _ in range(a.reps):
        for m in dec:                   # alternated: all three see the same clocks and the same neighbours' load
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            wave(m)
            e1.record(stream)
            e1.synchronize()
            ms[m].append(e0.elapsed_time(e1))
            assert int((ret != 0).sum().item()) == 0, ("decoder return", m)
    res = {"streams": N, "reps": a.reps, "card": card(), "torch_device": torch.cuda.get_device_name(0), "launches_per_wave": launches}
    for m, v in ms.items():
        v = np.array(v)
        res[m] = {"ms_per_wave_median": round(float(np.median(v)), 3), "min": round(float(v.min()), 3), "max": round(float(v.max()), 3)}
    res["32k_core_over_32k_full"] = round(res["32k_core"]["ms_per_wave_median"] / res["32k_full"]["ms_per_wave_median"], 3)
    res["32k_core_over_16k"] = round(res["32k_core"]["ms_per_wave_median"] / res["16k"]["ms_per_wave_median"], 3)
    print(json.dumps(res))
    for d in dec.values():
        d.close()


if __name__ == "__main__":
    main()
