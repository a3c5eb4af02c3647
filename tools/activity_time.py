#!/usr/bin/env python3
"""Time of one activity call (sb_activity_kernel) after a decoder wave of 16 kHz and of 32 kHz streams, timed with CUDA
events, beside the bytes it must read: the PCM rows (2 bytes per sample) plus a return code (4 B), a flags byte and two
output bytes per stream.

    python tools/activity_time.py [--streams 65536] [--reps 50] [--warmup 5]

Each batch decodes one 40 ms packet wave (golden.npz's clip packet 7 at 16 kHz, golden_32k.npz's hb40 packet 7 at 32 kHz,
lostflag 4) with decode_device, then activity_device is timed `reps` times, the two rates alternated.  Prints one JSON
line with the card's name and power limit beside the numbers."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from dec32_time import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    import torch
    import solo_b200
    from tests.golden import make_golden_32k as mk
    from tests.util import GOLDEN, load_golden
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the activity kernel has no CPU implementation to time")
    N, cap, dev = a.streams, 256, torch.device("cuda", 0)
    stream = torch.cuda.current_stream().cuda_stream
    g, f = load_golden(), np.load(os.path.join(GOLDEN, "golden_32k.npz"))
    pk = {16000: (bytes(g["fix_bits"][7, :int(g["fix_nbytes"][7, 0])]), tuple(int(v) for v in g["fix_nbytes"][7])),
          32000: mk.packets(f, "hb40")[7]}
    flags = torch.full((N,), 4, dtype=torch.int32, device=dev)
    ret = torch.zeros(N, dtype=torch.int32, device=dev)
    level = torch.zeros(N, dtype=torch.uint8, device=dev)
    vad = torch.zeros(N, dtype=torch.uint8, device=dev)
    run = {}
    for sr, (b, nb) in pk.items():
        row = np.zeros(cap, np.uint8)
        row[:len(b)] = np.frombuffer(b, np.uint8)
        bits = torch.from_numpy(row).to(dev).expand(N, cap).contiguous()
        nbt = torch.tensor(nb, dtype=torch.int16, device=dev).expand(N, 2).contiguous()
        d = solo_b200.DecoderBatch(N, samplerate=sr)
        pcm = torch.zeros((N, d.samples), dtype=torch.int16, device=dev)
        d.decode_device(pcm.data_ptr(), bits.data_ptr(), cap, nbt.data_ptr(), flags.data_ptr(), ret.data_ptr(), stream)
        torch.cuda.synchronize()
        assert int((ret != 0).sum().item()) == 0
        run[sr] = (d, pcm)

    def call(sr):
        d, pcm = run[sr]
        d.activity_device(pcm.data_ptr(), level.data_ptr(), vad.data_ptr(), stream)

    for _ in range(a.warmup):
        for sr in run:
            call(sr)
    torch.cuda.synchronize()
    ms = {sr: [] for sr in run}
    for _ in range(a.reps):
        for sr in run:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call(sr)
            e1.record()
            e1.synchronize()
            ms[sr].append(e0.elapsed_time(e1))
    res = {"streams": N, "reps": a.reps, "card": card(), "torch_device": torch.cuda.get_device_name(0)}
    for sr, v in ms.items():
        v = np.array(v)
        d, pcm = run[sr]
        nbytes = pcm.numel() * 2 + N * (4 + 1 + 2)
        med = float(np.median(v))
        res["%dk" % (sr // 1000)] = {"us_median": round(med * 1e3, 1), "us_min": round(float(v.min()) * 1e3, 1),
                                     "MB_per_call": round(nbytes / 1e6, 1), "GB_per_s_median": round(nbytes / (med * 1e-3) / 1e9, 1)}
    print(json.dumps(res))
    for d, pcm in run.values():
        d.close()


if __name__ == "__main__":
    main()
