#!/usr/bin/env python3
"""Decoder time per packet wave of 32 kHz streams (16 kHz SILK core), beside the 16 kHz decoder on the same card:
decode_device of a 32 kHz float-mode, a 32 kHz fixed-point-mode and a 16 kHz float-mode batch of `streams` streams,
alternated in one run and timed with CUDA events.

    python tools/dec32_time.py [--streams 65536] [--reps 20] [--warmup 3]

The 32 kHz batches decode one 40 ms packet of golden_32k.npz's hb40 stream (24 kb/s, lostflag 4) in every row, the 16 kHz
batch a wave of speech-replay packets (13.6 kb/s); each batch decodes its wave `reps` times after `warmup` untimed waves.
Also reports the device memory the first 32 kHz wave took beyond the batches' own allocations (the driver's reservation for
the decoder kernel's per-thread stack).  Prints one JSON line with the card's name and power limit beside the numbers."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


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
    free0 = torch.cuda.mem_get_info(0)[0]
    dec = {"32k_flp": solo_b200.DecoderBatch(N, samplerate=32000), "32k_fix": solo_b200.DecoderBatch(N, samplerate=32000, arith="fix")}
    free1 = torch.cuda.mem_get_info(0)[0]
    inp = {"32k_flp": (bits32, nb32), "32k_fix": (bits32, nb32)}

    def wave(m):
        bb, nn = inp[m]
        dec[m].decode_device(pcm.data_ptr(), bb.data_ptr(), cap, nn.data_ptr(), flags.data_ptr(), ret.data_ptr(), stream.cuda_stream)

    wave("32k_flp")
    torch.cuda.synchronize()
    free2 = torch.cuda.mem_get_info(0)[0]
    dec["16k_flp"] = solo_b200.DecoderBatch(N)
    inp["16k_flp"] = (bits16, nb16)
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
    res = {"streams": N, "reps": a.reps, "card": card(), "torch_device": torch.cuda.get_device_name(0),
           "batch_alloc_mib_two_32k_batches": round((free0 - free1) / 2 ** 20, 1),
           "first_32k_wave_extra_mib": round((free1 - free2) / 2 ** 20, 1)}
    for m, v in ms.items():
        v = np.array(v)
        res[m] = {"ms_per_wave_median": round(float(np.median(v)), 3), "min": round(float(v.min()), 3), "max": round(float(v.max()), 3)}
    res["32k_flp_over_16k_flp"] = round(res["32k_flp"]["ms_per_wave_median"] / res["16k_flp"]["ms_per_wave_median"], 3)
    print(json.dumps(res))
    for d in dec.values():
        d.close()


if __name__ == "__main__":
    main()
