#!/usr/bin/env python3
"""Decoder time per packet wave by arithmetic: decode_device of a float-mode (SOLO_B200_DEC_FLP) and a fixed-point-mode
(SOLO_B200_DEC_FIX) batch of the same streams, alternated in one run and timed with CUDA events.

    python tools/dec_arith_time.py [--streams 65536] [--reps 20] [--warmup 3]

One wave of speech-replay packets (13.6 kb/s, lostflag 4) is encoded once; each batch then decodes it `reps` times
after `warmup` untimed waves per mode.  Prints one JSON line: per mode the median and spread (min / max) of the ms per
wave, with the card's name and power limit beside them."""
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
    from tests.util import load_clip, speech_replay
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the decoder has no CPU implementation to time")
    N, cap, dev = a.streams, 128, torch.device("cuda", 0)
    x = torch.from_numpy(speech_replay(load_clip(), N, 1, first_packet=7)[0]).to(dev)
    bits = torch.zeros((N, cap), dtype=torch.uint8, device=dev)
    nb = torch.zeros((N, 2), dtype=torch.int16, device=dev)
    flags = torch.full((N,), 4, dtype=torch.int32, device=dev)
    ret = torch.zeros(N, dtype=torch.int32, device=dev)
    pcm = torch.zeros((N, 640), dtype=torch.int16, device=dev)
    stream = torch.cuda.current_stream()
    enc = solo_b200.EncoderBatch(N, rate=13600)
    enc.encode_device(x.data_ptr(), bits.data_ptr(), cap, nb.data_ptr(), stream.cuda_stream)
    dec = {m: solo_b200.DecoderBatch(N, arith=m) for m in ("flp", "fix")}

    def wave(m):
        dec[m].decode_device(pcm.data_ptr(), bits.data_ptr(), cap, nb.data_ptr(), flags.data_ptr(), ret.data_ptr(), stream.cuda_stream)

    for _ in range(a.warmup):
        for m in dec:
            wave(m)
    torch.cuda.synchronize()
    ms = {m: [] for m in dec}
    for _ in range(a.reps):
        for m in dec:                   # alternated: both modes see the same clocks and the same neighbours' load
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            wave(m)
            e1.record(stream)
            e1.synchronize()
            ms[m].append(e0.elapsed_time(e1))
    assert int((ret != 0).sum().item()) == 0, "decoder return"
    res = {"streams": N, "reps": a.reps, "card": card(), "torch_device": torch.cuda.get_device_name(0)}
    for m, v in ms.items():
        v = np.array(v)
        res[m] = {"ms_per_wave_median": round(float(np.median(v)), 3), "min": round(float(v.min()), 3), "max": round(float(v.max()), 3)}
    res["fix_over_flp"] = round(res["fix"]["ms_per_wave_median"] / res["flp"]["ms_per_wave_median"], 3)
    print(json.dumps(res))
    enc.close()
    for d in dec.values():
        d.close()


if __name__ == "__main__":
    main()
