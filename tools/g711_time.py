#!/usr/bin/env python3
"""Time of one G.711 gateway uplink (sb_g711_vad_kernel + sb_g711_synth_kernel) and one downlink (sb_g711_downlink_kernel)
for 65 536 streams, 40 ms and 20 ms rows, half of them mu-law and half A-law, timed with CUDA events over device-resident
buffers, beside the bytes each call must move (G.711 bytes and 16 kHz rows, the lost masks and activity bytes).

    python tools/g711_time.py [--reps 50] [--warmup 5] [--kernels]

Inputs are seeded: the uplink's payloads are random bytes (any byte is a valid code), one stream in eight loses a frame;
the downlink's rows are seeded noise.  Prints one JSON line with the card's name and power limit beside the numbers.
--kernels adds, from a separate torch.profiler pass after the timed one, each gateway kernel's mean device time."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from dec32_time import card  # noqa: E402

HBM_TBPS = 3.35                                 # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--kernels", action="store_true")
    a = ap.parse_args()
    import numpy as np
    import torch
    import solo_b200
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the gateway kernels have no CPU implementation to time")
    N, dev = 65536, torch.device("cuda", 0)
    stream = torch.cuda.current_stream().cuda_stream
    rng = np.random.Generator(np.random.PCG64(1))
    res = {"streams": N, "reps": a.reps, "card": card(), "torch_device": torch.cuda.get_device_name(0)}
    for fs in (40, 20):
        spp8, spp16 = 8 * fs, 16 * fs
        g = solo_b200.G711Gateway(N, fs, "pcmu")
        g.reset(np.arange(1, N, 2), "pcma")
        pay = torch.from_numpy(rng.integers(0, 256, (N, spp8), dtype=np.uint8)).to(dev)
        lost = torch.from_numpy(np.where(rng.random(N) < 0.125, 1, 0).astype(np.int32)).to(dev)
        pcm = torch.zeros((N, spp16), dtype=torch.int16, device=dev)
        level, flags = torch.zeros(N, dtype=torch.uint8, device=dev), torch.zeros(N, dtype=torch.uint8, device=dev)
        rows = torch.from_numpy(np.clip(rng.normal(0, 6000, (N, spp16)), -32768, 32767).astype(np.int16)).to(dev)
        out = torch.zeros((N, spp8), dtype=torch.uint8, device=dev)
        calls = {
            "uplink": (lambda: g.uplink_device(pay.data_ptr(), lost.data_ptr(), pcm.data_ptr(), level.data_ptr(),
                                               flags.data_ptr(), stream), N * (spp8 + 4 + 2 * spp16 + 2)),
            "downlink": (lambda: g.downlink_device(rows.data_ptr(), out.data_ptr(), stream), N * (2 * spp16 + spp8)),
        }
        for _ in range(a.warmup):
            for f, _ in calls.values():
                f()
        torch.cuda.synchronize()
        ms = {name: [] for name in calls}
        for _ in range(a.reps):
            for name, (f, _) in calls.items():     # alternated, so that both see the same machine
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                f()
                e1.record()
                e1.synchronize()
                ms[name].append(e0.elapsed_time(e1))
        for name, (_, nbytes) in calls.items():
            v = np.array(ms[name])
            med = float(np.median(v))
            res["%s_%dms" % (name, fs)] = {"ms_median": round(med, 4), "ms_min": round(float(v.min()), 4),
                                           "MB_per_call": round(nbytes / 1e6, 1),
                                           "share_of_hbm_peak": round(nbytes / (med * 1e-3) / (HBM_TBPS * 1e12), 3)}
        if a.kernels:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(10):
                    for f, _ in calls.values():
                        f()
                torch.cuda.synchronize()
            res["kernels_%dms" % fs] = {e.key: round(e.device_time_total / e.count / 1e3, 4) for e in prof.key_averages()
                                        if "g711" in e.key}
        g.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
