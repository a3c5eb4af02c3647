#!/usr/bin/env python3
"""Cost of receive-queue timing: one tick of a timed queue (solo_b200_rx_insert_timed_device + solo_b200_rx_pull_device)
against one tick of an untimed queue (solo_b200_rx_insert_device + pull_device) on the same arrays, alternated in one run
and timed with CUDA events; median of --reps ticks of each after --warmup.

    python tools/rx_timing_time.py [--reps 50] [--warmup 5]

The traffic is tools/rx_time.py's: 65 536 streams, depth 8, desc_cap 128, cap 256, about 132 k arrivals per tick (both
descriptions of golden-sized packets, 10 % one tick early, 1 % duplicated, shuffled), plus receive times of index * 640
and a seeded delay of up to two packets.  Also checks that both queues pulled the same rows and counted the same.  Prints
one JSON line with the card's name and power limit beside the numbers."""
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
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import numpy as np
    import torch
    import solo_b200
    from tests.server_ref import rx_time_traffic
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the receive-queue kernels have no CPU implementation to time")
    N, depth, desc_cap, cap, ts, dev = 65536, 8, 128, 256, 640, torch.device("cuda", 0)
    stream = torch.cuda.current_stream().cuda_stream
    rng = np.random.Generator(np.random.PCG64(1))
    s, d, lens, payload, off, early = rx_time_traffic(N, rng)
    A = len(s)
    delay = rng.integers(0, 2 * ts, A)
    td = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    d_s, d_d, d_off, d_len, d_pay = td(s), td(d), td(off), td(lens), td(payload)
    d_early = td(early.astype(np.int32))
    d_delay = td(delay.astype(np.int32))
    d_idx = torch.zeros(A, dtype=torch.int32, device=dev)
    d_arr = torch.zeros(A, dtype=torch.int32, device=dev)
    out = {w: (torch.zeros((N, cap), dtype=torch.uint8, device=dev), torch.zeros((N, 2), dtype=torch.int16, device=dev),
               torch.zeros(N, dtype=torch.int32, device=dev)) for w in (True, False)}
    qs = {True: solo_b200.RxQueue(N, depth, desc_cap), False: solo_b200.RxQueue(N, depth, desc_cap)}
    qs[True].enable_timing(ts, A)
    tick_of = {True: 0, False: 0}

    def tick(timed):
        t = tick_of[timed]
        torch.add(d_early, t, out=d_idx)                # index = t, or t + 1 for the early pairs (outside the window)
        torch.add(d_idx * ts, d_delay, out=d_arr)       # receive time, mod 2^32 in int32
        bits, nb, lf = out[timed]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        qs[timed].insert_device(d_s.data_ptr(), d_idx.data_ptr(), d_d.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), A,
                                d_pay.data_ptr(), payload.size, stream, d_arrival=d_arr.data_ptr() if timed else None)
        qs[timed].pull_device(0, bits.data_ptr(), cap, nb.data_ptr(), lf.data_ptr(), stream)
        e1.record()
        tick_of[timed] = t + 1
        return e0, e1

    for _ in range(a.warmup):
        for w in (True, False):
            tick(w)
    torch.cuda.synchronize()
    ms = {True: [], False: []}
    for _ in range(a.reps):
        for w in (True, False):
            e0, e1 = tick(w)
            e1.synchronize()
            ms[w].append(e0.elapsed_time(e1))
    same_rows = all(torch.equal(x, y) for x, y in zip(out[True], out[False]))
    same_counters = bool(np.array_equal(qs[True].stats()[0], qs[False].stats()[0]))
    jitter, highest, received, margin = qs[True].timing()
    timed, plain = float(np.median(ms[True])), float(np.median(ms[False]))
    print(json.dumps({
        "streams": N, "depth": depth, "desc_cap": desc_cap, "cap": cap, "arrivals_per_tick": A, "reps": a.reps,
        "card": card(), "torch_device": torch.cuda.get_device_name(0),
        "timed_insert_pull_us_median": round(timed * 1e3, 1), "timed_insert_pull_us_min": round(min(ms[True]) * 1e3, 1),
        "untimed_insert_pull_us_median": round(plain * 1e3, 1), "untimed_insert_pull_us_min": round(min(ms[False]) * 1e3, 1),
        "timing_cost_us": round((timed - plain) * 1e3, 1),
        "same_rows": same_rows, "same_counters": same_counters,
        "mean_reported_jitter": round(float(jitter.mean()), 2), "received_total": int(received.sum()),
        "margin_total": [int(v) for v in margin.sum(0)]}))
    for q in qs.values():
        q.close()


if __name__ == "__main__":
    main()
