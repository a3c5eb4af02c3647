#!/usr/bin/env python3
"""Time of one receive-queue tick (solo_b200_rx_insert_device + solo_b200_rx_pull_device) for 65 536 streams, depth 8,
desc_cap 128, cap 256, timed with CUDA events, beside the bytes it moves; then the queue's share of a device tick:
insert + pull + decode_device against decode_device alone, alternated in the same run.

    python tools/rx_time.py [--reps 50] [--warmup 5] [--tick-reps 8]

Each tick carries 131 072 arrivals plus 1 % duplicates: both descriptions of every stream's packet, split from golden.npz's
packets (stream s sends packet s mod 191), in a seeded shuffled order.  A fixed 10 % of the (stream, description) pairs
arrive one tick early, as part of the previous tick's array, so every description still arrives once.  Prints one JSON line
with the card's name and power limit beside the numbers."""
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
    ap.add_argument("--tick-reps", type=int, default=8)
    a = ap.parse_args()
    import numpy as np
    import torch
    import solo_b200
    from tests.server_ref import rx_time_traffic
    from tests.util import load_golden
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the receive-queue kernels have no CPU implementation to time")
    N, depth, desc_cap, cap, dev = 65536, 8, 128, 256, torch.device("cuda", 0)
    stream = torch.cuda.current_stream().cuda_stream
    rng = np.random.Generator(np.random.PCG64(1))
    s, d, lens, payload, off, early = rx_time_traffic(N, rng)
    A = len(s)
    td = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    d_s, d_d, d_off, d_len, d_pay = td(s), td(d), td(off), td(lens), td(payload)
    d_early = td(early.astype(np.int32))
    d_idx = torch.zeros(A, dtype=torch.int32, device=dev)
    d_bits = torch.zeros((N, cap), dtype=torch.uint8, device=dev)
    d_nb = torch.zeros((N, 2), dtype=torch.int16, device=dev)
    d_lf = torch.zeros(N, dtype=torch.int32, device=dev)
    q = solo_b200.RxQueue(N, depth, desc_cap)
    state = {"t": 0}

    def rx_tick():
        t = state["t"]
        torch.add(d_early, t, out=d_idx)        # index = t, or t + 1 for the early pairs (outside the timed window)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        q.insert_device(d_s.data_ptr(), d_idx.data_ptr(), d_d.data_ptr(), d_off.data_ptr(), d_len.data_ptr(), A,
                        d_pay.data_ptr(), payload.size, stream)
        q.pull_device(0, d_bits.data_ptr(), cap, d_nb.data_ptr(), d_lf.data_ptr(), stream)
        e1.record()
        state["t"] = t + 1
        return e0, e1

    for _ in range(a.warmup):
        rx_tick()
    torch.cuda.synchronize()
    ms = []
    for _ in range(a.reps):
        e0, e1 = rx_tick()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    lf = d_lf.cpu().numpy()
    cnt, bad = q.stats()
    ms = np.array(ms)
    med = float(np.median(ms))
    # bytes the tick must move, from the shapes: payload read and stored, the arrival arrays read by the three passes
    # (17 B each), the touched slots' metadata (index 4, lengths 4, election words 16, commit word 4) read and written,
    # per stream last / counters / nbytes / lostflag, and the rows: read from the store and written
    g = load_golden()
    p = np.repeat(np.arange(N), 2) % g["fix_nbytes"].shape[0]      # the packet of each original arrival
    rows = int(g["fix_nbytes"][p, 0].astype(np.int32).sum())
    slot_meta = N * 28 * 2
    nbytes = 2 * payload.size + 3 * 17 * A + slot_meta + N * (4 + 32 + 4 + 4) + 2 * rows
    res = {"streams": N, "depth": depth, "desc_cap": desc_cap, "cap": cap, "arrivals_per_tick": A, "reps": a.reps,
           "card": card(), "torch_device": torch.cuda.get_device_name(0),
           "insert_pull_us_median": round(med * 1e3, 1), "insert_pull_us_min": round(float(ms.min()) * 1e3, 1),
           "MB_per_tick": round(nbytes / 1e6, 2), "MB_payload_in": round(payload.size / 1e6, 2),
           "MB_rows_out": round(rows / 1e6, 2), "GB_per_s_median": round(nbytes / (med * 1e-3) / 1e9, 1),
           "share_of_hbm_peak": round(nbytes / (med * 1e-3) / (HBM_TBPS * 1e12), 3),
           "last_tick_lostflag_4_share": round(float((lf == 4).mean()), 4),
           "counters_total": [int(v) for v in cnt.sum(0)], "bad_stream": bad}

    # the queue's share of a device tick: insert + pull + decode against decode alone
    dec = solo_b200.DecoderBatch(N)
    dpcm = torch.zeros((N, 640), dtype=torch.int16, device=dev)

    def tick(with_rx):
        if with_rx:
            e0, e1 = rx_tick()
        else:
            e0 = torch.cuda.Event(enable_timing=True)
            e0.record()
        dec.decode_device(dpcm.data_ptr(), d_bits.data_ptr(), cap, d_nb.data_ptr(), d_lf.data_ptr(), 0, stream)
        e2 = torch.cuda.Event(enable_timing=True)
        e2.record()
        return e0, e2

    for w in (True, False):
        tick(w)
    torch.cuda.synchronize()
    tms = {True: [], False: []}
    for _ in range(a.tick_reps):
        for w in (True, False):
            e0, e2 = tick(w)
            e2.synchronize()
            tms[w].append(e0.elapsed_time(e2))
    full, base = float(np.median(tms[True])), float(np.median(tms[False]))
    res["tick"] = {"ms_insert_pull_decode": round(full, 3), "ms_decode": round(base, 3),
                   "queue_share": round((full - base) / full, 4), "reps": a.tick_reps}
    print(json.dumps(res))
    q.close()
    dec.close()


if __name__ == "__main__":
    main()
