#!/usr/bin/env python3
"""Time of one send-queue pack (solo_b200_tx_pack_device) for 65 536 streams, cap 256, timed with CUDA events, beside the
bytes it moves; then the queue's share of a device tick: encode_device + pack against encode_device alone, alternated in
the same run.

    python tools/tx_time.py [--reps 50] [--warmup 5] [--tick-reps 8]

Rows are golden.npz's packets (stream s sends packet s mod 191) with a seeded 5 % of the rows marked DTX (nbytes[0] = 0).
Prints one JSON line with the card's name and power limit beside the numbers."""
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
    from tests.util import load_clip, load_golden, speech_replay
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the send-queue kernels have no CPU implementation to time")
    N, cap, dev = 65536, 256, torch.device("cuda", 0)
    stream = torch.cuda.current_stream().cuda_stream
    rng = np.random.Generator(np.random.PCG64(1))
    g = load_golden()
    P = g["fix_nbytes"].shape[0]
    p = np.arange(N) % P
    bits = np.zeros((N, cap), np.uint8)
    w = min(g["fix_bits"].shape[1], cap)
    bits[:, :w] = g["fix_bits"][p, :w]
    nb = g["fix_nbytes"][p].astype(np.int16)
    nb[rng.random(N) < 0.05, 0] = 0
    td = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)  # noqa: E731
    d_bits, d_nb = td(bits), td(nb)
    d_pay = torch.zeros(N * cap, dtype=torch.uint8, device=dev)
    ent = [torch.zeros(2 * N, dtype=t, device=dev) for t in (torch.int32, torch.int32, torch.uint8, torch.int32, torch.int32)]
    d_ct, d_tot = torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int64, device=dev)
    q = solo_b200.TxQueue(N)

    def pack(rows):
        q.pack_device(rows.data_ptr(), cap, d_nb.data_ptr(), d_pay.data_ptr(), d_pay.numel(), *(e.data_ptr() for e in ent),
                      d_ct.data_ptr(), d_tot.data_ptr(), stream)

    def timed_pack():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        pack(d_bits)
        e1.record()
        return e0, e1

    for _ in range(a.warmup):
        timed_pack()
    torch.cuda.synchronize()
    ms = []
    for _ in range(a.reps):
        e0, e1 = timed_pack()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    count, total = int(d_ct.item()), int(d_tot.item())
    sent = nb[:, 0] > 0
    assert count == int(sent.sum() * 2 - ((nb[:, 0] == nb[:, 1]) & sent).sum()) and total == int(nb[sent, 0].sum())
    ms = np.array(ms)
    med = float(np.median(ms))
    # bytes the pack must move, from the shapes: nbytes read twice (sizes and pack passes), the payload read from the rows
    # and written, 14 bytes of entries per datagram, per stream next and counters read and written, the scan words
    # (8 B per stream, written and read; the block totals are negligible)
    nbytes = 2 * 4 * N + 2 * total + 14 * count + N * 2 * (4 + 16) + 2 * 8 * N
    res = {"streams": N, "cap": cap, "dtx_rows": int((~sent).sum()), "datagrams": count, "payload_bytes": total,
           "reps": a.reps, "card": card(), "torch_device": torch.cuda.get_device_name(0),
           "pack_us_median": round(med * 1e3, 1), "pack_us_min": round(float(ms.min()) * 1e3, 1),
           "MB_per_pack": round(nbytes / 1e6, 2), "MB_rows_if_copied_whole": round(N * cap / 1e6, 2),
           "MB_compact_copy": round((total + 14 * count) / 1e6, 2),
           "GB_per_s_median": round(nbytes / (med * 1e-3) / 1e9, 1),
           "share_of_hbm_peak": round(nbytes / (med * 1e-3) / (HBM_TBPS * 1e12), 3)}

    # the queue's share of a device tick: encode + pack against encode alone
    enc = solo_b200.EncoderBatch(N)
    x = speech_replay(load_clip(), N, 1)[0]
    d_x = td(x)
    d_out = torch.zeros((N, cap), dtype=torch.uint8, device=dev)

    def tick(with_tx):
        e0, e2 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        enc.encode_device(d_x.data_ptr(), d_out.data_ptr(), cap, d_nb.data_ptr(), stream)
        if with_tx:
            pack(d_out)
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
    res["tick"] = {"ms_encode_pack": round(full, 3), "ms_encode": round(base, 3),
                   "queue_share": round((full - base) / full, 4), "reps": a.tick_reps}
    print(json.dumps(res))
    q.close()
    enc.close()


if __name__ == "__main__":
    main()
