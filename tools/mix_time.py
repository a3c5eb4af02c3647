#!/usr/bin/env python3
"""Time of one solo_b200_mix_device call (sb_mix_select_kernel + sb_mix_kernel) for 65 536 streams of 640-sample rows,
k = 3, in four room layouts, timed with CUDA events, beside the bytes the mix must move: the member rows it writes plus
each talker row read once.  Then the mixer's share of a whole device tick: decode_device + activity_device + mix_device +
downlink encode_device against decode_device + encode_device alone, at 16 384 rooms of 4, alternated.

    python tools/mix_time.py [--reps 50] [--warmup 5] [--tick-reps 8]

Layouts: 16 384 rooms of 4; 256 rooms of 256; one room of 65 536; the mixed layout of tests/server_ref.py (8 192 rooms
of 4, 64 of 256, one of 12 000, 4 384 streams in no room).  Rows, levels and flags are seeded random (about 60 % of the
streams eligible).  Prints one JSON line with the card's name and power limit beside the numbers."""
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
    from tests.server_ref import mixed_layout
    from tests.util import load_golden
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the mix kernels have no CPU implementation to time")
    N, spp, k, dev = 65536, 640, 3, torch.device("cuda", 0)
    stream = torch.cuda.current_stream().cuda_stream
    rng = np.random.Generator(np.random.PCG64(1))
    perm = rng.permutation(N).astype(np.int32)
    layouts = {"16384x4": np.split(perm, 16384), "256x256": np.split(perm, 256), "1x65536": [perm],
               "mixed": mixed_layout(N)[0]}
    pcm = torch.from_numpy(rng.integers(-12000, 12000, (N, spp), dtype=np.int16)).to(dev)
    out = torch.zeros_like(pcm)
    level = torch.from_numpy(rng.integers(0, 128, N, dtype=np.uint8)).to(dev)
    flags = torch.from_numpy(rng.choice(np.array([0, 1, 2, 3, 12], np.uint8), N)).to(dev)
    dl = {}
    for name, rooms in layouts.items():
        rs, mb = solo_b200.rooms_csr(rooms)
        dl[name] = (torch.from_numpy(rs).to(dev), torch.from_numpy(mb).to(dev), len(rooms),
                    torch.zeros((len(rooms), k), dtype=torch.int32, device=dev), int(rs[-1]))

    def call(name, o=out, src=pcm, lv=level, fl=flags):
        rs, mb, R, tk, _ = dl[name]
        solo_b200.mix_device(src.data_ptr(), o.data_ptr(), spp, N, lv.data_ptr(), fl.data_ptr(), rs.data_ptr(),
                             mb.data_ptr(), R, k, tk.data_ptr(), stream)

    for _ in range(a.warmup):
        for name in dl:
            call(name)
    torch.cuda.synchronize()
    ms = {name: [] for name in dl}
    for _ in range(a.reps):
        for name in dl:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call(name)
            e1.record()
            e1.synchronize()
            ms[name].append(e0.elapsed_time(e1))
    res = {"streams": N, "spp": spp, "k": k, "reps": a.reps, "card": card(), "torch_device": torch.cuda.get_device_name(0)}
    for name, v in ms.items():
        v = np.array(v)
        _, _, R, tk, M = dl[name]
        talkers = int((tk >= 0).sum().item())
        nbytes = (M + talkers) * spp * 2
        med = float(np.median(v))
        res[name] = {"us_median": round(med * 1e3, 1), "us_min": round(float(v.min()) * 1e3, 1), "rooms": R,
                     "talker_rows": talkers, "MB_per_call": round(nbytes / 1e6, 1),
                     "GB_per_s_median": round(nbytes / (med * 1e-3) / 1e9, 1),
                     "share_of_hbm_peak": round(nbytes / (med * 1e-3) / (HBM_TBPS * 1e12), 3)}

    # the mixer's share of a device tick at 16 384 rooms of 4
    g = load_golden()
    cap = 256
    row = np.zeros(cap, np.uint8)
    n0 = int(g["fix_nbytes"][7, 0])
    row[:n0] = g["fix_bits"][7, :n0]
    bits = torch.from_numpy(row).to(dev).expand(N, cap).contiguous()
    nbt = torch.from_numpy(g["fix_nbytes"][7].astype(np.int16)).to(dev).expand(N, 2).contiguous()
    lost = torch.full((N,), 4, dtype=torch.int32, device=dev)
    dec = solo_b200.DecoderBatch(N)
    enc = solo_b200.EncoderBatch(N, rate=13600)
    dpcm = torch.zeros((N, spp), dtype=torch.int16, device=dev)
    down = torch.zeros((N, spp), dtype=torch.int16, device=dev)
    dbits = torch.zeros((N, cap), dtype=torch.uint8, device=dev)
    dnb = torch.zeros((N, 2), dtype=torch.int16, device=dev)

    def tick(with_mix):
        dec.decode_device(dpcm.data_ptr(), bits.data_ptr(), cap, nbt.data_ptr(), lost.data_ptr(), 0, stream)
        if with_mix:
            dec.activity_device(dpcm.data_ptr(), level.data_ptr(), flags.data_ptr(), stream)
            call("16384x4", o=down, src=dpcm)
        enc.encode_device(down.data_ptr(), dbits.data_ptr(), cap, dnb.data_ptr(), stream)

    for w in (True, False):
        tick(w)
    torch.cuda.synchronize()
    tms = {True: [], False: []}
    for _ in range(a.tick_reps):
        for w in (True, False):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            tick(w)
            e1.record()
            e1.synchronize()
            tms[w].append(e0.elapsed_time(e1))
    full, base = float(np.median(tms[True])), float(np.median(tms[False]))
    res["tick_16384x4"] = {"ms_decode_activity_mix_encode": round(full, 3), "ms_decode_encode": round(base, 3),
                           "mixer_and_activity_share": round((full - base) / full, 4), "reps": a.tick_reps}
    print(json.dumps(res))
    dec.close(), enc.close()


if __name__ == "__main__":
    main()
