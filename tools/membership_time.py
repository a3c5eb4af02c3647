#!/usr/bin/env python3
"""Cost of stream membership changes on the device beside the packet waves they interrupt, in 65 536-stream 16 kHz encoder
and decoder batches (40 ms packets, float decoder), on one card:

  reset_64 / reset_4096      : enc reset + dec reset of 64 / 4 096 streams (host clock around the two calls; each
                               stages its list, launches one kernel and synchronises the caller's stream, here a
                               non-default one of the tool's own)
  move_4096                  : export_states + import_states of 4 096 encoder and 4 096 decoder streams through blobs in
                               this GPU's memory; move_4096_peer the same with the blobs in a second GPU's memory, when
                               there is one
  import_state_loop_64       : the same 64 encoder and decoder streams through the per-stream import_state (one device
                               synchronise and one blocking copy each), for comparison with reset_64
  tick / tick_with_64_resets : decode_device + encode_device of every stream on one CUDA stream, without and with the
                               64 + 64 resets enqueued after them (host clock around the tick and its synchronise)

    python tools/membership_time.py [--streams 65536] [--reps 10] [--warmup 2]

Medians over `reps` repetitions after `warmup` untimed ones, the variants of a repetition alternated.  Prints one JSON line
with the card's name and power limit beside the numbers."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.dec32_time import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import numpy as np
    import torch
    import solo_b200
    from tests.util import load_clip, speech_replay
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: the membership calls have no CPU implementation to time")
    N, cap, dev = a.streams, 256, torch.device("cuda", 0)
    stream = torch.cuda.Stream()                # the tick's own stream, as a server would run it
    st = stream.cuda_stream
    enc, dec = solo_b200.EncoderBatch(N, rate=13600), solo_b200.DecoderBatch(N)
    x = torch.from_numpy(speech_replay(load_clip(), N, 1, first_packet=7)[0]).to(dev)
    bits = torch.zeros((N, cap), dtype=torch.uint8, device=dev)
    nb = torch.zeros((N, 2), dtype=torch.int16, device=dev)
    flags = torch.full((N,), 4, dtype=torch.int32, device=dev)
    ret = torch.zeros(N, dtype=torch.int32, device=dev)
    pcm = torch.zeros((N, 640), dtype=torch.int16, device=dev)
    enc.encode_device(x.data_ptr(), bits.data_ptr(), cap, nb.data_ptr(), st)     # a wave of real payloads to decode
    torch.cuda.synchronize()
    eb, db = solo_b200.state_bytes()
    rng = np.random.Generator(np.random.PCG64(1))
    lists = {m: rng.permutation(N)[:m].astype(np.int32) for m in (64, 4096)}
    blobs = {"local": (torch.zeros((4096, eb), dtype=torch.uint8, device=dev), torch.zeros((4096, db), dtype=torch.uint8, device=dev))}
    if torch.cuda.device_count() >= 2:
        solo_b200.enable_peer_access(0, 1)
        d1 = torch.device("cuda", 1)
        blobs["peer"] = (torch.zeros((4096, eb), dtype=torch.uint8, device=d1), torch.zeros((4096, db), dtype=torch.uint8, device=d1))
    host64 = [(enc.export_state(int(s)), dec.export_state(int(s))) for s in lists[64]]

    def reset(m):
        enc.reset(lists[m], stream=st)
        dec.reset(lists[m], stream=st)

    def move(where):
        be, bd = blobs[where]
        L = lists[4096]
        enc.export_states(L, be.data_ptr(), stream=st)
        enc.import_states(L, be.data_ptr(), stream=st)
        dec.export_states(L, bd.data_ptr(), stream=st)
        dec.import_states(L, bd.data_ptr(), stream=st)

    def import_loop():
        for s, (be, bd) in zip(lists[64], host64):
            enc.import_state(int(s), be)
            dec.import_state(int(s), bd)

    def tick(resets):
        dec.decode_device(pcm.data_ptr(), bits.data_ptr(), cap, nb.data_ptr(), flags.data_ptr(), ret.data_ptr(), st)
        enc.encode_device(x.data_ptr(), bits.data_ptr(), cap, nb.data_ptr(), st)
        if resets:
            reset(64)
        stream.synchronize()

    cases = {"reset_64": lambda: reset(64), "reset_4096": lambda: reset(4096), "move_4096": lambda: move("local"),
             "import_state_loop_64": import_loop, "tick": lambda: tick(False), "tick_with_64_resets": lambda: tick(True)}
    if "peer" in blobs:
        cases["move_4096_peer"] = lambda: move("peer")
    launches = {}
    for name, f in cases.items():
        k0 = solo_b200.kernel_launches()
        f()
        torch.cuda.synchronize()
        launches[name] = solo_b200.kernel_launches() - k0
    for _ in range(a.warmup):
        for f in cases.values():
            f()
    torch.cuda.synchronize()
    ms = {name: [] for name in cases}
    for _ in range(a.reps):
        for name, f in cases.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            ms[name].append(1e3 * (time.perf_counter() - t0))
    res = {"streams": N, "reps": a.reps, "card": card(), "torch_device": torch.cuda.get_device_name(0),
           "gpus": torch.cuda.device_count(), "launches": launches}
    for name, v in ms.items():
        v = np.array(v)
        res[name] = {"ms_median": round(float(np.median(v)), 3), "min": round(float(v.min()), 3), "max": round(float(v.max()), 3)}
    print(json.dumps(res))
    enc.close(); dec.close()


if __name__ == "__main__":
    main()
