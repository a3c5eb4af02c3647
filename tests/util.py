"""Shared helpers of the test-suite (input synthesis at 16 and 32 kHz, the reference driver's loss process, what the receiver
decodes)."""
import os
import re
import struct
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")


def load_clip():
    return np.load(os.path.join(GOLDEN, "speech_clip.npz"))["pcm"]


def load_golden():
    return np.load(os.path.join(GOLDEN, "golden.npz"))


def _lcg(s):
    return (907633515 + s * 196314165) & 0xFFFFFFFF


def _s32(x):
    return x - (1 << 32) if x >= (1 << 31) else x


def loss_flags(n_packets, loss_perc, seed=1):
    """lostflag sequence of the reference decoder driver (JC1_SDK_SRC_FLP/test/dec_main.c:24,227-307):
    per packet two LCG draws (one per description), float32 compare against loss/100; both kept -> 4,
    MD2 lost -> 2, MD1 lost -> 3, both lost -> 1."""
    rs = seed
    out = []
    thr = np.float32(loss_perc) / np.float32(100.0)
    for _ in range(n_packets):
        lost = []
        for _j in range(2):
            rs = _lcg(rs)
            v = np.float32(np.float32((_s32(rs) >> 16) + (1 << 15)) / np.float32(65535.0))
            lost.append(0 if v >= thr else 1)
        out.append({(0, 0): 4, (0, 1): 2, (1, 0): 3, (1, 1): 1}[tuple(lost)])
    return out


def trim_payload(b, nb, flag):
    """What the caller hands to AGR_Sate_Decoder_Decode for a given lostflag (dec_main.c:245-307)."""
    n0, n1 = int(nb[0]), int(nb[1])
    if flag == 2:
        return b[:n0 - n1], (n0 - n1, 0)
    if flag == 3:
        return b[n0 - n1:n0], (n1, 0)
    return b[:n0], (n0, n1)


def receive(bits, nb, flag):
    """(payload, nbytes, lostflag) the receiver hands to the decoder for one encoded packet: a DTX packet (nb[0] <= 0,
    nothing was sent) is concealed as a lost one, any other packet is trimmed for its lostflag."""
    if nb[0] <= 0:
        return bytes(16), (16, 8), 1
    return trim_payload(bits, nb, flag) + (int(flag),)


def bitfile(pk):
    """The reference CLI's .bit file of a list of (payload, (n0, n1), n) packets."""
    return b"".join(struct.pack("<hh", *nb) + (b if nb[0] else b"") for b, nb, n in pk)


def encode_signal(enc, pcm):
    """The packets of a whole signal through one encoder (enc.samples per packet); closes the encoder."""
    k = enc.samples
    pk = [enc.encode(pcm[i * k:(i + 1) * k]) for i in range(len(pcm) // k)]
    enc.close()
    return pk


def speech_replay(clip, n_streams, n_packets, first_packet=0):
    """SURVEY.md 8(d) synthetic batch (i): stream s reads the clip circularly from sample offset
    (s*7919*640) mod len(clip), scaled by 2^-(s mod 4).  Returns int16 [n_packets, n_streams, 640]."""
    n = len(clip)
    s = np.arange(n_streams, dtype=np.int64)
    off = (s * 7919 * 640) % n
    out = np.empty((n_packets, n_streams, 640), np.int16)
    idx = np.arange(640, dtype=np.int64)
    sh = (s & 3).astype(np.int16)
    for p in range(n_packets):
        ii = (off[:, None] + (first_packet + p) * 640 + idx[None, :]) % n
        out[p] = clip[ii] >> sh[:, None]
    return out


def synth_inputs(clip):
    """(name, int16 signal, encoder kwargs): parity cases beyond the plain clip (SURVEY.md 8(d) ii/iii + rates)."""
    rng = np.random.Generator(np.random.PCG64(1234))
    t = np.arange(640 * 60)
    cases = [
        ("rate6000", clip, dict(rate=6000)),
        ("rate15600", clip, dict(rate=15600)),
        ("rate24000", clip, dict(rate=24000)),
        ("rate100000", clip[:640 * 60], dict(rate=100000)),
        ("rate_default", clip[:640 * 60], dict(rate=0)),
        ("shift2", clip >> 2, {}),
        ("clip4x", np.clip(clip.astype(np.int32) * 4, -32768, 32767).astype(np.int16), {}),
        ("noise2000", np.clip(rng.normal(0, 2000, 640 * 80), -32768, 32767).astype(np.int16), {}),
        ("noise20000", np.clip(rng.normal(0, 20000, 640 * 40), -32768, 32767).astype(np.int16), {}),
        ("zeros", np.zeros(640 * 40, np.int16), {}),
        ("dc1000", np.full(640 * 40, 1000, np.int16), {}),
        ("square100", np.where((t // 80) % 2 == 0, 32767, -32767).astype(np.int16), {}),
        ("sine200", (8000 * np.sin(2 * np.pi * 200 * t / 16000)).astype(np.int16), {}),
        ("dtx", np.concatenate([clip[:640 * 60], np.zeros(640 * 60, np.int16), clip[:640 * 40]]), dict(dtx=1)),
        ("mdi", clip[:640 * 80], dict(use_md_index=1)),
    ]
    return cases


def signal_classes(clip, n_rows, n_packets, seed=5):
    """int16 [n_packets, n_rows, 640]; row s belongs to class s % 8:
    0 speech, 1 noise sigma 2000, 2 noise sigma 20000, 3 zeros, 4 DC 1000, 5 +-32767 square, 6 200 Hz sine, 7 4x clipped speech."""
    rng = np.random.Generator(np.random.PCG64(seed))
    L = n_packets * 640
    t = np.arange(L)
    out = np.zeros((n_rows, L), np.int16)
    for s in range(n_rows):
        k = s % 8
        off = (s * 7919 * 640) % (len(clip) - 1)
        sp = np.take(clip, (off + t) % len(clip))
        if k == 0:
            out[s] = sp
        elif k == 1:
            out[s] = np.clip(rng.normal(0, 2000, L), -32768, 32767).astype(np.int16)
        elif k == 2:
            out[s] = np.clip(rng.normal(0, 20000, L), -32768, 32767).astype(np.int16)
        elif k == 3:
            out[s] = 0
        elif k == 4:
            out[s] = 1000
        elif k == 5:
            out[s] = np.where(((t + 13 * s) // 80) % 2 == 0, 32767, -32767).astype(np.int16)
        elif k == 6:
            out[s] = (8000 * np.sin(2 * np.pi * 200 * (t + 7 * s) / 16000)).astype(np.int16)
        else:
            out[s] = np.clip(sp.astype(np.int32) * 4, -32768, 32767).astype(np.int16)
    return np.ascontiguousarray(out.reshape(n_rows, n_packets, 640).transpose(1, 0, 2))


def near_silent_classes(clip, n_rows, n_packets, samples=640, seed=9):
    """int16 [n_packets, n_rows, samples]; row s belongs to class s % 8:
    0 speech, 1-3 white noise sigma 1, 3, 8, 4 DC +1 / -1 (alternating between rows of the class), 5 isolated one-sample
    clicks in zeros, 6 speech at 2^-10, 7 speech fading into silence and back out (period 30 packets)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    L = n_packets * samples
    t = np.arange(L)
    out = np.zeros((n_rows, L), np.int16)
    for s in range(n_rows):
        k = s % 8
        off = (s * 7919 * 640) % (len(clip) - 1)
        sp = np.take(clip, (off + t) % len(clip)).astype(np.float64)
        if k == 0:
            v = sp
        elif k in (1, 2, 3):
            v = rng.normal(0, (1, 3, 8)[k - 1], L)
        elif k == 4:
            v = np.full(L, 1 if (s // 8) % 2 == 0 else -1)
        elif k == 5:
            v = np.zeros(L)
            pos = np.cumsum(rng.integers(200, 3000, L // 200 + 1))
            pos = pos[pos < L]
            v[pos] = rng.choice([-1, 1], pos.size) * rng.integers(1, 2000, pos.size)
        elif k == 6:
            v = sp / 1024.0
        else:
            ph = (t % (30 * samples)) / (30.0 * samples)
            env = np.clip(np.abs(2.0 * ph - 1.0) * 3.0 - 1.0, 0.0, 1.0)     # loud - fade - silent - fade - loud
            v = sp * env
        out[s] = np.clip(np.round(v), -32768, 32767).astype(np.int16)
    return np.ascontiguousarray(out.reshape(n_rows, n_packets, samples).transpose(1, 0, 2))


def upsample2(clip):
    """The clip at 32 kHz by an integer-exact rule: every 16 kHz sample x[n] is followed by the rounded-down mean of x[n]
    and x[n + 1] (the last one by itself).  No content above 8 kHz beyond the rule's images."""
    x = clip.astype(np.int32)
    nxt = np.concatenate([x[1:], x[-1:]])
    y = np.empty(2 * len(x), np.int32)
    y[0::2] = x
    y[1::2] = (x + nxt) >> 1
    return y.astype(np.int16)


def with_high_band(clip, seed=32):
    """upsample2(clip) plus seeded white noise of standard deviation 400 (content across 0-16 kHz, so that the 8-16 kHz
    band carries a signal), clipped to int16."""
    rng = np.random.Generator(np.random.PCG64(seed))
    y = upsample2(clip).astype(np.float64) + rng.normal(0.0, 400.0, 2 * len(clip))
    return np.clip(np.round(y), -32768, 32767).astype(np.int16)


def chirp(n_samples, amp=8000):
    """A linear chirp from 100 Hz to 15 kHz over n_samples at 32 kHz."""
    t = np.arange(n_samples) / 32000.0
    T = n_samples / 32000.0
    ph = 2 * np.pi * (100.0 * t + (15000.0 - 100.0) * t * t / (2 * T))
    return np.round(amp * np.sin(ph)).astype(np.int16)


def loss_with_bursts(T, n_rows, seed=3):
    """Per-stream lostflags: the reference driver's 20 % process, one burst of 10-14 lost packets per stream at a random
    place, every fifth row loss-free."""
    rng = np.random.Generator(np.random.PCG64(seed))
    flags = np.array([loss_flags(T, 20, seed=1 + s) for s in range(n_rows)], np.int32)
    for s in range(n_rows):
        n = int(rng.integers(10, 15))
        a = int(rng.integers(1, T - n))
        flags[s, a:a + n] = 1
    flags[::5] = 4
    return flags


def fuzz_decoder(iters, seed, corpus32=None):
    """Run tests/hostsim/fuzz_dec.cpp under AddressSanitizer and UBSan: the 16 kHz modes, or with corpus32 (a .bit file of
    32 kHz packets) the 32 kHz modes.  Checks that it ran clean; returns {mode: (decoded, rejected)}."""
    import pytest
    from tests.hostsim import build_hostsim
    try:
        exe = build_hostsim.build_fuzzer()
    except (subprocess.CalledProcessError, FileNotFoundError):
        pytest.skip("sanitizer build not available")
    p = subprocess.run([exe, str(iters), str(seed)] + ([str(corpus32)] if corpus32 else []), capture_output=True, text=True,
                       timeout=900)
    assert p.returncode == 0 and "no memory errors" in p.stdout, p.stdout[-2000:] + p.stderr[-4000:]
    print(p.stdout)
    return {m: (int(a), int(b)) for m, a, b in re.findall(r"^(.+): (\d+) decoded, (\d+) rejected$", p.stdout, re.M)}
