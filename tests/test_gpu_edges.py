"""Near-silence end to end, and device configurations no other batched test runs.

Real calls spend much of their time in near-silence: a quiet room's noise floor of a few LSB, a +-1 DC offset, clicks.
That input drives Burg's small-energy arithmetic with non-zero data, the VAD and the gain quantiser at the bottom of their
ranges, and DTX with comfort noise.  Here it runs in neighbouring streams with speech, in an odd-sized batch, through
encode_device / decode_device with DTX, 20 ms packets, joint mode 1 and use_md_index = 1, under a per-stream loss process
with bursts of 10 or more packets.  Every row is compared with the unmodified reference given the same configuration:
payloads byte-exact, PCM 0 LSB.  A CPU test runs the same class through the host model of the kernels.

Batched encodes with a cap below the packet size check the kernels' cap guards: bytes [0, min(cap, total)) of each row
equal the reference's, the length fields describe the whole packet, and nothing is written outside the row."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from tests.util import load_clip, loss_flags, trim_payload

PCM_TOL = 0


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


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the host model of the kernels against the reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref():
    from oracle import ref as r
    if not r.available():
        pytest.skip("oracle/_ref not built")
    return r


def test_host_model_near_silence_matches_reference(ref):
    from tests.hostsim.sim import SimDecoder, SimEncoder
    T, N = 40, 16
    x = near_silent_classes(load_clip(), N, T)
    flags = loss_with_bursts(T, N)
    for s in range(N):
        kw = dict(dtx=1) if s % 2 else dict(use_md_index=1)
        se, re_ = SimEncoder(**kw), ref.RefEncoder("fix", **kw)
        mdi = kw.get("use_md_index", 0)
        sd, rd = SimDecoder(use_md_index=mdi), ref.RefDecoder("flp", use_md_index=mdi)
        for p in range(T):
            b, nb, n = se.encode(x[p, s])
            rb, rnb, rn = re_.encode(x[p, s])
            assert (b, nb, n) == (rb, rnb, rn), ("payload", s, s % 8, p)
            f = int(flags[s, p])
            if rnb[0] <= 0:
                pb, pnb, f = bytes(16), (16, 8), 1
            else:
                pb, pnb = trim_payload(rb, rnb, f)
            y, r = sd.decode(pb, pnb, f)
            ry, rr = rd.decode(pb, pnb, f)
            assert r == rr == 0 and np.array_equal(y, ry), ("pcm", s, s % 8, p, f)
        for o in (se, re_, sd, rd):
            o.close()


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sb():
    import solo_b200
    solo_b200.lib()
    return solo_b200


def run_device_against_reference(sb, ref, x, rate=13600, dtx=0, use_md_index=0, framesize_ms=40, joint_hb=0, workers=16):
    """x: [T, N, samples].  encode_device / decode_device vs one reference encoder + decoder per row; the device decoder
    gets the host-trimmed payloads and a DTX row as a lost packet, exactly as the reference decoder does."""
    import torch
    T, N, S = x.shape
    cap = 256
    dev = torch.device("cuda", 0)
    eb = sb.EncoderBatch(N, rate=rate, dtx=dtx, use_md_index=use_md_index, framesize_ms=framesize_ms, joint_hb=joint_hb)
    db = sb.DecoderBatch(N, use_md_index=use_md_index, framesize_ms=framesize_ms, joint_hb=joint_hb)
    kw = dict(use_md_index=use_md_index, framesize_ms=framesize_ms, joint_hb=joint_hb)
    renc = [ref.RefEncoder("fix", rate=rate, dtx=dtx, **kw) for _ in range(N)]
    rdec = [ref.RefDecoder("flp", **kw) for _ in range(N)]
    flags = loss_with_bursts(T, N)
    d_pcm = torch.zeros((N, S), dtype=torch.int16, device=dev)
    d_bits = torch.zeros((N, cap), dtype=torch.uint8, device=dev)
    d_nb = torch.zeros((N, 2), dtype=torch.int16, device=dev)
    d_tb = torch.zeros((N, cap), dtype=torch.uint8, device=dev)
    d_tnb = torch.zeros((N, 2), dtype=torch.int16, device=dev)
    d_f = torch.zeros(N, dtype=torch.int32, device=dev)
    d_out = torch.zeros((N, S), dtype=torch.int16, device=dev)
    d_ret = torch.zeros(N, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    dtx_rows = 0

    def ref_row(args):
        s, p = args
        b, rnb, n = renc[s].encode(x[p, s])
        f = int(flags[s, p])
        if rnb[0] <= 0:      # DTX packet: nothing is sent, the receiver conceals
            pb, pnb, f = bytes(16), (16, 8), 1
        else:
            pb, pnb = trim_payload(b, rnb, f)
        y, r = rdec[s].decode(pb, pnb, f)
        return b, rnb, n, pb, pnb, f, y, r

    with ThreadPoolExecutor(workers) as pool:
        for p in range(T):
            d_pcm.copy_(torch.from_numpy(x[p]))
            eb.encode_device(d_pcm.data_ptr(), d_bits.data_ptr(), cap, d_nb.data_ptr(), st)
            rows = list(pool.map(ref_row, [(s, p) for s in range(N)]))
            torch.cuda.synchronize()
            bits, nb = d_bits.cpu().numpy(), d_nb.cpu().numpy()
            tb = np.zeros((N, cap), np.uint8)
            tnb = np.zeros((N, 2), np.int16)
            f_eff = np.zeros(N, np.int32)
            want = np.zeros((N, S), np.int16)
            for s, (b, rnb, n, pb, pnb, f, y, r) in enumerate(rows):
                assert tuple(nb[s]) == rnb, ("length fields", p, s, s % 8)
                assert bytes(bits[s, :max(n, 0)]) == b[:max(n, 0)], ("payload", p, s, s % 8)
                assert r == 0
                dtx_rows += rnb[0] <= 0
                tb[s, :len(pb)] = np.frombuffer(pb, np.uint8)
                tnb[s] = pnb
                f_eff[s] = f
                want[s] = y
            d_tb.copy_(torch.from_numpy(tb)); d_tnb.copy_(torch.from_numpy(tnb)); d_f.copy_(torch.from_numpy(f_eff))
            db.decode_device(d_out.data_ptr(), d_tb.data_ptr(), cap, d_tnb.data_ptr(), d_f.data_ptr(), d_ret.data_ptr(), st)
            torch.cuda.synchronize()
            assert int((d_ret != 0).sum().item()) == 0, ("decoder return", p)
            d = np.abs(d_out.cpu().numpy().astype(np.int32) - want.astype(np.int32)).max(axis=1)
            assert d.max() <= PCM_TOL, ("pcm", p, int(d.argmax()), int(d.argmax()) % 8, int(f_eff[d.argmax()]), int(d.max()))
    for o in renc + rdec:
        o.close()
    eb.close(); db.close()
    return dtx_rows


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", [
    dict(dtx=1),
    dict(dtx=1, use_md_index=1, framesize_ms=20),
    dict(dtx=1, joint_hb=1),
    dict(use_md_index=1),
], ids=["40ms_dtx", "20ms_dtx_mdi", "joint1_dtx", "40ms_mdi"])
def test_near_silence_next_to_speech_on_the_device(sb, ref, cfg):
    S = 16 * cfg.get("framesize_ms", 40)
    x = near_silent_classes(load_clip(), 37, 60, samples=S)
    dtx_rows = run_device_against_reference(sb, ref, x, **cfg)
    if cfg.get("dtx"):
        assert dtx_rows > 0, "no stream entered DTX: the near-silent rows did not reach comfort-noise coding"


def _cap_inputs(N, T, seed=21):
    clip = load_clip()
    x = near_silent_classes(clip, N, T, seed=seed)
    # loud, noisy rows produce the largest packets at high rates
    rng = np.random.Generator(np.random.PCG64(seed))
    for s in range(0, N, 3):
        x[:, s] = np.clip(rng.normal(0, 12000, (T, 640)), -32768, 32767).astype(np.int16)
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["host", "device"])
def test_batched_encode_below_the_packet_size(sb, ref, entry):
    import torch
    N, T = 29, 6
    rates = np.array([6000, 10000, 13600, 24000, 40000, 64000, 100000] * 5)[:N]
    dtx = (np.arange(N) % 4 == 3).astype(np.int32)           # every fourth row with DTX (silent classes go quiet)
    x = _cap_inputs(N, T)
    # the largest packet of this input, from the reference
    want = []
    for s in range(N):
        e = ref.RefEncoder("fix", rate=int(rates[s]), dtx=int(dtx[s]))
        want.append([e.encode(x[p, s]) for p in range(T)])
        e.close()
    biggest = max(n for row in want for (_, _, n) in row)
    assert biggest > 64
    assert sum(rnb[0] <= 0 for row in want for (_, rnb, _) in row) > 0, "no DTX row dropped a packet: the DTX case is not run"
    for cap in sorted({16, 17, 31, 64, biggest - 1, biggest}):
        eb = sb.EncoderBatch(N)
        eb.set_control(rate=rates, dtx=dtx)
        dev = torch.device("cuda", 0)
        canary = 0xA5
        for p in range(T):
            if entry == "host":
                bits = np.full((N + 1, cap), canary, np.uint8)      # a canary row after the batch
                nb = np.zeros((N, 2), np.int16)
                eb.encode(x[p], cap=cap, bits=bits[:N], nbytes=nb)
                tail = bits[N]
            else:
                d_bits = torch.full((N + 1, cap), canary, dtype=torch.uint8, device=dev)
                d_nb = torch.zeros((N, 2), dtype=torch.int16, device=dev)
                d_pcm = torch.from_numpy(np.ascontiguousarray(x[p])).to(dev)
                eb.encode_device(d_pcm.data_ptr(), d_bits.data_ptr(), cap, d_nb.data_ptr(), torch.cuda.current_stream().cuda_stream)
                torch.cuda.synchronize()
                bits, nb = d_bits.cpu().numpy(), d_nb.cpu().numpy()
                tail = bits[N]
            assert (tail == canary).all(), ("bytes written past the last row", cap, p)
            for s in range(N):
                b, rnb, n = want[s][p]
                assert tuple(nb[s]) == rnb, ("length fields", cap, p, s)
                k = min(cap, max(n, 0))
                assert bytes(bits[s, :k]) == b[:k], ("payload prefix", cap, p, s)
        eb.close()
