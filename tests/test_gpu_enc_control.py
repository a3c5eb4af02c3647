"""Encoder settings changed between packets on the GPU: per-stream target rate, DTX and expected packet loss through the
three entry points (set_control_device, set_control_host, solo_b200_encoder_set_control), with different schedules in
neighbouring streams of a warp / block.  Every checked row is compared with the unmodified reference fed the same schedule:
payload bytes and length fields against libjc1_fix.so (tests/enc_control_ref.py writes the settings into its handle), decoded
PCM under a per-stream 50 % loss process against libjc1_flp.so.  Tolerances: payloads bit-exact, PCM 0 LSB."""
import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from tests.test_gpu_hetero import signal_classes
from tests.enc_control_ref import RefEncoder as ControlledRefEncoder
from tests.util import load_clip, loss_flags, speech_replay, trim_payload

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sb():
    import solo_b200
    solo_b200.lib()
    return solo_b200


@pytest.fixture(scope="module")
def ref():
    from oracle import ref as r
    if not r.available():
        pytest.skip("oracle/_ref not built")
    r.lib("fix"), r.lib("flp")          # loaded once, before thread pools drive the reference
    return r


def schedules(N, T, seed, silence=None):
    """int32 [T, N] rate / dtx / loss arrays, -1 = unchanged: every stream its own schedule.  Rates log-uniform in
    [3 000, 120 000] b/s, loss 0-100, DTX toggled (per stream, at different packets) inside the silent stretch."""
    rng = np.random.Generator(np.random.PCG64(seed))
    rate = np.where(rng.random((T, N)) < 0.3, np.exp(rng.uniform(np.log(3000), np.log(120000), (T, N))), -1).astype(np.int32)
    loss = np.where(rng.random((T, N)) < 0.3, rng.integers(0, 101, (T, N)), -1).astype(np.int32)
    dtx = np.full((T, N), -1, np.int32)
    if silence:
        a, b = silence
        dtx[a] = rng.integers(0, 2, N)
        for _ in range(3):
            p = rng.integers(a + 1, b, N)
            dtx[p, np.arange(N)] = rng.integers(0, 2, N)
    rate[1, ::7], rate[2, 3::7] = 3000, 120000               # both clamps of the SILK core's [5000, 100000]
    return rate, dtx, loss


def ref_control(enc, rate, dtx, loss):
    c = {k: int(v) for k, v in (("rate", rate), ("dtx", dtx), ("loss", loss)) if v != -1}
    if c:
        enc.set_control(**c)


def test_4096_streams_50_packets_device_and_host_flavour_match_the_reference(sb, ref):
    """4 096 streams x 50 packets of the eight signal classes, each stream with its own schedule, through
    set_control_device + encode_device on a non-default CUDA stream: every row equals the reference.  A second batch
    driven through set_control_host + encode_host gives the same bytes.  1 024 sampled rows are decoded under a 50 % loss
    process per stream, PCM identical to libjc1_flp.so."""
    import torch
    N, T, cap = 4096, 50, 1024          # room for a 100 kb/s packet of full-scale noise
    silence = (20, 32)
    x = signal_classes(load_clip(), N, T, seed=17)
    x[silence[0]:silence[1]] = 0
    rate, dtx, loss = schedules(N, T, seed=3, silence=silence)
    no_loss_array = {p for p in range(T) if p % 7 == 3}     # packets whose call passes NULL for the loss array
    dev = torch.device("cuda", 0)
    cs = torch.cuda.Stream()
    eb_d, eb_h = sb.EncoderBatch(N), sb.EncoderBatch(N)
    renc = [ControlledRefEncoder() for _ in range(N)]
    sample = list(range(0, N, 4))
    db = sb.DecoderBatch(len(sample))
    rdec = [ref.RefDecoder("flp") for _ in sample]
    flags = np.array([loss_flags(T, 50, seed=1 + s) for s in sample], np.int32)
    d_x = torch.zeros((N, 640), dtype=torch.int16, device=dev)
    d_bits, d_nb = torch.zeros((N, cap), dtype=torch.uint8, device=dev), torch.zeros((N, 2), dtype=torch.int16, device=dev)
    d_ctrl = torch.zeros((3, N), dtype=torch.int32, device=dev)

    def ref_row(args):
        s, p = args
        ref_control(renc[s], rate[p, s], dtx[p, s], -1 if p in no_loss_array else loss[p, s])
        return renc[s].encode(x[p, s])

    stats = {"zero": 0}
    with ThreadPoolExecutor(32) as pool:
        for p in range(T):
            with torch.cuda.stream(cs):
                d_x.copy_(torch.from_numpy(x[p]), non_blocking=False)
                d_ctrl.copy_(torch.from_numpy(np.stack([rate[p], dtx[p], loss[p]])))
                lp = None if p in no_loss_array else d_ctrl[2].data_ptr()
                eb_d.set_control_device(d_ctrl[0].data_ptr(), d_ctrl[1].data_ptr(), lp, cs.cuda_stream)
                eb_d.encode_device(d_x.data_ptr(), d_bits.data_ptr(), cap, d_nb.data_ptr(), cs.cuda_stream)
            eb_h.set_control(rate=rate[p], dtx=dtx[p], loss=None if p in no_loss_array else loss[p])
            hbits, hnb = eb_h.encode(x[p], cap=cap)
            rows = list(pool.map(ref_row, [(s, p) for s in range(N)]))
            cs.synchronize()
            bits, nb = d_bits.cpu().numpy(), d_nb.cpu().numpy()
            assert np.array_equal(nb, hnb), p
            dbits, dnb, f_eff, want = np.zeros((len(sample), cap), np.uint8), np.zeros((len(sample), 2), np.int16), np.zeros(len(sample), np.int32), []
            for s, (b, rnb, n) in enumerate(rows):
                assert tuple(nb[s]) == rnb and bytes(bits[s, :max(n, 0)]) == b[:max(n, 0)], (p, s, s % 8, rate[p, s], dtx[p, s], loss[p, s])
                assert bytes(hbits[s, :max(n, 0)]) == b[:max(n, 0)], (p, s)
                stats["zero"] += rnb[0] == 0
            for i, s in enumerate(sample):
                b, rnb, n = rows[s]
                f = int(flags[i, p])
                pb, pnb = (bytes(16), (16, 8)) if rnb[0] <= 0 else trim_payload(b, rnb, f)
                f = 1 if rnb[0] <= 0 else f
                dbits[i, :len(pb)] = np.frombuffer(pb, np.uint8)
                dnb[i], f_eff[i] = pnb, f
            want = list(pool.map(lambda i: rdec[i].decode(bytes(dbits[i, :dnb[i, 0]]), tuple(dnb[i]), int(f_eff[i])), range(len(sample))))
            pcm, ret = db.decode(dbits, dnb, f_eff)
            assert (ret == 0).all() and all(r == 0 for _, r in want)
            assert np.array_equal(pcm, np.stack([y for y, _ in want])), p
    assert stats["zero"] > 0                                 # DTX dropped packets
    for o in renc + rdec:
        o.close()
    eb_d.close(); eb_h.close(); db.close()


def test_drop_in_handles_follow_schedules(sb, ref):
    """solo_b200_encoder_set_control on AGR_Sate_Encoder_Init handles (40 ms, 20 ms, joint mode 1, DTX) matches the
    reference handle given the same calls."""
    clip = load_clip()
    T = 40
    for k, kw in enumerate((dict(), dict(framesize_ms=20), dict(joint_hb=1), dict(dtx=1))):
        spp = 16 * kw.get("framesize_ms", 40)
        hk = dict(kw)
        if hk.pop("joint_hb", 0):
            hk.update(joint_enable=1, joint_mode=1)
        e, r = sb.SoloEncoder(**hk), ControlledRefEncoder(**kw)
        rate, dtx, loss = schedules(1, T, seed=40 + k, silence=(15, 30))
        xs = clip[spp * 20:spp * (20 + T)].copy()
        xs[15 * spp:30 * spp] = 0
        for p in range(T):
            c = {n: int(v[p, 0]) for n, v in (("rate", rate), ("dtx", dtx), ("loss", loss)) if v[p, 0] != -1}
            if c:
                e.set_control(**c)
                r.set_control(**c)
            assert e.encode(xs[p * spp:(p + 1) * spp]) == r.encode(xs[p * spp:(p + 1) * spp]), (kw, p, c)
        e.close(); r.close()


def test_export_import_in_the_middle_of_a_schedule(sb, ref):
    """A stream leaves its batch (slot 5 of 16) half way through its schedule and joins another one (slot 2 of 4): its
    settings travel with the state, and the rest of the schedule gives the reference's packets."""
    N, T0, T1, cap = 16, 12, 12, 1024
    x = speech_replay(load_clip(), N, T0 + T1)
    rate, dtx, loss = schedules(N, T0 + T1, seed=8)
    loss[T0 - 2, 5], rate[T0 - 1, 5] = 37, 24000              # settings made just before the export
    eb = sb.EncoderBatch(N)
    r = ControlledRefEncoder()
    for p in range(T0):
        eb.set_control(rate=rate[p], dtx=dtx[p], loss=loss[p])
        bits, nb = eb.encode(x[p], cap=cap)
        ref_control(r, rate[p, 5], dtx[p, 5], loss[p, 5])
        b, rnb, n = r.encode(x[p, 5])
        assert tuple(nb[5]) == rnb and bytes(bits[5, :n]) == b
    blob = eb.export_state(5)
    eb.close()
    eb2 = sb.EncoderBatch(4, rate=9000)
    y = speech_replay(load_clip(), 4, 3, first_packet=40)
    for p in range(3):
        eb2.encode(y[p], cap=cap)
    eb2.import_state(2, blob)
    for p in range(T0, T0 + T1):
        xin = speech_replay(load_clip(), 4, 1, first_packet=50 + p)[0]
        xin[2] = x[p, 5]
        c = [np.full(4, -1, np.int32) for _ in range(3)]
        for k, v in enumerate((rate, dtx, loss)):
            c[k][2] = v[p, 5]
        eb2.set_control(rate=c[0], dtx=c[1], loss=c[2])
        bits, nb = eb2.encode(xin, cap=cap)
        ref_control(r, rate[p, 5], dtx[p, 5], loss[p, 5])
        b, rnb, n = r.encode(x[p, 5])
        assert tuple(nb[2]) == rnb and bytes(bits[2, :n]) == b, p
    eb2.close(); r.close()


def test_current_values_change_nothing_and_bad_arguments_apply_nothing(sb):
    """Setting the values a batch already has, before every packet, is byte-identical to never calling.  Out-of-range
    values make the host call and the handle call return -1 with nothing applied (the next packet shows it); a NULL or
    foreign handle and a NULL batch are refused."""
    N, T, cap = 67, 8, 256
    x = speech_replay(load_clip(), N, T)
    a, b, c = sb.EncoderBatch(N, rate=13600, dtx=1), sb.EncoderBatch(N, rate=13600, dtx=1), sb.EncoderBatch(N, rate=13600, dtx=1)
    ok = np.full(N, 24000, np.int32)
    for p in range(T):
        b.set_control(rate=13600, dtx=1, loss=0)
        for bad in (dict(rate=0), dict(rate=-2), dict(dtx=2), dict(dtx=-3), dict(loss=101), dict(loss=-4),
                    dict(rate=np.where(np.arange(N) == N - 1, 0, ok), loss=30)):
            with pytest.raises(sb.SoloError):
                c.set_control(**bad)
        ra, na = a.encode(x[p], cap=cap)
        rb, nbb = b.encode(x[p], cap=cap)
        rc, nc = c.encode(x[p], cap=cap)
        assert np.array_equal(na, nbb) and np.array_equal(na, nc), p
        for s in range(N):
            assert bytes(ra[s, :na[s, 0]]) == bytes(rb[s, :na[s, 0]]) == bytes(rc[s, :na[s, 0]]), (p, s)
    L = sb.lib()
    assert L.solo_b200_enc_batch_set_control_host(None, None, None, None) == -1
    assert L.solo_b200_enc_batch_set_control_device(None, None, None, None, None) == -1
    a.close(); b.close(); c.close()
    clip = load_clip()
    e, e0 = sb.SoloEncoder(rate=13600), sb.SoloEncoder(rate=13600)
    d = sb.SoloDecoder()
    for p in range(6):
        for bad in ((0, -1, -1), (-1, 2, -1), (-1, -1, 101), (24000, 0, -7)):
            assert L.solo_b200_encoder_set_control(e.h, *bad) == -1
        assert e.encode(clip[p * 640:(p + 1) * 640]) == e0.encode(clip[p * 640:(p + 1) * 640]), p
    assert L.solo_b200_encoder_set_control(None, 24000, -1, -1) == -1
    assert L.solo_b200_encoder_set_control(d.h, 24000, -1, -1) == -1          # a decoder handle
    junk = (C.c_uint32 * 16)()
    assert L.solo_b200_encoder_set_control(C.addressof(junk), 24000, -1, -1) == -1
    e.close(); e0.close(); d.close()


def test_full_65536_stream_wave_after_a_control_call(sb, ref):
    """A control call for all 65 536 streams of a full batch (device arrays, then again before packet 3) ahead of the packet
    waves; sampled rows against the reference."""
    import torch
    N, T, cap = 65536, 6, 1024
    clip = load_clip()
    rate, dtx, loss = schedules(N, T, seed=21)
    rate[0] = np.exp(np.random.Generator(np.random.PCG64(2)).uniform(np.log(3000), np.log(120000), N)).astype(np.int32)
    dev = torch.device("cuda", 0)
    sample = sorted(set(list(range(0, N, 257)) + [1, 2, 3, 31, 32, N - 1]))
    renc = {s: ControlledRefEncoder() for s in sample}
    eb = sb.EncoderBatch(N)
    d_bits, d_nb = torch.zeros((N, cap), dtype=torch.uint8, device=dev), torch.zeros((N, 2), dtype=torch.int16, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    idx = torch.tensor(sample, device=dev)
    for p in range(T):
        xh = speech_replay(clip, N, 1, first_packet=p)[0]
        if p in (0, 3):
            d_c = torch.from_numpy(np.stack([rate[p], dtx[p], loss[p]])).to(dev)
            eb.set_control_device(d_c[0].data_ptr(), d_c[1].data_ptr(), d_c[2].data_ptr(), st)
        eb.encode_device(torch.from_numpy(xh).to(dev).data_ptr(), d_bits.data_ptr(), cap, d_nb.data_ptr(), st)
        torch.cuda.synchronize()
        bits, nb = d_bits[idx].cpu().numpy(), d_nb[idx].cpu().numpy()
        for i, s in enumerate(sample):
            if p in (0, 3):
                ref_control(renc[s], rate[p, s], dtx[p, s], loss[p, s])
            b, rnb, n = renc[s].encode(xh[s])
            assert tuple(nb[i]) == rnb and bytes(bits[i, :n]) == b, (p, s)
    for o in renc.values():
        o.close()
    eb.close()
