"""Encoder settings changed between packets on the GPU: per-stream target rate, DTX and expected packet loss through the
three entry points (set_control_device, set_control_host, solo_b200_encoder_set_control), with different schedules in
neighbouring streams of a warp / block.  Every checked row is compared with the unmodified reference fed the same schedule:
payload bytes and length fields against libjc1_fix.so (oracle.ref.RefEncoder.set_control writes the settings into its
handle), decoded PCM under a per-stream 50 % loss process against libjc1_flp.so.  Tolerances: payloads bit-exact, PCM 0 LSB."""
import ctypes as C

import numpy as np
import pytest

from tests.parity import DevicePath, RefRows, control_args, lockstep, ref, sb  # noqa: F401  (fixtures)
from tests.util import load_clip, loss_flags, signal_classes, speech_replay

pytestmark = pytest.mark.gpu


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
    eb_d, eb_h = sb.EncoderBatch(N), sb.EncoderBatch(N)
    dp = DevicePath(sb, eb_d, cap=cap, stream=torch.cuda.Stream())
    sample = list(range(0, N, 4))
    db = sb.DecoderBatch(len(sample))
    rr = RefRows(ref, range(N), decode="ref", pcm_rows=sample)
    flags = np.array([loss_flags(T, 50, seed=1 + s) for s in sample], np.int32)
    for p in range(T):
        lp = None if p in no_loss_array else loss[p]
        dp.encode(x[p], control=(rate[p], dtx[p], lp))
        eb_h.set_control(rate=rate[p], dtx=dtx[p], loss=lp)
        hbits, hnb = eb_h.encode(x[p], cap=cap)
        bits, nb, _ = dp.rows()
        assert np.array_equal(nb, hnb), p
        rx = rr.step(x[p], bits, nb, flags[:, p], control=(rate[p], dtx[p], np.full(N, -1) if lp is None else lp))
        for s, (b, _, n) in enumerate(rr.packets):
            assert bytes(hbits[s, :max(n, 0)]) == b, (p, s)
        pcm, ret = db.decode(*rx)
        assert (ret == 0).all()
        rr.check_pcm(pcm)
    assert rr.dtx_rows > 0                                   # DTX dropped packets
    rr.close()
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
        rate, dtx, loss = schedules(1, T, seed=40 + k, silence=(15, 30))
        xs = clip[spp * 20:spp * (20 + T)].copy()
        xs[15 * spp:30 * spp] = 0
        control = [control_args(rate[p, 0], dtx[p, 0], loss[p, 0]) for p in range(T)]
        lockstep((sb.SoloEncoder(**hk), None), (ref.RefEncoder("fix", **kw), None), xs.reshape(T, spp), control=control, tag=(kw,))


def test_export_import_in_the_middle_of_a_schedule(sb, ref):
    """A stream leaves its batch (slot 5 of 16) half way through its schedule and joins another one (slot 2 of 4): its
    settings travel with the state, and the rest of the schedule gives the reference's packets."""
    N, T0, T1, cap = 16, 12, 12, 1024
    x = speech_replay(load_clip(), N, T0 + T1)
    rate, dtx, loss = schedules(N, T0 + T1, seed=8)
    loss[T0 - 2, 5], rate[T0 - 1, 5] = 37, 24000              # settings made just before the export
    eb = sb.EncoderBatch(N)
    r = ref.RefEncoder("fix")
    for p in range(T0):
        eb.set_control(rate=rate[p], dtx=dtx[p], loss=loss[p])
        bits, nb = eb.encode(x[p], cap=cap)
        r.set_control(**control_args(rate[p, 5], dtx[p, 5], loss[p, 5]))
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
        r.set_control(**control_args(rate[p, 5], dtx[p, 5], loss[p, 5]))
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
    N, T, cap = 65536, 6, 1024
    clip = load_clip()
    rate, dtx, loss = schedules(N, T, seed=21)
    rate[0] = np.exp(np.random.Generator(np.random.PCG64(2)).uniform(np.log(3000), np.log(120000), N)).astype(np.int32)
    sample = sorted(set(list(range(0, N, 257)) + [1, 2, 3, 31, 32, N - 1]))
    eb = sb.EncoderBatch(N)
    dp, rr = DevicePath(sb, eb, cap=cap), RefRows(ref, sample)
    for p in range(T):
        xh = speech_replay(clip, N, 1, first_packet=p)[0]
        control = (rate[p], dtx[p], loss[p]) if p in (0, 3) else None
        dp.encode(xh, control=control)
        bits, nb, _ = dp.rows(sample)
        rr.step(xh[sample], bits, nb, control=None if control is None else tuple(c[sample] for c in control))
    rr.close()
    eb.close()
