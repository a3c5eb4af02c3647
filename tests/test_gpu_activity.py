"""Activity reports on the GPU (sb_activity_kernel through the C ABI), at 0 tolerance: every level equals the host function of
the PCM row it reports on, every flags byte the host model's (tests/hostsim), and the packet calls' outputs
and launch counts are the same with and without activity calls."""
import hashlib

import numpy as np
import pytest

from solo_b200 import api
from tests.golden import make_golden_32k as mk
from tests.parity import DeviceDecoder, batch_rows, received, sb, sim  # noqa: F401  (fixtures)
from tests.util import load_clip, load_golden, loss_flags, receive, signal_classes

pytestmark = pytest.mark.gpu
CAP = 256
RATES = (6000, 13600, 24000)


def levels(sim, rows):
    return np.array([sim.row_level(r) for r in rows], np.uint8)


def test_encoder_batch(sb, sim):
    """N = 256 streams of the eight signal classes at 6 / 13.6 / 24 kb/s, 40 packets, through encode + activity (host
    entry points), encode_device + activity_device and encode alone: level = the host function of the input rows, flags =
    the host model's, and payloads / nbytes byte-identical in all three (and equal to the host model's)."""
    import torch
    N, T = 256, 40
    x = signal_classes(load_clip(), N, T)
    rate = np.array([RATES[s % 3] for s in range(N)], np.int32)
    ea, eb, ed = (sb.EncoderBatch(N) for _ in range(3))
    for e in (ea, eb, ed):
        e.set_control(rate=rate)
    hm = [sim.SimEncoder(rate=int(rate[s])) for s in range(N)]
    dev = torch.device("cuda", 0)
    d_pcm = torch.zeros((N, 640), dtype=torch.int16, device=dev)
    d_bits = torch.zeros((N, CAP), dtype=torch.uint8, device=dev)
    d_nb = torch.zeros((N, 2), dtype=torch.int16, device=dev)
    d_lv = torch.zeros(N, dtype=torch.uint8, device=dev)
    d_fl = torch.zeros(N, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    seen = set()
    for p in range(T):
        ba, na = ea.encode(x[p], cap=CAP)
        lv, fl = ea.activity()
        bb, nb_ = eb.encode(x[p], cap=CAP)
        d_pcm.copy_(torch.from_numpy(x[p]))
        ed.encode_device(d_pcm.data_ptr(), d_bits.data_ptr(), CAP, d_nb.data_ptr(), st)
        ed.activity_device(d_pcm.data_ptr(), d_lv.data_ptr(), d_fl.data_ptr(), st)
        torch.cuda.synchronize()
        assert np.array_equal(ba, bb) and np.array_equal(na, nb_), p
        assert np.array_equal(d_bits.cpu().numpy(), ba) and np.array_equal(d_nb.cpu().numpy(), na), p
        assert np.array_equal(lv, levels(sim, x[p])), p
        assert np.array_equal(d_lv.cpu().numpy(), lv) and np.array_equal(d_fl.cpu().numpy(), fl), p
        for s in range(N):
            b, nb, _ = hm[s].encode(x[p, s])
            assert nb == tuple(int(v) for v in na[s]) and bytes(ba[s, :max(nb[0], 0)]) == b[:max(nb[0], 0)], (p, s)
            assert fl[s] == hm[s].flags, (p, s, int(fl[s]), hm[s].flags)
        seen.update(int(v) for v in fl)
    assert {0, 3} <= seen
    for e in (ea, eb, ed):
        e.close()
    for h in hm:
        h.close()


def test_clip_payloads_with_activity_calls_equal_the_reference(sb):
    """The clip through a batch with an activity call after every packet: payloads equal golden.npz's (the reference FIX
    encoder's) byte for byte."""
    g = load_golden()
    clip = load_clip()
    e = sb.EncoderBatch(3, rate=13600)
    for p in range(60):
        bits, nb = e.encode(np.tile(clip[p * 640:(p + 1) * 640], (3, 1)), cap=128)
        e.activity()
        n0 = int(g["fix_nbytes"][p, 0])
        assert tuple(nb[1]) == tuple(g["fix_nbytes"][p]) and bytes(bits[1, :n0]) == bytes(g["fix_bits"][p, :n0]), p
    e.close()


def dec_cases():
    """(name, samplerate, decoder kwargs, arith, packets, pinned md5 key or None, pinned flags or None)."""
    g, f = load_golden(), mk.load()
    pk16 = [(bytes(g["fix_bits"][p, :int(g["fix_nbytes"][p, 0])]), tuple(int(v) for v in g["fix_nbytes"][p])) for p in range(60)]
    out = [("16k-40ms-flp", 16000, dict(framesize_ms=40), "flp", pk16, None, None)]
    for s, arith in (("hb40", "flp"), ("hb40", "fix"), ("hb20", "flp"), ("joint", "flp"), ("joint", "fix")):
        out.append(("32k-%s-%s" % (s, arith), 32000, mk.STREAMS[s][1], arith, mk.packets(f, s)[:60],
                    "%s_%s_loss_packet_md5" % (arith, s), mk.flags_of(f, s, "loss")[:60]))
    return out


def enc16(sim, cfg):
    clip = load_clip()
    e = sim.SimEncoder(rate=13600, **cfg)
    k = e.samples
    pk = [e.encode(clip[p * k:(p + 1) * k])[:2] for p in range(60)]
    e.close()
    return pk


@pytest.mark.parametrize("case", range(8))
def test_decoder_batches_under_per_stream_loss(sb, sim, case):
    """N = 64 streams per batch, each under its own 50 % loss process (row 0: the fixture's loss flags), through decode +
    activity (host) and decode_device + activity_device: level = the host function of the output rows, flags = the host
    model's, PCM = the host model's (row 0: the fixture's md5); chunking (1 or 3) changes nothing."""
    cases = dec_cases()
    cases += [("16k-20ms-flp", 16000, dict(framesize_ms=20), "flp", enc16(sim, dict(framesize_ms=20)), None, None),
              ("16k-joint-fix", 16000, dict(framesize_ms=40, joint_hb=1), "fix", enc16(sim, dict(framesize_ms=40, joint_hb=1)), None, None)]
    name, sr, cfg, arith, pk, md5key, pinned = cases[case]
    f32 = mk.load()
    N, T = 64, len(pk)
    flags = np.array([loss_flags(T, 50, seed=40 + s) for s in range(N)], np.int32)
    if pinned is not None:
        flags[0] = pinned
    dh = sb.DecoderBatch(N, arith=arith, samplerate=sr, **cfg)
    dd = DeviceDecoder(sb.DecoderBatch(N, arith=arith, samplerate=sr, **cfg), CAP)
    hm = [sim.SimDecoder(arith=arith, samplerate=sr, **cfg) for _ in range(N)]
    for p in range(T):
        sb.set_chunks(1 if p % 2 else 3)
        rx = [receive(pk[p][0], pk[p][1], int(flags[s, p])) for s in range(N)]
        tb, tnb, tf = batch_rows(rx, CAP)
        pcm, ret = dh.decode(tb, tnb, tf)
        lv, fl = dh.activity()
        assert (ret == 0).all()
        d_pcm, _ = dd.decode(tb, tnb, tf)
        d_lv, d_fl = dd.activity()
        assert np.array_equal(d_pcm, pcm) and np.array_equal(d_lv, lv) and np.array_equal(d_fl, fl), (name, p)
        assert np.array_equal(lv, levels(sim, pcm)), (name, p)
        for s in range(N):
            y, r = hm[s].decode(*rx[s])
            assert r == 0 and np.array_equal(y, pcm[s]) and hm[s].flags == fl[s], (name, p, s, int(fl[s]), hm[s].flags)
        if md5key:
            assert hashlib.md5(pcm[0].tobytes()).digest() == bytes(f32[md5key][p]), (name, p)
        conc = 0xC if cfg["framesize_ms"] == 40 else 0x4
        assert np.array_equal(fl & conc != 0, tf == 1), (name, p)
    sb.set_chunks(0)
    dh.close(), dd.db.close()
    for h in hm:
        h.close()


def test_sample_of_a_65536_stream_batch(sb, sim):
    """One 65 536-stream 16 kHz decoder batch under per-row loss, through decode_device + activity_device: a fixed sample
    of 1 024 rows has the host model's flags and the host function's level of its output rows, for 12 packets."""
    import torch
    g = load_golden()
    N, T = 65536, 12
    rows = np.unique(np.concatenate([[0, N - 1], np.random.Generator(np.random.PCG64(66)).choice(N, 1022, replace=False)]))
    lost = np.random.Generator(np.random.PCG64(67)).random((T, N)) < 0.5
    db = sb.DecoderBatch(N)
    hm = [sim.SimDecoder() for _ in rows]
    dev = DeviceDecoder(db, CAP)
    for p in range(T):
        n0 = int(g["fix_nbytes"][p, 0])
        tb, tnb, _ = batch_rows([(bytes(g["fix_bits"][p, :n0]), g["fix_nbytes"][p], 4)], CAP)      # broadcast on the device
        pcm, _ = dev.decode(tb, tnb, np.where(lost[p], 1, 4), rows=rows)
        lv, fl = dev.activity(rows=rows)
        assert np.array_equal(lv, levels(sim, pcm)), p
        for i, s in enumerate(rows):
            y, r = hm[i].decode(bytes(g["fix_bits"][p, :n0]), tuple(int(v) for v in g["fix_nbytes"][p]), 1 if lost[p, s] else 4)
            assert r == 0 and hm[i].flags == fl[i] and np.array_equal(y, pcm[i]), (p, int(s))
    db.close()
    for h in hm:
        h.close()
    del dev
    torch.cuda.empty_cache()


def test_drop_in_handles_report_what_the_batch_row_reports(sb):
    """Encoder handles and 16 / 32 kHz decoder handles report, packet by packet, the level / flags of a batch row that codes
    the same stream; before their first packet, and for NULL or foreign handles, the calls fail."""
    f = mk.load()
    clip = load_clip()
    he = sb.SoloEncoder(rate=13600, dtx=1)
    h16, h32 = sb.SoloDecoder(), sb.SoloDecoder(samplerate=32000)
    eb, d16, d32 = sb.EncoderBatch(2, rate=13600, dtx=1), sb.DecoderBatch(2), sb.DecoderBatch(2, samplerate=32000)
    lv = np.zeros(1, np.uint8)
    for h in (he, h16, h32):
        assert sb.lib().solo_b200_encoder_last_activity(he.h, lv.ctypes.data, lv.ctypes.data) == -1
        assert sb.lib().solo_b200_decoder_last_activity(h.h, lv.ctypes.data, lv.ctypes.data) == -1
    assert sb.lib().solo_b200_decoder_last_activity(None, lv.ctypes.data, lv.ctypes.data) == -1
    with pytest.raises(sb.SoloError):
        eb.activity()
    pk32, fl32 = mk.packets(f, "hb40"), mk.flags_of(f, "hb40", "loss")
    x = np.concatenate([clip[:640 * 30], np.zeros(640 * 20, np.int16)])
    fl16 = loss_flags(50, 50, seed=9)
    for p in range(50):
        b, nb, n = he.encode(x[p * 640:(p + 1) * 640])
        bits, nbb = eb.encode(np.tile(x[p * 640:(p + 1) * 640], (2, 1)), cap=CAP)
        assert he.last_activity() == tuple(int(a[1]) for a in eb.activity()), p
        rx = receive(b, nb, fl16[p])
        y, r = h16.decode(*rx)
        d16.decode(*batch_rows([rx] * 2, CAP))
        assert h16.last_activity() == tuple(int(a[0]) for a in d16.activity()), p
        rx = receive(pk32[p][0], pk32[p][1], fl32[p])
        y, r = h32.decode(*rx)
        d32.decode(*batch_rows([rx] * 2, CAP))
        assert h32.last_activity() == tuple(int(a[1]) for a in d32.activity()), p
    assert sb.lib().solo_b200_encoder_last_activity(h16.h, lv.ctypes.data, lv.ctypes.data) == -1     # foreign handle
    for o in (he, h16, h32, eb, d16, d32):
        o.close()


def test_malformed_rows_report_127_and_no_flags(sb):
    """A 32 kHz batch whose odd rows get garbage, 16 kHz streams' packets, lying lengths or bad lostflags: the even rows
    report what a clean batch's do, and every rejected row reports level 127 and flags 0."""
    f, g = mk.load(), load_golden()
    pk = mk.packets(f, "hb40")
    N = 200
    rng = np.random.Generator(np.random.PCG64(12))
    clean, mixed = sb.DecoderBatch(N, samplerate=32000), sb.DecoderBatch(N, samplerate=32000)
    rejected = 0
    for p in range(30):
        tb, tnb, tf = received([pk[p]] * N, [4] * N, CAP)
        pc, rc = clean.decode(tb, tnb, tf)
        lc, fc = clean.activity()
        mb, mnb, mf = tb.copy(), tnb.copy(), tf.copy()
        for s in range(1, N, 2):
            k = (s // 2 + p) % 4
            if k == 0:
                mb[s] = rng.integers(0, 256, CAP, dtype=np.uint8)
            elif k == 1:
                n0 = int(g["fix_nbytes"][p, 0])
                mb[s] = 0
                mb[s, :n0] = g["fix_bits"][p, :n0]
                mnb[s] = g["fix_nbytes"][p]
            elif k == 2:
                mnb[s] = (int(rng.integers(-5, 2000)), int(rng.integers(-5, 2000)))
            else:
                mf[s] = int(rng.integers(-3, 9))
        pm, rm = mixed.decode(mb, mnb, mf)
        lm, fm = mixed.activity()
        assert np.array_equal(lm[0::2], lc[0::2]) and np.array_equal(fm[0::2], fc[0::2]), p
        bad = rm < 0
        assert (lm[bad] == 127).all() and (fm[bad] == 0).all(), p
        rejected += int(bad.sum())
    assert rejected > 0
    clean.close(), mixed.close()


def test_launch_counts_and_wave_kind(sb):
    """A packet wave launches what it launched before (encoder 8, decoder 2 with one chunk); each activity call adds one
    launch.  Host activity after a device wave, and the reverse, are refused."""
    import torch
    sb.set_chunks(1)
    x = np.tile(load_clip()[:640], (8, 1))
    e, d = sb.EncoderBatch(8), sb.DecoderBatch(8)
    with pytest.raises(sb.SoloError):
        d.activity()
    k0 = sb.kernel_launches()
    bits, nb = e.encode(x, cap=CAP)
    k1 = sb.kernel_launches()
    e.activity()
    k2 = sb.kernel_launches()
    d.decode(bits, nb, np.full(8, 4, np.int32))
    k3 = sb.kernel_launches()
    d.activity()
    k4 = sb.kernel_launches()
    assert (k1 - k0, k2 - k1, k3 - k2, k4 - k3) == (8, 1, 2, 1)
    dev = torch.device("cuda", 0)
    d_x = torch.from_numpy(x).to(dev)
    d_b = torch.zeros((8, CAP), dtype=torch.uint8, device=dev)
    d_nb = torch.zeros((8, 2), dtype=torch.int16, device=dev)
    d_o = torch.zeros(8, dtype=torch.uint8, device=dev)
    with pytest.raises(sb.SoloError, match="host"):
        e.activity_device(d_x.data_ptr(), d_o.data_ptr(), d_o.data_ptr())
    e.encode_device(d_x.data_ptr(), d_b.data_ptr(), CAP, d_nb.data_ptr())
    with pytest.raises(sb.SoloError, match="device"):
        e.activity()
    torch.cuda.synchronize()
    sb.set_chunks(0)
    e.close(), d.close()
