"""32 kHz streams through the GPU decoder (the DecState32 instantiation of the decoder kernels), through the C ABI: the
batched host and device entry points, the drop-in handles and the state hand-over, in both decoder arithmetics.  Every PCM
comparison is exact (0 LSB): against golden_32k.npz's per-packet md5, or against the reference's decoders in oracle/_ref."""
import ctypes as C
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from solo_b200 import api
from tests.golden import make_golden_32k as mk
from tests.parity import DeviceDecoder, batch_rows, received, ref, sb  # noqa: F401  (fixtures)
from tests.util import load_golden, loss_flags, receive

pytestmark = pytest.mark.gpu
CAP = 256

CASES = mk.decode_cases()


@pytest.mark.parametrize("key,stream,kind,rule", CASES, ids=[c[0] for c in CASES])
def test_fixture_on_batched_host_and_device_calls(sb, key, stream, kind, rule):
    """N = 257 streams that all decode one fixture stream, through decode_host and decode_device: every row of every
    packet has the reference's PCM (per-packet md5, 0 LSB)."""
    f = mk.load()
    cfg = mk.STREAMS[stream][1]
    pk, flags = mk.packets(f, stream), mk.flags_of(f, stream, rule)
    want = f[key + "_packet_md5"]
    N = 257
    dh = sb.DecoderBatch(N, arith=kind, samplerate=32000, **cfg)
    dd = sb.DecoderBatch(N, arith=kind, samplerate=32000, **cfg)
    assert dh.samples == 32 * cfg["framesize_ms"]
    dev = DeviceDecoder(dd, CAP)
    for p in range(len(pk)):
        tb, tnb, tf = received([pk[p]] * N, [flags[p]] * N, CAP)
        pcm, ret = dh.decode(tb, tnb, tf)
        assert (ret == 0).all(), p
        assert (mk.packet_md5(pcm) == want[p]).all(), ("host entry point: PCM differs from the reference's (0 LSB bar)", key, p)
        assert np.array_equal(dev.decode(tb, tnb, tf)[0], pcm), ("device entry point differs from host entry point", key, p)
    dh.close(), dd.close()


@pytest.mark.parametrize("arith,stream,rule", [("flp", "hb40", "loss"), ("fix", "joint", "loss")])
def test_fixture_on_a_65536_stream_batch(sb, arith, stream, rule):
    """One wave of 65 536 32 kHz streams through decode_device; a fixed sample of 1 024 rows (first, last and spread) is
    checked against the fixture's per-packet md5 (0 LSB) for the first 30 packets."""
    import torch
    f = mk.load()
    cfg = mk.STREAMS[stream][1]
    key = "%s_%s_%s" % (arith, stream, rule)
    pk, flags, want = mk.packets(f, stream), mk.flags_of(f, stream, rule), f[key + "_packet_md5"]
    N = 65536
    rows = np.unique(np.concatenate([[0, N - 1], np.random.Generator(np.random.PCG64(65)).choice(N, 1022, replace=False)]))
    db = sb.DecoderBatch(N, arith=arith, samplerate=32000, **cfg)
    dev = DeviceDecoder(db, CAP)
    for p in range(30):
        pcm, _ = dev.decode(*received([pk[p]], [flags[p]], CAP), rows=rows)      # one row, broadcast on the device
        got = mk.packet_md5(pcm)
        assert (got == want[p]).all(), ("PCM differs from the reference's (0 LSB bar)", key, p, int(rows[np.argmax((got != want[p]).any(1))]))
    db.close()
    del dev
    torch.cuda.empty_cache()


@pytest.mark.parametrize("cfg", [dict(framesize_ms=40), dict(framesize_ms=20), dict(framesize_ms=40, joint_hb=1)],
                         ids=["40ms", "20ms", "joint"])
def test_per_stream_loss_against_reference(sb, ref, cfg):
    """N = 97 streams, each its own signal (the fixture's input at its own offset, FIX-encoded at 32 kHz by the reference)
    and its own 50 % loss process; every row of every packet equal to the reference's float decoder and, where that mode
    exists, to its fixed-point decoder (0 LSB)."""
    x = mk.inputs()["hb"]
    N, T = 97, 16
    kinds = ["flp"] + (["fix"] if cfg["framesize_ms"] == 40 else [])
    pool = ThreadPoolExecutor(32)
    enc = [ref.RefEncoder("fix", rate=16000 + 1000 * (s % 9), samplerate=32000, **cfg) for s in range(N)]
    k = enc[0].samples
    off = [(s * 7919) % (len(x) - k * T) for s in range(N)]
    pk = []
    for p in range(T):          # one packet of every stream at a time: each encoder sees its packets in order
        pk.append(list(pool.map(lambda s: enc[s].encode(x[off[s] + p * k:off[s] + (p + 1) * k])[:2], range(N))))
    flags = np.array([loss_flags(T, 50, seed=31 + s) for s in range(N)], np.int32)
    for kind in kinds:
        db = sb.DecoderBatch(N, arith=kind, samplerate=32000, **cfg)
        rd = [ref.RefDecoder(kind, samplerate=32000, **cfg) for _ in range(N)]
        for p in range(T):
            tb, tnb, tf = received(pk[p], flags[:, p], CAP)
            pcm, ret = db.decode(tb, tnb, tf)
            assert (ret == 0).all(), p
            want = list(pool.map(lambda s: rd[s].decode(bytes(tb[s, :tnb[s, 0]]), tuple(tnb[s]), int(tf[s])), range(N)))
            for s in range(N):
                assert want[s][1] == 0 and np.array_equal(pcm[s], want[s][0]), (kind, p, s, "PCM differs (0 LSB bar)")
        for d in rd:
            d.close()
        db.close()
    for e in enc:
        e.close()
    pool.shutdown()


def test_chunking_does_not_change_pcm(sb):
    """The host entry point's pipelining (1, 3 and 7 chunks) gives the same PCM on a 32 kHz batch."""
    f = mk.load()
    pk, flags = mk.packets(f, "hb40"), mk.flags_of(f, "hb40", "loss")
    N = 6000
    out = {}
    for c in (1, 3, 7):
        sb.set_chunks(c)
        db = sb.DecoderBatch(N, samplerate=32000)
        res = []
        for p in range(12):
            tb, tnb, tf = received([pk[p]] * N, [flags[p]] * N, CAP)
            # rows differ: stream s starts s % 5 packets later into the lossy sequence (lost packets in its place before)
            tf = np.where(np.arange(N) % 5 > p, 1, tf).astype(np.int32)
            pcm, ret = db.decode(tb, tnb, tf)
            assert (ret == 0).all()
            res.append(pcm.copy())
        out[c] = np.stack(res)
        db.close()
    sb.set_chunks(0)
    assert np.array_equal(out[1], out[3]) and np.array_equal(out[1], out[7])


def test_state_export_import_and_refused_cross_rate(sb):
    """A 32 kHz stream's state moved mid-stream into another batch continues bit for bit; a 16 kHz blob is refused by a 32
    kHz batch and a 32 kHz blob by a 16 kHz batch, with nothing copied."""
    f = mk.load()
    pk, flags, want = mk.packets(f, "hb40"), mk.flags_of(f, "hb40", "loss"), f["flp_hb40_loss_packet_md5"]
    assert sb.dec_state_bytes(32000) > sb.dec_state_bytes(16000) == sb.state_bytes()[1]
    a = sb.DecoderBatch(4, samplerate=32000)
    b = sb.DecoderBatch(3, samplerate=32000)
    d16 = sb.DecoderBatch(2)

    def step(batch, p):
        pcm, ret = batch.decode(*received([pk[p]] * batch.n, [flags[p]] * batch.n, CAP))
        assert (ret == 0).all()
        return pcm
    for p in range(20):
        step(a, p)
    blob = a.export_state(2)
    assert blob.size == sb.dec_state_bytes(32000)
    b.import_state(1, blob)
    before16 = d16.export_state(0)
    with pytest.raises(sb.SoloError):
        d16.import_state(0, blob)
    assert np.array_equal(d16.export_state(0), before16)
    with pytest.raises(sb.SoloError):
        b.import_state(0, before16)
    for p in range(20, 40):
        pa, pb = step(a, p), step(b, p)
        assert (mk.packet_md5(pa) == want[p]).all() and (mk.packet_md5(pb[1:2]) == want[p]).all(), p
    a.close(), b.close(), d16.close()


def test_drop_in_handles_of_both_rates_at_once(sb):
    """AGR_Sate_Decoder_Init handles of 16 and 32 kHz streams alive together (their arena segments never shared), each
    decoding its fixture: 32 kHz ones give nSamplesOut = 1280 and the reference float build's PCM (0 LSB), 16 kHz ones
    golden.npz's.  The encoder refuses 32 kHz with the reason in solo_b200_last_error()."""
    f, g = mk.load(), load_golden()
    pk32, fl32, want32 = mk.packets(f, "hb40"), mk.flags_of(f, "hb40", "mode4"), f["flp_hb40_mode4_packet_md5"]
    h32 = [sb.SoloDecoder(samplerate=32000) for _ in range(3)]
    h16 = [sb.SoloDecoder() for _ in range(2)]
    for p in range(25):
        for h in h32:
            b, nb = pk32[p]
            y, r = h.decode(b, nb, fl32[p])
            assert r == 0 and h.last_nsamples == 1280 and y.shape == (1280,)
            assert (mk.packet_md5(y[None]) == want32[p]).all(), p
        n0 = int(g["fix_nbytes"][p, 0])
        for h in h16:
            y, r = h.decode(bytes(g["fix_bits"][p, :n0]), tuple(int(v) for v in g["fix_nbytes"][p]), 4)
            assert r == 0 and h.last_nsamples == 640
            assert np.abs(y.astype(np.int32) - g["flp_pcm_mode4"][p * 640:(p + 1) * 640]).max() == 0, p
    st = np.zeros(4, np.int32)
    sb.lib().solo_b200_arena_stats(st.ctypes.data)
    assert st[2] >= 2        # at least one segment per sample rate
    for h in h32 + h16:
        h.close()
    with pytest.raises(sb.SoloError, match="32 kHz encoder"):
        sb.SoloEncoder(samplerate=32000)
    c = api.EncCtrl(2, 24000, 32000, 0, 40, 0, 0, 0)
    assert not sb.lib().solo_b200_enc_batch_create(4, C.byref(c), 0)
    assert "32 kHz encoder" in api._err()


def test_drop_in_fixed_point_arithmetic_from_environment(sb, monkeypatch):
    """SOLO_B200_DEC_ARITH=fix makes 32 kHz handles decode to the reference fixed-point build's PCM (0 LSB); 20 ms packets
    are refused in that mode, as at 16 kHz."""
    f = mk.load()
    monkeypatch.setenv("SOLO_B200_DEC_ARITH", "fix")
    for stream in ("hb40", "joint"):
        cfg = mk.STREAMS[stream][1]
        pk, fl, want = mk.packets(f, stream), mk.flags_of(f, stream, "loss"), f["fix_%s_loss_packet_md5" % stream]
        j = 1 if cfg.get("joint_hb") else 0
        h = sb.SoloDecoder(samplerate=32000, joint_enable=j, joint_mode=j)
        for p in range(len(pk)):
            b, nb = pk[p]
            pb, pnb, fl_p = receive(b, nb, fl[p])
            y, r = h.decode(pb, pnb, fl_p)
            assert r == 0 and (mk.packet_md5(y[None]) == want[p]).all(), (stream, p)
        h.close()
    with pytest.raises(sb.SoloError):
        sb.SoloDecoder(samplerate=32000, framesize_ms=20)


def test_apply_loss_device_feeds_a_32k_batch(sb):
    """Untrimmed fixture rows and per-row lostflags -> apply_loss_device -> decode_device: the fixture's lossy PCM (0 LSB)."""
    import torch
    f = mk.load()
    pk, flags, want = mk.packets(f, "hb40"), mk.flags_of(f, "hb40", "loss"), f["flp_hb40_loss_packet_md5"]
    N = 129
    db = sb.DecoderBatch(N, samplerate=32000)
    dev = DeviceDecoder(db, CAP)
    st = torch.cuda.current_stream().cuda_stream
    for p in range(40):
        b, nb = pk[p]
        fl = flags[p]
        if nb[0] <= 0:
            b, nb, fl = bytes(16), (16, 8), 1
        t_b, t_nb, t_f = (torch.from_numpy(a).cuda() for a in batch_rows([(b, nb, fl)] * N, CAP))
        sb.apply_loss_device(t_b.data_ptr(), t_nb.data_ptr(), t_f.data_ptr(), dev.tb.data_ptr(), dev.tnb.data_ptr(), CAP, N, st)
        pcm, _ = dev.decode(tf=t_f)
        assert (mk.packet_md5(pcm) == want[p]).all(), ("PCM differs (0 LSB bar)", p)
    db.close()


def test_malformed_rows_do_not_touch_their_neighbours(sb):
    """A 32 kHz batch whose odd rows get garbage, 16 kHz streams' packets (8 kHz core), lying lengths or short rows: the
    even rows decode exactly as a clean batch does (0 LSB), the bad rows report errors, and nothing faults."""
    f, g = mk.load(), load_golden()
    pk = mk.packets(f, "hb40")
    N = 200
    rng = np.random.Generator(np.random.PCG64(12))
    clean = sb.DecoderBatch(N, samplerate=32000)
    mixed = sb.DecoderBatch(N, samplerate=32000)
    bad_rows = np.arange(1, N, 2)
    errors = 0
    for p in range(30):
        tb, tnb, tf = received([pk[p]] * N, [4] * N, CAP)
        pc, rc = clean.decode(tb, tnb, tf)
        assert (rc == 0).all()
        mb, mnb, mf = tb.copy(), tnb.copy(), tf.copy()
        for s in bad_rows:
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
        assert np.array_equal(pm[0::2], pc[0::2]) and (rm[0::2] == 0).all(), p
        errors += int((rm[bad_rows] != 0).sum())
    assert errors > 0
    clean.close(), mixed.close()
