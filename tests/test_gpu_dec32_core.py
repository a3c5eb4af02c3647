"""Core output of 32 kHz streams on the GPU (solo_b200_dec_batch_create_out with out_samplerate 16000): the batched host and
device entry points, return codes, activity, launch counts and state hand-over, and a mixed 16 / 32 kHz MCU tick.  Every
row is compared exactly (0 LSB) with the low band the reference's decoders hand to their synthesis filter bank
(oracle.ref.RefDecoder with out_samplerate 16000, see tests/test_dec32_core.py)."""
import ctypes as C

import numpy as np
import pytest

from solo_b200 import api
from tests.core32 import CORE, MODE_IDS, MODES, malformed_sequence, mixed_loss, stream_of, tap  # noqa: F401  (tap: fixture)
from tests.golden import make_golden_32k as mk
from tests.parity import DeviceDecoder, batch_rows, received, ref, sb, sim  # noqa: F401  (fixtures)
from tests.server_ref import csr, to_dev
from tests.util import load_golden, receive

pytestmark = pytest.mark.gpu
CAP = 256


def dev():
    import torch
    return torch.device("cuda", 0)


def oracle_rows(ref, kind, cfg, pk, flags):
    """Low bands [T, rows, samples] of one tapped reference decoder per row of flags int32 [rows, T] over the packets pk.
    Sequential: the tap records one library-wide low band per call."""
    R, T = flags.shape
    out = np.zeros((T, R, 16 * cfg["framesize_ms"]), np.int16)
    for r in range(R):
        d = ref.RefDecoder(kind, **CORE, **cfg)
        for p in range(T):
            out[p, r], ret = d.decode(*receive(*pk[p], int(flags[r, p])))
            assert ret == 0
        d.close()
    return out


@pytest.mark.parametrize("name,cfg,kind", MODES, ids=MODE_IDS)
def test_host_and_device_calls_under_per_stream_loss(sb, ref, tap, name, cfg, kind):
    """N = 97 rows of a fixture stream, each under its own mixed loss process over lostflags 1-4, through decode_host and
    decode_device: every row of every packet equals the reference's low band (0 LSB)."""
    f = mk.load()
    pk = mk.packets(f, stream_of(cfg))
    N, T = 97, 24
    flags = np.array([mixed_loss(T, seed=500 + s) for s in range(N)], np.int32)
    want = oracle_rows(ref, kind, cfg, pk, flags)
    dh = sb.DecoderBatch(N, arith=kind, **CORE, **cfg)
    dd = sb.DecoderBatch(N, arith=kind, **CORE, **cfg)
    assert dh.samples == 16 * cfg["framesize_ms"]
    device = DeviceDecoder(dd, CAP)
    for p in range(T):
        tb, tnb, tf = received([pk[p]] * N, flags[:, p], CAP)
        pcm, ret = dh.decode(tb, tnb, tf)
        assert (ret == 0).all() and pcm.shape == (N, dh.samples), p
        assert np.array_equal(pcm, want[p]), ("host entry point differs from the reference's low band", p,
                                              int(np.argmax((pcm != want[p]).any(1))))
        assert np.array_equal(device.decode(tb, tnb, tf)[0], want[p]), ("device entry point", p)
    dh.close(), dd.close()


@pytest.mark.parametrize("arith,cfg", [("flp", dict(framesize_ms=40)), ("fix", dict(framesize_ms=40, joint_hb=1))], ids=["flp-40ms", "fix-joint"])
def test_a_65536_stream_batch(sb, ref, tap, arith, cfg):
    """One decode_device wave of 65 536 core-output streams per packet, row s under loss process s % 8; a fixed sample of
    1 024 rows (first, last and spread) equals the reference's low band of its process (0 LSB) for 20 packets."""
    import torch
    f = mk.load()
    pk = mk.packets(f, stream_of(cfg))
    N, T, K = 65536, 20, 8
    procs = np.array([mixed_loss(T, seed=900 + j) for j in range(K)], np.int32)
    want = oracle_rows(ref, arith, cfg, pk, procs)
    rows = np.unique(np.concatenate([[0, N - 1], np.random.Generator(np.random.PCG64(66)).choice(N, 1022, replace=False)]))
    db = sb.DecoderBatch(N, arith=arith, **CORE, **cfg)
    device = DeviceDecoder(db, CAP)
    proc_of = np.arange(N) % K
    d_proc = torch.from_numpy(proc_of).to(dev())
    for p in range(T):
        # the K processes' rows, gathered on the device: row s is process s % K's
        got, _ = device.decode(*(to_dev(a)[d_proc] for a in received([pk[p]] * K, procs[:, p], CAP)), rows=rows)
        assert np.array_equal(got, want[p][proc_of[rows]]), ("row differs from the reference's low band", p)
    db.close()
    del device
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name,cfg,kind", MODES, ids=MODE_IDS)
def test_return_codes_activity_and_neighbours(sb, sim, name, cfg, kind):
    """N = 120 rows whose odd rows get the damaged and other-core packets of malformed_sequence (row s starts s // 2 packets
    into it): ret equals a full-band 32 kHz batch's on every row; the even rows equal a clean core-output batch's (0 LSB);
    activity flags equal the full-band batch's, and the level is the documented formula on each accepted row (127 / 0 for
    a rejected one), through both activity entry points."""
    f, g = mk.load(), load_golden()
    stream = stream_of(cfg)
    pk = mk.packets(f, stream)
    N, T = 120, 16
    seq = malformed_sequence(f, g, stream, T + N // 2, seed=5)
    core = sb.DecoderBatch(N, arith=kind, **CORE, **cfg)
    core_dev = DeviceDecoder(sb.DecoderBatch(N, arith=kind, **CORE, **cfg), CAP)
    clean = sb.DecoderBatch(N, arith=kind, **CORE, **cfg)
    full = sb.DecoderBatch(N, arith=kind, samplerate=32000, **cfg)
    rejected = 0
    for p in range(T):
        tb, tnb, tf = batch_rows([receive(*pk[p], 4) if s % 2 == 0 else seq[p + s // 2] for s in range(N)], CAP)
        pm, rm = core.decode(tb, tnb, tf)
        pf, rf = full.decode(tb, tnb, tf)
        pc, rc = clean.decode(tb[0::2].repeat(2, 0), tnb[0::2].repeat(2, 0), tf[0::2].repeat(2, 0))
        assert np.array_equal(rm, rf), (p, np.nonzero(rm != rf)[0][:5])
        assert (rm[0::2] == 0).all() and np.array_equal(pm[0::2], pc[0::2]), p
        rejected += int((rm < 0).sum())
        lv, fl = core.activity()
        lvf, flf = full.activity()
        assert np.array_equal(fl, flf), p
        want_lv = np.array([sim.row_level(pm[s]) if rm[s] >= 0 else 127 for s in range(N)], np.uint8)
        assert np.array_equal(lv, want_lv) and (fl[rm < 0] == 0).all(), p
        pd, rd = core_dev.decode(tb, tnb, tf, check=False)
        assert np.array_equal(rd, rm) and np.array_equal(pd[rm >= 0], pm[rm >= 0]), p
        dlv, dfl = core_dev.activity()
        assert np.array_equal(dlv, lv) and np.array_equal(dfl, fl), p
    assert rejected > 0
    for o in (core, core_dev.db, clean, full):
        o.close()


def test_launch_counts(sb):
    """A core-output wave is the full 32 kHz wave less its synthesis launches: one launch per chunk instead of two.  The
    16 kHz and full-band 32 kHz batches launch what they did before (two per chunk)."""
    f = mk.load()
    N = 6400                # three chunks of at least 2048 streams each when three are asked for
    tb, tnb, tf = received([mk.packets(f, "hb40")[0]] * N, [4] * N, CAP)
    for chunks in (1, 3):
        sb.set_chunks(chunks)
        for kw, per_chunk in ((dict(samplerate=32000, out_samplerate=16000), 1), (dict(samplerate=32000), 2), (dict(), 2)):
            b = sb.DecoderBatch(N, **kw)
            k0 = sb.kernel_launches()
            b.decode(tb, tnb, tf)
            assert sb.kernel_launches() - k0 == per_chunk * chunks, (kw, chunks)
            d = DeviceDecoder(b, CAP)
            k0 = sb.kernel_launches()
            d.decode(tb, tnb, tf, check=False)         # a 16 kHz batch rejects the 32 kHz packet
            assert sb.kernel_launches() - k0 == per_chunk, kw
            b.close()
    sb.set_chunks(0)


def test_state_export_import_within_the_mode_and_refused_across(sb):
    """A core-output stream's state moved mid-stream into another core-output batch continues bit for bit; a core-output
    blob is refused by a full-band 32 kHz batch and a full-band blob by a core-output batch, with nothing copied."""
    f = mk.load()
    pk, flags = mk.packets(f, "hb40"), mk.flags_of(f, "hb40", "loss")
    a = sb.DecoderBatch(4, **CORE)
    b = sb.DecoderBatch(3, **CORE)
    full = sb.DecoderBatch(2, samplerate=32000)

    def step(batch, p):
        tb, tnb, tf = received([pk[p]] * batch.n, [flags[p]] * batch.n, CAP)
        pcm, ret = batch.decode(tb, tnb, tf)
        assert (ret == 0).all()
        return pcm
    for p in range(20):
        step(a, p), step(full, p)
    blob = a.export_state(2)
    assert blob.size == sb.dec_state_bytes(32000)
    b.import_state(1, blob)
    before_full, before_core = full.export_state(0), b.export_state(0)
    with pytest.raises(sb.SoloError, match="core-output"):
        full.import_state(0, blob)
    with pytest.raises(sb.SoloError, match="full-band"):
        b.import_state(0, before_full)
    assert np.array_equal(full.export_state(0), before_full) and np.array_equal(b.export_state(0), before_core)
    for p in range(20, 40):
        pa, pb = step(a, p), step(b, p)
        assert np.array_equal(pa[2], pb[1]), p
    a.close(), b.close(), full.close()


def test_other_output_rates_are_refused(sb):
    """out_samplerate is the stream's rate or, for 32 kHz streams, 16000: anything else is NULL with a reason."""
    for rate, out in ((16000, 32000), (32000, 8000), (32000, 24000), (16000, 8000)):
        c = api.DecCtrl(0, rate, 40, 0, 0, 0)
        assert not sb.lib().solo_b200_dec_batch_create_out(4, C.byref(c), 0, 0, out)
        assert "output rate" in api._err()
        with pytest.raises(sb.SoloError):
            sb.DecoderBatch(4, samplerate=rate, out_samplerate=out)
    c = api.DecCtrl(0, 32000, 40, 0, 0, 0)
    h = sb.lib().solo_b200_dec_batch_create_out(4, C.byref(c), 0, 0, 32000)
    assert h
    sb.lib().solo_b200_dec_batch_destroy(h)


def test_mcu_tick_with_a_mixed_room(sb, ref, tap, sim):
    """A 16 kHz batch (N16 rows, golden.npz's speech stream) and a 32 kHz core-output batch (N32 rows, the hb40 fixture
    stream) decode into one device matrix [N16 + N32][640]; each batch's activity_device writes its part of level / flags;
    mix_device mixes rooms holding rows of both; the downlink encode_device runs on the mix.  Talkers and mix rows equal
    the host model's mixer applied to the reference's rows (16 kHz: the float decoder's PCM; 32 kHz: the low band), with
    levels from those rows and flags from the host model's decoders."""
    import torch
    g, f = load_golden(), mk.load()
    pk32 = mk.packets(f, "hb40")
    T, N16, N32, k = 12, 6, 5, 3
    N = N16 + N32
    lost16 = np.array([mixed_loss(T, seed=70 + s) for s in range(N16)], np.int32)
    lost32 = np.array([mixed_loss(T, seed=80 + s) for s in range(N32)], np.int32)
    rooms = [np.array([0, 6, 1, 7], np.int32), np.array([2, 3, 8, 9, 10], np.int32), np.array([4, 5], np.int32)]
    rs, mb = csr(rooms)
    d16 = sb.DecoderBatch(N16)
    d32 = sb.DecoderBatch(N32, **CORE)
    down = sb.EncoderBatch(N, rate=13600)
    st = torch.cuda.current_stream().cuda_stream
    d_pcm = torch.zeros((N, 640), dtype=torch.int16, device=dev())
    d_mix = torch.zeros((N, 640), dtype=torch.int16, device=dev())
    d_lv, d_fl = (torch.zeros(N, dtype=torch.uint8, device=dev()) for _ in range(2))
    d_ret = torch.zeros(N, dtype=torch.int32, device=dev())
    d_rs, d_mb = to_dev(rs), to_dev(mb)
    d_tk = torch.zeros((len(rooms), k), dtype=torch.int32, device=dev())
    d_bits = torch.zeros((N, CAP), dtype=torch.uint8, device=dev())
    d_nb = torch.zeros((N, 2), dtype=torch.int16, device=dev())
    # per row: (the reference's decoder, the host model's), 16 kHz rows first, then the 32 kHz streams' core rows
    model = [(ref.RefDecoder("flp", **kw), sim.SimDecoder(**kw)) for kw in [{}] * N16 + [CORE] * N32]
    h_mix = np.zeros((N, 640), np.int16)
    talked = mixed = 0
    for p in range(T):
        n0 = int(g["fix_nbytes"][p, 0])
        p16 = (bytes(g["fix_bits"][p, :n0]), tuple(int(v) for v in g["fix_nbytes"][p]))
        rx = [receive(*p16, int(lost16[s, p])) for s in range(N16)] + [receive(*pk32[p], int(lost32[s, p])) for s in range(N32)]
        t_b, t_nb, t_f = (to_dev(a) for a in batch_rows(rx, CAP))
        d16.decode_device(d_pcm.data_ptr(), t_b.data_ptr(), CAP, t_nb.data_ptr(), t_f.data_ptr(), d_ret.data_ptr(), st)
        d32.decode_device(d_pcm[N16:].data_ptr(), t_b[N16:].data_ptr(), CAP, t_nb[N16:].data_ptr(), t_f[N16:].data_ptr(),
                          d_ret[N16:].data_ptr(), st)
        d16.activity_device(d_pcm.data_ptr(), d_lv.data_ptr(), d_fl.data_ptr(), st)
        d32.activity_device(d_pcm[N16:].data_ptr(), d_lv[N16:].data_ptr(), d_fl[N16:].data_ptr(), st)
        sb.mix_device(d_pcm.data_ptr(), d_mix.data_ptr(), 640, N, d_lv.data_ptr(), d_fl.data_ptr(), d_rs.data_ptr(),
                      d_mb.data_ptr(), len(rooms), k, d_tk.data_ptr(), st)
        down.encode_device(d_mix.data_ptr(), d_bits.data_ptr(), CAP, d_nb.data_ptr(), st)
        # the model: the reference's rows, levels from them, flags from the host model's decoders
        rows = np.zeros((N, 640), np.int16)
        flags = np.zeros(N, np.uint8)
        for s, (dr, ds) in enumerate(model):
            (y, r), (_, rs_) = dr.decode(*rx[s]), ds.decode(*rx[s])
            assert r == rs_ == 0, (p, s)
            rows[s], flags[s] = y, ds.flags
        level = np.array([sim.row_level(x) for x in rows], np.uint8)
        _, want_tk = sim.mix_model(rows, level, flags, rs, mb, k, h_mix)
        torch.cuda.synchronize()
        assert (d_ret.cpu().numpy() == 0).all(), p
        assert np.array_equal(d_pcm.cpu().numpy(), rows), p
        assert np.array_equal(d_lv.cpu().numpy(), level) and np.array_equal(d_fl.cpu().numpy(), flags), p
        assert np.array_equal(d_tk.cpu().numpy(), want_tk), p
        assert np.array_equal(d_mix.cpu().numpy(), h_mix), p
        assert (d_nb.cpu().numpy()[:, 0] > 0).any(), p
        talked += int((want_tk >= 0).sum())
        mixed += int(any(((t >= 0) & (t < N16)).any() and (t >= N16).any() for t in want_tk))
    assert talked > 0 and mixed > 0, (talked, mixed)
    for o in [o for pair in model for o in pair] + [d16, d32, down]:
        o.close()
