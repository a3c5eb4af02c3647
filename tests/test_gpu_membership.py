"""Stream membership on the device: reset, export_states and import_states of a list of streams (solo_b200_{enc,dec}_batch_
reset / *_states in include/solo_b200.h).

  - A reset stream is a fresh stream: from the next wave it gives exactly what a stream of a newly created batch with the
    same settings gives on the same input (payload bytes and length fields; PCM at 0 LSB, return codes, activity), and
    the reference's rows where oracle/_ref is built.  The streams that were not reset are untouched.
  - export_states writes export_state's blobs, import_states takes them, and a list of streams moved between two batches
    with different histories (on one GPU, or straight into another GPU's memory) continues bit for bit.
  - Refused calls change nothing; the calls are ordered on the caller's stream and launch what the header says.
  - A 64-participant MCU tick loop with churn: every joiner's uplink decode and downlink encode equal fresh streams'."""
import numpy as np
import pytest

from tests.golden import make_golden_32k as mk
from tests.parity import batch_rows, control_args, sb  # noqa: F401  (fixture)
from tests.util import GOLDEN, load_clip, loss_flags, receive, signal_classes, speech_replay

pytestmark = pytest.mark.gpu
N, CAP = 257, 512
ENC_CFG = {"40ms": dict(framesize_ms=40), "20ms": dict(framesize_ms=20), "joint": dict(framesize_ms=40, joint_hb=1)}
# decoder configurations: (DecoderBatch keyword arguments, arithmetics its reset entries take)
DEC_CFG = {"16k_flp": (dict(), ("flp", "fix")), "16k_fix": (dict(arith="fix"), ("flp", "fix")),
           "16k_20ms": (dict(framesize_ms=20), ("flp",)), "32k_full": (dict(samplerate=32000), ("flp", "fix")),
           "32k_core": (dict(samplerate=32000, out_samplerate=16000), ("flp", "fix"))}


def oracle():
    from oracle import ref
    return ref if ref.available() else None


def classes(n, T, spp, seed):
    """signal_classes rows cut into packets of spp samples: int16 [T, n, spp]."""
    k = 640 // spp
    x = signal_classes(load_clip(), n, (T + k - 1) // k, seed)
    return np.ascontiguousarray(x.transpose(1, 0, 2).reshape(n, -1, spp)[:, :T].transpose(1, 0, 2))


def reset_plan(n, seed, arith=None):
    """About a third of the streams in random order, with mixed settings and some entries at -1: (streams, rate, dtx,
    loss) int32 arrays, or (streams, arith) with arith drawn from -1 and the given arithmetics' codes."""
    rng = np.random.Generator(np.random.PCG64(seed))
    S = rng.permutation(n)[:n // 3].astype(np.int32)
    m = len(S)
    if arith is not None:
        return S, rng.choice([-1] + [sb_arith(a) for a in arith], m).astype(np.int32)
    rate = np.where(rng.random(m) < 0.25, -1, rng.integers(6000, 64000, m)).astype(np.int32)
    dtx = rng.integers(-1, 2, m).astype(np.int32)
    loss = np.where(rng.random(m) < 0.3, -1, rng.integers(0, 101, m)).astype(np.int32)
    return S, rate, dtx, loss


def sb_arith(a):
    return {"flp": 0, "fix": 1}[a]


def same_rows(bits_a, nb_a, bits_b, nb_b, tag):
    assert np.array_equal(nb_a, nb_b), ("nbytes",) + tag
    for i in range(len(nb_a)):
        n = max(int(nb_a[i, 0]), 0)
        assert bytes(bits_a[i, :n]) == bytes(bits_b[i, :n]), ("payload", i) + tag


def device_blobs(n, nbytes, device=0):
    import torch
    return torch.zeros((n, nbytes), dtype=torch.uint8, device=torch.device("cuda", device))


def all_states(b, nbytes):
    """Every stream's state, exported through export_states, as a host array."""
    import torch
    d = device_blobs(b.n, nbytes)
    b.export_states(np.arange(b.n), d.data_ptr())
    torch.cuda.synchronize()
    return d.cpu().numpy()


# ---- reset = fresh, encoder ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mdi", (0, 1))
@pytest.mark.parametrize("name", list(ENC_CFG))
def test_encoder_reset_equals_a_fresh_stream(sb, name, mdi):
    """257 streams of the eight signal classes (DTX on at create); after 5 packets a third of them are reset with mixed
    rate / DTX / loss (some -1).  For 10 more packets the reset rows equal a new batch created with those settings, and a
    sample the reference FIX encoder; the other rows equal a run without the reset."""
    cfg = ENC_CFG[name]
    spp, T0, T1 = 16 * cfg["framesize_ms"], 5, 10
    x = classes(N, T0 + T1, spp, seed=7 + mdi)
    kw = dict(rate=13600, dtx=1, use_md_index=mdi, **cfg)
    a, b = sb.EncoderBatch(N, **kw), sb.EncoderBatch(N, **kw)
    for p in range(T0):
        a.encode(x[p], cap=CAP)
        b.encode(x[p], cap=CAP)
    S, rate, dtx, loss = reset_plan(N, seed=11 + mdi)
    a.reset(S, rate=rate, dtx=dtx, loss=loss)
    f = sb.EncoderBatch(len(S), **kw)
    f.set_control(rate=rate, dtx=dtx, loss=loss)          # create + set_control = create with the settings
    keep = np.setdiff1d(np.arange(N), S)
    ref = oracle()
    sample = list(range(0, len(S), 9))
    refs = []
    if ref is not None:
        rk = dict(rate=13600, dtx=1, use_md_index=mdi, framesize_ms=cfg["framesize_ms"], joint_hb=cfg.get("joint_hb", 0))
        for i in sample:
            e = ref.RefEncoder("fix", **rk)
            c = control_args(rate[i], dtx[i], loss[i])
            if c:
                e.set_control(**c)
            refs.append(e)
    dtx_rows = 0
    for p in range(T0, T0 + T1):
        ba, na = a.encode(x[p], cap=CAP)
        bb, nb = b.encode(x[p], cap=CAP)
        bf, nf = f.encode(x[p][S], cap=CAP)
        same_rows(ba[S], na[S], bf, nf, (name, mdi, p, "reset"))
        same_rows(ba[keep], na[keep], bb[keep], nb[keep], (name, mdi, p, "kept"))
        dtx_rows += int((na[:, 0] <= 0).sum())
        for e, i in zip(refs, sample):
            rb, rnb, n = e.encode(x[p][S[i]])
            assert tuple(na[S[i]]) == rnb and bytes(ba[S[i], :max(n, 0)]) == rb, (name, mdi, p, int(S[i]))
    assert dtx_rows > 0
    for o in [a, b, f] + refs:
        o.close()


# ---- reset = fresh, decoder ------------------------------------------------------------------------------------------
def uplink(sb, name, n, T, seed):
    """Per stream, T (payload, (n0, n1)) packets for a decoder configuration: the batched encoder over the signal classes
    (DTX on) at 16 kHz, golden_32k.npz's hb40 stream from a per-stream starting packet at 32 kHz."""
    kw = DEC_CFG[name][0]
    if kw.get("samplerate") == 32000:
        pk = mk.packets(np.load(GOLDEN + "/golden_32k.npz"), "hb40")
        return [[pk[(7 * s + seed + p) % len(pk)] for p in range(T)] for s in range(n)]
    fs = kw.get("framesize_ms", 40)
    x = classes(n, T, 16 * fs, seed)
    e = sb.EncoderBatch(n, rate=16000, dtx=1, framesize_ms=fs)
    out = [[None] * T for _ in range(n)]
    for p in range(T):
        bits, nb = e.encode(x[p], cap=CAP)
        for s in range(n):
            out[s][p] = (bytes(bits[s, :max(int(nb[s, 0]), 0)]), (int(nb[s, 0]), int(nb[s, 1])))
    e.close()
    return out


@pytest.mark.parametrize("name", list(DEC_CFG))
def test_decoder_reset_equals_a_fresh_stream(sb, name):
    """257 streams under a 20 % loss process; at packet 4 a quarter of them get a payload of random bytes (a corrupted
    packet whose terminator can leave a stream continuing the old payload), then a third of all streams are reset with
    mixed arithmetics (some -1), some of them with loss on the first packet after the reset.  For 12 more packets the reset
    rows equal new batches of their arithmetic fed the same rows (PCM at 0 LSB, return codes, activity level and flags)
    and, for full-band rows, a sample the reference decoder; the other rows equal a run without the reset."""
    kw, ariths = DEC_CFG[name]
    T0, T1 = 5, 12
    T = T0 + T1
    pk = uplink(sb, name, N, T, seed=3)
    rng = np.random.Generator(np.random.PCG64(5))
    flags = np.array([loss_flags(T, 20, seed=1 + s) for s in range(N)], np.int32)
    S, ar = reset_plan(N, seed=13, arith=ariths)
    flags[S[::3], T0] = 1
    flags[S[1::6], T0] = 2
    corrupt = set(range(0, N, 4))
    a, b = sb.DecoderBatch(N, **kw), sb.DecoderBatch(N, **kw)
    base = {k: v for k, v in kw.items() if k != "arith"}
    create = sb_arith(kw.get("arith", "flp"))
    eff = np.where(ar == -1, create, ar)
    fresh = {k: sb.DecoderBatch(int((eff == k).sum()), arith=("flp", "fix")[k], **base) for k in set(eff.tolist())}
    ref = oracle()
    refs = {}
    if ref is not None and kw.get("out_samplerate") is None:
        rk = dict(framesize_ms=base.get("framesize_ms", 40), samplerate=base.get("samplerate", 16000))
        refs = {int(i): ref.RefDecoder(("flp", "fix")[int(eff[i])], **rk) for i in range(0, len(S), 11)}
    keep = np.setdiff1d(np.arange(N), S)
    for p in range(T):
        rx = [receive(*pk[s][p], int(flags[s, p])) for s in range(N)]
        if p == T0 - 1:
            for s in corrupt:
                ln = max(len(rx[s][0]), 20)
                rx[s] = (rng.integers(0, 256, ln).astype(np.uint8).tobytes(), (ln, min(ln, rx[s][1][1] or 8)), 4)
        tb, tnb, tf = batch_rows(rx, CAP)
        if p == T0:
            a.reset(S, arith=ar)
        pa, ra = a.decode(tb, tnb, tf)
        la, fa = a.activity()
        pb, rb = b.decode(tb, tnb, tf)
        lb, fb = b.activity()
        assert np.array_equal(pa[keep], pb[keep]) and np.array_equal(ra[keep], rb[keep]), (name, p, "kept")
        assert np.array_equal(la[keep], lb[keep]) and np.array_equal(fa[keep], fb[keep]), (name, p, "kept activity")
        if p < T0:
            continue
        for k, f in fresh.items():
            rows = S[eff == k]
            pf, rf = f.decode(tb[rows], tnb[rows], tf[rows])
            lf, ff = f.activity()
            assert np.array_equal(pa[rows], pf) and np.array_equal(ra[rows], rf), (name, p, k, "reset")
            assert np.array_equal(la[rows], lf) and np.array_equal(fa[rows], ff), (name, p, k, "reset activity")
        for i, d in refs.items():
            s = int(S[i])
            y, r = d.decode(bytes(tb[s, :tnb[s, 0]]), tuple(int(v) for v in tnb[s]), int(tf[s]))
            assert r == ra[s] == 0 and np.array_equal(y, pa[s]), (name, p, s)
    for o in [a, b] + list(fresh.values()) + list(refs.values()):
        o.close()


# ---- blobs -------------------------------------------------------------------------------------------------------------
def dec_batch(sb, name, n, device=0):
    return sb.DecoderBatch(n, device=device, **DEC_CFG[name][0])


def dec_bytes(sb, name):
    return sb.dec_state_bytes(DEC_CFG[name][0].get("samplerate", 16000))


def move_and_continue_encoder(sb, dev_a, dev_b):
    """Encoder streams of batch A (device dev_a) moved into other slots of batch B (dev_b, another history, another create
    rate) through export_states into memory of dev_b and import_states there; both continue with the same rows."""
    import torch
    n = 97
    x, y = speech_replay(load_clip(), n, 12), speech_replay(load_clip(), n, 12, first_packet=300)
    a, b = sb.EncoderBatch(n, rate=24000, device=dev_a), sb.EncoderBatch(n, rate=9000, dtx=1, device=dev_b)
    for p in range(4):
        a.encode(x[p], cap=CAP)
        b.encode(y[p], cap=CAP)
    SA = np.array([5, 96, 0, 40, 41, 17], np.int32)
    SB = np.array([3, 4, 90, 0, 50, 51], np.int32)
    nbytes = sb.state_bytes()[0]
    blobs = device_blobs(len(SA), nbytes, dev_b)
    a.export_states(SA, blobs.data_ptr())
    with torch.cuda.device(dev_b):
        torch.cuda.synchronize()
    host = blobs.cpu().numpy()
    for i, s in enumerate(SA):
        assert np.array_equal(host[i], a.export_state(int(s))), ("export_states != export_state", int(s))
    b.import_states(SB, blobs.data_ptr())
    for i, s in enumerate(SB):
        assert np.array_equal(host[i], b.export_state(int(s))), ("imported", int(s))
    for p in range(4, 12):
        yb = y[p].copy()
        yb[SB] = x[p][SA]
        ba, na = a.encode(x[p], cap=CAP)
        bb, nb = b.encode(yb, cap=CAP)
        same_rows(ba[SA], na[SA], bb[SB], nb[SB], ("encoder move", p))
    a.close(); b.close()


def move_and_continue_decoder(sb, name, dev_a, dev_b):
    import torch
    n, T = 97, 14
    pk = uplink(sb, name, n, T, seed=9)
    flags = np.array([loss_flags(T, 20, seed=50 + s) for s in range(n)], np.int32)
    a, b = dec_batch(sb, name, n, dev_a), dec_batch(sb, name, n, dev_b)
    SA = np.array([1, 2, 96, 33, 64, 10], np.int32)
    SB = np.array([95, 0, 1, 32, 7, 8], np.int32)
    for p in range(T):
        rx = [receive(*pk[s][p], int(flags[s, p])) for s in range(n)]
        ry = [receive(*pk[(s + 31) % n][(p + 3) % T], 4) for s in range(n)]   # b: another history
        if p >= 6:
            for i, s in enumerate(SB):
                ry[s] = rx[SA[i]]
        if p == 6:
            nbytes = dec_bytes(sb, name)
            blobs = device_blobs(len(SA), nbytes, dev_b)
            a.export_states(SA, blobs.data_ptr())
            with torch.cuda.device(dev_b):
                torch.cuda.synchronize()
            host = blobs.cpu().numpy()
            for i, s in enumerate(SA):
                assert np.array_equal(host[i], a.export_state(int(s))), (name, "export_states != export_state", int(s))
            b.import_states(SB, blobs.data_ptr())
            for i, s in enumerate(SB):
                assert np.array_equal(host[i], b.export_state(int(s))), (name, "imported", int(s))
        pa, ra = a.decode(*batch_rows(rx, CAP))
        pb, rb = b.decode(*batch_rows(ry, CAP))
        if p >= 6:
            assert np.array_equal(pa[SA], pb[SB]) and np.array_equal(ra[SA], rb[SB]), (name, "decoder move", p)
    a.close(); b.close()


def test_export_states_are_export_state_blobs_and_moves_continue(sb):
    """On one GPU: export_states bytes equal export_state's for every listed stream; import_states of them reads back
    the same; the moved encoder and decoder streams (every decoder kind) continue bit for bit in their new slots.  Blobs
    made by export_state go in through import_states as well."""
    import torch
    move_and_continue_encoder(sb, 0, 0)
    for name in DEC_CFG:
        move_and_continue_decoder(sb, name, 0, 0)
    # import_states of export_state's blobs, and the reverse
    a, b = sb.DecoderBatch(16, samplerate=32000), sb.DecoderBatch(16, samplerate=32000)
    pk = uplink(sb, "32k_full", 16, 3, seed=1)
    for p in range(3):
        a.decode(*batch_rows([receive(*pk[s][p], 4) for s in range(16)], CAP))
    host = np.stack([a.export_state(s) for s in (3, 4)])
    d = torch.from_numpy(host).cuda()
    b.import_states([9, 2], d.data_ptr())
    assert np.array_equal(b.export_state(9), host[0]) and np.array_equal(b.export_state(2), host[1])
    a.close(); b.close()


@pytest.mark.parametrize("kind", ["encoder"] + list(DEC_CFG))
def test_moves_straight_into_another_gpus_memory(sb, kind):
    """With two GPUs: the blobs are written by the first GPU's export straight into the second GPU's memory (peer access)
    and imported there; the moved streams continue bit for bit."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs (found %d)" % torch.cuda.device_count())
    sb.enable_peer_access(0, 1)
    if kind == "encoder":
        move_and_continue_encoder(sb, 0, 1)
    else:
        move_and_continue_decoder(sb, kind, 0, 1)


# ---- refusals ------------------------------------------------------------------------------------------------------------
def test_refused_calls_change_nothing(sb):
    """Each refused call raises SoloError and leaves every stream's state as it was (all states exported before and after):
    a stream outside [0, N), a stream listed twice, an out-of-range setting, FIX on a 20 ms batch, a 32 kHz blob of the
    other output mode (even one entry of several), a misaligned d_blobs.  n = 0 does nothing."""
    n = 40
    x = speech_replay(load_clip(), n, 3)
    e = sb.EncoderBatch(n, rate=13600)
    for p in range(3):
        e.encode(x[p], cap=CAP)
    eb = sb.state_bytes()[0]
    d20 = sb.DecoderBatch(n, framesize_ms=20)
    full, core = sb.DecoderBatch(n, samplerate=32000), sb.DecoderBatch(n, samplerate=32000, out_samplerate=16000)
    pk = uplink(sb, "32k_full", n, 3, seed=2)
    for p in range(3):
        rows = batch_rows([receive(*pk[s][p], 4) for s in range(n)], CAP)
        full.decode(*rows)
        core.decode(*rows)
    b32 = sb.dec_state_bytes(32000)
    b16 = sb.dec_state_bytes(16000)
    blobs = device_blobs(4, max(eb, b32) + 8)

    def unchanged(batch, nbytes, call):
        before = all_states(batch, nbytes)
        with pytest.raises(sb.SoloError):
            call()
        assert np.array_equal(before, all_states(batch, nbytes))

    ptr = blobs.data_ptr()
    L, minus1 = sb.lib(), np.array([-1], np.int32)      # the library's own check of a negative index (Python refuses it too)
    for batch, nbytes, call in ((e, eb, lambda: L.solo_b200_enc_batch_reset(e.h, minus1.ctypes.data, 1, None, None, None, None)),
                                (core, b32, lambda: L.solo_b200_dec_batch_import_states(core.h, minus1.ctypes.data, 1, ptr, None))):
        before = all_states(batch, nbytes)
        assert call() == -1
        assert np.array_equal(before, all_states(batch, nbytes))
    for bad in ([n], [-1], [3, 7, 3]):
        unchanged(e, eb, lambda: e.reset(bad))
        unchanged(e, eb, lambda: e.import_states(bad, ptr))
        unchanged(core, b32, lambda: core.reset(bad))
        unchanged(core, b32, lambda: core.import_states(bad, ptr))
        with pytest.raises(sb.SoloError):
            e.export_states(bad, ptr)
    for bad in (dict(rate=0), dict(dtx=2), dict(loss=101), dict(rate=[24000, -2]), dict(loss=[-1, -5])):
        unchanged(e, eb, lambda: e.reset([1, 2], **bad))
    unchanged(d20, b16, lambda: d20.reset([0, 5], arith=[-1, 1]))
    unchanged(d20, b16, lambda: d20.reset([0], arith=2))
    unchanged(e, eb, lambda: e.import_states([1], ptr + 4))
    unchanged(core, b32, lambda: core.import_states([1], ptr + 4))
    with pytest.raises(sb.SoloError):
        e.export_states([1], ptr + 4)
    # 32 kHz blobs of the other output mode: three core-output blobs and one full-band one, in either direction
    mixed = device_blobs(4, b32)
    core.export_states([0, 1, 2], mixed.data_ptr())
    full.export_states([3], mixed.data_ptr() + 3 * b32)
    unchanged(core, b32, lambda: core.import_states([5, 6, 7, 8], mixed.data_ptr()))
    unchanged(full, b32, lambda: full.import_states([5, 6, 7, 8], mixed.data_ptr()))
    unchanged(full, b32, lambda: full.import_states([9], mixed.data_ptr()))
    core.import_states([5, 6, 7], mixed.data_ptr())          # the right mode goes in
    # n = 0 launches nothing and changes nothing
    k0 = sb.kernel_launches()
    e.reset([]); e.export_states([], 0); e.import_states([], 0); core.reset([]); core.import_states([], 0)
    assert sb.kernel_launches() == k0
    for o in (e, d20, full, core):
        o.close()


# ---- ordering and launches ---------------------------------------------------------------------------------------------
def test_device_tick_on_one_stream_equals_synchronised_calls(sb):
    """decode_device -> encode_device -> reset (both batches) / export + import -> next waves, all enqueued on one
    non-default caller stream without host synchronisation, equal the same calls with a device synchronise between every
    two of them."""
    import torch
    n, T, cap = 130, 8, 256
    dev = torch.device("cuda", 0)
    x = speech_replay(load_clip(), n, T)
    pk = uplink(sb, "16k_flp", n, T, seed=4)
    rows = [batch_rows([receive(*pk[s][p], 4) for s in range(n)], cap) for p in range(T)]
    S = np.array([7, 3, 100, 64, 65], np.int32)

    def run(sync):
        st = torch.cuda.Stream()
        enc, dec = sb.EncoderBatch(n, rate=20000), sb.DecoderBatch(n)
        eb, db = sb.state_bytes()[0], sb.dec_state_bytes()
        eblob, dblob = device_blobs(2, eb), device_blobs(2, db)
        pcm = torch.zeros((n, 640), dtype=torch.int16, device=dev)
        bits, nb = torch.zeros((n, cap), dtype=torch.uint8, device=dev), torch.zeros((n, 2), dtype=torch.int16, device=dev)
        xin = torch.zeros((n, 640), dtype=torch.int16, device=dev)
        tb, tnb, tf = (torch.zeros((n, cap), dtype=torch.uint8, device=dev), torch.zeros((n, 2), dtype=torch.int16, device=dev),
                       torch.zeros(n, dtype=torch.int32, device=dev))
        ret = torch.zeros(n, dtype=torch.int32, device=dev)
        out = []

        def s():
            if sync:
                torch.cuda.synchronize()
        with torch.cuda.stream(st):
            for p in range(T):
                for buf, v in zip((tb, tnb, tf), rows[p]):
                    buf.copy_(torch.from_numpy(v), non_blocking=False)
                xin.copy_(torch.from_numpy(x[p]))
                s()
                dec.decode_device(pcm.data_ptr(), tb.data_ptr(), cap, tnb.data_ptr(), tf.data_ptr(), ret.data_ptr(), st.cuda_stream)
                s()
                enc.encode_device(xin.data_ptr(), bits.data_ptr(), cap, nb.data_ptr(), st.cuda_stream)
                s()
                if p == 3:
                    dec.reset(S, arith=[-1, 1, 0, 1, -1], stream=st.cuda_stream)
                    s()
                    enc.reset(S, rate=[-1, 8000, 30000, -1, 12000], dtx=1, stream=st.cuda_stream)
                    s()
                if p == 5:
                    enc.export_states([1, 2], eblob.data_ptr(), stream=st.cuda_stream)
                    s()
                    enc.import_states([2, 1], eblob.data_ptr(), stream=st.cuda_stream)
                    s()
                    dec.export_states([9, 10], dblob.data_ptr(), stream=st.cuda_stream)
                    s()
                    dec.import_states([11, 9], dblob.data_ptr(), stream=st.cuda_stream)
                    s()
                out.append((pcm.clone(), ret.clone(), bits.clone(), nb.clone()))
        st.synchronize()
        enc.close(); dec.close()
        return [tuple(t.cpu().numpy() for t in o) for o in out]

    a, b = run(False), run(True)
    for p, (oa, ob) in enumerate(zip(a, b)):
        for k, (u, v) in enumerate(zip(oa, ob)):
            assert np.array_equal(u, v), (p, k)


def test_launch_counts(sb):
    """A reset or an export is one launch; an import two for a 32 kHz decoder batch, one otherwise.  The packet calls
    launch what they did before these calls: eight for an encode, two for a full-band decode, one for core output."""
    import torch
    n, cap = 64, 256
    dev = torch.device("cuda", 0)
    x = torch.from_numpy(speech_replay(load_clip(), n, 1)[0]).to(dev)
    bits, nb = torch.zeros((n, cap), dtype=torch.uint8, device=dev), torch.zeros((n, 2), dtype=torch.int16, device=dev)
    flags, ret = torch.full((n,), 1, dtype=torch.int32, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)
    pcm = torch.zeros((n, 1280), dtype=torch.int16, device=dev)
    e = sb.EncoderBatch(n)
    decs = {name: dec_batch(sb, name, n) for name in DEC_CFG}
    blobs = device_blobs(4, sb.state_bytes()[0])

    def count(f):
        k0 = sb.kernel_launches()
        f()
        torch.cuda.synchronize()
        return sb.kernel_launches() - k0

    def waves():
        c = {"enc": count(lambda: e.encode_device(x.data_ptr(), bits.data_ptr(), cap, nb.data_ptr()))}
        for name, d in decs.items():
            c[name] = count(lambda: d.decode_device(pcm.data_ptr(), bits.data_ptr(), cap, nb.data_ptr(), flags.data_ptr(), ret.data_ptr()))
        return c

    before = waves()
    assert before == {"enc": 8, "16k_flp": 2, "16k_fix": 2, "16k_20ms": 2, "32k_full": 2, "32k_core": 1}, before
    L = [0, 5, 63, 9]
    assert count(lambda: e.reset(L, rate=20000)) == 1
    assert count(lambda: e.export_states(L, blobs.data_ptr())) == 1
    assert count(lambda: e.import_states(L, blobs.data_ptr())) == 1
    for name, d in decs.items():
        assert count(lambda: d.reset(L)) == 1, name
        assert count(lambda: d.export_states(L, blobs.data_ptr())) == 1, name
        assert count(lambda: d.import_states(L, blobs.data_ptr())) == (2 if name.startswith("32k") else 1), name
    assert waves() == before
    e.close()
    for d in decs.values():
        d.close()


# ---- MCU churn -----------------------------------------------------------------------------------------------------------
def test_mcu_churn_joiners_equal_fresh_streams(sb):
    """64 participants in four rooms of 16, one tick = rx insert -> pull -> decode -> activity -> mix (k = 3) -> encode
    -> tx pack, with 10 % of the uplink datagrams lost.  At ticks 5 and 10 some participants leave and new ones join their
    slots: the server resets those slots' receive queue, decoder, encoder and send queue, and each new client starts a
    fresh uplink at packet 0.  Every joiner's decoded uplink (PCM, return codes) and downlink payloads equal those of fresh
    streams fed the same rows and mix rows, and the joiner's first downlink datagram is numbered 0."""
    n, T, k, cap = 64, 16, 3, 256
    rng = np.random.Generator(np.random.PCG64(77))
    rooms = [list(range(r, n, 4)) for r in range(4)]
    cli = sb.EncoderBatch(n, rate=16000, dtx=1)        # the participants' own encoders (a joiner's is new)
    cli_tx = sb.TxQueue(n)
    rx, dec, enc, tx = sb.RxQueue(n, depth=8, desc_cap=128), sb.DecoderBatch(n), sb.EncoderBatch(n, rate=13600), sb.TxQueue(n)
    events = {5: np.array([3, 20, 41, 62, 8], np.int32), 10: np.array([20, 1, 50], np.int32)}
    offset = np.zeros(n, np.int64)                     # where each slot's current participant reads the clip
    clip = load_clip()
    joined = []                                        # (tick, slots, fresh decoder, fresh encoder)
    for t in range(T):
        if t in events:
            J = events[t]
            for s in J:
                offset[s] = 1000 + 97 * t + s
            cli.reset(J)
            cli_tx.reset(J, 0)
            rx.reset(J, np.zeros(len(J), np.int64))
            dec.reset(J)
            enc.reset(J)
            tx.reset(J, np.zeros(len(J), np.int64))
            joined.append((t, J, sb.DecoderBatch(len(J)), sb.EncoderBatch(len(J), rate=13600)))
        x = np.stack([speech_replay(clip, 1, 1, first_packet=int(offset[s]))[0, 0] for s in range(n)])
        offset += 1
        up_bits, up_nb = cli.encode(x, cap=cap)
        payload, stream, index, desc, off, lens = cli_tx.pack(up_bits, up_nb)
        keep = rng.random(len(stream)) >= 0.1
        pays = [payload[o:o + ln] for o, ln, kk in zip(off, lens, keep) if kk]
        rx.insert(stream[keep], index[keep], desc[keep], pays)
        bits, nbytes, lostflag = rx.pull(cap=cap)
        pcm, ret = dec.decode(bits, nbytes, lostflag)
        level, flags = dec.activity()
        mixed, _ = sb.mix(pcm, level, flags, rooms, k)
        down_bits, down_nb = enc.encode(mixed, cap=cap)
        _, dstream, dindex, _, _, _ = tx.pack(down_bits, down_nb)
        for t0, J, fd, fe in joined:
            fp, fr = fd.decode(bits[J], nbytes[J], lostflag[J])
            assert np.array_equal(fp, pcm[J]) and np.array_equal(fr, ret[J]), ("uplink", t0, t)
            fb, fnb = fe.encode(mixed[J], cap=cap)
            same_rows(down_bits[J], down_nb[J], fb, fnb, ("downlink", t0, t))
            if t == t0:
                for s in J:
                    assert all(int(i) == 0 for i in dindex[dstream == s]), ("first downlink index", t0, int(s))
        # slots that are rejoined at the next tick leave the earlier fresh comparison
        still = []
        for j in joined:
            if t + 1 in events and np.isin(j[1], events[t + 1]).any():
                j[2].close(); j[3].close()
            else:
                still.append(j)
        joined = still
    for _, _, fd, fe in joined:
        fd.close(); fe.close()
    for o in (cli, cli_tx, rx, dec, enc, tx):
        o.close()
