"""32 kHz streams through the GPU decoder over the matrix the CPU lockstep covers (tests/core32.py): eight signal classes,
rates up to 100 kb/s, DTX and comfort noise, use_md_index, loss from the first packet, loss bursts and single-description
loss, payloads over 256 bytes; every row of a batch a different combination, so that the rows of a warp take different
paths.  Full-band and core output, float and fixed point, through decode_host and decode_device: every row equals the
reference's at 0 LSB (its full-band PCM, or for core output the low band it hands to its synthesis filter bank, see
tests/test_dec32_core.py), with the host model run alongside to tell a device-only fault from a model fault.

Then PCM rows off 16-byte alignment: core-output rows and encoder input rows at a 2-byte offset against aligned ones, and
full-band decoders refusing rows their 8-byte stores cannot write."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from solo_b200 import api
from tests.core32 import CORE, flags_for, mixed_loss, signals32, tap  # noqa: F401  (tap: fixture)
from tests.parity import COMPARED, DeviceDecoder, batch_rows, ref, sb, sim  # noqa: F401  (fixtures)
from tests.server_ref import to_dev
from tests.util import load_clip, receive, speech_replay

pytestmark = pytest.mark.gpu
N, CAP = 97, 512        # N odd and not a multiple of 32; CAP above the largest payload the matrix makes (about 500 bytes)
# configuration: (decoder keyword arguments, packets per stream, the rates its rows cycle through)
CONFIG = {"40ms": (dict(framesize_ms=40), 24, (15600, 24000, 40000, 64000, 100000)),
          "20ms": (dict(framesize_ms=20), 40, (15600, 24000, 64000, 100000)),
          "joint": (dict(framesize_ms=40, joint_hb=1), 24, (14800, 24000, 40000, 100000))}
ARITHS = {"40ms": ("flp", "fix"), "20ms": ("flp",), "joint": ("flp", "fix")}
CASES = [(name, mdi, kind, out) for name in CONFIG for kind in ARITHS[name] for out in ("full", "core") for mdi in (0, 1)]
LOSS = ("none", "first", "bursts", "mixed")
SPEECH = ("speech_hb", "fade")          # the classes that start at a row-dependent offset into the signal
CLASSES = [name for name, _ in signals32(1)]
WAVES = [("40ms", 1, "flp", "full"), ("joint", 1, "fix", "core")]
_WANT = {}                              # the reference rows of the WAVES cases, kept for the 65 536-row waves


def layout(name):
    """(class, rate, DTX, loss kind) of every row: class s % 8, so that neighbouring rows never share one; rate and DTX
    cycle with s // 8, so that every class meets every (rate, DTX) pair; the loss kind from a seeded generator."""
    rates = CONFIG[name][2]
    rng = np.random.Generator(np.random.PCG64(97))
    return [(s % 8, rates[(s // 8) % len(rates)], (s // 8 // len(rates)) % 2, LOSS[int(rng.integers(0, len(LOSS)))])
            for s in range(N)]


def row_flags(name):
    """lostflags int32 [N, T] of the rows' loss processes."""
    T = CONFIG[name][1]
    return np.array([mixed_loss(T, seed=300 + s) if loss == "mixed" else flags_for(loss, T, s)
                     for s, (_, _, _, loss) in enumerate(layout(name))], np.int32)


def test_layout_covers_the_matrix():
    """Every class x rate x DTX combination occurs, and every loss kind with DTX on and off; each loss kind is what it
    says (no loss, four lost packets first, a burst of at least ten, some loss) and the mixed rows of a
    configuration take all four lostflags."""
    for name, (cfg, T, rates) in CONFIG.items():
        lay, flags = layout(name), row_flags(name)
        assert {(c, r, d) for c, r, d, _ in lay} == {(c, r, d) for c in range(8) for r in rates for d in (0, 1)}, name
        assert {(d, loss) for _, _, d, loss in lay} == {(d, loss) for d in (0, 1) for loss in LOSS}, name
        for s, (_, _, _, loss) in enumerate(lay):
            f = flags[s]
            runs = np.diff(np.flatnonzero(np.diff(np.concatenate([[0], f == 1, [0]]))))[::2]
            assert {"none": (f == 4).all(), "first": (f[:4] == 1).all(), "bursts": runs.size > 0 and runs.max() >= 10,
                    "mixed": (f != 4).any()}[loss], (name, s, loss, f)
        assert set(flags[[loss == "mixed" for *_, loss in lay]].ravel()) == {1, 2, 3, 4}, name


@pytest.fixture(scope="module")
def packets(ref):
    """packets(configuration, use_md_index): per row, T (payload, (n0, n1)) packets of the reference FIX encoder at 32 kHz
    over the row's class, rate and DTX, made once for the configuration's decoder modes, one encoder per row on a thread
    pool.  The payloads fit CAP and some exceed 256 bytes."""
    made = {}

    def get(name, mdi):
        if (name, mdi) not in made:
            cfg, T, _ = CONFIG[name]
            k = 32 * cfg["framesize_ms"]
            sig = signals32(2 * T * k // 1280)      # twice what a row reads: room for the speech classes' offsets
            lay = layout(name)

            def row(s):
                c, rate, dtx, _ = lay[s]
                cls, x = sig[c]
                off = (s * 7919) % (T * k) if cls in SPEECH else 0
                e = ref.RefEncoder("fix", rate=rate, dtx=dtx, use_md_index=mdi, samplerate=32000, **cfg)
                pk = [e.encode(x[off + p * k:off + (p + 1) * k])[:2] for p in range(T)]
                e.close()
                return pk
            with ThreadPoolExecutor(32) as pool:
                pk = list(pool.map(row, range(N)))
            n0 = np.array([[nb[0] for _, nb in r] for r in pk])
            assert n0.max() <= CAP, ("a payload would be cut", name, mdi, int(n0.max()))
            assert (n0 > 256).any() and (n0 <= 0).any(), (name, mdi, "payloads over 256 bytes and DTX packets", int(n0.max()))
            made[(name, mdi)] = pk
        return made[(name, mdi)]
    return get


def decoder_args(name, mdi, kind, out):
    """The decoder keyword arguments of a case: oracle.ref.RefDecoder (arith `kind` first), sim.SimDecoder, DecoderBatch."""
    return dict(CONFIG[name][0], use_md_index=mdi, **(CORE if out == "core" else dict(samplerate=32000)))


def reference_rows(ref, sim, pk, flags, name, mdi, kind, out):
    """(reference rows, host model rows) int16 [T, N, samples] and the host model's activity flags uint8 [T, N], of one
    decoder per row over what the receiver makes of the row's packets under its lostflags.  The reference returns 0 for
    every packet.  Tapped (core output) reference decoders run one after another, the others on a thread pool."""
    kw = decoder_args(name, mdi, kind, out)
    T = CONFIG[name][1]

    def ref_row(s):
        d = ref.RefDecoder(kind, **kw)
        ys = []
        for p in range(T):
            y, r = d.decode(*receive(*pk[s][p], int(flags[s, p])))
            assert r == 0, ("reference decoder", name, mdi, kind, out, s, p, r)
            ys.append(y)
        d.close()
        return np.stack(ys)
    if out == "core":
        want = [ref_row(s) for s in range(N)]
    else:
        with ThreadPoolExecutor(32) as pool:
            want = list(pool.map(ref_row, range(N)))
    model, mflags = [], np.zeros((T, N), np.uint8)
    for s in range(N):
        d = sim.SimDecoder(arith=kind, **kw)
        ys = []
        for p in range(T):
            y, r = d.decode(*receive(*pk[s][p], int(flags[s, p])))
            assert r == 0, ("host model", name, mdi, kind, out, s, p, r)
            ys.append(y)
            mflags[p, s] = d.flags
        d.close()
        model.append(np.stack(ys))
    return np.stack(want, 1), np.stack(model, 1), mflags


@pytest.mark.parametrize("name,mdi,kind,out", CASES, ids=["%s-mdi%d-%s-%s" % c for c in CASES])
def test_heterogeneous_rows_against_the_reference(request, sb, ref, sim, packets, name, mdi, kind, out):
    """N = 97 rows, each its own class, rate, DTX and loss process, through decode_host and decode_device: every row of
    every packet equals the reference's (0 LSB); activity flags equal the host model's and levels are those of the
    reference's rows, through both activity entry points; DTX rows report received frames without voice and lost
    packets concealed frames."""
    if out == "core":
        request.getfixturevalue("tap")
    cfg, T, _ = CONFIG[name]
    lay, flags, pk = layout(name), row_flags(name), packets(name, mdi)
    want, model, mflags = reference_rows(ref, sim, pk, flags, name, mdi, kind, out)
    if (name, mdi, kind, out) in WAVES:
        _WANT[(name, mdi, kind, out)] = want
    kw = dict(decoder_args(name, mdi, kind, out), arith=kind)
    dh = sb.DecoderBatch(N, **kw)
    device = DeviceDecoder(sb.DecoderBatch(N, **kw), CAP)
    assert dh.samples == want.shape[2] == (16 if out == "core" else 32) * cfg["framesize_ms"]
    nf = cfg["framesize_ms"] // 20
    quiet = concealed = 0
    for p in range(T):
        tb, tnb, tf = batch_rows([receive(*pk[s][p], int(flags[s, p])) for s in range(N)], CAP)
        hp, hr = dh.decode(tb, tnb, tf)
        dp, dr = device.decode(tb, tnb, tf, check=False)
        assert (hr == 0).all() and (dr == 0).all(), (p, np.flatnonzero(hr)[:5], np.flatnonzero(dr)[:5])
        for entry, got in (("decode_device", dp), ("decode_host", hp)):
            bad = np.flatnonzero((got != want[p]).any(1))
            if bad.size:
                s = int(bad[0])
                c, rate, dtx, loss = lay[s]
                pytest.fail("%s: row %d (%s, %d b/s, DTX %d, loss %s) packet %d (lostflag %d) differs from the reference "
                            "by up to %d LSB; the host model %s the reference" % (
                                entry, s, CLASSES[c], rate, dtx, loss, p, tf[s],
                                int(np.abs(got[s].astype(int) - want[p, s]).max()),
                                "agrees with" if np.array_equal(model[p, s], want[p, s]) else "differs from"))
        assert np.array_equal(model[p], want[p]), ("host model differs from the reference", p)
        COMPARED["pcm"] += 2 * N
        want_lv = np.array([sim.row_level(y) for y in want[p]], np.uint8)
        for entry, (lv, fl) in (("activity", dh.activity()), ("activity_device", device.activity())):
            assert np.array_equal(fl, mflags[p]), (entry, p, np.flatnonzero(fl != mflags[p])[:5])
            assert np.array_equal(lv, want_lv), (entry, p, np.flatnonzero(lv != want_lv)[:5])
        for s in range(N):
            f = int(mflags[p, s])
            if tf[s] != 1 and lay[s][2]:
                quiet += sum(not f & (1 << j) for j in range(nf))          # a received frame coded without voice
            if tf[s] == 1:
                assert all(f & (4 << j) for j in range(nf)), (p, s, f)
                concealed += 1
    assert quiet > 0 and concealed > 0, (quiet, concealed)
    dh.close(), device.db.close()


@pytest.mark.parametrize("name,mdi,kind,out", WAVES, ids=["%s-mdi%d-%s-%s" % c for c in WAVES])
def test_a_65536_row_wave(request, sb, ref, sim, packets, name, mdi, kind, out):
    """The 97 rows of a matrix case gathered on the device into one decode_device wave of 65 536 rows (row s is row
    s % 97's); a fixed sample of 1 024 rows (first, last and spread) equals the reference's rows for 20 packets."""
    if out == "core":
        request.getfixturevalue("tap")
    import torch
    flags, pk = row_flags(name), packets(name, mdi)
    want = _WANT.get((name, mdi, kind, out))
    if want is None:
        want = reference_rows(ref, sim, pk, flags, name, mdi, kind, out)[0]
    M = 65536
    rows = np.unique(np.concatenate([[0, M - 1], np.random.Generator(np.random.PCG64(67)).choice(M, 1022, replace=False)]))
    db = sb.DecoderBatch(M, arith=kind, **decoder_args(name, mdi, kind, out))
    device = DeviceDecoder(db, CAP)
    src = torch.from_numpy(np.arange(M) % N).to(device.pcm.device)
    for p in range(20):
        rx = batch_rows([receive(*pk[s][p], int(flags[s, p])) for s in range(N)], CAP)
        got, _ = device.decode(*(to_dev(a)[src] for a in rx), rows=rows)
        bad = np.flatnonzero((got != want[p][rows % N]).any(1))
        assert bad.size == 0, ("row differs from the reference's", p, int(rows[bad[0]]))
        COMPARED["pcm"] += len(rows)
    db.close()
    del device
    torch.cuda.empty_cache()


def offset_rows(torch, n, samples, offset_bytes, canary):
    """An int16 [n, samples] view whose first row starts offset_bytes past a 16-byte boundary, inside a buffer filled with
    `canary` that has 16 bytes or more of it on each side; returns (buffer, view, start index)."""
    buf = torch.full((n * samples + 32,), canary, dtype=torch.int16, device=torch.device("cuda", 0))
    assert buf.data_ptr() % 16 == 0
    a = 8 + offset_bytes // 2
    view = buf[a:a + n * samples].view(n, samples)
    assert view.data_ptr() % 16 == offset_bytes
    return buf, view, a


def test_core_rows_off_16_byte_alignment(sb, ref, packets):
    """A core-output batch decoding into rows that start 2 bytes past a 16-byte boundary (the row store's scalar path)
    gives the rows of an aligned batch fed the same packets (0 LSB), writes nothing outside its rows, and activity_device
    on the offset rows (the activity kernel's 2-byte loads) reports what it reports on the aligned ones."""
    import torch
    name, mdi, kind, out = "joint", 1, "fix", "core"
    flags, pk = row_flags(name), packets(name, mdi)
    kw = dict(decoder_args(name, mdi, kind, out), arith=kind)
    aligned = DeviceDecoder(sb.DecoderBatch(N, **kw), CAP)
    S = aligned.db.samples
    canary = 0x5A5A
    buf, view, a = offset_rows(torch, N, S, 2, canary)
    offset = DeviceDecoder(sb.DecoderBatch(N, **kw), CAP, pcm=view)
    for p in range(8):
        rx = batch_rows([receive(*pk[s][p], int(flags[s, p])) for s in range(N)], CAP)
        pa, _ = aligned.decode(*rx)
        po, _ = offset.decode(*rx)
        assert np.array_equal(po, pa), (p, np.flatnonzero((po != pa).any(1))[:5])
        assert (pa != 0).any(), p
        COMPARED["pcm"] += N
        b = buf.cpu().numpy()
        assert (b[:a] == canary).all() and (b[a + N * S:] == canary).all(), p
        la, fa = aligned.activity()
        lo, fo = offset.activity()
        assert np.array_equal(lo, la) and np.array_equal(fo, fa), p
    aligned.db.close(), offset.db.close()


def test_encoder_rows_off_16_byte_alignment(sb):
    """encode_device of a 16 kHz batch (N = 97 speech-replay rows) from input rows 2 bytes past a 16-byte boundary (the
    band-split kernel's plain loads instead of the bulk copy): payloads and length fields byte-identical to an aligned
    batch's, and activity_device on those rows reports what it reports on the aligned ones."""
    import torch
    T = 6
    x = speech_replay(load_clip(), N, T)
    dev = torch.device("cuda", 0)
    st = torch.cuda.current_stream()
    ea, eo = sb.EncoderBatch(N), sb.EncoderBatch(N)
    xa = torch.zeros((N, 640), dtype=torch.int16, device=dev)
    _, xo, _ = offset_rows(torch, N, 640, 2, 0)
    bits = [torch.zeros((N, 256), dtype=torch.uint8, device=dev) for _ in range(2)]
    nb = [torch.zeros((N, 2), dtype=torch.int16, device=dev) for _ in range(2)]
    act = [[torch.zeros(N, dtype=torch.uint8, device=dev) for _ in range(2)] for _ in range(2)]
    for p in range(T):
        for i, (e, xi) in enumerate(((ea, xa), (eo, xo))):
            xi.copy_(torch.from_numpy(x[p]))
            e.encode_device(xi.data_ptr(), bits[i].data_ptr(), 256, nb[i].data_ptr(), st.cuda_stream)
            e.activity_device(xi.data_ptr(), act[i][0].data_ptr(), act[i][1].data_ptr(), st.cuda_stream)
        st.synchronize()
        assert torch.equal(nb[0], nb[1]) and torch.equal(bits[0], bits[1]), (p, "payloads")
        assert (nb[0][:, 0] > 0).all(), p
        assert torch.equal(act[0][0], act[1][0]) and torch.equal(act[0][1], act[1][1]), (p, "activity")
        COMPARED["payload"] += N
    ea.close(), eo.close()


@pytest.mark.parametrize("kw,refused", [(dict(), (2, 4, 6, 1)), (dict(samplerate=32000), (2, 4, 6, 1)), (CORE, (1,))],
                         ids=["16k", "32k-full", "32k-core"])
def test_decode_device_refuses_misaligned_rows(sb, kw, refused):
    """decode_device returns -1 before any launch, naming the alignment, when d_pcm is not 8-byte aligned for a full-band
    batch (16 kHz, or 32 kHz at its own rate) or not 2-byte aligned for a core-output one; the rows and return codes are
    untouched.  At the alignment the batch needs, the same call decodes (a lost packet on every row)."""
    import torch
    db = sb.DecoderBatch(N, **kw)
    need = 2 if db.samplerate != db.out_samplerate else 8
    canary = 0x5A5A
    buf = torch.full((N * db.samples + 32,), canary, dtype=torch.int16, device=torch.device("cuda", 0))
    device = DeviceDecoder(db, CAP)
    device.decode(tnb=np.array([[16, 8]] * N, np.int16), tf=np.ones(N, np.int32), rows=[])     # lost packets in place
    device.ret.fill_(-99)
    st = torch.cuda.current_stream().cuda_stream
    for off in refused:
        k0 = sb.kernel_launches()
        r = sb.lib().solo_b200_dec_batch_decode_device(db.h, buf.data_ptr() + 16 + off, device.tb.data_ptr(), CAP,
                                                       device.tnb.data_ptr(), device.flags.data_ptr(), device.ret.data_ptr(), st)
        assert r == -1 and "%d-byte aligned" % need in api._err(), (off, r, api._err())
        assert sb.kernel_launches() == k0, off
    torch.cuda.synchronize()
    assert (buf.cpu().numpy() == canary).all() and (device.ret.cpu().numpy() == -99).all()
    view = buf[8 + need // 2:8 + need // 2 + N * db.samples].view(N, db.samples)
    assert view.data_ptr() % 16 == need
    pcm, ret = DeviceDecoder(db, CAP, pcm=view).decode(device.tb, device.tnb, device.flags)
    assert (ret == 0).all()
    db.close()
