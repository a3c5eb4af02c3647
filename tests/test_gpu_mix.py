"""The conference mixer on the GPU (sb_mix_select_kernel + sb_mix_kernel through solo_b200_mix_host / _device), at 0
tolerance against the numpy restatement of tests/server_ref.py: random layouts at every row length, a 65 536-stream layout,
argument checking, out-of-range members on the device path, 32 kHz rows, and a whole MCU tick (decode, activity, mix,
downlink encode) on the device against the same tick through host calls and numpy mixing."""
import numpy as np
import pytest

from tests.golden import make_golden_32k as mk
from tests.parity import DeviceDecoder, batch_packets, received, sb  # noqa: F401  (fixture)
from tests.server_ref import POISON, csr, mixed_layout, numpy_mix, to_dev
from tests.util import load_clip, loss_flags, signal_classes

pytestmark = pytest.mark.gpu
CAP = 256


def dev():
    import torch
    return torch.device("cuda", 0)


def mix_on_device(sb, pcm, level, flags, room_start, members, n_rooms, k, out_init):
    """solo_b200_mix_device on copies of the arrays; returns (out, talkers) on the host."""
    import torch
    d_in, d_out, d_lv, d_fl, d_rs, d_mb = (to_dev(a) for a in (pcm, out_init, level, flags, room_start, members))
    d_tk = torch.full((max(n_rooms, 1), k), 7777, dtype=torch.int32, device=dev())
    sb.mix_device(d_in.data_ptr(), d_out.data_ptr(), pcm.shape[1], pcm.shape[0], d_lv.data_ptr(), d_fl.data_ptr(),
                  d_rs.data_ptr(), d_mb.data_ptr(), n_rooms, k, d_tk.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return d_out.cpu().numpy(), d_tk.cpu().numpy()[:n_rooms]


def random_layout(rng, n):
    """Rooms of random sizes (some empty, one large) over a random permutation of most of the n streams."""
    perm = rng.permutation(n).astype(np.int32)
    used = int(n * 0.85)
    cuts = np.sort(rng.choice(np.arange(1, used), 60, replace=False))
    rooms = np.split(perm[:used], cuts)
    rooms.insert(3, perm[:0])
    rooms.insert(17, perm[:0])
    return rooms


@pytest.mark.parametrize("spp", (320, 640, 1280))
def test_random_layouts_host_and_device(sb, spp):
    """n = 3 000 streams, random rooms, levels, flags and rows, k = 1..8: out and talkers of both entry points equal numpy,
    rows in no room keep the poison pattern byte for byte."""
    rng = np.random.Generator(np.random.PCG64(spp))
    n = 3000
    for k in range(1, 9):
        rooms = random_layout(rng, n)
        pcm = rng.integers(-32768, 32768, (n, spp), dtype=np.int16)
        pcm[rng.random(n) < 0.2] = 32767
        level = rng.integers(0, 128, n, dtype=np.uint8)
        level[rng.random(n) < 0.3] = 20                              # ties
        flags = rng.choice(np.array([0, 1, 2, 3, 4, 8, 12], np.uint8), n)
        want, wt = numpy_mix(pcm, level, flags, rooms, k, np.full((n, spp), POISON, np.int16))
        out, t = sb.mix(pcm, level, flags, rooms, k, out=np.full((n, spp), POISON, np.int16))
        assert np.array_equal(t, wt) and np.array_equal(out, want), k
        rs, mb = csr(rooms)
        out, t = mix_on_device(sb, pcm, level, flags, rs, mb, len(rooms), k, np.full((n, spp), POISON, np.int16))
        assert np.array_equal(t, wt) and np.array_equal(out, want), k


def test_65536_streams(sb):
    """The mixed layout at spp 640, k = 3: every talker list equals numpy, and so does a sample of 1 024 rows (room
    members of every room size and streams in no room, which keep the poison pattern)."""
    import torch
    n, spp, k = 65536, 640, 3
    rng = np.random.Generator(np.random.PCG64(2))
    rooms, spare = mixed_layout(n)
    pcm = rng.integers(-20000, 20000, (n, spp), dtype=np.int16)
    level = rng.integers(0, 128, n, dtype=np.uint8)
    flags = rng.choice(np.array([0, 1, 2, 3, 12], np.uint8), n)
    rs, mb = csr(rooms)
    out, t = mix_on_device(sb, pcm, level, flags, rs, mb, len(rooms), k, np.full((n, spp), POISON, np.int16))
    # numpy: the talkers of every room, then the sampled rows
    room_of = np.full(n, -1, np.int64)
    for r, mem in enumerate(rooms):
        room_of[mem] = r
    _, wt = numpy_mix(np.zeros((n, 1), np.int16), level, flags, rooms, k, np.zeros((n, 1), np.int16))
    assert np.array_equal(t, wt)
    special = np.concatenate([rooms[0], rooms[8191], rooms[8192][:8], rooms[-1][:8], spare[:8]])
    rest = np.setdiff1d(np.arange(n), special)
    sample = np.concatenate([special, np.random.Generator(np.random.PCG64(3)).choice(rest, 1024 - len(special), replace=False)])
    for i in sample:
        r = room_of[i]
        if r < 0:
            assert (out[i] == POISON).all(), i
            continue
        js = [j for j in wt[r] if j >= 0 and j != i]
        want = np.clip(pcm[js].astype(np.int32).sum(0), -32768, 32767) if js else np.zeros(spp)
        assert np.array_equal(out[i], want.astype(np.int16)), i
    torch.cuda.empty_cache()


def call_host(sb, pcm, out, spp, n, level, flags, room_start, members, n_rooms, k, talkers):
    return sb.lib().solo_b200_mix_host(pcm.ctypes.data, out.ctypes.data, spp, n, level.ctypes.data, flags.ctypes.data,
                                       room_start.ctypes.data, members.ctypes.data, n_rooms, k, talkers.ctypes.data)


def test_host_checks_every_argument(sb):
    """Each bad argument to solo_b200_mix_host returns -1, sets the error text and leaves out and talkers untouched."""
    n, spp, k = 50, 640, 3
    rng = np.random.Generator(np.random.PCG64(4))
    pcm = rng.integers(-1000, 1000, (n, spp), dtype=np.int16)
    level, flags = np.zeros(n, np.uint8), np.full(n, 3, np.uint8)
    good_rs, good_mb = np.array([0, 3, 3, 10], np.int32), np.arange(10, dtype=np.int32)[::-1].copy()
    cases = [dict(spp=600), dict(spp=0), dict(n=0), dict(n=-1), dict(k=0), dict(k=9), dict(n_rooms=-1),
             dict(room_start=np.array([1, 3, 3, 10], np.int32)),
             dict(room_start=np.array([0, 3, 2, 10], np.int32)),
             dict(members=np.array([9, 8, 7, 6, 5, 4, 3, 2, 1, -1], np.int32)),
             dict(members=np.array([9, 8, 7, 6, 5, 4, 3, 2, 1, n], np.int32)),
             dict(members=np.array([9, 9, 7, 6, 5, 4, 3, 2, 1, 0], np.int32)),      # twice in one room
             dict(members=np.array([9, 8, 7, 6, 5, 4, 3, 2, 1, 8], np.int32))]      # in two rooms
    for c in cases:
        a = dict(spp=spp, n=n, k=k, n_rooms=3, room_start=good_rs, members=good_mb)
        a.update(c)
        out = np.full((n, spp), POISON, np.int16)
        talkers = np.full((3, 9), 55, np.int32)
        r = call_host(sb, pcm, out, a["spp"], a["n"], level, flags, a["room_start"], a["members"], a["n_rooms"], a["k"], talkers)
        assert r == -1, c
        assert sb.api._err(), c
        assert (out == POISON).all() and (talkers == 55).all(), c
    out = np.full((n, spp), POISON, np.int16)
    talkers = np.full((3, k), 55, np.int32)
    assert call_host(sb, pcm, out, spp, n, level, flags, good_rs, good_mb, 3, k, talkers) == 0
    want, wt = numpy_mix(pcm, level, flags, [good_mb[:3], good_mb[3:3], good_mb[3:10]], k, np.full((n, spp), POISON, np.int16))
    assert np.array_equal(out, want) and np.array_equal(talkers, wt)


def test_device_skips_out_of_range_members(sb):
    """Member entries outside [0, n) on the device path are neither talkers nor written; every other row is what the
    layout without them gives.  Bad scalars, misaligned or overlapping rows are refused before any launch."""
    import torch
    n, spp, k = 2000, 640, 4
    rng = np.random.Generator(np.random.PCG64(5))
    rooms = random_layout(rng, n)
    pcm = rng.integers(-15000, 15000, (n, spp), dtype=np.int16)
    level = rng.integers(0, 128, n, dtype=np.uint8)
    level[:] = np.minimum(level, 100)
    flags = rng.choice(np.array([0, 1, 3], np.uint8), n)
    bad = [np.array([-1, n, n + 7, -(2 ** 31), 2 ** 31 - 1], np.int32)[rng.permutation(5)[:rng.integers(1, 6)]] for _ in rooms]
    dirty = [rng.permutation(np.concatenate([m, b])).astype(np.int32) for m, b in zip(rooms, bad)]
    want, wt = numpy_mix(pcm, level, flags, rooms, k, np.full((n, spp), POISON, np.int16))
    rs, mb = csr(dirty)
    out, t = mix_on_device(sb, pcm, level, flags, rs, mb, len(dirty), k, np.full((n, spp), POISON, np.int16))
    assert np.array_equal(t, wt) and np.array_equal(out, want)
    k0 = sb.kernel_launches()
    x = torch.zeros((n + 1, spp), dtype=torch.int16, device=dev())
    d_rs, d_mb, d_b = to_dev(rs), to_dev(mb), torch.zeros(n, dtype=torch.uint8, device=dev())
    d_tk = torch.zeros((len(dirty), k), dtype=torch.int32, device=dev())
    args = lambda i, o, s, nn, kk: (i, o, s, nn, d_b.data_ptr(), d_b.data_ptr(), d_rs.data_ptr(), d_mb.data_ptr(),
                                    len(dirty), kk, d_tk.data_ptr())
    for a in (args(x.data_ptr(), x[1].data_ptr(), spp, n, k),              # overlapping rows
              args(x.data_ptr() + 2, x[n].data_ptr(), spp, 1, k),          # misaligned
              args(x.data_ptr(), x[n].data_ptr(), 500, 1, k),              # bad spp
              args(x.data_ptr(), x[n].data_ptr(), spp, 1, 0),              # bad k
              args(x.data_ptr(), x[n].data_ptr(), spp, 0, k)):             # bad n
        with pytest.raises(sb.SoloError):
            sb.mix_device(*a)
    assert sb.kernel_launches() == k0


def test_32khz_decoder_rows(sb):
    """A 32 kHz decoder batch (1 280-sample rows) decodes golden_32k.npz's hb40 packets under per-stream loss; its device
    rows, levels and flags go through mix_device and the result equals numpy on the same rows."""
    import torch
    pk = mk.packets(mk.load(), "hb40")
    N, T, k = 64, 12, 3
    lost = np.array([loss_flags(T, 30, seed=80 + s) for s in range(N)], np.int32)
    d = DeviceDecoder(sb.DecoderBatch(N, samplerate=32000), CAP)
    rooms = [np.arange(0, 40, 2), np.arange(1, 40, 2)[::-1], np.arange(40, 52), np.array([60])]
    rs, mb = csr(rooms)
    st = torch.cuda.current_stream().cuda_stream
    d_out = torch.full((N, 1280), POISON, dtype=torch.int16, device=dev())
    d_rs, d_mb = to_dev(rs), to_dev(mb)
    d_tk = torch.zeros((len(rooms), k), dtype=torch.int32, device=dev())
    seen = 0
    for p in range(T):
        pcm, _ = d.decode(*received([pk[p + 5]] * N, lost[:, p], CAP))
        lv, fl = d.activity()
        sb.mix_device(d.pcm.data_ptr(), d_out.data_ptr(), 1280, N, d.level.data_ptr(), d.vad.data_ptr(), d_rs.data_ptr(),
                      d_mb.data_ptr(), len(rooms), k, d_tk.data_ptr(), st)
        torch.cuda.synchronize()
        want, wt = numpy_mix(pcm, lv, fl, rooms, k, np.full((N, 1280), POISON, np.int16))
        assert np.array_equal(d_tk.cpu().numpy(), wt) and np.array_equal(d_out.cpu().numpy(), want), p
        seen += int((wt >= 0).sum())
    assert seen > 0
    d.db.close()


def test_mcu_tick_device_equals_host(sb):
    """N = 256 uplinks of the eight signal classes, 20 packets under per-stream 20 % loss.  Path 1: uplink payloads ->
    decode_device -> activity_device -> mix_device -> downlink encode_device, no PCM on the host.  Path 2: the same with
    the *_host calls and numpy mixing.  Downlink payloads and nbytes are byte-identical; each mix call adds at most two
    kernel launches."""
    import torch
    N, T, k = 256, 20, 3
    x = signal_classes(load_clip(), N, T)
    lost = np.array([loss_flags(T, 20, seed=300 + s) for s in range(N)], np.int32)
    perm = np.random.Generator(np.random.PCG64(6)).permutation(N).astype(np.int32)
    cuts = np.cumsum([1, 2, 3, 4, 5, 8, 16, 33, 64, 100])
    rooms = np.split(perm[:cuts[-1]], cuts[:-1])                  # 20 streams in no room: their downlink rows stay zero
    rs, mb = csr(rooms)
    up = sb.EncoderBatch(N, rate=13600)
    d1, d2 = sb.DecoderBatch(N), sb.DecoderBatch(N)
    e1, e2 = sb.EncoderBatch(N, rate=13600), sb.EncoderBatch(N, rate=13600)
    st = torch.cuda.current_stream().cuda_stream
    d_pcm = torch.zeros((N, 640), dtype=torch.int16, device=dev())
    d_mix = torch.zeros((N, 640), dtype=torch.int16, device=dev())
    d_lv, d_fl = (torch.zeros(N, dtype=torch.uint8, device=dev()) for _ in range(2))
    d_rs, d_mb = to_dev(rs), to_dev(mb)
    d_tk = torch.zeros((len(rooms), k), dtype=torch.int32, device=dev())
    d_bits = torch.zeros((N, CAP), dtype=torch.uint8, device=dev())
    d_nb = torch.zeros((N, 2), dtype=torch.int16, device=dev())
    h_mix = np.zeros((N, 640), np.int16)
    talked = 0
    for p in range(T):
        bits, nb = up.encode(x[p], cap=CAP)
        tb, tnb, tf = received(batch_packets(bits, nb), lost[:, p], CAP)
        # path 1
        t_b, t_nb, t_f = to_dev(tb), to_dev(tnb), to_dev(tf)
        d1.decode_device(d_pcm.data_ptr(), t_b.data_ptr(), CAP, t_nb.data_ptr(), t_f.data_ptr(), 0, st)
        d1.activity_device(d_pcm.data_ptr(), d_lv.data_ptr(), d_fl.data_ptr(), st)
        k0 = sb.kernel_launches()
        sb.mix_device(d_pcm.data_ptr(), d_mix.data_ptr(), 640, N, d_lv.data_ptr(), d_fl.data_ptr(), d_rs.data_ptr(),
                      d_mb.data_ptr(), len(rooms), k, d_tk.data_ptr(), st)
        assert sb.kernel_launches() - k0 <= 2
        e1.encode_device(d_mix.data_ptr(), d_bits.data_ptr(), CAP, d_nb.data_ptr(), st)
        # path 2
        pcm, ret = d2.decode(tb, tnb, tf)
        assert (ret == 0).all()
        lv, fl = d2.activity()
        _, wt = numpy_mix(pcm, lv, fl, rooms, k, h_mix)
        b2, n2 = e2.encode(h_mix, cap=CAP)
        torch.cuda.synchronize()
        assert np.array_equal(d_tk.cpu().numpy(), wt), p
        assert np.array_equal(d_mix.cpu().numpy(), h_mix), p
        b1, n1 = d_bits.cpu().numpy(), d_nb.cpu().numpy()
        assert np.array_equal(n1, n2), p
        for s in range(N):
            m = max(int(n2[s, 0]), 0)
            assert bytes(b1[s, :m]) == bytes(b2[s, :m]), (p, s)
        talked += int((wt >= 0).sum())
    assert talked > 0
    for o in (up, d1, d2, e1, e2):
        o.close()
