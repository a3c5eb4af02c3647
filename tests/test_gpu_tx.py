"""The send queue and the downlink contributor lists on the GPU (sb_tx_sizes / scan / pack kernels through solo_b200_tx_*,
sb_mix_contributors_kernel), at 0 tolerance against the restatements of tests/server_ref.py: random rows at N = 257 and at
N = 65 536 (a 1 024-stream sample modelled, count, offsets and byte total checked in full), both entry-point forms, a real
encode_device wave against split_packet, malformed nbytes, repeatability, the launch budget and the scalar refusals;
then a loopback on the device: encode -> pack -> a seeded network -> receive queue -> decode reproduces encode ->
apply_loss_device -> decode for the same per-packet loss."""
import numpy as np
import pytest

from tests.parity import sb  # noqa: F401  (fixture)
from tests.server_ref import (BAD, DTX, M32, OCTETS, SENT, DevicePack, HostPack, PyTx, contributors_literal, csr_rooms,
                              random_rows, select_talkers, split_row, to_dev)
from tests.util import load_clip, speech_replay

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("form", [DevicePack, HostPack])
def test_queue_equals_model_257(sb, form):
    n = 257
    rng = np.random.Generator(np.random.PCG64(257))
    q, m = form(sb, n), PyTx(n)
    for w in range(12):
        if w in (4, 9):
            st = rng.choice(n, 20, replace=False)
            start = np.where(rng.random(20) < 0.5, M32 - rng.integers(1, 4, 20), rng.integers(0, M32, 20))
            q.reset(st, start)
            m.reset(st, start)
        bits, nb = random_rows(rng, n, (128, 256, 144)[w % 3])
        assert q.pack(bits, nb) == m.pack(bits, nb), w
    assert np.array_equal(q.stats(), m.stats())
    tot = m.cnt.sum(0)
    assert tot[SENT] and tot[DTX] and tot[BAD]


@pytest.mark.parametrize("form", [DevicePack, HostPack])
def test_queue_65536(sb, form):
    """65 536 streams of random rows: the count, every offset and length, and the byte total against a vectorised
    restatement; every datagram of a 1 024-stream sample against the row-by-row restatement."""
    N, cap = 65536, 256
    rng = np.random.Generator(np.random.PCG64(65536))
    bits, nb = random_rows(rng, N, cap)
    payload, ents = form(sb, N).pack(bits, nb)
    n0, n1 = nb[:, 0].astype(np.int64), nb[:, 1].astype(np.int64)
    sent = (n0 > 0) & (n1 >= 4) & (n1 <= n0) & (n0 <= cap)
    lens = np.stack([np.where(sent, n0 - n1, 0), np.where(sent, n1, 0)], 1).ravel()
    want_len = lens[lens > 0]
    want_off = np.concatenate([[0], np.cumsum(want_len)[:-1]])
    e = np.array(ents, np.int64)
    assert len(ents) == len(want_len) and len(payload) == int(lens.sum())
    assert np.array_equal(e[:, 4], want_len) and np.array_equal(e[:, 3], want_off)
    assert np.array_equal(e[:, 0], np.repeat(np.arange(N), (lens.reshape(N, 2) > 0).sum(1)))
    sample = np.sort(rng.choice(N, 1024, replace=False))
    by_stream = {}
    for k, (s, i, d, o, ln) in enumerate(ents):
        by_stream.setdefault(s, []).append((i, d, payload[o:o + ln]))
    for s in sample:
        cls, descs = split_row(bits[s], int(nb[s, 0]), int(nb[s, 1]), cap)
        want = [(0, d, data) for d, data in enumerate(descs, 1) if data]
        assert by_stream.get(int(s), []) == want, s


def test_encoder_wave_equals_split_packet(sb):
    """Every datagram of an encode_device wave (speech replay of the clip, DTX on) is split_packet's slice of its row."""
    import torch
    N, cap = 1024, 256
    x = speech_replay(load_clip(), N, 6)
    enc = sb.EncoderBatch(N, rate=13600, dtx=1)
    q = DevicePack(sb, N)
    d_x = torch.zeros((N, 640), dtype=torch.int16, device="cuda")
    d_bits = torch.zeros((N, cap), dtype=torch.uint8, device="cuda")
    d_nb = torch.zeros((N, 2), dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    n_dtx = 0
    for p in range(6):
        d_x.copy_(torch.from_numpy(x[p]))
        enc.encode_device(d_x.data_ptr(), d_bits.data_ptr(), cap, d_nb.data_ptr(), st)
        bits, nb = d_bits.cpu().numpy(), d_nb.cpu().numpy()
        payload, ents = q.pack(bits, nb)
        got = {}
        for s, i, d, o, ln in ents:
            assert i == p
            got.setdefault(s, []).append((d, payload[o:o + ln]))
        for s in range(N):
            if nb[s, 0] <= 0:
                n_dtx += 1
                assert s not in got
                continue
            p1, p2 = sb.split_packet(bytes(bits[s, :nb[s, 0]]), tuple(nb[s]))
            assert got[s] == [(d, b) for d, b in ((1, p1), (2, p2)) if b], (p, s)
    cnt = q.stats()
    assert (cnt[:, SENT] + cnt[:, DTX] == 6).all() and (cnt[:, BAD] == 0).all() and cnt[:, OCTETS].sum() > 0
    assert cnt[:, DTX].sum() == n_dtx
    enc.close()


def test_malformed_nbytes_and_repeatability(sb):
    """Every int16 extreme in nbytes on the device gives exactly the model's output; two queues given the same calls give
    identical datagrams and counters."""
    n, cap = 300, 128
    rng = np.random.Generator(np.random.PCG64(7))
    ext = np.array([-32768, -32767, -1, 0, 1, 3, 4, 5, cap - 1, cap, cap + 1, 32767], np.int16)
    a, b, m = DevicePack(sb, n), DevicePack(sb, n), PyTx(n)
    for w in range(6):
        bits, nb = random_rows(rng, n, cap)
        sel = rng.random(n) < 0.5
        nb[sel] = rng.choice(ext, (int(sel.sum()), 2))
        ra, rb = a.pack(bits, nb), b.pack(bits, nb)
        assert ra == rb == m.pack(bits, nb), w
    assert np.array_equal(a.stats(), m.stats()) and np.array_equal(b.stats(), m.stats())


def test_launch_budget_and_refusals(sb):
    """pack: three launches; reset: one; contributors_device: one (none without rooms).  encode_device launches as many
    kernels with a queue alive as without.  Scalars out of range are refused with -1."""
    import torch
    n, cap = 64, 256
    st = torch.cuda.current_stream().cuda_stream
    enc = sb.EncoderBatch(n)
    d_x = torch.zeros((n, 640), dtype=torch.int16, device="cuda")
    d_bits = torch.zeros((n, cap + 16), dtype=torch.uint8, device="cuda")
    d_nb = torch.zeros((n, 2), dtype=torch.int16, device="cuda")

    def launches(f):
        k = sb.kernel_launches()
        f()
        torch.cuda.synchronize()
        return sb.kernel_launches() - k

    def encode():
        enc.encode_device(d_x.data_ptr(), d_bits.data_ptr(), cap, d_nb.data_ptr(), st)

    before = launches(encode)
    q = DevicePack(sb, n)
    bits, nb = random_rows(np.random.Generator(np.random.PCG64(1)), n, cap)
    assert launches(lambda: q.pack(bits, nb)) == 3
    assert launches(lambda: q.q.reset([1, 2], [5, 6])) == 1
    assert launches(encode) == before
    rs, mb = to_dev(np.array([0, 3, 4], np.int32)), to_dev(np.array([5, 9, 2, 7], np.int32))
    tk, lv = to_dev(np.array([[9, 2], [7, -1]], np.int32)), to_dev(np.arange(n, dtype=np.uint8))
    cs = torch.zeros((n, 2), dtype=torch.int32, device="cuda")
    cl = torch.zeros((n, 2), dtype=torch.uint8, device="cuda")
    args = (rs.data_ptr(), mb.data_ptr())
    tail = (tk.data_ptr(), lv.data_ptr(), n, cs.data_ptr(), cl.data_ptr(), st)
    assert launches(lambda: sb.mix_contributors_device(*args, 2, 2, *tail)) == 1
    assert cs[5].tolist() == [9, 2] and cs[9].tolist() == [2, -1] and cs[7].tolist() == [-1, -1] and cs[0].tolist() == [-1, -1]
    assert cl[9].tolist() == [2, 127] and cl[0].tolist() == [127, 127]
    assert launches(lambda: sb.mix_contributors_device(*args, 0, 2, *tail)) == 0
    for k in (0, 9):
        with pytest.raises(sb.SoloError):
            sb.mix_contributors_device(*args, 2, k, *tail)
    with pytest.raises(sb.SoloError):
        sb.mix_contributors([[0, 1], [1]], np.zeros((2, 2), np.int32), np.zeros(n, np.uint8), n)   # listed twice
    with pytest.raises(sb.SoloError):
        sb.mix_contributors([[0, n]], np.zeros((1, 2), np.int32), np.zeros(n, np.uint8), n)       # outside [0, n)
    d_pay = torch.zeros(n * cap + 16, dtype=torch.uint8, device="cuda")
    ent = q.ent + [q.ct, q.tot]

    def pack(bits_ptr, c, pay_ptr, pay_cap):
        q.q.pack_device(bits_ptr, c, d_nb.data_ptr(), pay_ptr, pay_cap, *(x.data_ptr() for x in ent), st)

    pack(d_bits.data_ptr(), cap, d_pay.data_ptr(), n * cap)             # accepted
    for bad in ((d_bits.data_ptr(), 8, d_pay.data_ptr(), n * cap),      # cap below 16
                (d_bits.data_ptr(), 24, d_pay.data_ptr(), n * cap),     # cap not a multiple of 16
                (d_bits.data_ptr(), cap, d_pay.data_ptr(), n * cap - 1),  # payload_cap below the worst case
                (d_bits.data_ptr() + 1, cap, d_pay.data_ptr(), n * cap),  # d_bits not aligned
                (d_bits.data_ptr(), cap, d_pay.data_ptr() + 4, n * cap),  # d_payload not aligned
                (d_bits.data_ptr(), 1 << 30, d_pay.data_ptr(), 1 << 40)):  # n * cap above 2^31 - 1
        with pytest.raises(sb.SoloError):
            pack(*bad)
    for streams in ([0, 0], [-1], [n]):
        with pytest.raises(sb.SoloError):
            q.q.reset(streams, [1] * len(streams))
    with pytest.raises(sb.SoloError):
        sb.TxQueue(0)
    enc.close()


def test_contributors_equal_literal_loop(sb):
    """65 536 streams in rooms of 1, 4, 256 and one of 12 000, 3 384 in no room, talkers as the mixer selects them: both
    forms against INTEGRATION.md's loop, for k = 1, 3 and 8; the device form with members outside [0, n) too."""
    import torch
    n = 65536
    rng = np.random.Generator(np.random.PCG64(6465))
    sizes = [1] * 1000 + [4] * 8192 + [256] * 64 + [12000]
    st = torch.cuda.current_stream().cuda_stream
    for k in (1, 3, 8):
        room_start, members = csr_rooms(rng, n, sizes)
        level = rng.integers(0, 256, n).astype(np.uint8)
        flags = np.where(rng.random(n) < 0.4, rng.integers(1, 16, n), 0).astype(np.uint8)
        tk = select_talkers(room_start, members, level, flags, k, n)
        want = contributors_literal(room_start, members, len(sizes), k, tk, level, n)
        got = sb.mix_contributors([members[room_start[r]:room_start[r + 1]] for r in range(len(sizes))], tk, level, n)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), k
        bad_members = members.copy()
        at = rng.choice(len(members), 50, replace=False)
        bad_members[at] = rng.choice([-1, n, -(1 << 31)], 50)
        want = contributors_literal(room_start, bad_members, len(sizes), k, tk, level, n)
        d = [to_dev(x) for x in (room_start, bad_members, tk, level)]
        cs = torch.zeros((n, k), dtype=torch.int32, device="cuda")
        cl = torch.zeros((n, k), dtype=torch.uint8, device="cuda")
        sb.mix_contributors_device(d[0].data_ptr(), d[1].data_ptr(), len(sizes), k, d[2].data_ptr(), d[3].data_ptr(), n,
                                   cs.data_ptr(), cl.data_ptr(), st)
        assert np.array_equal(cs.cpu().numpy(), want[0]) and np.array_equal(cl.cpu().numpy(), want[1]), k


def test_loopback_equals_direct_path(sb):
    """257 streams, 44 ticks of encode_device.  Each tick's wave is packed on the device; the datagrams then cross a seeded
    network (10 % dropped, 5 % duplicated, each copy delayed 0 to D ticks, 4 % of the copies D + 1 or D + 2 ticks: late,
    the arrivals of a tick shuffled) into an RxQueue, which plays packet t - D at tick t; the pulled rows are decoded.
    The direct path decodes each wave through apply_loss_device with the lostflag the network implies.  Both decoders'
    PCM must be identical, and the rx and tx counters what the process implies."""
    import torch
    N, P, D, depth, desc_cap, cap = 257, 44, 3, 8, 128, 256
    x = speech_replay(load_clip(), N, P)
    enc = sb.EncoderBatch(N, rate=13600)
    dec_a, dec_b = sb.DecoderBatch(N), sb.DecoderBatch(N)
    tx, rx = sb.TxQueue(N), sb.RxQueue(N, depth, desc_cap)
    s_ = torch.cuda.Stream()
    dev = torch.device("cuda", 0)
    d_x = torch.zeros((N, 640), dtype=torch.int16, device=dev)
    d_bits = torch.zeros((N, cap), dtype=torch.uint8, device=dev)
    d_nb = torch.zeros((N, 2), dtype=torch.int16, device=dev)
    d_pay = torch.zeros(N * cap, dtype=torch.uint8, device=dev)
    ent = [torch.zeros(2 * N, dtype=t, device=dev) for t in (torch.int32, torch.int32, torch.uint8, torch.int32, torch.int32)]
    d_ct, d_tot = torch.zeros(1, dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int64, device=dev)
    d_flag, t_bits, t_nb = (torch.zeros(N, dtype=torch.int32, device=dev), torch.zeros((N, cap), dtype=torch.uint8, device=dev),
                            torch.zeros((N, 2), dtype=torch.int16, device=dev))
    r_bits, r_nb, r_lf = (torch.zeros((N, cap), dtype=torch.uint8, device=dev), torch.zeros((N, 2), dtype=torch.int16, device=dev),
                          torch.zeros(N, dtype=torch.int32, device=dev))
    pcm_a, pcm_b = (torch.zeros((P, N, 640), dtype=torch.int16, device=dev) for _ in range(2))
    ret_a, ret_b = (torch.zeros((P, N), dtype=torch.int32, device=dev) for _ in range(2))
    rng = np.random.Generator(np.random.PCG64(2024))
    sched = {}                          # arrival tick -> [(stream, index, desc, bytes)]
    on_time = {}                        # (stream, packet, desc) -> on-time copies
    late = np.zeros(N, np.int64)
    octets = np.zeros(N, np.int64)
    keep_alive = []
    st = s_.cuda_stream
    for t in range(P + D):
        with torch.cuda.stream(s_):
            if t < P:
                d_x.copy_(torch.from_numpy(x[t]))
                enc.encode_device(d_x.data_ptr(), d_bits.data_ptr(), cap, d_nb.data_ptr(), st)
                tx.pack_device(d_bits.data_ptr(), cap, d_nb.data_ptr(), d_pay.data_ptr(), d_pay.numel(),
                               *(e.data_ptr() for e in ent), d_ct.data_ptr(), d_tot.data_ptr(), st)
        s_.synchronize()
        if t < P:                       # the network: what each datagram of packet t does
            c, tot = int(d_ct.item()), int(d_tot.item())
            pay = d_pay[:tot].cpu().numpy().tobytes()
            ss, ix, de, of, ln = (e[:c].cpu().numpy() for e in ent)
            assert (ix.view(np.uint32) == t).all()
            got = np.zeros((N, 2), bool)
            for a in range(c):
                s, d, data = int(ss[a]), int(de[a]), pay[of[a]:of[a] + ln[a]]
                octets[s] += len(data)
                for copy in range(1 + (rng.random() < 0.05)):
                    if rng.random() < 0.10:
                        continue
                    delay = int(rng.integers(D + 1, D + 3)) if rng.random() < 0.04 else int(rng.integers(0, D + 1))
                    if delay <= D:
                        on_time[(s, t, d)] = on_time.get((s, t, d), 0) + 1
                        got[s, d - 1] = True
                    elif t + delay < P + D:
                        late[s] += 1
                    sched.setdefault(t + delay, []).append((s, t, d, data))
            flag = np.where(got[:, 0] & got[:, 1], 4, np.where(got[:, 0], 2, np.where(got[:, 1], 3, 1))).astype(np.int32)
        arr = sched.pop(t, [])
        arr = [arr[i] for i in rng.permutation(len(arr))]
        lens = np.array([len(a[3]) for a in arr], np.int32)
        off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int32) if arr else np.zeros(0, np.int32)
        host = [np.array([a[0] for a in arr], np.int32), np.array([a[1] for a in arr], np.uint32).view(np.int32),
                np.array([a[2] for a in arr], np.uint8), off, lens, np.frombuffer(b"".join(a[3] for a in arr) + b"\0", np.uint8)]
        with torch.cuda.stream(s_):
            dv = [torch.from_numpy(np.array(h)).to(dev, non_blocking=False) for h in host]
            keep_alive.append(dv)
            if t < P:                   # the direct path of packet t
                d_flag.copy_(torch.from_numpy(flag))
                sb.apply_loss_device(d_bits.data_ptr(), d_nb.data_ptr(), d_flag.data_ptr(), t_bits.data_ptr(), t_nb.data_ptr(),
                                     cap, N, st)
                dec_a.decode_device(pcm_a[t].data_ptr(), t_bits.data_ptr(), cap, t_nb.data_ptr(), d_flag.data_ptr(),
                                    ret_a[t].data_ptr(), st)
            rx.insert_device(*(v.data_ptr() for v in dv[:5]), len(arr), dv[5].data_ptr(), int(lens.sum()), st)
            if t >= D:                  # the loopback path plays packet t - D
                rx.pull_device(0, r_bits.data_ptr(), cap, r_nb.data_ptr(), r_lf.data_ptr(), st)
                dec_b.decode_device(pcm_b[t - D].data_ptr(), r_bits.data_ptr(), cap, r_nb.data_ptr(), r_lf.data_ptr(),
                                    ret_b[t - D].data_ptr(), st)
    s_.synchronize()
    assert (ret_a.cpu().numpy() == 0).all() and (ret_b.cpu().numpy() == 0).all()
    assert torch.equal(pcm_a, pcm_b)
    cnt, bad = rx.stats()
    want = np.zeros((N, 8), np.int64)
    for (s, p, d), copies in on_time.items():
        want[s, 0] += 1
        want[s, 1] += copies - 1
    want[:, 2] = late
    for s in range(N):
        for p in range(P):
            h = sum((s, p, d) in on_time for d in (1, 2))
            want[s, 5 + (2 - h)] += 1
    assert bad == 0 and np.array_equal(cnt.astype(np.int64), want)
    tc = tx.stats()
    assert (tc[:, SENT] == P).all() and np.array_equal(tc[:, OCTETS].astype(np.int64), octets) and (tc[:, DTX] == 0).all()
    assert want[:, 1].sum() > 0 and want[:, 2].sum() > 0 and want[:, 6].sum() > 0 and want[:, 7].sum() > 0
    for o in (enc, dec_a, dec_b, tx, rx):
        o.close()
