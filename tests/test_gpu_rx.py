"""The receive queue on the GPU (sb_rx_elect / classify / commit / pull kernels through solo_b200_rx_*), at 0 tolerance
against the restatement of tests/server_ref.py: seeded arrival processes at N = 257 and at N = 65 536 (a 1 024-stream sample
modelled), both entry-point forms, NULL and explicit play, arrival order, malformed device inputs, the launch budget, and a
whole receive -> decode run on the device that reproduces the reference decoder's PCM under golden.npz's 50 % loss."""
import numpy as np
import pytest

from tests.parity import sb  # noqa: F401  (fixture)
from tests.server_ref import DeviceForm, HostForm, M32, PyRx, check_pull, make_ops, replay, run_model, to_dev
from tests.util import load_golden

pytestmark = pytest.mark.gpu


def check_against_model(impl, ops, n, depth, desc_cap):
    """Replay ops on impl; rows (up to nbytes[0]), nbytes, lostflag and counters must equal the restatement's."""
    m, want = run_model(ops, n, depth, desc_cap)
    for got, w in zip(replay(impl, ops), want):
        check_pull(got, w)
    cnt, bad = impl.stats()
    assert np.array_equal(cnt.astype(np.int64), m.cnt) and bad == m.bad
    return m


@pytest.mark.parametrize("form", [DeviceForm, HostForm])
@pytest.mark.parametrize("explicit_play", [False, True])
def test_queue_equals_model_257(sb, form, explicit_play):
    n, depth, cap = 257, 8, 128
    rng = np.random.Generator(np.random.PCG64(11 + explicit_play))
    ops, _ = make_ops(rng, n, depth, cap, 24, explicit_play=explicit_play)
    m = check_against_model(form(sb, n, depth, cap), ops, n, depth, cap)
    assert all(m.cnt.sum(0) > 0) and m.bad > 0


@pytest.mark.parametrize("depth,desc_cap", [(2, 16), (32, 48), (4, 1024)])
def test_queue_equals_model_other_shapes(sb, depth, desc_cap):
    n = 65
    rng = np.random.Generator(np.random.PCG64(depth + desc_cap))
    ops, _ = make_ops(rng, n, depth, desc_cap, 12, explicit_play=True)
    check_against_model(DeviceForm(sb, n, depth, desc_cap), ops, n, depth, desc_cap)


def test_queue_equals_model_65536_sample(sb):
    """65 536 streams: 1 024 sampled streams run a modelled arrival process, the others receive both descriptions of every
    packet on time; the sample is compared with the model, the others with the lossless outcome."""
    N, n, depth, cap = 65536, 1024, 8, 128
    rng = np.random.Generator(np.random.PCG64(65536))
    sample = np.sort(rng.choice(N, n, replace=False)).astype(np.int32)
    other = np.setdiff1d(np.arange(N, dtype=np.int32), sample)
    ops, _ = make_ops(rng, n, depth, cap, 6, explicit_play=True)
    q = DeviceForm(sb, N, depth, cap)
    m = PyRx(n, depth, cap)
    tick = 0
    for op in ops:
        if op[0] == "reset":
            q.reset(sample[op[1]], op[2])
            m.reset(op[1], op[2])
        elif op[0] == "insert":
            stream, index, desc, off, lens, payload = op[1:]
            mapped = np.where((stream >= 0) & (stream < n), sample[np.clip(stream, 0, n - 1)], np.where(stream < 0, -1, N))
            k = len(other)
            fill = np.frombuffer(rng.bytes(2 * k * 20), np.uint8)
            q.insert(mapped.astype(np.int32), index, desc, off, lens, payload)
            q.insert(np.concatenate([other, other]), np.full(2 * k, tick, np.uint32),
                     np.concatenate([np.ones(k, np.uint8), np.full(k, 2, np.uint8)]), (20 * np.arange(2 * k)).astype(np.int32),
                     np.full(2 * k, 20, np.int32), fill)
            m.insert(*op[1:])
        else:
            play = None
            if op[1] is not None:
                play = np.full(N, tick, np.uint32)
                play[sample] = op[1]
            bits, nb, lf = q.pull(play)
            rows, wnb, wlf = m.pull(op[1])
            assert np.array_equal(nb[sample], wnb) and np.array_equal(lf[sample], wlf)
            for i, row in enumerate(rows):
                assert bytes(bits[sample[i], :len(row)]) == row, i
            assert (lf[other] == 4).all() and (nb[other] == (40, 20)).all()
            f = fill.reshape(2, k, 20)
            assert np.array_equal(bits[other, :20], f[0]) and np.array_equal(bits[other, 20:40], f[1])
            tick += 1
    cnt, bad = q.stats()
    assert np.array_equal(cnt[sample].astype(np.int64), m.cnt) and bad == m.bad
    assert (cnt[other] == [2 * tick, 0, 0, 0, 0, tick, 0, 0]).all()


def test_order_and_repeatability(sb):
    """The same arrivals in a permuted array give the model's result for that order; the same array twice, on two queues,
    gives identical rows and counters."""
    n, depth, cap = 257, 4, 64
    rng = np.random.Generator(np.random.PCG64(3))
    ops, _ = make_ops(rng, n, depth, cap, 10)
    perm_ops = []
    for op in ops:
        if op[0] == "insert":
            p = rng.permutation(len(op[1]))
            op = ("insert",) + tuple(x[p] for x in op[1:6]) + (op[6],)
        perm_ops.append(op)
    check_against_model(DeviceForm(sb, n, depth, cap), perm_ops, n, depth, cap)
    a, b = DeviceForm(sb, n, depth, cap), DeviceForm(sb, n, depth, cap)
    for op in ops:
        if op[0] == "insert":
            a.insert(*op[1:])
            b.insert(*op[1:])
        elif op[0] == "reset":
            a.reset(*op[1:])
            b.reset(*op[1:])
        else:
            ra, rb = a.pull(op[1]), b.pull(op[1])
            assert all(np.array_equal(x, y) for x, y in zip(ra, rb))
    assert all(np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y for x, y in zip(a.stats(), b.stats()))


def test_malformed_device_inputs_do_not_spread(sb):
    """Arrivals with extreme offsets, lengths, streams and desc values, mixed into a clean tick's array on the device path,
    change only the malformed / bad-stream counts: every row and every other counter is as in the clean run."""
    n, depth, cap = 257, 8, 128
    rng = np.random.Generator(np.random.PCG64(9))
    ops, _ = make_ops(rng, n, depth, cap, 8)
    clean, dirty = DeviceForm(sb, n, depth, cap), DeviceForm(sb, n, depth, cap)
    i32 = np.iinfo(np.int32)
    extra, n_bad = np.zeros(n, np.int64), 0       # the malformed arrivals each stream's counter has seen since its reset
    for op in ops:
        if op[0] == "insert":
            stream, index, desc, off, lens, payload = op[1:]
            k = 64
            bs = rng.integers(0, n, k).astype(np.int32)
            bd = rng.integers(1, 3, k).astype(np.uint8)
            bo = rng.integers(0, payload.size, k).astype(np.int32)
            bl = np.full(k, 10, np.int32)
            kind = np.arange(k) % 8
            bo[kind == 0] = i32.min
            bo[kind == 1] = i32.max
            bl[kind == 2] = i32.max
            bl[kind == 3] = i32.min
            bl[kind == 4] = -5
            bd[kind == 5] = 255
            bs[kind == 6] = i32.min
            bs[kind == 7] = i32.max
            np.add.at(extra, bs[kind < 6], 1)
            n_bad += int((kind >= 6).sum())
            at = np.sort(rng.integers(0, len(stream) + 1, k))     # the clean arrivals keep their order
            cat = lambda x, y: np.insert(x, at, y)  # noqa: E731
            clean.insert(*op[1:])
            dirty.insert(cat(stream, bs), cat(index, rng.integers(0, M32, k, dtype=np.uint32)), cat(desc, bd),
                         cat(off, bo), cat(lens, bl), payload)
        elif op[0] == "reset":
            clean.reset(*op[1:])
            dirty.reset(*op[1:])
            extra[op[1]] = 0
        else:
            a, b = clean.pull(op[1]), dirty.pull(op[1])
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
    (ca, ba), (cb, bb) = clean.stats(), dirty.stats()
    assert np.array_equal(np.delete(ca, 4, 1), np.delete(cb, 4, 1))
    assert bb - ba == n_bad and np.array_equal(cb[:, 4].astype(np.int64) - ca[:, 4], extra)


def test_launch_budget_and_existing_calls(sb):
    """insert: three launches (none for no arrivals); pull: one; reset: one.  A decode_device call launches the same number
    of kernels with a queue alive as without."""
    import torch
    n = 64
    dec = sb.DecoderBatch(n)
    g = load_golden()
    n0, n1 = (int(v) for v in g["fix_nbytes"][0])
    bits = np.zeros((n, 256), np.uint8)
    bits[:, :n0] = g["fix_bits"][0, :n0]
    d_bits, d_nb = to_dev(bits), to_dev(np.tile(np.array([n0, n1], np.int16), (n, 1)))
    d_lf, d_pcm = to_dev(np.full(n, 4, np.int32)), torch.zeros((n, 640), dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def launches(f):
        k = sb.kernel_launches()
        f()
        torch.cuda.synchronize()
        return sb.kernel_launches() - k

    before = launches(lambda: dec.decode_device(d_pcm.data_ptr(), d_bits.data_ptr(), 256, d_nb.data_ptr(), d_lf.data_ptr(), 0, st))
    q = DeviceForm(sb, n, 8, 128)
    z = np.zeros(0, np.int32)
    assert launches(lambda: q.insert(z, z.astype(np.uint32), z.astype(np.uint8), z, z, np.zeros(16, np.uint8))) == 0
    one = np.ones(1, np.int32)
    assert launches(lambda: q.insert(one, one.astype(np.uint32), one.astype(np.uint8), 0 * one, one, np.ones(4, np.uint8))) == 3
    assert launches(lambda: q.pull()) == 1
    assert launches(lambda: q.q.reset([1, 2], [5, 6])) == 1
    assert launches(lambda: dec.decode_device(d_pcm.data_ptr(), d_bits.data_ptr(), 256, d_nb.data_ptr(), d_lf.data_ptr(), 0, st)) == before
    with pytest.raises(sb.SoloError):
        q.q.pull(cap=255)                               # below 2 * desc_cap
    for streams in ([0, 0], [-1], [n]):                 # listed twice, outside [0, n)
        with pytest.raises(sb.SoloError):
            q.q.reset(streams, [1] * len(streams))
    dec.close()


def test_payload_list_insert(sb):
    """RxQueue.insert with a list of payloads and pull on the host: a packet split, sent in reverse order, merged back."""
    g = load_golden()
    n0, n1 = (int(v) for v in g["fix_nbytes"][5])
    row = bytes(g["fix_bits"][5, :n0])
    p1, p2 = sb.split_packet(row, (n0, n1))
    q = sb.RxQueue(3, depth=4, desc_cap=64)
    q.insert([1, 1, 2, 9], [0, 0, 0, 0], [2, 1, 1, 1], [p2, p1, p1, p1])
    bits, nb, lf = q.pull(cap=128)
    assert list(lf) == [1, 4, 2] and tuple(nb[1]) == (n0, n1) and bytes(bits[1, :n0]) == row
    assert bytes(bits[2, :len(p1)]) == p1 and tuple(nb[2]) == (len(p1), 0)
    cnt, bad = q.stats()
    assert bad == 1 and list(cnt[1]) == [2, 0, 0, 0, 0, 1, 0, 0] and list(cnt[0]) == [0] * 7 + [1]
    q.close()


def test_receive_then_decode_reproduces_reference_pcm(sb):
    """257 streams each split golden.npz's packets into descriptions and deliver them as loss50_flags says: shuffled per
    tick (each stream its own seed), every description 0 to D - 1 ticks early, some twice, and the descriptions the loss
    process dropped one tick after their packet played.  Every tick runs insert_device, pull_device and decode_device on
    one CUDA stream; every stream's PCM equals flp_pcm_loss50 and its counters what its delivery implies."""
    import torch
    g = load_golden()
    bits_g, nb_g, flags = g["fix_bits"], g["fix_nbytes"], [int(v) for v in g["loss50_flags"]]
    P, n, depth, desc_cap, cap = len(flags), 257, 8, 128, 256
    want_pcm = g["flp_pcm_loss50"].reshape(P, -1)
    desc_of = []
    for p in range(P):
        n0, n1 = int(nb_g[p, 0]), int(nb_g[p, 1])
        desc_of.append((bytes(bits_g[p, :n0 - n1]), bytes(bits_g[p, n0 - n1:n0])) if n0 > 0 else (b"", b""))
    sched = [[] for _ in range(P + 1)]     # tick -> [(stream, index, desc, bytes)]
    expect = np.zeros((n, 8), np.int64)
    for s in range(n):
        r = np.random.Generator(np.random.PCG64(1000 + s))
        for p in range(P):
            keep = {4: (1, 2), 2: (1,), 3: (2,), 1: ()}[flags[p]]
            for d in (1, 2):
                data = desc_of[p][d - 1]
                if not data:
                    continue
                if d in keep:
                    t = max(0, p - int(r.integers(0, depth)))
                    sched[t].append((s, p, d, data))
                    expect[s, 0] += 1
                    if r.random() < 0.1:                        # a duplicate, still before playout
                        sched[int(r.integers(t, p + 1))].append((s, p, d, data))
                        expect[s, 1] += 1
                else:
                    sched[p + 1].append((s, p, d, data))       # after its packet played
                    expect[s, 2] += p + 1 < P
            held = [d for d in (1, 2) if desc_of[p][d - 1] and d in keep]
            expect[s, 5 + (2 - len(held))] += 1
    q = sb.RxQueue(n, depth, desc_cap)
    dec = sb.DecoderBatch(n)
    st = torch.cuda.Stream()
    d_bits = torch.zeros((n, cap), dtype=torch.uint8, device="cuda")
    d_nb = torch.zeros((n, 2), dtype=torch.int16, device="cuda")
    d_lf = torch.zeros(n, dtype=torch.int32, device="cuda")
    d_pcm = torch.zeros((P, n, 640), dtype=torch.int16, device="cuda")
    d_ret = torch.zeros((P, n), dtype=torch.int32, device="cuda")
    keep_alive = []
    with torch.cuda.stream(st):
        for t in range(P):
            arr = sched[t]
            r = np.random.Generator(np.random.PCG64(t))
            arr = [arr[i] for i in r.permutation(len(arr))]
            lens = np.array([len(a[3]) for a in arr], np.int32)
            off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int32) if arr else np.zeros(0, np.int32)
            host = [np.array([a[0] for a in arr], np.int32), np.array([a[1] for a in arr], np.uint32).view(np.int32),
                    np.array([a[2] for a in arr], np.uint8), off, lens,
                    np.frombuffer(b"".join(a[3] for a in arr) + b"\0", np.uint8)]
            dv = [torch.from_numpy(np.array(x)).pin_memory().to("cuda", non_blocking=True) for x in host]
            keep_alive.append(dv)
            q.insert_device(*(x.data_ptr() for x in dv[:5]), len(arr), dv[5].data_ptr(), int(lens.sum()), st.cuda_stream)
            q.pull_device(0, d_bits.data_ptr(), cap, d_nb.data_ptr(), d_lf.data_ptr(), st.cuda_stream)
            dec.decode_device(d_pcm[t].data_ptr(), d_bits.data_ptr(), cap, d_nb.data_ptr(), d_lf.data_ptr(),
                              d_ret[t].data_ptr(), st.cuda_stream)
    st.synchronize()
    pcm, ret = d_pcm.cpu().numpy(), d_ret.cpu().numpy()
    assert (ret == 0).all()
    for s in range(n):
        assert np.array_equal(pcm[:, s], want_pcm), s
    cnt, bad = q.stats()
    assert bad == 0 and np.array_equal(cnt.astype(np.int64), expect)
    q.close()
    dec.close()
