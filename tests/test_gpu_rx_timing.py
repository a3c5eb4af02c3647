"""Receive-queue timing on the GPU (sb_rx_timing_keys / sort / walk kernels through solo_b200_rx_insert_timed_* and
solo_b200_rx_timing), at 0 tolerance against the host model (a timed sim.SimRx, the same sb_rx.cuh rules in array
order): seeded arrival processes at N = 257 through both entry points, the rx_time.py traffic at N = 65 536, every arrival on
one stream at n = max_arrivals, garbage arrays, repeatability, reset, and a send queue -> network -> receive queue
loopback with known delays whose jitter has a closed form.  A timed queue and an untimed one fed the same arrays must
pull the same rows and report the same counters."""
import numpy as np
import pytest

from tests.hostsim.sim import SimRx
from tests.parity import sb  # noqa: F401  (fixture)
from tests.server_ref import DeviceForm, HostForm, M32, PyRx, add_arrivals, make_ops, replay, rx_time_traffic
from tests.util import load_golden

pytestmark = pytest.mark.gpu


def check_timing(q, m):
    for got, want in zip(q.timing(), m.timing()):
        assert got.dtype == want.dtype and np.array_equal(got, want)


def timed_model(n, depth, desc_cap, ts):
    m = SimRx(n, depth, desc_cap)
    m.enable_timing(ts)
    return m


def run_pair(sb, ops, n, depth, desc_cap, ts, form, max_arrivals):
    """Replay timed ops on a timed queue, an untimed queue and the host model.  Pulls and counters of the two queues must
    agree and equal the restatement's counters, and the timed queue's timing must equal the model's after every insert.
    Returns the timed queue."""
    timed, plain = form(sb, n, depth, desc_cap), form(sb, n, depth, desc_cap)
    timed.enable_timing(ts, max_arrivals)
    q, m = PyRx(n, depth, desc_cap), timed_model(n, depth, desc_cap, ts)
    for op in ops:
        if op[0] == "insert":
            q.insert(*op[1:7])
            m.insert(*op[1:])
            timed.insert(*op[1:])
            plain.insert(*op[1:7])
            check_timing(timed, m)
        elif op[0] == "reset":
            for x in (timed, plain, q, m):
                x.reset(op[1], op[2])
            check_timing(timed, m)
        else:
            a, b = timed.pull(op[1]), plain.pull(op[1])
            q.pull(op[1])
            m.pull(op[1])
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
    ca, cb = timed.stats(), plain.stats()
    assert np.array_equal(ca[0], cb[0]) and ca[1] == cb[1]
    assert np.array_equal(ca[0].astype(np.int64), q.cnt)
    plain.close()
    return timed


@pytest.mark.parametrize("form", [DeviceForm, HostForm], ids=["insert_device", "insert_host"])
@pytest.mark.parametrize("explicit_play", [False, True])
def test_timed_queue_equals_model_257(sb, form, explicit_play):
    n, depth, desc_cap, ts = 257, 8, 128, 640
    rng = np.random.Generator(np.random.PCG64(257 + explicit_play))
    ops, _ = make_ops(rng, n, depth, desc_cap, 16, explicit_play=explicit_play)
    ops = add_arrivals(rng, ops, ts, M32 - 7000)
    q = run_pair(sb, ops, n, depth, desc_cap, ts, form, 4096)
    jitter, highest, received, margin = q.timing()
    assert (highest >> np.uint64(32)).max() >= 1 and (margin.sum(0) > 0).all() and received.sum() > 0
    q.close()


def test_host_and_device_forms_agree_and_repeat(sb):
    """The same timed calls through insert_timed_host, and twice through insert_timed_device: identical timing."""
    n, depth, desc_cap, ts = 300, 4, 64, 320
    rng = np.random.Generator(np.random.PCG64(9))
    ops, _ = make_ops(rng, n, depth, desc_cap, 8)
    ops = add_arrivals(rng, ops, ts, 5)
    res = []
    for form in (HostForm, DeviceForm, DeviceForm):
        q = form(sb, n, depth, desc_cap)
        q.enable_timing(ts, 8192)
        replay(q, ops)
        res.append(q.timing())
        q.close()
    for r in res[1:]:
        assert all(np.array_equal(x, y) for x, y in zip(r, res[0]))


def test_timed_queue_equals_model_65536(sb):
    """65 536 streams and about 132 k arrivals per tick (the rx_time.py traffic) with receive times: index * 640 plus a
    per-arrival delay, the clock wrapping during the run.  Every stream's timing is compared."""
    N, depth, desc_cap, ts = 65536, 8, 128, 640
    rng = np.random.Generator(np.random.PCG64(65536))
    s, d, lens, payload, off, early = rx_time_traffic(N, rng)
    A = len(s)
    timed, plain = DeviceForm(sb, N, depth, desc_cap), DeviceForm(sb, N, depth, desc_cap)
    timed.enable_timing(ts, A)
    m = timed_model(N, depth, desc_cap, ts)
    for t in range(4):
        index = ((t + early) % M32).astype(np.uint32)
        arrival = ((M32 - 2 * ts + index.astype(np.int64) * ts + rng.integers(0, 2 * ts, A)) % M32).astype(np.uint32)
        m.insert(s, index, d, off, lens, payload, arrival)
        timed.insert(s, index, d, off, lens, payload, arrival)
        plain.insert(s, index, d, off, lens, payload)
        check_timing(timed, m)
        a, b = timed.pull(), plain.pull()
        m.pull()
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
    ca, cb = timed.stats(), plain.stats()
    assert np.array_equal(ca[0], cb[0]) and ca[1] == cb[1]
    jitter, highest, received, margin = timed.timing()
    assert received.min() > 0 and margin[:, 0].sum() > 0 and margin[:, 1].sum() > 0


@pytest.mark.parametrize("N,target", [(65536, 40000), (257, 0), (1, 0)])
def test_all_arrivals_on_one_stream(sb, N, target):
    """n = max_arrivals arrivals, all valid and on one stream, in an order with reordering and duplicates: one group of
    the sort holds every arrival, and its walk follows array order."""
    desc_cap, ts, A = 64, 640, 140000
    rng = np.random.Generator(np.random.PCG64(N))
    q = DeviceForm(sb, N, 32, desc_cap)
    q.enable_timing(ts, A)
    m = timed_model(N, 32, desc_cap, ts)
    stream = np.full(A, target, np.int32)
    index = (np.arange(A) // 2 + rng.integers(-40, 40, A)) % M32
    index = index.astype(np.uint32)
    desc = rng.integers(1, 3, A).astype(np.uint8)
    lens = np.full(A, 4, np.int32)
    off = rng.integers(0, 60, A).astype(np.int32)
    payload = rng.integers(0, 256, 64).astype(np.uint8)
    arrival = ((index.astype(np.int64) * ts + rng.integers(0, 3000, A)) % M32).astype(np.uint32)
    m.insert(stream, index, desc, off, lens, payload, arrival)
    q.insert(stream, index, desc, off, lens, payload, arrival)
    check_timing(q, m)
    assert int(q.timing()[2][target]) == A


def test_garbage_arrays(sb):
    """Arrays of random words: out-of-range and negative streams, bad descriptions, lengths and offsets, any index and
    arrival.  The timing still equals the model, and the counters equal an untimed queue's."""
    N, depth, desc_cap, ts = 1000, 8, 32, 0x9E3779B1
    rng = np.random.Generator(np.random.PCG64(77))
    timed, plain = DeviceForm(sb, N, depth, desc_cap), DeviceForm(sb, N, depth, desc_cap)
    timed.enable_timing(ts, 50000)
    m = timed_model(N, depth, desc_cap, ts)
    for t in range(3):
        A = 50000
        w = rng.integers(0, M32, (6, A), dtype=np.uint64).astype(np.uint32)
        stream = np.where(w[0] % 3 == 0, w[0] % (N + 50), w[0]).astype(np.uint32).view(np.int32)
        stream = np.where(w[0] % 7 == 1, -(w[0] % 9).astype(np.int32) - 1, stream).astype(np.int32)
        desc = (w[1] % 4).astype(np.uint8)
        lens = np.where(w[2] % 5 == 0, w[2].view(np.int32), (w[2] % 40).astype(np.int32)).astype(np.int32)
        off = np.where(w[3] % 5 == 0, w[3].view(np.int32), (w[3] % 300).astype(np.int32)).astype(np.int32)
        index = np.where(w[4] % 2 == 0, t + w[4] % 12, w[4]).astype(np.uint32)
        arrival = w[5]
        payload = rng.integers(0, 256, 256).astype(np.uint8)
        m.insert(stream, index, desc, off, lens, payload, arrival)
        timed.insert(stream, index, desc, off, lens, payload, arrival)
        plain.insert(stream, index, desc, off, lens, payload)
        check_timing(timed, m)
        a, b = timed.pull(), plain.pull()
        m.pull()
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
    ca, cb = timed.stats(), plain.stats()
    assert np.array_equal(ca[0], cb[0]) and ca[1] == cb[1] and ca[1] > 0
    assert m.received.sum() > 0


def test_reset_clears_listed_streams_and_launches(sb):
    """A timed queue's reset clears the listed streams' timing (two launches); an untimed insert leaves timing alone; the
    device call refuses n_arrivals > max_arrivals and a queue without timing."""
    import torch
    n, desc_cap, ts = 40, 32, 640
    q = DeviceForm(sb, n, 8, desc_cap)
    k = 2 * n
    stream = np.repeat(np.arange(n, dtype=np.int32), 2)
    index = np.tile(np.array([0, 3], np.uint32), n)
    args = (stream, index, np.ones(k, np.uint8), np.zeros(k, np.int32), np.full(k, 4, np.int32),
            np.zeros(8, np.uint8))
    arrival = np.arange(k, dtype=np.uint32) * 100
    with pytest.raises(sb.SoloError):
        q.timing()
    with pytest.raises(sb.SoloError):
        q.insert(*args, arrival)
    q.enable_timing(ts, k)
    with pytest.raises(sb.SoloError):
        q.enable_timing(ts, k)
    with pytest.raises(sb.SoloError):
        q.insert(*(np.concatenate([x, x[:1]]) for x in args[:5]), args[5], np.concatenate([arrival, arrival[:1]]))
    q.insert(*args, arrival)
    before = q.timing()
    q.insert(*args)                                           # untimed: timing unchanged
    assert all(np.array_equal(x, y) for x, y in zip(q.timing(), before))
    listed = np.array([3, 17, 39], np.int32)
    l0 = sb.kernel_launches()
    q.reset(listed, np.zeros(3, np.uint32))
    assert sb.kernel_launches() - l0 == 2
    after = q.timing()
    keep = np.setdiff1d(np.arange(n), listed)
    for x, y in zip(after, before):
        assert not x[listed].any() and np.array_equal(x[keep], y[keep])
    l0 = sb.kernel_launches()
    q.insert(*args, arrival)
    assert sb.kernel_launches() - l0 == 3 + 2 + 3 * 1     # N = 40: one 8-bit digit
    torch.cuda.synchronize()
    assert int(q.timing()[1][3]) == 3 and int(q.timing()[2][3]) == 2
    q.close()


def test_loopback_jitter_has_closed_form(sb):
    """Encoder-sized rows -> send queue -> a network that delays description 1 by 0 and description 2 by k_s timestamp
    units -> timed receive queue, in arrival order.  Every |D| after a stream's first arrival is k_s, so its jitter
    climbs to the recurrence's fixed point 16 k_s - 8 and reports k_s - 1 (0 for k_s = 0); highest is the last index
    sent and received counts every datagram."""
    N, cap, ts, ticks = 64, 256, 640, 240
    g = load_golden()
    P = g["fix_nbytes"].shape[0]
    bits = np.zeros((N, cap), np.uint8)
    nb = np.zeros((N, 2), np.int16)
    for s in range(N):
        r = s % P
        bits[s, :g["fix_bits"].shape[1]] = g["fix_bits"][r][:cap]
        nb[s] = g["fix_nbytes"][r]
    k = (np.arange(N) * 37) % 300
    k[::9] = 0
    tx = sb.TxQueue(N)
    rx = HostForm(sb, N, 8, 128)
    rx.enable_timing(ts, 2 * N)
    sent = np.zeros(N, np.int64)
    for t in range(ticks):
        payload, stream, index, desc, off, lens = tx.pack(bits, nb)
        arrival = (index.astype(np.int64) * ts + 1000 + np.where(desc == 2, k[stream], 0)) % M32
        order = np.lexsort((np.arange(len(stream)), arrival))          # the network delivers in arrival order
        stream, index, desc, off, lens, arrival = (x[order] for x in (stream, index, desc, off, lens, arrival))
        rx.insert(stream, index, desc, off, lens, payload, arrival.astype(np.uint32))
        rx.pull()
        np.add.at(sent, stream, 1)
    jitter, highest, received, margin = rx.timing()
    assert np.array_equal(jitter, np.maximum(k - 1, 0).astype(np.uint32))
    assert (highest == ticks - 1).all() and np.array_equal(received.astype(np.int64), sent)
    assert np.array_equal(margin[:, 0].astype(np.int64), sent)         # every datagram arrives for the next pull
    tx.close()
    rx.close()
