"""Receive-queue timing on the CPU: the host model (tests/hostsim/server.cpp's rx_model_timing, the kernels' per-arrival
rules of sb_rx.cuh compiled by g++, in a timed sim.SimRx) against a direct statement of RFC 3550 A.1 / A.8 and of the
margin rule in include/solo_b200.h (tests/server_ref.PyTiming), on seeded arrival processes and on cases with a known
answer.  The model's pulls and counters are checked against PyRx on the way.

The processes are tests/server_ref.make_ops's (reordering, duplicates, late arrivals, ring overrun, malformed entries,
streams out of range, resets, index wrap across 2^32) with receive times added: a network delay per arrival, a receiver
clock that wraps at 2^32, and transit jumps of 2^31."""
import numpy as np
import pytest

from tests.parity import sim  # noqa: F401  (fixture)
from tests.server_ref import M32, PyRx, PyTiming, add_arrivals, check_pull, make_ops


def same(model, py):
    return all(np.array_equal(x, y) for x, y in zip(model.timing(), py.read()))


def replay(sim, ops, n, depth, desc_cap, ts):
    """Apply the timed ops to the host model of a timed queue and to the restatements: PyRx, whose `last` feeds PyTiming.
    The timing must agree after every insert and reset, the pulls and counters of the two queues throughout.  Returns
    (model, timing restatement)."""
    h, q, py = sim.SimRx(n, depth, desc_cap), PyRx(n, depth, desc_cap), PyTiming(n, desc_cap, ts)
    h.enable_timing(ts)
    for op in ops:
        if op[0] == "insert":
            stream, index, desc, off, lens, payload, arrival = op[1:]
            py.insert(np.array(q.last, np.uint32), stream, index, desc, off, lens, arrival, len(payload))
            q.insert(*op[1:7])
            h.insert(*op[1:])
            assert same(h, py)
        elif op[0] == "reset":
            for x in (h, q):
                x.reset(op[1], op[2])
            py.reset(op[1])
            assert same(h, py)
        else:
            check_pull(h.pull(op[1]), q.pull(op[1]))
    cnt, bad = h.stats()
    assert np.array_equal(cnt.astype(np.int64), q.cnt) and bad == q.bad
    return h, py


@pytest.mark.parametrize("depth,desc_cap,ts,explicit_play", [(8, 128, 640, False), (8, 128, 640, True),
                                                             (2, 16, 320, True), (32, 64, 0x9E3779B1, False)])
def test_model_equals_rfc_statement(sim, depth, desc_cap, ts, explicit_play):
    rng = np.random.Generator(np.random.PCG64(depth * 7919 + desc_cap + explicit_play))
    n = 37
    ops, _ = make_ops(rng, n, depth, desc_cap, 30, explicit_play=explicit_play)
    ops = add_arrivals(rng, ops, ts, M32 - 5000)         # the receiver's clock wraps early on
    _, py = replay(sim, ops, n, depth, desc_cap, ts)
    jitter, highest, received, margin = py.read()
    # the process reached what it is meant to cover: index wrap (a cycle), transit jumps (jitter past 2^27 units),
    # every margin bin, and resets between calls
    assert (highest >> np.uint64(32)).max() >= 1
    assert jitter.max() > (1 << 27)
    assert (margin.sum(0)[:min(depth + 2, 8)] > 0).all()     # indices reach depth + 2 ahead
    assert any(op[0] == "reset" for op in ops)


def test_model_step_by_step(sim):
    """The state after every insert, not only at the end, in the given and in permuted array orders."""
    rng = np.random.Generator(np.random.PCG64(3))
    n, depth, desc_cap, ts = 9, 4, 32, 640
    ops, _ = make_ops(rng, n, depth, desc_cap, 12)
    for trial in range(3):
        if trial:
            perm = []
            for op in ops:
                if op[0] == "insert":
                    p = rng.permutation(len(op[1]))
                    op = ("insert",) + tuple(x[p] for x in op[1:6]) + (op[6],)
                perm.append(op)
            ops = perm
        replay(sim, add_arrivals(rng, ops, ts, 12345), n, depth, desc_cap, ts)


def run_stream(sim, ts, sends):
    """One stream: per tick, (index, arrival) pairs in arrival order, then a pull.  Returns (model, restatement)."""
    pay = np.zeros(64, np.uint8)
    ops = []
    for tick in sends:
        if tick:
            idx = np.array([p for p, _ in tick], np.uint32)
            arr = np.array([a % M32 for _, a in tick], np.uint32)
            k = len(tick)
            ops.append(("insert", np.zeros(k, np.int32), idx, np.ones(k, np.uint8), np.zeros(k, np.int32),
                        np.full(k, 8, np.int32), pay, arr))
        ops.append(("pull", None))
    return replay(sim, ops, 1, 32, 64, ts)


@pytest.mark.parametrize("delay", [0, 17, 5000, M32 - 3])
def test_constant_delay_gives_zero_jitter(sim, delay):
    ts = 640
    sends = [[(t, t * ts + delay + 123456789)] for t in range(50)]
    h, _ = run_stream(sim, ts, sends)
    jitter, highest, received, margin = h.timing()
    assert int(jitter[0]) == 0 and int(h.jitter[0]) == 0 and int(received[0]) == 50 and int(highest[0]) == 49


@pytest.mark.parametrize("k", [1, 2, 40, 640, 100000])
def test_alternating_delay_converges_to_fixed_point(sim, k):
    """Delays 0, k, 0, k, ...: |D| = k for every packet after the first, and J += k - ((J + 8) >> 4) climbs to the
    recurrence's fixed point 16k - 8 (the smallest J with (J + 8) >> 4 = k) and stays; reported, (16k - 8) >> 4 = k - 1."""
    ts = 640
    sends = [[(t, t * ts + (k if t % 2 else 0))] for t in range(16 * 200)]
    h, _ = run_stream(sim, ts, sends)
    assert int(h.jitter[0]) == 16 * k - 8
    assert int(h.timing()[0][0]) == k - 1


@pytest.mark.parametrize("m", [0, 1, 3, 7, 12])
def test_margin_of_packets_m_ticks_early(sim, m):
    """Packet t + m + 1 arrives at tick t, before the pull that plays t + 1: every arrival is m pulls early, so the
    histogram is all in bin min(m, 7)."""
    ts = 640
    sends = [[(t + m, (t + m) * ts - m * ts)] for t in range(30)]
    h, _ = run_stream(sim, ts, sends)
    margin = h.timing()[3][0]
    assert int(margin[min(m, 7)]) == 30 and int(margin.sum()) == 30


def test_highest_across_wrap_and_reset(sim):
    """highest counts a cycle when the index wraps past 2^32, ignores older indices, and restarts after a reset."""
    ts = 1
    h, py = sim.SimRx(2, 16, 16), PyTiming(2, 16, ts)
    h.enable_timing(ts)
    start = np.array([M32 - 9, 1], np.uint32)
    h.reset([0, 1], start)
    last = start - np.uint32(1)
    idx = np.array([M32 - 3, M32 - 1, 2, M32 - 2, 1, 5, 4], np.uint32)
    k = len(idx)
    cols = (np.zeros(k, np.int32), idx, np.full(k, 2, np.uint8), np.zeros(k, np.int32), np.ones(k, np.int32))
    arrival, pay = np.arange(k, dtype=np.uint32), np.zeros(1, np.uint8)
    h.insert(*cols, pay, arrival)
    py.insert(last, *cols, arrival, 1)
    assert same(h, py)
    assert int(h.timing()[1][0]) == (1 << 32) | 5
    h.reset([0], start[:1])
    py.reset([0])
    one = (np.zeros(1, np.int32), np.array([7], np.uint32)) + tuple(x[:1] for x in cols[2:])
    h.insert(*one, pay, arrival[:1])
    py.insert(last, *one, arrival[:1], 1)
    assert same(h, py)
    assert int(h.timing()[1][0]) == 7 and int(h.timing()[2][0]) == 1
