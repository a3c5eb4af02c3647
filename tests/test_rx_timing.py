"""Receive-queue timing on the CPU: the host model (tests/hostsim/rx.cpp's rx_model_timing, the kernels' per-arrival rules
of sb_rx.cuh compiled by g++, driven by sim.SimRxTiming) against a direct statement of RFC 3550 A.1 / A.8 and of the
margin rule in include/solo_b200.h, on seeded arrival processes and on cases with a known answer.

The processes are tests/test_rx.py's (reordering, duplicates, late arrivals, ring overrun, malformed entries, streams out
of range, resets, index wrap across 2^32) with receive times added: a network delay per arrival, a receiver clock that
wraps at 2^32, and transit jumps of 2^31."""
import numpy as np
import pytest

from tests.hostsim.rx_timing import SimRxTiming
from tests.test_rx import M32, PyRx, make_ops


# ---- the rules, stated directly ----------------------------------------------------------------------------------------
class PyTiming:
    """Per stream None (no valid arrival since the reset) or [transit, jitter, cycles, max_seq, received]; margin [n, 8]."""

    def __init__(self, n, desc_cap, ts):
        self.n, self.desc_cap, self.ts = n, desc_cap, ts
        self.st = [None] * n
        self.margin = np.zeros((n, 8), np.int64)

    def insert(self, last, stream, index, desc, off, lens, arrival, payload_bytes):
        for a in range(len(stream)):
            s, p, d, o, ln = int(stream[a]), int(index[a]), int(desc[a]), int(off[a]), int(lens[a])
            if not 0 <= s < self.n or d not in (1, 2) or not 1 <= ln <= self.desc_cap or o < 0 or o + ln > payload_bytes:
                continue
            ahead = (p - int(last[s])) % M32             # current: 1 <= ahead < 2^31
            if 1 <= ahead < (1 << 31):
                self.margin[s, min(ahead - 1, 7)] += 1
            transit = (int(arrival[a]) - p * self.ts) % M32     # RFC 3550 A.8: arrival - RTP timestamp
            st = self.st[s]
            if st is None:
                self.st[s] = [transit, 0, 0, p, 1]
                continue
            D = (transit - st[0]) % M32
            D = D - M32 if D >= (1 << 31) else D
            st[1] = (st[1] + abs(D) - (((st[1] + 8) % M32) >> 4)) % M32    # J += |D| - (J + 8) / 16, in uint32
            udelta = (p - st[3]) % M32                   # A.1: an index ahead of max_seq, one cycle up past 2^32
            if 0 < udelta < (1 << 31):
                if p < st[3]:
                    st[2] = (st[2] + 1) % M32
                st[3] = p
            st[0] = transit
            st[4] = (st[4] + 1) % M32

    def reset(self, streams):
        for s in streams:
            self.st[int(s)] = None
            self.margin[int(s)] = 0

    def read(self):
        """(jitter >> 4, highest, received, margin) as solo_b200_rx_timing reports them."""
        z = [0, 0, 0, 0, 0]
        st = [x if x is not None else z for x in self.st]
        return (np.array([x[1] >> 4 for x in st], np.uint32), np.array([(x[2] << 32) | x[3] for x in st], np.uint64),
                np.array([x[4] for x in st], np.uint32), self.margin.astype(np.uint32))


# ---- seeded processes with receive times ------------------------------------------------------------------------------
def add_arrivals(rng, ops, ts, clock0):
    """ops of make_ops, each insert with receive times: clock0 + index * ts + a delay of up to 3 packets, some arrivals
    shifted by 2^31 (a transit jump) and some at a random time.  Returns the timed ops."""
    out = []
    for op in ops:
        if op[0] != "insert":
            out.append(op)
            continue
        index = op[2].astype(np.int64)
        arr = clock0 + index * ts + rng.integers(0, 3 * ts + 1, len(index))
        u = rng.random(len(index))
        arr = np.where(u < 0.02, arr + (1 << 31), arr)
        arr = np.where((u >= 0.02) & (u < 0.03), rng.integers(0, M32, len(index)), arr)
        out.append(op + ((arr % M32).astype(np.uint32),))
    return out


def replay(ops, n, depth, desc_cap, ts, impls):
    """Apply the timed ops to the queue restatement (for `last`) and to each timing implementation."""
    q = PyRx(n, depth, desc_cap)
    for op in ops:
        if op[0] == "insert":
            stream, index, desc, off, lens, payload, arrival = op[1:]
            last = np.array(q.last, np.uint32)
            for t in impls:
                t.insert(last, stream, index, desc, off, lens, arrival, len(payload))
            q.insert(stream, index, desc, off, lens, payload)
        elif op[0] == "reset":
            for t in impls:
                t.reset(op[1])
            q.reset(op[1], op[2])
        else:
            q.pull(op[1])
    return q


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a.read(), b.read()))


@pytest.mark.parametrize("depth,desc_cap,ts,explicit_play", [(8, 128, 640, False), (8, 128, 640, True),
                                                             (2, 16, 320, True), (32, 64, 0x9E3779B1, False)])
def test_model_equals_rfc_statement(depth, desc_cap, ts, explicit_play):
    rng = np.random.Generator(np.random.PCG64(depth * 7919 + desc_cap + explicit_play))
    n = 37
    ops, _ = make_ops(rng, n, depth, desc_cap, 30, explicit_play=explicit_play)
    ops = add_arrivals(rng, ops, ts, M32 - 5000)         # the receiver's clock wraps early on
    sim, py = SimRxTiming(n, desc_cap, ts), PyTiming(n, desc_cap, ts)
    replay(ops, n, depth, desc_cap, ts, [sim, py])
    assert same(sim, py)
    jitter, highest, received, margin = py.read()
    # the process reached what it is meant to cover: index wrap (a cycle), transit jumps (jitter past 2^27 units),
    # every margin bin, and resets between calls
    assert (highest >> np.uint64(32)).max() >= 1
    assert jitter.max() > (1 << 27)
    assert (margin.sum(0)[:min(depth + 2, 8)] > 0).all()     # indices reach depth + 2 ahead
    assert any(op[0] == "reset" for op in ops)


def test_model_step_by_step():
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
        timed = add_arrivals(rng, ops, ts, 12345)
        sim, py = SimRxTiming(n, desc_cap, ts), PyTiming(n, desc_cap, ts)
        q = PyRx(n, depth, desc_cap)
        for op in timed:
            if op[0] == "insert":
                last = np.array(q.last, np.uint32)
                for t in (sim, py):
                    t.insert(last, *op[1:6], op[7], len(op[6]))
                q.insert(*op[1:7])
                assert same(sim, py)
            elif op[0] == "reset":
                for t in (sim, py):
                    t.reset(op[1])
                q.reset(op[1], op[2])
            else:
                q.pull(op[1])


def run_stream(ts, sends):
    """One stream: per tick, (index, arrival) pairs in arrival order, then a pull.  Returns (model, restatement)."""
    sim, py = SimRxTiming(1, 64, ts), PyTiming(1, 64, ts)
    q = PyRx(1, 32, 64)
    pay = np.zeros(64, np.uint8)
    for tick in sends:
        if tick:
            idx = np.array([p for p, _ in tick], np.uint32)
            arr = np.array([a % M32 for _, a in tick], np.uint32)
            k = len(tick)
            args = (np.zeros(k, np.int32), idx, np.ones(k, np.uint8), np.zeros(k, np.int32), np.full(k, 8, np.int32), arr, 64)
            last = np.array(q.last, np.uint32)
            sim.insert(last, *args)
            py.insert(last, *args)
            q.insert(*args[:5], pay)
        q.pull()
    assert same(sim, py)
    return sim, py


@pytest.mark.parametrize("delay", [0, 17, 5000, M32 - 3])
def test_constant_delay_gives_zero_jitter(delay):
    ts = 640
    sends = [[(t, t * ts + delay + 123456789)] for t in range(50)]
    sim, _ = run_stream(ts, sends)
    jitter, highest, received, margin = sim.read()
    assert int(jitter[0]) == 0 and int(sim.jitter[0]) == 0 and int(received[0]) == 50 and int(highest[0]) == 49


@pytest.mark.parametrize("k", [1, 2, 40, 640, 100000])
def test_alternating_delay_converges_to_fixed_point(k):
    """Delays 0, k, 0, k, ...: |D| = k for every packet after the first, and J += k - ((J + 8) >> 4) climbs to the
    recurrence's fixed point 16k - 8 (the smallest J with (J + 8) >> 4 = k) and stays; reported, (16k - 8) >> 4 = k - 1."""
    ts = 640
    sends = [[(t, t * ts + (k if t % 2 else 0))] for t in range(16 * 200)]
    sim, _ = run_stream(ts, sends)
    assert int(sim.jitter[0]) == 16 * k - 8
    assert int(sim.read()[0][0]) == k - 1


@pytest.mark.parametrize("m", [0, 1, 3, 7, 12])
def test_margin_of_packets_m_ticks_early(m):
    """Packet t + m + 1 arrives at tick t, before the pull that plays t + 1: every arrival is m pulls early, so the
    histogram is all in bin min(m, 7)."""
    ts = 640
    sends = [[(t + m, (t + m) * ts - m * ts)] for t in range(30)]
    sim, _ = run_stream(ts, sends)
    margin = sim.read()[3][0]
    assert int(margin[min(m, 7)]) == 30 and int(margin.sum()) == 30


def test_highest_across_wrap_and_reset():
    """highest counts a cycle when the index wraps past 2^32, ignores older indices, and restarts after a reset."""
    ts = 1
    sim, py = SimRxTiming(2, 16, ts), PyTiming(2, 16, ts)
    last = np.array([M32 - 10, 0], np.uint32)
    idx = np.array([M32 - 3, M32 - 1, 2, M32 - 2, 1, 5, 4], np.uint32)
    k = len(idx)
    args = (np.zeros(k, np.int32), idx, np.full(k, 2, np.uint8), np.zeros(k, np.int32), np.ones(k, np.int32),
            np.arange(k, dtype=np.uint32), 1)
    for t in (sim, py):
        t.insert(last, *args)
    assert same(sim, py)
    assert int(sim.read()[1][0]) == (1 << 32) | 5
    for t in (sim, py):
        t.reset([0])
        t.insert(last, np.zeros(1, np.int32), np.array([7], np.uint32), *(x[:1] for x in args[2:6]), 1)
    assert same(sim, py)
    assert int(sim.read()[1][0]) == 7 and int(sim.read()[2][0]) == 1
