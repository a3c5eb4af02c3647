"""The receive queue on the CPU: the host build of its source (tests/hostsim/rx.cpp: sb_rx.cuh compiled by g++, the insert
kernels' passes in their order with the atomics as plain read-modify-writes, and the pull kernel's rule) against an
independent restatement of the semantics in include/solo_b200.h that takes the arrivals one at a time in array order.

Seeded arrival processes cover reordering within the depth, duplicates with identical and different bytes, late arrivals,
ring overrun (an index `depth` ahead), bursts of `depth` packets in one call, malformed arrivals, streams out of range,
index wrap across 2^32, jumps of `play` (forward and back) and resets.  The shared merge rule is checked against
solo_b200_merge_packets on every length combination."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.parity import sb  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "rx.cpp")
M32 = 1 << 32
STORED, DUPLICATE, LATE, DROPPED, MALFORMED, PLAYED_BOTH, PLAYED_ONE, PLAYED_NONE = range(8)


# ---- the semantics, restated --------------------------------------------------------------------------------------------
def current(p, last):
    return 1 <= (p - last) % M32 < (1 << 31)


def merge(d1, d2):
    """(row, (n0, n1), lostflag) of solo_b200_merge_packets for the descriptions held (b"" = missing)."""
    if d1 and d2:
        return d1 + d2, (len(d1) + len(d2), len(d2)), 4
    if d1:
        return d1, (len(d1), 0), 2
    if d2:
        return d2, (len(d2), 0), 3
    return bytes(16), (16, 8), 1


class PyRx:
    """Per stream: last, slots {j: [index, {desc: bytes}]}, 8 counters; plus the queue-wide bad-stream count."""

    def __init__(self, n, depth, desc_cap):
        self.n, self.depth, self.desc_cap = n, depth, desc_cap
        self.last = [M32 - 1] * n
        self.slots = [{} for _ in range(n)]
        self.cnt = np.zeros((n, 8), np.int64)
        self.bad = 0

    def _held_dist(self, s, j):
        h = self.slots[s].get(j)
        return (h[0] - self.last[s]) % M32 if h and h[1] and current(h[0], self.last[s]) else 0

    def insert(self, stream, index, desc, off, lens, payload):
        valid = []
        for a in range(len(stream)):
            s, p, d, o, ln = int(stream[a]), int(index[a]), int(desc[a]), int(off[a]), int(lens[a])
            if not 0 <= s < self.n:
                self.bad += 1
            elif d not in (1, 2) or not 1 <= ln <= self.desc_cap or o < 0 or o + ln > len(payload):
                self.cnt[s, MALFORMED] += 1
            elif not current(p, self.last[s]):
                self.cnt[s, LATE] += 1
            else:
                valid.append(a)
        newest = {}                 # (stream, slot) -> newest distance among the held index and the valid arrivals
        for a in valid:
            s, p = int(stream[a]), int(index[a])
            key = (s, p % self.depth)
            newest[key] = max(newest.get(key, self._held_dist(*key)), (p - self.last[s]) % M32)
        for a in valid:             # in array order: the first arrival of each (index, desc) is stored
            s, p, d, o, ln = int(stream[a]), int(index[a]), int(desc[a]), int(off[a]), int(lens[a])
            j = p % self.depth
            if (p - self.last[s]) % M32 != newest[(s, j)]:
                self.cnt[s, DROPPED] += 1
                continue
            h = self.slots[s].get(j)
            if h is None or h[0] != p:
                if h is not None:
                    self.cnt[s, DROPPED] += len(h[1])       # held descriptions discarded
                h = self.slots[s][j] = [p, {}]
            if d in h[1]:
                self.cnt[s, DUPLICATE] += 1
            else:
                h[1][d] = bytes(payload[o:o + ln])
                self.cnt[s, STORED] += 1

    def pull(self, play=None):
        rows, nbytes, flags = [], np.zeros((self.n, 2), np.int16), np.zeros(self.n, np.int32)
        for s in range(self.n):
            t = int(play[s]) if play is not None else (self.last[s] + 1) % M32
            j = t % self.depth
            h = self.slots[s].get(j)
            held = h[1] if h and h[0] == t else {}
            row, nb, f = merge(held.get(1, b""), held.get(2, b""))
            rows.append(row)
            nbytes[s], flags[s] = nb, f
            self.cnt[s, {4: PLAYED_BOTH, 2: PLAYED_ONE, 3: PLAYED_ONE, 1: PLAYED_NONE}[f]] += 1
            self.last[s] = t
            if h and h[1] and not current(h[0], t):
                if h[0] != t:
                    self.cnt[s, DROPPED] += len(h[1])
                del self.slots[s][j]
        return rows, nbytes, flags

    def reset(self, streams, start):
        for s, t in zip(streams, start):
            self.slots[s] = {}
            self.cnt[s] = 0
            self.last[s] = (int(t) - 1) % M32


# ---- seeded arrival processes -------------------------------------------------------------------------------------------
def make_ops(rng, n, depth, desc_cap, ticks, explicit_play=False):
    """A list of ("insert", stream, index, desc, off, len, payload) / ("pull", play or None) / ("reset", streams, start)
    operations, generated against PyRx so that the indices stay near each stream's playout point.  Returns (ops, model)
    with the model after all of them."""
    m = PyRx(n, depth, desc_cap)
    ops = []
    for tick in range(ticks):
        if tick % 7 == 3:           # rejoin a few streams, some just below the 2^32 wrap
            st = rng.choice(n, max(1, n // 16), replace=False).astype(np.int32)
            start = np.where(rng.random(len(st)) < 0.5, M32 - rng.integers(1, 4, len(st)), rng.integers(0, M32, len(st)))
            start = start.astype(np.uint32)
            ops.append(("reset", st, start))
            m.reset(st, start)
        rec = []                    # (stream, index, desc, bytes)
        for s in range(n):
            base = m.last[s]
            k = rng.integers(0, 7)
            if rng.random() < 0.05:     # a burst of `depth` packets, both descriptions, in shuffled order
                for q in range(1, depth + 1):
                    for d in (1, 2):
                        rec.append([s, base + q, d, rng.bytes(int(rng.integers(1, desc_cap + 1)))])
            for _ in range(k):
                u = rng.random()
                if u < 0.6:
                    off = int(rng.integers(1, depth + 1))           # within the depth
                elif u < 0.75:
                    off = int(rng.integers(-3, 1))                  # late: already played
                elif u < 0.85:
                    off = depth + int(rng.integers(1, 3))           # ring overrun
                else:
                    off = int(rng.integers(1, 3))
                rec.append([s, base + off, int(rng.integers(1, 3)), rng.bytes(int(rng.integers(1, desc_cap + 1)))])
        for i in range(len(rec) // 8):  # duplicates: identical bytes, or other bytes
            r = list(rec[int(rng.integers(0, len(rec)))])
            if rng.random() < 0.5:
                r[3] = rng.bytes(int(rng.integers(1, desc_cap + 1)))
            rec.append(r)
        order = rng.permutation(len(rec))
        rec = [rec[i] for i in order]
        stream = np.array([r[0] for r in rec], np.int32)
        index = np.array([r[1] % M32 for r in rec], np.uint32)
        desc = np.array([r[2] for r in rec], np.uint8)
        lens = np.array([len(r[3]) for r in rec], np.int32)
        off = np.zeros(len(rec), np.int32)
        off[1:] = np.cumsum(lens[:-1])
        payload = np.frombuffer(b"".join(r[3] for r in rec) + bytes(3), np.uint8).copy()
        # malformed and out-of-range entries
        bad = rng.random(len(rec))
        desc[bad < 0.01] = 0
        desc[(bad >= 0.01) & (bad < 0.02)] = 3
        lens[(bad >= 0.02) & (bad < 0.025)] = 0
        lens[(bad >= 0.025) & (bad < 0.03)] = desc_cap + 1
        off[(bad >= 0.03) & (bad < 0.035)] = -1
        sel = (bad >= 0.035) & (bad < 0.04)
        off[sel] = len(payload) - lens[sel] + 1
        stream[(bad >= 0.04) & (bad < 0.045)] = -1
        stream[(bad >= 0.045) & (bad < 0.05)] = n
        ops.append(("insert", stream, index, desc, off, lens, payload))
        m.insert(stream, index, desc, off, lens, payload)
        play = None
        if explicit_play:
            nxt = np.array([(v + 1) % M32 for v in m.last], np.int64)
            u = rng.random(n)
            nxt = np.where(u < 0.1, nxt + rng.integers(2, 2 * depth, n), nxt)       # jump ahead
            nxt = np.where((u >= 0.1) & (u < 0.13), nxt - rng.integers(2, 5, n), nxt)   # go back
            play = (nxt % M32).astype(np.uint32)
        ops.append(("pull", play))
        m.pull(play)
    return ops, m


def run_model(ops, n, depth, desc_cap):
    """(model, [its pull results]) after applying ops to PyRx."""
    m = PyRx(n, depth, desc_cap)
    out = []
    for op in ops:
        if op[0] == "insert":
            m.insert(*op[1:])
        elif op[0] == "reset":
            m.reset(op[1], op[2])
        else:
            out.append(m.pull(op[1]))
    return m, out


# ---- the host build ----------------------------------------------------------------------------------------------------
def load_lib(out):
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-w", SRC, "-o", out])
    lib = C.CDLL(out)
    vp, ci = C.c_void_p, C.c_int
    lib.rx_model_insert.argtypes = [ci, ci, ci] + [vp] * 13 + [ci, vp, C.c_int64]
    lib.rx_model_pull.argtypes = [ci, ci, ci] + [vp] * 6 + [vp, ci, vp, vp]
    lib.rx_model_merge.argtypes = [ci, ci, vp, vp]
    lib.rx_model_merge.restype = ci
    return lib


@pytest.fixture(scope="module")
def L(tmp_path_factory):
    return load_lib(str(tmp_path_factory.mktemp("rx") / "librx.so"))


class HostRx:
    """The queue's device state arrays on the host, driven by the host build."""

    def __init__(self, L, n, depth, desc_cap):
        self.L, self.n, self.depth, self.desc_cap = L, n, depth, desc_cap
        self.last = np.full(n, M32 - 1, np.uint32)
        self.idx = np.zeros(n * depth, np.uint32)
        self.len = np.zeros(n * depth * 2, np.uint16)
        self.elect = np.zeros(n * depth * 2, np.uint64)
        self.rep = np.full(n * depth, 0xFFFFFFFF, np.uint32)
        self.cnt = np.zeros((n, 8), np.uint32)
        self.bad = np.zeros(1, np.uint64)
        self.store = np.zeros(n * depth * 2 * desc_cap + 16, np.uint8)

    def insert(self, stream, index, desc, off, lens, payload):
        a = [np.ascontiguousarray(x, t) for x, t in ((stream, np.int32), (index, np.uint32), (desc, np.uint8),
                                                     (off, np.int32), (lens, np.int32), (payload, np.uint8))]
        self.L.rx_model_insert(self.n, self.depth, self.desc_cap, *(x.ctypes.data for x in (
            self.last, self.idx, self.len, self.elect, self.rep, self.cnt, self.bad, self.store)), *(x.ctypes.data for x in a[:5]),
            len(a[0]), a[5].ctypes.data, a[5].size)

    def pull(self, play=None):
        cap = 2 * self.desc_cap
        bits = np.zeros((self.n, cap), np.uint8)
        nb = np.zeros((self.n, 2), np.int16)
        lf = np.zeros(self.n, np.int32)
        p = np.ascontiguousarray(play, np.uint32) if play is not None else None
        self.L.rx_model_pull(self.n, self.depth, self.desc_cap, self.last.ctypes.data, self.idx.ctypes.data,
                             self.len.ctypes.data, self.cnt.ctypes.data, self.store.ctypes.data,
                             p.ctypes.data if p is not None else None, bits.ctypes.data, cap, nb.ctypes.data, lf.ctypes.data)
        return bits, nb, lf

    def reset(self, streams, start):
        for s, t in zip(streams, start):
            self.last[s] = (int(t) - 1) % M32
            self.cnt[s] = 0
            self.len[s * 2 * self.depth:(s + 1) * 2 * self.depth] = 0


def check_pull(got, want):
    bits, nb, lf = got
    rows, wnb, wlf = want
    assert np.array_equal(nb, wnb) and np.array_equal(lf, wlf)
    for s, row in enumerate(rows):
        assert bytes(bits[s, :len(row)]) == row, s


def replay(impl, ops):
    pulls = []
    for op in ops:
        if op[0] == "insert":
            impl.insert(*op[1:])
        elif op[0] == "reset":
            impl.reset(op[1], op[2])
        else:
            pulls.append(impl.pull(op[1]))
    return pulls


@pytest.mark.parametrize("depth,desc_cap,explicit_play", [(8, 128, False), (8, 128, True), (2, 16, True), (32, 64, False),
                                                          (4, 1024, True)])
def test_host_build_equals_restatement(L, depth, desc_cap, explicit_play):
    rng = np.random.Generator(np.random.PCG64(depth * 1000 + desc_cap + explicit_play))
    n = 37
    ops, m = make_ops(rng, n, depth, desc_cap, 30, explicit_play=explicit_play)
    h = HostRx(L, n, depth, desc_cap)
    got = replay(h, ops)
    _, want = run_model(ops, n, depth, desc_cap)
    for g, w in zip(got, want):
        check_pull(g, w)
    assert np.array_equal(h.cnt.astype(np.int64), m.cnt) and int(h.bad[0]) == m.bad
    assert not h.elect.any() and (h.rep == 0xFFFFFFFF).all()      # election words are empty between calls
    # every case the process is meant to produce happened
    tot = m.cnt.sum(0)
    assert all(tot[k] > 0 for k in range(8)) and m.bad > 0, tot


def test_permuted_arrivals_follow_array_order(L):
    """The same arrivals in another order give the restatement's result for that order (the first of duplicates wins)."""
    rng = np.random.Generator(np.random.PCG64(5))
    n, depth, cap = 9, 4, 32
    ops, _ = make_ops(rng, n, depth, cap, 6)
    for trial in range(3):
        perm_ops = []
        for op in ops:
            if op[0] == "insert":
                p = rng.permutation(len(op[1]))
                op = ("insert",) + tuple(x[p] for x in op[1:6]) + (op[6],)
            perm_ops.append(op)
        h = HostRx(L, n, depth, cap)
        got = replay(h, perm_ops)
        m, want = run_model(perm_ops, n, depth, cap)
        for g, w in zip(got, want):
            check_pull(g, w)
        assert np.array_equal(h.cnt.astype(np.int64), m.cnt)


def test_wrap_and_overrun_by_hand(L):
    """Packets across the 2^32 wrap, an index `depth` ahead that supersedes a held one, and a late copy."""
    n, depth, cap = 1, 4, 16
    for impl in (HostRx(L, n, depth, cap), PyRx(n, depth, cap)):
        impl.reset([0], [M32 - 2])                      # plays 2^32 - 2, 2^32 - 1, 0, 1, ...
        pay = np.arange(1, 65, dtype=np.uint8)
        impl.insert(np.zeros(4, np.int32), np.array([M32 - 1, 0, M32 - 2, 3], np.uint32), np.array([1, 2, 2, 1], np.uint8),
                    np.array([0, 4, 8, 12], np.int32), np.array([4, 4, 4, 4], np.int32), pay)
        got = [impl.pull() for _ in range(2)]
        impl.insert(np.zeros(3, np.int32), np.array([M32 - 1, 4, 7], np.uint32), np.array([1, 1, 2], np.uint8),
                    np.array([0, 20, 30], np.int32), np.array([3, 5, 6], np.int32), pay)
        got += [impl.pull() for _ in range(3)]
        if isinstance(impl, HostRx):
            cnt, first = impl.cnt.astype(np.int64), got
        else:
            want = got
            assert np.array_equal(cnt, impl.cnt), (cnt, impl.cnt)
            for g, w in zip(first, want):
                check_pull(g, w)
            # index 3 supersedes 2^32 - 1 in its slot; 2^32 - 2 plays description 2 only; the late copy of 2^32 - 1 counts
            # late; 4 and 7 then supersede the held 0 and 3 (dropped), so 0, 1 and 2 play nothing
            assert [int(w[2][0]) for w in want] == [3, 1, 1, 1, 1]
            assert list(impl.cnt[0]) == [5, 0, 1, 3, 0, 0, 1, 4]


@pytest.mark.parametrize("cap", [0, 15, 16, 40, 400])
def test_merge_rule_equals_merge_packets(L, sb, cap):
    """rx_merge (sb_rx.cuh) against solo_b200_merge_packets for every pair of lengths 0..40 and a few large ones."""
    lengths = list(range(41)) + [200, 255, 256]
    a = np.arange(1, 301, dtype=np.uint8)
    b = np.arange(101, 401, dtype=np.uint16).astype(np.uint8)
    for n1 in lengths:
        for n2 in lengths:
            nb = np.zeros(2, np.int16)
            lf = C.c_int32()
            row = L.rx_model_merge(n1, n2, nb.ctypes.data, C.byref(lf))
            out = np.full(max(cap, 1), 0xEE, np.uint8)
            wnb = np.zeros(2, np.int16)
            wlf = C.c_int32()
            r = sb.lib().solo_b200_merge_packets(a.ctypes.data if n1 else None, n1, b.ctypes.data if n2 else None, n2,
                                                 out.ctypes.data, cap, wnb.ctypes.data, C.byref(wlf))
            if n1 + n2 > cap and n1 + n2 > 0:
                assert r == -1
                continue
            assert r == 0 and tuple(nb) == tuple(wnb) and lf.value == wlf.value, (n1, n2, cap)
            want = bytes(a[:n1]) + bytes(b[:n2]) if n1 + n2 else bytes(16)
            assert row == len(want)
            if n1 + n2 or cap >= 16:
                assert bytes(out[:row]) == want
