"""The receive queue on the CPU: the host build of its source (tests/hostsim/server.cpp driven by sim.SimRx: sb_rx.cuh
compiled by g++, the insert kernels' passes in their order with the atomics as plain read-modify-writes, and the pull
kernel's rule) against an independent restatement of the semantics in include/solo_b200.h (tests/server_ref.PyRx) that
takes the arrivals one at a time in array order.

Seeded arrival processes cover reordering within the depth, duplicates with identical and different bytes, late arrivals,
ring overrun (an index `depth` ahead), bursts of `depth` packets in one call, malformed arrivals, streams out of range,
index wrap across 2^32, jumps of `play` (forward and back) and resets.  The shared merge rule is checked against
solo_b200_merge_packets on every length combination."""
import ctypes as C

import numpy as np
import pytest

from tests.parity import sb, sim  # noqa: F401  (fixtures)
from tests.server_ref import M32, PyRx, check_pull, make_ops, replay, run_model


@pytest.mark.parametrize("depth,desc_cap,explicit_play", [(8, 128, False), (8, 128, True), (2, 16, True), (32, 64, False),
                                                          (4, 1024, True)])
def test_host_build_equals_restatement(sim, depth, desc_cap, explicit_play):
    rng = np.random.Generator(np.random.PCG64(depth * 1000 + desc_cap + explicit_play))
    n = 37
    ops, m = make_ops(rng, n, depth, desc_cap, 30, explicit_play=explicit_play)
    h = sim.SimRx(n, depth, desc_cap)
    got = replay(h, ops)
    _, want = run_model(ops, n, depth, desc_cap)
    for g, w in zip(got, want):
        check_pull(g, w)
    assert np.array_equal(h.cnt.astype(np.int64), m.cnt) and int(h.bad[0]) == m.bad
    assert not h.elect.any() and (h.rep == 0xFFFFFFFF).all()      # election words are empty between calls
    # every case the process is meant to produce happened
    tot = m.cnt.sum(0)
    assert all(tot[k] > 0 for k in range(8)) and m.bad > 0, tot


def test_permuted_arrivals_follow_array_order(sim):
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
        h = sim.SimRx(n, depth, cap)
        got = replay(h, perm_ops)
        m, want = run_model(perm_ops, n, depth, cap)
        for g, w in zip(got, want):
            check_pull(g, w)
        assert np.array_equal(h.cnt.astype(np.int64), m.cnt)


def test_wrap_and_overrun_by_hand(sim):
    """Packets across the 2^32 wrap, an index `depth` ahead that supersedes a held one, and a late copy."""
    n, depth, cap = 1, 4, 16
    for impl in (sim.SimRx(n, depth, cap), PyRx(n, depth, cap)):
        impl.reset([0], [M32 - 2])                      # plays 2^32 - 2, 2^32 - 1, 0, 1, ...
        pay = np.arange(1, 65, dtype=np.uint8)
        impl.insert(np.zeros(4, np.int32), np.array([M32 - 1, 0, M32 - 2, 3], np.uint32), np.array([1, 2, 2, 1], np.uint8),
                    np.array([0, 4, 8, 12], np.int32), np.array([4, 4, 4, 4], np.int32), pay)
        got = [impl.pull() for _ in range(2)]
        impl.insert(np.zeros(3, np.int32), np.array([M32 - 1, 4, 7], np.uint32), np.array([1, 1, 2], np.uint8),
                    np.array([0, 20, 30], np.int32), np.array([3, 5, 6], np.int32), pay)
        got += [impl.pull() for _ in range(3)]
        if isinstance(impl, sim.SimRx):
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
def test_merge_rule_equals_merge_packets(sim, sb, cap):
    """rx_merge (sb_rx.cuh) against solo_b200_merge_packets for every pair of lengths 0..40 and a few large ones."""
    lengths = list(range(41)) + [200, 255, 256]
    a = np.arange(1, 301, dtype=np.uint8)
    b = np.arange(101, 401, dtype=np.uint16).astype(np.uint8)
    for n1 in lengths:
        for n2 in lengths:
            row, nb, lf = sim.merge(n1, n2)
            out = np.full(max(cap, 1), 0xEE, np.uint8)
            wnb = np.zeros(2, np.int16)
            wlf = C.c_int32()
            r = sb.lib().solo_b200_merge_packets(a.ctypes.data if n1 else None, n1, b.ctypes.data if n2 else None, n2,
                                                 out.ctypes.data, cap, wnb.ctypes.data, C.byref(wlf))
            if n1 + n2 > cap and n1 + n2 > 0:
                assert r == -1
                continue
            assert r == 0 and tuple(nb) == tuple(wnb) and lf == wlf.value, (n1, n2, cap)
            want = bytes(a[:n1]) + bytes(b[:n2]) if n1 + n2 else bytes(16)
            assert row == len(want)
            if n1 + n2 or cap >= 16:
                assert bytes(out[:row]) == want
