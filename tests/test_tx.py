"""The send queue and the downlink contributor lists on the CPU: the host build of their source (tests/hostsim/server.cpp
driven by sim.SimTx and sim.contributors: sb_tx.cuh compiled by g++, the pack kernels' three passes in their order and the
contributor kernel's per-member rule) against independent restatements (tests/server_ref.py).

The pack restatement builds datagrams row by row from the rules in include/solo_b200.h; it covers DTX rows, every kind of
bad row, an empty description 1, rows of the host encoder at 40 ms, 20 ms and joint mode 1, index wrap across 2^32,
octet-counter wrap, reset, N = 1 and random rows across several blocks of the sizes pass.  The contributor restatement is
a literal transcription of INTEGRATION.md's CSRC loop, over rooms of 1, 4 and 256 members, streams in no room, k = 1..8,
fewer talkers than k and members outside [0, n)."""
import numpy as np
import pytest

from tests.parity import sb, sim  # noqa: F401  (fixtures)
from tests.server_ref import (BAD, DTX, M32, OCTETS, SENT, PyTx, contributors_literal, csr_rooms, random_rows,
                              select_talkers, split_row)
from tests.util import load_clip


def check_same(a, b):
    (pa, ea), (pb, eb) = a, b
    assert ea == eb
    assert pa == pb


def run_both(sim, n, waves, resets=None):
    """Pack the waves [(bits, nbytes)] on the host build and the restatement (resets: {wave: (streams, start)} before it);
    every pack and the final counters must agree.  Returns the restatement."""
    h, m = sim.SimTx(n), PyTx(n)
    for w, (bits, nb) in enumerate(waves):
        if resets and w in resets:
            h.reset(*resets[w])
            m.reset(*resets[w])
        check_same(h.pack(bits, nb), m.pack(bits, nb))
    assert np.array_equal(h.stats(), m.stats())
    assert [int(v) for v in h.next] == m.next
    return m


def test_rule_equals_split_packet(sb):
    """split_row against solo_b200_split_packet on every (n0, n1) in a grid, with cap above every n0."""
    row = np.arange(256, dtype=np.uint8)
    for n0 in range(-3, 40):
        for n1 in range(-3, 44):
            cls, descs = split_row(row, n0, n1, 256)
            try:
                p1, p2 = sb.split_packet(bytes(row[:max(n0, 0)]), (n0, n1))
                assert cls in (SENT, DTX) and descs == ([p1, p2] if cls == SENT else []), (n0, n1)
            except sb.SoloError:
                assert cls == BAD, (n0, n1)


def test_dtx_bad_and_empty_rows(sim):
    cap = 64
    rows = [(0, 0), (-1, 8), (-32768, 5), (40, 3), (40, -1), (40, -32768), (40, 41), (65, 8), (32767, 8),
            (12, 12), (4, 4), (40, 8), (40, 4), (64, 8)]
    bits = np.random.Generator(np.random.PCG64(1)).integers(0, 256, (len(rows), cap), dtype=np.uint8)
    nb = np.array(rows, np.int16)
    m = run_both(sim, len(rows), [(bits, nb)] * 3)
    cnt = m.stats()
    assert list(cnt[:3, DTX]) == [3] * 3 and list(cnt[3:9, BAD]) == [3] * 6 and (cnt[9:, SENT] == 3).all()
    payload, ents = m.pack(bits, nb)
    assert [e[2] for e in ents if e[0] in (9, 10)] == [2, 2]               # description 1 empty: not emitted
    assert all(e[1] == 3 for e in ents)                                     # every row's index advanced three times


@pytest.mark.parametrize("cfg", [dict(framesize_ms=40), dict(framesize_ms=20), dict(framesize_ms=40, joint_hb=1),
                                 dict(framesize_ms=40, dtx=1)])
def test_host_encoder_rows(sim, cfg):
    """Rows of the host encoder (3 streams of the clip, 12 packets): each datagram is what split_packet gives."""
    clip = load_clip()
    n, P, cap = 3, 12, 256
    encs = [sim.SimEncoder(**cfg) for _ in range(n)]
    S = encs[0].samples
    waves = []
    for p in range(P):
        bits, nb = np.zeros((n, cap), np.uint8), np.zeros((n, 2), np.int16)
        for s, e in enumerate(encs):
            x = clip[(p * S + s * 4001) % (len(clip) - S):][:S] >> s
            b, nb[s], _ = e.encode(x)
            bits[s, :len(b)] = np.frombuffer(b, np.uint8)
        waves.append((bits, nb))
    for e in encs:
        e.close()
    tails = {(40, 0): 8, (20, 0): 4, (40, 1): 4}[(cfg["framesize_ms"], cfg.get("joint_hb", 0))]
    assert all(int(nb[s, 1]) >= tails for _, nb in waves for s in range(n) if nb[s, 0] > 0)
    m = run_both(sim, n, waves)
    assert m.cnt[:, BAD].sum() == 0 and m.cnt[:, SENT].sum() + m.cnt[:, DTX].sum() == n * P


def test_index_wrap_and_reset(sim):
    rng = np.random.Generator(np.random.PCG64(2))
    n = 5
    waves = [random_rows(rng, n, 128) for _ in range(8)]
    resets = {0: ([0, 3], [M32 - 2, M32 - 1]), 4: ([3, 1], [7, M32 - 3]), 6: ([], [])}
    m = run_both(sim, n, waves, resets)
    assert m.next[0] == 6 and m.next[3] == 11 and m.next[1] == 1


def test_octet_counter_wrap(sim):
    """The octet counter is mod 2^32: start both just below it."""
    rng = np.random.Generator(np.random.PCG64(3))
    n = 4
    h, m = sim.SimTx(n), PyTx(n)
    h.cnt[:, OCTETS] = M32 - 100
    m.cnt[:, OCTETS] = M32 - 100
    for _ in range(3):
        bits, nb = random_rows(rng, n, 128, dtx=0, bad=0)
        check_same(h.pack(bits, nb), m.pack(bits, nb))
    assert np.array_equal(h.stats(), m.stats()) and (m.cnt[:, OCTETS] > M32).all()


def test_single_stream(sim):
    rng = np.random.Generator(np.random.PCG64(4))
    run_both(sim, 1, [random_rows(rng, 1, 64, dtx=0.3, bad=0.3) for _ in range(40)])


@pytest.mark.parametrize("n,cap", [(37, 128), (600, 256), (1031, 144)])
def test_random_rows(sim, n, cap):
    rng = np.random.Generator(np.random.PCG64(n + cap))
    waves = [random_rows(rng, n, cap) for _ in range(5)]
    st = rng.choice(n, n // 8, replace=False)
    m = run_both(sim, n, waves, {3: (st, rng.integers(0, M32, len(st)))})
    tot = m.cnt.sum(0)
    assert tot[SENT] > 0 and tot[DTX] > 0 and tot[BAD] > 0


# ---- the contributor lists ----------------------------------------------------------------------------------------------
LAYOUTS = {"ones": [1] * 40, "fours": [4] * 60, "big": [256, 256], "mixed": [1, 4, 256, 4, 1, 0, 17, 4],
           "none": []}


@pytest.mark.parametrize("name", sorted(LAYOUTS))
@pytest.mark.parametrize("k", range(1, 9))
def test_contributors_equal_literal_loop(sim, name, k):
    rng = np.random.Generator(np.random.PCG64(k * 100 + len(name)))
    n = 600
    room_start, members = csr_rooms(rng, n, LAYOUTS[name], out_of_range=3 if name == "mixed" else 0)
    level = rng.integers(0, 256, n).astype(np.uint8)                # bit 7 set on some: the & 0x7f
    flags = np.where(rng.random(n) < (0.15 if k > 4 else 0.6), rng.integers(1, 16, n), 0).astype(np.uint8)
    tk = select_talkers(room_start, members, level, flags, k, n)
    got = sim.contributors(room_start, members, k, tk, level, n)
    want = contributors_literal(room_start, members, len(room_start) - 1, k, tk, level, n)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    in_room = np.zeros(n, bool)
    in_room[members[(members >= 0) & (members < n)]] = True
    assert (got[0][~in_room] == -1).all() and (got[1][~in_room] == 127).all()
    if name in ("ones", "fours", "mixed") and k > 1:
        assert ((tk < 0).sum(1) > 0).any()                              # some room has fewer talkers than k
