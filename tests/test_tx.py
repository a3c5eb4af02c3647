"""The send queue and the downlink contributor lists on the CPU: the host build of their source (tests/hostsim/tx.cpp:
sb_tx.cuh compiled by g++, the pack kernels' three passes in their order and the contributor kernel's per-member rule)
against independent restatements.

The pack restatement builds datagrams row by row from the rules in include/solo_b200.h; it covers DTX rows, every kind of
bad row, an empty description 1, rows of the host encoder at 40 ms, 20 ms and joint mode 1, index wrap across 2^32,
octet-counter wrap, reset, N = 1 and random rows across several blocks of the sizes pass.  The contributor restatement is
a literal transcription of INTEGRATION.md's CSRC loop, over rooms of 1, 4 and 256 members, streams in no room, k = 1..8,
fewer talkers than k and members outside [0, n)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.parity import sb, sim  # noqa: F401  (fixtures)
from tests.util import load_clip

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "tx.cpp")
M32 = 1 << 32
SENT, OCTETS, DTX, BAD = range(4)


# ---- the pack semantics, restated --------------------------------------------------------------------------------------
def split_row(row, n0, n1, cap):
    """(counter, [description bytes]) of one encoded row under the header's rules."""
    if n0 <= 0:
        return DTX, []
    if n1 < 4 or n1 > n0 or n0 > cap:
        return BAD, []
    return SENT, [bytes(row[:n0 - n1]), bytes(row[n0 - n1:n0])]


class PyTx:
    """Per stream: next index and the four counters (kept exact, reported mod 2^32)."""

    def __init__(self, n):
        self.n = n
        self.next = [0] * n
        self.cnt = np.zeros((n, 4), np.int64)

    def pack(self, bits, nbytes):
        """-> (payload bytes, [(stream, index, desc, off, len)])."""
        cap = bits.shape[1]
        payload, ents = b"", []
        for s in range(self.n):
            cls, descs = split_row(bits[s], int(nbytes[s, 0]), int(nbytes[s, 1]), cap)
            idx = self.next[s]
            self.next[s] = (idx + 1) % M32
            self.cnt[s, cls] += 1
            for d, data in enumerate(descs, 1):
                if data:
                    ents.append((s, idx, d, len(payload), len(data)))
                    payload += data
                    self.cnt[s, OCTETS] += len(data)
        return payload, ents

    def reset(self, streams, start):
        for s, t in zip(streams, start):
            self.next[s] = int(t) % M32
            self.cnt[s] = 0

    def stats(self):
        return (self.cnt % M32).astype(np.uint32)


# ---- the host build -----------------------------------------------------------------------------------------------------
def load_lib(out):
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-w", SRC, "-o", out])
    lib = C.CDLL(out)
    vp, ci = C.c_void_p, C.c_int
    lib.tx_model_pack.argtypes = [ci, vp, ci, vp] + [vp] * 9
    lib.tx_model_pack.restype = ci
    lib.tx_model_contributors.argtypes = [vp, vp, ci, ci, vp, vp, ci, vp, vp]
    return lib


@pytest.fixture(scope="module")
def L(tmp_path_factory):
    return load_lib(str(tmp_path_factory.mktemp("tx") / "libtx.so"))


class HostTx:
    """The queue's device state arrays on the host, driven by the host build."""

    def __init__(self, L, n):
        self.L, self.n = L, n
        self.next = np.zeros(n, np.uint32)
        self.cnt = np.zeros((n, 4), np.uint32)

    def pack(self, bits, nbytes):
        bits = np.ascontiguousarray(bits, np.uint8)
        nbytes = np.ascontiguousarray(nbytes, np.int16)
        e = 2 * self.n
        payload = np.zeros(self.n * bits.shape[1], np.uint8)
        st, ix, de, of, ln = (np.zeros(e, t) for t in (np.int32, np.uint32, np.uint8, np.int32, np.int32))
        total = C.c_int64()
        c = self.L.tx_model_pack(self.n, bits.ctypes.data, bits.shape[1], nbytes.ctypes.data, self.next.ctypes.data,
                                 self.cnt.ctypes.data, payload.ctypes.data, st.ctypes.data, ix.ctypes.data, de.ctypes.data,
                                 of.ctypes.data, ln.ctypes.data, C.byref(total))
        return bytes(payload[:total.value]), list(zip(*(x[:c].tolist() for x in (st, ix, de, of, ln))))

    def reset(self, streams, start):
        for s, t in zip(streams, start):
            self.next[s] = int(t) % M32
            self.cnt[s] = 0

    def stats(self):
        return self.cnt.copy()


def random_rows(rng, n, cap, dtx=0.05, bad=0.05):
    """bits uint8 [n, cap], nbytes int16 [n, 2]: golden-like sent rows (60-120 bytes, a 4- or 8-byte high-band tail in
    description 2), about `dtx` DTX rows and `bad` rows of every kind, a few empty descriptions 1."""
    bits = rng.integers(0, 256, (n, cap), dtype=np.uint8)
    n0 = rng.integers(60, min(cap, 121) + 1, n)
    n1 = rng.integers(4, 60, n)
    n1 = np.minimum(n1, n0)
    u = rng.random(n)
    n1[u < 0.02] = n0[u < 0.02]                                     # description 1 empty
    kind = rng.integers(0, 6, n)
    badrow = (u >= 0.02) & (u < 0.02 + bad)
    n1[badrow & (kind == 0)] = rng.integers(-5, 4, n)[badrow & (kind == 0)]      # n1 < 4 (and negative)
    n1[badrow & (kind == 1)] = n0[badrow & (kind == 1)] + 1                      # n1 > n0
    n0[badrow & (kind == 2)] = cap + 1                                           # n0 > cap
    n0[badrow & (kind == 3)] = 32767
    n1[badrow & (kind == 4)] = -32768
    n1[badrow & (kind == 5)] = 32767
    dt = (u >= 0.02 + bad) & (u < 0.02 + bad + dtx)
    n0[dt] = rng.choice([0, -1, -32768], int(dt.sum()))
    nbytes = np.stack([n0, n1], 1).astype(np.int16)
    return bits, nbytes


def check_same(a, b):
    (pa, ea), (pb, eb) = a, b
    assert ea == eb
    assert pa == pb


def run_both(L, n, waves, resets=None):
    """Pack the waves [(bits, nbytes)] on the host build and the restatement (resets: {wave: (streams, start)} before it);
    every pack and the final counters must agree.  Returns the restatement."""
    h, m = HostTx(L, n), PyTx(n)
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


def test_dtx_bad_and_empty_rows(L):
    cap = 64
    rows = [(0, 0), (-1, 8), (-32768, 5), (40, 3), (40, -1), (40, -32768), (40, 41), (65, 8), (32767, 8),
            (12, 12), (4, 4), (40, 8), (40, 4), (64, 8)]
    bits = np.random.Generator(np.random.PCG64(1)).integers(0, 256, (len(rows), cap), dtype=np.uint8)
    nb = np.array(rows, np.int16)
    m = run_both(L, len(rows), [(bits, nb)] * 3)
    cnt = m.stats()
    assert list(cnt[:3, DTX]) == [3] * 3 and list(cnt[3:9, BAD]) == [3] * 6 and (cnt[9:, SENT] == 3).all()
    payload, ents = m.pack(bits, nb)
    assert [e[2] for e in ents if e[0] in (9, 10)] == [2, 2]               # description 1 empty: not emitted
    assert all(e[1] == 3 for e in ents)                                     # every row's index advanced three times


@pytest.mark.parametrize("cfg", [dict(framesize_ms=40), dict(framesize_ms=20), dict(framesize_ms=40, joint_hb=1),
                                 dict(framesize_ms=40, dtx=1)])
def test_host_encoder_rows(L, sim, cfg):
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
    m = run_both(L, n, waves)
    assert m.cnt[:, BAD].sum() == 0 and m.cnt[:, SENT].sum() + m.cnt[:, DTX].sum() == n * P


def test_index_wrap_and_reset(L):
    rng = np.random.Generator(np.random.PCG64(2))
    n = 5
    waves = [random_rows(rng, n, 128) for _ in range(8)]
    resets = {0: ([0, 3], [M32 - 2, M32 - 1]), 4: ([3, 1], [7, M32 - 3]), 6: ([], [])}
    m = run_both(L, n, waves, resets)
    assert m.next[0] == 6 and m.next[3] == 11 and m.next[1] == 1


def test_octet_counter_wrap(L):
    """The octet counter is mod 2^32: start both just below it."""
    rng = np.random.Generator(np.random.PCG64(3))
    n = 4
    h, m = HostTx(L, n), PyTx(n)
    h.cnt[:, OCTETS] = M32 - 100
    m.cnt[:, OCTETS] = M32 - 100
    for _ in range(3):
        bits, nb = random_rows(rng, n, 128, dtx=0, bad=0)
        check_same(h.pack(bits, nb), m.pack(bits, nb))
    assert np.array_equal(h.stats(), m.stats()) and (m.cnt[:, OCTETS] > M32).all()


def test_single_stream(L):
    rng = np.random.Generator(np.random.PCG64(4))
    run_both(L, 1, [random_rows(rng, 1, 64, dtx=0.3, bad=0.3) for _ in range(40)])


@pytest.mark.parametrize("n,cap", [(37, 128), (600, 256), (1031, 144)])
def test_random_rows(L, n, cap):
    rng = np.random.Generator(np.random.PCG64(n + cap))
    waves = [random_rows(rng, n, cap) for _ in range(5)]
    st = rng.choice(n, n // 8, replace=False)
    m = run_both(L, n, waves, {3: (st, rng.integers(0, M32, len(st)))})
    tot = m.cnt.sum(0)
    assert tot[SENT] > 0 and tot[DTX] > 0 and tot[BAD] > 0


# ---- the contributor lists ----------------------------------------------------------------------------------------------
def select_talkers(room_start, members, level, flags, k, n):
    """The mixer's talkers of each room (include/solo_b200.h: the up-to-k eligible members with the smallest
    (level, index)), padded with -1."""
    R = len(room_start) - 1
    tk = np.full((R, k), -1, np.int32)
    for r in range(R):
        c = sorted((int(level[j]), int(j)) for j in members[room_start[r]:room_start[r + 1]] if 0 <= j < n and flags[j] & 3)
        for t, (_, j) in enumerate(c[:k]):
            tk[r, t] = j
    return tk


def contributors_literal(room_start, members, R, k, talkers, level, n):
    """INTEGRATION.md's loop, with the CSRC list kept as stream indices and the header extension bytes as levels."""
    csrc = np.full((n, k), -1, np.int32)
    lvl = np.full((n, k), 127, np.uint8)
    talkers = talkers.ravel()
    for r in range(R):
        for m in range(room_start[r], room_start[r + 1]):
            i, cc = int(members[m]), 0
            if not 0 <= i < n:
                continue
            t = 0
            while t < k and talkers[r * k + t] >= 0:
                j = int(talkers[r * k + t])
                t += 1
                if j == i:
                    continue
                csrc[i, cc] = j
                lvl[i, cc] = level[j] & 0x7F
                cc += 1
    return csrc, lvl


def layout(rng, n, sizes, out_of_range=0):
    """CSR rooms of the given sizes over a random permutation of [0, n) (the rest in no room), with `out_of_range`
    members replaced by -1 or n."""
    perm = rng.permutation(n)
    assert sum(sizes) <= n
    room_start = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    members = perm[:sum(sizes)].astype(np.int32)
    if out_of_range:
        at = rng.choice(len(members), out_of_range, replace=False)
        members[at] = rng.choice([-1, n, 1 << 30], out_of_range)
    return room_start, members


def model_contributors(L, room_start, members, k, talkers, level, n):
    csrc, lvl = np.zeros((n, k), np.int32), np.zeros((n, k), np.uint8)
    rs, mb, tk, lv = (np.ascontiguousarray(x, t) for x, t in ((room_start, np.int32), (members, np.int32),
                                                                 (talkers, np.int32), (level, np.uint8)))
    L.tx_model_contributors(rs.ctypes.data, mb.ctypes.data, len(rs) - 1, k, tk.ctypes.data, lv.ctypes.data, n,
                            csrc.ctypes.data, lvl.ctypes.data)
    return csrc, lvl


LAYOUTS = {"ones": [1] * 40, "fours": [4] * 60, "big": [256, 256], "mixed": [1, 4, 256, 4, 1, 0, 17, 4],
           "none": []}


@pytest.mark.parametrize("name", sorted(LAYOUTS))
@pytest.mark.parametrize("k", range(1, 9))
def test_contributors_equal_literal_loop(L, name, k):
    rng = np.random.Generator(np.random.PCG64(k * 100 + len(name)))
    n = 600
    room_start, members = layout(rng, n, LAYOUTS[name], out_of_range=3 if name == "mixed" else 0)
    level = rng.integers(0, 256, n).astype(np.uint8)                # bit 7 set on some: the & 0x7f
    flags = np.where(rng.random(n) < (0.15 if k > 4 else 0.6), rng.integers(1, 16, n), 0).astype(np.uint8)
    tk = select_talkers(room_start, members, level, flags, k, n)
    got = model_contributors(L, room_start, members, k, tk, level, n)
    want = contributors_literal(room_start, members, len(room_start) - 1, k, tk, level, n)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    in_room = np.zeros(n, bool)
    in_room[members[(members >= 0) & (members < n)]] = True
    assert (got[0][~in_room] == -1).all() and (got[1][~in_room] == 127).all()
    if name in ("ones", "fours", "mixed") and k > 1:
        assert ((tk < 0).sum(1) > 0).any()                              # some room has fewer talkers than k
