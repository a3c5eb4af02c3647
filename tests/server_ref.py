"""What the server-side tests compare against and drive: independent restatements of the mixer, the receive queue with
its timing and the send queue (include/solo_b200.h), the seeded traffic the tests and tools feed them, and adapters that
drive the queues through their device and host entry points (torch is imported only by those)."""
import numpy as np

from tests.util import load_golden

M32 = 1 << 32
STORED, DUPLICATE, LATE, DROPPED, MALFORMED, PLAYED_BOTH, PLAYED_ONE, PLAYED_NONE = range(8)   # RX_COUNTERS
SENT, OCTETS, DTX, BAD = range(4)                                                                # TX_COUNTERS
POISON = -21846                                 # 0xAAAA: rows of streams in no room must keep it


# ---- the receive queue, restated --------------------------------------------------------------------------------------
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


def replay(impl, ops):
    """Apply ops to a queue (a timed insert when the op carries receive times); returns its pull results."""
    pulls = []
    for op in ops:
        if op[0] == "insert":
            impl.insert(*op[1:])
        elif op[0] == "reset":
            impl.reset(op[1], op[2])
        else:
            pulls.append(impl.pull(op[1]))
    return pulls


def check_pull(got, want):
    """A queue's pull (bits, nbytes, lostflag) against PyRx's (rows, nbytes, lostflag): rows up to nbytes[0]."""
    bits, nb, lf = got
    rows, wnb, wlf = want
    assert np.array_equal(nb, wnb) and np.array_equal(lf, wlf)
    for s, row in enumerate(rows):
        assert bytes(bits[s, :len(row)]) == row, s


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


# ---- the send queue and the contributor lists, restated ----------------------------------------------------------------
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


# ---- the mixer, restated -----------------------------------------------------------------------------------------------
def csr(rooms):
    room_start = np.zeros(len(rooms) + 1, np.int32)
    room_start[1:] = np.cumsum([len(r) for r in rooms])
    members = np.concatenate([np.asarray(r, np.int32) for r in rooms] + [np.zeros(0, np.int32)])
    return room_start, members


def numpy_mix(pcm, level, flags, rooms, k, out):
    """The rule of include/solo_b200.h, restated: sort each room's eligible members by (level, index), keep k, and give
    every member the clamped int32 sum of the kept rows minus its own."""
    talkers = np.full((len(rooms), k), -1, np.int32)
    for r, mem in enumerate(rooms):
        el = sorted((int(level[j]), int(j)) for j in mem if flags[j] & 3)[:k]
        t = [j for _, j in el]
        talkers[r, :len(t)] = t
        total = pcm[t].astype(np.int32).sum(0) if t else np.zeros(pcm.shape[1], np.int32)
        for i in mem:
            own = pcm[i].astype(np.int32) if int(i) in t else 0
            out[i] = np.clip(total - own, -32768, 32767).astype(np.int16)
    return out, talkers


# ---- seeded traffic ----------------------------------------------------------------------------------------------------
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


def rx_time_traffic(N, rng):
    """tools/rx_time.py's tick: both descriptions of every stream's golden-sized packet (stream s sends packet s mod 191),
    1 % of them sent twice, a fixed 10 % of the (stream, description) pairs one tick early (a duplicate as early as its
    original), shuffled.  Returns (stream, desc, lens, payload, off, early)."""
    g = load_golden()
    P = g["fix_nbytes"].shape[0]
    s = np.repeat(np.arange(N, dtype=np.int32), 2)
    d = np.tile(np.array([1, 2], np.uint8), N)
    p = s % P
    n0, n1 = g["fix_nbytes"][p, 0].astype(np.int32), g["fix_nbytes"][p, 1].astype(np.int32)
    lens = np.where(d == 1, n0 - n1, n1).astype(np.int32)
    src = np.where(d == 1, 0, n0 - n1)                          # the description's first byte in its packet row
    dup = rng.choice(2 * N, 2 * N // 100, replace=False)
    s, d, lens, src, p = (np.concatenate([x, x[dup]]) for x in (s, d, lens, src, p))
    early = rng.random(2 * N) < 0.10
    early = np.concatenate([early, early[dup]])
    order = rng.permutation(len(s))
    s, d, lens, src, p, early = (x[order] for x in (s, d, lens, src, p, early))
    off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int32)
    bits = g["fix_bits"]                                        # read from the archive once, not per description
    payload = np.concatenate([bits[pi, si:si + li] for pi, si, li in zip(p, src, lens)]).astype(np.uint8)
    return s, d, lens, payload, off, early.astype(np.int64)


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


def shuffled_rooms(k, rng, sizes=None, spare=40):
    """Rooms of the given sizes (default 0, 1, 2, k, k + 1, 33, 1000) over a random permutation of the streams, in shuffled
    room order, and `spare` streams in no room; returns (n, rooms)."""
    sizes = list(sizes if sizes is not None else (0, 1, 2, k, k + 1, 33, 1000))
    rng.shuffle(sizes)
    n = sum(sizes) + spare
    perm = rng.permutation(n).astype(np.int32)
    rooms, o = [], 0
    for s in sizes:
        rooms.append(perm[o:o + s])
        o += s
    return n, rooms


def csr_rooms(rng, n, sizes, out_of_range=0):
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


def mixed_layout(n=65536, seed=1):
    """8 192 rooms of 4, 64 rooms of 256 and one room of 12 000 over a permutation of the streams; 4 384 in no room."""
    perm = np.random.Generator(np.random.PCG64(seed)).permutation(n).astype(np.int32)
    sizes = [4] * 8192 + [256] * 64 + [12000]
    rooms, o = [], 0
    for s in sizes:
        rooms.append(perm[o:o + s])
        o += s
    assert n - o == 4384
    return rooms, perm[o:]


# ---- the queues through their device and host entry points (GPU tests) -------------------------------------------------
def to_dev(a):
    """A host array on cuda:0 (uint32 as int32 of the same bits)."""
    import torch
    a = np.array(a)
    if a.dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(a).to(torch.device("cuda", 0))


class DeviceForm:
    """RxQueue driven through insert_device / pull_device on the current torch stream; an insert with receive times is a
    timed insert."""

    def __init__(self, sb, n, depth, desc_cap):
        self.q, self.n, self.cap = sb.RxQueue(n, depth, desc_cap), n, 2 * desc_cap

    def insert(self, stream, index, desc, off, lens, payload, arrival=None):
        import torch
        a = [to_dev(x) for x in (stream, index, desc, off, lens, payload)]
        da = to_dev(arrival) if arrival is not None else None
        self.q.insert_device(*(x.data_ptr() for x in a[:5]), len(stream), a[5].data_ptr(), payload.size,
                             torch.cuda.current_stream().cuda_stream, d_arrival=da.data_ptr() if da is not None else None)
        torch.cuda.synchronize()

    def pull(self, play=None):
        import torch
        d_bits = torch.zeros((self.n, self.cap), dtype=torch.uint8, device="cuda")
        d_nb = torch.zeros((self.n, 2), dtype=torch.int16, device="cuda")
        d_lf = torch.zeros(self.n, dtype=torch.int32, device="cuda")
        d_play = to_dev(np.asarray(play, np.uint32)) if play is not None else None
        self.q.pull_device(d_play.data_ptr() if d_play is not None else 0, d_bits.data_ptr(), self.cap, d_nb.data_ptr(),
                           d_lf.data_ptr(), torch.cuda.current_stream().cuda_stream)
        return d_bits.cpu().numpy(), d_nb.cpu().numpy(), d_lf.cpu().numpy()

    def reset(self, streams, start):
        self.q.reset(streams, start)

    def stats(self):
        import torch
        torch.cuda.synchronize()
        return self.q.stats()

    def enable_timing(self, ts_per_index, max_arrivals):
        self.q.enable_timing(ts_per_index, max_arrivals)

    def timing(self):
        import torch
        torch.cuda.synchronize()
        return self.q.timing()

    def close(self):
        self.q.close()


class HostForm(DeviceForm):
    """The same through solo_b200_rx_insert_host / insert_timed_host (raw arrays, so malformed offsets reach them) and
    pull_host."""

    def insert(self, stream, index, desc, off, lens, payload, arrival=None):
        from solo_b200.api import lib
        a = [np.ascontiguousarray(x) for x in (stream, index, desc, off, lens, payload)]
        if arrival is None:
            r = lib().solo_b200_rx_insert_host(self.q.h, *(x.ctypes.data for x in a[:5]), len(stream), a[5].ctypes.data,
                                               a[5].size)
        else:
            ar = np.ascontiguousarray(arrival, np.uint32)
            r = lib().solo_b200_rx_insert_timed_host(self.q.h, *(x.ctypes.data for x in a[:5]), ar.ctypes.data, len(stream),
                                                     a[5].ctypes.data, a[5].size)
        assert r == 0

    def pull(self, play=None):
        return self.q.pull(play, cap=self.cap)


class DevicePack:
    """TxQueue driven through pack_device on torch buffers, on the current torch stream."""

    def __init__(self, sb, n):
        import torch
        self.q, self.n = sb.TxQueue(n), n
        self.ent = [torch.zeros(2 * n, dtype=t, device="cuda") for t in (torch.int32, torch.int32, torch.uint8, torch.int32,
                                                                          torch.int32)]
        self.ct = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.tot = torch.zeros(1, dtype=torch.int64, device="cuda")

    def pack(self, bits, nbytes):
        import torch
        d_bits, d_nb = to_dev(bits), to_dev(nbytes)
        cap = bits.shape[1]
        d_pay = torch.full((self.n * cap,), 0xA5, dtype=torch.uint8, device="cuda")
        self.q.pack_device(d_bits.data_ptr(), cap, d_nb.data_ptr(), d_pay.data_ptr(), d_pay.numel(),
                           *(x.data_ptr() for x in self.ent), self.ct.data_ptr(), self.tot.data_ptr(),
                           torch.cuda.current_stream().cuda_stream)
        c, t = int(self.ct.item()), int(self.tot.item())
        st, ix, de, of, ln = (x[:c].cpu().numpy() for x in self.ent)
        return bytes(d_pay[:t].cpu().numpy()), list(zip(st.tolist(), (ix.view(np.uint32)).tolist(), de.tolist(), of.tolist(),
                                                       ln.tolist()))

    def reset(self, streams, start):
        self.q.reset(streams, start)

    def stats(self):
        import torch
        torch.cuda.synchronize()
        return self.q.stats()


class HostPack(DevicePack):
    def pack(self, bits, nbytes):
        payload, st, ix, de, of, ln = self.q.pack(bits, nbytes)
        return bytes(payload), list(zip(st.tolist(), ix.tolist(), de.tolist(), of.tolist(), ln.tolist()))
