"""Drivers of the parity tests.

lockstep runs two per-stream codecs side by side: the host model of the kernels, the drop-in handles or the reference.
RefRows runs the reference per checked row beside a batch.  DeviceDecoder drives a decoder batch through its device entry
points, and DevicePath an encoder batch and its decoder batch.
The fixtures sb, ref and sim are imported by the test modules that use them.
Bar: payloads and both length fields byte-identical; return values 0; PCM within PCM_TOL."""
import collections
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from tests.util import receive

PCM_TOL = 0                             # LSB; the north star allows 1
COMPARED = collections.Counter()        # payload rows and PCM rows the drivers have compared, to check how far a test reaches


@pytest.fixture(scope="module")
def sb():
    import solo_b200
    solo_b200.lib()
    return solo_b200


@pytest.fixture(scope="module")
def ref():
    from oracle import ref as r
    if not r.available():
        pytest.skip("oracle/_ref not built")
    r.lib("fix"), r.lib("flp")          # loaded once, before thread pools drive the reference
    return r


@pytest.fixture(scope="module")
def sim():
    from tests.hostsim import sim as s
    s.lib()
    return s


def control_args(rate, dtx, loss):
    """set_control keyword arguments of one stream's settings, -1 = unchanged."""
    return {k: int(v) for k, v in (("rate", rate), ("dtx", dtx), ("loss", loss)) if v != -1}


def ref_and_model(ref, sim, **cfg):
    """(FIX encoder, FLP decoder) of the reference and (encoder, decoder) of the host model, of one configuration."""
    dcfg = {k: v for k, v in cfg.items() if k not in ("rate", "dtx")}
    return (ref.RefEncoder("fix", **cfg), ref.RefDecoder("flp", **dcfg)), (sim.SimEncoder(**cfg), sim.SimDecoder(**dcfg))


def lockstep(a, b, x, flags=None, control=None, tag=()):
    """a, b: (encoder, decoder) pairs; x: int16 [packets, samples].  Per packet p, control[p] (set_control arguments, if
    given) goes to both encoders, and both encode x[p]: (payload, length fields, return value) must be equal.  With flags,
    both decoders decode what the receiver makes of the packet under flags[p]: both return 0, and their PCM has x[p]'s
    length and differs by at most PCM_TOL.  Closes all four; returns a's packets."""
    (ea, da), (eb, db) = a, b
    out = []
    for p in range(len(x)):
        if control is not None and control[p]:
            ea.set_control(**control[p])
            eb.set_control(**control[p])
        pk = ea.encode(x[p])
        assert pk == eb.encode(x[p]), ("payload", p) + tuple(tag)
        COMPARED["payload"] += 1
        out.append(pk)
        if flags is not None:
            rx = receive(pk[0], pk[1], flags[p])
            (ya, ra), (yb, rb) = da.decode(*rx), db.decode(*rx)
            assert ra == rb == 0 and ya.shape == yb.shape == (len(x[p]),), ("decoder", p, ra, rb) + tuple(tag)
            assert np.abs(ya.astype(np.int32) - yb.astype(np.int32)).max() <= PCM_TOL, ("pcm", p, rx[2]) + tuple(tag)
            COMPARED["pcm"] += 1
    for o in (ea, da, eb, db):
        if o is not None:
            o.close()
    return out


def batch_packets(bits, nb):
    """A batch's rows as (payload, (n0, n1)) packets."""
    return [(bytes(bits[i, :max(int(nb[i, 0]), 0)]), (int(nb[i, 0]), int(nb[i, 1]))) for i in range(len(nb))]


def batch_rows(rx, cap):
    """(payload, nbytes, lostflag) triples as a batch decoder's input: payloads uint8 [rows, cap] (a payload longer than cap
    cut to it), nbytes int16 [rows, 2], lostflags int32 [rows]."""
    tb, tnb, tf = np.zeros((len(rx), cap), np.uint8), np.zeros((len(rx), 2), np.int16), np.zeros(len(rx), np.int32)
    for i, (b, tnb[i], tf[i]) in enumerate(rx):
        tb[i, :min(len(b), cap)] = np.frombuffer(b, np.uint8)[:cap]
    return tb, tnb, tf


def received(packets, flags, cap):
    """What the receiver hands a batch decoder: `receive` of each (payload, (n0, n1)) packet under its lostflag, as
    batch_rows."""
    return batch_rows([receive(b, nb, f) for (b, nb), f in zip(packets, flags)], cap)


class RefRows:
    """The reference beside a batch: a FIX encoder for each checked row (rows: batch indices) and, when decode is "ref" or
    "gpu", an FLP decoder for each of pcm_rows (a subset of rows, all of them by default), all made from one configuration
    (rate, dtx, use_md_index, framesize_ms, joint_hb).  They advance one packet per step(), on a thread pool (the reference
    is plain C behind ctypes, which releases the GIL).  decode="ref": each decoder gets what the receiver makes of the
    reference's own payload; decode="gpu": of the batch's payload."""

    def __init__(self, ref, rows, decode=None, pcm_rows=None, **cfg):
        self.rows = list(rows)
        self.enc = [ref.RefEncoder("fix", **cfg) for _ in self.rows]
        pos = {s: i for i, s in enumerate(self.rows)}
        self.pcm_rows = self.rows if pcm_rows is None else list(pcm_rows)
        self.pcm_pos = [pos[s] for s in self.pcm_rows]
        dcfg = {k: v for k, v in cfg.items() if k not in ("rate", "dtx")}
        self.dec = [ref.RefDecoder("flp", **dcfg) for _ in self.pcm_rows] if decode else []
        self.decode = decode
        self.pool = ThreadPoolExecutor(32)
        self.p = -1
        self.dtx_rows = 0           # (row, packet) pairs the reference encoder sent nothing for

    def step(self, x, bits, nb, flags=None, control=None):
        """One packet.  x, bits, nb: the checked rows' input and the batch's payloads and length fields (row i is rows[i]);
        control: (rate, dtx, loss) arrays over rows for set_control first, -1 = unchanged.  Checks the length fields and
        payload bytes; with decoders, decodes under flags (over pcm_rows) and returns the received (payloads, nbytes,
        lostflags) of pcm_rows for the batch decoder."""
        self.p += 1

        def encode(i):
            c = {} if control is None else control_args(*(v[i] for v in control))
            if c:
                self.enc[i].set_control(**c)
            return self.enc[i].encode(x[i])

        self.packets = list(self.pool.map(encode, range(len(self.rows))))
        for i, (b, rnb, n) in enumerate(self.packets):
            assert tuple(nb[i]) == rnb and bytes(bits[i, :max(n, 0)]) == b, ("payload", self.p, self.rows[i])
            self.dtx_rows += rnb[0] <= 0
        COMPARED["payload"] += len(self.packets)
        if not self.dec:
            return None
        src = self.packets if self.decode == "ref" else batch_packets(bits, nb)
        tb, tnb, tf = rx = received([src[i][:2] for i in self.pcm_pos], flags, bits.shape[1])
        self.want = list(self.pool.map(lambda k: self.dec[k].decode(bytes(tb[k, :tnb[k, 0]]), tuple(tnb[k]), int(tf[k])),
                                       range(len(tf))))
        assert all(r == 0 for _, r in self.want), ("reference decoder", self.p)
        return rx

    def check_pcm(self, pcm):
        """pcm: the batch's decoded rows of pcm_rows for the last step, within PCM_TOL of the reference's."""
        want = np.stack([y for y, _ in self.want])
        assert pcm.shape == want.shape, (pcm.shape, want.shape)
        d = np.abs(pcm.astype(np.int32) - want.astype(np.int32)).max(axis=1)
        assert d.max() <= PCM_TOL, ("pcm", self.p, self.pcm_rows[int(d.argmax())], int(d.max()))
        COMPARED["pcm"] += len(want)

    def close(self):
        for o in self.enc + self.dec:
            o.close()
        self.pool.shutdown()


class DeviceDecoder:
    """A decoder batch through decode_device and activity_device on torch buffers of its own (cuda:0), in order on `stream`
    (default: the current stream).  Same call shapes as the batch's host calls, decode and activity.  pcm: a cuda:0 int16
    tensor [N, samples] to decode into instead of its own (a view at any offset, to place the rows)."""

    def __init__(self, db, cap=256, stream=None, pcm=None):
        import torch
        self.torch, self.db, self.cap = torch, db, cap
        self.stream = torch.cuda.current_stream() if stream is None else stream
        N, dev = db.n, torch.device("cuda", 0)
        self.tb, self.tnb = torch.zeros((N, cap), dtype=torch.uint8, device=dev), torch.zeros((N, 2), dtype=torch.int16, device=dev)
        self.flags, self.ret = torch.zeros(N, dtype=torch.int32, device=dev), torch.full((N,), -99, dtype=torch.int32, device=dev)
        self.pcm = torch.zeros((N, db.samples), dtype=torch.int16, device=dev) if pcm is None else pcm
        assert self.pcm.shape == (N, db.samples) and self.pcm.is_contiguous()
        self.level, self.vad = torch.zeros(N, dtype=torch.uint8, device=dev), torch.zeros(N, dtype=torch.uint8, device=dev)

    def decode(self, tb=None, tnb=None, tf=None, rows=None, check=True):
        """Decode payloads [N, cap], nbytes [N, 2] and lostflags [N]: host arrays or cuda:0 tensors, each copied into the
        decoder's input buffer on the device, where a leading dimension of 1 is broadcast over the batch; None decodes what
        that buffer holds.  check: every row must return 0.  Returns (pcm, ret) of rows (all rows by default) as host
        arrays."""
        torch = self.torch
        with torch.cuda.stream(self.stream):
            for buf, a in ((self.tb, tb), (self.tnb, tnb), (self.flags, tf)):
                if a is not None:
                    buf.copy_(torch.as_tensor(np.ascontiguousarray(a) if isinstance(a, np.ndarray) else a).to(buf.device))
            self.db.decode_device(self.pcm.data_ptr(), self.tb.data_ptr(), self.cap, self.tnb.data_ptr(), self.flags.data_ptr(),
                                  self.ret.data_ptr(), self.stream.cuda_stream)
        self.stream.synchronize()
        assert not check or int((self.ret != 0).sum().item()) == 0, "decoder return"
        return self._rows(self.pcm, rows), self._rows(self.ret, rows)

    def activity(self, rows=None):
        """activity_device after the last decode: (level, flags) of rows (all rows by default) as host arrays."""
        with self.torch.cuda.stream(self.stream):
            self.db.activity_device(self.pcm.data_ptr(), self.level.data_ptr(), self.vad.data_ptr(), self.stream.cuda_stream)
        return self._rows(self.level, rows), self._rows(self.vad, rows)

    def _rows(self, t, rows):
        self.stream.synchronize()
        return (t if rows is None else t[self.torch.as_tensor(rows, dtype=self.torch.long, device=t.device)]).cpu().numpy()


class DevicePath:
    """A batch through its device entry points on torch buffers of its own (cuda:0), in order on `stream` (default: the
    current stream): set_control_device, encode_device, then apply_loss_device or host-made payloads, decode_device."""

    def __init__(self, sb, eb, db=None, cap=256, stream=None):
        import torch
        self.torch, self.sb, self.eb, self.cap = torch, sb, eb, cap
        self.stream = torch.cuda.current_stream() if stream is None else stream
        self.dec = DeviceDecoder(db, cap, self.stream) if db is not None else None
        N, S, dev = eb.n, eb.samples, torch.device("cuda", 0)
        self.x = torch.zeros((N, S), dtype=torch.int16, device=dev)
        self.bits, self.nb = torch.zeros((N, cap), dtype=torch.uint8, device=dev), torch.zeros((N, 2), dtype=torch.int16, device=dev)
        self.ctrl = torch.zeros((3, N), dtype=torch.int32, device=dev)

    def encode(self, x, control=None):
        """x: int16 [N, samples] host array.  control: (rate, dtx, loss) int32 arrays [N] for set_control_device first;
        None for one of them passes a NULL array."""
        torch, st = self.torch, self.stream.cuda_stream
        with torch.cuda.stream(self.stream):
            self.x.copy_(torch.from_numpy(x))
            if control is not None:
                ptr = []
                for k, v in enumerate(control):
                    if v is not None:
                        self.ctrl[k].copy_(torch.from_numpy(np.ascontiguousarray(v, np.int32)))
                    ptr.append(None if v is None else self.ctrl[k].data_ptr())
                self.eb.set_control_device(*ptr, st)
            self.eb.encode_device(self.x.data_ptr(), self.bits.data_ptr(), self.cap, self.nb.data_ptr(), st)

    def decode(self, flags, rx=None):
        """Decode under lostflags [N]: the encoded payloads trimmed on the device (apply_loss_device), or rx = (payloads,
        nbytes) made on the host.  Every row must return 0."""
        d = self.dec           # rows=[]: nothing comes back to the host here, rows() reads the PCM
        if rx is not None:
            d.decode(rx[0], rx[1], flags, rows=[])
            return
        with self.torch.cuda.stream(self.stream):
            d.flags.copy_(self.torch.from_numpy(np.ascontiguousarray(flags, np.int32)))
            self.sb.apply_loss_device(self.bits.data_ptr(), self.nb.data_ptr(), d.flags.data_ptr(), d.tb.data_ptr(),
                                      d.tnb.data_ptr(), self.cap, self.eb.n, self.stream.cuda_stream)
        d.decode(rows=[])

    def rows(self, idx=None):
        """(payloads, length fields, PCM -- None without a decoder batch) of rows idx (all rows by default) as host
        arrays."""
        self.stream.synchronize()
        if idx is None:
            return self.bits.cpu().numpy(), self.nb.cpu().numpy(), self.dec and self.dec.pcm.cpu().numpy()
        i = self.torch.tensor(idx, device=self.bits.device)
        return self.bits[i].cpu().numpy(), self.nb[i].cpu().numpy(), self.dec and self.dec.pcm[i].cpu().numpy()
