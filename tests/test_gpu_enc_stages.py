"""The voice-activity kernel and the high-band half of the entropy-coding kernel, run on the GPU stage by stage and compared
bit-exactly with the unmodified reference encoder.

The encoder tests see these stages only through payload bytes, where thresholds and quantisation hide errors: the VAD's band
qualities and tilt reach the bitstream only through later decisions, and the high-band gains only as 5-bit indices.  Here
the reference runs whole packets (oracle/enc_ref.c: AGR_Sate_Encoder_Encode on a real handle with the product's settings,
with linker taps on SKP_Silk_VAD_GetSA_Q8, the quantiser's excitation and the high-band LSP index, excitation and gain
quantiser), and the device code runs in its product kernel's launch layout (tests/gpu_ops/ops.cu):
  * vad_packet (sb_enc_vad_kernel's layout), from the reference's own VAD state at the reset, mid-stream and around the
    noise estimator's 1000-frame ramp, on the reference's low-band frames: every frame's speech activity, band qualities,
    tilt and state;
  * enc_store_high_band (the last step of sb_enc_finish_kernel, in its two-threads-per-stream mapping): gains, their
    32-level VQ and bit packing, on the reference's LSP indices, high-band energies and quantiser excitation of every
    packet, compared with the high-band bytes of the reference's payload.  The low-band length it stores behind is the
    reference's own, so its length fields are checked only as assembled from that; the description coding, the pairing
    and shuffles of the finish kernel and the drop / reject decision are not covered here;
  * the gain VQ over every int16 gain, against AGR_Sate_gain_quant_highband_fix, ties and wrapped distances included.
An unmarked test runs the host model's functions of these stages against the same records, and another checks, on the
reference alone, that the case table reaches each regime it is built for."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.util import load_clip

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS_LIB = os.path.join(ROOT, "tests", "_gpu_ops", "libsb_gpu_ops.so")
FRAME, NV, CAP = 160, 28, 1024
I16 = 1 << 16


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _ok(r):
    assert r == 0, "CUDA harness call failed with error %d" % r


def w32(x):
    return ((int(x) + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def sqrt_approx(x):
    from tests.test_gpu_ops import sqrt_approx as f
    return f(x)


def _first_diff(what, got, want):
    got, want = np.asarray(got), np.asarray(want)
    bad = np.argwhere(got != want)
    if len(bad):
        i = tuple(int(v) for v in bad[0])
        raise AssertionError("%s: %d elements differ, first at element %s: got %s, reference %s"
                             % (what, len(bad), i, got[i], want[i]))


# ---------------------------------------------------------------------------------------------------------------------
# cases: signals x settings
# ---------------------------------------------------------------------------------------------------------------------
def _tone(f_hz, n, amp=12000, phase=0.3):
    return amp * np.sin(2 * np.pi * f_hz / 16000 * np.arange(n) + phase)


def signal(kind, n, rng):
    t = np.arange(n)
    if kind == "speech":
        return np.resize(load_clip(), n)
    if kind == "hb_sine":                    # a 6 kHz sine: energy only above 4 kHz, a near-silent low band
        return _tone(6000, n, 20000)
    if kind == "hb_noise":                   # noise shifted to 4-8 kHz by (-1)^n modulation of low-passed noise
        lo = np.convolve(rng.normal(0, 9000, n + 15), np.ones(16) / 4, "valid")[:n]
        return lo * np.where(t % 2 == 0, 1, -1)
    if kind.startswith("tone"):              # one tone in each VAD band of the 8 kHz low band
        return _tone(int(kind[4:]), n)
    if kind == "step":                       # silence, then a full-scale square at 1 kHz
        return np.where(t < n // 2, 0, np.where((t // 8) % 2 == 0, 32767, -32768))
    if kind == "square":
        return np.where((t // 16) % 2 == 0, 32767, -32767)
    if kind == "lsb":
        return rng.integers(-1, 2, n)
    if kind == "late_onset":                 # quiet noise, then speech from the frame before the VAD counter reaches 1000
        x = np.resize(load_clip(), n).astype(np.float64)
        x[:984 * 320] = rng.integers(-2, 3, 984 * 320)
        return x
    if kind == "dtx":                        # talk spurts between silences long enough for DTX entry and its re-sends
        x = np.resize(load_clip(), n).astype(np.float64)
        x[n // 8: 7 * n // 8] = rng.integers(-2, 3, 6 * n // 8)
        return x
    raise ValueError(kind)


# name, signal, packets, settings (rate, dtx, framesize_ms, joint, mdi, loss)
CASES = [
    ("speech/6k", "speech", 60, (6000, 0, 40, 0, 0, 0)),
    ("speech/13k6/20ms/mdi", "speech", 80, (13600, 0, 20, 0, 1, 0)),
    ("speech/24k/joint/loss10", "speech", 60, (24000, 0, 40, 1, 0, 10)),
    ("speech/100k/loss100", "speech", 60, (100000, 0, 40, 0, 1, 100)),
    ("hb_sine", "hb_sine", 30, (13600, 0, 40, 0, 0, 0)),
    ("hb_sine/joint", "hb_sine", 30, (13600, 0, 40, 1, 0, 0)),
    ("hb_noise/20ms", "hb_noise", 40, (24000, 0, 20, 0, 0, 10)),
    ("hb_noise/joint", "hb_noise", 30, (13600, 0, 40, 1, 1, 0)),
    ("tone250/20ms", "tone250", 40, (13600, 0, 20, 0, 0, 0)),
    ("tone750/mdi", "tone750", 30, (13600, 0, 40, 0, 1, 0)),
    ("tone1500/joint", "tone1500", 30, (24000, 0, 40, 1, 0, 0)),
    ("tone3000/loss10", "tone3000", 30, (13600, 0, 40, 0, 0, 10)),
    ("step/20ms", "step", 40, (13600, 0, 20, 0, 0, 0)),
    ("square", "square", 30, (24000, 0, 40, 0, 0, 0)),
    ("lsb/joint/mdi", "lsb", 30, (13600, 0, 40, 1, 1, 0)),
    ("dtx", "dtx", 120, (13600, 1, 40, 0, 0, 0)),
    ("dtx/20ms", "dtx", 160, (13600, 1, 20, 0, 1, 0)),
    ("onset/long", "late_onset", 520, (13600, 0, 40, 0, 0, 0)),  # 1040 frames: the VAD's noise-estimator ramp ends
]
# first packet of each VAD run: the reset state, mid-stream, and for the long case one run across the ramp's end and one
# after it (the VAD counter starts at 15 and counts frames, so packet p of a 40 ms stream starts at 15 + 2 p: 987 and 1007).
# The long case's speech starts one frame before the counter reaches 1000, so the band energies jump past the noise levels
# in the frame whose update is the first without the ramp's floor on its smoothing coefficient.
VAD_RUN = 12


def vad_starts(name, npk):
    return [0, npk // 2] + ([486, 496] if name == "onset/long" else [])


class Ref:
    def __init__(self):
        from oracle import enc_ref, ref
        if not ref.available() or not enc_ref.available():
            pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
        self.enc = enc_ref.RefEnc()
        self.fix = ref.lib("fix").lib
        self.fix.AGR_Sate_gain_quant_highband_fix.restype = C.c_int32
        self.fix.AGR_Sate_gain_quant_highband_fix.argtypes = [C.c_int16, C.c_void_p, C.c_int32]
        self.gain_cb = np.ctypeslib.as_array((C.c_int16 * 32).in_dll(self.fix, "AGR_Sate_highband_gain_cdbk_fix")).copy()
        self.recs = {}
        for i, (name, kind, npk, st) in enumerate(CASES):
            L = 16 * st[2]
            x = np.clip(np.round(signal(kind, npk * L, np.random.default_rng(100 + i))), -32768, 32767).astype(np.int16)
            self.recs[name] = self.enc.run(x.reshape(npk, L), *st)

    def gain_index(self, gain):
        return self.fix.AGR_Sate_gain_quant_highband_fix(int(gain), _p(self.gain_cb), 32)


@pytest.fixture(scope="module")
def ref():
    return Ref()


@pytest.fixture(scope="module")
def ops():
    if not os.path.exists(OPS_LIB):
        pytest.fail(OPS_LIB + " missing: __graft_entry__.build() builds it")
    return C.CDLL(OPS_LIB)


@pytest.fixture(scope="module")
def host():
    from tests.hostsim import sim
    L = sim.lib()
    L.hs_vad_packet.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.hs_hb_store.argtypes = [C.c_void_p] * 5 + [C.c_int, C.c_void_p]
    return L


def nf_of(st):
    return 1 if st[2] == 20 else 2


def hb_frame_of(st):
    return 320 if st[3] else 160


# ---------------------------------------------------------------------------------------------------------------------
# voice activity
# ---------------------------------------------------------------------------------------------------------------------
def vad_runs(ref):
    """[(name, settings, first packet, packet records)]; neighbouring runs belong to different cases, and 20 ms and 40 ms
    streams alternate within a warp."""
    runs = []
    for name, _, npk, st in CASES:
        for p0 in vad_starts(name, npk):
            runs.append((name, st, p0, ref.recs[name][p0:p0 + VAD_RUN]))
    runs.sort(key=lambda r: r[2] % 7)
    assert len(runs) % 64, "the last block of the launch is partly empty"
    return runs


def check_vad(what, nf, rec, out, st_after):
    """out [npk][2][6] and st_after [npk][28] (device or host model) against the packets' records"""
    for p in range(len(rec)):
        for f in range(nf):
            where = "%s packet %d frame %d VAD" % (what, p, f)
            want = [rec["sa_Q8"][p, f]] + list(rec["quality_Q15"][p, f]) + [rec["tilt_Q15"][p, f]]
            _first_diff(where + " outputs (SA_Q8, quality_Q15[4], tilt_Q15)", out[p, f], want)
        _first_diff("%s packet %d VAD state after" % (what, p), st_after[p], rec["vad_after"][p, nf - 1])


def ref_vad_consistent(rec, nf):
    assert (rec["n_vad"] == nf).all()
    flat = rec["vad_before"][:, :nf].reshape(-1, NV), rec["vad_after"][:, :nf].reshape(-1, NV)
    _first_diff("reference: VAD state before a frame == after the previous one", flat[0][1:], flat[1][:-1])


@pytest.mark.gpu
def test_vad_against_reference(ops, ref):
    runs = vad_runs(ref)
    n, npk = len(runs), VAD_RUN
    nf = np.array([nf_of(st) for _, st, _, _ in runs], np.int32)
    st0 = np.stack([r["vad_before"][0, 0] for _, _, _, r in runs]).astype(np.int32)
    low = np.zeros((n, npk, 2, FRAME), np.int16)
    for i, (_, _, _, r) in enumerate(runs):
        low[i, :len(r)] = r["low"]
    out = np.zeros((n, npk, 2, 6), np.int32)
    st_after = np.zeros((n, npk, NV), np.int32)
    _ok(ops.sb_ops_vad(n, npk, _p(nf), _p(st0), _p(low), _p(out), _p(st_after)))
    for i, (name, st, p0, r) in enumerate(runs):
        ref_vad_consistent(r, nf[i])
        check_vad("%s from packet %d:" % (name, p0), nf[i], r, out[i, :len(r)], st_after[i, :len(r)])


# ---------------------------------------------------------------------------------------------------------------------
# high band of the payload
# ---------------------------------------------------------------------------------------------------------------------
def hb_inputs(rec, st):
    """one packet's inputs of enc_store_high_band from the reference's record: cfg, lsp_idx [2], nrg0 [2][4], r16 [2][FRAME]"""
    nf, F = nf_of(st), hb_frame_of(st)
    nhb, SF = nf * FRAME // F, F // 4
    nb0, nb1 = int(rec["nbytes"][0]), int(rec["nbytes"][1])
    lb = nb0 - 4 * nhb if nb0 else 0
    cfg = np.array([nf, F, lb, nb1 - 4 * nhb if nb0 else 0], np.int32)
    nrg0 = np.zeros((2, 4), np.int32)
    for k in range(nhb):
        for s in range(4):
            nrg0[k, s] = sqrt_approx(w32(int((rec["hb_exc"][k, s, :SF].astype(np.int64) ** 2).sum())))
    r16 = (rec["res_Q10"] >> 10).astype(np.int16)
    return cfg, rec["hb_lsp_idx"].astype(np.int32), nrg0, r16


def hb_packets(ref):
    """every packet of every case, as (name, settings, packet index, record), interleaved across cases"""
    out = []
    for name, _, npk, st in CASES:
        rec = ref.recs[name]
        nhb = nf_of(st) * FRAME // hb_frame_of(st)
        assert (rec["n_lsp"] == nhb).all() and (rec["n_gain"] == 4 * nhb).all() and (rec["n_res"] == nf_of(st)).all(), name
        out += [(name, st, p, rec[p]) for p in range(npk)]
    out.sort(key=lambda r: r[2])
    if len(out) % 2 == 0:                        # odd: the last block is partly filled
        out.append(out[0])
    return out


def check_hb(where, st, rec, bits, nb, total):
    """The high-band bytes are an independent check.  nBytesOut and the packet size follow from the reference's low-band
    length, which is an input here: they check only how enc_store_high_band adds the high-band bytes to it (and that a
    DTX-dropped packet's high band starts at offset 0)."""
    nhb = nf_of(st) * FRAME // hb_frame_of(st)
    lb = int(rec["nbytes"][0]) - 4 * nhb if rec["nbytes"][0] else 0
    _first_diff(where + " high-band bytes", bits[lb:lb + 4 * nhb], rec["payload"][lb:lb + 4 * nhb])
    _first_diff(where + " nBytesOut", nb, rec["nbytes"])
    assert total == rec["ret"], "%s: packet size %d, reference %d" % (where, total, rec["ret"])


@pytest.mark.gpu
def test_high_band_payload_against_reference(ops, ref):
    pk = hb_packets(ref)
    n = len(pk)
    ins = [hb_inputs(r, st) for _, st, _, r in pk]
    cfg, lsp, nrg0, r16 = (np.ascontiguousarray(np.stack([x[j] for x in ins])) for j in range(4))
    bits = np.zeros((n, CAP), np.uint8)
    nb = np.zeros((n, 2), np.int16)
    total = np.zeros((n, 2), np.int32)
    _ok(ops.sb_ops_hb_store(n, CAP, _p(cfg), _p(lsp), _p(nrg0), _p(r16), _p(bits), _p(nb), _p(total)))
    for i, (name, st, p, r) in enumerate(pk):
        where = "%s packet %d" % (name, p)
        check_hb(where, st, r, bits[i], nb[i], total[i, 0])
        assert total[i, 1] == total[i, 0], where + ": the two threads' packet sizes"
        lb = int(cfg[i, 2])
        assert (bits[i, :lb] == 0xA5).all(), where + ": bytes written over the descriptions"
        assert (bits[i, r["ret"]:] == 0xA5).all(), where + ": bytes written past the packet"


def sweep_inputs():
    """every int16 gain, eight per stream: nrg1 = sqrt_approx(15^2 + 4^2) = 15, so gain = (int16)(nrg0 + 1)"""
    g = np.arange(-32768, 32768)
    assert sqrt_approx(241) == 15
    n = len(g) // 8 + 1                          # odd: the last block is partly filled
    nrg0 = np.zeros((n, 2, 4), np.int32)
    nrg0.reshape(-1)[:len(g)] = (g % I16) - 1    # nrg0 + 1 in [0, 65535]: (int16) of it is g
    r16 = np.zeros((n, 2, FRAME), np.int16)
    r16[:, :, 0::40] = 15
    r16[:, :, 1::40] = 4
    cfg = np.tile(np.array([2, 160, 0, 0], np.int32), (n, 1))
    lsp = np.tile(np.array([0x5A5, 0xFFF], np.int32), (n, 1))
    return g, cfg, lsp, nrg0, r16


@pytest.mark.gpu
def test_gain_vq_every_gain(ops, ref):
    g, cfg, lsp, nrg0, r16 = sweep_inputs()
    n = len(cfg)
    bits = np.zeros((n, CAP), np.uint8)
    nb = np.zeros((n, 2), np.int16)
    total = np.zeros((n, 2), np.int32)
    _ok(ops.sb_ops_hb_store(n, CAP, _p(cfg), _p(lsp), _p(nrg0), _p(r16), _p(bits), _p(nb), _p(total)))
    w = bits[:, :8].reshape(n, 2, 4).astype(np.uint32)
    w = (w[..., 0] << 24) | (w[..., 1] << 16) | (w[..., 2] << 8) | w[..., 3]
    idx = np.stack([(w >> (15 - 5 * s)) & 31 for s in range(4)], -1).reshape(-1)[:len(g)]
    want = np.array([ref.gain_index(v) for v in g])
    bad = np.flatnonzero(idx != want)
    assert not len(bad), "gain VQ: %d gains differ, first gain %d: device index %d, reference %d" % (len(bad), g[bad[0]], idx[bad[0]], want[bad[0]])
    assert ((w >> 20) == lsp).all(), "gain sweep: LSP index field"


# ---------------------------------------------------------------------------------------------------------------------
# host model and regimes (no GPU)
# ---------------------------------------------------------------------------------------------------------------------
def test_host_model_stages_against_reference(ref, host):
    for name, st, p0, r in vad_runs(ref):
        nf = nf_of(st)
        ref_vad_consistent(r, nf)
        s = np.ascontiguousarray(r["vad_before"][0, 0]).astype(np.int32)
        out = np.zeros((len(r), 2, 6), np.int32)
        st_after = np.zeros((len(r), NV), np.int32)
        for p in range(len(r)):
            host.hs_vad_packet(_p(s), nf, _p(np.ascontiguousarray(r["low"][p])), _p(out[p]))
            st_after[p] = s
        check_vad("host model %s from packet %d:" % (name, p0), nf, r, out, st_after)
    for name, st, p, r in hb_packets(ref):
        cfg, lsp, nrg0, r16 = hb_inputs(r, st)
        bits = np.full(CAP, 0xA5, np.uint8)
        nb = np.zeros(2, np.int16)
        total = host.hs_hb_store(_p(cfg), _p(lsp), _p(nrg0), _p(r16), _p(bits), CAP, _p(nb))
        check_hb("host model %s packet %d" % (name, p), st, r, bits, nb, total)


def test_case_tables_reach_every_listed_regime(ref):
    """Counts, over the case table, of the regimes these tests exist for."""
    wrapped = 0
    for name, _, npk, st in CASES:
        rec = ref.recs[name]
        nhb, SF = nf_of(st) * FRAME // hb_frame_of(st), hb_frame_of(st) // 4
        for r in rec:
            _, _, nrg0, r16 = hb_inputs(r, st)
            flat = r16.reshape(-1)
            for k in range(nhb):
                for s in range(4):
                    e = flat[k * hb_frame_of(st) + s * SF:k * hb_frame_of(st) + (s + 1) * SF].astype(np.int64)
                    nrg1 = sqrt_approx(w32(int((e * e).sum())))
                    gain = w32((int(nrg0[k, s]) + 1) << 4) // (nrg1 + 1)
                    assert ((gain + 32768) % I16) - 32768 == r["hb_gain"][k, s], (name, "tapped gain")
                    wrapped += gain > 32767
    # a loud high band over a near-silent low band: the unquantised gain wraps in its int16 cast
    assert wrapped > 0, "no high-band gain wraps"
    # the sweep's gains: exact ties between two codebook entries (the VQ keeps the first), and wrapped differences
    g = np.arange(-32768, 32768)[:, None]
    t = ((g - ref.gain_cb.astype(np.int64)[None, :] + 32768) % I16) - 32768
    d = t * t
    assert (np.sum(d == d.min(1, keepdims=True), 1) > 1).sum() > 0, "no ties in the gain sweep"
    assert (np.abs(g - ref.gain_cb[None, :]) > 32767).any(), "no wrapped gain differences in the sweep"
    # the VAD runs: from the reset state, across the end of the noise estimator's ramp (counter 1000)
    runs = vad_runs(ref)
    c0 = [int(r["vad_before"][0, 0, NV - 2]) for _, _, _, r in runs]
    c1 = [int(r["vad_after"][-1, nf_of(st) - 1, NV - 2]) for _, st, _, r in runs]
    assert 15 in c0, "no VAD run from the reset state"
    assert any(a < 1000 <= b for a, b in zip(c0, c1)), "no VAD run across counter 1000"
    assert any(a >= 1000 for a in c0), "no VAD run entirely after the ramp"
    # DTX: entry, dropped packets and the re-send after MAX_CONSECUTIVE_DTX frames
    for name in ("dtx", "dtx/20ms"):
        rec = ref.recs[name]
        assert rec["in_dtx"].any(), (name, "DTX never entered")
        assert (rec["nbytes"][:, 0] == 0).any(), (name, "no DTX-dropped packet")
        resend = (rec["in_dtx"][:-1] == 1) & (rec["in_dtx"][1:] == 0) & (rec["no_speech_counter"][1:] > 0)
        assert resend.any(), (name, "no re-send inside a DTX period")
