"""The band-split, high-band analysis and synthesis filter-bank code of the codec's kernels, run on the GPU routine by routine
and compared bit-exactly with the unmodified reference.

The encoder and decoder tests see these kernels only through payload bytes and decoded PCM, where quantisation hides many
errors (a wrong tie-break or a wrong NLSF vector that lands on the same codebook index).  Here the device code runs in its
product kernel's launch layout (tests/gpu_ops/ops.cu, compiled with the library's flags) and every intermediate the reference
exposes is compared at 0 LSB:
  * high-band frames (c_hb_analyse_packet, sb_enc_hb_warp_kernel's layout) against the reference's AGR_Bwe_encode_frame_FIX
    on a real encoder handle (oracle/hb_ref.c, with linker taps on the LSP search, NLSF2A_stable and the analysis filter);
  * the LSP search alone (c_hb_lsp_quant) against AGR_Sate_lsp_quant_highband;
  * the synthesis filter bank (qmf_synth_group, qmf_synth_group_fix) against AGR_Sate_qmf_synth of the float and the
    fixed-point build, followed by the int16 conversion of AGR_BWE_decode_frame_FLP.c (the fixed-point build's filter bank
    saturates itself);
  * the band split (qmf_output_pair, sb_enc_qmf_kernel's staging) against AGR_Sate_qmf_decomp.
The unmarked test at the end runs the case tables through the reference alone and checks that each regime the tables are
built for is reached, so that a table cannot silently stop covering it."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.util import chirp, load_clip

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS_LIB = os.path.join(ROOT, "tests", "_gpu_ops", "libsb_gpu_ops.so")
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
ORDER, PACKET, SYN_N2MAX = 8, 640, 640
# (frame length, high-band samples per packet) of the three high-band settings: 40 ms packets, 20 ms packets, joint mode 1
SETTINGS = {"40ms": (160, 320), "20ms": (160, 160), "joint": (320, 320)}
WNF_Q32 = int(float(np.float32(2.5e-5)) * 2.0 ** 32 + 0.5)       # SKP_FIX_CONST(FIND_LPC_COND_FAC, 32)
CHIRP_Q16 = int(float(np.float32(0.99995)) * 65536.0 + 0.5)     # SKP_FIX_CONST(FIND_LPC_CHIRP, 16)

HB_OUT = np.dtype([
    ("lsp_idx", "<i4"), ("nrg0", "<i4", 4), ("nlsf_pre", "<i4", ORDER), ("nlsf_q", "<i4", ORDER), ("weight", "<i4", ORDER),
    ("coef", "<i2", ORDER), ("x_hb_buf", "<i2", 680), ("hb_first", "<i4")], align=True)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _ok(r):
    assert r == 0, "CUDA harness call failed with error %d" % r


def w32(x):
    return ((int(x) + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def sqrt_approx(x):
    from tests.test_gpu_ops import sqrt_approx as f
    return f(x)


def trunc_i32(v):
    """(SKP_int32) of a float on the reference's x86 target: truncation, INT_MIN out of range."""
    from tests.test_gpu_ops import trunc_i32 as f
    return f(float(v))


# ---------------------------------------------------------------------------------------------------------------------
# libraries
# ---------------------------------------------------------------------------------------------------------------------
class Ref:
    def __init__(self):
        from oracle import hb_ref, ref
        if not ref.available() or not hb_ref.available():
            pytest.skip("oracle/_ref not built (needs the reference sources at build time)")
        self.fix = ref.lib("fix").lib
        self.flp = ref.lib("flp").lib
        self.hb = hb_ref.RefHb()
        self.cb1 = np.ctypeslib.as_array((C.c_int16 * 2048).in_dll(self.fix, "AGR_Sate_highband_lsp_cdbk1_fix")).reshape(256, ORDER).copy()
        self.cb2 = np.ctypeslib.as_array((C.c_int16 * 128).in_dll(self.fix, "AGR_Sate_highband_lsp_cdbk2_fix")).reshape(16, ORDER).copy()
        self.qmf_fix = np.ctypeslib.as_array((C.c_int16 * 64).in_dll(self.fix, "AGR_Sate_qmf_coeffs_fix")).copy()
        self.qmf_flt = np.ctypeslib.as_array((C.c_float * 64).in_dll(self.flp, "AGR_Sate_qmf_coeffs")).copy()
        self.fix.AGR_Sate_lsp_quant_highband.restype = C.c_int32
        for setting, (F, _) in SETTINGS.items():
            assert self.hb.frame_size(setting) == F, ("the reference's BWE_FrameSize", setting)

    def lsp_quant(self, nlsf):
        v = np.ascontiguousarray(nlsf, np.int32).copy()
        idx = self.fix.AGR_Sate_lsp_quant_highband(_p(v), C.c_int32(ORDER))
        return idx, v

    def laroia(self, nlsf):
        w, v = np.zeros(ORDER, np.int32), np.ascontiguousarray(nlsf, np.int32)
        self.fix.SKP_Silk_NLSF_VQ_weights_laroia(_p(w), _p(v), C.c_int(ORDER))
        return w

    def decomp(self, x, mem):
        """AGR_Sate_qmf_decomp of one packet; mem [64] int16 in / out."""
        x = np.ascontiguousarray(x, np.int16)
        lo, hi = np.zeros(len(x) // 2, np.int16), np.zeros(len(x) // 2, np.int16)
        self.fix.AGR_Sate_qmf_decomp(_p(x), _p(self.qmf_fix), _p(lo), _p(hi), C.c_int32(len(x)), C.c_int32(64), _p(mem), None)
        return lo, hi

    def synth(self, fix, low, high, mem1, mem2):
        """AGR_Sate_qmf_synth of one packet and the int16 PCM the decoder makes of it; mem1 / mem2 [64] in / out."""
        N = 2 * len(low)
        if fix:
            x1, x2, y = np.ascontiguousarray(low, np.int16), np.ascontiguousarray(high, np.float32).astype(np.int16), np.zeros(N, np.int16)
            self.fix.AGR_Sate_qmf_synth(_p(x1), _p(x2), _p(self.qmf_fix), _p(y), C.c_int32(N), C.c_int32(64), _p(mem1), _p(mem2), None)
            return y, None
        x1, x2, y = np.ascontiguousarray(low, np.float32), np.ascontiguousarray(high, np.float32), np.zeros(N, np.float32)
        self.flp.AGR_Sate_qmf_synth(_p(x1), _p(x2), _p(self.qmf_flt), _p(y), C.c_int32(N), C.c_int32(64), _p(mem1), _p(mem2), None)
        # AGR_BWE_decode_frame_FLP.c:222-229
        pcm = np.array([min(32767, max(-32768, trunc_i32(v))) for v in y], np.int16)
        return pcm, y

    def front_nlsf(self, lpc_in):
        """SKP_Silk_find_LPC_FIX's path without interpolation, step by step: Burg, chirp, A2NLSF.  Returns the NLSF vector and
        whether A2NLSF widened the polynomial."""
        rn, rq, a = C.c_int32(0), C.c_int(0), np.zeros(16, np.int32)
        x = np.ascontiguousarray(lpc_in, np.int16)
        self.fix.SKP_Silk_burg_modified(C.byref(rn), C.byref(rq), _p(a), _p(x), C.c_int(88), C.c_int(4), C.c_int32(WNF_Q32), C.c_int(ORDER))
        self.fix.SKP_Silk_bwexpander_32(_p(a), C.c_int(ORDER), C.c_int32(CHIRP_Q16))
        a0, nl = a.copy(), np.zeros(ORDER, np.int32)
        self.fix.SKP_Silk_A2NLSF(_p(nl), _p(a), C.c_int(ORDER))
        return nl, bool((a != a0).any())


@pytest.fixture(scope="module")
def ref():
    return Ref()


@pytest.fixture(scope="module")
def ops():
    if not os.path.exists(OPS_LIB):
        pytest.fail(OPS_LIB + " missing: __graft_entry__.build() builds it")
    L = C.CDLL(OPS_LIB)
    assert L.sb_ops_hb_out_bytes() == HB_OUT.itemsize
    return L


def _first_diff(what, got, want):
    got, want = np.asarray(got), np.asarray(want)
    bad = np.argwhere(got != want)
    if len(bad):
        i = tuple(int(v) for v in bad[0])
        raise AssertionError("%s: %d elements differ, first at element %s: device %s, reference %s"
                             % (what, len(bad), i, got[i], want[i]))


# ---------------------------------------------------------------------------------------------------------------------
# high-band frames
# ---------------------------------------------------------------------------------------------------------------------
def _sines(rng, L):
    """Two or three full-scale sinusoids a fraction of a grid step apart: A2NLSF finds two roots in one interval of its cosine
    grid and widens the polynomial."""
    t = np.arange(L)
    f0, df = rng.uniform(0.02, 0.48), rng.uniform(0, 0.003)
    x = sum(rng.uniform(8000, 16000) * np.sin(2 * np.pi * (f0 + i * df) * t + rng.uniform(0, 6.3)) for i in range(int(rng.integers(2, 4))))
    return np.clip(np.round(x), -32768, 32767)


def _speech_high(ref, L, offset):
    clip = load_clip()
    mem = np.zeros(64, np.int16)
    out = []
    for p in range(len(clip) // PACKET):
        out.append(ref.decomp(clip[p * PACKET:(p + 1) * PACKET], mem)[1])
    h = np.concatenate(out)
    return np.resize(np.roll(h, -offset), L)


def hb_signal(ref, kind, L, rng, F):
    if kind == "zeros":
        return np.zeros(L)
    if kind == "pm1":
        return rng.integers(-1, 2, L)
    if kind == "dc":
        return np.full(L, rng.choice([1, 1000, -20000, 32767, -32768]))
    if kind == "nyquist":
        s = rng.choice([32767, -32768])
        return np.where(np.arange(L) % 2 == 0, s, -32767 if s > 0 else 32767)
    if kind == "noise_full":
        return rng.integers(-32768, 32768, L)
    if kind == "sines":
        return _sines(rng, L)
    if kind == "speech":
        return _speech_high(ref, L, int(rng.integers(0, 20000)))
    if kind == "steps":      # a different class every frame
        kinds = ["zeros", "pm1", "dc", "nyquist", "noise_full", "sines", "speech"]
        return np.concatenate([hb_signal(ref, kinds[int(rng.integers(len(kinds)))], F, rng, F) for _ in range(L // F)])
    raise ValueError(kind)


HB_KINDS = ("zeros", "pm1", "dc", "nyquist", "noise_full", "sines", "speech", "steps")


def hb_cases(ref):
    """[(name, setting, high [nfr, F])]: every class for both frame lengths (and both packet lengths of F = 160); speech and
    step changes over 52 frames, the rest over 6 (every case starts from the reset state, so its first frame is one after
    reset).  Several seeds per class, so that neighbouring warps take different cases and different F; one more speech case
    leaves the last block of the launch partly empty."""
    out = []
    for kind in HB_KINDS:
        for seed in range(3):
            for setting, (F, n) in SETTINGS.items():
                rng = np.random.default_rng(1000 * HB_KINDS.index(kind) + 10 * seed + len(setting))
                nfr = 52 if kind in ("speech", "steps") else 6
                x = hb_signal(ref, kind, nfr * F, rng, F).astype(np.int16)
                out.append(("%s/%d/%s" % (kind, seed, setting), setting, x.reshape(nfr, F)))
    x = hb_signal(ref, "speech", 52 * 160, np.random.default_rng(99), 160).astype(np.int16)
    out.append(("speech/3/40ms", "40ms", x.reshape(52, 160)))
    return out


def ref_hb_frames(ref, setting, high):
    rec = ref.hb.run(setting, high)
    assert (rec["n_quant"] == 1).all() and (rec["n_nlsf2a"] == 4).all() and (rec["n_filter"] == 4).all()
    F = high.shape[1]
    SF = F // 4
    nrg = np.zeros((len(high), 4), np.int64)
    wrapped = np.zeros((len(high), 4), bool)
    for f in range(len(high)):
        for k in range(4):
            e = int((rec["exc"][f, k * SF:(k + 1) * SF].astype(np.int64) ** 2).sum())
            wrapped[f, k] = e > I32_MAX
            nrg[f, k] = sqrt_approx(w32(e))
    return rec, nrg, wrapped


def dev_hb(ops, cases, per_frame):
    n = len(cases)
    nfr = max(len(x) for _, _, x in cases)
    npk = max(len(x) * x.shape[1] // SETTINGS[s][1] for _, s, x in cases)
    kc = np.array([SETTINGS[s] for _, s, _ in cases], np.int32)
    high = np.zeros((n, npk, PACKET // 2), np.int16)
    for i, (_, s, x) in enumerate(cases):
        m = SETTINGS[s][1]
        flat = x.reshape(-1)
        for p in range(len(flat) // m):
            high[i, p, :m] = flat[p * m:(p + 1) * m]
    out = np.zeros((n, npk, 2), HB_OUT)
    _ok(ops.sb_ops_hb(n, npk, per_frame, _p(kc), _p(high), _p(out)))
    res = []
    for i, (_, s, x) in enumerate(cases):
        fpp = SETTINGS[s][1] // SETTINGS[s][0]
        res.append(out[i, :, :fpp].reshape(-1)[:len(x)])
    assert nfr == max(len(r) for r in res)
    return res


@pytest.mark.gpu
def test_hb_frames_against_reference(ops, ref):
    """Every frame's working set (one c_hb_analyse_packet call per frame), then the same cases through whole packets (the
    product's loop over the frames of a packet) for the per-frame results and the state after each packet."""
    cases = hb_cases(ref)
    assert len(cases) % 4, "the last block of the launch is partly empty"
    got = dev_hb(ops, cases, 1)
    packets = dev_hb(ops, cases, 0)
    for (name, setting, x), d, q in zip(cases, got, packets):
        rec, nrg, _ = ref_hb_frames(ref, setting, x)
        fpp = SETTINGS[setting][1] // SETTINGS[setting][0]
        for f in range(len(x)):
            where = "%s frame %d (whole packets)" % (name, f)
            _first_diff(where + " lsp_idx", q["lsp_idx"][f], rec["lsp_idx"][f])
            _first_diff(where + " hb_nrg0", q["nrg0"][f], nrg[f])
            if f % fpp == fpp - 1:
                _first_diff(where + " x_hb_buf after the packet", q["x_hb_buf"][f], rec["x_hb_buf"][f])
                assert q["hb_first"][f] == 0, where + " hb_first after the packet"
        for f in range(len(x)):
            where = "%s frame %d" % (name, f)
            _first_diff(where + " pre-VQ NLSF_Q15", d["nlsf_pre"][f], rec["nlsf_in"][f])
            _first_diff(where + " Laroia weights", d["weight"][f], ref.laroia(rec["nlsf_in"][f]))
            _first_diff(where + " lsp_idx", d["lsp_idx"][f], rec["lsp_idx"][f])
            _first_diff(where + " quantised NLSF_Q15", d["nlsf_q"][f], rec["nlsf_q"][f])
            _first_diff(where + " HB_prev_NLSFq_Q15", d["nlsf_q"][f], rec["prev_nlsfq"][f])
            for k in range(4):
                _first_diff(where + " NLSF2A_stable coef (sub-frame %d)" % k, d["coef"][f], rec["coef"][f, k])
            _first_diff(where + " hb_nrg0", d["nrg0"][f], nrg[f])
            _first_diff(where + " x_hb_buf after the slide", d["x_hb_buf"][f], rec["x_hb_buf"][f])
            assert d["hb_first"][f] == 0, where + " hb_first (1 in the reset state)"


# ---------------------------------------------------------------------------------------------------------------------
# LSP search
# ---------------------------------------------------------------------------------------------------------------------
def _i16(v):
    return ((np.asarray(v, np.int64) + 32768) & 0xFFFF) - 32768


def _wrap32(v):
    return ((np.asarray(v, np.int64) + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def vq_search(cb1, cb2, w, x):
    """AGR_Sate_lsp_quant_highband's two searches in big integers, for classifying cases: (first-stage distances [256] (wrapped,
    and unwrapped sums), second-stage distances [16] (wrapped, unwrapped), idx1, idx2)."""
    x = np.asarray(x, np.int64)
    t = _i16(x[None, :] - cb1.astype(np.int64))
    d1_raw = (t * t).sum(1)                                   # SMLABB: (int16) tmp * (int16) tmp, summed mod 2^32
    d1 = _wrap32(d1_raw)
    idx1 = int(np.argmin(d1)) if d1.min() < I32_MAX else 0
    r = x - cb1[idx1].astype(np.int64)
    t2 = _wrap32(r[None, :] - cb2.astype(np.int64))
    sq = _i16(t2) * _i16(t2)                                  # SMULBB
    terms = (sq * _i16(np.asarray(w, np.int64))[None, :]) >> 16   # SMLAWB: (b * (int16) c) >> 16
    d2_raw = terms.sum(1)
    d2 = _wrap32(d2_raw)
    idx2 = int(np.argmin(d2)) if d2.min() < I32_MAX else 0
    return d1, d1_raw, d2, d2_raw, idx1, idx2


def _equidistant(a, b, reach=40):
    """An integer point next to the midpoint of rows a and b at exactly equal squared distance from both, or None: with
    u = b - a, |x - a|^2 - |x - b|^2 = sum u (2x - a - b), solved by moving three components of the rounded midpoint."""
    u = b - a
    x = (a + b) // 2
    D = int((u * (2 * x - a - b)).sum())
    if D % 2:
        return None
    need = -D // 2                    # sum u_j d_j = need
    nz = np.nonzero(u)[0]
    if len(nz) < 3:
        return None
    j = nz[np.argsort(np.abs(u[nz]))[:3]]
    r = np.arange(-reach, reach + 1)
    d0, d1 = np.meshgrid(r, r)
    rem = need - u[j[0]] * d0 - u[j[1]] * d1
    d2 = rem // u[j[2]]
    ok = (rem % u[j[2]] == 0) & (np.abs(d2) <= reach)
    if not ok.any():
        return None
    k = np.argmin(np.where(ok, np.abs(d0) + np.abs(d1) + np.abs(d2), 1 << 30))
    x = x.copy()
    x[j[0]] += d0.flat[k]
    x[j[1]] += d1.flat[k]
    x[j[2]] += d2.flat[k]
    return x


def vq_cases(ref):
    """NLSF vectors [n, 8] (int32) for the LSP search:
      first-stage ties at the minimum between rows e and e + 32k (one lane's rows) and between rows of different lanes,
      found next to the midpoints of near codebook rows;
      second-stage ties: a first-stage row plus a point next to the midpoint of two second-stage rows;
      wrapping SMLABB / SMLAWB sums: components far outside the codebook's range (|x - cb| beyond 2^15);
      codebook rows themselves, and random sorted vectors as the analysis produces them.
    The INT_MAX fallback of the second stage (every one of the 16 distances equal to INT_MAX) is not constructed: a single
    residual would need 16 wrapped sums of eight weighted squares all equal to 2^31 - 1, and no search has found one; the
    branch test asserts it is never reached, so the kernel's equality test against INT_MAX stays unexercised."""
    cb1, cb2 = ref.cb1.astype(np.int64), ref.cb2.astype(np.int64)
    rng = np.random.default_rng(77)
    same_lane, other_lane, ties2 = [], [], []
    for a in range(256):
        by_dist = np.argsort(((cb1 - cb1[a]) ** 2).sum(1))
        partners = [int(b) for b in by_dist[1:6]] + [int(b) for b in by_dist if b != a and (b - a) % 32 == 0][:3]
        for b in partners:
            if b < a and (b - a) % 32:
                continue
            x = _equidistant(cb1[a], cb1[b])
            if x is None:
                continue
            d1 = vq_search(ref.cb1, ref.cb2, ref.laroia(x), x)[0]
            if d1[a] == d1.min() == d1[b]:
                (same_lane if (b - a) % 32 == 0 else other_lane).append(x)
    for _ in range(1000):
        i = int(rng.integers(256))
        a, b = rng.choice(16, 2, replace=False)
        mid = cb1[i] + (cb2[a] + cb2[b]) // 2
        for _ in range(8):
            x = mid + rng.integers(-1, 2, ORDER)
            _, _, d2, _, i1, _ = vq_search(ref.cb1, ref.cb2, ref.laroia(x), x)
            if i1 == i and d2[a] == d2.min() == d2[b]:
                ties2.append(x)
                break
    wrap = []
    for _ in range(60):
        x = rng.integers(0, 32768, ORDER) + rng.choice([-1, 1], ORDER) * rng.integers(20000, 1 << 20, ORDER)
        wrap.append(np.sort(x) if rng.random() < 0.5 else x)
    for _ in range(60):       # clustered components far outside the codebook: large Laroia weights on large residuals
        wrap.append(rng.integers(-40000, 70000) + np.cumsum(rng.choice([1, 2, 3, 50, 3000, 20000], ORDER)))
    plain = [cb1[int(i)] for i in rng.integers(0, 256, 32)] + [np.sort(rng.integers(0, 32768, ORDER)) for _ in range(64)]
    rows = same_lane + other_lane + ties2 + wrap + plain
    return np.array(rows, np.int64).astype(np.int32), dict(same_lane=len(same_lane), other_lane=len(other_lane), ties2=len(ties2))


@pytest.mark.gpu
def test_lsp_search_against_reference(ops, ref):
    x, _ = vq_cases(ref)
    n = len(x)
    idx, q, w = np.zeros(n, np.int32), np.zeros((n, ORDER), np.int32), np.zeros((n, ORDER), np.int32)
    _ok(ops.sb_ops_hb_vq(n, _p(np.ascontiguousarray(x)), _p(idx), _p(q), _p(w)))
    for i in range(n):
        ri, rq = ref.lsp_quant(x[i])
        where = "LSP case %d %s" % (i, [int(v) for v in x[i]])
        _first_diff(where + " weights", w[i], ref.laroia(x[i]))
        _first_diff(where + " index", idx[i], ri)
        _first_diff(where + " quantised vector", q[i], rq)
        _first_diff(where + " residual", x[i].astype(np.int64) - q[i], x[i].astype(np.int64) - rq)


# ---------------------------------------------------------------------------------------------------------------------
# synthesis filter bank
# ---------------------------------------------------------------------------------------------------------------------
SYN_KINDS = ("random", "loud", "tiny", "extremes")


def syn_case(kind, fix, N2, npk, rng, coef_sign):
    """low [npk, N2] int16, high [npk, N2] float32.  A fixed-point stream's high band and filter memories hold int16 values
    (sb_dec.cuh), so the synthesis kernel's __float2int_rz and the host model's (i32) cast convert them alike; its cases
    keep to that range."""
    if kind == "random":          # fractional high band, speech-like levels
        low = rng.integers(-12000, 12000, (npk, N2))
        high = rng.normal(0, 3000, (npk, N2)) + rng.uniform(-1, 1, (npk, N2))
    elif kind == "loud":          # sums past +-32768 and just past 32767 / -32768: the clamps after truncation
        s = rng.choice([-1, 1], (npk, 1))
        low = np.clip(s * coef_sign(N2) * rng.integers(20000, 32768, (npk, N2)), -32768, 32767)
        high = s * coef_sign(N2) * rng.uniform(0, 30000, (npk, N2)) * rng.choice([0.0, 1.0], (npk, N2), p=[0.3, 0.7])
    elif kind == "tiny":          # outputs in (-1, 0) and (0, 1)
        low = rng.integers(-1, 2, (npk, N2)) * (rng.random((npk, N2)) < 0.05)
        high = rng.uniform(-0.9, 0.9, (npk, N2))
    else:                         # int16 extremes in the filter's sign pattern: wrapping int32 sums, the -32767 clamp
        s = rng.choice([-1, 1], (npk, 1))
        pat = s * coef_sign(N2)
        low = np.where(pat > 0, 32767, -32768) * (rng.random((npk, N2)) < 0.9)
        high = np.where(pat > 0, 32767.0, -32768.0) * rng.choice([-1.0, 1.0], (npk, N2))
    if fix:
        high = np.trunc(np.clip(high, -32768, 32767))
    return low.astype(np.int16), high.astype(np.float32)


def syn_cases(ref):
    """[(name, fix, N2, low [npk, N2], high [npk, N2], mem0 [128])], float and fixed-point streams alternating, so that they sit
    in neighbouring warps; N2 = 160, 320 (16 kHz, 20 and 40 ms) and 640 (32 kHz, 40 ms); 24 packets with carried memories.
    One more stream leaves the last block of the launch partly empty."""
    a = ref.qmf_fix.astype(np.int64)

    def coef_sign(N2):
        # a band pattern whose products with the filter taps mostly share one sign, so the sums grow past int16 / int32
        return np.where(np.resize(np.concatenate([a[0::2], a[1::2]]), N2)[::-1] >= 0, 1, -1)

    out = []
    for kind in SYN_KINDS:
        for N2 in (160, 320, 640):
            for fix in (0, 1):
                rng = np.random.default_rng(SYN_KINDS.index(kind) * 100 + N2 + fix)
                low, high = syn_case(kind, fix, N2, 24, rng, coef_sign)
                mem = np.zeros(128, np.float32)
                out.append(("%s/N2=%d/%s" % (kind, N2, "fix" if fix else "float"), fix, N2, low, high, mem))
    low, high = syn_case("random", 0, 640, 24, np.random.default_rng(7), coef_sign)
    out.append(("random/N2=640/float/2", 0, 640, low, high, np.zeros(128, np.float32)))
    return out


def ref_syn(ref, fix, low, high):
    t = np.int16 if fix else np.float32
    m1, m2 = np.zeros(64, t), np.zeros(64, t)
    pcm, raw, mems = [], [], []
    for p in range(len(low)):
        y, r = ref.synth(fix, low[p], high[p], m1, m2)
        pcm.append(y)
        raw.append(r)
        mems.append(np.concatenate([m1, m2]).astype(np.float32))
    return np.array(pcm), raw, np.array(mems)


@pytest.mark.gpu
def test_synthesis_against_reference(ops, ref):
    cases = syn_cases(ref)
    n, npk = len(cases), len(cases[0][3])
    assert n % 4, "the last block of the launch is partly empty"
    fix = np.array([c[1] for c in cases], np.int32)
    n2 = np.array([c[2] for c in cases], np.int32)
    mem0 = np.ascontiguousarray(np.stack([c[5] for c in cases]), np.float32)
    low = np.zeros((n, npk, SYN_N2MAX), np.int16)
    high = np.zeros((n, npk, SYN_N2MAX), np.float32)
    for i, c in enumerate(cases):
        low[i, :, :c[2]] = c[3]
        high[i, :, :c[2]] = c[4]
    pcm = np.zeros((n, npk, 2 * SYN_N2MAX), np.int16)
    mem = np.zeros((n, npk, 128), np.float32)
    _ok(ops.sb_ops_synth(n, npk, _p(fix), _p(n2), _p(mem0), _p(low), _p(high), _p(pcm), _p(mem)))
    for i, (name, f, N2, lo, hi, _) in enumerate(cases):
        rp, _, rm = ref_syn(ref, f, lo, hi)
        for p in range(npk):
            _first_diff("%s packet %d PCM" % (name, p), pcm[i, p, :2 * N2], rp[p])
            # only the odd entries are filter memory (AGR_BWE_qmf.c:178-181); the even ones stay as they started
            _first_diff("%s packet %d memories" % (name, p), mem[i, p], rm[p])


# ---------------------------------------------------------------------------------------------------------------------
# band split
# ---------------------------------------------------------------------------------------------------------------------
SPLIT_KINDS = ("impulses", "dc", "alternating", "chirp", "random")


def split_signal(kind, L, rng):
    if kind == "impulses":
        x = np.zeros(L, np.int64)
        x[rng.integers(0, L, L // 50)] = rng.choice([32767, -32768, 1, -1, 5000], L // 50)
        return x
    if kind == "dc":
        return np.full(L, rng.choice([32767, -32768, 1, -1, 12345]))
    if kind == "alternating":     # full-scale Nyquist: the high band beyond +-32767 on both sides
        return np.where(np.arange(L) % 2 == int(rng.integers(2)), 32767, -32768)
    if kind == "chirp":
        return chirp(L, amp=int(rng.integers(8000, 32767)))
    return rng.integers(-32768, 32768, L)


def split_cases():
    out = []
    for kind in SPLIT_KINDS:
        for spp in (640, 320):
            for seed in range(2):
                rng = np.random.default_rng(SPLIT_KINDS.index(kind) * 10 + seed + spp)
                x = np.clip(split_signal(kind, 20 * spp, rng), -32768, 32767).astype(np.int16)
                out.append(("%s/%d/%d" % (kind, spp, seed), spp, x.reshape(20, spp)))
    return out


def ref_split(ref, x):
    mem = np.zeros(64, np.int16)
    bands, mems = [], []
    for p in range(len(x)):
        lo, hi = ref.decomp(x[p], mem)
        bands.append(np.concatenate([lo, hi]))
        mems.append(mem.copy())
    return np.array(bands), np.array(mems)


@pytest.mark.gpu
def test_band_split_against_reference(ops, ref):
    cases = split_cases()
    n, npk = len(cases), 20
    spp = np.array([c[1] for c in cases], np.int32)
    pcm = np.zeros((n, npk, PACKET), np.int16)
    for i, (_, s, x) in enumerate(cases):
        pcm[i, :, :s] = x
    bands = np.zeros((n, npk, PACKET), np.int16)
    mem = np.zeros((n, npk, 64), np.int16)
    _ok(ops.sb_ops_qmf_split(n, npk, _p(spp), _p(np.zeros((n, 64), np.int16)), _p(pcm), _p(bands), _p(mem)))
    for i, (name, s, x) in enumerate(cases):
        rb, rm = ref_split(ref, x)
        for p in range(npk):
            _first_diff("%s packet %d bands [low | high]" % (name, p), bands[i, p, :s], rb[p])
            _first_diff("%s packet %d memory" % (name, p), mem[i, p, :63], rm[p, :63])


# ---------------------------------------------------------------------------------------------------------------------
# the tables reach what they are for (reference only)
# ---------------------------------------------------------------------------------------------------------------------
def fix_synth_sums(a, low, high, m1, m2):
    """The fixed-point filter bank's four MAC sums per group in big integers (AGR_BWE_qmf.c:134-168): [N2 / 2, 4]."""
    N2 = len(low)
    xx1 = np.concatenate([np.asarray(low, np.int64)[::-1], np.asarray(m1, np.int64)[1::2]])
    xx2 = np.concatenate([np.asarray(high, np.int64)[::-1], np.asarray(m2, np.int64)[1::2]])
    i = np.arange(0, N2, 2)
    y = np.zeros((len(i), 4), np.int64)
    x10, x20 = xx1[N2 - 2 - i], xx2[N2 - 2 - i]
    for j in range(0, 32, 2):
        a0, a1 = a[2 * j], a[2 * j + 1]
        x11, x21 = xx1[N2 - 1 + j - i], xx2[N2 - 1 + j - i]
        y[:, 0] += a0 * x11 - a0 * x21
        y[:, 1] += a1 * x11 + a1 * x21
        y[:, 2] += a0 * x10 - a0 * x20
        y[:, 3] += a1 * x10 + a1 * x20
        a0, a1 = a[2 * j + 2], a[2 * j + 3]
        x10, x20 = xx1[N2 + j - i], xx2[N2 + j - i]
        y[:, 0] += a0 * x10 - a0 * x20
        y[:, 1] += a1 * x10 + a1 * x20
        y[:, 2] += a0 * x11 - a0 * x21
        y[:, 3] += a1 * x11 + a1 * x21
    return y


def test_case_tables_reach_every_listed_regime(ref):
    # ---- high-band frames: wrapped sub-frame energies (and the zero square root they give), A2NLSF widening, both frame
    #      lengths, runs of 50 frames and more.  Two regimes of the frame's routines are out of reach of any input, and the
    #      tables are held to their absence:
    #      * A2NLSF's white-spectrum fallback (NLSF[k] = (k + 1) * (2^15 / 9), after 30 failed widenings): the frame's
    #        polynomial is Burg's minimum-phase filter after the 0.99995 chirp, whose roots the widening separates within a
    #        few steps.  Silence gives an ordinary root search (Burg's all-zero predictor), not the fallback.  The fallback
    #        of c_a2nlsf itself is compared on large random polynomials in test_gpu_ops.py.
    #      * NLSF2A_stable's bandwidth-expansion loop: the frame filters it is called with are cb1[i] + cb2[j], and none of
    #        the 4 096 sums gives an unstable filter (checked below), so the high band never enters that loop.
    from tests.test_gpu_ops import white_nlsf
    white_vec = list(white_nlsf(ORDER))
    plain, stable = np.zeros(ORDER, np.int16), np.zeros(ORDER, np.int16)
    unstable_sums = 0
    for i in range(256):
        for j in range(16):
            v = np.ascontiguousarray(ref.cb1[i].astype(np.int32) + ref.cb2[j].astype(np.int32))
            ref.fix.SKP_Silk_NLSF2A(_p(plain), _p(v), C.c_int(ORDER))
            ref.fix.SKP_Silk_NLSF2A_stable(_p(stable), _p(v), C.c_int(ORDER))
            unstable_sums += list(plain) != list(stable)
    assert unstable_sums == 0, ("a quantised high-band vector needs NLSF2A_stable's expansion", unstable_sums)
    wrapped = zero_sqrt = widened = white = expanded = long_runs = 0
    per_F = {160: 0, 320: 0}
    for name, setting, x in hb_cases(ref):
        rec, nrg, wr = ref_hb_frames(ref, setting, x)
        F = x.shape[1]
        per_F[F] += len(x)
        long_runs += len(x) >= 50
        wrapped += int(wr.sum())
        zero_sqrt += int((wr & (nrg == 0)).sum())
        buf = np.zeros(2 * 1280 + 480, np.int16)
        for f in range(len(x)):
            buf[F + 40:2 * F + 40] = x[f]
            lpc_in = np.concatenate([buf[F - ORDER + 80 * k:F - ORDER + 80 * k + 88] for k in range(4)])
            nl, wid = ref.front_nlsf(lpc_in)
            assert list(nl) == list(rec["nlsf_in"][f]), ("the front of the frame is find_LPC_FIX's", name, f)
            widened += wid
            white += list(nl) == white_vec
            ref.fix.SKP_Silk_NLSF2A(_p(plain), _p(np.ascontiguousarray(rec["nlsf_q"][f], np.int32)), C.c_int(ORDER))
            expanded += list(plain) != list(rec["coef"][f, 0])
            buf[:680] = rec["x_hb_buf"][f]
    assert wrapped >= 20 and zero_sqrt >= 1 and widened >= 5 and long_runs >= 10 and min(per_F.values()) >= 200, \
        ("high-band frames", wrapped, zero_sqrt, widened, long_runs, per_F)
    assert white == 0 and expanded == 0, ("regimes documented as out of reach were reached: update the notes", white, expanded)

    # ---- LSP search: ties of each kind, wrapping distances, the (absent) INT_MAX fallback
    x, counts = vq_cases(ref)
    wrap1 = wrap2 = fallback = 0
    for v in x:
        d1, d1r, d2, d2r, i1, i2 = vq_search(ref.cb1, ref.cb2, ref.laroia(v), v)
        assert (i1 | (i2 << 8)) == ref.lsp_quant(v)[0], ("the statement is the reference's search", list(v))
        wrap1 += bool((d1 != d1r).any())
        wrap2 += bool((d2 != d2r).any())
        fallback += bool((d2 == I32_MAX).all())
    assert counts["same_lane"] >= 5 and counts["other_lane"] >= 20 and counts["ties2"] >= 20, counts
    assert wrap1 >= 20 and wrap2 >= 5 and fallback == 0, (wrap1, wrap2, fallback)

    # ---- synthesis: float clamps at +32767 and -32768, outputs in (-1, 0), fixed-point int32 wrap and the -32767 clamp
    hi_clamp = lo_clamp = neg_frac = fix_wrap = fix_lo = fix_hi = 0
    a = ref.qmf_fix.astype(np.int64)
    for name, fix, N2, low, high, _ in syn_cases(ref):
        if fix:
            m1, m2 = np.zeros(64, np.int16), np.zeros(64, np.int16)
            for p in range(len(low)):
                y_exact = fix_synth_sums(a, low[p], high[p].astype(np.int16), m1, m2)
                fix_wrap += int(((y_exact > I32_MAX) | (y_exact < I32_MIN)).sum())
                y, _ = ref.synth(1, low[p], high[p], m1, m2)
                fix_lo += int((y == -32767).sum())
                fix_hi += int((y == 32767).sum())
        else:
            _, raw, _ = ref_syn(ref, 0, low, high)
            r = np.concatenate(raw)
            hi_clamp += int((r >= 32768).sum())
            lo_clamp += int((r < -32768).sum())
            neg_frac += int(((r > -1) & (r < 0)).sum())
    assert hi_clamp >= 50 and lo_clamp >= 50 and neg_frac >= 50 and fix_wrap >= 20 and fix_lo >= 50 and fix_hi >= 50, \
        ("synthesis", hi_clamp, lo_clamp, neg_frac, fix_wrap, fix_lo, fix_hi)

    # ---- band split: both output clamps
    top = bottom = 0
    for name, spp, x in split_cases():
        b, _ = ref_split(ref, x)
        top += int((b == 32767).sum())
        bottom += int((b == -32767).sum())
    assert top >= 20 and bottom >= 20, ("band split clamps", top, bottom)
