"""The quantiser kernel's device code (nsq_packet_warp, sb_nsq_warp.cuh) frame by frame against the reference's
SKP_Silk_NSQ_del_dec, at lags, gains and decision paths that the encoder-level tests do not reach.

Each case is a start state and 4-6 frames (three 40 ms packets, or five 20 ms packets).  The frames are captured from the host
model's encoder (what its quantiser stage received: frame control and prefiltered input) on speech, noise, silence, LSB noise
and sines, and then perturbed along one axis each; a case starts from the reset state (the reference's own, read through
oracle/nsq_ref.c) or from a state captured in mid-stream.  Every case goes through
  * the reference (oracle/_ref/libjc1_fix_nsq.so), one frame per call;
  * the scalar model (sb_nsq.cuh) and the kernel's code on emulated warps, two different cases per warp (unmarked tests);
  * the kernel's code on the GPU in the production layout (tests/gpu_ops/ops.cu sb_ops_nsq, `gpu`).
Outputs compared bit for bit, after every frame: the pulses of both descriptions, the centre excitation as the encoder keeps
it ((int16)(r >> 10)), the seed written back; after every packet: the three quantiser states.  Of sLPC_Q14 only the 10 newest
values are compared: the reference keeps 32, reads the newest 10 (LPC order) and nothing else, and the kernel stores those.

Contract -- what the encoder can hand the quantiser, which every case respects:
  * pitchL = lag + SKP_Silk_CB_lags_stage2[k][contour] with lag in [16, 144] and the three 8 kHz contours (0,0,0,0),
    (2,1,0,-1), (-1,0,1,2): lags 15..146, sub-frame steps within the contour.  Unvoiced frames: pitchL, LTPCoef_Q14,
    HarmShapeGain_Q14 and LTP_scale_Q14 as the encoder leaves them (pitchL 0, HarmShapeGain 0).
  * Gains_Q16 = log2lin(min(smulwb(INV_SCALE_Q16, ind) + OFFSET, 3967)) along index walks the gain quantiser allows: a
    packet's first index in [0, 63], then steps of -4 .. +40; indices below 0 (gains under 2.0, only reachable when the
    encoder's own gain falls below 2.0) are left out.
  * DeltaGains_Q16: the eight values of the MD gain quantiser (gain_quant.c:75, 140).  Left out: the unquantised values
    SKP_Silk_gains_quant passes through when the inverse falls outside its eight steps -- they depend on a float the
    encoder computes from md_delta_gain_par, whose range is not stated anywhere.
  * LTP_scale_Q14: the three values of SKP_Silk_LTPScales_table_Q14.  NLSFInterpCoef_Q2: 0 .. 4.  QuantOffsetType 0 / 1
    with either signal type, Seed 0 .. 3.
  * Lambda_Q10, Tilt_Q14, LF_shp_Q14, HarmShapeGain_Q14 (voiced): the smallest and largest values the host model's
    encoder produced over the capture signals at 8 and 100 kb/s.
  * Input: the captured xfw, full scale (+-32767) under the smallest gains (residual clamp at +-64 pulses, sat16 of the
    output), silence, +-1 LSB.
The unmarked reach test runs the tables through a coverage build of the same reference library and checks that the source
lines they are meant to reach are reached (anchors found by their text when the library is built: oracle/cov_anchors.py)."""
import ctypes as C
import functools
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from oracle import nsq_ref
from tests.hostsim import sim
from tests.util import load_clip

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS_LIB = os.path.join(ROOT, "tests", "_gpu_ops", "libsb_gpu_ops.so")

CONTOURS = ((0, 0, 0, 0), (2, 1, 0, -1), (-1, 0, 1, 2))       # SKP_Silk_CB_lags_stage2, the 8 kHz columns
LTP_SCALES = (15565, 11469, 8192)                              # SKP_Silk_LTPScales_table_Q14
INV_SCALE_Q16 = (65536 * (((86 - 6) * 128) // 6)) // (64 - 1)  # gain_quant.c:32 (MIN / MAX_QGAIN_DB 6 / 86, 64 levels)
GAIN_OFFSET = (6 * 128) // 6 + 16 * 128                        # gain_quant.c:30


def _reference():
    if not nsq_ref.available():
        pytest.skip("oracle/_ref/libjc1_fix_nsq.so not built (needs the reference sources at build time)")
    return nsq_ref.RefNsq()


def gain_q16(R, ind):
    """gains_dequant for an accumulated index (gain_quant.c:133)."""
    R.L.SKP_Silk_log2lin.restype = C.c_int32
    x = min(((INV_SCALE_Q16 * ind) >> 16) + GAIN_OFFSET, 3967)
    return int(R.L.SKP_Silk_log2lin(C.c_int32(x)))


def delta_gains():
    from tests.test_gpu_ops import inverse32_varq
    return [inverse32_varq((k + 1) * (32768 // 8) + 32767, 32) for k in range(8)]


# ---------------------------------------------------------------------------------------------------------------------
# captures
# ---------------------------------------------------------------------------------------------------------------------
def _signals():
    clip = load_clip()
    rng = np.random.Generator(np.random.PCG64(11))
    n = 640 * 24
    t = np.arange(n)
    return {
        "speech": clip[640 * 10:640 * 10 + n],
        "speech_late": clip[640 * 100:640 * 100 + n],
        "noise": np.clip(rng.normal(0, 3000, n), -32768, 32767).astype(np.int16),
        "silence": np.zeros(n, np.int16),
        "lsb": rng.integers(-1, 2, n).astype(np.int16),
        "sine200": (8000 * np.sin(2 * np.pi * 200 * t / 16000)).astype(np.int16),
        "sine60": (12000 * np.sin(2 * np.pi * 60 * t / 16000)).astype(np.int16),
    }


@functools.lru_cache(maxsize=None)
def captures(framesize_ms, rate=13600):
    """{signal: (frames [packets, nf], states before each packet [packets, 3])} from the host model's encoder."""
    res = {}
    for name, x in _signals().items():
        e = sim.SimEncoder(rate=rate, framesize_ms=framesize_ms)
        k = e.samples
        fr, st = zip(*[e.capture(x[i * k:(i + 1) * k]) for i in range(len(x) // k)])
        e.close()
        res[name] = (np.stack(fr), np.stack(st))
    return res


@functools.lru_cache(maxsize=None)
def encoder_ends():
    """Smallest / largest value of the shaping and rate controls over every captured frame (voiced frames for the
    harmonic shaping), at two rates."""
    fr = np.concatenate([f.reshape(-1) for r in (8000, 100000) for f, _ in captures(40, r).values()]
                        + [f.reshape(-1) for f, _ in captures(40).values()])
    v = fr[fr["sigtype"] == 0]
    return {"Lambda_Q10": (int(fr["Lambda_Q10"].min()), int(fr["Lambda_Q10"].max())),
            "Tilt_Q14": (int(fr["Tilt_Q14"].min()), int(fr["Tilt_Q14"].max())),
            "LF_shp_Q14": (int(fr["LF_shp_Q14"].min()), int(fr["LF_shp_Q14"].max())),
            "HarmShapeGain_Q14": (int(v["HarmShapeGain_Q14"].min()), int(v["HarmShapeGain_Q14"].max()))}


# ---------------------------------------------------------------------------------------------------------------------
# case tables
# ---------------------------------------------------------------------------------------------------------------------
def _voiced_run(fr, npk, nf):
    """First packet index p such that packets p .. p+npk-1 are voiced in every frame."""
    v = (fr["sigtype"] == 0).all(axis=1)
    for p in range(len(v) - npk + 1):
        if v[p:p + npk].all():
            return p
    raise AssertionError("no voiced run of %d packets in the capture" % npk)


@functools.lru_cache(maxsize=None)
def case_table(nf):
    """[(name, st0 [3], frames [npk * nf])], ordered so that neighbouring cases differ, odd count."""
    R = _reference()
    reset = R.reset_state()
    cap = captures(20 * nf)
    npk = 3 if nf == 2 else 5
    nfr = npk * nf
    ends = encoder_ends()
    cases = []

    def add(name, sig, p, edit=None, start="mid"):
        fr, st = cap[sig]
        f = fr[p:p + npk].reshape(-1).copy()
        s = reset.copy() if start == "reset" else st[p].copy()
        if edit:
            edit(f)
        cases.append((name, s, f))

    sp = _voiced_run(cap["speech"][0], npk, nf)
    sp2 = _voiced_run(cap["speech_late"][0], npk, nf)
    # starting frames as captured: reset and mid-stream starts of every signal class
    for sig in ("speech", "noise", "silence", "lsb", "sine200", "sine60"):
        add(sig + "@reset", sig, 0, start="reset")
        add(sig + "@mid", sig, 4)
    add("speech_voiced", "speech", sp)

    # pitch: the lowest lags (decision delays 12..15), the 32-sample cap, the top of the range, contour steps
    def lags(seq):
        def ed(f):
            for i in range(len(f)):
                f["pitchL"][i] = [seq[i % len(seq)] + c for c in CONTOURS[i % 3]] if np.isscalar(seq[0]) else seq[i % len(seq)]
        return ed
    for L in (16, 17, 18):
        add("lag%d" % L, "speech", sp, lags([L]))
    add("lag15_contour", "speech", sp, lambda f: f["pitchL"].__setitem__(slice(None), (15, 16, 17, 18)))
    add("lag37_38", "speech", sp2, lags([[37] * 4, [38] * 4]))
    add("lag143_146", "speech", sp, lambda f: f["pitchL"].__setitem__(slice(None), (143, 144, 145, 146)))
    add("lag146_143", "speech", sp2, lambda f: f["pitchL"].__setitem__(slice(None), (146, 145, 144, 143)))
    add("lag144_146", "speech", sp, lags([[144] * 4, (146, 145, 144, 143), (143, 144, 145, 146)]))
    add("lag16_to_144", "speech", sp2, lags([[16] * 4, [144] * 4]))

    # voiced with a small last lag, then unvoiced: the unvoiced frame's decision delay comes from lagPrev
    def to_unvoiced(L):
        def ed(f):
            u = cap["noise"][0][4:4 + npk].reshape(-1)
            for i in range(1, len(f), 2):
                f[i] = u[i]
            for i in range(0, len(f), 2):
                f["pitchL"][i] = (L + 1, L, L, L)
        return ed
    add("voiced16_unvoiced", "speech", sp, to_unvoiced(16))
    add("voiced40_unvoiced", "speech", sp2, to_unvoiced(40))

    # NLSF interpolation factor (rewhitening and flush at sub-frame 2 unless it is 4) and the LTP scaling
    for q in range(5):
        add("interp%d" % q, "speech", sp if q % 2 else sp2, lambda f, q=q: f["NLSFInterpCoef_Q2"].__setitem__(slice(None), q))
    for s in LTP_SCALES:
        add("ltp_scale%d" % s, "speech", sp, lambda f, s=s: f["LTP_scale_Q14"].__setitem__(slice(None), s))

    # gains along the quantiser's index walks
    def walk(first, steps):
        ind = [first]
        for d in steps:
            ind.append(ind[-1] + d)
        return [gain_q16(R, i) for i in ind]
    g_up = walk(0, ([40, 27] + [0] * 2 + [-4] * 4) * nfr)[:4 * nfr]
    g_dn = walk(63, ([-4] * 7 + [40]) * nfr)[:4 * nfr]
    for name, g in (("gain_bottom", walk(0, [0] * (4 * nfr - 1))), ("gain_top", walk(63, [4] + [0] * (4 * nfr - 2))),
                    ("gain_up40_down4", g_up), ("gain_down4_up40", g_dn)):
        for sig in ("speech", "noise"):
            p = sp if sig == "speech" else 2
            add(name + "_" + sig, sig, p, lambda f, g=g: f["Gains_Q16"].__setitem__(slice(None), np.reshape(g, (-1, 4))))

    # rate / shaping controls at the ends the encoder produced
    def setf(field, v, voiced_only=False):
        def ed(f):
            m = f["sigtype"] == 0 if voiced_only else np.ones(len(f), bool)
            f[field][m] = v
        return ed
    for field in ("Lambda_Q10", "Tilt_Q14", "LF_shp_Q14"):
        lo, hi = ends[field]
        add(field + "_lo", "speech", sp, setf(field, lo))
        add(field + "_hi", "noise", 3, setf(field, hi))
    lo, hi = ends["HarmShapeGain_Q14"]
    add("harm_lo", "speech", sp, setf("HarmShapeGain_Q14", lo, True))
    add("harm_hi", "speech", sp2, setf("HarmShapeGain_Q14", hi, True))
    dg = delta_gains()
    add("delta_gain_lo", "speech", sp, setf("DeltaGains_Q16", min(dg)))
    add("delta_gain_hi", "noise", 2, setf("DeltaGains_Q16", max(dg)))
    add("delta_gain_mid", "sine200", 2, setf("DeltaGains_Q16", dg[3]))

    # quantisation offset type x signal type, seeds
    for sig, p in (("speech", sp), ("noise", 3)):
        for qo in (0, 1):
            add("offset%d_%s" % (qo, sig), sig, p, setf("QuantOffsetType", qo))
    for s in range(4):
        add("seed%d" % s, "speech" if s % 2 else "noise", sp if s % 2 else 5, setf("Seed", s))

    # input extremes: full scale under the smallest gains, silence and +-1 LSB under the voiced controls
    def full_scale(f):
        rng = np.random.Generator(np.random.PCG64(len(cases)))
        f["x"] = np.where(rng.integers(0, 2, f["x"].shape) == 1, 32767, -32767)
        f["Gains_Q16"] = gain_q16(R, 0)
    add("fullscale_bottom_gain_speech", "speech", sp, full_scale)
    add("fullscale_bottom_gain_noise", "noise", 2, full_scale)
    add("fullscale_square", "speech", sp2, lambda f: (f["x"].__setitem__(slice(None), np.where((np.arange(160) // 20) % 2, 32767, -32768)),
                                                     f["Gains_Q16"].__setitem__(slice(None), gain_q16(R, 4))))
    add("silence_voiced", "speech", sp, lambda f: f["x"].__setitem__(slice(None), 0))
    add("lsb_voiced", "speech", sp2, lambda f: f["x"].__setitem__(slice(None), np.where(np.arange(160) % 3 == 0, 1, -1)))

    for name, s, f in cases:
        assert len(f) == nfr and np.all((f["pitchL"][f["sigtype"] == 0] >= 15) & (f["pitchL"][f["sigtype"] == 0] <= 146)), name
    # neighbours differ: the extremes of the table (sorted by the first frame's lowest lag, unvoiced last) side by side
    key = [min(f["pitchL"][0]) if f["sigtype"][0] == 0 else 1000 + i for i, (_, _, f) in enumerate(cases)]
    srt = [cases[i] for i in np.argsort(key, kind="stable")]
    order = []
    while srt:
        order.append(srt.pop(0))
        if srt:
            order.append(srt.pop())
    if len(order) % 2 == 0:
        order.append(order[0])
    return order


def _stack(table):
    return (np.stack([s for _, s, _ in table]), np.stack([f for _, _, f in table]))


@functools.lru_cache(maxsize=None)
def ref_outputs(nf):
    """The reference over the table: (out [n, frames], states after every packet [n, packets, 3])."""
    R = _reference()
    out, st = zip(*[R.run(s, f) for _, s, f in case_table(nf)])
    return np.stack(out), np.stack(st)[:, nf - 1::nf]


STATE_FIELDS = ("xq", "sLTP_shp_Q10", "sLPC_Q14", "sAR2_Q14", "sLF_AR_shp_Q12", "lagPrev", "prev_inv_gain_Q16")
QZ = ("centre", "description 1", "description 2")


def compare(table, nf, got, want, what):
    out, st = got
    rout, rst = want
    for c, (name, _, _) in enumerate(table):
        for f in range(out.shape[1]):
            for field, g, w in (("q_md[0]", out[c, f]["q_md"][0], rout[c, f]["q_md"][0]),
                                ("q_md[1]", out[c, f]["q_md"][1], rout[c, f]["q_md"][1]),
                                ("r16", out[c, f]["r16"], rout[c, f]["r16"]), ("Seed", out[c, f]["Seed"], rout[c, f]["Seed"])):
                bad = np.flatnonzero(np.atleast_1d(g != w))
                assert not len(bad), "%s: case %s, packet %d, frame %d, %s differs first at [%d]: %s vs reference %s" % (
                    what, name, f // nf, f % nf, field, bad[0], np.atleast_1d(g)[bad[0]], np.atleast_1d(w)[bad[0]])
        for p in range(st.shape[1]):
            for qz in range(3):
                for field in STATE_FIELDS:
                    g, w = np.atleast_1d(st[c, p, qz][field]), np.atleast_1d(rst[c, p, qz][field])
                    if field == "sLPC_Q14":
                        g, w = g[22:], w[22:]
                    bad = np.flatnonzero(g != w)
                    assert not len(bad), "%s: case %s, state after packet %d, %s quantiser, %s differs first at [%d]: %s vs reference %s" % (
                        what, name, p, QZ[qz], field, bad[0], g[bad[0]], w[bad[0]])


TABLES = (2, 1)   # 40 ms and 20 ms packets


@pytest.mark.parametrize("nf", TABLES)
def test_scalar_model_matches_reference(nf):
    """The host model's quantiser (sb_nsq.cuh) over the case tables, frame by frame."""
    table = case_table(nf)
    st0, fr = _stack(table)
    compare(table, nf, sim.nsq_run(st0, fr, nf), ref_outputs(nf), "scalar model")


@pytest.mark.parametrize("nf", TABLES)
def test_kernel_code_on_emulated_warps_matches_reference(nf):
    """The kernel's device code (sb_nsq_warp.cuh) compiled for the host, 16 emulated lanes per case and two different cases
    per warp (the emulation's barriers wait for exactly the lanes a collective names); the last warp's second group shadows
    the last case, as an odd batch does.  Scratch outputs are poisoned before every packet."""
    table = case_table(nf)
    st0, fr = _stack(table)
    compare(table, nf, sim.nsq_run(st0, fr, nf, emu="gw16"), ref_outputs(nf), "emulated kernel")


def _gcov_counts(gcda_dir, src):
    """{line: count} of one source file from gcov's JSON (the .gcno copied beside the .gcda)."""
    base = os.path.splitext(src)[0]
    shutil.copy(os.path.join(nsq_ref.COV_DIR, "obj", base + ".gcno"), gcda_dir)
    r = subprocess.run(["gcov", "--json-format", "--stdout", "-o", gcda_dir, base + ".gcda"], cwd=gcda_dir,
                       capture_output=True, text=True, check=True)
    counts = {}
    for doc in r.stdout.splitlines():
        if not doc.startswith("{"):
            continue
        for f in json.loads(doc)["files"]:
            if os.path.basename(f["file"]) == src:
                for ln in f["lines"]:
                    counts[ln["line_number"]] = counts.get(ln["line_number"], 0) + ln["count"]
    return counts


MIN_COUNT = {"rdcx1_low": 10000, "rdcx1_high": 10000, "rdcx1_mid": 10000, "randsync": 1000, "reset_k2": 20,
             "rewhite": 200, "ltp_scale": 500, "gain_adj": 1000, "judge_sample": 10000}


def test_case_tables_reach_their_branches(tmp_path):
    """The tables through a coverage build of the reference library (in a subprocess: the counts are written at exit, to
    GCOV_PREFIX), then the count of every anchor line; more replacement passes than samples (several de-synchronised states
    in one sample); and from the outputs: a pulse of magnitude 64 (the residual clamp), a saturated output sample, the
    32767 clamp of the inverse gain."""
    if not os.path.exists(nsq_ref.COV_LIB):
        pytest.skip("oracle/_ref/cov not built (needs the reference sources at build time)")
    if shutil.which("gcov") is None:
        pytest.skip("gcov not installed")
    anchors = nsq_ref.read_anchors()
    sat = False
    for nf in TABLES:
        table = case_table(nf)
        st0, fr = _stack(table)
        np.savez(tmp_path / ("t%d.npz" % nf), st0=st0, fr=fr)
        rout, rst = ref_outputs(nf)
        assert (np.abs(rout["q_md"].astype(np.int32)) == 64).any(), "no pulse at the residual clamp (nf=%d)" % nf
        sat |= bool((np.abs(rst["xq"].astype(np.int32)) >= 32767).any())
        inv = [2 ** 32 // int(g) for g in fr["Gains_Q16"].reshape(-1)]
        assert max(inv) > 32767, "no gain small enough for the clamp of the inverse"
    assert sat, "no saturated output sample"
    prefix = tmp_path / "gcda"
    code = ("import sys, numpy as np; sys.path.insert(0, %r)\n"
            "from oracle import nsq_ref\n"
            "R = nsq_ref.RefNsq(nsq_ref.COV_LIB)\n"
            "for nf in %r:\n"
            "    t = np.load(%r %% nf)\n"
            "    for s, f in zip(t['st0'], t['fr']): R.run(s, f)\n") % (ROOT, TABLES, str(tmp_path / "t%d.npz"))
    # the library records each .gcda under the absolute path of its build directory; stripping more leading directories
    # than that path has puts every file straight into the prefix, wherever the tree was built
    env = dict(os.environ, GCOV_PREFIX=str(prefix), GCOV_PREFIX_STRIP="4096")
    run = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    src = anchors["gain_adj"][0]
    gcda = prefix / (os.path.splitext(src)[0] + ".gcda")
    assert gcda.is_file(), "no %s written; files under the prefix: %s; stderr: %s" % (
        gcda.name, sorted(os.path.relpath(os.path.join(d, f), prefix) for d, _, fs in os.walk(prefix) for f in fs)[:20], run.stderr)
    counts = _gcov_counts(str(prefix), src)
    seen = {name: counts.get(line, 0) for name, (_, line) in anchors.items()}
    print("anchor counts:", json.dumps(seen))
    for name, n in MIN_COUNT.items():
        assert seen[name] >= n, "%s (%s:%d) reached %d times, want >= %d" % (name, src, anchors[name][1], seen[name], n)
    assert seen["judge_pass"] > seen["judge_sample"], "never more than one replacement pass in a sample"


@pytest.mark.gpu
@pytest.mark.parametrize("nf", TABLES)
def test_kernel_on_gpu_matches_reference(nf):
    """The device code on the H100 (sb_ops_nsq: nsq_packet_warp in sb_enc_nsq_kernel's layout, one launch per packet)."""
    if not os.path.exists(OPS_LIB):
        pytest.fail(OPS_LIB + " missing: __graft_entry__.build() builds it")
    L = C.CDLL(OPS_LIB)
    L.nsq_io_sizes.argtypes = [C.c_void_p]
    nsq_ref.check_sizes(L)
    L.sb_ops_nsq.argtypes = [C.c_int] * 3 + [C.c_void_p] * 4
    table = case_table(nf)
    st0, fr = _stack(table)
    n, nfr = fr.shape
    out = np.zeros((n, nfr), nsq_ref.FRAME_OUT)
    st = np.zeros((n, nfr // nf, 3), nsq_ref.STATE)
    r = L.sb_ops_nsq(n, nfr // nf, nf, st0.ctypes.data, fr.ctypes.data, out.ctypes.data, st.ctypes.data)
    assert r == 0, "CUDA harness call failed with error %d" % r
    compare(table, nf, (out, st), ref_outputs(nf), "GPU kernel")
