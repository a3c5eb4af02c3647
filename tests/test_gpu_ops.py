"""Single routines of the analysis kernel, run on the GPU one warp per case and compared bit-exactly with the reference.

The encoder-level GPU tests reach only the branches that their signals reach.  Here the warp-cooperative routines of
sb_coop.cuh and the device forms of the sb_common.cuh primitives run on their own (tests/gpu_ops/ops.cu, compiled with the
library's flags) over case tables built to reach every branch, and each result is compared with:
  * the unmodified reference (oracle/_ref/libjc1_fix.so) where it exports the function: SKP_Silk_burg_modified, A2NLSF,
    schur, schur64, k2a, k2a_Q16, warped_autocorrelation_FIX, quant_LTP_gains_FIX, lin2log, log2lin, sigm_Q15;
  * a plain big-integer statement of the reference macro (SKP_Silk_macros.h, SKP_Silk_Inlines.h,
    SKP_Silk_SigProc_FIX.h) for the primitives it inlines.
Every case stays inside the reference's input contract; cases the reference leaves undefined are named where they are left
out.  The unmarked test at the end runs the case tables through the reference alone and checks that each branch the tables
are meant to reach is reached, so that a table cannot silently stop covering its branch."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.util import load_clip

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPS_LIB = os.path.join(ROOT, "tests", "_gpu_ops", "libsb_gpu_ops.so")

I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
XMAX = 4 * 88                 # burg case buffer per half (sb_ops_burg_xmax)
SHAPE_WIN, SHAPE_ORDER = 120, 16
WARPING_Q16 = 7864
# SKP_FIX_CONST(2.5e-5f, 32): the float literal times 2^32, + 0.5, in double
WNF_Q32 = int(float(np.float32(2.5e-5)) * 2.0 ** 32 + 0.5)


# ---------------------------------------------------------------------------------------------------------------------
# libraries
# ---------------------------------------------------------------------------------------------------------------------
def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def ref_lib():
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref not built")
    L = ref.lib("fix").lib
    for name in ("SKP_Silk_schur", "SKP_Silk_schur64", "SKP_Silk_lin2log", "SKP_Silk_log2lin", "SKP_Silk_sigm_Q15"):
        getattr(L, name).restype = C.c_int32
    return L


@pytest.fixture(scope="module")
def ref():
    return ref_lib()


@pytest.fixture(scope="module")
def ops():
    if not os.path.exists(OPS_LIB):
        pytest.fail(OPS_LIB + " missing: __graft_entry__.build() builds it")
    L = C.CDLL(OPS_LIB)
    assert L.sb_ops_burg_xmax() == XMAX
    return L


def _ok(r):
    assert r == 0, "CUDA harness call failed with error %d" % r


# ---------------------------------------------------------------------------------------------------------------------
# big-integer statements of the reference macros
# ---------------------------------------------------------------------------------------------------------------------
def w32(x):
    return ((int(x) + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def s16(x):
    return ((int(x) + (1 << 15)) & 0xFFFF) - (1 << 15)


def clz32(x):
    x &= 0xFFFFFFFF
    return 32 - x.bit_length()


def cdiv(a, b):          # C integer division (truncates toward zero)
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def smulwb(a, b):        # macros.h:34 (== floor(a * (int16)b / 2^16))
    return (a * s16(b)) >> 16


def smulwt(a, b):        # macros.h:40
    return (a * (w32(b) >> 16)) >> 16


def smmul(a, b):
    return (a * b) >> 32


def rshift_round(a, s):
    return (a >> 1) + (a & 1) if s == 1 else ((a >> (s - 1)) + 1) >> 1


def smulww(a, b):        # macros.h:61: SMULWB(a, b) + a * RSHIFT_ROUND(b, 16), wrapping
    return w32(smulwb(a, b) + a * rshift_round(b, 16))


def sat32(x):
    return max(I32_MIN, min(I32_MAX, x))


def lshift_sat32(a, s):  # SigProc_FIX.h:576
    return w32(max(I32_MIN >> s, min(I32_MAX >> s, a)) << s)


def div32_varq(a32, b32, q):          # Inlines.h:124-166 (a32 != INT_MIN: SKP_abs leaves it negative, headroom -1)
    a_h = clz32(abs(a32)) - 1
    a_n = w32(a32 << a_h)
    b_h = clz32(abs(b32)) - 1
    b_n = w32(b32 << b_h)
    inv = cdiv(I32_MAX >> 2, b_n >> 16)
    res = smulwb(a_n, inv)
    a_n = w32(a_n - w32(smmul(b_n, res) << 3))
    res = w32(res + smulwb(a_n, inv))
    ls = 29 + a_h - b_h - q
    if ls <= 0:
        return lshift_sat32(res, -ls)
    return res >> ls if ls < 32 else 0


def inverse32_varq(b32, q):           # Inlines.h:170-207
    b_h = clz32(abs(b32)) - 1
    b_n = w32(b32 << b_h)
    inv = cdiv(I32_MAX >> 2, b_n >> 16)
    res = w32(inv << 16)
    err = w32(w32(-smulwb(b_n, inv)) << 3)
    res = w32(res + smulww(err, inv))
    ls = 61 - b_h - q
    if ls <= 0:
        return lshift_sat32(res, -ls)
    return res >> ls if ls < 32 else 0


def sqrt_approx(x):                   # Inlines.h:71-96 with CLZ_FRAC (Inlines.h:57-66) and the generic ROR32
    if x <= 0:
        return 0
    lz = clz32(x)
    rot = 24 - lz
    u = x & 0xFFFFFFFF
    r = ((u << (32 - rot)) | (u >> rot)) if rot > 0 else (((u << -rot) | (u >> (32 + rot))) if rot < 0 else u)
    frac = r & 0x7F
    y = 32768 if lz & 1 else 46214
    y >>= lz >> 1
    return y + smulwb(y, 213 * frac)


def float2int(x):
    # SigProc_FIX.h:629 on the reference's x86 target: cvttsd2si returns INT_MIN for NaN and out-of-range values (ISO C
    # leaves that cast undefined; the device form states the x86 result explicitly)
    v = x + 0.5 if x > 0 else x - 0.5
    return trunc_i32(v)


def trunc_i32(v):
    if not (-2147483649.0 < v < 2147483648.0):
        return I32_MIN
    return int(v)


# ---------------------------------------------------------------------------------------------------------------------
# primitives on the device
# ---------------------------------------------------------------------------------------------------------------------
OP = {n: i for i, n in enumerate((
    "smulwb", "smulwt", "smmul", "add_sat32", "sub_sat32", "clz32", "clz64", "div_q29", "div32_varq", "inverse32_varq",
    "sqrt_approx", "lin2log", "log2lin", "sigm_q15", "lshift_sat32", "popc32", "ctz32", "float2int", "trunc_i32", "smulww"))}

EDGE32 = [0, 1, -1, 2, -2, 3, 255, -256, 32767, -32768, 32768, -32769, 65535, 65536, -65536, 0x12345678, -0x12345678,
          (1 << 30) - 1, 1 << 30, -(1 << 30), I32_MAX - 1, I32_MAX, I32_MIN + 1, I32_MIN]


def dev_prim(ops, name, a, b=None, c=None, f=None):
    n = len(a) if f is None else len(f)
    A = np.ascontiguousarray(np.asarray(a if a is not None else np.zeros(n), np.int64))
    B = np.ascontiguousarray(np.asarray(b if b is not None else np.zeros(n), np.int64))
    Cc = np.ascontiguousarray(np.asarray(c if c is not None else np.zeros(n), np.int64))
    F = np.ascontiguousarray(np.asarray(f if f is not None else np.zeros(n), np.float64))
    out = np.zeros(n, np.int64)
    _ok(ops.sb_ops_prim(OP[name], _p(A), _p(B), _p(Cc), _p(F), _p(out), n))
    return out


def rand32(rng, n):
    """Uniform int32 mixed with values at every magnitude (uniform draws are almost all near full scale)."""
    u = rng.integers(I32_MIN, I32_MAX, n, endpoint=True)
    sh = rng.integers(0, 31, n)
    return np.where(rng.random(n) < 0.5, u, u >> sh)


def _mismatch(name, args, got, want):
    bad = np.nonzero(np.asarray(got) != np.asarray(want))[0]
    if len(bad):
        i = int(bad[0])
        raise AssertionError("%s: %d of %d differ, first at %s: device %d, reference %d"
                             % (name, len(bad), len(got), tuple(int(np.asarray(x)[i]) for x in args), int(got[i]), int(want[i])))


@pytest.mark.gpu
def test_smulwb_smulwt_every_b16_against_edge_a(ops):
    b16 = np.arange(-32768, 32768, dtype=np.int64)
    for a in EDGE32:
        av = np.full(b16.size, a, np.int64)
        # smulwb reads the low half of b, smulwt the high half: exercise both with the other half filled
        bw = (b16 & 0xFFFF) | (np.int64(0x5A5A) << 16)
        bw = np.where(bw >= 1 << 31, bw - (1 << 32), bw)
        _mismatch("smulwb", (av, bw), dev_prim(ops, "smulwb", av, bw), (av * b16) >> 16)
        bt = (b16 << 16) | 0xA5A5
        bt = np.where(bt >= 1 << 31, bt - (1 << 32), bt)
        _mismatch("smulwt", (av, bt), dev_prim(ops, "smulwt", av, bt), (av * b16) >> 16)


@pytest.mark.gpu
def test_products_and_saturating_sums(ops):
    rng = np.random.Generator(np.random.PCG64(71))
    e = np.array(EDGE32, np.int64)
    a = np.concatenate([np.repeat(e, e.size), rand32(rng, 200000)])
    b = np.concatenate([np.tile(e, e.size), rand32(rng, 200000)])
    _mismatch("smmul", (a, b), dev_prim(ops, "smmul", a, b), (a * b) >> 32)
    _mismatch("add_sat32", (a, b), dev_prim(ops, "add_sat32", a, b), np.clip(a + b, I32_MIN, I32_MAX))
    _mismatch("sub_sat32", (a, b), dev_prim(ops, "sub_sat32", a, b), np.clip(a - b, I32_MIN, I32_MAX))
    want = [smulww(int(x), int(y)) for x, y in zip(a[:50000], b[:50000])]
    _mismatch("smulww", (a[:50000], b[:50000]), dev_prim(ops, "smulww", a[:50000], b[:50000]), want)


@pytest.mark.gpu
def test_bit_utilities(ops):
    rng = np.random.Generator(np.random.PCG64(72))
    x = np.concatenate([np.array(EDGE32, np.int64), [w32(1 << k) for k in range(32)], [w32((1 << k) - 1) for k in range(33)],
                        rand32(rng, 100000)]).astype(np.int64)
    _mismatch("clz32", (x,), dev_prim(ops, "clz32", x), [clz32(int(v)) for v in x])
    _mismatch("popc32", (x,), dev_prim(ops, "popc32", x), [bin(int(v) & 0xFFFFFFFF).count("1") for v in x])
    nz = x[x != 0]
    _mismatch("ctz32", (nz,), dev_prim(ops, "ctz32", nz), [((int(v) & -int(v)) & 0xFFFFFFFF).bit_length() - 1 for v in nz])
    h = np.concatenate([[0, 1, -1, 1 << 32, (1 << 32) - 1, -(1 << 32), (1 << 62), -(1 << 63), (1 << 63) - 1],
                        [1 << k for k in range(63)], rng.integers(-(1 << 63), (1 << 63) - 1, 50000, dtype=np.int64),
                        rng.integers(0, 1 << 32, 50000, dtype=np.int64)]).astype(np.int64)
    _mismatch("clz64", (h,), dev_prim(ops, "clz64", h), [64 - (int(v) & 0xFFFFFFFFFFFFFFFF).bit_length() for v in h])
    sh = np.concatenate([np.repeat(np.arange(31), len(EDGE32)), rng.integers(0, 31, 50000)])
    v = np.concatenate([np.tile(np.array(EDGE32, np.int64), 31), rand32(rng, 50000)])
    _mismatch("lshift_sat32", (v, sh), dev_prim(ops, "lshift_sat32", v, sh), [lshift_sat32(int(p), int(s)) for p, s in zip(v, sh)])


@pytest.mark.gpu
def test_div_q29_every_normalised_divisor(ops):
    """Exhaustive over the divisors DIV32_varQ / INVERSE32_varQ produce (16384 <= |d| <= 32768): the float reciprocal
    (__frcp_rn, __float2int_rz) plus the correction step must equal the reference's C division SKP_DIV32_16."""
    d = np.concatenate([np.arange(16384, 32769), -np.arange(16384, 32769)]).astype(np.int64)
    n = I32_MAX >> 2
    want = np.where(d > 0, n // d, -(n // -d))
    _mismatch("div_q29", (d,), dev_prim(ops, "div_q29", d), want)


@pytest.mark.gpu
def test_div32_varq_and_inverse32_varq(ops):
    rng = np.random.Generator(np.random.PCG64(73))
    e = [v for v in EDGE32 if v != I32_MIN]      # INT_MIN: SKP_abs leaves it negative and the headroom is -1 (undefined)
    a, b, q = [], [], []
    for x in e:
        for y in e:
            if y != 0:
                for qq in (0, 14, 16, 31):
                    a.append(x); b.append(y); q.append(qq)
    ra, rb = rand32(rng, 30000), rand32(rng, 30000)
    keep = (ra != I32_MIN) & (rb != I32_MIN) & (rb != 0)
    a += list(ra[keep]); b += list(rb[keep]); q += list(rng.integers(0, 32, int(keep.sum())))
    a, b, q = (np.array(v, np.int64) for v in (a, b, q))
    _mismatch("div32_varq", (a, b, q), dev_prim(ops, "div32_varq", a, b, q),
              [div32_varq(int(x), int(y), int(z)) for x, y, z in zip(a, b, q)])
    qi = np.maximum(q, 1)                        # Qres > 0 (Inlines.h:180)
    _mismatch("inverse32_varq", (b, qi), dev_prim(ops, "inverse32_varq", b, None, qi), [inverse32_varq(int(y), int(z)) for y, z in zip(b, qi)])


@pytest.mark.gpu
def test_sqrt_lin2log_log2lin_sigm(ops, ref):
    rng = np.random.Generator(np.random.PCG64(74))
    x = np.concatenate([np.array(EDGE32, np.int64), np.arange(-16, 4096), [1 << k for k in range(31)], rand32(rng, 60000)])
    _mismatch("sqrt_approx", (x,), dev_prim(ops, "sqrt_approx", x), [sqrt_approx(int(v)) for v in x])
    pos = x[x > 0]                               # lin2log: positive input (CLZ_FRAC of 0 rotates by 24 - 32)
    _mismatch("lin2log", (pos,), dev_prim(ops, "lin2log", pos), [ref.SKP_Silk_lin2log(int(v)) for v in pos])
    lg = np.arange(-1, 31 * 128 + 1, dtype=np.int64)      # every input from -1 to 31 * 128
    _mismatch("log2lin", (lg,), dev_prim(ops, "log2lin", lg), [ref.SKP_Silk_log2lin(int(v)) for v in lg])
    s = np.arange(-32768, 32768, dtype=np.int64)          # every int16
    _mismatch("sigm_q15", (s,), dev_prim(ops, "sigm_q15", s), [ref.SKP_Silk_sigm_Q15(int(v)) for v in s])


@pytest.mark.gpu
def test_float2int_and_trunc(ops):
    rng = np.random.Generator(np.random.PCG64(75))
    f = np.concatenate([[0.0, -0.0, 0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 0.49999999999999994, -0.49999999999999994,
                         2147483646.5, 2147483647.0, 2147483647.4, 2147483647.5, 2147483648.0, -2147483648.0,
                         -2147483648.4, -2147483648.5, -2147483649.0, 1e300, -1e300, np.inf, -np.inf, np.nan],
                        rng.normal(0, 1e4, 20000), rng.uniform(-3e9, 3e9, 20000)])
    _mismatch("float2int", (f,), dev_prim(ops, "float2int", None, f=f), [float2int(float(v)) for v in f])
    _mismatch("trunc_i32", (f,), dev_prim(ops, "trunc_i32", None, f=f), [trunc_i32(float(v)) for v in f])


# ---------------------------------------------------------------------------------------------------------------------
# case tables (shared by the GPU comparisons and the branch-reach test)
# ---------------------------------------------------------------------------------------------------------------------
def _frame(rng, kind, n, level):
    t = np.arange(n)
    if kind == "noise":
        v = rng.normal(0, level, n)
    elif kind == "lsb":          # +-level LSB, uniform
        v = rng.integers(-level, level + 1, n)
    elif kind == "dc":
        v = np.full(n, level)
    elif kind == "nyquist":
        v = level * np.where(t % 2 == 0, 1, -1)
    elif kind == "impulse":
        v = np.zeros(n); v[rng.integers(0, n)] = level
    elif kind == "tone":
        v = level * np.sin(2 * np.pi * rng.uniform(0.01, 0.49) * t + rng.uniform(0, 6.3))
    elif kind == "square":
        v = np.where((t // 7) % 2 == 0, level, -level)
    else:                        # speech
        clip = load_clip()
        o = int(rng.integers(0, len(clip) - n))
        v = clip[o:o + n].astype(np.float64) * level
    return np.clip(np.round(v), -32768, 32767).astype(np.int16)


def _at_energy(rng, n, lo, hi):
    """White noise scaled so that its energy (sum of squares) lies in [lo, hi)."""
    for _ in range(100):
        v = rng.normal(0, 1, n)
        e = float(np.sum(v * v))
        g = np.sqrt(rng.uniform(lo, hi) / e)
        x = np.clip(np.round(v * g), -32768, 32767).astype(np.int16)
        if lo <= int(np.sum(x.astype(np.int64) ** 2)) < hi:
            return x
    raise AssertionError("no frame at that energy")


def burg_cases(D):
    """(nb0, nb1, L, WhiteNoiseFrac_Q32, x0, x1) as the encoder calls c_burg2: order 10 over four 50-sample blocks and the
    second half of them (find_LPC), order 8 over four 88-sample blocks (high band).  Per branch:
      rshifts <= -2 (the mlaw / smlaww arithmetic): +-1..+-8 LSB noise, single LSB clicks, energies giving rshifts -2, -3;
      rshifts = MAX_RSHIFTS with energy >= 2^31 (sum_sqr_shift fallback): full-scale noise, square and Nyquist;
      early termination |num| >= nrg: pure tones, Nyquist alternation, DC;
      the ordinary range in between: speech and noise at several levels."""
    rng = np.random.Generator(np.random.PCG64(100 + D))
    L = 50 if D == 10 else 88
    nbs = [(4, 2), (4, 4)] if D == 10 else [(4, 4)]
    kinds = [("lsb", 1), ("lsb", 2), ("lsb", 3), ("lsb", 8), ("noise", 1), ("noise", 3), ("noise", 8), ("impulse", 1),
             ("impulse", -1), ("impulse", 8), ("dc", 1), ("dc", -1), ("nyquist", 1), ("nyquist", 8), ("nyquist", 32767),
             ("tone", 3), ("tone", 1000), ("tone", 32000), ("square", 32767), ("noise", 20000), ("noise", 32767),
             ("speech", 1.0), ("speech", 1 / 8), ("speech", 1 / 1024), ("noise", 500), ("dc", 32767), ("dc", -32768)]
    frames = []
    for k, lev in kinds:
        for _ in range(3):
            frames.append(_frame(rng, k, 4 * L, lev))
    # rshifts = 3 - clz32(energy) for energies below 2^30: -2 <-> [2^26, 2^27), -3 <-> [2^25, 2^26)
    for lo, hi in ((1 << 26, 1 << 27), (1 << 25, 1 << 26), (1 << 24, 1 << 25), (1 << 30, 1 << 31)):
        for _ in range(4):
            frames.append(_at_energy(rng, 4 * L, lo, hi))
    frames.append(np.zeros(4 * L, np.int16))
    cases = []
    for i, f in enumerate(frames):
        for nb0, nb1 in nbs:
            other = frames[(i * 7 + 3) % len(frames)]
            # the second half's frame starts where find_LPC's does (block nb0 - nb1) when nb1 < nb0
            x1 = other[(nb0 - nb1) * L:] if nb1 < nb0 else other
            cases.append((nb0, nb1, L, WNF_Q32, f, np.ascontiguousarray(x1[:nb1 * L])))
    return cases


def ref_burg(ref, x, nb, L, wnf, D):
    x = np.ascontiguousarray(x, np.int16)
    rn, rq, A = C.c_int32(0), C.c_int(0), np.zeros(16, np.int32)
    ref.SKP_Silk_burg_modified(C.byref(rn), C.byref(rq), _p(A), _p(x), C.c_int(L), C.c_int(nb), C.c_int32(wnf), C.c_int(D))
    return rn.value, rq.value, A[:D].copy()


def _poly_from_roots(roots):
    p = np.array([1.0 + 0j])
    for r in roots:
        p = np.convolve(p, [1.0, -r])
    return p.real


def a2nlsf_cases(D):
    """a_Q16 [D] (A(z) = 1 - sum a[k] z^-(k+1)), per branch:
      regular: Burg-like predictors of stable filters (roots inside the circle);
      widening retry loop: roots on and just outside the unit circle, double roots;
      white-spectrum fallback after 30 widenings: large random coefficients and roots far outside the circle;
      the forced-root path and |ylo| >= 65536 interpolation: every walk with an alternating-polynomial step, and large
      coefficients (the polynomials scale with a_Q16)."""
    rng = np.random.Generator(np.random.PCG64(200 + D))
    out = []

    def add(roots, gain=1.0):
        p = _poly_from_roots(roots)
        a = -p[1:D + 1] * gain
        q = np.round(a * 65536.0)
        if np.all(np.abs(q) < 2 ** 30):
            out.append(q.astype(np.int64))

    def pairs(radii):
        r = []
        for rad in radii:
            th = rng.uniform(0.05, np.pi - 0.05)
            r += [rad * np.exp(1j * th), rad * np.exp(-1j * th)]
        return r

    for _ in range(40):
        add(pairs(rng.uniform(0.3, 0.97, D // 2)))
    for rad in (0.999, 1.0, 1.0001, 1.01, 1.05, 1.2, 1.5, 2.0, 3.0):
        for _ in range(6):
            add(pairs(np.concatenate([[rad], rng.uniform(0.3, 0.95, D // 2 - 1)])))
    for _ in range(6):
        add(pairs(np.full(D // 2, rng.uniform(1.0, 1.3))))
    for _ in range(6):                  # double roots
        r = pairs(rng.uniform(0.9, 1.0, D // 4))
        add((r + r + pairs([0.5] * (D // 2 - 2 * (D // 4))))[:D])
    for mag in (1 << 16, 1 << 18, 1 << 20, 1 << 22, 1 << 24):
        for _ in range(6):
            out.append(rng.integers(-mag, mag, D).astype(np.int64))
    out.append(np.zeros(D, np.int64))
    return out


def ref_a2nlsf(ref, a, D):
    a32 = np.ascontiguousarray(np.asarray(a, np.int32))
    nl = np.zeros(D, np.int32)
    ref.SKP_Silk_A2NLSF(_p(nl), _p(a32), C.c_int(D))
    return nl, a32


def a2nlsf_walk(ref, a, D):
    """SKP_Silk_A2NLSF (A2NLSF.c:46-287, QPoly 16, no oversampled cosine table, 3 bisections) in big integers, counting
    the branches that its outputs do not show: a root found in the same grid interval as the previous one (the search
    restarts there with the forced value +-4096 as ylo) and the interpolation for |ylo| >= 65536.
    Returns (NLSF, widened a_Q16, roots in the same interval, |ylo| >= 65536 interpolations)."""
    cos = np.ctypeslib.as_array((C.c_int * 129).in_dll(ref, "SKP_Silk_LSFCosTab_FIX_Q12")).tolist()
    dd = D // 2
    a = [int(v) for v in a]

    def init():
        P, Q = [0] * (dd + 1), [0] * (dd + 1)
        P[dd] = Q[dd] = 1 << 16
        for k in range(dd):
            P[k] = w32(-a[dd - k - 1] - a[dd + k])
            Q[k] = w32(-a[dd - k - 1] + a[dd + k])
        for k in range(dd, 0, -1):
            P[k - 1] = w32(P[k - 1] - P[k])
            Q[k - 1] = w32(Q[k - 1] + Q[k])
        for p in (P, Q):
            for k in range(2, dd + 1):
                for n in range(dd, k, -1):
                    p[n - 2] = w32(p[n - 2] - p[n])
                p[k - 2] = w32(p[k - 2] - w32(p[k] << 1))
        return P, Q

    def ev(p, x):
        y, xq = p[dd], x << 4
        for n in range(dd - 1, -1, -1):
            y = w32(p[n] + smulww(y, xq))
        return y

    def start(PQ):
        ylo = ev(PQ[0], cos[0])
        if ylo < 0:
            return PQ[1], ev(PQ[1], cos[0]), 1, [0]
        return PQ[0], ylo, 0, []

    nlsf = [0] * D
    PQ = init()
    p, ylo, root_ix, _ = start(PQ)
    xlo, k, i, forced, same, big = cos[0], 1, 0, False, 0, 0
    while True:
        xhi = cos[k]
        yhi = ev(p, xhi)
        if (ylo <= 0 <= yhi) or (ylo >= 0 >= yhi):
            same += forced
            ffrac = -256
            for m in range(3):
                xmid = rshift_round(xlo + xhi, 1)
                ymid = ev(p, xmid)
                if (ylo <= 0 <= ymid) or (ylo >= 0 >= ymid):
                    xhi, yhi = xmid, ymid
                else:
                    xlo, ylo = xmid, ymid
                    ffrac += 128 >> m
            if abs(ylo) < 65536:
                den = w32(ylo - yhi)
                nom = w32((ylo << 5) + (den >> 1))
                if den != 0:
                    ffrac += cdiv(nom, den)
            else:
                big += 1
                ffrac += cdiv(ylo, w32(ylo - yhi) >> 5)
            nlsf[root_ix] = min((k << 8) + ffrac, 32767)
            root_ix += 1
            if root_ix >= D:
                break
            p = PQ[root_ix & 1]
            xlo = cos[k - 1]
            ylo = (1 - (root_ix & 2)) << 12
            forced = True
        else:
            forced = False
            k += 1
            xlo, ylo = xhi, yhi
            if k > 128:
                i += 1
                if i > 30:
                    return list(white_nlsf(D)), a, same, big
                t = chirp = 65536 - (10 + i) * i
                for j in range(D - 1):
                    a[j] = smulww(a[j], t)
                    t = smulww(chirp, t)
                a[D - 1] = smulww(a[D - 1], t)
                PQ = init()
                p, ylo, root_ix, _ = start(PQ)
                xlo, k = cos[0], 1
    return nlsf, a, same, big


def white_nlsf(D):
    n0 = (1 << 15) // (D + 1)
    return np.array([n0] + [(k + 1) * n0 for k in range(1, D)], np.int32)


def schur_py(c, order):
    """SKP_Silk_schur (schur.c:40-93) in big integers; returns (rc_Q15, energy, in_contract, clipped).  in_contract is False
    when a step would overflow int32 (signed overflow in the reference: undefined, so such cases are not tested)."""
    lz = clz32(c[0])
    if lz < 2:
        C0 = [v >> 1 for v in c]
    elif lz > 2:
        C0 = [v << (lz - 2) for v in c]
    else:
        C0 = list(c)
    ok = all(I32_MIN <= v <= I32_MAX for v in C0)
    Ca, Cb = list(C0), list(C0)
    rc, clipped = [], False
    for k in range(order):
        d = max(Cb[0] >> 15, 1)
        if Ca[k + 1] == I32_MIN and d == 1:
            ok = False
        r = -cdiv(Ca[k + 1], d)
        if r > 32767 or r < -32768:
            clipped = True
        r = max(-32768, min(32767, r))
        rc.append(r)
        for n in range(order - k):
            t1, t2 = Ca[n + k + 1], Cb[n]
            for v in (2 * t1, 2 * t2):
                ok &= I32_MIN <= v <= I32_MAX
            Ca[n + k + 1] = t1 + smulwb(2 * t2, r)
            Cb[n] = t2 + smulwb(2 * t1, r)
            ok &= I32_MIN <= Ca[n + k + 1] <= I32_MAX and I32_MIN <= Cb[n] <= I32_MAX
    return rc, Cb[0], ok, clipped


def schur_cases(order, positive_definite_only=False):
    """c [order + 1] with c[0] > 0: autocorrelations of real frames (positive definite), then non-positive-definite rows
    (|c[k]| close to or above c[0], random signs) that drive the reflection coefficient into its int16 clip; only rows
    whose recursion stays inside int32 are kept (see schur_py)."""
    rng = np.random.Generator(np.random.PCG64(300 + order))
    out = []
    for kind, lev in (("noise", 1000), ("tone", 8000), ("speech", 1.0), ("lsb", 1), ("nyquist", 100), ("impulse", 3), ("dc", 5)):
        for _ in range(6):
            x = _frame(rng, kind, 240, lev).astype(np.int64)
            r = [int(np.dot(x[:240 - k], x[k:])) for k in range(order + 1)]
            sh = max(0, max(abs(v) for v in r).bit_length() - 31)
            r = [v >> sh for v in r]
            if r[0] > 0:
                out.append(r)
    if positive_definite_only:
        return out
    tries = 0
    while len(out) < 160 and tries < 20000:
        tries += 1
        c0 = int(rng.integers(1, 1 << int(rng.integers(4, 31))))
        spread = float(rng.choice([0.3, 0.45, 0.6, 0.9, 1.3]))
        c = [c0] + [int(v) for v in np.round(c0 * rng.uniform(-spread, spread, order))]
        c = [max(I32_MIN + 1, min(I32_MAX, v)) for v in c]
        if schur_py(c, order)[2]:
            out.append(c)
    return out


def schur64_cases():
    """c [17] for schur64_r at the shaping order: autocorrelations of real frames and rows with c[0] <= 0 (the early
    return).  Non-positive-definite rows are left out: their residual energy can reach 0, and DIV32_varQ by 0 is outside
    the reference's contract (it traps)."""
    return schur_cases(16, positive_definite_only=True) + [[0] * 17, [-5] + [3] * 16, [I32_MIN] + [0] * 16]


def warped_cases():
    """Four windows [4][120] and a warping value per case: full-scale, few-LSB and all-zero windows (the shift selection
    at both ends of its range) at the warpings the encoder uses (WARPING_Q16 + coding quality * 0.01 in Q18)."""
    rng = np.random.Generator(np.random.PCG64(500))
    kinds = [("lsb", 1), ("lsb", 3), ("impulse", 1), ("noise", 8), ("noise", 32767), ("square", 32767), ("nyquist", 32767),
             ("dc", -32768), ("tone", 32000), ("speech", 1.0), ("speech", 1 / 1024), ("noise", 300)]
    warps = [WARPING_Q16, WARPING_Q16 + 164, WARPING_Q16 + 327, WARPING_Q16 + 655]
    out = []
    for i in range(len(kinds) * 3):
        w = np.stack([_frame(rng, kinds[(i + j) % len(kinds)][0], SHAPE_WIN, kinds[(i + j) % len(kinds)][1]) for j in range(4)])
        out.append((w, warps[i % len(warps)]))
    out.append((np.zeros((4, SHAPE_WIN), np.int16), WARPING_Q16))
    return out


def ltp_cases():
    """(B_Q14 [20], W_Q18 [100], mu_Q8): LTP gains in and beyond the codebooks' range with weights from near zero up to
    large diagonal-dominant matrices (products stay inside the reference's int32 arithmetic)."""
    rng = np.random.Generator(np.random.PCG64(600))
    out = []
    for scale in (0, 1, 1 << 8, 1 << 14, 1 << 18, 1 << 20):
        for _ in range(10):
            B = rng.integers(-4000, 20000, 20).astype(np.int16)
            W = np.zeros((4, 5, 5), np.int64)
            for j in range(4):
                m = rng.normal(0, 1, (5, 5))
                m = m @ m.T + np.eye(5)
                W[j] = np.round(m / np.abs(m).max() * scale)
            out.append((B, W.reshape(-1).astype(np.int32), 8))
    out.append((np.zeros(20, np.int16), np.zeros(100, np.int32), 8))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# routines on the device vs the reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("D", [10, 8])
def test_burg_both_halves(ops, ref, D):
    cases = burg_cases(D)
    n = len(cases)
    hdr = np.zeros((n, 4), np.int32)
    xb = np.zeros((n, 2, XMAX), np.int16)
    for i, (nb0, nb1, L, wnf, x0, x1) in enumerate(cases):
        hdr[i] = (nb0, nb1, L, wnf)
        xb[i, 0, :x0.size] = x0
        xb[i, 1, :x1.size] = x1
    nrg, q, A = np.zeros((n, 2), np.int32), np.zeros((n, 2), np.int32), np.zeros((n, 2, 16), np.int32)
    _ok(ops.sb_ops_burg(D, _p(hdr), _p(xb), n, _p(nrg), _p(q), _p(A)))
    for i, (nb0, nb1, L, wnf, x0, x1) in enumerate(cases):
        for h, (x, nb) in enumerate(((x0, nb0), (x1, nb1))):
            rn, rq, rA = ref_burg(ref, x, nb, L, wnf, D)
            got = (int(nrg[i, h]), int(q[i, h]), list(A[i, h, :D]))
            assert got == (rn, rq, list(rA)), ("burg", D, i, h, got, (rn, rq, list(rA)))


@pytest.mark.gpu
@pytest.mark.parametrize("D", [10, 8])
def test_a2nlsf_including_widening_and_fallback(ops, ref, D):
    cases = a2nlsf_cases(D)
    n = len(cases)
    a = np.zeros((n, 16), np.int32)
    for i, c in enumerate(cases):
        a[i, :D] = c
    nl = np.zeros((n, 16), np.int32)
    _ok(ops.sb_ops_a2nlsf(D, _p(a), n, _p(nl)))
    for i, c in enumerate(cases):
        rn, ra = ref_a2nlsf(ref, c, D)
        assert list(nl[i, :D]) == list(rn), ("NLSF", D, i, list(c))
        assert list(a[i, :D]) == list(ra), ("a_Q16 after widening", D, i, list(c))


@pytest.mark.gpu
@pytest.mark.parametrize("order", [10, 16])
def test_schur_and_k2a(ops, ref, order):
    cs = schur_cases(order)
    rng = np.random.Generator(np.random.PCG64(310 + order))
    n = len(cs)
    c = np.zeros((n, 17), np.int32)
    for i, r in enumerate(cs):
        c[i, :order + 1] = r
    rc_in = rng.integers(-32768, 32768, (n, 16)).astype(np.int16)
    rc_in[: n // 2] //= 4                          # also ordinary stable filters
    rc, nrg, A = np.zeros((n, 16), np.int16), np.zeros(n, np.int32), np.zeros((n, 16), np.int32)
    _ok(ops.sb_ops_schur(_p(c), _p(rc_in), order, n, _p(rc), _p(nrg), _p(A)))
    for i in range(n):
        rrc = np.zeros(16, np.int16)
        rn = ref.SKP_Silk_schur(_p(rrc), _p(np.ascontiguousarray(c[i])), C.c_int32(order))
        assert (list(rc[i, :order]), int(nrg[i])) == (list(rrc[:order]), rn), ("schur", order, i, list(c[i, :order + 1]))
        rA = np.zeros(16, np.int32)
        ref.SKP_Silk_k2a(_p(rA), _p(np.ascontiguousarray(rc_in[i])), C.c_int32(order))
        assert list(A[i, :order]) == list(rA[:order]), ("k2a", order, i)


@pytest.mark.gpu
def test_schur64_and_k2a_q16_at_the_shaping_order(ops, ref):
    cs = schur64_cases()
    rng = np.random.Generator(np.random.PCG64(401))
    n = len(cs)
    c = np.ascontiguousarray(np.array(cs, np.int64).astype(np.int32))
    rc_in = rng.integers(-65536, 65536, (n, 16)).astype(np.int32)
    rc_in[: n // 2] //= 3
    rc, nrg, A = np.zeros((n, 16), np.int32), np.zeros(n, np.int32), np.zeros((n, 16), np.int32)
    _ok(ops.sb_ops_schur64(_p(c), _p(rc_in), n, _p(rc), _p(nrg), _p(A)))
    for i in range(n):
        rrc = np.zeros(16, np.int32)
        rn = ref.SKP_Silk_schur64(_p(rrc), _p(np.ascontiguousarray(c[i])), C.c_int32(16))
        assert (list(rc[i]), int(nrg[i])) == (list(rrc), rn), ("schur64", i, list(c[i]))
        rA = np.zeros(16, np.int32)
        ref.SKP_Silk_k2a_Q16(_p(rA), _p(np.ascontiguousarray(rc_in[i])), C.c_int32(16))
        assert list(A[i]) == list(rA), ("k2a_Q16", i)


@pytest.mark.gpu
def test_warped_autocorrelation(ops, ref):
    cases = warped_cases()
    n = len(cases)
    x = np.ascontiguousarray(np.stack([w for w, _ in cases]).astype(np.int16))
    warp = np.array([v for _, v in cases], np.int32)
    corr, scale = np.zeros((n, 4, 17), np.int32), np.zeros((n, 4), np.int32)
    _ok(ops.sb_ops_warped_autocorr(_p(x), _p(warp), n, _p(corr), _p(scale)))
    for i in range(n):
        for j in range(4):
            rc, rs = np.zeros(17, np.int32), C.c_int(0)
            ref.SKP_Silk_warped_autocorrelation_FIX(_p(rc), C.byref(rs), _p(np.ascontiguousarray(x[i, j])), C.c_int16(int(warp[i])),
                                                    C.c_int(SHAPE_WIN), C.c_int(SHAPE_ORDER))
            assert (list(corr[i, j]), int(scale[i, j])) == (list(rc), rs.value), ("warped autocorrelation", i, j, int(warp[i]))


@pytest.mark.gpu
def test_quant_ltp_gains(ops, ref):
    cases = ltp_cases()
    n = len(cases)
    B = np.ascontiguousarray(np.stack([b for b, _, _ in cases]))
    W = np.ascontiguousarray(np.stack([w for _, w, _ in cases]))
    mu = np.array([m for _, _, m in cases], np.int32)
    cbk, per = np.zeros((n, 4), np.int32), np.zeros(n, np.int32)
    Bd = B.copy()
    _ok(ops.sb_ops_quant_ltp_gains(_p(Bd), _p(W), _p(mu), n, _p(cbk), _p(per)))
    for i in range(n):
        rB, rc, rp = B[i].copy(), np.zeros(4, np.int32), C.c_int(0)
        ref.SKP_Silk_quant_LTP_gains_FIX(_p(rB), _p(rc), C.byref(rp), _p(np.ascontiguousarray(W[i])), C.c_int(int(mu[i])), C.c_int(0))
        assert (list(Bd[i]), list(cbk[i]), int(per[i])) == (list(rB), list(rc), rp.value), ("quant_LTP_gains", i)


# ---------------------------------------------------------------------------------------------------------------------
# pitch analysis and NLSF MSVQ: the routines with scalar instances, run in the analysis kernel's 8-warp block layout
# ---------------------------------------------------------------------------------------------------------------------
PITCH_LEN = 320               # 40 ms at 8 kHz
THRES1_Q16 = int(float(np.float32(0.7)) * 65536.0 + 0.5)     # SKP_FIX_CONST(0.7f, 16), the encoder's first-stage threshold


def pitch_cases():
    """(signal [320] at 8 kHz, prevLag, search_thres2_Q15, LTPCorr_Q15 of the previous frame).  Per branch:
      voiced at the lag limits: pulse trains and harmonic tones with periods 16, 17 (minimum lag) and 143, 144 (maximum);
      voiced in between, with and without the previous-lag bias (prevLag > 0, previous correlation 0 / mid / full);
      unvoiced: silence (the first-stage 'uniform' exit), near-silent noise and white noise;
      the scaling shifts of both stages: full-scale pulse trains and square waves."""
    rng = np.random.Generator(np.random.PCG64(700))
    t = np.arange(PITCH_LEN)
    clip = load_clip()
    sigs = []
    for P in (16, 17, 18, 24, 40, 64, 100, 142, 143, 144, 144, 144):
        for amp in (3000, 32767):
            ph = int(rng.integers(0, P))
            pulse = np.where((t + ph) % P == 0, amp, 0)
            sigs.append(pulse)
            tone = sum(np.cos(2 * np.pi * h * (t + ph) / P) / h for h in range(1, 6))
            sigs.append(tone / np.abs(tone).max() * amp)
    sigs += [np.zeros(PITCH_LEN), rng.integers(-2, 3, PITCH_LEN), rng.normal(0, 3000, PITCH_LEN),
             np.where((t // 8) % 2 == 0, 32767, -32767)]
    for _ in range(12):
        o = int(rng.integers(0, len(clip) - 2 * PITCH_LEN))
        sigs.append(clip[o:o + 2 * PITCH_LEN:2].astype(np.float64) * rng.choice([1.0, 0.25]))
    out = []
    for i, s in enumerate(sigs):
        x = np.clip(np.round(s), -32768, 32767).astype(np.int16)
        prev = (0, 0, 16, 60, 144)[i % 5]
        thr = (6554, 11469, 16384, 22938)[i % 4]          # 0.2 .. 0.7 in Q15, the range the encoder's threshold takes
        corr = (0, 16384, 32767)[i % 3] if prev else 0
        out.append((x, prev, thr, corr))
    return out


def ref_pitch(ref, x, prev, thr, corr):
    pitch, lag, cont, c = (C.c_int * 4)(), C.c_int(0), C.c_int(0), C.c_int(corr)
    x = np.ascontiguousarray(x, np.int16)
    r = ref.SKP_Silk_pitch_analysis_core(_p(x), pitch, C.byref(lag), C.byref(cont), C.byref(c), C.c_int(prev),
                                         C.c_int32(THRES1_Q16), C.c_int(thr), C.c_int(8), C.c_int(2), C.c_int(0))
    return list(pitch) + [lag.value, cont.value, c.value, r]


class _CBS(C.Structure):            # SKP_Silk_NLSF_CBS (SKP_Silk_structs.h)
    _fields_ = [("nVectors", C.c_int32), ("CB_NLSF_Q15", C.POINTER(C.c_int16)), ("Rates_Q5", C.POINTER(C.c_int16))]


class _CB(C.Structure):             # SKP_Silk_NLSF_CB_struct
    _fields_ = [("nStages", C.c_int32), ("CBStages", C.POINTER(_CBS)), ("NDeltaMin_Q15", C.c_void_p), ("CDF", C.c_void_p),
                ("StartPtr", C.c_void_p), ("MiddleIx", C.c_void_p)]


def ref_codebook(ref, sigtype):
    """The reference's order-10 codebook of a signal type (control_codec_FIX.c: psNLSF_CB[sigtype]) and its stages as arrays."""
    cb = _CB.in_dll(ref, "SKP_Silk_NLSF_CB%d_10" % sigtype)
    stages = []
    for s in range(cb.nStages):
        st = cb.CBStages[s]
        n = st.nVectors
        stages.append((np.ctypeslib.as_array(st.CB_NLSF_Q15, (n * 10,)).reshape(n, 10).astype(np.int64),
                       np.ctypeslib.as_array(st.Rates_Q5, (n,)).astype(np.int64)))
    return cb, stages


def msvq_search(stages, nlsf, w, mu):
    """The survivor search of NLSF_MSVQ_encode_FIX.c (16 survivors, stable order by value then scan position), returning
    per stage the sorted candidate values and the number of survivors kept, and the first survivor's path."""
    res = [np.array(nlsf, np.int64)]
    rate = [0]
    paths = [[]]
    log = []
    for CB, R in stages:
        vals = []
        for n, r in enumerate(res):
            d = r[None, :] - CB                                  # [nVec, 10]
            err = np.zeros(len(CB), np.int64)
            for m in range(10):
                dd = d[:, m]
                err = err + ((dd * dd * int(w[m])) >> 16)          # SMLAWB(err, SMULBB(diff, diff), w)
            vals += list(zip((err + (rate[n] + R) * mu).tolist(), range(n * len(CB), (n + 1) * len(CB))))
        vals.sort()
        surv = min(16, len(vals))
        best0 = vals[0][0]
        if best0 < I32_MAX // 16:
            thr = best0 + ((16 * best0 * 6554) >> 16)           # SMLAWB(best0, 16 * best0, 0.1 in Q16)
            while vals[surv - 1][0] > thr and surv > 8:
                surv -= 1
        log.append(([v for v, _ in vals], surv))
        nres, nrate, npaths = [], [], []
        for v, e in vals[:surv]:
            n, i = divmod(e, len(CB))
            nres.append(res[n] - CB[i]); nrate.append(rate[n] + int(R[i])); npaths.append(paths[n] + [i])
        res, rate, paths = nres, nrate, npaths
    return log, paths[0]


def msvq_cases():
    """(sigtype, NLSF_Q15 [10], previous quantised NLSF [10], W_Q6 [10], mu_Q15, mu_fluc_red_Q16, deactivate_fluc_red).
    Targets: sorted random vectors and codebook vectors themselves; weights: Laroia-sized values, equal small weights and
    all-zero weights, whose distances tie at the survivor boundaries; mu over the range process_NLSFs gives it, fluctuation reduction on and off.  Weights stay at most
    3000 so that the weighted error sums of the reference stay inside int32."""
    rng = np.random.Generator(np.random.PCG64(800))
    out = []

    def rnd_nlsf():
        v = np.sort(rng.integers(200, 32500, 10))
        return np.maximum.accumulate(v + np.arange(10) * 60).clip(0, 32700)

    for i in range(96):
        sigtype = i % 2
        kind = (i // 2) % 4
        nl = rnd_nlsf()
        if kind == 0:
            w = rng.integers(100, 3000, 10)
        elif kind == 1:
            w = np.full(10, int(rng.integers(1, 4)))
        elif kind == 2:
            w = np.zeros(10, np.int64)
        else:
            w = rng.integers(500, 3000, 10)
            nl = None                      # a codebook vector: filled in by the caller from the reference tables
        mu = int(rng.integers(33, 165)) if sigtype else int(rng.integers(33, 67))
        fluc = int(rng.integers(0, 13108))
        out.append((sigtype, nl, rnd_nlsf(), w.astype(np.int64), mu, fluc, int(i % 3 == 0)))
    # mu = 0 with zero weights: every pair of a stage ties, which no input reaches with mu >= 1 (the codebook rates differ).
    # process_NLSFs never passes mu = 0, but the routine has no such precondition, and this is what reaches the kernel's
    # sequential path for more than 64 pairs at the survivor bound.
    for i in range(8):
        out.append((i % 2, rnd_nlsf(), rnd_nlsf(), np.zeros(10, np.int64), 0, int(rng.integers(0, 13108)), int(i >= 4)))
    return out


def msvq_table(ref):
    cases = []
    rng = np.random.Generator(np.random.PCG64(801))
    books = {s: ref_codebook(ref, s)[1] for s in (0, 1)}
    for sigtype, nl, prev, w, mu, fluc, deact in msvq_cases():
        if nl is None:
            CB = books[sigtype][0][0]
            nl = CB[int(rng.integers(0, len(CB)))]
        cases.append((sigtype, np.asarray(nl, np.int64), np.asarray(prev, np.int64), w, mu, fluc, deact))
    return cases


def ref_msvq(ref, sigtype, nl, prev, w, mu, fluc, deact):
    cb, _ = ref_codebook(ref, sigtype)
    idx = np.zeros(6, np.int32)
    q = np.ascontiguousarray(np.asarray(nl, np.int32))
    ref.SKP_Silk_NLSF_MSVQ_encode_FIX(_p(idx), _p(q), C.byref(cb), _p(np.ascontiguousarray(np.asarray(prev, np.int32))),
                                      _p(np.ascontiguousarray(np.asarray(w, np.int32))), C.c_int(mu), C.c_int(fluc), C.c_int(16),
                                      C.c_int(10), C.c_int(deact))
    return list(idx), list(q)


@pytest.mark.gpu
def test_pitch_analysis_core_in_the_block_layout(ops, ref):
    cases = pitch_cases()
    n = len(cases)
    hdr = np.array([(prev, THRES1_Q16, thr, corr) for _, prev, thr, corr in cases], np.int32)
    sig = np.ascontiguousarray(np.stack([x for x, _, _, _ in cases]).astype(np.int16))
    out = np.zeros((n, 8), np.int32)
    _ok(ops.sb_ops_pitch(_p(hdr), _p(sig), n, _p(out)))
    for i, (x, prev, thr, corr) in enumerate(cases):
        want = ref_pitch(ref, x, prev, thr, corr)
        assert list(out[i]) == want, ("pitch: lags[4], lagIndex, contourIndex, LTPCorr, sigtype", i, prev, thr, corr)


@pytest.mark.gpu
def test_nlsf_msvq_encode_in_the_block_layout(ops, ref):
    cases = msvq_table(ref)
    n = len(cases)
    hdr = np.array([(mu, fluc, deact, sigtype) for sigtype, _, _, _, mu, fluc, deact in cases], np.int32)
    nl = np.ascontiguousarray(np.stack([c[1] for c in cases]).astype(np.int32))
    prev = np.ascontiguousarray(np.stack([c[2] for c in cases]).astype(np.int32))
    w = np.ascontiguousarray(np.stack([c[3] for c in cases]).astype(np.int32))
    idx, q = np.zeros((n, 6), np.int32), np.zeros((n, 10), np.int32)
    _ok(ops.sb_ops_msvq(_p(hdr), _p(nl), _p(prev), _p(w), n, _p(idx), _p(q)))
    for i, c in enumerate(cases):
        ri, rq = ref_msvq(ref, *c)
        assert (list(idx[i]), list(q[i])) == (ri, rq), ("MSVQ: indices, quantised NLSF", i, c[0], c[4], c[5], c[6])


# ---------------------------------------------------------------------------------------------------------------------
# the tables reach their branches (reference only, no GPU)
# ---------------------------------------------------------------------------------------------------------------------
def test_case_tables_reach_every_listed_branch():
    ref = ref_lib()
    for D in (10, 8):
        regimes = {"le_m2_nonzero": 0, "eq_m2": 0, "eq_m3": 0, "min_clamp": 0, "max_e_ge_2_31": 0, "positive": 0,
                   "early_stop": 0}
        for nb0, nb1, L, wnf, x0, x1 in burg_cases(D):
            for x, nb in ((x0, nb0), (x1, nb1)):
                _, rq, A = ref_burg(ref, x, nb, L, wnf, D)
                rs = -rq
                e = int(np.sum(x[:nb * L].astype(np.int64) ** 2))
                regimes["le_m2_nonzero"] += rs <= -2 and e > 0
                regimes["eq_m2"] += rs == -2
                regimes["eq_m3"] += rs == -3
                regimes["min_clamp"] += rs == -16 and e > 0
                regimes["max_e_ge_2_31"] += rs == 7 and e >= 1 << 31
                regimes["positive"] += 0 < rs < 7
                # |num| >= nrg at step n ends the recursion with A[n:] = 0 (full-scale DC / Nyquist: at n = 0); a run of at
                # least two trailing zeros is not a rounding accident of the last coefficient
                regimes["early_stop"] += e > 0 and not A[D - 2:].any()
        assert all(v >= 3 for v in regimes.values()), ("burg", D, regimes)

        cases = a2nlsf_cases(D)
        white = widened = plain = 0
        for a in cases:
            nl, a_out = ref_a2nlsf(ref, a, D)
            w = list(a_out) != list(a)
            white += list(nl) == list(white_nlsf(D)) and w
            widened += w and list(nl) != list(white_nlsf(D))
            plain += not w
        assert white >= 5 and widened >= 5 and plain >= 20, ("A2NLSF", D, white, widened, plain)
        same = big = 0
        for a in cases:
            nl, a_out = ref_a2nlsf(ref, a, D)
            wn, wa, s_, b_ = a2nlsf_walk(ref, a, D)
            assert (list(nl), list(a_out)) == (wn, wa), ("the walk is the reference's A2NLSF", D, list(a))
            same += s_ > 0
            big += b_ > 0
        assert same >= 3 and big >= 3, ("A2NLSF: roots in the same interval, |ylo| >= 65536 interpolations", D, same, big)

    for order in (10, 16):
        cs = schur_cases(order)
        assert all(schur_py(c, order)[2] for c in cs)
        clipped = sum(schur_py(c, order)[3] for c in cs)
        assert clipped >= 20 and len(cs) - clipped >= 20, ("schur", order, clipped, len(cs))
        # the big-integer statement used to keep the rows inside the contract is the reference's recursion
        for c in cs[:40]:
            rrc = np.zeros(16, np.int16)
            rn = ref.SKP_Silk_schur(_p(rrc), _p(np.array(c + [0] * (17 - len(c)), np.int32)), C.c_int32(order))
            rc, e, _, _ = schur_py(c, order)
            assert (list(rrc[:order]), rn) == (rc, e)

    scales = set()
    for w, warp in warped_cases():
        for j in range(4):
            rc, rs = np.zeros(17, np.int32), C.c_int(0)
            ref.SKP_Silk_warped_autocorrelation_FIX(_p(rc), C.byref(rs), _p(np.ascontiguousarray(w[j])), C.c_int16(warp),
                                                    C.c_int(SHAPE_WIN), C.c_int(SHAPE_ORDER))
            scales.add(rs.value)
    # -(QC + lsh) with lsh clamped to 30 - QC (few-LSB windows) and lsh < 0 (full scale)
    assert -30 in scales and max(scales) > -10, sorted(scales)

    pers = set()
    for B, W, mu in ltp_cases():
        rB, rc, rp = B.copy(), np.zeros(4, np.int32), C.c_int(0)
        ref.SKP_Silk_quant_LTP_gains_FIX(_p(rB), _p(rc), C.byref(rp), _p(np.ascontiguousarray(W)), C.c_int(mu), C.c_int(0))
        pers.add(rp.value)
    assert pers == {0, 1, 2}, pers

    voiced_min = voiced_max = silent_unvoiced = biased = unvoiced = 0
    for x, prev, thr, corr in pitch_cases():
        r = ref_pitch(ref, x, prev, thr, corr)
        voiced = r[7] == 0
        voiced_min += voiced and r[4] == 0              # lag 16
        voiced_max += voiced and r[4] == 144 - 16       # lag 144
        silent_unvoiced += not x.any() and not voiced
        biased += voiced and prev > 0 and corr > 0
        unvoiced += not voiced
    assert voiced_min >= 2 and voiced_max >= 2 and silent_unvoiced >= 1 and biased >= 5 and unvoiced >= 4, \
        ("pitch", voiced_min, voiced_max, silent_unvoiced, biased, unvoiced)

    books = {s: ref_codebook(ref, s)[1] for s in (0, 1)}
    boundary_ties = long_ties = untied = 0
    for sigtype, nl, prev, w, mu, fluc, deact in msvq_table(ref):
        log, path = msvq_search(books[sigtype], nl, w, mu)
        if deact:       # without fluctuation reduction the first survivor is the result: the statement is the reference's
            assert path == ref_msvq(ref, sigtype, nl, prev, w, mu, fluc, deact)[0], (sigtype, list(nl), list(w), mu)
        tie = any(surv < len(v) and v[surv - 1] == v[surv] for v, surv in log)
        boundary_ties += tie
        untied += not tie
        # more than 64 pairs at or below the 16th value: the kernel's compacted short list overflows
        long_ties += any(len(v) > 16 and sum(1 for u in v if u <= v[15]) > 64 for v, _ in log)
    assert boundary_ties >= 20 and long_ties >= 5 and untied >= 20, ("MSVQ", boundary_ties, long_ties, untied)
