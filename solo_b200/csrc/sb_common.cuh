// solo_b200 -- level-0 integer arithmetic kit shared by every per-stream codec routine.
//
// Every routine in solo_b200/csrc/*.cuh is written once as a __host__ __device__ function:
//   * nvcc compiles it into the sm_90a kernels of libsolo_b200.so (the product path);
//   * tests/hostsim compiles the same source with g++ so that the kernel logic can be checked
//     against the compiled reference (oracle/_ref) in a container without a GPU.
// The host build is test infrastructure only; libsolo_b200.so never executes codec maths on the CPU.
//
// Semantics reproduced here (bit-exactly) are those of the reference's fixed-point macro layer:
//   JC1_SDK_SRC_ARM/src/libSATECodec/SKP_Silk_macros.h:34-123       (SMULWB .. CLZ32)
//   JC1_SDK_SRC_ARM/src/libSATECodec/SKP_Silk_SigProc_FIX.h:505-650 (shifts, saturation, RAND)
//   JC1_SDK_SRC_ARM/src/libSATECodec/SKP_Silk_Inlines.h:43-278      (CLZ_FRAC, SQRT_APPROX, DIV32_varQ, ...)
// The reference relies on two's-complement wrap-around in many places (SURVEY.md App. A, Q17); all
// additions / multiplications / left shifts below are therefore done on uint32_t and cast back.
#pragma once
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define SB_HD __host__ __device__ __forceinline__
#define SB_FN __host__ __device__ inline
// Large routines with several call sites: one out-of-line copy instead of one per site.  The thread-per-stream kernels are
// 0.6 - 1.2 MB of SASS when everything is inlined, far beyond the instruction caches of an SM.
#ifdef SB_OUTLINE_BIG
#define SB_FN_BIG __host__ __device__ __noinline__ inline
#else
#define SB_FN_BIG __host__ __device__ inline
#endif
#else
#define SB_HD inline
#define SB_FN inline
#define SB_FN_BIG inline
#endif
// the two approximate-division helpers (~40 instructions, > 100 call sites in the analysis kernel): one out-of-line copy where
// code size matters more than the call (the warp-per-stream kernels execute most instructions once per packet)
#if defined(__CUDACC__) && defined(SB_DIV_OUTLINE)
#define SB_HD_DIV __host__ __device__ __noinline__ inline
#else
#define SB_HD_DIV SB_HD
#endif

namespace sb {

typedef int8_t i8;
typedef int16_t i16;
typedef int32_t i32;
typedef int64_t i64;
typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

#define SB_I32_MAX 0x7FFFFFFF
#define SB_I32_MIN ((int32_t)0x80000000)

// ---- compile-time float -> fixed conversion (SKP_FIX_CONST, SigProc_FIX.h:602) --------------------
// The reference multiplies a *float* literal by a power of two (exact) and adds 0.5 in double.
// Call with the literal carrying the same suffix as in the reference's tuning tables.
constexpr i32 fixc_(double c, int q) { return (i32)(c * (double)((i64)1 << q) + 0.5); }
template <i32 V> struct cx_ { static constexpr i32 v = V; };
#define SB_FIXC(C, Q) (::sb::cx_< ::sb::fixc_((C), (Q)) >::v)

// ---- wrap-around primitives ---------------------------------------------------------------------
SB_HD i32 addw(i32 a, i32 b) { return (i32)((u32)a + (u32)b); }
SB_HD i32 subw(i32 a, i32 b) { return (i32)((u32)a - (u32)b); }
SB_HD i32 mulw(i32 a, i32 b) { return (i32)((u32)a * (u32)b); }
SB_HD i32 negw(i32 a) { return (i32)(0u - (u32)a); }
SB_HD i32 shl(i32 a, int s) { return (i32)((u32)a << s); }
SB_HD i64 shl64(i64 a, int s) { return (i64)((u64)a << s); }
SB_HD i32 mlaw(i32 a, i32 b, i32 c) { return addw(a, mulw(b, c)); }

SB_HD i32 imin(i32 a, i32 b) { return a < b ? a : b; }
SB_HD i32 imax(i32 a, i32 b) { return a > b ? a : b; }
SB_HD i32 iabs(i32 a) { return a > 0 ? a : negw(a); }  // SKP_abs (INT_MIN stays INT_MIN)
SB_HD i32 sat16(i32 a) { return a > 32767 ? 32767 : (a < -32768 ? -32768 : a); }
// SKP_LIMIT: order of the two limits is arbitrary in the reference
SB_HD i32 limit(i32 a, i32 l1, i32 l2) {
    return l1 > l2 ? (a > l1 ? l1 : (a < l2 ? l2 : a)) : (a > l2 ? l2 : (a < l1 ? l1 : a));
}

// ---- 16x16 / 32x16 / 32x32 products ----------------------------------------------------------------
SB_HD i32 smulbb(i32 a, i32 b) { return (i32)(i16)a * (i32)(i16)b; }
SB_HD i32 smlabb(i32 a, i32 b, i32 c) { return addw(a, smulbb(b, c)); }
SB_HD i32 smulbt(i32 a, i32 b) { return (i32)(i16)a * (b >> 16); }
SB_HD i32 smlabt(i32 a, i32 b, i32 c) { return addw(a, smulbt(b, c)); }
SB_HD i32 smultt(i32 a, i32 b) { return (a >> 16) * (b >> 16); }
// (a * (int16)b) >> 16, exact (macros.h:34)
// Device form: (a * b16) >> 16 == high word of a * (b16 << 16); one IMAD.HI instead of a 64-bit product.
SB_HD i32 smulwb(i32 a, i32 b) {
#ifdef __CUDA_ARCH__
    return __mulhi(a, (i32)((u32)b << 16));
#else
    return (i32)(((i64)a * (i64)(i16)b) >> 16);
#endif
}
SB_HD i32 smlawb(i32 a, i32 b, i32 c) { return addw(a, smulwb(b, c)); }
SB_HD i32 smulwt(i32 a, i32 b) {
#ifdef __CUDA_ARCH__
    return __mulhi(a, (i32)((u32)b & 0xFFFF0000u));
#else
    return (i32)(((i64)a * (i64)(b >> 16)) >> 16);
#endif
}
SB_HD i32 smlawt(i32 a, i32 b, i32 c) { return addw(a, smulwt(b, c)); }
SB_HD i32 rshift_round(i32 a, int s) { return s == 1 ? (a >> 1) + (a & 1) : ((a >> (s - 1)) + 1) >> 1; }
SB_HD i64 rshift_round64(i64 a, int s) { return s == 1 ? (a >> 1) + (a & 1) : ((a >> (s - 1)) + 1) >> 1; }
// SMULWW = SMULWB(a,b) + a * RSHIFT_ROUND(b,16)  (macros.h:61) == low 32 bits of (a*b)>>16
SB_HD i32 smulww(i32 a, i32 b) { return (i32)(u32)(u64)(((i64)a * (i64)b) >> 16); }
SB_HD i32 smlaww(i32 a, i32 b, i32 c) { return addw(a, smulww(b, c)); }
SB_HD i32 smmul(i32 a, i32 b) {
#ifdef __CUDA_ARCH__
    return __mulhi(a, b);
#else
    return (i32)(((i64)a * (i64)b) >> 32);
#endif
}
SB_HD i64 smull(i32 a, i32 b) { return (i64)a * (i64)b; }

// ---- saturating arithmetic (macros.h:69-75, SigProc_FIX.h:560-580) -----------------------------------
SB_HD i32 add_sat32(i32 a, i32 b) {
#ifdef __CUDA_ARCH__
    i32 r;
    asm("add.sat.s32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
#else
    i64 s = (i64)a + (i64)b;
    return s > SB_I32_MAX ? SB_I32_MAX : (s < (i64)SB_I32_MIN ? SB_I32_MIN : (i32)s);
#endif
}
SB_HD i32 sub_sat32(i32 a, i32 b) {
#ifdef __CUDA_ARCH__
    i32 r;
    asm("sub.sat.s32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
#else
    i64 s = (i64)a - (i64)b;
    return s > SB_I32_MAX ? SB_I32_MAX : (s < (i64)SB_I32_MIN ? SB_I32_MIN : (i32)s);
#endif
}
SB_HD i32 add_pos_sat32(i32 a, i32 b) { i32 s = addw(a, b); return (s & 0x80000000) ? SB_I32_MAX : s; }
SB_HD i32 lshift_sat32(i32 a, int s) {
    return shl(limit(a, SB_I32_MIN >> s, SB_I32_MAX >> s), s);
}
SB_HD i32 add_sat16(i32 a, i32 b) { return sat16(addw((i32)(i16)a, b)); }

// ---- bit utilities ------------------------------------------------------------------------------
SB_HD int clz32(i32 x) {
#ifdef __CUDA_ARCH__
    return __clz(x);
#else
    return x == 0 ? 32 : __builtin_clz((u32)x);
#endif
}
SB_HD int clz64(i64 x) {
    i32 up = (i32)(x >> 32);
    return up == 0 ? 32 + clz32((i32)x) : clz32(up);
}
SB_HD i32 ror32(i32 a, int rot) {  // SigProc_FIX.h:475-484 (generic form)
    u32 x = (u32)a;
    if (rot == 0) return a;
    if (rot < 0) { u32 m = (u32)(-rot); return (i32)((x << m) | (x >> (32 - m))); }
    return (i32)((x << (32 - rot)) | (x >> rot));
}
SB_HD void clz_frac(i32 in, i32* lz, i32* frac_q7) {
    i32 l = clz32(in);
    *lz = l;
    *frac_q7 = ror32(in, 24 - l) & 0x7f;
}
// Inlines.h:71-96
SB_HD i32 sqrt_approx(i32 x) {
    if (x <= 0) return 0;
    i32 lz, frac;
    clz_frac(x, &lz, &frac);
    i32 y = (lz & 1) ? 32768 : 46214;
    y >>= (lz >> 1);
    return smlawb(y, y, smulbb(213, frac));
}
SB_HD i32 norm16(i16 a) {
    i32 a32 = a;
    if (a32 == 0) return 0;
    a32 ^= (a32 >> 31);
    return clz32(a32) - 17;
}
SB_HD i32 norm32(i32 a) {
    if (shl(a, 1) == 0) return 0;
    a ^= (a >> 31);
    return clz32(a) - 1;
}
// lin2log.c:41-48 ; log2lin.c:40-60
SB_HD i32 lin2log(i32 x) {
    i32 lz, frac;
    clz_frac(x, &lz, &frac);
    return shl(31 - lz, 7) + smlawb(frac, mulw(frac, 128 - frac), 179);
}
SB_HD i32 log2lin(i32 in_q7) {
    if (in_q7 < 0) return 0;
    if (in_q7 >= (31 << 7)) return SB_I32_MAX;
    i32 out = shl(1, in_q7 >> 7);
    i32 frac = in_q7 & 0x7F;
    i32 t = smlawb(frac, mulw(frac, 128 - frac), -174);
    if (in_q7 < 2048) out = addw(out, mulw(out, t) >> 7);
    else out = mlaw(out, out >> 7, t);
    return out;
}
// sigm_Q15.c:54-79
SB_HD i32 sigm_q15(i32 in_q5) {
    const i32 slope[6] = {237, 153, 73, 30, 12, 7};
    const i32 pos[6] = {16384, 23955, 28861, 31213, 32178, 32548};
    const i32 neg[6] = {16384, 8812, 3906, 1554, 589, 219};
    if (in_q5 < 0) {
        in_q5 = -in_q5;
        if (in_q5 >= 6 * 32) return 0;
        i32 ind = in_q5 >> 5;
        return neg[ind] - smulbb(slope[ind], in_q5 & 0x1F);
    }
    if (in_q5 >= 6 * 32) return 32767;
    i32 ind = in_q5 >> 5;
    return pos[ind] + smulbb(slope[ind], in_q5 & 0x1F);
}

// (SKP_int32_MAX >> 2) / d as the reference's C division computes it, for the divisors its normalisation produces
// (16384 <= |d| <= 32768): float reciprocal + one exact correction step instead of a generic 32-bit integer division
// (exhaustively checked against the integer division for every such d: tests/test_hostsim_parity.py).
SB_HD i32 div_q29(i32 d) {
    const i32 N = SB_I32_MAX >> 2;
    if ((u32)(iabs(d) - 16384) > 16384u) return d == 0 ? 0 : N / d;   // not reachable from normalised inputs
#ifdef __CUDA_ARCH__
    i32 q = __float2int_rz((float)N * __frcp_rn((float)d));
#else
    i32 q = (i32)((float)N * (1.0f / (float)d));
#endif
    const i32 rem = N - q * d;
    if (d > 0) { if (rem < 0) q--; else if (rem >= d) q++; }
    else { if (rem < 0) q++; else if (rem >= -d) q--; }
    return q;
}

// ---- approximate division (Inlines.h:124-217); reproduced step by step, never an exact divide --------
SB_HD_DIV i32 div32_varq(i32 a32, i32 b32, int qres) {
    int a_headrm = clz32(iabs(a32)) - 1;
    i32 a_nrm = shl(a32, a_headrm);
    int b_headrm = clz32(iabs(b32)) - 1;
    i32 b_nrm = shl(b32, b_headrm);
    i32 b_inv = div_q29(b_nrm >> 16);
    i32 result = smulwb(a_nrm, b_inv);
    a_nrm = subw(a_nrm, shl(smmul(b_nrm, result), 3));
    result = smlawb(result, a_nrm, b_inv);
    int lshift = 29 + a_headrm - b_headrm - qres;
    if (lshift <= 0) return lshift_sat32(result, -lshift);
    if (lshift < 32) return result >> lshift;
    return 0;
}
SB_HD_DIV i32 inverse32_varq(i32 b32, int qres) {
    int b_headrm = clz32(iabs(b32)) - 1;
    i32 b_nrm = shl(b32, b_headrm);
    i32 b_inv = div_q29(b_nrm >> 16);
    i32 result = shl(b_inv, 16);
    i32 err_q32 = shl(negw(smulwb(b_nrm, b_inv)), 3);
    result = smlaww(result, err_q32, b_inv);
    int lshift = 61 - b_headrm - qres;
    if (lshift <= 0) return lshift_sat32(result, -lshift);
    if (lshift < 32) return result >> lshift;
    return 0;
}

// Inlines.h:219-275 (sine approximation, input 65536 == 2*pi)
SB_HD i32 sin_approx_q24(i32 x) {
    i32 y_q30;
    x &= 65535;
    if (x <= 32768) {
        if (x < 16384) x = 16384 - x; else x -= 16384;
        if (x < 1100) return smlawb(1 << 24, mulw(x, x), -5053);
        x = smulwb(shl(x, 8), x);
        y_q30 = smlawb(1059577, x, -5013);
        y_q30 = smlaww(-82778932, x, y_q30);
        y_q30 = smlaww(1073735400 + 66, x, y_q30);
    } else {
        if (x < 49152) x = 49152 - x; else x -= 49152;
        if (x < 1100) return smlawb(-(1 << 24), mulw(x, x), 5053);
        x = smulwb(shl(x, 8), x);
        y_q30 = smlawb(-1059577, x, 5013);
        y_q30 = smlaww(82778932, x, y_q30);
        y_q30 = smlaww(-1073735400, x, y_q30);
    }
    return rshift_round(y_q30, 6);
}
SB_HD i32 cos_approx_q24(i32 x) { return sin_approx_q24(x + 16384); }

// dither / PLC / CNG generator (SigProc_FIX.h:650)
SB_HD i32 lcg_rand(i32 seed) { return mlaw(907633515, seed, 196314165); }

// round-half-away float->int (SigProc_FIX.h:629-632)
// float / double -> int32 by truncation, with the out-of-range behaviour of the reference's build target made explicit:
// x86 cvttss2si / cvttsd2si return INT_MIN ("integer indefinite") for NaN and for values outside int32, where CUDA's cvt
// would saturate and ISO C leaves it undefined.  Only reachable with corrupted payloads (a blown-up synthesis filter).
SB_HD i32 trunc_i32(double x) { return (x > -2147483649.0 && x < 2147483648.0) ? (i32)x : SB_I32_MIN; }
SB_HD i32 float2int(double x) { return trunc_i32((x > 0) ? x + 0.5 : x - 0.5); }

}  // namespace sb
