// solo_b200 -- signal-processing primitives of the SILK core (level 0), one stream per caller.
// Every routine cites the reference routine whose integer behaviour it reproduces; paths are
// relative to /root/reference/JC1_SDK_SRC_ARM/src/libSATECodec/.
#pragma once
#include "sb_par.cuh"
#include "sb_tables.cuh"

namespace sb {

// ---- inner products (SKP_Silk_inner_prod_aligned.c:44-75) -----------------------------------------
SB_HD i32 inner_prod16(const i16* a, const i16* b, int len) {
    i32 s = 0;
    for (int i = 0; i < len; i++) s = addw(s, (i32)a[i] * (i32)b[i]);
    return s;
}
SB_HD i64 inner_prod16_64(const i16* a, const i16* b, int len) {
    i64 s = 0;
    for (int i = 0; i < len; i++) s += (i64)((i32)a[i] * (i32)b[i]);
    return s;
}

// ---- SKP_Silk_sum_sqr_shift.c:40-98 -------------------------------------------------------------
// The reference takes a different accumulation path when the input pointer is only 2-byte aligned
// (SURVEY.md App. A Q21).  All its buffers are 4-byte aligned arrays, so the path is decided by the
// parity of the element offset, which every call site passes as `odd_start`.
SB_FN void sum_sqr_shift(i32* energy, i32* shift, const i16* x, int len, int odd_start) {
    i32 nrg; int i, shft = 0;
    if (odd_start) { nrg = (i32)x[0] * (i32)x[0]; i = 1; } else { nrg = 0; i = 0; }
    len--;
    while (i < len) {
        nrg = addw(nrg, (i32)x[i] * (i32)x[i]);
        nrg = addw(nrg, (i32)x[i + 1] * (i32)x[i + 1]);
        i += 2;
        if (nrg < 0) { nrg = (i32)((u32)nrg >> 2); shft = 2; break; }
    }
    for (; i < len; i += 2) {
        i32 t = (i32)x[i] * (i32)x[i];
        t = addw(t, (i32)x[i + 1] * (i32)x[i + 1]);
        nrg = (i32)((u32)nrg + ((u32)t >> shft));
        if (nrg < 0) { nrg = (i32)((u32)nrg >> 2); shft += 2; }
    }
    if (i == len) {
        i32 t = (i32)x[i] * (i32)x[i];
        nrg = addw(nrg, t >> shft);
    }
    if (nrg & 0xC0000000) { nrg = (i32)((u32)nrg >> 2); shft += 2; }
    *shift = shft;
    *energy = nrg;
}

// ---- SKP_Silk_autocorr.c:40-77 --------------------------------------------------------------------
SB_FN void autocorr(i32* results, i32* scale, const i16* x, int n, int count) {
    int cc = imin(n, count);
    i64 corr64 = inner_prod16_64(x, x, n) + 1;
    int lz = clz64(corr64);
    int nrs = 35 - lz;
    *scale = nrs;
    if (nrs <= 0) {
        results[0] = shl((i32)corr64, -nrs);
        for (int i = 1; i < cc; i++) results[i] = shl(inner_prod16(x, x + i, n - i), -nrs);
    } else {
        results[0] = (i32)(corr64 >> nrs);
        for (int i = 1; i < cc; i++) results[i] = (i32)(inner_prod16_64(x, x + i, n - i) >> nrs);
    }
}

// ---- SKP_Silk_schur.c:40-93 (order <= 16) ---------------------------------------------------------
SB_FN i32 schur(i16* rc_Q15, const i32* c, int order) {
    i32 C[17][2];
    int lz = clz32(c[0]);
    for (int k = 0; k < order + 1; k++) {
        i32 v = lz < 2 ? (c[k] >> 1) : (lz > 2 ? shl(c[k], lz - 2) : c[k]);
        C[k][0] = C[k][1] = v;
    }
    for (int k = 0; k < order; k++) {
        i32 rc = negw(C[k + 1][0] / imax(C[0][1] >> 15, 1));
        rc = sat16(rc);
        rc_Q15[k] = (i16)rc;
        for (int n = 0; n < order - k; n++) {
            i32 t1 = C[n + k + 1][0], t2 = C[n][1];
            C[n + k + 1][0] = smlawb(t1, shl(t2, 1), rc);
            C[n][1] = smlawb(t2, shl(t1, 1), rc);
        }
    }
    return C[0][1];
}

// ---- SKP_Silk_k2a.c:40-60 -------------------------------------------------------------------------
SB_FN void k2a(i32* A_Q24, const i16* rc_Q15, int order) {
    i32 Atmp[16];
    for (int k = 0; k < order; k++) {
        for (int n = 0; n < k; n++) Atmp[n] = A_Q24[n];
        for (int n = 0; n < k; n++) A_Q24[n] = smlawb(A_Q24[n], shl(Atmp[k - n - 1], 1), rc_Q15[k]);
        A_Q24[k] = negw(shl((i32)rc_Q15[k], 9));
    }
}

// ---- SKP_Silk_schur64.c:42-91, SKP_Silk_k2a_Q16.c:40-60, SKP_Silk_bwexpander_32.c:31-47 at a fixed order -------------
// Every array in registers (fully unrolled): in the analysis kernel these run as one scalar instance per shaping window,
// where a local-memory array would put a ~30-cycle load into every step of a long dependent chain.
template <int ORD> SB_HD i32 schur64_r(i32 (&rc_Q16)[ORD], const i32 (&c)[ORD + 1]) {
    i32 C0[ORD + 1], C1[ORD + 1];
    if (c[0] <= 0) {
#pragma unroll
        for (int k = 0; k < ORD; k++) rc_Q16[k] = 0;
        return 0;
    }
#pragma unroll
    for (int k = 0; k < ORD + 1; k++) C0[k] = C1[k] = c[k];
#pragma unroll
    for (int k = 0; k < ORD; k++) {
        const i32 rc_Q31 = div32_varq(negw(C0[k + 1]), C1[0], 31);
        rc_Q16[k] = rshift_round(rc_Q31, 15);
#pragma unroll
        for (int n = 0; n < ORD - k; n++) {
            const i32 t1 = C0[n + k + 1], t2 = C1[n];
            C0[n + k + 1] = addw(t1, smmul(shl(t2, 1), rc_Q31));
            C1[n] = addw(t2, smmul(shl(t1, 1), rc_Q31));
        }
    }
    return C1[0];
}
template <int ORD> SB_HD void k2a_q16_r(i32 (&A_Q24)[ORD], const i32 (&rc_Q16)[ORD]) {
#pragma unroll
    for (int k = 0; k < ORD; k++) {
        i32 Atmp[ORD];
#pragma unroll
        for (int n = 0; n < k; n++) Atmp[n] = A_Q24[n];
#pragma unroll
        for (int n = 0; n < k; n++) A_Q24[n] = smlaww(A_Q24[n], Atmp[k - n - 1], rc_Q16[k]);
        A_Q24[k] = negw(shl(rc_Q16[k], 8));
    }
}
template <int ORD> SB_HD void bwexpander_32_r(i32 (&ar)[ORD], i32 chirp_Q16) {
    i32 t = chirp_Q16;
#pragma unroll
    for (int i = 0; i < ORD - 1; i++) { ar[i] = smulww(ar[i], t); t = smulww(chirp_Q16, t); }
    ar[ORD - 1] = smulww(ar[ORD - 1], t);
}

// ---- SKP_Silk_bwexpander.c:31-48 / SKP_Silk_bwexpander_32.c:31-47 -------------------------------------
SB_FN void bwexpander(i16* ar, int d, i32 chirp_Q16) {
    i32 cm1 = chirp_Q16 - 65536;
    for (int i = 0; i < d - 1; i++) {
        ar[i] = (i16)rshift_round(mulw(chirp_Q16, ar[i]), 16);
        chirp_Q16 += rshift_round(mulw(chirp_Q16, cm1), 16);
    }
    ar[d - 1] = (i16)rshift_round(mulw(chirp_Q16, ar[d - 1]), 16);
}
SB_FN void bwexpander_32(i32* ar, int d, i32 chirp_Q16) {
    i32 t = chirp_Q16;
    for (int i = 0; i < d - 1; i++) {
        ar[i] = smulww(ar[i], t);
        t = smulww(chirp_Q16, t);
    }
    ar[d - 1] = smulww(ar[d - 1], t);
}

// ---- SKP_Silk_LPC_inv_pred_gain.c:42-153 --------------------------------------------------------------
SB_FN int lpc_inv_pred_gain_qa(i32* invGain_Q30, i32 A_QA[2][16], int order) {
    const i32 A_LIMIT = SB_FIXC(0.99975, 16);
    i32* Anew = A_QA[order & 1];
    *invGain_Q30 = 1 << 30;
    for (int k = order - 1; k > 0; k--) {
        if (Anew[k] > A_LIMIT || Anew[k] < -A_LIMIT) return 1;
        i32 rc_Q31 = negw(shl(Anew[k], 31 - 16));
        i32 rc_mult1_Q30 = (SB_I32_MAX >> 1) - smmul(rc_Q31, rc_Q31);
        i32 rc_mult2_Q16 = inverse32_varq(rc_mult1_Q30, 46);
        *invGain_Q30 = shl(smmul(*invGain_Q30, rc_mult1_Q30), 2);
        i32* Aold = Anew;
        Anew = A_QA[k & 1];
        int headrm = clz32(rc_mult2_Q16) - 1;
        rc_mult2_Q16 = shl(rc_mult2_Q16, headrm);
        for (int n = 0; n < k; n++) {
            i32 tmp = subw(Aold[n], shl(smmul(Aold[k - n - 1], rc_Q31), 1));
            Anew[n] = shl(smmul(tmp, rc_mult2_Q16), 16 - headrm);
        }
    }
    if (Anew[0] > A_LIMIT || Anew[0] < -A_LIMIT) return 1;
    i32 rc_Q31 = negw(shl(Anew[0], 31 - 16));
    i32 rc_mult1_Q30 = (SB_I32_MAX >> 1) - smmul(rc_Q31, rc_Q31);
    *invGain_Q30 = shl(smmul(*invGain_Q30, rc_mult1_Q30), 2);
    return 0;
}
SB_FN int lpc_inv_pred_gain_q12(i32* invGain_Q30, const i16* A_Q12, int order) {
    i32 A[2][16];
    i32* Anew = A[order & 1];
    for (int k = 0; k < order; k++) Anew[k] = shl((i32)A_Q12[k], 4);
    return lpc_inv_pred_gain_qa(invGain_Q30, A, order);
}
SB_FN int lpc_inv_pred_gain_q24(i32* invGain_Q30, const i32* A_Q24, int order) {
    i32 A[2][16];
    i32* Anew = A[order & 1];
    for (int k = 0; k < order; k++) Anew[k] = rshift_round(A_Q24[k], 8);
    return lpc_inv_pred_gain_qa(invGain_Q30, A, order);
}

// ---- SKP_Silk_MA.c:41-62 (MA_Prediction) and :65-118 (LPC_analysis_filter), both only ever called with a zeroed state
// on this path == direct-form FIR whose taps before in[0] are zero:
//   out[k] = sat16(rshift_round((in[k] << 12) - sum_d B[d] * in[k-1-d], 12))
// MA_Prediction subtracts with wrap-around, LPC_analysis_filter with saturation.  The sum is taken mod 2^32, so missing
// taps may be added as zeros: the last ORD inputs slide through registers and the coefficients are loaded once.
template <int ORD, bool SAT> SB_FN void fir_zero_state(const i16* in, const i16* B_Q12, i16* out, int len) {
    i32 b[ORD], w[ORD];
#pragma unroll
    for (int d = 0; d < ORD; d++) { b[d] = B_Q12[d]; w[d] = 0; }
    for (int k = 0; k < len; k++) {
        i32 acc = 0;
#pragma unroll
        for (int d = 0; d < ORD; d++) acc = addw(acc, w[d] * b[d]);
        const i32 x = in[k];
        const i32 o = SAT ? sub_sat32(shl(x, 12), acc) : subw(shl(x, 12), acc);
        out[k] = (i16)sat16(rshift_round(o, 12));
#pragma unroll
        for (int d = ORD - 1; d > 0; d--) w[d] = w[d - 1];
        w[0] = x;
    }
}
template <bool SAT> SB_FN void fir_zero_state_any(const i16* in, const i16* B_Q12, i16* out, int len, int order) {
    if (order == 10) { fir_zero_state<10, SAT>(in, B_Q12, out, len); return; }
    if (order == 8) { fir_zero_state<8, SAT>(in, B_Q12, out, len); return; }
    for (int k = 0; k < len; k++) {
        i32 acc = 0;
        int dmax = imin(order, k);
        for (int d = 0; d < dmax; d++) acc = addw(acc, (i32)in[k - 1 - d] * (i32)B_Q12[d]);
        i32 o = SAT ? sub_sat32(shl((i32)in[k], 12), acc) : subw(shl((i32)in[k], 12), acc);
        out[k] = (i16)sat16(rshift_round(o, 12));
    }
}
SB_FN void ma_prediction_zero_state(const i16* in, const i16* B_Q12, i16* out, int len, int order) {
    fir_zero_state_any<false>(in, B_Q12, out, len, order);
}
SB_FN void lpc_analysis_filter_zero_state(const i16* in, const i16* B_Q12, i16* out, int len, int order) {
    fir_zero_state_any<true>(in, B_Q12, out, len, order);
}

// ---- SKP_Silk_apply_sine_window.c:47-118 (scalar form; identical numerics on little-endian, Q24)
SB_FN void apply_sine_window(i16* px_win, const i16* px, int win_type, int length) {
    int k = (length >> 2) - 4;
    i32 f_Q16 = SB_T(sine_freq_table_q16)[k];
    i32 c_Q16 = smulwb(f_Q16, -f_Q16);
    i32 S0, S1;
    if (win_type == 1) { S0 = 0; S1 = f_Q16 + (length >> 3); }
    else { S0 = 1 << 16; S1 = (1 << 16) + (c_Q16 >> 1) + (length >> 4); }
    for (k = 0; k < length; k += 4) {
        px_win[k] = (i16)smulwb((S0 + S1) >> 1, px[k]);
        px_win[k + 1] = (i16)smulwb(S1, px[k + 1]);
        S0 = smulwb(S1, c_Q16) + shl(S1, 1) - S0 + 1;
        S0 = imin(S0, 1 << 16);
        px_win[k + 2] = (i16)smulwb((S0 + S1) >> 1, px[k + 2]);
        px_win[k + 3] = (i16)smulwb(S0, px[k + 3]);
        S1 = smulwb(S0, c_Q16) + shl(S0, 1) - S1;
        S1 = imin(S1, 1 << 16);
    }
}

// ---- SKP_Silk_resampler_down2.c:41-78 --------------------------------------------------------------
SB_FN void resampler_down2(i32* S, i16* __restrict__ out, const i16* __restrict__ in, int inLen) {   // out and in never overlap
    int len2 = inLen >> 1;
    const i32 c0 = SB_T(resampler_down2_0)[0], c1 = SB_T(resampler_down2_1)[0];
    i32 S0 = S[0], S1 = S[1];
    for (int k = 0; k < len2; k++) {
        i32 in32 = shl((i32)in[2 * k], 10);
        i32 Y = subw(in32, S0);
        i32 X = smlawb(Y, Y, c1);
        i32 out32 = addw(S0, X);
        S0 = addw(in32, X);
        in32 = shl((i32)in[2 * k + 1], 10);
        Y = subw(in32, S1);
        X = smulwb(Y, c0);
        out32 = addw(out32, S1);
        out32 = addw(out32, X);
        S1 = addw(in32, X);
        out[k] = (i16)sat16(rshift_round(out32, 11));
    }
    S[0] = S0; S[1] = S1;
}

// ---- SKP_Silk_ana_filt_bank_1.c:45-80 (in-place on outL == in is safe: in[2k], in[2k+1] are read before outL[k] is written)
SB_FN void ana_filt_bank_1(const i16* in, i32* S, i16* outL, i16* outH, int N) {
    const i32 A20 = (i16)(5394 << 1), A21 = (i16)(20623 << 1);
    int N2 = N >> 1;
    i32 S0 = S[0], S1 = S[1];
    i32 x0 = in[0], x1 = in[1];          // the next input pair is fetched before outL[k] is stored (outL may be in: index k < 2k + 2)
    for (int k = 0; k < N2; k++) {
        const i32 a = x0, b = x1;
        if (k + 1 < N2) { x0 = in[2 * k + 2]; x1 = in[2 * k + 3]; }
        i32 in32 = shl(a, 10);
        i32 Y = subw(in32, S0);
        i32 X = smlawb(Y, Y, A21);
        i32 out_1 = addw(S0, X);
        S0 = addw(in32, X);
        in32 = shl(b, 10);
        Y = subw(in32, S1);
        X = smulwb(Y, A20);
        i32 out_2 = addw(S1, X);
        S1 = addw(in32, X);
        outL[k] = (i16)sat16(rshift_round(addw(out_2, out_1), 11));
        outH[k] = (i16)sat16(rshift_round(subw(out_2, out_1), 11));
    }
    S[0] = S0; S[1] = S1;
}

// ---- SKP_Silk_biquad_alt.c:38-72 ------------------------------------------------------------------
SB_FN void biquad_alt(const i16* __restrict__ in, const i32* B_Q28, const i32* A_Q28, i32* S, i16* __restrict__ out, int len) {   // in and out never overlap
    const i32 A0_L = (-A_Q28[0]) & 0x3FFF, A0_U = (-A_Q28[0]) >> 14;
    const i32 A1_L = (-A_Q28[1]) & 0x3FFF, A1_U = (-A_Q28[1]) >> 14;
    const i32 B0 = B_Q28[0], B1 = B_Q28[1], B2 = B_Q28[2];
    i32 S0 = S[0], S1 = S[1];
    for (int k = 0; k < len; k++) {
        const i32 inval = in[k];
        const i32 out32_Q14 = shl(smlawb(S0, B0, inval), 2);
        S0 = addw(S1, rshift_round(smulwb(out32_Q14, A0_L), 14));
        S0 = smlawb(S0, out32_Q14, A0_U);
        S0 = smlawb(S0, B1, inval);
        S1 = rshift_round(smulwb(out32_Q14, A1_L), 14);
        S1 = smlawb(S1, out32_Q14, A1_U);
        S1 = smlawb(S1, B2, inval);
        out[k] = (i16)sat16(addw(out32_Q14, (1 << 14) - 1) >> 14);
    }
    S[0] = S0; S[1] = S1;
}

// ---- SKP_Silk_sort.c:34-124 (partial insertion sorts; tie-breaking is part of the bitstream, Q22)
SB_FN void insertion_sort_decreasing_i16(i16* a, i32* index, int L, int K) {
    for (int i = 0; i < K; i++) index[i] = i;
    for (int i = 1; i < K; i++) {
        i32 value = a[i]; int j;
        for (j = i - 1; j >= 0 && value > a[j]; j--) { a[j + 1] = a[j]; index[j + 1] = index[j]; }
        a[j + 1] = (i16)value; index[j + 1] = i;
    }
    for (int i = K; i < L; i++) {
        i32 value = a[i];
        if (value > a[K - 1]) {
            int j;
            for (j = K - 2; j >= 0 && value > a[j]; j--) { a[j + 1] = a[j]; index[j + 1] = index[j]; }
            a[j + 1] = (i16)value; index[j + 1] = i;
        }
    }
}

// ---- SKP_Silk_burg_modified.c:49-228 (QA = 25) --------------------------------------------------------
SB_FN void burg_modified(i32* res_nrg, i32* res_nrg_Q, i32* A_Q16, const i16* x, int subfr_length, int nb_subfr,
                         i32 WhiteNoiseFrac_Q32, int D) {
    const int QA = 25, MAX_RSHIFTS = 32 - QA, MIN_RSHIFTS = -16, HEAD = 2;
    i32 C0, rshifts;
    i32 C_first_row[16], C_last_row[16], Af_QA[16], CAf[17], CAb[17];
    sum_sqr_shift(&C0, &rshifts, x, nb_subfr * subfr_length, 0);
    if (rshifts > MAX_RSHIFTS) {
        C0 = shl(C0, rshifts - MAX_RSHIFTS);
        rshifts = MAX_RSHIFTS;
    } else {
        int lz = clz32(C0) - 1;
        int extra = HEAD - lz;
        if (extra > 0) { extra = imin(extra, MAX_RSHIFTS - rshifts); C0 = C0 >> extra; }
        else { extra = imax(extra, MIN_RSHIFTS - rshifts); C0 = shl(C0, -extra); }
        rshifts += extra;
    }
    for (int i = 0; i < 16; i++) C_first_row[i] = 0;
    if (rshifts > 0) {
        for (int s = 0; s < nb_subfr; s++) {
            const i16* xp = x + s * subfr_length;
            for (int n = 1; n < D + 1; n++)
                C_first_row[n - 1] = addw(C_first_row[n - 1], (i32)(inner_prod16_64(xp, xp + n, subfr_length - n) >> rshifts));
        }
    } else {
        for (int s = 0; s < nb_subfr; s++) {
            const i16* xp = x + s * subfr_length;
            for (int n = 1; n < D + 1; n++)
                C_first_row[n - 1] = addw(C_first_row[n - 1], shl(inner_prod16(xp, xp + n, subfr_length - n), -rshifts));
        }
    }
    for (int i = 0; i < 16; i++) C_last_row[i] = C_first_row[i];
    CAb[0] = CAf[0] = addw(addw(C0, smmul(WhiteNoiseFrac_Q32, C0)), 1);
    for (int n = 0; n < D; n++) {
        if (rshifts > -2) {
            for (int s = 0; s < nb_subfr; s++) {
                const i16* xp = x + s * subfr_length;
                i32 x1 = negw(shl((i32)xp[n], 16 - rshifts));
                i32 x2 = negw(shl((i32)xp[subfr_length - n - 1], 16 - rshifts));
                i32 tmp1 = shl((i32)xp[n], QA - 16);
                i32 tmp2 = shl((i32)xp[subfr_length - n - 1], QA - 16);
                for (int k = 0; k < n; k++) {
                    C_first_row[k] = smlawb(C_first_row[k], x1, xp[n - k - 1]);
                    C_last_row[k] = smlawb(C_last_row[k], x2, xp[subfr_length - n + k]);
                    i32 At = Af_QA[k];
                    tmp1 = smlawb(tmp1, At, xp[n - k - 1]);
                    tmp2 = smlawb(tmp2, At, xp[subfr_length - n + k]);
                }
                tmp1 = shl(negw(tmp1), 32 - QA - rshifts);
                tmp2 = shl(negw(tmp2), 32 - QA - rshifts);
                for (int k = 0; k <= n; k++) {
                    CAf[k] = smlawb(CAf[k], tmp1, xp[n - k]);
                    CAb[k] = smlawb(CAb[k], tmp2, xp[subfr_length - n + k - 1]);
                }
            }
        } else {
            for (int s = 0; s < nb_subfr; s++) {
                const i16* xp = x + s * subfr_length;
                i32 x1 = negw(shl((i32)xp[n], -rshifts));
                i32 x2 = negw(shl((i32)xp[subfr_length - n - 1], -rshifts));
                i32 tmp1 = shl((i32)xp[n], 17);
                i32 tmp2 = shl((i32)xp[subfr_length - n - 1], 17);
                for (int k = 0; k < n; k++) {
                    C_first_row[k] = mlaw(C_first_row[k], x1, xp[n - k - 1]);
                    C_last_row[k] = mlaw(C_last_row[k], x2, xp[subfr_length - n + k]);
                    i32 At1 = rshift_round(Af_QA[k], QA - 17);
                    tmp1 = mlaw(tmp1, xp[n - k - 1], At1);
                    tmp2 = mlaw(tmp2, xp[subfr_length - n + k], At1);
                }
                tmp1 = negw(tmp1);
                tmp2 = negw(tmp2);
                for (int k = 0; k <= n; k++) {
                    CAf[k] = smlaww(CAf[k], tmp1, shl((i32)xp[n - k], -rshifts - 1));
                    CAb[k] = smlaww(CAb[k], tmp2, shl((i32)xp[subfr_length - n + k - 1], -rshifts - 1));
                }
            }
        }
        i32 tmp1 = C_first_row[n], tmp2 = C_last_row[n];
        i32 num = 0;
        i32 nrg = addw(CAb[0], CAf[0]);
        for (int k = 0; k < n; k++) {
            i32 At = Af_QA[k];
            int lz = clz32(iabs(At)) - 1;
            lz = imin(32 - QA, lz);
            i32 At1 = shl(At, lz);
            int sh = 32 - QA - lz;
            tmp1 = addw(tmp1, shl(smmul(C_last_row[n - k - 1], At1), sh));
            tmp2 = addw(tmp2, shl(smmul(C_first_row[n - k - 1], At1), sh));
            num = addw(num, shl(smmul(CAb[n - k], At1), sh));
            nrg = addw(nrg, shl(smmul(addw(CAb[k + 1], CAf[k + 1]), At1), sh));
        }
        CAf[n + 1] = tmp1;
        CAb[n + 1] = tmp2;
        num = addw(num, tmp2);
        num = shl(negw(num), 1);
        i32 rc_Q31;
        if (iabs(num) < nrg) {
            rc_Q31 = div32_varq(num, nrg, 31);
        } else {
            for (int k = n; k < D; k++) Af_QA[k] = 0;
            break;
        }
        for (int k = 0; k < (n + 1) >> 1; k++) {
            i32 t1 = Af_QA[k], t2 = Af_QA[n - k - 1];
            Af_QA[k] = addw(t1, shl(smmul(t2, rc_Q31), 1));
            Af_QA[n - k - 1] = addw(t2, shl(smmul(t1, rc_Q31), 1));
        }
        Af_QA[n] = rc_Q31 >> (31 - QA);
        for (int k = 0; k <= n + 1; k++) {
            i32 t1 = CAf[k], t2 = CAb[n - k + 1];
            CAf[k] = addw(t1, shl(smmul(t2, rc_Q31), 1));
            CAb[n - k + 1] = addw(t2, shl(smmul(t1, rc_Q31), 1));
        }
    }
    i32 nrg = CAf[0];
    i32 tmp1 = 1 << 16;
    for (int k = 0; k < D; k++) {
        i32 At1 = rshift_round(Af_QA[k], QA - 16);
        nrg = smlaww(nrg, CAf[k + 1], At1);
        tmp1 = smlaww(tmp1, At1, At1);
        A_Q16[k] = negw(At1);
    }
    *res_nrg = smlaww(nrg, smmul(WhiteNoiseFrac_Q32, C0), negw(tmp1));
    *res_nrg_Q = -rshifts;
}

// ---- SKP_Silk_A2NLSF.c:46-287 ---------------------------------------------------------------------
SB_HD void a2nlsf_trans_poly(i32* p, int dd) {
    for (int k = 2; k <= dd; k++) {
        for (int n = dd; n > k; n--) p[n - 2] = subw(p[n - 2], p[n]);
        p[k - 2] = subw(p[k - 2], shl(p[k], 1));
    }
}
SB_HD i32 a2nlsf_eval_poly(const i32* p, i32 x, int dd) {
    i32 y32 = p[dd];
    i32 x_Q16 = shl(x, 4);
    for (int n = dd - 1; n >= 0; n--) y32 = smlaww(p[n], y32, x_Q16);
    return y32;
}
SB_FN void a2nlsf_init(const i32* a_Q16, i32* P, i32* Q, int dd) {
    P[dd] = 1 << 16;
    Q[dd] = 1 << 16;
    for (int k = 0; k < dd; k++) {
        P[k] = subw(negw(a_Q16[dd - k - 1]), a_Q16[dd + k]);
        Q[k] = addw(negw(a_Q16[dd - k - 1]), a_Q16[dd + k]);
    }
    for (int k = dd; k > 0; k--) {
        P[k - 1] = subw(P[k - 1], P[k]);
        Q[k - 1] = addw(Q[k - 1], Q[k]);
    }
    a2nlsf_trans_poly(P, dd);
    a2nlsf_trans_poly(Q, dd);
}
SB_FN void a2nlsf(i32* NLSF, i32* a_Q16, int d) {
    const int BIN = 3, TABSZ = 128, MAX_ITER = 30;
    i32 P[9], Q[9];
    int dd = d >> 1;
    a2nlsf_init(a_Q16, P, Q, dd);
    const i32* p = P;
    i32 xlo = SB_T(lsf_cos_q12)[0];
    i32 ylo = a2nlsf_eval_poly(p, xlo, dd);
    int root_ix;
    if (ylo < 0) { NLSF[0] = 0; p = Q; ylo = a2nlsf_eval_poly(p, xlo, dd); root_ix = 1; }
    else root_ix = 0;
    int k = 1, i = 0;
    while (1) {
        i32 xhi = SB_T(lsf_cos_q12)[k];
        i32 yhi = a2nlsf_eval_poly(p, xhi, dd);
        if ((ylo <= 0 && yhi >= 0) || (ylo >= 0 && yhi <= 0)) {
            i32 ffrac = -256;
            for (int m = 0; m < BIN; m++) {
                i32 xmid = rshift_round(xlo + xhi, 1);
                i32 ymid = a2nlsf_eval_poly(p, xmid, dd);
                if ((ylo <= 0 && ymid >= 0) || (ylo >= 0 && ymid <= 0)) { xhi = xmid; yhi = ymid; }
                else { xlo = xmid; ylo = ymid; ffrac = ffrac + (128 >> m); }
            }
            if (iabs(ylo) < 65536) {
                i32 den = subw(ylo, yhi);
                i32 nom = addw(shl(ylo, 8 - BIN), den >> 1);
                if (den != 0) ffrac += nom / den;
            } else {
                ffrac += ylo / (subw(ylo, yhi) >> (8 - BIN));
            }
            NLSF[root_ix] = imin(shl(k, 8) + ffrac, 32767);
            root_ix++;
            if (root_ix >= d) break;
            p = (root_ix & 1) ? Q : P;
            xlo = SB_T(lsf_cos_q12)[k - 1];
            ylo = shl(1 - (root_ix & 2), 12);
        } else {
            k++;
            xlo = xhi;
            ylo = yhi;
            if (k > TABSZ) {
                i++;
                if (i > MAX_ITER) {
                    NLSF[0] = (1 << 15) / (d + 1);
                    for (k = 1; k < d; k++) NLSF[k] = smulbb(k + 1, NLSF[0]);
                    return;
                }
                bwexpander_32(a_Q16, d, 65536 - smulbb(10 + i, i));
                a2nlsf_init(a_Q16, P, Q, dd);
                p = P;
                xlo = SB_T(lsf_cos_q12)[0];
                ylo = a2nlsf_eval_poly(p, xlo, dd);
                if (ylo < 0) { NLSF[0] = 0; p = Q; ylo = a2nlsf_eval_poly(p, xlo, dd); root_ix = 1; }
                else root_ix = 0;
                k = 1;
            }
        }
    }
}

// ---- SKP_Silk_NLSF2A.c:40-150 ---------------------------------------------------------------------
SB_HD void nlsf2a_find_poly(i32* out, const i32* cLSF, int dd) {
    out[0] = 1 << 20;
    out[1] = negw(cLSF[0]);
    for (int k = 1; k < dd; k++) {
        i32 ftmp = cLSF[2 * k];
        out[k + 1] = subw(shl(out[k - 1], 1), (i32)rshift_round64(smull(ftmp, out[k]), 20));
        for (int n = k; n > 1; n--)
            out[n] = addw(out[n], subw(out[n - 2], (i32)rshift_round64(smull(ftmp, out[n - 1]), 20)));
        out[1] = subw(out[1], ftmp);
    }
}
SB_FN void nlsf2a(i16* a, const i32* NLSF, int d) {
    i32 cos_LSF_Q20[16], P[9], Q[9], a_int32[16];
    for (int k = 0; k < d; k++) {
        i32 f_int = NLSF[k] >> 8;
        i32 f_frac = NLSF[k] - shl(f_int, 8);
        i32 cos_val = SB_T(lsf_cos_q12)[f_int];
        i32 delta = SB_T(lsf_cos_q12)[f_int + 1] - cos_val;
        cos_LSF_Q20[k] = addw(shl(cos_val, 8), mulw(delta, f_frac));
    }
    int dd = d >> 1;
    nlsf2a_find_poly(P, &cos_LSF_Q20[0], dd);
    nlsf2a_find_poly(Q, &cos_LSF_Q20[1], dd);
    for (int k = 0; k < dd; k++) {
        i32 Ptmp = addw(P[k + 1], P[k]);
        i32 Qtmp = subw(Q[k + 1], Q[k]);
        a_int32[k] = negw(rshift_round(addw(Ptmp, Qtmp), 9));
        a_int32[d - k - 1] = rshift_round(subw(Qtmp, Ptmp), 9);
    }
    int i;
    for (i = 0; i < 10; i++) {
        i32 maxabs = 0, idx = 0;
        for (int k = 0; k < d; k++) {
            i32 absval = iabs(a_int32[k]);
            if (absval > maxabs) { maxabs = absval; idx = k; }
        }
        if (maxabs > 32767) {
            maxabs = imin(maxabs, 98369);
            i32 sc_Q16 = 65470 - mulw(65470 >> 2, maxabs - 32767) / (mulw(maxabs, idx + 1) >> 2);
            bwexpander_32(a_int32, d, sc_Q16);
        } else break;
    }
    if (i == 10) for (int k = 0; k < d; k++) a_int32[k] = sat16(a_int32[k]);
    for (int k = 0; k < d; k++) a[k] = (i16)a_int32[k];
}
// SKP_Silk_NLSF2A_stable.c:31-58
SB_FN void nlsf2a_stable(i16* pAR_Q12, const i32* pNLSF, int order) {
    i32 invGain;
    nlsf2a(pAR_Q12, pNLSF, order);
    int i;
    for (i = 0; i < 20; i++) {
        if (lpc_inv_pred_gain_q12(&invGain, pAR_Q12, order) == 1) bwexpander(pAR_Q12, order, 65536 - smulbb(10 + i, i));
        else break;
    }
    if (i == 20) for (i = 0; i < order; i++) pAR_Q12[i] = 0;
}
// SKP_Silk_interpolate.c:31-49
SB_HD void interpolate(i32* xi, const i32* x0, const i32* x1, int ifact_Q2, int d) {
    for (int i = 0; i < d; i++) xi[i] = x0[i] + (mulw(x1[i] - x0[i], ifact_Q2) >> 2);
}

// ---- SKP_Silk_NLSF_stabilize.c:42-138 -----------------------------------------------------------------
SB_FN void nlsf_stabilize(i32* NLSF_Q15, const i32* NDeltaMin_Q15, int L) {
    int loops;
    for (loops = 0; loops < 20; loops++) {
        i32 min_diff = NLSF_Q15[0] - NDeltaMin_Q15[0];
        int I = 0;
        for (int i = 1; i <= L - 1; i++) {
            i32 diff = NLSF_Q15[i] - (NLSF_Q15[i - 1] + NDeltaMin_Q15[i]);
            if (diff < min_diff) { min_diff = diff; I = i; }
        }
        i32 diff = (1 << 15) - (NLSF_Q15[L - 1] + NDeltaMin_Q15[L]);
        if (diff < min_diff) { min_diff = diff; I = L; }
        if (min_diff >= 0) return;
        if (I == 0) NLSF_Q15[0] = NDeltaMin_Q15[0];
        else if (I == L) NLSF_Q15[L - 1] = (1 << 15) - NDeltaMin_Q15[L];
        else {
            i32 min_center = 0;
            for (int k = 0; k < I; k++) min_center += NDeltaMin_Q15[k];
            min_center += NDeltaMin_Q15[I] >> 1;
            i32 max_center = 1 << 15;
            for (int k = L; k > I; k--) max_center -= NDeltaMin_Q15[k];
            max_center -= (NDeltaMin_Q15[I] - (NDeltaMin_Q15[I] >> 1));
            i32 center = limit(rshift_round(NLSF_Q15[I - 1] + NLSF_Q15[I], 1), min_center, max_center);
            NLSF_Q15[I - 1] = center - (NDeltaMin_Q15[I] >> 1);
            NLSF_Q15[I] = NLSF_Q15[I - 1] + NDeltaMin_Q15[I];
        }
    }
    if (loops == 20) {
        for (int i = 1; i < L; i++) {
            i32 value = NLSF_Q15[i]; int j;
            for (j = i - 1; j >= 0 && value < NLSF_Q15[j]; j--) NLSF_Q15[j + 1] = NLSF_Q15[j];
            NLSF_Q15[j + 1] = value;
        }
        NLSF_Q15[0] = imax(NLSF_Q15[0], NDeltaMin_Q15[0]);
        for (int i = 1; i < L; i++) NLSF_Q15[i] = imax(NLSF_Q15[i], NLSF_Q15[i - 1] + NDeltaMin_Q15[i]);
        NLSF_Q15[L - 1] = imin(NLSF_Q15[L - 1], (1 << 15) - NDeltaMin_Q15[L]);
        for (int i = L - 2; i >= 0; i--) NLSF_Q15[i] = imin(NLSF_Q15[i], NLSF_Q15[i + 1] - NDeltaMin_Q15[i + 1]);
    }
}

// ---- SKP_Silk_NLSF_VQ_weights_laroia.c:40-79 --------------------------------------------------------
SB_FN void nlsf_vq_weights_laroia(i32* pW_Q6, const i32* pNLSF_Q15, int D) {
    i32 t1 = (1 << 21) / imax(pNLSF_Q15[0], 3);
    i32 t2 = (1 << 21) / imax(pNLSF_Q15[1] - pNLSF_Q15[0], 3);
    pW_Q6[0] = imin(t1 + t2, 32767);
    for (int k = 1; k < D - 1; k += 2) {
        t1 = (1 << 21) / imax(pNLSF_Q15[k + 1] - pNLSF_Q15[k], 3);
        pW_Q6[k] = imin(t1 + t2, 32767);
        t2 = (1 << 21) / imax(pNLSF_Q15[k + 2] - pNLSF_Q15[k + 1], 3);
        pW_Q6[k + 1] = imin(t1 + t2, 32767);
    }
    t1 = (1 << 21) / imax((1 << 15) - pNLSF_Q15[D - 1], 3);
    pW_Q6[D - 1] = imin(t1 + t2, 32767);
}

// ---- NLSF codebook accessors (tables_NLSF_CB{0,1}_10.c; order 16: tables_NLSF_CB{0,1}_16.c) ----------------------------
struct NlsfCb {
    const i16* cb_q15;       // all stages, concatenated
    const i16* rates_q5;
    const i32* ndelta_min;   // [order + 1]
    const i32* nvec;         // [stages]: 6 at order 10, 10 at order 16
    const u16* cdf;
    const i32* cdf_start;    // [stages] element offsets into cdf
    const i32* cdf_mid;      // [stages]
};
template <int D = 10> SB_HD NlsfCb nlsf_cb(int sigtype) {
    static_assert(D == 10 || D == 16, "NLSF codebooks exist for orders 10 and 16");
    NlsfCb c;
    if constexpr (D == 10) {
        if (sigtype == 0) {
            c.cb_q15 = SB_T(nlsf_cb0_q15); c.rates_q5 = SB_T(nlsf_cb0_rates_q5); c.ndelta_min = SB_T(nlsf_cb0_ndelta_min_q15);
            c.nvec = SB_T(nlsf_cb0_nvec); c.cdf = SB_T(nlsf_cb0_cdf); c.cdf_start = SB_T(nlsf_cb0_cdf_start); c.cdf_mid = SB_T(nlsf_cb0_cdf_mid);
        } else {
            c.cb_q15 = SB_T(nlsf_cb1_q15); c.rates_q5 = SB_T(nlsf_cb1_rates_q5); c.ndelta_min = SB_T(nlsf_cb1_ndelta_min_q15);
            c.nvec = SB_T(nlsf_cb1_nvec); c.cdf = SB_T(nlsf_cb1_cdf); c.cdf_start = SB_T(nlsf_cb1_cdf_start); c.cdf_mid = SB_T(nlsf_cb1_cdf_mid);
        }
    } else {
        if (sigtype == 0) {
            c.cb_q15 = SB_T(nlsf16_cb0_q15); c.rates_q5 = SB_T(nlsf16_cb0_rates_q5); c.ndelta_min = SB_T(nlsf16_cb0_ndelta_min_q15);
            c.nvec = SB_T(nlsf16_cb0_nvec); c.cdf = SB_T(nlsf16_cb0_cdf); c.cdf_start = SB_T(nlsf16_cb0_cdf_start); c.cdf_mid = SB_T(nlsf16_cb0_cdf_mid);
        } else {
            c.cb_q15 = SB_T(nlsf16_cb1_q15); c.rates_q5 = SB_T(nlsf16_cb1_rates_q5); c.ndelta_min = SB_T(nlsf16_cb1_ndelta_min_q15);
            c.nvec = SB_T(nlsf16_cb1_nvec); c.cdf = SB_T(nlsf16_cb1_cdf); c.cdf_start = SB_T(nlsf16_cb1_cdf_start); c.cdf_mid = SB_T(nlsf16_cb1_cdf_mid);
        }
    }
    return c;
}
// number of MSVQ stages of the order-D codebooks
template <int D> struct NlsfStages { enum { N = D == 16 ? 10 : 6 }; };
// SKP_Silk_NLSF_MSVQ_decode.c:31-98 (order 10 with 6 stages, order 16 with 10)
template <int D = 10> SB_FN void nlsf_msvq_decode(i32* pNLSF_Q15, const NlsfCb& cb, const i32* idx) {
    enum { NST = NlsfStages<D>::N };
    const i16* e = cb.cb_q15 + idx[0] * D;
    for (int i = 0; i < D; i++) pNLSF_Q15[i] = e[i];
    int base = cb.nvec[0];
    for (int s = 1; s < NST; s++) {
        e = cb.cb_q15 + (base + idx[s]) * D;
        for (int i = 0; i < D; i++) pNLSF_Q15[i] += e[i];
        base += cb.nvec[s];
    }
    nlsf_stabilize(pNLSF_Q15, cb.ndelta_min, D);
}

}  // namespace sb
