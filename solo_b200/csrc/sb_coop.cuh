// solo_b200 -- encoder analysis stage in its warp-cooperative form: ONE stream = ONE warp.
//
// Every routine here is called by all 32 lanes of the warp that owns the stream (convergently), works on arrays in shared
// memory and keeps scalars in registers.  The work of a routine is laid out over the lanes in one of four ways:
//   * lanes over outputs      -- FIR filters, correlations per lag, code-vector errors: no communication at all;
//   * lanes over terms + sum  -- wrap-around integer sums (mod 2^32 / 2^64 addition is associative, so the bits match the
//                                reference's sequential accumulation);
//   * lanes over stages       -- the warped all-pass chains run as a skewed wavefront (lane = stage, one shuffle per step);
//   * lane per instance       -- short recursions that exist several times per frame (4 shaping windows, 4 LTP sub-frames,
//                                4 interpolation candidates) run as one scalar instance per lane.
// Short scalar recursions that exist once or a few times per stream (high-pass biquad, decimator chains, Schur / step-up
// recursions per window, LTP normal equations per sub-frame, NLSF -> LPC conversions) run as "instances": the block's streams
// side by side on consecutive threads (c_instances, sb_par.cuh).  Pure recurrences that depend on nothing else in the frame
// are not here at all: the voice-activity detector runs before this kernel, the shaping-filter finishing and the prefilter
// after it, as thread-per-instance kernels (solo_b200.cu).
// The per-frame control arithmetic between the lane-parallel cores (thresholds, scores, gains, shaping parameters, the
// per-window shaping filter) is not restated here: it is the SB_HD helpers next to the scalar routines of sb_enc_*.cuh /
// sb_sigproc.cuh, which both forms call.  tests/hostsim compiles both forms and checks this file (32 fibres per stream,
// sb_par.cuh SB_EMU) against the golden bitstream and the scalar model on a machine without a GPU.
#pragma once
#include "sb_enc.cuh"
#include "sb_par.cuh"

#if SB_COOP_ACTIVE
namespace sb {

// ---------------------------------------------------------------------------------------------------------------------
// primitives
// ---------------------------------------------------------------------------------------------------------------------
SB_HD int popc32(u32 x) {
#ifdef __CUDA_ARCH__
    return __popc(x);
#else
    return __builtin_popcount(x);
#endif
}
SB_HD int ctz32(u32 x) {   // x != 0
#ifdef __CUDA_ARCH__
    return __ffs((int)x) - 1;
#else
    return __builtin_ctz(x);
#endif
}
// Zero-state FIR (SKP_Silk_MA_Prediction / SKP_Silk_LPC_analysis_filter with a cleared state, SKP_Silk_MA.c:41-118):
// out[k] = sat16(rshift_round((in[k] << 12) - sum_{d < min(ORD, k)} B[d] * in[k-1-d], 12)); lanes over outputs.
template <int ORD, bool SAT> SB_CFN void c_fir_zero_state(const i16* in, const i16* B_Q12, i16* out, int len) {
    i32 b[ORD];
#pragma unroll
    for (int d = 0; d < ORD; d++) b[d] = B_Q12[d];
    SB_PARFOR(k, 0, len) {
        i32 acc = 0;
        if (k >= ORD) {
#pragma unroll
            for (int d = 0; d < ORD; d++) acc = addw(acc, (i32)in[k - 1 - d] * b[d]);
        } else {
#pragma unroll
            for (int d = 0; d < ORD; d++) if (d < k) acc = addw(acc, (i32)in[k - 1 - d] * b[d]);
        }
        const i32 x = in[k];
        const i32 o = SAT ? sub_sat32(shl(x, 12), acc) : subw(shl(x, 12), acc);
        out[k] = (i16)sat16(rshift_round(o, 12));
    }
}

// SKP_Silk_schur (schur.c:40-93), order <= 31: lane n keeps C[n][1] and C[n+k+1][0] in registers; the second slides down
// one lane per step.  c: correlations (shared memory); rc_Q15: shared; returns the residual energy on every lane.
SB_CFN i32 c_schur(i16* rc_Q15, const i32* c, int order) {
    const int lane = SB_LANE;
    const int lz = clz32(c[0]);
    i32 a = 0, b = 0;
    if (lane <= order) { const i32 v = c[lane]; a = lz < 2 ? (v >> 1) : (lz > 2 ? shl(v, lz - 2) : v); }
    b = wshfl_down(a, 1);
    for (int k = 0; k < order; k++) {
        const i32 c00 = wbcast(b, 0), c01 = wbcast(a, 0);
        const i32 rc = sat16(negw(c00 / imax(c01 >> 15, 1)));
        if (lane == 0) rc_Q15[k] = (i16)rc;
        if (lane < order - k) {
            const i32 t1 = b, t2 = a;
            b = smlawb(t1, shl(t2, 1), rc);
            a = smlawb(t2, shl(t1, 1), rc);
        }
        b = wshfl_down(b, 1);
    }
    return wbcast(a, 0);
}
// SKP_Silk_k2a (k2a.c:40-60): lane n keeps A[n]; returns it (valid for n < order).  rc_Q15: shared memory.
SB_CFN i32 c_k2a(const i16* rc_Q15, int order) {
    const int lane = SB_LANE;
    i32 A = 0;
    for (int k = 0; k < order; k++) {
        const i32 rc = rc_Q15[k];
        const i32 t = wshfl(A, (k - lane - 1) & 31);
        if (lane < k) A = smlawb(A, shl(t, 1), rc);
        if (lane == k) A = negw(shl(rc, 9));
    }
    return A;
}
// chirp factor that SKP_Silk_bwexpander (bwexpander.c:31-48) applies to coefficient `lane` (d coefficients)
SB_CFN i32 c_bwexpander_chirp16(int d, i32 chirp_Q16) {
    const int lane = SB_LANE;
    const i32 cm1 = chirp_Q16 - 65536;
    i32 mine = chirp_Q16;
    for (int i = 0; i < d - 1; i++) {
        if (lane == i) mine = chirp_Q16;
        chirp_Q16 += rshift_round(mulw(chirp_Q16, cm1), 16);
    }
    if (lane >= d - 1) mine = chirp_Q16;
    return mine;
}
// factor that SKP_Silk_bwexpander_32 (bwexpander_32.c:31-47) multiplies into coefficient `lane`
SB_CFN i32 c_bwexpander32_factor(int d, i32 chirp_Q16) {
    const int lane = SB_LANE;
    i32 t = chirp_Q16, mine = chirp_Q16;
    for (int i = 0; i < d - 1; i++) {
        if (lane == i) mine = t;
        t = smulww(chirp_Q16, t);
    }
    if (lane >= d - 1) mine = t;
    return mine;
}

// ---------------------------------------------------------------------------------------------------------------------
// pitch analysis (SKP_Silk_find_pitch_lags_FIX.c:32-125, SKP_Silk_pitch_analysis_core.c:65-560 at 8 kHz, complexity 2)
// ---------------------------------------------------------------------------------------------------------------------
struct PitchScr {
    i16 Wsig[PITCH_LPC_WIN];
    i16 sig8[2 * FRAME];
    i16 sig4[FRAME];
    i16 C1[2][66];        // first-stage correlations, index lag - 8
    i16 C2[4][48];        // second-stage correlations by candidate slot
    i16 d_comp[48];
    i16 dc[160];          // candidate marks / their running sums, index lag
    i32 d_srch[24];
    u8 slot[152];         // lag -> candidate slot + 1 (0: not computed, correlation 0)
    i32 acorr[12];
    i16 rc_Q15[16];
    i16 A_Q12[16];
    i32 dn[2][FRAME];     // outputs of the two all-pass chains of the 2:1 decimator
};

SB_CFN int c_pitch_analysis_core(PitchScr* P, const i16* signal, i32* pitch_out, i32* lagIndex, i32* contourIndex, i32* LTPCorr_Q15,
                                i32 prevLag, i32 search_thres1_Q16, i32 search_thres2_Q15) {
    enum { FL8 = 320, FL4 = 160, SF8 = 40, MINL8 = 16, MAXL8 = 144, MINL4 = 8, MAXL4 = 72, NCB = 11, NL4 = MAXL4 - MINL4 + 1 };
    const int lane = SB_LANE;
    i16* sig8 = P->sig8;
    i16* sig4 = P->sig4;
    SB_PARFOR(i, 0, FL8) sig8[i] = signal[i];
    SB_SYNC();
    // 2:1 decimator: one recurrence over the frame (lane 0)
    // (SKP_Silk_resampler_down2.c:41-78 from a cleared state): the two all-pass chains (even / odd input samples) as two scalar
    // instances, their outputs added afterwards -- out32 is a wrap-around sum of the four terms, so the order is free
    c_instances<2>([&](int d, int k) {
        PitchScr* Pj = xoff(P, d);
        const i16* __restrict__ in = Pj->sig8;
        i32* __restrict__ o = Pj->dn[k];
        i32 S = 0;
        if (k == 0) {
            const i32 c1 = SB_T(resampler_down2_1)[0];
#pragma unroll 8
            for (int q = 0; q < FL4; q++) { const i32 in32 = shl((i32)in[2 * q], 10); const i32 Y = subw(in32, S); const i32 X = smlawb(Y, Y, c1); o[q] = addw(S, X); S = addw(in32, X); }
        } else {
            const i32 c0 = SB_T(resampler_down2_0)[0];
#pragma unroll 8
            for (int q = 0; q < FL4; q++) { const i32 in32 = shl((i32)in[2 * q + 1], 10); const i32 Y = subw(in32, S); const i32 X = smulwb(Y, c0); o[q] = addw(S, X); S = addw(in32, X); }
        }
    });
    SB_PARFOR(i, 0, FL4) sig4[i] = (i16)sat16(rshift_round(addw(P->dn[0][i], P->dn[1][i]), 11));
    SB_SYNC();
    // low-pass (descending in-place loop of the reference = old values on the right-hand side) + scaling
    i32 v[5];
#pragma unroll
    for (int j = 0; j < 5; j++) { const int i = lane + 32 * j; v[j] = i > 0 ? add_sat16(sig4[i], sig4[i - 1]) : (i32)sig4[0]; }
    SB_SYNC();
    i32 shift = pitch_find_scaling(wmax(imax(imax(imax(iabs(v[0]), iabs(v[1])), imax(iabs(v[2]), iabs(v[3]))), iabs(v[4]))), imax(SF8, FL4 >> 1));
#pragma unroll
    for (int j = 0; j < 5; j++) sig4[lane + 32 * j] = (i16)((i16)v[j] >> shift);
    SB_SYNC();

    // ---- first stage at 4 kHz: lanes over (half, lag) ----
    const i16* target0 = &sig4[FL4 >> 1];
    i32 e8 = 0;     // energy of the first basis vector (lag 8) of half `lane` (lanes 0, 1)
    if (lane < 2) { const i16* b = target0 + lane * SF8 - MINL4; for (int i = 0; i < SF8; i++) e8 = addw(e8, (i32)b[i] * (i32)b[i]); }
    const i32 e8_0 = wbcast(e8, 0), e8_1 = wbcast(e8, 1);
    SB_PARFOR(t, 0, 2 * NL4) {
        const int k = t >= NL4, d = MINL4 + t - k * NL4;
        const i16* target = target0 + k * SF8;
        const i16* basis = target - d;
        i32 cross = 0, e = 0;
#pragma unroll 8
        for (int i = 0; i < SF8; i++) { const i32 bv = basis[i]; cross = addw(cross, (i32)target[i] * bv); e = addw(e, bv * bv); }
        const i32 ek = k ? e8_1 : e8_0;
        const i32 normalizer = addw(add_sat32(ek, smulbb(SF8, 4000)), subw(e, ek));   // recursion of the reference, unrolled
        P->C1[k][d - MINL4] = (i16)sat16(cross / (sqrt_approx(normalizer) + 1));
    }
    SB_SYNC();
    i32 cs[3];
#pragma unroll
    for (int j = 0; j < 3; j++) {
        const int i = lane + 32 * j;
        if (i < NL4) {
            i32 sum = ((i32)P->C1[0][i] + (i32)P->C1[1][i]) >> 1;
            cs[j] = smlawb(sum, sum, shl(-(i + MINL4), 4));
        }
    }
    SB_SYNC();
#pragma unroll
    for (int j = 0; j < 3; j++) { const int i = lane + 32 * j; if (i < NL4) P->C1[0][i] = (i16)cs[j]; }
    SB_SYNC();
    int length_d_srch = 4 + 2 * 2;
    {   // the eight largest of the 65 smoothed correlations, in the order the reference's stable partial insertion sort
        // (sort.c:79-124) leaves them: by value, equal values by position.  Eight rounds of a warp-wide arg-max.
        i32 v3[3];
#pragma unroll
        for (int j = 0; j < 3; j++) { const int i = lane + 32 * j; v3[j] = i < NL4 ? (i32)P->C1[0][i] : SB_I32_MIN; }
        SB_SYNC();
        for (int r = 0; r < 4 + 2 * 2; r++) {
            i32 bv = v3[0], bi = lane;
            if (v3[1] > bv) { bv = v3[1]; bi = lane + 32; }
            if (v3[2] > bv) { bv = v3[2]; bi = lane + 64; }
            wargmax(bv, bi);        // ties: smallest position
            if (lane == (bi & 31)) { const int j = bi >> 5; if (j == 0) v3[0] = SB_I32_MIN; else if (j == 1) v3[1] = SB_I32_MIN; else v3[2] = SB_I32_MIN; }
            if (lane == 0) { P->C1[0][r] = (i16)bv; P->d_srch[r] = bi; }
        }
    }
    i32 energy;
    {
        i32 part = 0;
        SB_PARFOR(i, 0, FL4 >> 1) part = addw(part, (i32)target0[i] * (i32)target0[i]);
        energy = add_pos_sat32(wsum(part), 1000);
    }
    SB_SYNC();
    const i32 Cmax = P->C1[0][0];
    i32 threshold = smulbb(Cmax, Cmax);
    if ((energy >> (4 + 2)) > threshold) {     // uniform
        if (lane < 4) pitch_out[lane] = 0;
        if (lane == 0) { *LTPCorr_Q15 = 0; *lagIndex = 0; *contourIndex = 0; }
        SB_SYNC();
        return 1;
    }
    threshold = smulwb(search_thres1_Q16, Cmax);
    {
        const bool ok = lane < length_d_srch && P->C1[0][lane] > threshold;
        const u32 bad = ~wballot(ok) & ((1u << length_d_srch) - 1);
        if (bad) length_d_srch = ctz32(bad);         // the list ends at the first entry below the threshold
    }
    SB_PARFOR(i, 0, 160) P->dc[i] = 0;
    SB_SYNC();
    if (lane < length_d_srch) { const i32 d = (P->d_srch[lane] + MINL4) << 1; P->dc[d] = 1; }
    SB_SYNC();
    // running sums over 3, then over 4 lags (the reference's in-place descending loops read unmodified lower entries)
    i32 w5[5];
#pragma unroll
    for (int j = 0; j < 5; j++) { const int i = MINL8 + lane + 32 * j; w5[j] = i <= MAXL8 + 3 ? P->dc[i] + P->dc[i - 1] + P->dc[i - 2] : 0; }
    SB_SYNC();
#pragma unroll
    for (int j = 0; j < 5; j++) { const int i = MINL8 + lane + 32 * j; if (i <= MAXL8 + 3) P->dc[i] = (i16)w5[j]; }
    SB_SYNC();
    length_d_srch = 0;
#pragma unroll
    for (int j = 0; j < 5; j++) {
        const int i = MINL8 + lane + 32 * j;
        const bool on = i < MAXL8 + 1 && P->dc[i + 1] > 0;
        const u32 m = wballot(on);
        if (on) P->d_srch[length_d_srch + popc32(m & ((1u << lane) - 1))] = i;
        length_d_srch += popc32(m);
    }
#pragma unroll
    for (int j = 0; j < 5; j++) { const int i = MINL8 + lane + 32 * j; w5[j] = i <= MAXL8 + 3 ? P->dc[i] + P->dc[i - 1] + P->dc[i - 2] + P->dc[i - 3] : 0; }
    SB_SYNC();
    int length_d_comp = 0;
    SB_PARFOR(i, 0, 152) P->slot[i] = 0;
    SB_SYNC();
#pragma unroll
    for (int j = 0; j < 5; j++) {
        const int i = MINL8 + lane + 32 * j;
        const bool on = i < MAXL8 + 4 && w5[j] > 0;
        const u32 m = wballot(on);
        if (on) {
            const int q = length_d_comp + popc32(m & ((1u << lane) - 1));
            P->d_comp[q] = (i16)(i - 2);
            P->slot[i - 2] = (u8)(q + 1);
        }
        length_d_comp += popc32(m);
    }

    // ---- second stage at 8 kHz: lanes over (sub-frame, candidate lag) ----
    {
        i32 m8 = 0;
        SB_PARFOR(i, 0, FL8) m8 = imax(m8, iabs((i32)sig8[i]));
        shift = pitch_find_scaling(wmax(m8), SF8);
    }
    if (shift > 0) SB_PARFOR(i, 0, FL8) sig8[i] = (i16)(sig8[i] >> shift);
    SB_SYNC();
    i32 et = 0;      // energy of target sub-frame `lane` (lanes 0..3)
    if (lane < 4) { const i16* tp = &sig8[FL4 + lane * SF8]; for (int i = 0; i < SF8; i++) et = addw(et, (i32)tp[i] * (i32)tp[i]); }
    const i32 et0 = wbcast(et, 0), et1 = wbcast(et, 1), et2 = wbcast(et, 2), et3 = wbcast(et, 3);
    SB_PARFOR(t, 0, 4 * length_d_comp) {
        const int k = t / length_d_comp, j = t - k * length_d_comp;
        const int d = P->d_comp[j];
        const i16* target = &sig8[FL4 + k * SF8];
        const i16* basis = target - d;
        i32 cross_corr = 0, energy_basis = 0;
#pragma unroll 8
        for (int i = 0; i < SF8; i++) { const i32 bv = basis[i]; cross_corr = addw(cross_corr, (i32)target[i] * bv); energy_basis = addw(energy_basis, bv * bv); }
        const i32 energy_target = k == 0 ? et0 : (k == 1 ? et1 : (k == 2 ? et2 : et3));
        P->C2[k][j] = (i16)pitch_stage2_corr(cross_corr, energy_target, energy_basis);
    }
    SB_SYNC();
    // ---- search over the short list (one candidate lag per lane) ----
    const i16* cbl = SB_T(pitch_cb_lags_stage2);   // [4][11]
    const i32 ltpcorr_prev = *LTPCorr_Q15;
    i32 key = SB_I32_MIN, my_cc = SB_I32_MIN, my_cb = 0, my_d = 0;
    if (lane < length_d_srch) {
        const int d = P->d_srch[lane];
        i32 CCmax_new = SB_I32_MIN; int CBimax_new = 0;
        for (int j = 0; j < NCB; j++) {
            i32 cc = 0;
#pragma unroll
            for (int i = 0; i < 4; i++) { const int sl = P->slot[d + cbl[i * NCB + j]]; cc += sl ? (i32)P->C2[i][sl - 1] : 0; }
            if (cc > CCmax_new) { CCmax_new = cc; CBimax_new = j; }
        }
        key = pitch_lag_score(CCmax_new, CBimax_new, d, prevLag, ltpcorr_prev, search_thres2_Q15);
        my_cc = CCmax_new; my_cb = CBimax_new; my_d = d;
    }
    i32 best = key, who = lane;
    wargmax(best, who);        // first of equal maxima, as the ascending scan with a strict comparison keeps it
    SB_SYNC();                 // every lane has read the previous correlation (ltpcorr_prev) before lane 0 replaces it
    if (best == SB_I32_MIN) {  // uniform
        if (lane < 4) pitch_out[lane] = 0;
        if (lane == 0) { *LTPCorr_Q15 = 0; *lagIndex = 0; *contourIndex = 0; }
        SB_SYNC();
        return 1;
    }
    const i32 CCmax = imax(wshfl(my_cc, who), 0);
    const i32 CBimax = wshfl(my_cb, who), lag = wshfl(my_d, who);
    if (lane < 4) pitch_out[lane] = lag + cbl[lane * NCB + CBimax];
    if (lane == 0) { *LTPCorr_Q15 = sqrt_approx(shl(CCmax, 13)); *lagIndex = lag - MINL8; *contourIndex = CBimax; }
    SB_SYNC();
    return 0;
}

// x points at x_buf + FRAME; res receives 336 samples of LPC residual.  All lanes return (and c gets) the signal type.
SB_CFN void c_find_pitch_lags(EncSilk* st, EncCtrl* c, PitchScr* P, i16* res, const i16* x) {
    enum { BUF_LEN = LA_PITCH + 2 * FRAME, ORD = 10 };
    const int lane = SB_LANE;
    const i16* x_buf = x - FRAME;
    const i16* x_buf_ptr = x_buf + BUF_LEN - PITCH_LPC_WIN;
    // 24 ms window: sine slopes on two lanes (16 samples each), flat part copied by all
    if (lane == 0) apply_sine_window(P->Wsig, x_buf_ptr, 1, LA_PITCH);
    if (lane == 1) apply_sine_window(P->Wsig + PITCH_LPC_WIN - LA_PITCH, x_buf_ptr + PITCH_LPC_WIN - LA_PITCH, 2, LA_PITCH);
    SB_PARFOR(i, 0, PITCH_LPC_WIN - 2 * LA_PITCH) P->Wsig[LA_PITCH + i] = x_buf_ptr[LA_PITCH + i];
    SB_SYNC();
    // autocorrelation, 11 lags (SKP_Silk_autocorr, autocorr.c:40-77): lanes over samples, 64-bit partial sums
    i64 acc[ORD + 1];
#pragma unroll
    for (int i = 0; i <= ORD; i++) acc[i] = 0;
    for (int j = 0; j < PITCH_LPC_WIN / 32; j++) {
        const int n = lane + 32 * j;
        const i32 xn = P->Wsig[n];
#pragma unroll
        for (int i = 0; i <= ORD; i++) if (n + i < PITCH_LPC_WIN) acc[i] += (i64)(xn * (i32)P->Wsig[n + i]);
    }
#pragma unroll
    for (int i = 0; i <= ORD; i++) acc[i] = wsum64(acc[i]);
    {
        const i64 corr64 = acc[0] + 1;
        const int nrs = 35 - clz64(corr64);
#pragma unroll
        for (int i = 0; i <= ORD; i++) {
            const i64 s = i == 0 ? corr64 : acc[i];
            const i32 r = nrs <= 0 ? shl((i32)s, -nrs) : (i32)(s >> nrs);
            if (lane == i) P->acorr[i] = i == 0 ? smlawb(r, r, SB_FIXC(1e-3f, 16)) : r;
        }
    }
    SB_SYNC();
    const i32 ac0 = P->acorr[0];
    const i32 res_nrg = c_schur(P->rc_Q15, P->acorr, ORD);
    const i32 predGain = pitch_pred_gain_q16(ac0, res_nrg);
    SB_SYNC();
    const i32 A_Q24 = c_k2a(P->rc_Q15, ORD);
    {
        const i32 chirp = c_bwexpander_chirp16(ORD, SB_FIXC(0.99f, 16));
        if (lane < ORD) P->A_Q12[lane] = (i16)rshift_round(mulw(chirp, (i32)(i16)sat16(A_Q24 >> 12)), 16);
    }
    SB_SYNC();
    c_fir_zero_state<ORD, false>(x_buf, P->A_Q12, res, BUF_LEN);
    SB_SYNC();
    if (lane < ORD) res[lane] = 0;
    const i32 thrhld_Q15 = pitch_thrhld_q15(st->speech_activity_Q8, st->prev_sigtype, c->input_tilt_Q15);
    const i32 prevLag = st->prevLag;
    SB_SYNC();
    SB_PHASE();
    const int sigtype = c_pitch_analysis_core(P, res, c->pitchL, &c->lagIndex, &c->contourIndex, &st->LTPCorr_Q15, prevLag,
                                              SB_FIXC(0.7f, 16), thrhld_Q15);
    if (lane == 0) { c->sigtype = sigtype; c->predGain_Q16 = predGain; }
    SB_SYNC();
}

// ---------------------------------------------------------------------------------------------------------------------
// noise-shape analysis (SKP_Silk_noise_shape_analysis_FIX.c:137-531)
// ---------------------------------------------------------------------------------------------------------------------
struct ShapeScr {
    i16 xw[NB_SUBFR][SHAPE_WIN];
    i32 acorr[NB_SUBFR][SHAPE_ORDER + 1];
    i32 scale[NB_SUBFR];
    i32 par3[3];                 // warping_Q16, BWExp1_Q16, BWExp2_Q16 for the per-window instances
    i32 gains[NB_SUBFR][2];      // their results: Gains_Q16, GainsPre_Q14 before the frame-level tweaks
    i32 ar[NB_SUBFR][2][SHAPE_ORDER];   // AR2_Q24, AR1_Q24 between the instance stages
    i32 invgain[NB_SUBFR][2];
};

// Warped autocorrelation of the four shaping windows at once (SKP_Silk_warped_autocorrelation_FIX.c:36-85): the 16
// all-pass sections run as a wavefront, lane g of an 8-lane group owns sections 2g and 2g+1 of its window and works on
// sample t - g at step t; a section's right-hand state is its own previous output, so one shuffle per step suffices.
SB_CFN void c_warped_autocorr4(ShapeScr* S, i32 warping_Q16) {
    const int QC = 10, QS = 14;
    const int lane = SB_LANE, g = lane & 7, win = lane >> 3;
    const i16* input = S->xw[win];
    const i32 w = (i16)warping_Q16;
    i32 p0 = 0, p1 = 0, p2 = 0, out = 0;
    i64 c0 = 0, c1 = 0, c2 = 0;
    for (int t = 0; t < SHAPE_WIN + 7; t++) {
        const int n = t - g;
        const i32 from_prev = wshfl_up(out, 1);
        if (n >= 0 && n < SHAPE_WIN) {
            const i32 s0 = shl((i32)input[n], QS);
            const i32 in = g == 0 ? s0 : from_prev;
            const i32 tmp2 = smlawb(p0, subw(p1, in), w);
            const i32 tmp1 = smlawb(p1, subw(p2, tmp2), w);
            c0 += smull(in, s0) >> (2 * QS - QC);
            c1 += smull(tmp2, s0) >> (2 * QS - QC);
            if (g == 7) c2 += smull(tmp1, s0) >> (2 * QS - QC);
            p0 = in; p1 = tmp2; p2 = tmp1; out = tmp1;
        }
    }
    const i64 corr0 = wshfl64(c0, win * 8);
    int lsh = clz64(corr0) - 35;
    lsh = limit(lsh, -12 - QC, 30 - QC);
    i32* corr = S->acorr[win];
    if (lsh >= 0) {
        corr[2 * g] = (i32)shl64(c0, lsh); corr[2 * g + 1] = (i32)shl64(c1, lsh);
        if (g == 7) corr[16] = (i32)shl64(c2, lsh);
    } else {
        corr[2 * g] = (i32)(c0 >> (-lsh)); corr[2 * g + 1] = (i32)(c1 >> (-lsh));
        if (g == 7) corr[16] = (i32)(c2 >> (-lsh));
    }
    if (g == 0) S->scale[win] = -(QC + lsh);
}

// pitch_res points at res_pitch + FRAME, x at x_buf + FRAME.
SB_CFN void c_noise_shape_analysis(EncSilk* st, EncCtrl* c, ShapeScr* S, const i16* pitch_res, const i16* x) {
    const int lane = SB_LANE;
    // ---- scalars, computed by every lane from shared data; lane 0 stores ----
    const i32 sigtype = c->sigtype;
    const i32 speech_activity_Q8 = st->speech_activity_Q8, LTPCorr_Q15 = st->LTPCorr_Q15;
    // sparseness of the residual (unvoiced): ten 2 ms energies, one per lane
    i32 energy_variation_Q7 = 0;
    if (sigtype != 0) {      // uniform
        i32 log_energy_Q7 = 0;
        if (lane < 10) {
            i32 nrg, scale;
            sum_sqr_shift(&nrg, &scale, pitch_res + 16 * lane, 16, 0);
            nrg += 16 >> scale;
            log_energy_Q7 = lin2log(nrg);
        }
        const i32 prev = wshfl_up(log_energy_Q7, 1);
        energy_variation_Q7 = wsum((lane >= 1 && lane < 10) ? iabs(log_energy_Q7 - prev) : 0);
    }
    const ShapeCtl s = shape_control(sigtype, st->SNR_dB_Q7, st->SNRPerMD_dB_Q7, c->input_quality_bands_Q15, speech_activity_Q8,
                                     LTPCorr_Q15, energy_variation_Q7, c->predGain_Q16);
    const i32 warping_Q16 = s.warping_Q16;

    // ---- the four 15 ms windows: slopes on eight lanes, flat parts copied by all ----
    {
        const int slope = (SHAPE_WIN - 40) >> 1;   // 40
        if (lane < 8) {
            const int k = lane >> 1, h = lane & 1;
            const i16* xp = x - LA_SHAPE + k * SUBFR + h * (slope + 40);
            apply_sine_window(S->xw[k] + h * (slope + 40), xp, h + 1, slope);
        }
        SB_PARFOR(i, 0, NB_SUBFR * 40) {
            const int k = i / 40, j = i - 40 * k;
            S->xw[k][slope + j] = (x - LA_SHAPE + k * SUBFR)[slope + j];
        }
    }
    SB_SYNC();
    SB_PHASE();
    c_warped_autocorr4(S, warping_Q16);
    SB_SYNC();
    SB_PHASE();
    // ---- per window: reflection coefficients, shaping filters, gains -- one scalar instance per window ----
    if (lane == 0) { S->par3[0] = warping_Q16; S->par3[1] = s.BWExp1_Q16; S->par3[2] = s.BWExp2_Q16; }
    c_instances<NB_SUBFR>([&](int d, int k) {
        ShapeScr* Sj = xoff(S, d);
        i32 auto_corr[SHAPE_ORDER + 1], AR1_Q24[SHAPE_ORDER], AR2_Q24[SHAPE_ORDER];
#pragma unroll
        for (int i = 0; i <= SHAPE_ORDER; i++) auto_corr[i] = Sj->acorr[k][i];
        Sj->gains[k][0] = shape_window(AR2_Q24, AR1_Q24, auto_corr, Sj->scale[k], Sj->par3[0], Sj->par3[1], Sj->par3[2]);
#pragma unroll
        for (int i = 0; i < SHAPE_ORDER; i++) { Sj->ar[k][0][i] = AR2_Q24[i]; Sj->ar[k][1][i] = AR1_Q24[i]; }
    });
    // (inverse prediction gains, pre-gains, coefficient limiting and the Q13 coefficients of the windows are finished by the
    //  shaping-filter kernel that runs after this one: nothing in the rest of the analysis reads them)
    // ---- gain tweaking: lane k owns sub-frame k ----
    const i32 md_gain_mult_Q16 = shape_gain_mult_q16(s.md_SNR_adj_dB_Q7);
    const i32 gain_mult_Q16 = shape_gain_mult_q16(s.SNR_adj_dB_Q7);
    const float md_delta_gain_par = (float)gain_mult_Q16 / (float)md_gain_mult_Q16;
    i32 avgGain_Q16 = st->avgGain_Q16;
    const i32 gain_k = shape_gain_tweak(S->gains[lane & 3][0], gain_mult_Q16, shape_gain_add_q16(avgGain_Q16));
    for (int k = 0; k < NB_SUBFR; k++) avgGain_Q16 = shape_avg_gain_q16(avgGain_Q16, wshfl(gain_k, k), speech_activity_Q8);
    // ---- low-frequency shaping, tilt, harmonic shaping ----
    const i32 LF_shp_k = shape_lf_shp_q14(sigtype, c->pitchL[lane & 3], c->input_quality_bands_Q15[0]);
    const HarmTilt h = shape_harm_tilt(sigtype, speech_activity_Q8, s.input_quality_Q14, s.coding_quality_Q14, LTPCorr_Q15);
    i32 hb = st->HarmBoost_smth_Q16, hs = st->HarmShapeGain_smth_Q16, ti = st->Tilt_smth_Q16;
    i32 hb_k = 0, hs_k = 0, ti_k = 0;
    for (int k = 0; k < NB_SUBFR; k++) {
        const i32 hb_q = shape_smooth_q14(hb, h.HarmBoost_Q16), hs_q = shape_smooth_q14(hs, h.HarmShapeGain_Q16), ti_q = shape_smooth_q14(ti, h.Tilt_Q16);
        if (lane == k) { hb_k = hb_q; hs_k = hs_q; ti_k = ti_q; }
    }
    SB_SYNC();     // every lane has read what it needs from c / st
    if (lane < NB_SUBFR) {
        c->Gains_Q16[lane] = gain_k;
        c->LF_shp_Q14[lane] = LF_shp_k;
        c->HarmBoost_Q14[lane] = hb_k;
        c->HarmShapeGain_Q14[lane] = hs_k;
        c->Tilt_Q14[lane] = ti_k;
    }
    if (lane == 0) {
        c->current_SNR_dB_Q7 = st->SNR_dB_Q7;
        c->current_SNRPerMD_dB_Q7 = st->SNRPerMD_dB_Q7;
        c->input_quality_Q14 = s.input_quality_Q14;
        c->coding_quality_Q14 = s.coding_quality_Q14;
        c->sparseness_Q8 = s.sparseness_Q8;
        c->QuantOffsetType = s.QuantOffsetType;
        c->md_delta_gain_par = md_delta_gain_par;
        st->avgGain_Q16 = avgGain_Q16;
        st->HarmBoost_smth_Q16 = hb; st->HarmShapeGain_smth_Q16 = hs; st->Tilt_smth_Q16 = ti;
        S->par3[1] = shape_pregain_mult_q16(s.coding_quality_Q14);
    }
    SB_SYNC();
}

// ---------------------------------------------------------------------------------------------------------------------
// prediction analysis (SKP_Silk_find_pred_coefs_FIX.c:31-131 and what it calls)
// ---------------------------------------------------------------------------------------------------------------------
// Two Burg analyses side by side (SKP_Silk_burg_modified.c:49-228, QA = 25): lanes 0..15 analyse nb0 blocks starting at x0,
// lanes 16..31 nb1 blocks starting at x1 (find_LPC runs the whole frame and its second half; a caller with one analysis
// passes the same arguments twice).  Lane k of a half keeps row k of C_first_row / C_last_row / Af / CAf / CAb in registers;
// sums over the prediction order are 16-lane reductions (addition mod 2^32 is order-free), index reversals are shuffles.
// All lanes of a half return that half's results; A_Q16 (shared memory, [2][16], not inside B) receives the coefficients.
struct BurgScr {
    i32 cfr[2][NB_SUBFR][16];    // per block: first-row correlations before they are summed over the blocks
};
template <int D> SB_CFN void c_burg2(i32* res_nrg, i32* res_nrg_Q, i32 (*A_Q16)[16], BurgScr* B, const i16* x0, int nb0, const i16* x1, int nb1, int L,
                                    i32 WhiteNoiseFrac_Q32) {
    const int QA = 25, MAX_RSHIFTS = 32 - QA, MIN_RSHIFTS = -16, HEAD = 2;
    const int lane = SB_LANE, h = lane >> 4, k = lane & 15, base = h << 4;
    const i16* x = h ? x1 : x0;
    const int nb = h ? nb1 : nb0;
    // ---- C0 = energy with the reference's shift logic ----
    i32 C0, rshifts;
    {
        i64 part = 0;
        for (int i = k; i < nb * L; i += 16) part += (i64)((i32)x[i] * (i32)x[i]);
        const i64 total = gsum64<16>(part);
        i32 e = 0, sft = 0;
        if (total < ((i64)1 << 31)) {
            e = (i32)total;
            if (e & 0xC0000000) { e = (i32)((u32)e >> 2); sft = 2; }
        } else if (k == 0) {
            sum_sqr_shift(&e, &sft, x, nb * L, 0);
        }
        C0 = wshfl(e, base); rshifts = wshfl(sft, base);
    }
    if (rshifts > MAX_RSHIFTS) {
        C0 = shl(C0, rshifts - MAX_RSHIFTS);
        rshifts = MAX_RSHIFTS;
    } else {
        const int lz = clz32(C0) - 1;
        int extra = HEAD - lz;
        if (extra > 0) { extra = imin(extra, MAX_RSHIFTS - rshifts); C0 = C0 >> extra; }
        else { extra = imax(extra, MIN_RSHIFTS - rshifts); C0 = shl(C0, -extra); }
        rshifts += extra;
    }
    // ---- first-row correlations: tasks (block, lag) over the 16 lanes of the half ----
    for (int t = k; t < nb * D; t += 16) {
        const int s = t / D, n = t - s * D + 1;
        const i16* xp = x + s * L;
        i64 acc = 0;
        for (int i = 0; i < L - n; i++) acc += (i64)((i32)xp[i] * (i32)xp[i + n]);
        B->cfr[h][s][n - 1] = rshifts > 0 ? (i32)(acc >> rshifts) : shl((i32)acc, -rshifts);
    }
    SB_SYNC();
    i32 Cf = 0, Cl, Af = 0, CAf = 0, CAb = 0;
    if (k < D) for (int s = 0; s < nb; s++) Cf = addw(Cf, B->cfr[h][s][k]);
    Cl = Cf;
    if (k == 0) CAb = CAf = addw(addw(C0, smmul(WhiteNoiseFrac_Q32, C0)), 1);
    bool done = false;
    for (int n = 0; n < D; n++) {
        // (a) per block: prediction errors at both ends (4 lanes per block, 16-lane halves hold up to 4 blocks)
        const int sblk = k >> 2, j = k & 3;
        i32 t1 = 0, t2 = 0;
        for (int r = 0; 4 * r < n; r++) {           // n is uniform: every lane takes part in every exchange
            const int kk = j + 4 * r;
            const i32 At = wshfl(Af, base + (kk & 15));
            if (kk < n && sblk < nb) {
                const i16* xp = x + sblk * L;
                if (rshifts > -2) {
                    t1 = smlawb(t1, At, xp[n - kk - 1]);
                    t2 = smlawb(t2, At, xp[L - n + kk]);
                } else {
                    const i32 At1 = rshift_round(At, QA - 17);
                    t1 = mlaw(t1, xp[n - kk - 1], At1);
                    t2 = mlaw(t2, xp[L - n + kk], At1);
                }
            }
        }
        t1 = gsum<4>(t1); t2 = gsum<4>(t2);
        if (sblk < nb) {
            const i16* xp = x + sblk * L;
            if (rshifts > -2) {
                t1 = addw(t1, shl((i32)xp[n], QA - 16)); t2 = addw(t2, shl((i32)xp[L - n - 1], QA - 16));
                t1 = shl(negw(t1), 32 - QA - rshifts); t2 = shl(negw(t2), 32 - QA - rshifts);
            } else {
                t1 = addw(t1, shl((i32)xp[n], 17)); t2 = addw(t2, shl((i32)xp[L - n - 1], 17));
                t1 = negw(t1); t2 = negw(t2);
            }
        }
        // (b) rank-one updates of the four rows, lane k = column k, blocks in turn
        for (int s = 0; s < NB_SUBFR; s++) {
            const i32 e1 = wshfl(t1, base + 4 * s), e2 = wshfl(t2, base + 4 * s);
            if (s < nb && !done) {
                const i16* xp = x + s * L;
                if (rshifts > -2) {
                    const i32 x1 = negw(shl((i32)xp[n], 16 - rshifts)), x2 = negw(shl((i32)xp[L - n - 1], 16 - rshifts));
                    if (k < n) { Cf = smlawb(Cf, x1, xp[n - k - 1]); Cl = smlawb(Cl, x2, xp[L - n + k]); }
                    if (k <= n) { CAf = smlawb(CAf, e1, xp[n - k]); CAb = smlawb(CAb, e2, xp[L - n + k - 1]); }
                } else {
                    const i32 x1 = negw(shl((i32)xp[n], -rshifts)), x2 = negw(shl((i32)xp[L - n - 1], -rshifts));
                    if (k < n) { Cf = mlaw(Cf, x1, xp[n - k - 1]); Cl = mlaw(Cl, x2, xp[L - n + k]); }
                    if (k <= n) { CAf = smlaww(CAf, e1, shl((i32)xp[n - k], -rshifts - 1)); CAb = smlaww(CAb, e2, shl((i32)xp[L - n + k - 1], -rshifts - 1)); }
                }
            }
        }
        // (c) reflection coefficient
        i32 tmp1 = wshfl(Cf, base + n), tmp2 = wshfl(Cl, base + n);
        {
            const i32 a = wshfl(Cl, base + ((n - k - 1) & 15)), b = wshfl(Cf, base + ((n - k - 1) & 15));
            const i32 cb = wshfl(CAb, base + ((n - k) & 15)), s1 = wshfl(CAb, base + ((k + 1) & 15)), s2 = wshfl(CAf, base + ((k + 1) & 15));
            i32 T1 = 0, T2 = 0, T3 = 0, T4 = 0;
            if (k < n) {
                int lz = clz32(iabs(Af)) - 1;
                lz = imin(32 - QA, lz);
                const i32 At1 = shl(Af, lz);
                const int sh = 32 - QA - lz;
                T1 = shl(smmul(a, At1), sh); T2 = shl(smmul(b, At1), sh);
                T3 = shl(smmul(cb, At1), sh); T4 = shl(smmul(addw(s1, s2), At1), sh);
            }
            tmp1 = addw(tmp1, gsum<16>(T1)); tmp2 = addw(tmp2, gsum<16>(T2));
            const i32 num0 = gsum<16>(T3);
            const i32 nrg = addw(addw(wshfl(CAb, base), wshfl(CAf, base)), gsum<16>(T4));
            i32 num = shl(negw(addw(num0, tmp2)), 1);
            const bool ok = iabs(num) < nrg;
            const i32 rc_Q31 = (ok && !done) ? div32_varq(num, nrg, 31) : 0;
            if (!done) {
                if (k == n + 1) { CAf = tmp1; CAb = tmp2; }
                if (!ok) { if (k >= n) Af = 0; done = true; }
            }
            // (d), (e): order update of the predictor and of the two correlation rows (old values on the right-hand side)
            const i32 tA = wshfl(Af, base + ((n - k - 1) & 15));
            const i32 ob = wshfl(CAb, base + ((n + 1 - k) & 15)), of = wshfl(CAf, base + ((n + 1 - k) & 15));
            if (!done) {
                if (k < n) Af = addw(Af, shl(smmul(tA, rc_Q31), 1));
                if (k == n) Af = rc_Q31 >> (31 - QA);
                if (k <= n + 1) {
                    const i32 cf_old = CAf, cb_old = CAb;
                    CAf = addw(cf_old, shl(smmul(ob, rc_Q31), 1));
                    CAb = addw(cb_old, shl(smmul(of, rc_Q31), 1));
                }
            }
        }
    }
    // ---- result ----
    const i32 At1 = k < D ? rshift_round(Af, QA - 16) : 0;
    const i32 caf_next = wshfl(CAf, base + ((k + 1) & 15));
    const i32 nrg = addw(wshfl(CAf, base), gsum<16>(k < D ? smulww(caf_next, At1) : 0));
    const i32 tt = addw(1 << 16, gsum<16>(k < D ? smulww(At1, At1) : 0));
    if (k < D) A_Q16[h][k] = negw(At1);
    *res_nrg = smlaww(nrg, smmul(WhiteNoiseFrac_Q32, C0), negw(tt));
    *res_nrg_Q = -rshifts;
}

// SKP_Silk_A2NLSF (A2NLSF.c:46-287).  The reference walks a 128-interval cosine grid and alternates between the two
// symmetric polynomials; here both polynomials are evaluated on the whole grid (lanes over grid points), sign changes are
// collected as bit masks, the walk becomes a scan for the next set bit, and the d bisections run on d lanes.
// a_Q16: shared memory (modified when the root search has to widen the bandwidth); NLSF: shared memory.
struct A2nlsfScr { i32 y[2][132]; i32 k_of[16]; i32 ylo_of[16]; };
template <int D> SB_CFN void c_a2nlsf(i32* NLSF, i32* a_Q16, A2nlsfScr* Z) {
    enum { DD = D / 2, BIN = 3, TABSZ = 128, MAX_ITER = 30 };
    const int lane = SB_LANE;
    const i32* cosv = SB_T(lsf_cos_q12);
    for (int iter = 0;; iter++) {
        i32 PQ[2][DD + 1];
        {
            i32 a[D];
#pragma unroll
            for (int i = 0; i < D; i++) a[i] = a_Q16[i];
            PQ[0][DD] = 1 << 16; PQ[1][DD] = 1 << 16;
#pragma unroll
            for (int k = 0; k < DD; k++) {
                PQ[0][k] = subw(negw(a[DD - k - 1]), a[DD + k]);
                PQ[1][k] = addw(negw(a[DD - k - 1]), a[DD + k]);
            }
#pragma unroll
            for (int k = DD; k > 0; k--) { PQ[0][k - 1] = subw(PQ[0][k - 1], PQ[0][k]); PQ[1][k - 1] = addw(PQ[1][k - 1], PQ[1][k]); }
#pragma unroll
            for (int q = 0; q < 2; q++) {
#pragma unroll
                for (int k = 2; k <= DD; k++) {
#pragma unroll
                    for (int n = DD; n > k; n--) PQ[q][n - 2] = subw(PQ[q][n - 2], PQ[q][n]);
                    PQ[q][k - 2] = subw(PQ[q][k - 2], shl(PQ[q][k], 1));
                }
            }
        }
        SB_SYNC();
        // both polynomials on the grid
        for (int g = lane; g <= TABSZ; g += 32) {
            const i32 x_Q16 = shl(cosv[g], 4);
#pragma unroll
            for (int q = 0; q < 2; q++) {
                i32 y32 = PQ[q][DD];
#pragma unroll
                for (int n = DD - 1; n >= 0; n--) y32 = smlaww(PQ[q][n], y32, x_Q16);
                Z->y[q][g] = y32;
            }
        }
        SB_SYNC();
        // sign changes between neighbouring grid points: bit g of word w <-> interval ending at grid point 32 w + g
        u32 sc[2][5];
#pragma unroll
        for (int w = 0; w < 5; w++) {
            const int g = 32 * w + lane;
#pragma unroll
            for (int q = 0; q < 2; q++) {
                bool on = false;
                if (g >= 1 && g <= TABSZ) { const i32 lo = Z->y[q][g - 1], hi = Z->y[q][g]; on = (lo <= 0 && hi >= 0) || (lo >= 0 && hi <= 0); }
                sc[q][w] = wballot(on);
            }
        }
        // the walk (every lane, identical)
        int root_ix = 0, q = 0, k = 1;
        bool forced = false; i32 fy = 0;
        if (Z->y[0][0] < 0) { root_ix = 1; q = 1; }
        bool fail = false;
        while (root_ix < D) {
            int kk = -1;
            if (forced) {
                const i32 hi = Z->y[q][k];
                if ((fy <= 0 && hi >= 0) || (fy >= 0 && hi <= 0)) kk = k;
            }
            int from = forced ? k + 1 : k;
            bool was_forced = forced && kk == k;
            if (kk < 0) {
                for (int w = from >> 5; w < 5 && kk < 0; w++) {
                    u32 m = sc[q][w];
                    if (w == (from >> 5)) m &= ~0u << (from & 31);
                    if (m) kk = 32 * w + ctz32(m);
                }
            }
            if (kk < 0 || kk > TABSZ) { fail = true; break; }
            if (lane == root_ix) { Z->k_of[root_ix] = kk; Z->ylo_of[root_ix] = was_forced ? fy : Z->y[q][kk - 1]; }
            root_ix++;
            q = root_ix & 1;
            k = kk;
            forced = true;
            fy = shl(1 - (root_ix & 2), 12);
        }
        if (!fail) {
            SB_SYNC();
            const int first = Z->y[0][0] < 0 ? 1 : 0;
            if (lane == 0 && first) NLSF[0] = 0;
            if (lane >= first && lane < D) {
                const int r = lane, qq = r & 1, kk = Z->k_of[r];
                i32 xlo = cosv[kk - 1], xhi = cosv[kk], ylo = Z->ylo_of[r], yhi = Z->y[qq][kk];
                i32 ffrac = -256;
                for (int m = 0; m < BIN; m++) {
                    const i32 xmid = rshift_round(xlo + xhi, 1);
                    const i32 x_Q16 = shl(xmid, 4);
                    i32 ymid = qq ? PQ[1][DD] : PQ[0][DD];
#pragma unroll
                    for (int n = DD - 1; n >= 0; n--) ymid = smlaww(qq ? PQ[1][n] : PQ[0][n], ymid, x_Q16);
                    if ((ylo <= 0 && ymid >= 0) || (ylo >= 0 && ymid <= 0)) { xhi = xmid; yhi = ymid; }
                    else { xlo = xmid; ylo = ymid; ffrac = ffrac + (128 >> m); }
                }
                if (iabs(ylo) < 65536) {
                    const i32 den = subw(ylo, yhi);
                    const i32 nom = addw(shl(ylo, 8 - BIN), den >> 1);
                    if (den != 0) ffrac += nom / den;
                } else {
                    ffrac += ylo / (subw(ylo, yhi) >> (8 - BIN));
                }
                NLSF[r] = imin(shl(kk, 8) + ffrac, 32767);
            }
            SB_SYNC();
            return;
        }
        // no root left on the grid: widen the bandwidth and start over (A2NLSF.c:251-283)
        const int i = iter + 1;
        if (i > MAX_ITER) {
            SB_SYNC();
            const i32 n0 = (1 << 15) / (D + 1);
            if (lane < D) NLSF[lane] = lane == 0 ? n0 : smulbb(lane + 1, n0);
            SB_SYNC();
            return;
        }
        const i32 f = c_bwexpander32_factor(D, 65536 - smulbb(10 + i, i));
        SB_SYNC();
        if (lane < D) a_Q16[lane] = smulww(a_Q16[lane], f);
        SB_SYNC();
    }
}

struct PredScr {
    alignas(4) i16 LPC_in_pre[NB_SUBFR * LPC_ORDER + FRAME];
    i32 WLTP[NB_SUBFR * LTP_ORDER * LTP_ORDER];
    LtpSubfr ltp[NB_SUBFR];
    i32 invGains_Q16[NB_SUBFR], local_gains[NB_SUBFR], Wght_Q15[NB_SUBFR];
    i32 NLSF_Q15[LPC_ORDER + 2];
    i32 NLSFW_Q6[LPC_ORDER + 2];
    i32 A_Q16[2][16];            // Burg results: whole frame, second half
    i32 flag_interp;             // this frame searches the NLSF interpolation factor
    i32 ie[8][2];                // residual energy and shift of (candidate, half-frame)
    i32 vq_meta[5];              // MSVQ: survivor set, survivors, fluctuation reduction off, its weight, signal type
    i32 vq_wsse[16];
    i32 nlsf_out[2][LPC_ORDER];  // quantised NLSFs of the two half-frames, for the gain kernel
    i16 a_tmp_Q12[4][LPC_ORDER + 2];
    union {
        struct { BurgScr burg; A2nlsfScr a2n; } lpc;
        i16 LPC_res[4][2 * (SUBFR + LPC_ORDER)];
        struct {
            i32 res[2][16 * LPC_ORDER];
            i32 rate[2][16];
            u32 path_lo[2][16]; u16 path_hi[2][16];
            i32 cand_v[64]; i16 cand_e[64];
            i32 best_v[16]; i16 best_e[16];
            i32 nlsf_s[16][LPC_ORDER + 1];
        } vq;
    } u;
};

// SKP_Silk_quant_LTP_gains_FIX (quant_LTP_gains_FIX.c:30-103): 8 lanes per sub-frame walk each codebook
SB_CFN void c_quant_ltp_gains(i16* B_Q14, i32* cbk_index, i32* periodicity_index, const i32* W_Q18, i32 mu_Q8) {
    const int lane = SB_LANE, j = lane >> 3, g = lane & 7;
    i32 best_rd = SB_I32_MAX, best_k = 0, best_idx = 0;
    const i16* in = B_Q14 + j * LTP_ORDER;
    const i32* W = W_Q18 + j * LTP_ORDER * LTP_ORDER;
    for (int k = 0; k < 3; k++) {
        const i16* cl = k == 0 ? SB_T(ltp_bits0_q6) : (k == 1 ? SB_T(ltp_bits1_q6) : SB_T(ltp_bits2_q6));
        const i16* cbk = k == 0 ? SB_T(ltp_vq0_q14) : (k == 1 ? SB_T(ltp_vq1_q14) : SB_T(ltp_vq2_q14));
        const int size = SB_T(ltp_vq_sizes)[k];
        i32 rd = SB_I32_MAX, idx = 0;
        for (int e = g; e < size; e += 8) {
            const i32 v = vq_wmat_ec_entry(in, W, cbk + e * LTP_ORDER, cl[e], mu_Q8);
            if (v < rd) { rd = v; idx = e; }
        }
        gargmin<8>(rd, idx);                 // first of equal minima
        i32 rate_dist = 0;
        for (int jj = 0; jj < NB_SUBFR; jj++) rate_dist = add_pos_sat32(rate_dist, wshfl(rd, 8 * jj));
        rate_dist = imin(SB_I32_MAX - 1, rate_dist);
        if (rate_dist < best_rd) { best_rd = rate_dist; best_k = k; best_idx = idx; }
    }
    SB_SYNC();
    const i16* cbk = best_k == 0 ? SB_T(ltp_vq0_q14) : (best_k == 1 ? SB_T(ltp_vq1_q14) : SB_T(ltp_vq2_q14));
    if (g < LTP_ORDER) B_Q14[j * LTP_ORDER + g] = cbk[best_idx * LTP_ORDER + g];
    if (g == 0) cbk_index[j] = best_idx;
    if (lane == 0) *periodicity_index = best_k;
    SB_SYNC();
}

// SKP_Silk_find_LPC_FIX (find_LPC_FIX.c:32-148), order 10, four blocks of 50 samples in x
SB_CFN void c_find_lpc(i32* NLSF_Q15, i32* interpIndex, const i32* prev_NLSFq_Q15, int useInterp, PredScr* Q) {
    enum { ORD = LPC_ORDER, SL = SUBFR + LPC_ORDER };
    const int lane = SB_LANE, h = lane >> 4;
    const i16* x = Q->LPC_in_pre;
    BurgScr* B = &Q->u.lpc.burg;
    i32 rn, rq;
    c_burg2<ORD>(&rn, &rq, Q->A_Q16, B, x, NB_SUBFR, useInterp ? x + (NB_SUBFR >> 1) * SL : x, useInterp ? (NB_SUBFR >> 1) : NB_SUBFR, SL, SB_FIXC(2.5e-5f, 32));
    SB_SYNC();
    {   // bwexpander_32(a, 10, 0.99995) on both results (coefficient index = lane inside each half)
        const int k = lane & 15;
        i32 t = SB_FIXC(0.99995f, 16), mine = t;
        for (int i = 0; i < ORD - 1; i++) { if (k == i) mine = t; t = smulww(SB_FIXC(0.99995f, 16), t); }
        if (k >= ORD - 1) mine = t;
        if (k < ORD) Q->A_Q16[h][k] = smulww(Q->A_Q16[h][k], mine);
    }
    i32 res_nrg = wshfl(rn, 0), res_nrg_Q = wshfl(rq, 0);
    const i32 res_tmp_nrg = wshfl(rn, 16), res_tmp_nrg_Q = wshfl(rq, 16);
    SB_SYNC();
    int interp = 4;
    const bool interpOn = useInterp == 1;      // per stream: the instance sections below are entered by every warp of the block
    if (lane == 0) Q->flag_interp = interpOn ? 1 : 0;
    if (interpOn) {
        lpc_first_half_nrg(res_nrg, res_nrg_Q, res_tmp_nrg, res_tmp_nrg_Q);
        c_a2nlsf<ORD>(NLSF_Q15, Q->A_Q16[1], &Q->u.lpc.a2n);
    }
    // the four interpolation candidates: NLSF -> LPC as four scalar instances, analysis filters over all lanes
    c_instances<4>([&](int d, int k) {
        PredScr* Qj = xoff(Q, d);
        if (!Qj->flag_interp) return;
        const i32* nlj = xoff(NLSF_Q15, d);
        const i32* pvj = xoff(prev_NLSFq_Q15, d);
        i32 NLSF0[ORD], nl[ORD], prevv[ORD];
        for (int i = 0; i < ORD; i++) { nl[i] = nlj[i]; prevv[i] = pvj[i]; }
        interpolate(NLSF0, prevv, nl, k, ORD);
        i16 a12[ORD];
        nlsf2a_stable(a12, NLSF0, ORD);
        for (int i = 0; i < ORD; i++) Qj->a_tmp_Q12[k][i] = a12[i];
    });
    if (interpOn) {     // (the grid scratch of c_a2nlsf, same union as LPC_res, is dead from here on)
        for (int t = lane; t < 4 * 2 * SL; t += 32) {
            const int cand = t / (2 * SL), kx = t - cand * 2 * SL;
            const i16* bq = Q->a_tmp_Q12[cand];
            i32 acc = 0;
#pragma unroll
            for (int d = 0; d < ORD; d++) if (d < kx) acc = addw(acc, (i32)x[kx - 1 - d] * (i32)bq[d]);
            const i32 xi = x[kx];
            Q->u.LPC_res[cand][kx] = (i16)sat16(rshift_round(sub_sat32(shl(xi, 12), acc), 12));
        }
    }
    c_instances<8>([&](int d, int k) {     // (candidate, half) residual energies
        PredScr* Qj = xoff(Q, d);
        if (!Qj->flag_interp) return;
        const int cand = k >> 1, half = k & 1;
        i32 e, sft;
        sum_sqr_shift(&e, &sft, Qj->u.LPC_res[cand] + ORD + half * SL, SL - ORD, (ORD + half * SL) & 1);
        Qj->ie[k][0] = e; Qj->ie[k][1] = sft;
    });
    if (interpOn) {
        for (int kq = 3; kq >= 0; kq--)
            if (lpc_interp_lower(res_nrg, res_nrg_Q, Q->ie[2 * kq][0], Q->ie[2 * kq][1], Q->ie[2 * kq + 1][0], Q->ie[2 * kq + 1][1])) interp = kq;
        SB_SYNC();
    }
    if (interp == 4) c_a2nlsf<ORD>(NLSF_Q15, Q->A_Q16[0], &Q->u.lpc.a2n);
    if (lane == 0) *interpIndex = interp;
    SB_SYNC();
}

// SKP_Silk_NLSF_MSVQ_encode_FIX (NLSF_MSVQ_encode_FIX.c:33-239), order 10, 6 stages, 16 survivors.
// Stage: lanes over (survivor, code vector) pairs; the 16 best pairs by (value, scan position) -- what the reference's stable
// partial insertion sort returns -- are found by bounding the 16th value with the lanes' own minima, compacting the pairs
// below the bound in scan order and ranking that short list.
SB_CFN void c_nlsf_msvq_encode(i32* NLSFIndices, i32* pNLSF_Q15, const NlsfCb& cb, const i32* pNLSF_q_Q15_prev, const i32* pW_Q6,
                              i32 NLSF_mu_Q15, i32 NLSF_mu_fluc_red_Q16, int deactivate_fluc_red, int sigtype, PredScr* Q) {
    enum { SURV = 16, NST = 6, ORD = LPC_ORDER, MAXC = 8 };
    const int lane = SB_LANE;
    auto& V = Q->u.vq;
    i32 wq[ORD];
#pragma unroll
    for (int m = 0; m < ORD; m++) wq[m] = pW_Q6[m];
    int cur = 0, nxt = 1;
    if (lane < ORD) V.res[0][lane] = pNLSF_Q15[lane];
    if (lane < SURV) { V.rate[0][lane] = 0; V.path_lo[0][lane] = 0; V.path_hi[0][lane] = 0; }
    SB_SYNC();
    int prev_survivors = 1, cur_survivors = 0, cb_off = 0;
    const int min_survivors = SURV / 2;
    for (int s = 0; s < NST; s++) {
        const int nVec = cb.nvec[s];
        const i16* CB = cb.cb_q15 + cb_off * ORD;
        const i16* Rates = cb.rates_q5 + cb_off;
        const int ncand = prev_survivors * nVec;
        const int lg = 31 - clz32(nVec);
        cur_survivors = imin(SURV, ncand);
        // values of my pairs e = lane, lane + 32, ...
        i32 val[MAXC];
        i32 mymin = SB_I32_MAX;
#pragma unroll
        for (int r = 0; r < MAXC; r++) {
            const int e = lane + 32 * r;
            val[r] = SB_I32_MAX;
            if (e < ncand) {
                const int n = e >> lg, i = e & (nVec - 1);      // nVec is a power of two in both codebooks
                const i32* in = &V.res[cur][n * ORD];
                const i16* v = CB + i * ORD;
                i32 sum_error = 0;
#pragma unroll
                for (int m = 0; m < ORD; m++) { const i32 diff = in[m] - (i32)v[m]; sum_error = smlawb(sum_error, smulbb(diff, diff), wq[m]); }
                val[r] = smlabb(sum_error, V.rate[cur][n] + Rates[i], NLSF_mu_Q15);
                mymin = imin(mymin, val[r]);
            }
        }
        // upper bound U for the SURV-th smallest value: the SURV-th smallest of the lanes' minima (>= SURV pairs are <= U)
        i32 U;
        {
            int rank = 0;
            for (int l = 0; l < 32; l++) { const i32 o = wshfl(mymin, l); rank += (o < mymin) || (o == mymin && l < lane); }
            U = wshfl(mymin, ctz32(wballot(rank == SURV - 1)));
        }
        // compact the pairs with value <= U in scan order (e ascending)
        int M = 0;
#pragma unroll
        for (int r = 0; r < MAXC; r++) {
            if (32 * r >= ncand) break;       // uniform
            const bool on = (lane + 32 * r) < ncand && val[r] <= U;
            const u32 m = wballot(on);
            if (on) { const int q = M + popc32(m & ((1u << lane) - 1)); if (q < 64) { V.cand_v[q] = val[r]; V.cand_e[q] = (i16)(lane + 32 * r); } }
            M += popc32(m);
        }
        SB_SYNC();
        if (M > 64) {
            // more than 64 pairs share the bound (long runs of equal values): lane 0 replays the reference's sort over everything
            // it needs the values again; rare enough to recompute them one by one
            if (lane == 0) {
                i32 kv[SURV]; int ke[SURV]; int filled = 0;
                for (int e = 0; e < ncand; e++) {
                    const int n = e / nVec, i = e - n * nVec;
                    const i32* in = &V.res[cur][n * ORD];
                    const i16* v = CB + i * ORD;
                    i32 sum_error = 0;
                    for (int m = 0; m < ORD; m++) { const i32 diff = in[m] - (i32)v[m]; sum_error = smlawb(sum_error, smulbb(diff, diff), wq[m]); }
                    const i32 vv = smlabb(sum_error, V.rate[cur][n] + Rates[i], NLSF_mu_Q15);
                    if (filled < cur_survivors) {
                        int jx = filled - 1;
                        for (; jx >= 0 && vv < kv[jx]; jx--) { kv[jx + 1] = kv[jx]; ke[jx + 1] = ke[jx]; }
                        kv[jx + 1] = vv; ke[jx + 1] = e; filled++;
                    } else if (vv < kv[SURV - 1]) {
                        int jx = SURV - 2;
                        for (; jx >= 0 && vv < kv[jx]; jx--) { kv[jx + 1] = kv[jx]; ke[jx + 1] = ke[jx]; }
                        kv[jx + 1] = vv; ke[jx + 1] = e;
                    }
                }
                for (int q = 0; q < cur_survivors; q++) { V.best_v[q] = kv[q]; V.best_e[q] = (i16)ke[q]; }
            }
        } else {
            // rank inside the short list: #{(v', q') < (v, q)}
            for (int q = lane; q < M; q += 32) {
                const i32 v = V.cand_v[q];
                int rank = 0;
                for (int o = 0; o < M; o++) { const i32 ov = V.cand_v[o]; rank += (ov < v) || (ov == v && o < q); }
                if (rank < SURV) { V.best_v[rank] = v; V.best_e[rank] = V.cand_e[q]; }
            }
        }
        SB_SYNC();
        const i32 best0 = V.best_v[0];
        if (best0 < SB_I32_MAX / SURV) {
            const i32 thr = smlawb(best0, mulw(SURV, best0), SB_FIXC(0.1f, 16));
            while (V.best_v[cur_survivors - 1] > thr && cur_survivors > min_survivors) cur_survivors--;
        }
        // survivors of this stage: residuals, rates, paths
        for (int t = lane; t < cur_survivors * ORD; t += 32) {
            const int kx = t / ORD, m = t - kx * ORD;
            const int e = V.best_e[kx];
            const int input_index = s > 0 ? e >> lg : 0, cb_index = s > 0 ? e & (nVec - 1) : e;
            V.res[nxt][kx * ORD + m] = V.res[cur][input_index * ORD + m] - (i32)CB[cb_index * ORD + m];
        }
        if (lane < cur_survivors) {
            const int e = V.best_e[lane];
            const int input_index = s > 0 ? e >> lg : 0, cb_index = s > 0 ? e & (nVec - 1) : e;
            V.rate[nxt][lane] = V.rate[cur][input_index] + Rates[cb_index];
            u64 pth = ((u64)V.path_hi[cur][input_index] << 32) | V.path_lo[cur][input_index];
            pth |= (u64)(u32)cb_index << (8 * s);
            V.path_lo[nxt][lane] = (u32)pth; V.path_hi[nxt][lane] = (u16)(pth >> 32);
        }
        SB_SYNC();
        cur ^= 1; nxt ^= 1;
        prev_survivors = cur_survivors;
        cb_off += nVec;
    }
    // survivors now in [cur]; V.best_v holds their rate-distortion values in order
    // fluctuation reduction: decode every survivor (one scalar instance each) and weigh its distance to the previous frame
    if (lane == 0) { Q->vq_meta[0] = cur; Q->vq_meta[1] = cur_survivors; Q->vq_meta[2] = deactivate_fluc_red; Q->vq_meta[3] = NLSF_mu_fluc_red_Q16; Q->vq_meta[4] = sigtype; }
    c_instances<SURV>([&](int d, int k) {
        PredScr* Qj = xoff(Q, d);
        if (Qj->vq_meta[2] == 1) return;
        i32 wsse = SB_I32_MAX;
        if (k < Qj->vq_meta[1]) {
            auto& Vj = Qj->u.vq;
            const int cj = Qj->vq_meta[0];
            const NlsfCb cbj = nlsf_cb(Qj->vq_meta[4]);
            const i32* prevj = xoff(pNLSF_q_Q15_prev, d);
            const u64 pth = ((u64)Vj.path_hi[cj][k] << 32) | Vj.path_lo[cj][k];
            i32 idx[NST];
#pragma unroll
            for (int i = 0; i < NST; i++) idx[i] = (i32)((pth >> (8 * i)) & 0xff);
            i32* nl = Vj.nlsf_s[k];
            nlsf_msvq_decode(nl, cbj, idx);
            i32 wsse_Q20 = 0;
            for (int i = 0; i < ORD; i++) {
                const i32 se = nl[i] - prevj[i];
                wsse_Q20 = smlawb(wsse_Q20, smulbb(se, se), Qj->NLSFW_Q6[i]);
            }
            wsse = add_pos_sat32(Vj.best_v[k], smulwb(wsse_Q20, Qj->vq_meta[3]));
        }
        Qj->vq_wsse[k] = wsse;
    });
    i32 bestIndex = 0;
    if (deactivate_fluc_red != 1) {      // per stream
        i32 wsse = lane < SURV ? Q->vq_wsse[lane] : SB_I32_MAX;
        i32 who = lane;
        wargmin(wsse, who);       // first of equal minima; a value equal to INT_MAX never wins in the reference either
        bestIndex = wsse < SB_I32_MAX ? who : 0;
    }
    SB_SYNC();
    const u64 pth = ((u64)V.path_hi[cur][bestIndex] << 32) | V.path_lo[cur][bestIndex];
    if (lane < NST) NLSFIndices[lane] = (i32)((pth >> (8 * lane)) & 0xff);
    c_instances<1>([&](int d, int) {
        PredScr* Qj = xoff(Q, d);
        const i32* ixj = xoff(NLSFIndices, d);
        i32* outj = xoff(pNLSF_Q15, d);
        i32 idx[NST], nl[ORD];
        for (int i = 0; i < NST; i++) idx[i] = ixj[i];
        nlsf_msvq_decode(nl, nlsf_cb(Qj->vq_meta[4]), idx);
        for (int i = 0; i < ORD; i++) outj[i] = nl[i];
    });
}

// SKP_Silk_process_NLSFs_FIX (process_NLSFs_FIX.c:31-127)
SB_CFN void c_process_nlsfs(EncSilk* st, EncCtrl* c, i32* pNLSF_Q15, PredScr* Q, const NlsfFastTabs* fast) {
    const int lane = SB_LANE;
    const int sigtype = c->sigtype, interpQ2 = c->NLSFInterpCoef_Q2;
    i32 NLSF_mu_Q15, NLSF_mu_fluc_red_Q16;
    nlsf_mu(NLSF_mu_Q15, NLSF_mu_fluc_red_Q16, sigtype, st->speech_activity_Q8, c->sparseness_Q8);
    const int doInterpolate = interpQ2 < (1 << 2);
    // Laroia weights: one scalar instance for the target vector, one for the interpolated one (eleven divisions each)
    c_instances<2>([&](int d, int k) {
        PredScr* Qj = xoff(Q, d);
        const i32* nlj = xoff(pNLSF_Q15, d);
        i32 nl[LPC_ORDER], w[LPC_ORDER];
        if (k == 0) { for (int i = 0; i < LPC_ORDER; i++) nl[i] = nlj[i]; }
        else {
            const EncSilk* sj = xoff(st, d);
            i32 a[LPC_ORDER], b[LPC_ORDER];
            for (int i = 0; i < LPC_ORDER; i++) { a[i] = sj->prev_NLSFq_Q15[i]; b[i] = nlj[i]; }
            interpolate(nl, a, b, xoff(c, d)->NLSFInterpCoef_Q2, LPC_ORDER);
        }
        nlsf_vq_weights_laroia(w, nl, LPC_ORDER);
        for (int i = 0; i < LPC_ORDER; i++) Qj->u.vq.nlsf_s[k][i] = w[i];
    });
    if (lane < LPC_ORDER) {
        const i32 w = Q->u.vq.nlsf_s[0][lane];
        Q->NLSFW_Q6[lane] = doInterpolate ? nlsf_interp_weight_q6(w, Q->u.vq.nlsf_s[1][lane], interpQ2) : w;
    }
    SB_SYNC();
    NlsfCb cb = nlsf_cb(sigtype);
    if (fast) {
        cb.cb_q15 = sigtype == 0 ? fast->cb0 : fast->cb1;
        cb.rates_q5 = sigtype == 0 ? fast->rates0 : fast->rates1;
    }
    c_nlsf_msvq_encode(c->NLSFIndices, pNLSF_Q15, cb, st->prev_NLSFq_Q15, Q->NLSFW_Q6, NLSF_mu_Q15, NLSF_mu_fluc_red_Q16,
                       st->first_frame_after_reset, sigtype, Q);
    // quantised NLSFs of the two half-frames (first half interpolated); the gain kernel turns them into prediction filters
    if (lane < LPC_ORDER) {
        const i32 q = pNLSF_Q15[lane];
        Q->nlsf_out[1][lane] = q;
        Q->nlsf_out[0][lane] = nlsf_first_half_q15(st->prev_NLSFq_Q15[lane], q, interpQ2);
    }
    SB_SYNC();
}

// SKP_Silk_find_pred_coefs_FIX (find_pred_coefs_FIX.c:31-131)
SB_CFN void c_find_pred_coefs(EncSilk* st, EncCtrl* c, PredScr* Q, const i16* res_pitch, int frame_in_packet, const NlsfFastTabs* fast) {
    const int lane = SB_LANE;
    const int sigtype = c->sigtype;
    {   // (find_pred_coefs states this step too: as a shared helper it grows this kernel's spill traffic)
        const i32 g = c->Gains_Q16[lane & 3];
        i32 min_gain_Q16 = SB_I32_MAX >> 6;
        for (int i = 0; i < NB_SUBFR; i++) min_gain_Q16 = imin(min_gain_Q16, c->Gains_Q16[i]);
        if (lane < NB_SUBFR) {
            i32 inv = div32_varq(min_gain_Q16, g, 16 - 2);
            inv = imax(inv, 363);
            Q->invGains_Q16[lane] = inv;
            Q->Wght_Q15[lane] = smulwb(inv, inv) >> 1;
            Q->local_gains[lane] = (1 << 16) / inv;
        }
    }
    SB_SYNC();
    const i16* xb = st->x_buf + FRAME - LPC_ORDER;
    // LTP analysis of the voiced streams: the four sub-frames as four scalar instances, then the part that couples them
    c_instances<NB_SUBFR>([&](int d, int k) {
        EncCtrl* cj = xoff(c, d);
        if (cj->sigtype != 0) return;
        PredScr* Qj = xoff(Q, d);
        const i16* rp = xoff(res_pitch, d);
        find_ltp_subfr(k, cj->LTPCoef_Q14 + k * LTP_ORDER, Qj->WLTP + k * LTP_ORDER * LTP_ORDER, &Qj->ltp[k], rp, rp + (FRAME >> 1),
                       cj->pitchL[k], Qj->Wght_Q15[k]);
    });
    c_instances<1>([&](int d, int) {
        EncCtrl* cj = xoff(c, d);
        if (cj->sigtype != 0) return;
        PredScr* Qj = xoff(Q, d);
        find_ltp_tail(cj->LTPCoef_Q14, &cj->LTPredCodGain_Q7, Qj->ltp, Qj->Wght_Q15);
        ltp_scale_ctrl(xoff(st, d), cj, frame_in_packet);      // independent of the gain quantisation below
    });
    if (sigtype == 0) {       // per stream
        c_quant_ltp_gains(c->LTPCoef_Q14, c->LTPIndex, &c->PERIndex, Q->WLTP, SB_FIXC(0.03f, 8));
        // SKP_Silk_LTP_analysis_filter_FIX (LTP_analysis_filter_FIX.c:30-80): lanes over outputs
        for (int t = lane; t < NB_SUBFR * (SUBFR + LPC_ORDER); t += 32) {
            const int k = t / (SUBFR + LPC_ORDER), i = t - k * (SUBFR + LPC_ORDER);
            Q->LPC_in_pre[t] = ltp_analysis_sample(xb, c->LTPCoef_Q14, c->pitchL, Q->invGains_Q16, k, i);
        }
    } else {
        for (int t = lane; t < NB_SUBFR * (SUBFR + LPC_ORDER); t += 32) {
            const int k = t / (SUBFR + LPC_ORDER), i = t - k * (SUBFR + LPC_ORDER);
            Q->LPC_in_pre[t] = (i16)smulwb(Q->invGains_Q16[k], (xb + k * SUBFR)[i]);
        }
        if (lane < NB_SUBFR * LTP_ORDER) c->LTPCoef_Q14[lane] = 0;
        if (lane == 0) c->LTPredCodGain_Q7 = 0;
    }
    SB_SYNC();
    SB_PHASE();
    c_find_lpc(Q->NLSF_Q15, &c->NLSFInterpCoef_Q2, st->prev_NLSFq_Q15, 1 * (1 - st->first_frame_after_reset), Q);
    SB_PHASE();
    c_process_nlsfs(st, c, Q->NLSF_Q15, Q, fast);
    SB_PHASE();
    // (prediction filters, residual energies and the gain processing follow in the gain kernel)
    if (lane < LPC_ORDER) st->prev_NLSFq_Q15[lane] = Q->NLSF_Q15[lane];
    SB_SYNC();
}

// ---------------------------------------------------------------------------------------------------------------------
// high band (AGR_BWE_encode_frame_FIX.c:8-82 first half, AGR_BWE_find_HB_LPC_FIX.c:4-49, AGR_BWE_quant_highband.c:23-104)
// ---------------------------------------------------------------------------------------------------------------------
struct HbScr {
    alignas(4) i16 LPC_in_pre[4 * (80 + HB_ORDER)];
    i32 A_Q16[2][16];
    i32 NLSF_Q15[HB_ORDER + 2];
    i32 weight[HB_ORDER];
    i16 coef[HB_ORDER];
    union { BurgScr burg; A2nlsfScr a2n; } u;
};
// AGR_Sate_lsp_quant_highband (AGR_BWE_quant_highband.c:23-104) on H->NLSF_Q15: Laroia weights into H->weight, 256-entry
// first stage over the lanes, 16-entry weighted second stage; the quantised vector replaces H->NLSF_Q15, lane 0 stores the
// index.  The caller synchronises the warp before it reads the results.
SB_CFN void c_hb_lsp_quant(HbScr* H, i32* lsp_idx_out) {
    const int lane = SB_LANE;
    if (lane == 0) { i32 w[HB_ORDER], nl[HB_ORDER]; for (int i = 0; i < HB_ORDER; i++) nl[i] = H->NLSF_Q15[i]; nlsf_vq_weights_laroia(w, nl, HB_ORDER); for (int i = 0; i < HB_ORDER; i++) H->weight[i] = w[i]; }
    SB_SYNC();
    i32 lsp[HB_ORDER];
#pragma unroll
    for (int j = 0; j < HB_ORDER; j++) lsp[j] = H->NLSF_Q15[j];
    const i16* cb1 = SB_T(hb_lsp_cb1_fix);
    const i16* cb2 = SB_T(hb_lsp_cb2_fix);
    i32 best = SB_I32_MAX, idx1 = 0;
    for (int e = lane; e < 256; e += 32) {
        const i32 dist = hb_lsp_dist1(lsp, e);
        if (dist < best) { best = dist; idx1 = e; }
    }
    wargmin(best, idx1);
#pragma unroll
    for (int j = 0; j < HB_ORDER; j++) lsp[j] -= cb1[idx1 * HB_ORDER + j];
    i32 best2 = SB_I32_MAX, idx2 = lane;
    if (lane < 16) best2 = hb_lsp_dist2(lsp, H->weight, lane);
    wargmin(best2, idx2);
    if (best2 == SB_I32_MAX) idx2 = 0;      // the reference's strict comparison never accepts INT_MAX
    SB_SYNC();
    if (lane < HB_ORDER) H->NLSF_Q15[lane] = (i32)cb1[idx1 * HB_ORDER + lane] + (i32)cb2[idx2 * HB_ORDER + lane];
    if (lane == 0) *lsp_idx_out = shl(idx2, 8) + idx1;
}
// One high-band frame of F samples: buffer update, order-8 LPC (Burg over four 88-sample blocks), two-stage LSP VQ,
// residual energy per sub-frame.  hb, H: shared memory; high: the new samples; outputs: global memory.
template <int F> SB_CFN void c_hb_analyse_frame(EncBands* hb, HbScr* H, const i16* high, i32* lsp_idx_out, i32* nrg0_out) {
    enum { LPCF = 80, BL = LPCF + HB_ORDER, SF = F >> 2 };
    const int lane = SB_LANE;
    SB_PARFOR(i, 0, F) hb->x_hb_buf[F + 40 + i] = high[i];
    SB_SYNC();
    SB_PARFOR(t, 0, 4 * BL) { const int k = t / BL, i = t - k * BL; H->LPC_in_pre[t] = hb->x_hb_buf[F - HB_ORDER + k * LPCF + i]; }
    SB_SYNC();
    i32 rn, rq;
    c_burg2<HB_ORDER>(&rn, &rq, H->A_Q16, &H->u.burg, H->LPC_in_pre, 4, H->LPC_in_pre, 4, BL, SB_FIXC(2.5e-5f, 32));
    SB_SYNC();
    {
        const i32 f = c_bwexpander32_factor(HB_ORDER, SB_FIXC(0.99995f, 16));
        if (lane < HB_ORDER) H->A_Q16[0][lane] = smulww(H->A_Q16[0][lane], f);
    }
    SB_SYNC();
    c_a2nlsf<HB_ORDER>(H->NLSF_Q15, H->A_Q16[0], &H->u.a2n);
    c_hb_lsp_quant(H, lsp_idx_out);
    SB_SYNC();
    if (lane == 0) { i32 nl[HB_ORDER]; i16 a12[HB_ORDER]; for (int i = 0; i < HB_ORDER; i++) nl[i] = H->NLSF_Q15[i]; nlsf2a_stable(a12, nl, HB_ORDER); for (int i = 0; i < HB_ORDER; i++) H->coef[i] = a12[i]; }
    SB_SYNC();
    // ---- residual energy of the four sub-frames (zero-state analysis filter per sub-frame) ----
    {
        i32 b[HB_ORDER];
#pragma unroll
        for (int d = 0; d < HB_ORDER; d++) b[d] = H->coef[d];
        const i16* p_hb = hb->x_hb_buf + F;
        i32 e0 = 0, e1 = 0, e2 = 0, e3 = 0;
        SB_PARFOR(t, 0, 4 * SF) {
            const int sub = t / SF, kx = t - sub * SF;
            const i16* in = p_hb + sub * SF;
            i32 acc = 0;
#pragma unroll
            for (int d = 0; d < HB_ORDER; d++) if (d < kx) acc = addw(acc, (i32)in[kx - 1 - d] * b[d]);
            const i32 ex = sat16(rshift_round(sub_sat32(shl((i32)in[kx], 12), acc), 12));
            const i32 sq = ex * ex;
            if (sub == 0) e0 = addw(e0, sq); else if (sub == 1) e1 = addw(e1, sq); else if (sub == 2) e2 = addw(e2, sq); else e3 = addw(e3, sq);
        }
        e0 = wsum(e0); e1 = wsum(e1); e2 = wsum(e2); e3 = wsum(e3);
        if (lane < 4) nrg0_out[lane] = sqrt_approx(lane == 0 ? e0 : (lane == 1 ? e1 : (lane == 2 ? e2 : e3)));
    }
    SB_SYNC();
    // buffer slides by one frame: [0,F) <- [F,2F), then [F,F+40) <- [2F,2F+40)
    {
        i32* xb = reinterpret_cast<i32*>(hb->x_hb_buf);
        SB_PARFOR(i, 0, F / 2) xb[i] = xb[F / 2 + i];
        SB_SYNC();
        SB_PARFOR(i, 0, 20) xb[F / 2 + i] = xb[F + i];
        if (lane == 0) hb->hb_first = 0;
        SB_SYNC();
    }
}
// Every high-band frame of the packet: n new samples in frames of F (the stream's hb_frame) -> scr->hb_lsp_idx, hb_nrg0.
SB_CFN void c_hb_analyse_packet(EncBands* hb, HbScr* H, const i16* high, int n, int F, EncScratch* scr) {
    for (int f = 0; f < n / F; f++) {
        if (F == HB_FRAME) c_hb_analyse_frame<HB_FRAME>(hb, H, high + f * F, &scr->hb_lsp_idx[f], scr->hb_nrg0[f]);
        else c_hb_analyse_frame<2 * HB_FRAME>(hb, H, high + f * F, &scr->hb_lsp_idx[f], scr->hb_nrg0[f]);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// frame / packet drivers
// ---------------------------------------------------------------------------------------------------------------------
// Working set of one stream during a packet (shared memory in the warp-per-stream kernel).
struct CoopWork {
    alignas(16) i16 low[2 * FRAME];        // low band of the packet (both 20 ms frames)
    i16 pIn_HP[FRAME];
    i16 res_pitch[2 * FRAME + LA_PITCH];
    EncCtrl c;
    i32 vad[2][6];             // per frame: speech activity Q8, four band qualities Q15, tilt Q15 (from the VAD kernel)
    i32 ar_keep[NB_SUBFR * 2 * SHAPE_ORDER];   // shaping filters of the frame, for the kernels that run after this one
    i32 par_keep[2];
    union {
        PitchScr pitch;
        ShapeScr shape;
        PredScr pred;
    } u;
};

// One stream's slot in the shared memory of the core-analysis kernel: persistent state + working set of the packet.
struct AnaSmem {
    EncSilk st;
    CoopWork W;
};
SB_CFN int sb_slot_bytes() { return (int)sizeof(AnaSmem); }

// SKP_Silk_encode_frame_FIX (encode_frame_FIX.c:34-131, 151-165, 199-208) up to the quantiser, one 20 ms frame.
SB_CFN void c_encode_frame_analysis(EncSilk* st, CoopWork* W, const i16* pIn, int frame_in_packet, const NlsfFastTabs* fast) {
    EncCtrl* c = &W->c;
    i16* x_frame = st->x_buf + FRAME;
    c_instances<1>([&](int d, int) {
        CoopWork* Wj = xoff(W, d);
        const i32* vad = Wj->vad[frame_in_packet];
        frame_analysis_begin(xoff(st, d), &Wj->c, Wj->pIn_HP, xoff(pIn, d), vad[0], vad + 1, vad[5]);
    });
    SB_PARFOR(i, 0, FRAME) x_frame[LA_SHAPE + i] = W->pIn_HP[i];   // LP_variable_cutoff is a copy (transition_frame_no == 0)
    SB_SYNC();
    SB_PHASE();
    c_find_pitch_lags(st, c, &W->u.pitch, W->res_pitch, x_frame);
    SB_PHASE();
    c_noise_shape_analysis(st, c, &W->u.shape, W->res_pitch + FRAME, x_frame);
    SB_PARFOR(i, 0, NB_SUBFR * 2 * SHAPE_ORDER) W->ar_keep[i] = (&W->u.shape.ar[0][0][0])[i];
    if (SB_LANE < 2) W->par_keep[SB_LANE] = W->u.shape.par3[SB_LANE == 0 ? 0 : 1];
    SB_SYNC();
    SB_PHASE();
    c_find_pred_coefs(st, c, &W->u.pred, W->res_pitch, frame_in_packet, fast);
    if (SB_LANE0) frame_analysis_end(st, c);
    SB_SYNC();
    {   // x_buf slides by one frame: [0,160) <- [160,320), then [160,200) <- [320,360) (each step reads only unwritten words)
        i32* xb = reinterpret_cast<i32*>(st->x_buf);
        SB_PARFOR(i, 0, FRAME / 2) xb[i] = xb[FRAME / 2 + i];
        SB_SYNC();
        SB_PARFOR(i, 0, LA_SHAPE / 2) xb[FRAME / 2 + i] = xb[FRAME + i];
        SB_SYNC();
    }
}

// Stage A for the SILK core of one packet.  st, W: shared memory; W->low already holds the low band; scr: global memory.
SB_CFN void c_enc_packet_analysis(EncSilk* st, CoopWork* W, EncScratch* scr, const NlsfFastTabs* fast = nullptr) {
    const int nf = st->frames_per_packet;
    if (SB_LANE < 12) {
        const int f = SB_LANE / 6, q = SB_LANE - 6 * f;
        W->vad[f][q] = q == 0 ? scr->vad_sa_Q8[f] : (q == 5 ? scr->vad_tilt_Q15[f] : scr->vad_quality_Q15[f][q - 1]);
    }
    SB_SYNC();
    for (int f = 0; f < nf; f++) {
        c_encode_frame_analysis(st, W, W->low + f * FRAME, f, fast);
        const i32* src = reinterpret_cast<const i32*>(&W->c);
        i32* dst = reinterpret_cast<i32*>(&scr->c[f]);
        SB_PARFOR(i, 0, (int)(sizeof(EncCtrl) / 4)) dst[i] = src[i];
        // the prefilter's input is the frame as the analysis saw it (delayed by the shaping look-ahead): after the slide of
        // x_buf at the end of the frame that is x_buf[0 .. FRAME)
        const i32* xs = reinterpret_cast<const i32*>(st->x_buf);
        i32* xd = reinterpret_cast<i32*>(scr->x_hp[f]);
        SB_PARFOR(i, 0, FRAME / 2) xd[i] = xs[i];
        SB_PARFOR(i, 0, NB_SUBFR * 2 * SHAPE_ORDER) (&scr->ar_Q24[f][0][0][0])[i] = W->ar_keep[i];
        if (SB_LANE < 2) scr->shape_par[f][SB_LANE] = W->par_keep[SB_LANE];
        SB_PARFOR(i, 0, 2 * LPC_ORDER) (&scr->nlsf_Q15[f][0][0])[i] = (&W->u.pred.nlsf_out[0][0])[i];
        SB_PARFOR(i, 0, (NB_SUBFR * LPC_ORDER + FRAME) / 2) reinterpret_cast<i32*>(scr->lpc_in_pre[f])[i] = reinterpret_cast<const i32*>(W->u.pred.LPC_in_pre)[i];
        if (SB_LANE < NB_SUBFR) scr->local_gains[f][SB_LANE] = W->u.pred.local_gains[SB_LANE];
        SB_SYNC();
    }
}

}  // namespace sb
#endif  // SB_COOP_ACTIVE
