// solo_b200 -- encoder front end of one 20 ms SILK frame: VAD, variable high-pass, pitch analysis.
// Reference paths relative to /root/reference/JC1_SDK_SRC_ARM/src/libSATECodec/.
#pragma once
#include "sb_sigproc.cuh"
#include "sb_state.cuh"

namespace sb {

// ---- SKP_Silk_VAD.c:41-70 ---------------------------------------------------------------------------
SB_FN void vad_init(VadState* v) {
    memset(v, 0, sizeof(VadState));
    for (int b = 0; b < 4; b++) v->NoiseLevelBias[b] = imax(50 / (b + 1), 1);
    for (int b = 0; b < 4; b++) {
        v->NL[b] = 100 * v->NoiseLevelBias[b];
        v->inv_NL[b] = SB_I32_MAX / v->NL[b];
    }
    v->counter = 15;
    for (int b = 0; b < 4; b++) v->NrgRatioSmth_Q8[b] = 100 * 256;
}

// ---- SKP_Silk_VAD.c:260-318 -------------------------------------------------------------------------
SB_FN void vad_get_noise_levels(const i32* pX, VadState* v) {
    i32 min_coef = v->counter < 1000 ? 32767 / ((v->counter >> 4) + 1) : 0;
    for (int k = 0; k < 4; k++) {
        i32 nl = v->NL[k];
        i32 nrg = add_pos_sat32(pX[k], v->NoiseLevelBias[k]);
        i32 inv_nrg = SB_I32_MAX / nrg;
        i32 coef;
        if (nrg > shl(nl, 3)) coef = 1024 >> 3;
        else if (nrg < nl) coef = 1024;
        else coef = smulwb(smulww(inv_nrg, nl), 1024 << 1);
        coef = imax(coef, min_coef);
        v->inv_NL[k] = smlawb(v->inv_NL[k], inv_nrg - v->inv_NL[k], coef);
        nl = SB_I32_MAX / v->inv_NL[k];
        nl = imin(nl, 0x00FFFFFF);
        v->NL[k] = nl;
    }
    v->counter++;
}

// ---- SKP_Silk_VAD.c:75-255 (frame length 160) ------------------------------------------------------
// X: scratch for the four band signals (the device kernel passes shared memory)
SB_FN void vad_get_sa_q8_x(VadState* v, i32* pSA_Q8, i32* pQuality_Q15, i32* pTilt_Q15, const i16* pIn, i16 (*X)[FRAME / 2]) {
    const i32 tiltWeights[4] = {30000, 6000, -12000, -12000};
    i32 Xnrg[4], NrgToNoiseRatio_Q8[4];
    ana_filt_bank_1(pIn, v->AnaState, X[0], X[3], FRAME);
    ana_filt_bank_1(X[0], v->AnaState1, X[0], X[2], FRAME >> 1);
    ana_filt_bank_1(X[0], v->AnaState2, X[0], X[1], FRAME >> 2);
    // differentiator on the lowest band
    int dfl = FRAME >> 3;
    X[0][dfl - 1] = (i16)(X[0][dfl - 1] >> 1);
    i16 HPstateTmp = X[0][dfl - 1];
    for (int i = dfl - 1; i > 0; i--) {
        X[0][i - 1] = (i16)(X[0][i - 1] >> 1);
        X[0][i] = (i16)(X[0][i] - X[0][i - 1]);
    }
    X[0][0] = (i16)(X[0][0] - v->HPstate);
    v->HPstate = HPstateTmp;
    i32 sumSquared = 0;
    for (int b = 0; b < 4; b++) {
        int dl = FRAME >> imin(4 - b, 3);
        int sl = dl >> 2, off = 0;
        Xnrg[b] = v->XnrgSubfr[b];
        for (int s = 0; s < 4; s++) {
            sumSquared = 0;
            for (int i = 0; i < sl; i++) {
                i32 x_tmp = X[b][i + off] >> 3;
                sumSquared = smlabb(sumSquared, x_tmp, x_tmp);
            }
            if (s < 3) Xnrg[b] = add_pos_sat32(Xnrg[b], sumSquared);
            else Xnrg[b] = add_pos_sat32(Xnrg[b], sumSquared >> 1);
            off += sl;
        }
        v->XnrgSubfr[b] = sumSquared;
    }
    vad_get_noise_levels(Xnrg, v);
    sumSquared = 0;
    i32 input_tilt = 0;
    for (int b = 0; b < 4; b++) {
        i32 speech_nrg = Xnrg[b] - v->NL[b];
        if (speech_nrg > 0) {
            if ((Xnrg[b] & 0xFF800000) == 0) NrgToNoiseRatio_Q8[b] = shl(Xnrg[b], 8) / (v->NL[b] + 1);
            else NrgToNoiseRatio_Q8[b] = Xnrg[b] / ((v->NL[b] >> 8) + 1);
            i32 SNR_Q7 = lin2log(NrgToNoiseRatio_Q8[b]) - 8 * 128;
            sumSquared = smlabb(sumSquared, SNR_Q7, SNR_Q7);
            if (speech_nrg < (1 << 20)) SNR_Q7 = smulwb(shl(sqrt_approx(speech_nrg), 6), SNR_Q7);
            input_tilt = smlawb(input_tilt, tiltWeights[b], SNR_Q7);
        } else {
            NrgToNoiseRatio_Q8[b] = 256;
        }
    }
    sumSquared = sumSquared / 4;
    i32 pSNR_dB_Q7 = (i16)(3 * sqrt_approx(sumSquared));
    i32 SA_Q15 = sigm_q15(smulwb(45000, pSNR_dB_Q7) - 128);
    *pTilt_Q15 = shl(sigm_q15(input_tilt) - 16384, 1);
    i32 speech_nrg = 0;
    for (int b = 0; b < 4; b++) speech_nrg += (b + 1) * ((Xnrg[b] - v->NL[b]) >> 4);
    if (speech_nrg <= 0) SA_Q15 = SA_Q15 >> 1;
    else if (speech_nrg < 32768) {
        speech_nrg = sqrt_approx(shl(speech_nrg, 15));
        SA_Q15 = smulwb(32768 + speech_nrg, SA_Q15);
    }
    *pSA_Q8 = imin(SA_Q15 >> 7, 255);
    i32 smooth_coef_Q16 = (i16)smulwb(4096, smulwb(SA_Q15, SA_Q15));
    for (int b = 0; b < 4; b++) {
        v->NrgRatioSmth_Q8[b] = smlawb(v->NrgRatioSmth_Q8[b], NrgToNoiseRatio_Q8[b] - v->NrgRatioSmth_Q8[b], smooth_coef_Q16);
        i32 SNR_Q7 = 3 * (lin2log(v->NrgRatioSmth_Q8[b]) - 8 * 128);
        pQuality_Q15[b] = sigm_q15((SNR_Q7 - 16 * 128) >> 4);
    }
}

SB_FN void vad_get_sa_q8(VadState* v, i32* pSA_Q8, i32* pQuality_Q15, i32* pTilt_Q15, const i16* pIn) {
    i16 X[4][FRAME / 2];
    vad_get_sa_q8_x(v, pSA_Q8, pQuality_Q15, pTilt_Q15, pIn, X);
}

// Voice activity of every frame of a packet ahead of the rest of the analysis (device: its own thread-per-stream kernel --
// the detector is three cascaded all-pass filter banks plus scalar bookkeeping, a pure recurrence that depends on nothing but
// the low-band signal and its own state).  low: nf * FRAME samples.
SB_FN void vad_packet(VadState* v, const i16* low, int nf, i32* sa_Q8, i32 (*quality_Q15)[4], i32* tilt_Q15) {
    for (int f = 0; f < nf; f++) vad_get_sa_q8(v, &sa_Q8[f], quality_Q15[f], &tilt_Q15[f], low + f * FRAME);
}

// ---- SKP_Silk_HP_variable_cutoff_FIX.c:37-118 ---------------------------------------------------------
SB_FN void hp_variable_cutoff(EncSilk* st, EncCtrl* c, i16* out, const i16* in) {
    if (st->prev_sigtype == 0) {
        i32 pitch_freq_Hz_Q16 = shl(8 * 1000, 16) / st->prevLag;
        i32 pitch_freq_log_Q7 = lin2log(pitch_freq_Hz_Q16) - (16 << 7);
        i32 quality_Q15 = c->input_quality_bands_Q15[0];
        pitch_freq_log_Q7 = subw(pitch_freq_log_Q7, smulwb(smulwb(shl(quality_Q15, 2), quality_Q15), pitch_freq_log_Q7 - 809));
        pitch_freq_log_Q7 = addw(pitch_freq_log_Q7, (SB_FIXC(0.6, 15) - quality_Q15) >> 9);
        i32 delta_freq_Q7 = pitch_freq_log_Q7 - (st->variable_HP_smth1_Q15 >> 8);
        if (delta_freq_Q7 < 0) delta_freq_Q7 = mulw(delta_freq_Q7, 3);
        delta_freq_Q7 = limit(delta_freq_Q7, -SB_FIXC(0.4f, 7), SB_FIXC(0.4f, 7));
        st->variable_HP_smth1_Q15 = smlawb(st->variable_HP_smth1_Q15, mulw(shl(st->speech_activity_Q8, 1), delta_freq_Q7), SB_FIXC(0.1f, 16));
    }
    st->variable_HP_smth2_Q15 = smlawb(st->variable_HP_smth2_Q15, st->variable_HP_smth1_Q15 - st->variable_HP_smth2_Q15, SB_FIXC(0.015f, 16));
    c->pitch_freq_low_Hz = log2lin(st->variable_HP_smth2_Q15 >> 8);
    c->pitch_freq_low_Hz = limit(c->pitch_freq_low_Hz, SB_FIXC(80.0f, 0), SB_FIXC(150.0f, 0));
    i32 Fc_Q19 = smulbb(1482, c->pitch_freq_low_Hz) / 8;
    i32 r_Q28 = SB_FIXC(1.0, 28) - mulw(SB_FIXC(0.92, 9), Fc_Q19);
    i32 B_Q28[3], A_Q28[2];
    B_Q28[0] = r_Q28;
    B_Q28[1] = shl(-r_Q28, 1);
    B_Q28[2] = r_Q28;
    i32 r_Q22 = r_Q28 >> 6;
    A_Q28[0] = smulww(r_Q22, smulww(Fc_Q19, Fc_Q19) - SB_FIXC(2.0, 22));
    A_Q28[1] = smulww(r_Q22, r_Q22);
    biquad_alt(in, B_Q28, A_Q28, st->In_HP_State, out, FRAME);
}

// ---- encode_frame_FIX.c:151-165: VAD flag and the DTX counter ----------------------------------------------
SB_FN void vad_flag_and_dtx(EncSilk* st, i32* vadFlag) {
    if (st->speech_activity_Q8 < SB_FIXC(0.1f, 8)) {
        st->vadFlag = 0;
        st->noSpeechCounter++;
        if (st->noSpeechCounter > 5) st->inDTX = 1;
        if (st->noSpeechCounter > 20 + 5) { st->noSpeechCounter = 5; st->inDTX = 0; }
    } else {
        st->noSpeechCounter = 0; st->inDTX = 0; st->vadFlag = 1;
    }
    *vadFlag = st->vadFlag;
}

// The pitch-search arithmetic below is written once for the scalar model and the analysis kernel (c_pitch_analysis_core,
// c_find_pitch_lags in sb_coop.cuh), which calls it on every lane or on the lane that owns a candidate.

// ---- SKP_Silk_pitch_analysis_core.c:680-706: down-shift of a signal whose largest |x| is x_maxabs ---------------
SB_HD i32 pitch_find_scaling(i32 x_maxabs, int sum_sqr_len) {
    // int16_array_maxabs (SKP_Silk_array_maxabs.c:40-66) takes |x| at the largest x^2 and reports 32767 from 1073676289 on
    const i32 x_max = x_maxabs * x_maxabs >= 1073676289 ? 32767 : x_maxabs;
    i32 nbits;
    if (x_max < 32767) nbits = 32 - clz32(smulbb(x_max, x_max));
    else nbits = 30;
    nbits += 17 - (clz32(sum_sqr_len) - 16);
    return nbits < 31 ? 0 : nbits - 30;
}
SB_FN i32 maxabs16(const i16* x, int n) {
    i32 m = 0;
    for (int i = 0; i < n; i++) m = imax(m, iabs((i32)x[i]));
    return m;
}
// stage-2 normalised correlation of a target sub-frame and one lag's basis vector (:399-420)
SB_HD i32 pitch_stage2_corr(i32 cross_corr, i32 energy_target, i32 energy_basis) {
    if (cross_corr <= 0) return 0;
    i32 energy = imax(energy_target, energy_basis);
    int lshift = limit(clz32(cross_corr) - 1, 0, 15);
    i32 temp32 = shl(cross_corr, lshift) / ((energy >> (15 - lshift)) + 1);
    temp32 = smulwb(cross_corr, temp32);
    temp32 = add_sat32(temp32, temp32);
    lshift = limit(clz32(temp32) - 1, 0, 15);
    energy = imin(energy_target, energy_basis);
    return (i16)(shl(temp32, lshift) / ((energy >> (15 - lshift)) + 1));
}
// Score of stage-2 candidate lag d, whose best contour CBimax sums to CCmax: the sum less the short-lag bias and the
// previous-lag bias (:427-455).  SB_I32_MIN if the candidate may not win: its sum is not above the threshold, or the
// contour's first lag is above the minimum lag.
SB_HD i32 pitch_lag_score(i32 CCmax, int CBimax, int d, i32 prevLag, i32 LTPCorr_Q15, i32 search_thres2_Q15) {
    const i32 corr_thres_Q15 = smulbb(search_thres2_Q15, search_thres2_Q15) >> 13;
    if (CCmax <= corr_thres_Q15 || SB_T(pitch_cb_lags_stage2)[CBimax] > 16) return SB_I32_MIN;
    const i32 lag_log2_Q7 = lin2log(d);
    i32 score = CCmax - (smulbb(4 * 6554, lag_log2_Q7) >> 7);
    if (prevLag > 0) {
        i32 dl = lag_log2_Q7 - lin2log(prevLag);
        dl = smulbb(dl, dl) >> 7;
        i32 prev_lag_bias_Q15 = smulbb(4 * 6554, LTPCorr_Q15) >> 15;
        prev_lag_bias_Q15 = mulw(prev_lag_bias_Q15, dl) / (dl + (1 << 6));
        score -= prev_lag_bias_Q15;
    }
    return score;
}

// ---- SKP_Silk_pitch_analysis_core.c:65-560 specialised to Fs = 8 kHz, complexity 2 (stage 3 is skipped
// at 8 kHz: App. A Q23).  Returns 0 voiced / 1 unvoiced.
SB_FN int pitch_analysis_core(const i16* signal, i32* pitch_out, i32* lagIndex, i32* contourIndex, i32* LTPCorr_Q15,
                              i32 prevLag, i32 search_thres1_Q16, i32 search_thres2_Q15) {
    enum { FL8 = 320, FL4 = 160, SF8 = 40, MINL8 = 16, MAXL8 = 144, MINL4 = 8, MAXL4 = 72, CW = 221, NCB = 11 };
    i16 signal_8kHz[FL8];
    i16 signal_4kHz[FL4];
    i16 C[4][CW];
    i32 d_srch[24];
    i16 d_comp[CW];
    i32 filt_state[2] = {0, 0};
    for (int i = 0; i < FL8; i++) signal_8kHz[i] = signal[i];
    resampler_down2(filt_state, signal_4kHz, signal_8kHz, FL8);
    for (int i = FL4 - 1; i > 0; i--) signal_4kHz[i] = (i16)add_sat16(signal_4kHz[i], signal_4kHz[i - 1]);
    i32 shift = pitch_find_scaling(maxabs16(signal_4kHz, FL4), imax(SF8, FL4 >> 1));
    if (shift > 0) for (int i = 0; i < FL4; i++) signal_4kHz[i] = (i16)(signal_4kHz[i] >> shift);

    // ---- first stage at 4 kHz ----
    for (int k = 0; k < 4; k++) for (int i = 0; i < CW; i++) C[k][i] = 0;
    const i16* target_ptr = &signal_4kHz[FL4 >> 1];
    for (int k = 0; k < 2; k++) {
        const i16* basis_ptr = target_ptr - MINL4;
        i32 cross_corr = inner_prod16(target_ptr, basis_ptr, SF8);
        i32 normalizer = inner_prod16(basis_ptr, basis_ptr, SF8);
        normalizer = add_sat32(normalizer, smulbb(SF8, 4000));
        i32 temp32 = cross_corr / (sqrt_approx(normalizer) + 1);
        C[k][MINL4] = (i16)sat16(temp32);
        for (int d = MINL4 + 1; d <= MAXL4; d++) {
            basis_ptr--;
            cross_corr = inner_prod16(target_ptr, basis_ptr, SF8);
            normalizer = addw(normalizer, subw(smulbb(basis_ptr[0], basis_ptr[0]), smulbb(basis_ptr[SF8], basis_ptr[SF8])));
            temp32 = cross_corr / (sqrt_approx(normalizer) + 1);
            C[k][d] = (i16)sat16(temp32);
        }
        target_ptr += SF8;
    }
    for (int i = MAXL4; i >= MINL4; i--) {
        i32 sum = (i32)C[0][i] + (i32)C[1][i];
        sum = sum >> 1;
        sum = smlawb(sum, sum, shl(-i, 4));
        C[0][i] = (i16)sum;
    }
    int length_d_srch = 4 + 2 * 2;
    insertion_sort_decreasing_i16(&C[0][MINL4], d_srch, MAXL4 - MINL4 + 1, length_d_srch);
    target_ptr = &signal_4kHz[FL4 >> 1];
    i32 energy = inner_prod16(target_ptr, target_ptr, FL4 >> 1);
    energy = add_pos_sat32(energy, 1000);
    i32 Cmax = C[0][MINL4];
    i32 threshold = smulbb(Cmax, Cmax);
    if ((energy >> (4 + 2)) > threshold) {
        for (int k = 0; k < 4; k++) pitch_out[k] = 0;
        *LTPCorr_Q15 = 0; *lagIndex = 0; *contourIndex = 0;
        return 1;
    }
    threshold = smulwb(search_thres1_Q16, Cmax);
    for (int i = 0; i < length_d_srch; i++) {
        if (C[0][MINL4 + i] > threshold) d_srch[i] = (d_srch[i] + MINL4) << 1;
        else { length_d_srch = i; break; }
    }
    for (int i = MINL8 - 5; i < MAXL8 + 5; i++) d_comp[i] = 0;
    for (int i = 0; i < length_d_srch; i++) d_comp[d_srch[i]] = 1;
    for (int i = MAXL8 + 3; i >= MINL8; i--) d_comp[i] = (i16)(d_comp[i] + d_comp[i - 1] + d_comp[i - 2]);
    length_d_srch = 0;
    for (int i = MINL8; i < MAXL8 + 1; i++) {
        if (d_comp[i + 1] > 0) { d_srch[length_d_srch] = i; length_d_srch++; }
    }
    for (int i = MAXL8 + 3; i >= MINL8; i--) d_comp[i] = (i16)(d_comp[i] + d_comp[i - 1] + d_comp[i - 2] + d_comp[i - 3]);
    int length_d_comp = 0;
    for (int i = MINL8; i < MAXL8 + 4; i++) {
        if (d_comp[i] > 0) { d_comp[length_d_comp] = (i16)(i - 2); length_d_comp++; }
    }

    // ---- second stage at 8 kHz ----
    shift = pitch_find_scaling(maxabs16(signal_8kHz, FL8), SF8);
    if (shift > 0) for (int i = 0; i < FL8; i++) signal_8kHz[i] = (i16)(signal_8kHz[i] >> shift);
    for (int k = 0; k < 4; k++) for (int i = 0; i < CW; i++) C[k][i] = 0;
    target_ptr = &signal_8kHz[FL4];
    for (int k = 0; k < 4; k++) {
        i32 energy_target = inner_prod16(target_ptr, target_ptr, SF8);
        for (int j = 0; j < length_d_comp; j++) {
            int d = d_comp[j];
            const i16* basis_ptr = target_ptr - d;
            C[k][d] = (i16)pitch_stage2_corr(inner_prod16(target_ptr, basis_ptr, SF8), energy_target, inner_prod16(basis_ptr, basis_ptr, SF8));
        }
        target_ptr += SF8;
    }
    i32 CCmax = SB_I32_MIN, CCmax_b = SB_I32_MIN;
    int CBimax = 0, lag = -1;
    const i16* cbl = SB_T(pitch_cb_lags_stage2);  // [4][11]
    for (int k = 0; k < length_d_srch; k++) {
        int d = d_srch[k];
        i32 CC[NCB];
        for (int j = 0; j < NCB; j++) {
            CC[j] = 0;
            for (int i = 0; i < 4; i++) CC[j] = CC[j] + (i32)C[i][d + cbl[i * NCB + j]];
        }
        i32 CCmax_new = SB_I32_MIN; int CBimax_new = 0;
        for (int i = 0; i < NCB; i++) if (CC[i] > CCmax_new) { CCmax_new = CC[i]; CBimax_new = i; }
        const i32 CCmax_new_b = pitch_lag_score(CCmax_new, CBimax_new, d, prevLag, *LTPCorr_Q15, search_thres2_Q15);
        if (CCmax_new_b > CCmax_b) { CCmax_b = CCmax_new_b; CCmax = CCmax_new; lag = d; CBimax = CBimax_new; }
    }
    if (lag == -1) {
        for (int k = 0; k < 4; k++) pitch_out[k] = 0;
        *LTPCorr_Q15 = 0; *lagIndex = 0; *contourIndex = 0;
        return 1;
    }
    CCmax = imax(CCmax, 0);
    *LTPCorr_Q15 = sqrt_approx(shl(CCmax, 13));
    for (int k = 0; k < 4; k++) pitch_out[k] = lag + cbl[k * NCB + CBimax];
    *lagIndex = lag - MINL8;
    *contourIndex = CBimax;
    return 0;
}

// ---- SKP_Silk_find_pitch_lags_FIX.c:32-125 -----------------------------------------------------------
// prediction gain of the order-10 whitening filter from the regularised energy and Schur's residual energy (:86-88)
SB_HD i32 pitch_pred_gain_q16(i32 auto_corr0, i32 res_nrg) { return div32_varq(auto_corr0, imax(res_nrg, 1), 16); }
// voicing threshold of the pitch search, order 10 (:108-115)
SB_HD i32 pitch_thrhld_q15(i32 speech_activity_Q8, i32 prev_sigtype, i32 input_tilt_Q15) {
    i32 thrhld_Q15 = SB_FIXC(0.45, 15);
    thrhld_Q15 = smlabb(thrhld_Q15, SB_FIXC(-0.004, 15), 10);
    thrhld_Q15 = smlabb(thrhld_Q15, SB_FIXC(-0.1, 7), speech_activity_Q8);
    thrhld_Q15 = smlabb(thrhld_Q15, SB_FIXC(0.15, 15), prev_sigtype);
    thrhld_Q15 = smlawb(thrhld_Q15, SB_FIXC(-0.1, 16), input_tilt_Q15);
    return (i16)sat16(thrhld_Q15);
}
// x points at x_buf + FRAME (start of the frame to encode); res receives 336 samples of LPC residual.
SB_FN void find_pitch_lags(EncSilk* st, EncCtrl* c, i16* res, const i16* x) {
    enum { BUF_LEN = LA_PITCH + 2 * FRAME, ORD = 10 };
    i16 Wsig[PITCH_LPC_WIN];
    i32 auto_corr[ORD + 1];
    i16 rc_Q15[ORD];
    i32 A_Q24[ORD];
    i16 A_Q12[ORD];
    const i16* x_buf = x - FRAME;
    const i16* x_buf_ptr = x_buf + BUF_LEN - PITCH_LPC_WIN;
    apply_sine_window(Wsig, x_buf_ptr, 1, LA_PITCH);
    for (int i = 0; i < PITCH_LPC_WIN - 2 * LA_PITCH; i++) Wsig[LA_PITCH + i] = x_buf_ptr[LA_PITCH + i];
    apply_sine_window(Wsig + PITCH_LPC_WIN - LA_PITCH, x_buf_ptr + PITCH_LPC_WIN - LA_PITCH, 2, LA_PITCH);
    i32 scale;
    autocorr(auto_corr, &scale, Wsig, PITCH_LPC_WIN, ORD + 1);
    auto_corr[0] = smlawb(auto_corr[0], auto_corr[0], SB_FIXC(1e-3f, 16));
    i32 res_nrg = schur(rc_Q15, auto_corr, ORD);
    c->predGain_Q16 = pitch_pred_gain_q16(auto_corr[0], res_nrg);
    k2a(A_Q24, rc_Q15, ORD);
    for (int i = 0; i < ORD; i++) A_Q12[i] = (i16)sat16(A_Q24[i] >> 12);
    bwexpander(A_Q12, ORD, SB_FIXC(0.99f, 16));
    ma_prediction_zero_state(x_buf, A_Q12, res, BUF_LEN, ORD);
    for (int i = 0; i < ORD; i++) res[i] = 0;
    c->sigtype = pitch_analysis_core(res, c->pitchL, &c->lagIndex, &c->contourIndex, &st->LTPCorr_Q15, st->prevLag, SB_FIXC(0.7f, 16),
                                     pitch_thrhld_q15(st->speech_activity_Q8, st->prev_sigtype, c->input_tilt_Q15));
}

}  // namespace sb
