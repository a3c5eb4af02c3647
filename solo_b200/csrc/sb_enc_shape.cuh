// solo_b200 -- noise-shape analysis and prefilter of one 20 ms frame.
// Reference paths relative to /root/reference/JC1_SDK_SRC_ARM/src/libSATECodec/.
#pragma once
#include "sb_sigproc.cuh"
#include "sb_state.cuh"

namespace sb {

// ---- SKP_Silk_warped_autocorrelation_FIX.c:36-85 (order 16, length 120) ----------------------------------
SB_FN void warped_autocorrelation(i32* corr, i32* scale, const i16* input, i32 warping_Q16, int length, int order) {
    const int QC = 10, QS = 14;
    i32 state_QS[SHAPE_ORDER + 1];
    i64 corr_QC[SHAPE_ORDER + 1];
    for (int i = 0; i <= SHAPE_ORDER; i++) { state_QS[i] = 0; corr_QC[i] = 0; }
    warping_Q16 = (i16)warping_Q16;
    for (int n = 0; n < length; n++) {
        i32 tmp1_QS = shl((i32)input[n], QS);
        for (int i = 0; i < order; i += 2) {
            i32 tmp2_QS = smlawb(state_QS[i], subw(state_QS[i + 1], tmp1_QS), warping_Q16);
            state_QS[i] = tmp1_QS;
            corr_QC[i] += smull(tmp1_QS, state_QS[0]) >> (2 * QS - QC);
            tmp1_QS = smlawb(state_QS[i + 1], subw(state_QS[i + 2], tmp2_QS), warping_Q16);
            state_QS[i + 1] = tmp2_QS;
            corr_QC[i + 1] += smull(tmp2_QS, state_QS[0]) >> (2 * QS - QC);
        }
        state_QS[order] = tmp1_QS;
        corr_QC[order] += smull(tmp1_QS, state_QS[0]) >> (2 * QS - QC);
    }
    int lsh = clz64(corr_QC[0]) - 35;
    lsh = limit(lsh, -12 - QC, 30 - QC);
    *scale = -(QC + lsh);
    if (lsh >= 0) for (int i = 0; i < order + 1; i++) corr[i] = (i32)shl64(corr_QC[i], lsh);
    else for (int i = 0; i < order + 1; i++) corr[i] = (i32)(corr_QC[i] >> (-lsh));
}

// ---- SKP_Silk_noise_shape_analysis_FIX.c:52-132 -----------------------------------------------------------
SB_FN void limit_warped_coefs(i32* syn_Q24, i32* ana_Q24, i32 lambda_Q16, i32 limit_Q24, int order) {
    int ind = 0;
    i32 nom_Q16, den_Q24, gain_syn_Q16, gain_ana_Q16;
    lambda_Q16 = -lambda_Q16;
    for (int i = order - 1; i > 0; i--) {
        syn_Q24[i - 1] = smlawb(syn_Q24[i - 1], syn_Q24[i], lambda_Q16);
        ana_Q24[i - 1] = smlawb(ana_Q24[i - 1], ana_Q24[i], lambda_Q16);
    }
    lambda_Q16 = -lambda_Q16;
    nom_Q16 = smlawb(SB_FIXC(1.0, 16), -lambda_Q16, lambda_Q16);
    den_Q24 = smlawb(SB_FIXC(1.0, 24), syn_Q24[0], lambda_Q16);
    gain_syn_Q16 = div32_varq(nom_Q16, den_Q24, 24);
    den_Q24 = smlawb(SB_FIXC(1.0, 24), ana_Q24[0], lambda_Q16);
    gain_ana_Q16 = div32_varq(nom_Q16, den_Q24, 24);
    for (int i = 0; i < order; i++) {
        syn_Q24[i] = smulww(gain_syn_Q16, syn_Q24[i]);
        ana_Q24[i] = smulww(gain_ana_Q16, ana_Q24[i]);
    }
    for (int iter = 0; iter < 10; iter++) {
        i32 maxabs_Q24 = -1;
        for (int i = 0; i < order; i++) {
            i32 a = syn_Q24[i], b = ana_Q24[i];
            a = (a ^ (a >> 31)) - (a >> 31);
            b = (b ^ (b >> 31)) - (b >> 31);
            i32 tmp = imax(a, b);
            if (tmp > maxabs_Q24) { maxabs_Q24 = tmp; ind = i; }
        }
        if (maxabs_Q24 <= limit_Q24) return;
        for (int i = 1; i < order; i++) {
            syn_Q24[i - 1] = smlawb(syn_Q24[i - 1], syn_Q24[i], lambda_Q16);
            ana_Q24[i - 1] = smlawb(ana_Q24[i - 1], ana_Q24[i], lambda_Q16);
        }
        gain_syn_Q16 = inverse32_varq(gain_syn_Q16, 32);
        gain_ana_Q16 = inverse32_varq(gain_ana_Q16, 32);
        for (int i = 0; i < order; i++) {
            syn_Q24[i] = smulww(gain_syn_Q16, syn_Q24[i]);
            ana_Q24[i] = smulww(gain_ana_Q16, ana_Q24[i]);
        }
        i32 chirp_Q16 = SB_FIXC(0.99, 16) - div32_varq(
            smulwb(maxabs_Q24 - limit_Q24, smlabb(SB_FIXC(0.8, 10), SB_FIXC(0.1, 10), iter)),
            mulw(maxabs_Q24, ind + 1), 22);
        bwexpander_32(syn_Q24, order, chirp_Q16);
        bwexpander_32(ana_Q24, order, chirp_Q16);
        lambda_Q16 = -lambda_Q16;
        for (int i = order - 1; i > 0; i--) {
            syn_Q24[i - 1] = smlawb(syn_Q24[i - 1], syn_Q24[i], lambda_Q16);
            ana_Q24[i - 1] = smlawb(ana_Q24[i - 1], ana_Q24[i], lambda_Q16);
        }
        lambda_Q16 = -lambda_Q16;
        nom_Q16 = smlawb(SB_FIXC(1.0, 16), -lambda_Q16, lambda_Q16);
        den_Q24 = smlawb(SB_FIXC(1.0, 24), syn_Q24[0], lambda_Q16);
        gain_syn_Q16 = div32_varq(nom_Q16, den_Q24, 24);
        den_Q24 = smlawb(SB_FIXC(1.0, 24), ana_Q24[0], lambda_Q16);
        gain_ana_Q16 = div32_varq(nom_Q16, den_Q24, 24);
        for (int i = 0; i < order; i++) {
            syn_Q24[i] = smulww(gain_syn_Q16, syn_Q24[i]);
            ana_Q24[i] = smulww(gain_ana_Q16, ana_Q24[i]);
        }
    }
}

// ---- SKP_Silk_noise_shape_analysis_FIX.c:137-531 ---------------------------------------------------------
// The per-frame control arithmetic below is written once for the scalar model and the analysis kernel
// (c_noise_shape_analysis, sb_coop.cuh), which calls it on every lane or on the lane that owns sub-frame / window k.

// Frame-level control: SNR adjustment, sparseness (unvoiced: energy_variation_Q7 of the residual's ten 2 ms energies),
// bandwidth expansion and warping (:155-268).
struct ShapeCtl {
    i32 input_quality_Q14, coding_quality_Q14, SNR_adj_dB_Q7, md_SNR_adj_dB_Q7, sparseness_Q8, QuantOffsetType;
    i32 BWExp1_Q16, BWExp2_Q16, warping_Q16;
};
SB_HD ShapeCtl shape_control(int sigtype, i32 SNR_dB_Q7, i32 SNRPerMD_dB_Q7, const i32* input_quality_bands_Q15,
                             i32 speech_activity_Q8, i32 LTPCorr_Q15, i32 energy_variation_Q7, i32 predGain_Q16) {
    ShapeCtl s;
    // inBandFEC_SNR_comp_Q8 == 0 (LBRR off)
    s.input_quality_Q14 = (input_quality_bands_Q15[0] + input_quality_bands_Q15[1]) >> 2;
    s.coding_quality_Q14 = sigm_q15(rshift_round(SNR_dB_Q7 - SB_FIXC(18.0, 7), 4)) >> 1;
    const i32 md_input_quality_Q14 = sigm_q15(rshift_round(SNRPerMD_dB_Q7 - SB_FIXC(18.0, 7), 4)) >> 1;
    i32 b_Q8 = SB_FIXC(1.0, 8) - speech_activity_Q8;
    b_Q8 = smulwb(shl(b_Q8, 8), b_Q8);
    auto snr_adj = [&](i32 snr_Q7, i32 quality_Q14) {
        const i32 a = smlawb(snr_Q7, smulbb(SB_FIXC(-4.0f, 7) >> (4 + 1), b_Q8), smulwb(SB_FIXC(1.0, 14) + quality_Q14, s.coding_quality_Q14));
        if (sigtype == 0) return smlawb(a, SB_FIXC(2.0f, 8), LTPCorr_Q15);
        return smlawb(a, smlawb(SB_FIXC(6.0, 9), -SB_FIXC(0.4, 18), snr_Q7), SB_FIXC(1.0, 14) - s.input_quality_Q14);
    };
    s.SNR_adj_dB_Q7 = snr_adj(SNR_dB_Q7, s.input_quality_Q14);
    s.md_SNR_adj_dB_Q7 = snr_adj(SNRPerMD_dB_Q7, md_input_quality_Q14);
    s.sparseness_Q8 = 0;
    s.QuantOffsetType = 0;
    if (sigtype != 0) {
        s.sparseness_Q8 = sigm_q15(smulwb(energy_variation_Q7 - SB_FIXC(5.0, 7), SB_FIXC(0.1, 16))) >> 7;
        s.QuantOffsetType = s.sparseness_Q8 > SB_FIXC(0.75f, 8) ? 0 : 1;
        s.SNR_adj_dB_Q7 = smlawb(s.SNR_adj_dB_Q7, SB_FIXC(2.0f, 15), s.sparseness_Q8 - SB_FIXC(0.5, 8));
        s.md_SNR_adj_dB_Q7 = smlawb(s.md_SNR_adj_dB_Q7, SB_FIXC(2.0f, 15), s.sparseness_Q8 - SB_FIXC(0.5, 8));
    }
    const i32 strength_Q16 = smulwb(predGain_Q16, SB_FIXC(1e-3f, 16));
    s.BWExp1_Q16 = s.BWExp2_Q16 = div32_varq(SB_FIXC(0.95f, 16), smlaww(SB_FIXC(1.0, 16), strength_Q16, strength_Q16), 16);
    const i32 delta_Q16 = smulwb(SB_FIXC(1.0, 16) - smulbb(3, s.coding_quality_Q14), SB_FIXC(0.01f, 16));
    s.BWExp1_Q16 = subw(s.BWExp1_Q16, delta_Q16);
    s.BWExp2_Q16 = addw(s.BWExp2_Q16, delta_Q16);
    s.BWExp1_Q16 = shl(s.BWExp1_Q16, 14) / (s.BWExp2_Q16 >> 2);
    s.warping_Q16 = smlawb(WARPING_Q16, s.coding_quality_Q14, SB_FIXC(0.01, 18));
    return s;
}

// One window's shaping filters from its warped autocorrelation (Q-domain exponent `scale`; auto_corr is overwritten):
// regularisation, Schur, step-up, warped gain, AR2 = bandwidth expansion BWExp2, AR1 = AR2 expanded by BWExp1 (:300-344).
// Returns the window's gain before the frame-level tweaks.
SB_HD i32 shape_window(i32 (&AR2_Q24)[SHAPE_ORDER], i32 (&AR1_Q24)[SHAPE_ORDER], i32 (&auto_corr)[SHAPE_ORDER + 1], i32 scale,
                       i32 warping_Q16, i32 BWExp1_Q16, i32 BWExp2_Q16) {
    i32 refl_coef_Q16[SHAPE_ORDER];
    auto_corr[0] = addw(auto_corr[0], imax(smulwb(auto_corr[0] >> 4, SB_FIXC(1e-5f, 20)), 1));
    i32 nrg = schur64_r<SHAPE_ORDER>(refl_coef_Q16, auto_corr);
    k2a_q16_r<SHAPE_ORDER>(AR2_Q24, refl_coef_Q16);
    int Qnrg = -scale;
    if (Qnrg & 1) { Qnrg -= 1; nrg >>= 1; }
    const i32 tmp32 = sqrt_approx(nrg);
    Qnrg >>= 1;
    i32 gain_Q16 = lshift_sat32(tmp32, 16 - Qnrg);
    {   // warped_gain (:33-50)
        const i32 lambda_Q16 = -warping_Q16;
        i32 gain_Q24 = AR2_Q24[SHAPE_ORDER - 1];
#pragma unroll
        for (int i = SHAPE_ORDER - 2; i >= 0; i--) gain_Q24 = smlawb(AR2_Q24[i], gain_Q24, lambda_Q16);
        gain_Q24 = smlawb(SB_FIXC(1.0, 24), gain_Q24, -lambda_Q16);
        gain_Q16 = smulww(gain_Q16, inverse32_varq(gain_Q24, 40));
    }
    if (gain_Q16 < 0) gain_Q16 = SB_I32_MAX;
    bwexpander_32_r<SHAPE_ORDER>(AR2_Q24, BWExp2_Q16);
#pragma unroll
    for (int i = 0; i < SHAPE_ORDER; i++) AR1_Q24[i] = AR2_Q24[i];
    bwexpander_32_r<SHAPE_ORDER>(AR1_Q24, BWExp1_Q16);
    return gain_Q16;
}

// gain tweaking (:346-384): the SNR-dependent multiplier, the offset that follows the running average, one gain
SB_HD i32 shape_gain_mult_q16(i32 SNR_adj_dB_Q7) { return log2lin(negw(smlawb(-SB_FIXC(16.0, 7), SNR_adj_dB_Q7, SB_FIXC(0.16, 16)))); }
SB_HD i32 shape_gain_add_q16(i32 avgGain_Q16) {
    const i32 gain_add_Q16 = log2lin(smlawb(SB_FIXC(16.0, 7), SB_FIXC(4.0f, 7), SB_FIXC(0.16, 16)));
    return add_sat32(gain_add_Q16, smulww(avgGain_Q16, log2lin(smlawb(SB_FIXC(16.0, 7), SB_FIXC(-50.0f, 7), SB_FIXC(0.16, 16)))));
}
SB_HD i32 shape_gain_tweak(i32 gain_Q16, i32 gain_mult_Q16, i32 gain_add_Q16) {
    gain_Q16 = smulww(gain_Q16, gain_mult_Q16);
    if (gain_Q16 < 0) gain_Q16 = SB_I32_MAX;
    return add_pos_sat32(gain_Q16, gain_add_Q16);
}
// the running average after one sub-frame's tweaked gain
SB_HD i32 shape_avg_gain_q16(i32 avgGain_Q16, i32 gain_Q16, i32 speech_activity_Q8) {
    return add_sat32(avgGain_Q16, smulwb(gain_Q16 - avgGain_Q16, rshift_round(smulbb(speech_activity_Q8, SB_FIXC(1e-3f, 10)), 2)));
}
// de-essing factor: fs == 8 kHz takes no branch (:438-457), so it is the pre-gain multiplier alone
SB_HD i32 shape_pregain_mult_q16(i32 coding_quality_Q14) {
    return SB_FIXC(1.0, 16) + rshift_round(mlaw(SB_FIXC(0.05f, 26), coding_quality_Q14, SB_FIXC(0.1f, 12)), 10);
}
// low-frequency shaping of a sub-frame with pitch lag pitchL (voiced; the same for every sub-frame when unvoiced) (:459-477)
SB_HD i32 shape_lf_shp_q14(int sigtype, i32 pitchL, i32 input_quality_band0_Q15) {
    const i32 strength_Q16 = mulw(SB_FIXC(3.0f, 0), SB_FIXC(1.0, 16) + smulbb(SB_FIXC(0.5f, 1), input_quality_band0_Q15 - SB_FIXC(1.0, 15)));
    i32 b_Q14, LF_shp_Q14;
    if (sigtype == 0) {
        b_Q14 = SB_FIXC(0.2, 14) / 8 + SB_FIXC(3.0, 14) / imax(pitchL, 1);
        LF_shp_Q14 = shl(SB_FIXC(1.0, 14) - b_Q14 - smulwb(strength_Q16, b_Q14), 16);
    } else {
        b_Q14 = 21299 / 8;
        LF_shp_Q14 = shl(SB_FIXC(1.0, 14) - b_Q14 - smulwb(strength_Q16, smulwb(SB_FIXC(0.6, 16), b_Q14)), 16);
    }
    return LF_shp_Q14 | (u16)(b_Q14 - SB_FIXC(1.0, 14));
}
// targets of the three smoothed shaping parameters (:470-505)
struct HarmTilt { i32 HarmBoost_Q16, HarmShapeGain_Q16, Tilt_Q16; };
SB_HD HarmTilt shape_harm_tilt(int sigtype, i32 speech_activity_Q8, i32 input_quality_Q14, i32 coding_quality_Q14, i32 LTPCorr_Q15) {
    HarmTilt h;
    h.HarmBoost_Q16 = smulwb(smulwb(SB_FIXC(1.0, 17) - shl(coding_quality_Q14, 3), LTPCorr_Q15), SB_FIXC(0.1f, 16));
    h.HarmBoost_Q16 = smlawb(h.HarmBoost_Q16, SB_FIXC(1.0, 16) - shl(input_quality_Q14, 2), SB_FIXC(0.1f, 16));
    h.HarmShapeGain_Q16 = 0;
    h.Tilt_Q16 = -SB_FIXC(0.3f, 16);
    if (sigtype == 0) {
        h.Tilt_Q16 -= smulwb(SB_FIXC(1.0, 16) - SB_FIXC(0.3f, 16), smulwb(SB_FIXC(0.35f, 24), speech_activity_Q8));
        h.HarmShapeGain_Q16 = smlawb(SB_FIXC(0.3f, 16),
            SB_FIXC(1.0, 16) - smulwb(SB_FIXC(1.0, 18) - shl(coding_quality_Q14, 4), input_quality_Q14), SB_FIXC(0.2f, 16));
        h.HarmShapeGain_Q16 = smulwb(shl(h.HarmShapeGain_Q16, 1), sqrt_approx(shl(LTPCorr_Q15, 15)));
    }
    return h;
}
// one sub-frame step of a smoothed parameter (state Q16) towards its target; returns the sub-frame's Q14 value
SB_HD i32 shape_smooth_q14(i32& smth_Q16, i32 target_Q16) {
    smth_Q16 = smlawb(smth_Q16, target_Q16 - smth_Q16, SB_FIXC(0.4f, 16));
    return rshift_round(smth_Q16, 2);
}

// pitch_res points at res_pitch + FRAME, x at x_buf + FRAME.  Stops, as the analysis kernel does, after the bandwidth
// expansion of each window: ar_Q24[k] = {AR2, AR1} and shape_par = {warping_Q16, de-essing multiplier Q16} go to
// shape_post_window, which finishes the filters and the pre-gains.
SB_FN void noise_shape_analysis(EncSilk* st, EncCtrl* c, const i16* pitch_res, const i16* x, i32 (*ar_Q24)[2][SHAPE_ORDER], i32* shape_par) {
    i32 auto_corr[SHAPE_ORDER + 1], AR1_Q24[SHAPE_ORDER], AR2_Q24[SHAPE_ORDER];
    i16 x_windowed[SHAPE_WIN];
    i32 scale = 0, nrg;
    const i16* x_ptr = x - LA_SHAPE;

    // sparseness of the unvoiced residual
    i32 energy_variation_Q7 = 0;
    if (c->sigtype != 0) {
        const int nSamples = 16;
        i32 log_energy_prev_Q7 = 0;
        const i16* pr = pitch_res;
        for (int k = 0; k < 10; k++) {
            sum_sqr_shift(&nrg, &scale, pr, nSamples, 0);
            nrg += nSamples >> scale;
            i32 log_energy_Q7 = lin2log(nrg);
            if (k > 0) energy_variation_Q7 += iabs(log_energy_Q7 - log_energy_prev_Q7);
            log_energy_prev_Q7 = log_energy_Q7;
            pr += nSamples;
        }
    }
    const ShapeCtl s = shape_control(c->sigtype, st->SNR_dB_Q7, st->SNRPerMD_dB_Q7, c->input_quality_bands_Q15, st->speech_activity_Q8,
                                     st->LTPCorr_Q15, energy_variation_Q7, c->predGain_Q16);
    c->current_SNR_dB_Q7 = st->SNR_dB_Q7;
    c->current_SNRPerMD_dB_Q7 = st->SNRPerMD_dB_Q7;
    c->input_quality_Q14 = s.input_quality_Q14;
    c->coding_quality_Q14 = s.coding_quality_Q14;
    c->sparseness_Q8 = s.sparseness_Q8;
    c->QuantOffsetType = s.QuantOffsetType;

    for (int k = 0; k < NB_SUBFR; k++) {
        const int flat_part = 40, slope_part = (SHAPE_WIN - 40) >> 1;
        apply_sine_window(x_windowed, x_ptr, 1, slope_part);
        for (int i = 0; i < flat_part; i++) x_windowed[slope_part + i] = x_ptr[slope_part + i];
        apply_sine_window(x_windowed + slope_part + flat_part, x_ptr + slope_part + flat_part, 2, slope_part);
        x_ptr += SUBFR;
        warped_autocorrelation(auto_corr, &scale, x_windowed, s.warping_Q16, SHAPE_WIN, SHAPE_ORDER);
        c->Gains_Q16[k] = shape_window(AR2_Q24, AR1_Q24, auto_corr, scale, s.warping_Q16, s.BWExp1_Q16, s.BWExp2_Q16);
        for (int i = 0; i < SHAPE_ORDER; i++) { ar_Q24[k][0][i] = AR2_Q24[i]; ar_Q24[k][1][i] = AR1_Q24[i]; }
    }

    const i32 md_gain_mult_Q16 = shape_gain_mult_q16(s.md_SNR_adj_dB_Q7);
    const i32 gain_mult_Q16 = shape_gain_mult_q16(s.SNR_adj_dB_Q7);
    c->md_delta_gain_par = (float)gain_mult_Q16 / (float)md_gain_mult_Q16;
    const i32 gain_add_Q16 = shape_gain_add_q16(st->avgGain_Q16);
    for (int k = 0; k < NB_SUBFR; k++) {
        c->Gains_Q16[k] = shape_gain_tweak(c->Gains_Q16[k], gain_mult_Q16, gain_add_Q16);
        st->avgGain_Q16 = shape_avg_gain_q16(st->avgGain_Q16, c->Gains_Q16[k], st->speech_activity_Q8);
    }
    shape_par[0] = s.warping_Q16;
    shape_par[1] = shape_pregain_mult_q16(s.coding_quality_Q14);

    const HarmTilt h = shape_harm_tilt(c->sigtype, st->speech_activity_Q8, s.input_quality_Q14, s.coding_quality_Q14, st->LTPCorr_Q15);
    for (int k = 0; k < NB_SUBFR; k++) {
        c->LF_shp_Q14[k] = shape_lf_shp_q14(c->sigtype, c->pitchL[k], c->input_quality_bands_Q15[0]);
        c->HarmBoost_Q14[k] = shape_smooth_q14(st->HarmBoost_smth_Q16, h.HarmBoost_Q16);
        c->HarmShapeGain_Q14[k] = shape_smooth_q14(st->HarmShapeGain_smth_Q16, h.HarmShapeGain_Q16);
        c->Tilt_Q14[k] = shape_smooth_q14(st->Tilt_smth_Q16, h.Tilt_Q16);
    }
}

// ---- SKP_Silk_prefilter_FIX.c:43-82 (warped LPC analysis filter, order 16) ------------------------------------
SB_FN void warped_lpc_analysis_filter(i32* state, i16* res, const i16* coef_Q13, const i16* input, i32 lambda_Q16, int length) {
    i32 sv[SHAPE_ORDER + 1], cq[SHAPE_ORDER];      // register copies: state and coefficients do not change place during the call
#pragma unroll
    for (int i = 0; i <= SHAPE_ORDER; i++) sv[i] = state[i];
#pragma unroll
    for (int i = 0; i < SHAPE_ORDER; i++) cq[i] = coef_Q13[i];
    for (int n = 0; n < length; n++) {
        const i32 xin = input[n];
        i32 tmp2 = smlawb(sv[0], sv[1], lambda_Q16);
        sv[0] = shl(xin, 14);
        i32 tmp1 = smlawb(sv[1], subw(sv[2], tmp2), lambda_Q16);
        sv[1] = tmp2;
        i32 acc_Q11 = smulwb(tmp2, cq[0]);
#pragma unroll
        for (int i = 2; i < SHAPE_ORDER; i += 2) {
            tmp2 = smlawb(sv[i], subw(sv[i + 1], tmp1), lambda_Q16);
            sv[i] = tmp1;
            acc_Q11 = smlawb(acc_Q11, tmp1, cq[i - 1]);
            tmp1 = smlawb(sv[i + 1], subw(sv[i + 2], tmp2), lambda_Q16);
            sv[i + 1] = tmp2;
            acc_Q11 = smlawb(acc_Q11, tmp2, cq[i]);
        }
        sv[SHAPE_ORDER] = tmp1;
        acc_Q11 = smlawb(acc_Q11, tmp1, cq[SHAPE_ORDER - 1]);
        res[n] = (i16)sat16(xin - rshift_round(acc_Q11, 11));
    }
#pragma unroll
    for (int i = 0; i <= SHAPE_ORDER; i++) state[i] = sv[i];
}

// ---- SKP_Silk_prefilter_FIX.c:85-224 -------------------------------------------------------------------
struct PrefState {      // the prefilter's part of EncSilk
    i16 pf_sLTP_shp[LTP_BUF];
    i32 pf_sAR_shp[SHAPE_ORDER + 1];
    i32 pf_sLTP_shp_buf_idx, pf_sLF_AR_shp_Q12, pf_sLF_MA_shp_Q12, pf_sHarmHP, pf_lagPrev;
};
SB_FN void prefilter(PrefState* st, const EncCtrl* c, i16* xw, const i16* x) {
    i32 x_filt_Q12[SUBFR];
    i16 st_res[SUBFR];
    const i16* px = x;
    i16* pxw = xw;
    i32 lag = st->pf_lagPrev;
    for (int k = 0; k < NB_SUBFR; k++) {
        if (c->sigtype == 0) lag = c->pitchL[k];
        i32 HarmShapeGain_Q12 = smulwb(c->HarmShapeGain_Q14[k], 16384 - c->HarmBoost_Q14[k]);
        i32 HarmShapeFIRPacked_Q12 = HarmShapeGain_Q12 >> 2;
        HarmShapeFIRPacked_Q12 |= shl(HarmShapeGain_Q12 >> 1, 16);
        i32 Tilt_Q14 = c->Tilt_Q14[k];
        i32 LF_shp_Q14 = c->LF_shp_Q14[k];
        warped_lpc_analysis_filter(st->pf_sAR_shp, st_res, &c->AR1_Q13[k * SHAPE_ORDER], px, WARPING_Q16, SUBFR);
        i32 B0 = rshift_round(c->GainsPre_Q14[k], 2);
        i32 tmp_32 = smlabb(SB_FIXC(0.05f, 26), c->HarmBoost_Q14[k], HarmShapeGain_Q12);
        tmp_32 = smlabb(tmp_32, c->coding_quality_Q14, SB_FIXC(0.1f, 12));
        tmp_32 = smulwb(tmp_32, -c->GainsPre_Q14[k]);
        tmp_32 = rshift_round(tmp_32, 12);
        i32 B1 = sat16(tmp_32);
        x_filt_Q12[0] = smlabb(smulbb(st_res[0], B0), st->pf_sHarmHP, B1);
        for (int j = 1; j < SUBFR; j++) x_filt_Q12[j] = smlabb(smulbb(st_res[j], B0), st_res[j - 1], B1);
        st->pf_sHarmHP = st_res[SUBFR - 1];
        // SKP_Silk_prefilt_FIX (:174-224)
        {
            i16* LTP_shp_buf = st->pf_sLTP_shp;
            i32 idx0 = st->pf_sLTP_shp_buf_idx;
            i32 sLF_AR = st->pf_sLF_AR_shp_Q12, sLF_MA = st->pf_sLF_MA_shp_Q12;
            for (int i = 0; i < SUBFR; i++) {
                i32 n_LTP_Q12;
                if (lag > 0) {
                    i32 idx = lag + idx0;
                    n_LTP_Q12 = smulbb(LTP_shp_buf[(idx - 2) & LTP_MASK], HarmShapeFIRPacked_Q12);
                    n_LTP_Q12 = smlabt(n_LTP_Q12, LTP_shp_buf[(idx - 1) & LTP_MASK], HarmShapeFIRPacked_Q12);
                    n_LTP_Q12 = smlabb(n_LTP_Q12, LTP_shp_buf[(idx) & LTP_MASK], HarmShapeFIRPacked_Q12);
                } else n_LTP_Q12 = 0;
                i32 n_Tilt_Q10 = smulwb(sLF_AR, Tilt_Q14);
                i32 n_LF_Q10 = smlawb(smulwt(sLF_AR, LF_shp_Q14), sLF_MA, LF_shp_Q14);
                sLF_AR = subw(x_filt_Q12[i], shl(n_Tilt_Q10, 2));
                sLF_MA = subw(sLF_AR, shl(n_LF_Q10, 2));
                idx0 = (idx0 - 1) & LTP_MASK;
                LTP_shp_buf[idx0] = (i16)sat16(rshift_round(sLF_MA, 12));
                pxw[i] = (i16)sat16(rshift_round(subw(sLF_MA, n_LTP_Q12), 12));
            }
            st->pf_sLF_AR_shp_Q12 = sLF_AR;
            st->pf_sLF_MA_shp_Q12 = sLF_MA;
            st->pf_sLTP_shp_buf_idx = idx0;
        }
        px += SUBFR;
        pxw += SUBFR;
    }
    st->pf_lagPrev = c->pitchL[NB_SUBFR - 1];
}

// ---- after the analysis kernel (device: two thread-per-instance kernels; scalar recursions at full lane efficiency) ----
// (1) one shaping window: inverse prediction gains of AR2 / AR1 -> GainsPre, coefficient limiting, Q13 coefficients
//     (noise_shape_analysis_FIX.c:392-415; the analysis kernel stops after the bandwidth expansion of the window)
SB_FN void shape_post_window(EncScratch* scr, int f, int k) {
    i32 AR1_Q24[SHAPE_ORDER], AR2_Q24[SHAPE_ORDER];
    for (int i = 0; i < SHAPE_ORDER; i++) { AR2_Q24[i] = scr->ar_Q24[f][k][0][i]; AR1_Q24[i] = scr->ar_Q24[f][k][1][i]; }
    i32 pre_nrg_Q30, nrg;
    lpc_inv_pred_gain_q24(&pre_nrg_Q30, AR2_Q24, SHAPE_ORDER);
    lpc_inv_pred_gain_q24(&nrg, AR1_Q24, SHAPE_ORDER);
    pre_nrg_Q30 = shl(smulwb(pre_nrg_Q30, SB_FIXC(0.7, 15)), 1);
    const i32 gains_pre = SB_FIXC(0.3, 14) + div32_varq(pre_nrg_Q30, nrg, 14);
    limit_warped_coefs(AR2_Q24, AR1_Q24, scr->shape_par[f][0], SB_FIXC(3.999, 24), SHAPE_ORDER);
    EncCtrl* c = &scr->c[f];
    for (int i = 0; i < SHAPE_ORDER; i++) {
        c->AR1_Q13[k * SHAPE_ORDER + i] = (i16)sat16(rshift_round(AR1_Q24[i], 11));
        c->AR2_Q13[k * SHAPE_ORDER + i] = (i16)sat16(rshift_round(AR2_Q24[i], 11));
    }
    c->GainsPre_Q14[k] = smulwb(scr->shape_par[f][1], gains_pre);
}
// (2) the prefilter of every frame of the packet (its output feeds only the quantiser)
SB_FN void prefilter_packet(EncSilk* st, EncScratch* scr, int nf) {
    PrefState ps;        // thread-private copy: on the device the recursion then runs out of registers / local memory
    for (int i = 0; i < LTP_BUF; i++) ps.pf_sLTP_shp[i] = st->pf_sLTP_shp[i];
    for (int i = 0; i <= SHAPE_ORDER; i++) ps.pf_sAR_shp[i] = st->pf_sAR_shp[i];
    ps.pf_sLTP_shp_buf_idx = st->pf_sLTP_shp_buf_idx; ps.pf_sLF_AR_shp_Q12 = st->pf_sLF_AR_shp_Q12; ps.pf_sLF_MA_shp_Q12 = st->pf_sLF_MA_shp_Q12;
    ps.pf_sHarmHP = st->pf_sHarmHP; ps.pf_lagPrev = st->pf_lagPrev;
    for (int f = 0; f < nf; f++) prefilter(&ps, &scr->c[f], scr->xfw[f], scr->x_hp[f]);
    for (int i = 0; i < LTP_BUF; i++) st->pf_sLTP_shp[i] = ps.pf_sLTP_shp[i];
    for (int i = 0; i <= SHAPE_ORDER; i++) st->pf_sAR_shp[i] = ps.pf_sAR_shp[i];
    st->pf_sLTP_shp_buf_idx = ps.pf_sLTP_shp_buf_idx; st->pf_sLF_AR_shp_Q12 = ps.pf_sLF_AR_shp_Q12; st->pf_sLF_MA_shp_Q12 = ps.pf_sLF_MA_shp_Q12;
    st->pf_sHarmHP = ps.pf_sHarmHP; st->pf_lagPrev = ps.pf_lagPrev;
}

}  // namespace sb
