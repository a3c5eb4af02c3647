// solo_b200 -- prediction analysis of one 20 ms frame: LTP, Burg LPC, NLSF interpolation search,
// NLSF multi-stage VQ, residual energies, gain processing and quantisation.
// Reference paths relative to /root/reference/JC1_SDK_SRC_ARM/src/libSATECodec/.
#pragma once
#include "sb_sigproc.cuh"
#include "sb_state.cuh"

namespace sb {

// ---- SKP_Silk_corrMatrix_FIX.c:35-68 (order 5, L 40) ------------------------------------------------------
SB_FN void corr_vector(const i16* x, const i16* t, int L, int order, i32* Xt, int rshifts) {
    const i16* ptr1 = &x[order - 1];
    if (rshifts > 0) {
        for (int lag = 0; lag < order; lag++) {
            i32 ip = 0;
            for (int i = 0; i < L; i++) ip = addw(ip, smulbb(ptr1[i], t[i]) >> rshifts);
            Xt[lag] = ip;
            ptr1--;
        }
    } else {
        for (int lag = 0; lag < order; lag++) { Xt[lag] = inner_prod16(ptr1, t, L); ptr1--; }
    }
}
// ---- SKP_Silk_corrMatrix_FIX.c:71-153; x_odd = parity of x's element offset (sum_sqr_shift alignment path)
SB_FN void corr_matrix(const i16* x, int L, int order, int head_room, i32* XX, i32* rshifts, int x_odd) {
    i32 energy, rshifts_local;
    sum_sqr_shift(&energy, &rshifts_local, x, L + order - 1, x_odd);
    int hr = imax(head_room - clz32(energy), 0);
    energy = energy >> hr;
    rshifts_local += hr;
    for (int i = 0; i < order - 1; i++) energy = subw(energy, smulbb(x[i], x[i]) >> rshifts_local);
    if (rshifts_local < *rshifts) { energy = energy >> (*rshifts - rshifts_local); rshifts_local = *rshifts; }
    XX[0] = energy;
    const i16* ptr1 = &x[order - 1];
    for (int j = 1; j < order; j++) {
        energy = subw(energy, smulbb(ptr1[L - j], ptr1[L - j]) >> rshifts_local);
        energy = addw(energy, smulbb(ptr1[-j], ptr1[-j]) >> rshifts_local);
        XX[j * order + j] = energy;
    }
    const i16* ptr2 = &x[order - 2];
    if (rshifts_local > 0) {
        for (int lag = 1; lag < order; lag++) {
            energy = 0;
            for (int i = 0; i < L; i++) energy = addw(energy, smulbb(ptr1[i], ptr2[i]) >> rshifts_local);
            XX[lag * order + 0] = energy;
            XX[0 * order + lag] = energy;
            for (int j = 1; j < order - lag; j++) {
                energy = subw(energy, smulbb(ptr1[L - j], ptr2[L - j]) >> rshifts_local);
                energy = addw(energy, smulbb(ptr1[-j], ptr2[-j]) >> rshifts_local);
                XX[(lag + j) * order + j] = energy;
                XX[j * order + lag + j] = energy;
            }
            ptr2--;
        }
    } else {
        for (int lag = 1; lag < order; lag++) {
            energy = inner_prod16(ptr1, ptr2, L);
            XX[lag * order + 0] = energy;
            XX[0 * order + lag] = energy;
            for (int j = 1; j < order - lag; j++) {
                energy = subw(energy, smulbb(ptr1[L - j], ptr2[L - j]));
                energy = smlabb(energy, ptr1[-j], ptr2[-j]);
                XX[(lag + j) * order + j] = energy;
                XX[j * order + lag + j] = energy;
            }
            ptr2--;
        }
    }
    *rshifts = rshifts_local;
}

// ---- SKP_Silk_solve_LS_FIX.c:41-241 (M = 5) -----------------------------------------------------------------
SB_FN void solve_ldl5(i32* A, const i32* b, i32* x_Q16) {
    const int M = 5;
    i32 L_Q16[M * M], Y[M], invD_Q36[M], invD_Q48[M], v_Q0[M], D_Q0[M];
    i32 diag_min_value = imax(smmul(add_sat32(A[0], A[M * M - 1]), SB_FIXC(1e-5f, 31)), 1 << 9);
    int status = 1;
    for (int loop = 0; loop < M && status == 1; loop++) {
        status = 0;
        for (int j = 0; j < M; j++) {
            const i32* ptr1 = &L_Q16[j * M];
            i32 tmp_32 = 0;
            for (int i = 0; i < j; i++) {
                v_Q0[i] = smulww(D_Q0[i], ptr1[i]);
                tmp_32 = smlaww(tmp_32, v_Q0[i], ptr1[i]);
            }
            tmp_32 = subw(A[j * M + j], tmp_32);
            if (tmp_32 < diag_min_value) {
                tmp_32 = subw(smulbb(loop + 1, diag_min_value), tmp_32);
                for (int i = 0; i < M; i++) A[i * M + i] = addw(A[i * M + i], tmp_32);
                status = 1;
                break;
            }
            D_Q0[j] = tmp_32;
            i32 q36 = inverse32_varq(tmp_32, 36);
            i32 q40 = shl(q36, 4);
            i32 err = subw(1 << 24, smulww(tmp_32, q40));
            i32 q48 = smulww(err, q40);
            invD_Q36[j] = q36;
            invD_Q48[j] = q48;
            L_Q16[j * M + j] = 65536;
            ptr1 = &A[j * M];
            const i32* ptr2 = &L_Q16[(j + 1) * M];
            for (int i = j + 1; i < M; i++) {
                tmp_32 = 0;
                for (int k = 0; k < j; k++) tmp_32 = smlaww(tmp_32, v_Q0[k], ptr2[k]);
                tmp_32 = subw(ptr1[i], tmp_32);
                L_Q16[i * M + j] = addw(smmul(tmp_32, q48), smulww(tmp_32, q36) >> 4);
                ptr2 += M;
            }
        }
    }
    // L*Y = b
    for (int i = 0; i < M; i++) {
        i32 t = 0;
        for (int j = 0; j < i; j++) t = smlaww(t, L_Q16[i * M + j], Y[j]);
        Y[i] = subw(b[i], t);
    }
    for (int i = 0; i < M; i++) {
        i32 t = Y[i];
        Y[i] = addw(smmul(t, invD_Q48[i]), smulww(t, invD_Q36[i]) >> 4);
    }
    for (int i = M - 1; i >= 0; i--) {
        i32 t = 0;
        for (int j = M - 1; j > i; j--) t = smlaww(t, L_Q16[j * M + i], x_Q16[j]);
        x_Q16[i] = subw(Y[i], t);
    }
}

// ---- SKP_Silk_residual_energy16_FIX.c:31-103 (D = 5, cQ = 14) ---------------------------------------------
SB_FN i32 residual_energy16_covar(const i16* c, const i32* wXX, const i32* wXx, i32 wxx) {
    const int D = 5, cQ = 14;
    int lshifts = 16 - cQ, Qxtra = lshifts;
    i32 c_max = 0, cn[5];
    for (int i = 0; i < D; i++) c_max = imax(c_max, iabs((i32)c[i]));
    Qxtra = imin(Qxtra, clz32(c_max) - 17);
    i32 w_max = imax(wXX[0], wXX[D * D - 1]);
    Qxtra = imin(Qxtra, clz32(mulw(D, smulwb(w_max, c_max) >> 4)) - 5);
    Qxtra = imax(Qxtra, 0);
    for (int i = 0; i < D; i++) cn[i] = shl((i32)c[i], Qxtra);
    lshifts -= Qxtra;
    i32 tmp = 0;
    for (int i = 0; i < D; i++) tmp = smlawb(tmp, wXx[i], cn[i]);
    i32 nrg = subw(wxx >> (1 + lshifts), tmp);
    i32 tmp2 = 0;
    for (int i = 0; i < D; i++) {
        tmp = 0;
        const i32* pRow = &wXX[i * D];
        for (int j = i + 1; j < D; j++) tmp = smlawb(tmp, pRow[j], cn[j]);
        tmp = smlawb(tmp, pRow[i] >> 1, cn[i]);
        tmp2 = smlawb(tmp2, tmp, cn[i]);
    }
    nrg = addw(nrg, shl(tmp2, lshifts));
    if (nrg < 1) nrg = 1;
    else if (nrg > (SB_I32_MAX >> (lshifts + 2))) nrg = SB_I32_MAX >> 1;
    else nrg = shl(nrg, lshifts + 1);
    return nrg;
}

// ---- SKP_Silk_find_LTP_FIX.c:39-231 -----------------------------------------------------------------------
// r_first == res_pitch (element offset 0 of a 4-byte aligned buffer), r_last == res_pitch + FRAME/2.
// Split in two so that the cooperative kernel can run the four sub-frames on four lanes: the body of the sub-frame loop
// (:67-148) and the part that couples the sub-frames (:150-231).
struct LtpSubfr { i32 rr, nrg, w, corr_rshifts; };
SB_FN void find_ltp_subfr(int k, i16* b_Q14_ptr, i32* WLTP_ptr, LtpSubfr* o, const i16* r_first, const i16* r_last, i32 lag_k, i32 Wght_Q15_k) {
    const int HEAD = 2;
    i32 b_Q16[LTP_ORDER], Rr[LTP_ORDER];
    const i16* r_ptr = (k < (NB_SUBFR >> 1) ? &r_first[FRAME] : &r_last[FRAME] - (NB_SUBFR >> 1) * SUBFR) + k * SUBFR;
    const i16* lag_ptr = r_ptr - (lag_k + LTP_ORDER / 2);
    i32 rr, rr_shifts;
    sum_sqr_shift(&rr, &rr_shifts, r_ptr, SUBFR, 0);
    int LZs = clz32(rr);
    if (LZs < HEAD) { rr = rshift_round(rr, HEAD - LZs); rr_shifts += (HEAD - LZs); }
    i32 corr_rshifts = rr_shifts;
    corr_matrix(lag_ptr, SUBFR, LTP_ORDER, HEAD, WLTP_ptr, &corr_rshifts, lag_k & 1);
    corr_vector(lag_ptr, r_ptr, SUBFR, LTP_ORDER, Rr, corr_rshifts);
    if (corr_rshifts > rr_shifts) rr = rr >> (corr_rshifts - rr_shifts);
    i32 regu = 1;
    regu = smlawb(regu, rr, SB_FIXC(0.01f / 3, 16));
    regu = smlawb(regu, WLTP_ptr[0], SB_FIXC(0.01f / 3, 16));
    regu = smlawb(regu, WLTP_ptr[(LTP_ORDER - 1) * LTP_ORDER + LTP_ORDER - 1], SB_FIXC(0.01f / 3, 16));
    for (int i = 0; i < LTP_ORDER; i++) WLTP_ptr[i * LTP_ORDER + i] = addw(WLTP_ptr[i * LTP_ORDER + i], regu);
    rr = addw(rr, regu);
    solve_ldl5(WLTP_ptr, Rr, b_Q16);
    for (int i = 0; i < LTP_ORDER; i++) b_Q14_ptr[i] = (i16)sat16(rshift_round(b_Q16[i], 2));
    const i32 nrg = residual_energy16_covar(b_Q14_ptr, WLTP_ptr, Rr, rr);
    int extra_shifts = imin(corr_rshifts, HEAD);
    i32 denom32 = addw(lshift_sat32(smulwb(nrg, Wght_Q15_k), 1 + extra_shifts), smulwb(SUBFR, 655) >> (corr_rshifts - extra_shifts));
    denom32 = imax(denom32, 1);
    i32 temp32 = shl(Wght_Q15_k, 16) / denom32;
    temp32 = temp32 >> (31 + corr_rshifts - extra_shifts - 26);
    i32 WLTP_max = 0;
    for (int i = 0; i < LTP_ORDER * LTP_ORDER; i++) WLTP_max = imax(WLTP_ptr[i], WLTP_max);
    int lshift = clz32(WLTP_max) - 1 - 3;
    if (26 - 18 + lshift < 31) temp32 = imin(temp32, shl(1, 26 - 18 + lshift));
    for (int i = 0; i < LTP_ORDER * LTP_ORDER; i++) WLTP_ptr[i] = (i32)(smull(WLTP_ptr[i], temp32) >> 8);
    o->rr = rr; o->nrg = nrg; o->corr_rshifts = corr_rshifts;
    o->w = WLTP_ptr[(LTP_ORDER >> 1) * LTP_ORDER + (LTP_ORDER >> 1)];
}
SB_FN void find_ltp_tail(i16* b_Q14, i32* LTPredCodGain_Q7, const LtpSubfr* sf, const i32* Wght_Q15) {
    i32 delta_b_Q14[LTP_ORDER], d_Q14[NB_SUBFR];
    int maxRshifts = 0;
    for (int k = 0; k < NB_SUBFR; k++) maxRshifts = imax(sf[k].corr_rshifts, maxRshifts);
    {
        i32 LPC_LTP_res_nrg = 0, LPC_res_nrg = 0;
        for (int k = 0; k < NB_SUBFR; k++) {
            LPC_res_nrg = addw(LPC_res_nrg, addw(smulwb(sf[k].rr, Wght_Q15[k]), 1) >> (1 + (maxRshifts - sf[k].corr_rshifts)));
            LPC_LTP_res_nrg = addw(LPC_LTP_res_nrg, addw(smulwb(sf[k].nrg, Wght_Q15[k]), 1) >> (1 + (maxRshifts - sf[k].corr_rshifts)));
        }
        LPC_LTP_res_nrg = imax(LPC_LTP_res_nrg, 1);
        i32 div_Q16 = div32_varq(LPC_res_nrg, LPC_LTP_res_nrg, 16);
        *LTPredCodGain_Q7 = smulbb(3, lin2log(div_Q16) - (16 << 7));
    }
    i16* b_Q14_ptr = b_Q14;
    for (int k = 0; k < NB_SUBFR; k++) {
        d_Q14[k] = 0;
        for (int i = 0; i < LTP_ORDER; i++) d_Q14[k] += b_Q14_ptr[i];
        b_Q14_ptr += LTP_ORDER;
    }
    i32 max_abs_d_Q14 = 0, max_w_bits = 0;
    for (int k = 0; k < NB_SUBFR; k++) {
        max_abs_d_Q14 = imax(max_abs_d_Q14, iabs(d_Q14[k]));
        max_w_bits = imax(max_w_bits, 32 - clz32(sf[k].w) + sf[k].corr_rshifts - maxRshifts);
    }
    int extra_shifts = max_w_bits + 32 - clz32(max_abs_d_Q14) - 14;
    extra_shifts -= (32 - 1 - 2 + maxRshifts);
    extra_shifts = imax(extra_shifts, 0);
    int maxRshifts_wxtra = maxRshifts + extra_shifts;
    i32 temp32 = (262 >> (maxRshifts + extra_shifts)) + 1;
    i32 wd = 0;
    for (int k = 0; k < NB_SUBFR; k++) {
        temp32 = addw(temp32, sf[k].w >> (maxRshifts_wxtra - sf[k].corr_rshifts));
        wd = addw(wd, shl(smulww(sf[k].w >> (maxRshifts_wxtra - sf[k].corr_rshifts), d_Q14[k]), 2));
    }
    i32 m_Q12 = div32_varq(wd, temp32, 12);
    b_Q14_ptr = b_Q14;
    for (int k = 0; k < NB_SUBFR; k++) {
        if (2 - sf[k].corr_rshifts > 0) temp32 = sf[k].w >> (2 - sf[k].corr_rshifts);
        else temp32 = lshift_sat32(sf[k].w, sf[k].corr_rshifts - 2);
        i32 g_Q26 = mulw(SB_FIXC(0.1f, 26) / ((SB_FIXC(0.1f, 26) >> 10) + temp32),
                         lshift_sat32(sub_sat32(m_Q12, d_Q14[k] >> 2), 4));
        temp32 = 0;
        for (int i = 0; i < LTP_ORDER; i++) {
            delta_b_Q14[i] = b_Q14_ptr[i] > 1638 ? b_Q14_ptr[i] : 1638;
            temp32 += delta_b_Q14[i];
        }
        temp32 = g_Q26 / temp32;
        for (int i = 0; i < LTP_ORDER; i++)
            b_Q14_ptr[i] = (i16)limit((i32)b_Q14_ptr[i] + smulwb(lshift_sat32(temp32, 4), delta_b_Q14[i]), -16000, 28000);
        b_Q14_ptr += LTP_ORDER;
    }
}
SB_FN void find_ltp(i16* b_Q14, i32* WLTP, i32* LTPredCodGain_Q7, const i16* r_first, const i16* r_last, const i32* lag,
                    const i32* Wght_Q15, i32* corr_rshifts) {
    LtpSubfr sf[NB_SUBFR];
    for (int k = 0; k < NB_SUBFR; k++) {
        find_ltp_subfr(k, b_Q14 + k * LTP_ORDER, WLTP + k * LTP_ORDER * LTP_ORDER, &sf[k], r_first, r_last, lag[k], Wght_Q15[k]);
        corr_rshifts[k] = sf[k].corr_rshifts;
    }
    find_ltp_tail(b_Q14, LTPredCodGain_Q7, sf, Wght_Q15);
}

// ---- SKP_Silk_VQ_nearest_neighbor_FIX.c:31-159 (scalar form of the packed arithmetic) -----------------------
// weighted error + rate cost of one code vector (row) for input in_Q14
SB_HD i32 vq_wmat_ec_entry(const i16* in_Q14, const i32* W_Q18, const i16* row, i32 cl_Q6, i32 mu_Q8) {
    i32 d0 = (i16)(in_Q14[0] - row[0]), d1 = (i16)(in_Q14[1] - row[1]), d2 = (i16)(in_Q14[2] - row[2]);
    i32 d3 = (i16)(in_Q14[3] - row[3]), d4 = (i16)(in_Q14[4] - row[4]);
    i32 sum1 = smulbb(mu_Q8, cl_Q6);
    i32 sum2 = smulwb(W_Q18[1], d1);
    sum2 = smlawb(sum2, W_Q18[2], d2);
    sum2 = smlawb(sum2, W_Q18[3], d3);
    sum2 = smlawb(sum2, W_Q18[4], d4);
    sum2 = shl(sum2, 1);
    sum2 = smlawb(sum2, W_Q18[0], d0);
    sum1 = smlawb(sum1, sum2, d0);
    sum2 = smulwb(W_Q18[7], d2);
    sum2 = smlawb(sum2, W_Q18[8], d3);
    sum2 = smlawb(sum2, W_Q18[9], d4);
    sum2 = shl(sum2, 1);
    sum2 = smlawb(sum2, W_Q18[6], d1);
    sum1 = smlawb(sum1, sum2, d1);
    sum2 = smulwb(W_Q18[13], d3);
    sum2 = smlawb(sum2, W_Q18[14], d4);
    sum2 = shl(sum2, 1);
    sum2 = smlawb(sum2, W_Q18[12], d2);
    sum1 = smlawb(sum1, sum2, d2);
    sum2 = smulwb(W_Q18[19], d4);
    sum2 = shl(sum2, 1);
    sum2 = smlawb(sum2, W_Q18[18], d3);
    sum1 = smlawb(sum1, sum2, d3);
    sum2 = smulwb(W_Q18[24], d4);
    sum1 = smlawb(sum1, sum2, d4);
    return sum1;
}
SB_FN void vq_wmat_ec(i32* ind, i32* rate_dist_Q14, const i16* in_Q14, const i32* W_Q18, const i16* cb_Q14, const i16* cl_Q6,
                      i32 mu_Q8, int L) {
    *rate_dist_Q14 = SB_I32_MAX;
    const i16* row = cb_Q14;
    for (int k = 0; k < L; k++) {
        const i32 sum1 = vq_wmat_ec_entry(in_Q14, W_Q18, row, cl_Q6[k], mu_Q8);
        if (sum1 < *rate_dist_Q14) { *rate_dist_Q14 = sum1; *ind = k; }
        row += LTP_ORDER;
    }
}

// ---- SKP_Silk_quant_LTP_gains_FIX.c:30-103 (lowComplexity == 0) ----------------------------------------------
SB_FN void quant_ltp_gains(i16* B_Q14, i32* cbk_index, i32* periodicity_index, const i32* W_Q18, i32 mu_Q8) {
    i32 temp_idx[NB_SUBFR];
    i32 min_rate_dist = SB_I32_MAX;
    for (int k = 0; k < 3; k++) {
        const i16* cl = k == 0 ? SB_T(ltp_bits0_q6) : (k == 1 ? SB_T(ltp_bits1_q6) : SB_T(ltp_bits2_q6));
        const i16* cbk = k == 0 ? SB_T(ltp_vq0_q14) : (k == 1 ? SB_T(ltp_vq1_q14) : SB_T(ltp_vq2_q14));
        int cbk_size = SB_T(ltp_vq_sizes)[k];
        i32 rate_dist = 0;
        for (int j = 0; j < NB_SUBFR; j++) {
            i32 rd;
            vq_wmat_ec(&temp_idx[j], &rd, B_Q14 + j * LTP_ORDER, W_Q18 + j * LTP_ORDER * LTP_ORDER, cbk, cl, mu_Q8, cbk_size);
            rate_dist = add_pos_sat32(rate_dist, rd);
        }
        rate_dist = imin(SB_I32_MAX - 1, rate_dist);
        if (rate_dist < min_rate_dist) {
            min_rate_dist = rate_dist;
            for (int j = 0; j < NB_SUBFR; j++) cbk_index[j] = temp_idx[j];
            *periodicity_index = k;
        }
    }
    int p = *periodicity_index;
    const i16* cbk = p == 0 ? SB_T(ltp_vq0_q14) : (p == 1 ? SB_T(ltp_vq1_q14) : SB_T(ltp_vq2_q14));
    for (int j = 0; j < NB_SUBFR; j++)
        for (int k = 0; k < LTP_ORDER; k++) B_Q14[j * LTP_ORDER + k] = cbk[cbk_index[j] * LTP_ORDER + k];
}

// ---- SKP_Silk_LTP_scale_ctrl_FIX.c:39-81 ---------------------------------------------------------------------------
SB_FN void ltp_scale_ctrl(EncSilk* st, EncCtrl* c, int frame_in_packet) {
    st->HPLTPredCodGain_Q7 = imax(c->LTPredCodGain_Q7 - st->prevLTPredCodGain_Q7, 0) + rshift_round(st->HPLTPredCodGain_Q7, 1);
    st->prevLTPredCodGain_Q7 = c->LTPredCodGain_Q7;
    i32 g_out_Q5 = rshift_round((c->LTPredCodGain_Q7 >> 1) + (st->HPLTPredCodGain_Q7 >> 1), 3);
    i32 g_limit_Q15 = sigm_q15(g_out_Q5 - (3 << 5));
    c->LTP_scaleIndex = 0;
    if (frame_in_packet == 0) {
        int round_loss = st->packetLoss_perc + (st->frames_per_packet - 1);
        i32 thrld1 = SB_T(ltpscale_thresholds_q15)[imin(round_loss, 10)];
        i32 thrld2 = SB_T(ltpscale_thresholds_q15)[imin(round_loss + 1, 10)];
        if (g_limit_Q15 > thrld1) c->LTP_scaleIndex = 2;
        else if (g_limit_Q15 > thrld2) c->LTP_scaleIndex = 1;
    }
    c->LTP_scale_Q14 = SB_T(ltpscales_q14)[c->LTP_scaleIndex];
}

// ---- SKP_Silk_LTP_analysis_filter_FIX.c:30-80 --------------------------------------------------------------
// Output i of sub-frame k's block of SUBFR + LPC_ORDER samples, x pointing at the first block's start: the LTP residual
// scaled by the sub-frame's inverse gain.  The analysis kernel computes one output per lane (c_find_pred_coefs).
SB_HD i16 ltp_analysis_sample(const i16* x, const i16* LTPCoef_Q14, const i32* pitchL, const i32* invGains_Q16, int k, int i) {
    const i16* x_ptr = x + k * SUBFR;
    const i16* x_lag_ptr = x_ptr - pitchL[k] + i;
    const i16* B = &LTPCoef_Q14[k * LTP_ORDER];
    i32 est = smulbb(x_lag_ptr[LTP_ORDER / 2], B[0]);
#pragma unroll
    for (int j = 1; j < LTP_ORDER; j++) est = smlabb(est, x_lag_ptr[LTP_ORDER / 2 - j], B[j]);
    est = rshift_round(est, 14);
    const i32 r = sat16((i32)x_ptr[i] - est);
    return (i16)smulwb(invGains_Q16[k], r);
}

// ---- SKP_Silk_find_LPC_FIX.c:32-148 --------------------------------------------------------------------
// The energy comparisons are written once for this scalar model and the analysis kernel (c_find_lpc, sb_coop.cuh).
// Residual energy of the first half: the whole frame's less the second half's, in the coarser of the two Q-domains (:83-93).
SB_HD void lpc_first_half_nrg(i32& res_nrg, i32& res_nrg_Q, i32 res_tmp_nrg, i32 res_tmp_nrg_Q) {
    const int shift = res_tmp_nrg_Q - res_nrg_Q;
    if (shift >= 0) {
        if (shift < 32) res_nrg = subw(res_nrg, res_tmp_nrg >> shift);
    } else {
        res_nrg = subw(res_nrg >> (-shift), res_tmp_nrg);
        res_nrg_Q = res_tmp_nrg_Q;
    }
}
// Interpolation candidate with half-frame residual energies res_nrg0 / res_nrg1 (right shifts rshift0 / rshift1): true,
// and its energy becomes the best, if it is lower than the best so far (:119-140).
SB_HD bool lpc_interp_lower(i32& res_nrg, i32& res_nrg_Q, i32 res_nrg0, i32 rshift0, i32 res_nrg1, i32 rshift1) {
    i32 res_nrg_interp_Q;
    int shift = rshift0 - rshift1;
    if (shift >= 0) { res_nrg1 = res_nrg1 >> shift; res_nrg_interp_Q = -rshift0; }
    else { res_nrg0 = res_nrg0 >> (-shift); res_nrg_interp_Q = -rshift1; }
    const i32 res_nrg_interp = addw(res_nrg0, res_nrg1);
    shift = res_nrg_interp_Q - res_nrg_Q;
    bool lower;
    if (shift >= 0) lower = (res_nrg_interp >> shift) < res_nrg;
    else if (-shift < 32) lower = res_nrg_interp < (res_nrg >> (-shift));
    else lower = false;
    if (lower) { res_nrg = res_nrg_interp; res_nrg_Q = res_nrg_interp_Q; }
    return lower;
}
// x: nb_subfr blocks of subfr_length samples (each with `order` preceding samples); x is 4-byte aligned.
SB_FN void find_lpc(i32* NLSF_Q15, i32* interpIndex, const i32* prev_NLSFq_Q15, int useInterp, int order, const i16* x,
                    int subfr_length) {
    i32 a_Q16[16], a_tmp_Q16[16], NLSF0_Q15[16];
    i16 a_tmp_Q12[16];
    i16 LPC_res[2 * (SUBFR + 16)];
    i32 res_nrg, res_nrg_Q;
    *interpIndex = 4;
    burg_modified(&res_nrg, &res_nrg_Q, a_Q16, x, subfr_length, NB_SUBFR, SB_FIXC(2.5e-5f, 32), order);
    bwexpander_32(a_Q16, order, SB_FIXC(0.99995f, 16));
    if (useInterp == 1) {
        i32 res_tmp_nrg, res_tmp_nrg_Q;
        burg_modified(&res_tmp_nrg, &res_tmp_nrg_Q, a_tmp_Q16, x + (NB_SUBFR >> 1) * subfr_length, subfr_length, NB_SUBFR >> 1,
                      SB_FIXC(2.5e-5f, 32), order);
        bwexpander_32(a_tmp_Q16, order, SB_FIXC(0.99995f, 16));
        lpc_first_half_nrg(res_nrg, res_nrg_Q, res_tmp_nrg, res_tmp_nrg_Q);
        a2nlsf(NLSF_Q15, a_tmp_Q16, order);
        for (int k = 3; k >= 0; k--) {
            interpolate(NLSF0_Q15, prev_NLSFq_Q15, NLSF_Q15, k, order);
            nlsf2a_stable(a_tmp_Q12, NLSF0_Q15, order);
            lpc_analysis_filter_zero_state(x, a_tmp_Q12, LPC_res, 2 * subfr_length, order);
            i32 res_nrg0, res_nrg1, rshift0, rshift1;
            sum_sqr_shift(&res_nrg0, &rshift0, LPC_res + order, subfr_length - order, order & 1);
            sum_sqr_shift(&res_nrg1, &rshift1, LPC_res + order + subfr_length, subfr_length - order, (order + subfr_length) & 1);
            if (lpc_interp_lower(res_nrg, res_nrg_Q, res_nrg0, rshift0, res_nrg1, rshift1)) *interpIndex = k;
        }
    }
    if (*interpIndex == 4) a2nlsf(NLSF_Q15, a_Q16, order);
}

// ---- SKP_Silk_NLSF_MSVQ_encode_FIX.c:33-239 + NLSF_VQ_rate_distortion_FIX.c + NLSF_VQ_sum_error_FIX.c ----------
// (order 10, 6 stages, 16 survivors)
SB_FN void nlsf_msvq_encode(i32* NLSFIndices, i32* pNLSF_Q15, const NlsfCb& cb, const i32* pNLSF_q_Q15_prev, const i32* pW_Q6,
                            i32 NLSF_mu_Q15, i32 NLSF_mu_fluc_red_Q16, int deactivate_fluc_red) {
    enum { SURV = 16, NST = 6, ORD = 10 };
    i32 pRateDist_Q18[SURV];
    i32 log_v[SURV * 16 > 64 ? SURV * 16 : 64];   // candidates that entered the running best-16, in scan order
    i16 log_e[SURV * 16 > 64 ? SURV * 16 : 64];
    // survivor sets of two consecutive stages: ping-pong buffers instead of the reference's copy-back (:224-229)
    i32 rate_buf[2][SURV], pTempIndices[SURV];
    u64 path_buf[2][SURV];           // the six stage indices of a survivor, 8 bits each
    i32 res_buf[2][SURV * ORD];
    i32 *pRate_Q5 = rate_buf[0], *pRate_new_Q5 = rate_buf[1];
    u64 *pPath = path_buf[0], *pPath_new = path_buf[1];
    pPath[0] = 0;
    i32 *pRes_Q15 = res_buf[0], *pRes_new_Q15 = res_buf[1];
    for (int i = 0; i < SURV; i++) pRate_Q5[i] = 0;
    for (int i = 0; i < ORD; i++) pRes_Q15[i] = pNLSF_Q15[i];
    int prev_survivors = 1, cur_survivors = 0;
    const int min_survivors = SURV / 2;
    int cb_off = 0;
    for (int s = 0; s < NST; s++) {
        const int nVec = cb.nvec[s];
        const i16* CB = cb.cb_q15 + cb_off * ORD;
        const i16* Rates = cb.rates_q5 + cb_off;
        cur_survivors = imin(SURV, smulbb(prev_survivors, nVec));
        // Weighted errors + rate cost of every (survivor, code vector) pair and the 16 best of them, equivalent to filling
        // pRateDist_Q18[prev_survivors * nVec] and running SKP_Silk_insertion_sort_increasing over it (sort.c:34-76:
        // ascending, an element goes behind equal values that came earlier).  Written for SIMT execution, where a branch
        // costs every stream of the warp as soon as one stream takes it:
        //   1. the scan keeps only the sorted VALUES of the current best 16 in registers (one min/max pair per slot, no
        //      flags, no indices) and appends every candidate that enters the list to a log;
        //   2. afterwards the log -- in scan order -- is filtered with the final 16th value and the 16 survivors are
        //      insertion-sorted exactly as the reference would sort them.
        // Every element of the final best-16 was below the threshold when it was scanned, so it is in the log.
        i32 ka[SURV];
#pragma unroll
        for (int j = 0; j < SURV; j++) ka[j] = SB_I32_MAX;
        int nlog = 0;
        for (int n = 0; n < prev_survivors; n++) {
            i32 in[ORD];
#pragma unroll
            for (int m = 0; m < ORD; m++) in[m] = pRes_Q15[n * ORD + m];
            const i32 rate_n = pRate_Q5[n];
            const i16* v = CB;
            for (int i = 0; i < nVec; i++) {
                i32 sum_error = 0;
#pragma unroll
                for (int m = 0; m < ORD; m++) {
                    i32 diff = in[m] - (i32)v[m];
                    sum_error = smlawb(sum_error, smulbb(diff, diff), pW_Q6[m]);
                }
                v += ORD;
                const i32 val = smlabb(sum_error, rate_n + Rates[i], NLSF_mu_Q15);
                const int e = n * nVec + i;
                if (e < SURV || val < ka[SURV - 1]) {
                    log_v[nlog] = val; log_e[nlog] = (i16)e; nlog++;
#pragma unroll
                    for (int j = SURV - 1; j >= 1; j--) ka[j] = imin(ka[j], imax(ka[j - 1], val));
                    ka[0] = imin(ka[0], val);
                }
            }
        }
        {
            const i32 T = ka[SURV - 1];
            int need_eq = SURV;                       // how many elements equal to T belong to the best 16
#pragma unroll
            for (int j = 0; j < SURV; j++) need_eq -= (ka[j] < T) ? 1 : 0;
            // compact the 16 survivors (scan order), then place each at its rank: #{(v', pos') < (v, pos)} -- the order an
            // insertion sort with strict comparisons produces
            i32 tv[SURV], te[SURV];
            for (int j = 0; j < SURV; j++) { tv[j] = SB_I32_MAX; te[j] = 0; }
            int m = 0;
            for (int q = 0; q < nlog; q++) {
                const i32 val = log_v[q];
                bool take = val < T;
                if (val == T && need_eq > 0) { take = true; need_eq--; }
                if (take && m < SURV) { tv[m] = val; te[m] = log_e[q]; m++; }
            }
            i32 rv[SURV];
#pragma unroll
            for (int a = 0; a < SURV; a++) rv[a] = tv[a];
#pragma unroll
            for (int a = 0; a < SURV; a++) {
                int rank = 0;
#pragma unroll
                for (int b = 0; b < SURV; b++) rank += (rv[b] < rv[a]) | ((rv[b] == rv[a]) & (b < a));
                pRateDist_Q18[rank] = rv[a]; pTempIndices[rank] = te[a];
            }
        }
        if (pRateDist_Q18[0] < SB_I32_MAX / SURV) {
            i32 thr = smlawb(pRateDist_Q18[0], mulw(SURV, pRateDist_Q18[0]), SB_FIXC(0.1f, 16));
            while (pRateDist_Q18[cur_survivors - 1] > thr && cur_survivors > min_survivors) cur_survivors--;
        }
        for (int k = 0; k < cur_survivors; k++) {
            int input_index, cb_index;
            if (s > 0) {
                if (nVec == 8) { input_index = pTempIndices[k] >> 3; cb_index = pTempIndices[k] & 7; }
                else { input_index = pTempIndices[k] / nVec; cb_index = pTempIndices[k] - smulbb(input_index, nVec); }
            } else { input_index = 0; cb_index = pTempIndices[k]; }
            const i32* __restrict__ pc = &pRes_Q15[input_index * ORD];
            const i16* __restrict__ e = &CB[cb_index * ORD];
            i32* __restrict__ pi = &pRes_new_Q15[k * ORD];
#pragma unroll
            for (int i = 0; i < ORD; i++) pi[i] = pc[i] - (i32)e[i];
            pRate_new_Q5[k] = pRate_Q5[input_index] + Rates[cb_index];
            pPath_new[k] = pPath[input_index] | ((u64)(u32)cb_index << (8 * s));
        }
        if (s < NST - 1) {
            i32* t;
            t = pRes_Q15; pRes_Q15 = pRes_new_Q15; pRes_new_Q15 = t;
            t = pRate_Q5; pRate_Q5 = pRate_new_Q5; pRate_new_Q5 = t;
            { u64* tp = pPath; pPath = pPath_new; pPath_new = tp; }
        }
        prev_survivors = cur_survivors;
        cb_off += nVec;
    }
    int bestIndex = 0;
    if (deactivate_fluc_red != 1) {
        i32 bestRateDist_Q20 = SB_I32_MAX;
        for (int s = 0; s < cur_survivors; s++) {
            i32 idx[NST];
            for (int i = 0; i < NST; i++) idx[i] = (i32)((pPath_new[s] >> (8 * i)) & 0xff);
            nlsf_msvq_decode(pNLSF_Q15, cb, idx);
            i32 wsse_Q20 = 0;
            for (int i = 0; i < ORD; i++) {
                i32 se = pNLSF_Q15[i] - pNLSF_q_Q15_prev[i];
                wsse_Q20 = smlawb(wsse_Q20, smulbb(se, se), pW_Q6[i]);
            }
            wsse_Q20 = add_pos_sat32(pRateDist_Q18[s], smulwb(wsse_Q20, NLSF_mu_fluc_red_Q16));
            if (wsse_Q20 < bestRateDist_Q20) { bestRateDist_Q20 = wsse_Q20; bestIndex = s; }
        }
    }
    for (int i = 0; i < NST; i++) NLSFIndices[i] = (i32)((pPath_new[bestIndex] >> (8 * i)) & 0xff);
    nlsf_msvq_decode(pNLSF_Q15, cb, NLSFIndices);
}

// ---- SKP_Silk_process_NLSFs_FIX.c:31-127 ----------------------------------------------------------------
// Low-latency copies of the two NLSF codebooks (vectors + rates, 4.2 KB): the analysis kernel keeps them in
// shared memory because the MSVQ gathers code vectors by data-dependent index ~1 000 times per frame.
struct NlsfFastTabs {
    i16 cb0[1200], rates0[120], cb1[720], rates1[72];
};
SB_FN void nlsf_fast_tabs_fill(NlsfFastTabs* T, int tid, int nthreads) {
    for (int i = tid; i < 1200; i += nthreads) T->cb0[i] = SB_T(nlsf_cb0_q15)[i];
    for (int i = tid; i < 120; i += nthreads) T->rates0[i] = SB_T(nlsf_cb0_rates_q5)[i];
    for (int i = tid; i < 720; i += nthreads) T->cb1[i] = SB_T(nlsf_cb1_q15)[i];
    for (int i = tid; i < 72; i += nthreads) T->rates1[i] = SB_T(nlsf_cb1_rates_q5)[i];
}
// The rules below are written once for this scalar model and the analysis kernel (c_process_nlsfs, sb_coop.cuh).
// rate weight and fluctuation-reduction weight of the NLSF quantiser (:52-63)
SB_HD void nlsf_mu(i32& NLSF_mu_Q15, i32& NLSF_mu_fluc_red_Q16, int sigtype, i32 speech_activity_Q8, i32 sparseness_Q8) {
    if (sigtype == 0) {
        NLSF_mu_Q15 = smlawb(66, -8388, speech_activity_Q8);
        NLSF_mu_fluc_red_Q16 = smlawb(6554, -838848, speech_activity_Q8);
    } else {
        NLSF_mu_Q15 = smlawb(164, -33554, speech_activity_Q8);
        NLSF_mu_fluc_red_Q16 = smlawb(13107, -1677696, speech_activity_Q8 + sparseness_Q8);
    }
    NLSF_mu_Q15 = imax(NLSF_mu_Q15, 1);
}
// one Laroia weight of the target NLSFs, w_Q6, merged with that of the first half's interpolated NLSFs, w0_Q6 (:71-82)
SB_HD i32 nlsf_interp_weight_q6(i32 w_Q6, i32 w0_Q6, int interpQ2) {
    return smlawb(w_Q6 >> 1, w0_Q6, shl(smulbb(interpQ2, interpQ2), 11));
}
// one quantised NLSF of the first half-frame: interpolated from the previous frame's unless interpQ2 == 4 (:108-118)
SB_HD i32 nlsf_first_half_q15(i32 prev_Q15, i32 q_Q15, int interpQ2) {
    return interpQ2 < (1 << 2) ? prev_Q15 + (mulw(q_Q15 - prev_Q15, interpQ2) >> 2) : q_Q15;
}
// Up to the quantised NLSFs of the two half-frames, nlsf_out = {interpolated first half, second half}; gains_packet turns
// them into the prediction filters (:108-127).
SB_FN void process_nlsfs(EncSilk* st, EncCtrl* c, i32* pNLSF_Q15, i32 (*nlsf_out)[LPC_ORDER]) {
    i32 pNLSFW_Q6[LPC_ORDER], pNLSF0_temp_Q15[LPC_ORDER], pNLSFW0_temp_Q6[LPC_ORDER];
    i32 NLSF_mu_Q15, NLSF_mu_fluc_red_Q16;
    nlsf_mu(NLSF_mu_Q15, NLSF_mu_fluc_red_Q16, c->sigtype, st->speech_activity_Q8, c->sparseness_Q8);
    nlsf_vq_weights_laroia(pNLSFW_Q6, pNLSF_Q15, LPC_ORDER);
    const int interpQ2 = c->NLSFInterpCoef_Q2;
    if (interpQ2 < (1 << 2)) {
        interpolate(pNLSF0_temp_Q15, st->prev_NLSFq_Q15, pNLSF_Q15, interpQ2, LPC_ORDER);
        nlsf_vq_weights_laroia(pNLSFW0_temp_Q6, pNLSF0_temp_Q15, LPC_ORDER);
        for (int i = 0; i < LPC_ORDER; i++) pNLSFW_Q6[i] = nlsf_interp_weight_q6(pNLSFW_Q6[i], pNLSFW0_temp_Q6[i], interpQ2);
    }
    nlsf_msvq_encode(c->NLSFIndices, pNLSF_Q15, nlsf_cb(c->sigtype), st->prev_NLSFq_Q15, pNLSFW_Q6, NLSF_mu_Q15, NLSF_mu_fluc_red_Q16,
                     st->first_frame_after_reset);
    for (int i = 0; i < LPC_ORDER; i++) {
        nlsf_out[1][i] = pNLSF_Q15[i];
        nlsf_out[0][i] = nlsf_first_half_q15(st->prev_NLSFq_Q15[i], pNLSF_Q15[i], interpQ2);
    }
}

// ---- SKP_Silk_residual_energy_FIX.c:32-92 ------------------------------------------------------------------
SB_FN void residual_energy(i32* nrgs, i32* nrgsQ, const i16* x, const i16 a_Q12[2][LPC_ORDER], const i32* gains) {
    const int offset = LPC_ORDER + SUBFR;
    i16 LPC_res[2 * (LPC_ORDER + SUBFR)];
    const i16* x_ptr = x;
    for (int i = 0; i < 2; i++) {
        lpc_analysis_filter_zero_state(x_ptr, a_Q12[i], LPC_res, 2 * offset, LPC_ORDER);
        const i16* p = LPC_res + LPC_ORDER;
        for (int j = 0; j < 2; j++) {
            i32 rshift;
            sum_sqr_shift(&nrgs[i * 2 + j], &rshift, p, SUBFR, 0);
            nrgsQ[i * 2 + j] = -rshift;
            p += offset;
        }
        x_ptr += 2 * offset;
    }
    for (int i = 0; i < NB_SUBFR; i++) {
        int lz1 = clz32(nrgs[i]) - 1;
        int lz2 = clz32(gains[i]) - 1;
        i32 tmp32 = shl(gains[i], lz2);
        tmp32 = smmul(tmp32, tmp32);
        nrgs[i] = smmul(tmp32, shl(nrgs[i], lz1));
        nrgsQ[i] += lz1 + 2 * lz2 - 32 - 32;
    }
}

// ---- SKP_Silk_find_pred_coefs_FIX.c:31-131 -----------------------------------------------------------------
// Up to the quantised NLSFs: frame f's hand-over to gains_packet (nlsf_Q15, lpc_in_pre, local_gains) goes to scr.
SB_FN void find_pred_coefs(EncSilk* st, EncCtrl* c, const i16* res_pitch, EncScratch* scr, int frame_in_packet) {
    i32 WLTP[NB_SUBFR * LTP_ORDER * LTP_ORDER];
    i32 invGains_Q16[NB_SUBFR], Wght_Q15[NB_SUBFR], LTP_corrs_rshift[NB_SUBFR];
    i32 NLSF_Q15[LPC_ORDER];
    i32* local_gains = scr->local_gains[frame_in_packet];
    i16* LPC_in_pre = scr->lpc_in_pre[frame_in_packet];
    // (the analysis kernel states this step separately: as a shared helper it grows the kernel's spill traffic)
    i32 min_gain_Q16 = SB_I32_MAX >> 6;
    for (int i = 0; i < NB_SUBFR; i++) min_gain_Q16 = imin(min_gain_Q16, c->Gains_Q16[i]);
    for (int i = 0; i < NB_SUBFR; i++) {
        invGains_Q16[i] = div32_varq(min_gain_Q16, c->Gains_Q16[i], 16 - 2);
        invGains_Q16[i] = imax(invGains_Q16[i], 363);
        i32 tmp = smulwb(invGains_Q16[i], invGains_Q16[i]);
        Wght_Q15[i] = tmp >> 1;
        local_gains[i] = (1 << 16) / invGains_Q16[i];
    }
    if (c->sigtype == 0) {
        find_ltp(c->LTPCoef_Q14, WLTP, &c->LTPredCodGain_Q7, res_pitch, res_pitch + (FRAME >> 1), c->pitchL, Wght_Q15, LTP_corrs_rshift);
        quant_ltp_gains(c->LTPCoef_Q14, c->LTPIndex, &c->PERIndex, WLTP, SB_FIXC(0.03f, 8));
        ltp_scale_ctrl(st, c, frame_in_packet);
        for (int k = 0; k < NB_SUBFR; k++)
            for (int i = 0; i < SUBFR + LPC_ORDER; i++)
                LPC_in_pre[k * (SUBFR + LPC_ORDER) + i] = ltp_analysis_sample(st->x_buf + FRAME - LPC_ORDER, c->LTPCoef_Q14, c->pitchL, invGains_Q16, k, i);
    } else {
        const i16* x_ptr = st->x_buf + FRAME - LPC_ORDER;
        i16* x_pre_ptr = LPC_in_pre;
        for (int i = 0; i < NB_SUBFR; i++) {
            for (int j = 0; j < SUBFR + LPC_ORDER; j++) x_pre_ptr[j] = (i16)smulwb(invGains_Q16[i], x_ptr[j]);
            x_pre_ptr += SUBFR + LPC_ORDER;
            x_ptr += SUBFR;
        }
        for (int i = 0; i < NB_SUBFR * LTP_ORDER; i++) c->LTPCoef_Q14[i] = 0;
        c->LTPredCodGain_Q7 = 0;
    }
    find_lpc(NLSF_Q15, &c->NLSFInterpCoef_Q2, st->prev_NLSFq_Q15, 1 * (1 - st->first_frame_after_reset), LPC_ORDER, LPC_in_pre,
             SUBFR + LPC_ORDER);
    process_nlsfs(st, c, NLSF_Q15, scr->nlsf_Q15[frame_in_packet]);
    for (int i = 0; i < LPC_ORDER; i++) st->prev_NLSFq_Q15[i] = NLSF_Q15[i];
}

// ---- SKP_Silk_gain_quant.c:42-107 ---------------------------------------------------------------------------
SB_FN void gains_quant(i32* ind, i32* gain_Q16, i32* prev_ind, int conditional, i32* ind2, i32* DeltaGains_Q16) {
    const i32 OFFSET = (6 * 128) / 6 + 16 * 128;
    const i32 SCALE_Q16 = (65536 * (64 - 1)) / (((86 - 6) * 128) / 6);
    const i32 INV_SCALE_Q16 = (65536 * (((86 - 6) * 128) / 6)) / (64 - 1);
    const i32 AlphaDis_Q16 = 32768 / 8;
    i32 inv_gain_Q16 = inverse32_varq(imax(*DeltaGains_Q16, 1), 32);
    inv_gain_Q16 -= 32767;
    *ind2 = 0;
    for (int k = 0; k < 8; k++) {
        if (inv_gain_Q16 > k * AlphaDis_Q16 && inv_gain_Q16 <= (k + 1) * AlphaDis_Q16) {
            *ind2 = k;
            inv_gain_Q16 = (k + 1) * AlphaDis_Q16;
        }
    }
    inv_gain_Q16 += 32767;
    *DeltaGains_Q16 = inverse32_varq(imax(inv_gain_Q16, 1), 32);
    for (int k = 0; k < NB_SUBFR; k++) {
        ind[k] = smulwb(SCALE_Q16, lin2log(gain_Q16[k]) - OFFSET);
        if (ind[k] < *prev_ind) ind[k]++;
        if (k == 0 && conditional == 0) {
            ind[k] = limit(ind[k], 0, 64 - 1);
            ind[k] = imax(ind[k], *prev_ind + -4);
            *prev_ind = ind[k];
        } else {
            ind[k] = limit(ind[k] - *prev_ind, -4, 40);
            *prev_ind += ind[k];
            ind[k] -= -4;
        }
        gain_Q16[k] = log2lin(imin(smulwb(INV_SCALE_Q16, *prev_ind) + OFFSET, 3967));
    }
}

// ---- SKP_Silk_process_gains_FIX.c:32-150 -------------------------------------------------------------------
SB_FN void process_gains(EncSilk* st, EncCtrl* c, int frame_in_packet) {
    if (c->sigtype == 0) {
        i32 s_Q16 = -sigm_q15(rshift_round(c->LTPredCodGain_Q7 - SB_FIXC(12.0, 7), 4));
        for (int k = 0; k < NB_SUBFR; k++) c->Gains_Q16[k] = smlawb(c->Gains_Q16[k], c->Gains_Q16[k], s_Q16);
    }
    i32 InvMaxSqrVal_Q16 = log2lin(smulwb(SB_FIXC(70.0, 7) - c->current_SNR_dB_Q7, SB_FIXC(0.33, 16))) / SUBFR;
    for (int k = 0; k < NB_SUBFR; k++) {
        i32 ResNrg = c->ResNrg[k];
        i32 ResNrgPart = smulww(ResNrg, InvMaxSqrVal_Q16);
        if (c->ResNrgQ[k] > 0) {
            if (c->ResNrgQ[k] < 32) ResNrgPart = rshift_round(ResNrgPart, c->ResNrgQ[k]);
            else ResNrgPart = 0;
        } else if (c->ResNrgQ[k] != 0) {
            if (ResNrgPart > (SB_I32_MAX >> (-c->ResNrgQ[k]))) ResNrgPart = SB_I32_MAX;
            else ResNrgPart = shl(ResNrgPart, -c->ResNrgQ[k]);
        }
        i32 gain = c->Gains_Q16[k];
        i32 gain_squared = add_sat32(ResNrgPart, smmul(gain, gain));
        if (gain_squared < 32767) {
            gain_squared = smlaww(shl(ResNrgPart, 16), gain, gain);
            gain = sqrt_approx(gain_squared);
            c->Gains_Q16[k] = lshift_sat32(gain, 8);
        } else {
            gain = sqrt_approx(gain_squared);
            c->Gains_Q16[k] = lshift_sat32(gain, 16);
        }
    }
    // MD delta gain: three IEEE operations inside the "fixed-point" encoder (App. A Q18); keep them exact
    // (compile with -fmad=false; division is IEEE-correct by default).
    float tmp_float = 1.0f / (float)c->md_delta_gain_par;
    tmp_float = tmp_float * 65536.0f;
    tmp_float = tmp_float > 131072.0f ? 131072.0f : (tmp_float < -131072.0f ? -131072.0f : tmp_float);
    i32 Delta_Gains_Q16 = float2int((double)tmp_float - (0.05 * (double)65536.0f));
    gains_quant(c->GainsIndices, c->Gains_Q16, &st->LastGainIndex, frame_in_packet, &c->DeltaGainsIndices, &Delta_Gains_Q16);
    c->DeltaGains_Q16 = Delta_Gains_Q16;
    if (c->sigtype == 0) {
        if (c->LTPredCodGain_Q7 + (c->input_tilt_Q15 >> 8) > SB_FIXC(1.0, 7)) c->QuantOffsetType = 0;
        else c->QuantOffsetType = 1;
    }
    i32 quant_offset_Q10 = SB_T(quant_offsets_q10)[c->sigtype * 2 + c->QuantOffsetType];
    c->Lambda_Q10 = SB_FIXC(1.2f, 10) + smulbb(SB_FIXC(-0.05f, 10), N_DD) + smulwb(SB_FIXC(-0.3f, 18), st->speech_activity_Q8) +
                    smulwb(SB_FIXC(-0.2f, 12), c->input_quality_Q14) + smulwb(SB_FIXC(-0.1f, 12), c->coding_quality_Q14) +
                    smulwb(SB_FIXC(1.5f, 16), quant_offset_Q10);
}

// ---- after the analysis kernel (device: one thread per stream): what only the quantiser and the entropy coder read ----
// quantised NLSFs -> the two prediction filters (process_NLSFs_FIX.c:108-127), residual energies (residual_energy_FIX.c),
// gain processing and quantisation (process_gains_FIX.c), VAD flag / DTX counter (encode_frame_FIX.c:151-165)
SB_FN void gains_packet(EncSilk* st, EncScratch* scr, int nf) {
    for (int f = 0; f < nf; f++) {
        EncCtrl* c = &scr->c[f];
        for (int k = 0; k < 2; k++) {
            i32 nl[LPC_ORDER];
            i16 a12[LPC_ORDER];
            for (int i = 0; i < LPC_ORDER; i++) nl[i] = scr->nlsf_Q15[f][k][i];
            nlsf2a_stable(a12, nl, LPC_ORDER);
            for (int i = 0; i < LPC_ORDER; i++) c->PredCoef_Q12[k][i] = a12[i];
        }
        i16 x[NB_SUBFR * LPC_ORDER + FRAME];
        i16 a[2][LPC_ORDER];
        i32 lg[NB_SUBFR];
        for (int i = 0; i < NB_SUBFR * LPC_ORDER + FRAME; i++) x[i] = scr->lpc_in_pre[f][i];
        for (int k = 0; k < 2; k++) for (int i = 0; i < LPC_ORDER; i++) a[k][i] = c->PredCoef_Q12[k][i];
        for (int i = 0; i < NB_SUBFR; i++) lg[i] = scr->local_gains[f][i];
        residual_energy(c->ResNrg, c->ResNrgQ, x, a, lg);
        st->speech_activity_Q8 = scr->vad_sa_Q8[f];
        process_gains(st, c, f);
        vad_flag_and_dtx(st, &scr->vadFlag[f]);
    }
    scr->dtx_drop = (st->useDTX && st->inDTX) ? 1 : 0;
}

}  // namespace sb
