// solo_b200 -- one SOLO packet through the decoder (float-build semantics: the PCM parity target).
// Low band: integer SILK decoder (range decode, MD excitation rebuild, LTP + LPC synthesis, PLC, CNG);
// high band: float LPC synthesis of the folded low-band excitation; float QMF synthesis; truncate to int16.
// As on the device, a packet takes two steps: dec_packet (the decode kernel) up to the two band signals, and dec_synth (the
// scalar model of the synthesis kernel, which shares qmf_synth_group) for the filter bank and the int16 output; the host
// model's dec_packet with a PCM output runs both.
// Reference (paths under /root/reference/JC1_SDK_SRC_FLP/src/):
//   libBWE/AGR_BWE_decode_frame_FLP.c:41-232, AGR_BWE_LPC_synthesizer.c:29-52, AGR_BWE_qmf.c:86-182,
//   AGR_BWE_quant_highband.c:114-128, AGR_BWE_SDK_API.c:172-279,
//   libSATECodec/SKP_Silk_dec_API.c:76-189, SKP_Silk_decode_frame.c:57-364, SKP_Silk_decode_parameters.c:31-297,
//   SKP_Silk_decode_pulses.c:33-110, SKP_Silk_shell_coder.c:123-155, SKP_Silk_code_signs.c:64-90,
//   SKP_Silk_decode_pitch.c:34-60, SKP_Silk_decode_core.c:44-213, SKP_Silk_gain_quant.c:110-142,
//   SKP_Silk_PLC.c:43-387, SKP_Silk_CNG.c:31-149, SKP_Silk_LPC_synthesis_filter.c:41-94,
//   SKP_Silk_wrappers_FLP.c:54-73, SKP_Silk_create_init_destroy.c:35-55, SKP_Silk_decoder_set_fs.c:31-86.
// Float code must be compiled without FMA contraction (-fmad=false / -ffp-contract=off).
// A stream may instead follow the reference's fixed-point build (DEC_FIX, per stream in DecState::arith): same low band,
// integer high-band synthesis and integer filter bank (JC1_SDK_SRC_ARM/src/libBWE/AGR_BWE_decode_frame_FIX.c:40-115,
// AGR_BWE_LPC_synthesizer.c:56-136, AGR_BWE_quant_highband.c:106-121, AGR_BWE_qmf.c:86-182 with FIXED_POINT).
// Everything below is templated on the rate of the SILK core, KHZ: 8 for 16 kHz streams (the 8 kHz core, order-10 LPC),
// 16 for 32 kHz streams (the 16 kHz core, order-16 LPC; AGR_BWE_SDK_API.c:196-200 and SKP_Silk_decoder_set_fs.c:40-50).
// The high band of a 32 kHz stream covers 8-16 kHz with the same 8th-order synthesis on frames of the core's length.
#pragma once
#include "sb_rangecoder.cuh"
#include "sb_sigproc.cuh"
#include "sb_state.cuh"

namespace sb {

// SILK core dimensions of a decoder (SKP_Silk_decoder_set_fs.c:37-50): frame and sub-frame length, LPC order
template <int KHZ> struct DecCore {
    static_assert(KHZ == 8 || KHZ == 16, "SOLO streams carry an 8 kHz core (16 kHz API) or a 16 kHz core (32 kHz API)");
    enum { FRAME = 20 * KHZ, SUBFR = 5 * KHZ, LPC_ORDER = KHZ == 8 ? 10 : 16 };
};
// the core dimensions as local constants of a templated routine (they hide the encoder's 8 kHz ones of sb_state.cuh)
#define SB_DEC_DIMS(KHZ) enum { FRAME = DecCore<KHZ>::FRAME, SUBFR = DecCore<KHZ>::SUBFR, LPC_ORDER = DecCore<KHZ>::LPC_ORDER }

template <int KHZ> struct DecMdT {
    SB_DEC_DIMS(KHZ);
    i32 LastGainIndex;
    i32 prevNLSF_Q15[LPC_ORDER];
    i32 typeOffsetPrev;
    i32 prevDeltaGainIndex;
};

// decoder arithmetic of a stream: the reference's float build (the default) or its fixed-point build
enum { DEC_FLP = 0, DEC_FIX = 1 };

template <int KHZ> struct DecStateT {
    SB_DEC_DIMS(KHZ);
    i32 useMDIndex;
    i32 frames_per_packet;  // 2: 40 ms packets, 1: 20 ms packets
    i32 hb_frame;           // FRAME, or 2 * FRAME with joint_mode 1
    i32 arith;              // DEC_FLP or DEC_FIX
    i32 seen_good;  // 0 until the first frame has been range-decoded (reference state is still at fs = 24 kHz)
    DecMdT<KHZ> md[2];
    i32 prev_inv_gain_Q16;
    i32 sLTP_Q16[2 * FRAME];
    i32 sLPC_Q14[16];
    i32 exc_Q10[FRAME];
    i16 outBuf[2 * FRAME];
    i32 lagPrev, first_frame_after_reset, moreInternalDecoderFrames, nFramesDecoded, FrameTermination;
    i32 nBytesLeft[2];
    // range decoder position of a payload that is still being consumed when the packet call returns (see DecStale)
    u32 rc_base_Q32[2], rc_range_Q16[2];
    i32 rc_bufferIx[2], rc_error[2], rc_bufLen[2];
    i32 vadFlag, lossCnt, prev_sigtype;
    // PLC (structs.h:268-280)
    i32 plc_pitchL_Q8, plc_last_frame_lost, plc_rand_seed, plc_conc_energy, plc_conc_energy_shift;
    i32 plc_prevGain_Q16[NB_SUBFR];
    i16 plc_LTPCoef_Q14[LTP_ORDER], plc_prevLPC_Q12[LPC_ORDER], plc_randScale_Q14, plc_prevLTP_scale_Q14;
    // 1: the stream decodes to its SILK core only (core output of a 32 kHz stream, dec_packet<KHZ, true>), so its high-band
    // and filter-bank memories never advance.  Kept in the state so that an exported blob records it.  It sits in what was
    // the padding after the int16 fields above: the state's size and every other field's offset are as without it.
    i16 core_only;
    // CNG (structs.h:283-290)
    i32 cng_exc_buf_Q10[FRAME];
    i32 cng_smth_NLSF_Q15[LPC_ORDER];
    i32 cng_synth_state[LPC_ORDER];
    i32 cng_smth_Gain_Q16, cng_rand_seed;
    // high band + QMF synthesis (AGR_BWE_structs.h).  A stream uses either the float fields (DEC_FLP) or their fixed-point
    // counterparts (DEC_FIX), so they share storage.  The filter-bank memories hold int16-valued samples in both modes.
    i32 hb_lossCnt, hb_first;
    union { float hb_prev_NLSFq[HB_ORDER]; i32 hb_prev_NLSF_Q15[HB_ORDER]; };
    union { float hb_prev_Gain; i32 hb_prev_Gain_fix; };
    union { float hb_sLPC[16]; i32 hb_synth_Q14[HB_ORDER]; };   // HB_synth_state: [HB_ORDER - 1] newest
    float g0_mem[64], g1_mem[64];
};
typedef DecStateT<8> DecState;      // 16 kHz streams
typedef DecStateT<16> DecState32;   // 32 kHz streams

template <int KHZ> struct DecCtrlT {
    SB_DEC_DIMS(KHZ);
    i32 pitchL[NB_SUBFR];
    i32 Gains_Q16[NB_SUBFR];
    i32 DeltaGains_Q16;
    i32 Seed;
    i16 PredCoef_Q12[2][LPC_ORDER];
    i16 LTPCoef_Q14[LTP_ORDER * NB_SUBFR];
    i32 LTP_scale_Q14;
    i32 PERIndex, RateLevelIndex, QuantOffsetType, sigtype, MDIndex, NLSFInterpCoef_Q2;
};

// SKP_Silk_init_decoder + AGR_Sate_Decoder_Init, expressed for the core the first good frame selects (the PLC and CNG
// reset themselves to it on their first call, PLC.c:52-55, CNG.c:89-94).
// dec_state_fields sets what Init sets on a zeroed state; dec_state_init zeroes the state first (the device's reset kernel
// zeroes it with word stores instead of this byte-wise memset, then calls dec_state_fields).
template <int KHZ> SB_FN void dec_state_fields(DecStateT<KHZ>* st, i32 useMDIndex, i32 framesize_ms, i32 joint_hb, i32 arith, i32 core_only) {
    SB_DEC_DIMS(KHZ);
    st->useMDIndex = useMDIndex;
    st->core_only = core_only ? 1 : 0;
    st->arith = arith == DEC_FIX ? DEC_FIX : DEC_FLP;
    st->frames_per_packet = framesize_ms == 20 ? 1 : 2;
    st->hb_frame = joint_hb ? 2 * FRAME : FRAME;
    st->first_frame_after_reset = 1;
    st->prev_inv_gain_Q16 = 65536;
    st->lagPrev = 100;
    st->md[0].LastGainIndex = 1;
    st->md[1].LastGainIndex = 1;
    st->plc_pitchL_Q8 = FRAME >> 1;  // SKP_Silk_PLC_Reset at the core rate
    // SKP_Silk_CNG_Reset (CNG.c:58-73) at the core's order
    i32 step = 32767 / (LPC_ORDER + 1), acc = 0;
    for (int i = 0; i < LPC_ORDER; i++) { acc += step; st->cng_smth_NLSF_Q15[i] = acc; }
    st->cng_rand_seed = 3176576;
    st->hb_first = 1;
}
template <int KHZ> SB_FN void dec_state_init(DecStateT<KHZ>* st, i32 useMDIndex, i32 framesize_ms = 40, i32 joint_hb = 0, i32 arith = DEC_FLP,
                                              i32 core_only = 0) {
    memset(st, 0, sizeof(DecStateT<KHZ>));
    dec_state_fields(st, useMDIndex, framesize_ms, joint_hb, arith, core_only);
}

// Length split of AGR_Sate_decode_process (AGR_BWE_decode_frame_FLP.c:171-190): {n0, n1} as passed by the
// caller -> {len(description in slot 0), len(description in slot 1)}; returns the byte offset of the HB bits.
SB_HD i32 dec_split_lengths(i16* nb, i32 lostflag, int hb_bytes) {
    i32 total = nb[0];
    i32 n0 = lostflag == 2 ? total : total - hb_bytes;
    i32 n1 = nb[1];
    if (n1) n1 -= hb_bytes;
    i32 hb_off = n0;
    n0 -= n1;
    nb[0] = (i16)n0;
    nb[1] = (i16)n1;
    return hb_off;
}

// ---- entropy decoding ---------------------------------------------------------------------------------
SB_HD void dec_split(int* c1, int* c2, RangeDec* rc, int p, const u16* shell_table) {
    if (p > 0) {
        rc_decode(c1, rc, &shell_table[SB_T(shell_table_offsets)[p]], p >> 1);
        *c2 = p - *c1;
    } else { *c1 = 0; *c2 = 0; }
}
SB_FN void shell_decoder(i32* p0, RangeDec* rc, int pulses4) {
    int p3[2], p2[4], p1[8];
    dec_split(&p3[0], &p3[1], rc, pulses4, SB_T(shell_table3));
    dec_split(&p2[0], &p2[1], rc, p3[0], SB_T(shell_table2));
    dec_split(&p1[0], &p1[1], rc, p2[0], SB_T(shell_table1));
    dec_split(&p0[0], &p0[1], rc, p1[0], SB_T(shell_table0));
    dec_split(&p0[2], &p0[3], rc, p1[1], SB_T(shell_table0));
    dec_split(&p1[2], &p1[3], rc, p2[1], SB_T(shell_table1));
    dec_split(&p0[4], &p0[5], rc, p1[2], SB_T(shell_table0));
    dec_split(&p0[6], &p0[7], rc, p1[3], SB_T(shell_table0));
    dec_split(&p2[2], &p2[3], rc, p3[1], SB_T(shell_table2));
    dec_split(&p1[4], &p1[5], rc, p2[2], SB_T(shell_table1));
    dec_split(&p0[8], &p0[9], rc, p1[4], SB_T(shell_table0));
    dec_split(&p0[10], &p0[11], rc, p1[5], SB_T(shell_table0));
    dec_split(&p1[6], &p1[7], rc, p2[3], SB_T(shell_table1));
    dec_split(&p0[12], &p0[13], rc, p1[6], SB_T(shell_table0));
    dec_split(&p0[14], &p0[15], rc, p1[7], SB_T(shell_table0));
}

// SKP_Silk_decode_pulses (decode_pulses.c:33-110)
template <int KHZ> SB_FN void decode_pulses(RangeDec* rc, DecCtrlT<KHZ>* c, i32* q) {
    SB_DEC_DIMS(KHZ);
    enum { ITER = FRAME / 16 };
    int sum_pulses[ITER], nLshifts[ITER];
    rc_decode(&c->RateLevelIndex, rc, &SB_T(rate_levels_cdf)[c->sigtype * 10], SB_T(rate_levels_cdf_offset)[0]);
    const u16* cdf_ptr = &SB_T(pulses_per_block_cdf)[c->RateLevelIndex * 21];
    const u16* cdf_last = &SB_T(pulses_per_block_cdf)[9 * 21];
    const int off = SB_T(pulses_per_block_cdf_offset)[0];
    for (int i = 0; i < ITER; i++) {
        nLshifts[i] = 0;
        rc_decode(&sum_pulses[i], rc, cdf_ptr, off);
        while (sum_pulses[i] == 18 + 1) {
            nLshifts[i]++;
            rc_decode(&sum_pulses[i], rc, cdf_last, off);
        }
    }
    for (int i = 0; i < ITER; i++) {
        if (sum_pulses[i] > 0) shell_decoder(&q[i * 16], rc, sum_pulses[i]);
        else for (int k = 0; k < 16; k++) q[i * 16 + k] = 0;
    }
    for (int i = 0; i < ITER; i++) {
        if (nLshifts[i] > 0) {
            int nLS = nLshifts[i];
            i32* pp = &q[i * 16];
            for (int k = 0; k < 16; k++) {
                i32 abs_q = pp[k];
                for (int j = 0; j < nLS; j++) {
                    int bit;
                    abs_q = shl(abs_q, 1);
                    rc_decode(&bit, rc, SB_T(lsb_cdf), 1);
                    abs_q += bit;
                }
                pp[k] = abs_q;
            }
        }
    }
    // SKP_Silk_decode_signs (code_signs.c:64-90)
    u16 cdf[3];
    int idx = smulbb(9, shl(c->sigtype, 1) + c->QuantOffsetType) + c->RateLevelIndex;
    cdf[0] = 0; cdf[1] = SB_T(sign_cdf)[idx]; cdf[2] = 65535;
    for (int i = 0; i < FRAME; i++) {
        if (q[i] > 0) {
            int data;
            rc_decode(&data, rc, cdf, 1);
            q[i] *= (shl(data, 1) - 1);
        }
    }
}

// SKP_Silk_gains_dequant (gain_quant.c:110-142), md_enable == 1
SB_FN void gains_dequant(i32* gain_Q16, const i32* ind, i32* prev_ind, int conditional, int ind2, i32* DeltaGains_Q16) {
    const i32 OFFSET = (6 * 128) / 6 + 16 * 128;
    const i32 INV_SCALE_Q16 = (65536 * (((86 - 6) * 128) / 6)) / (64 - 1);
    for (int k = 0; k < NB_SUBFR; k++) {
        if (k == 0 && conditional == 0) *prev_ind = ind[k];
        else *prev_ind += ind[k] + -4;
        gain_Q16[k] = log2lin(imin(smulwb(INV_SCALE_Q16, *prev_ind) + OFFSET, 3967));
    }
    i32 inv_gain_Q16 = (ind2 + 1) * (32768 / 8);
    inv_gain_Q16 += 32767;
    *DeltaGains_Q16 = inverse32_varq(imax(inv_gain_Q16, 1), 32);
}

// SKP_Silk_decode_parameters (decode_parameters.c:31-297), fullDecoding == 1, description slot kDesp
template <int KHZ> SB_FN void decode_parameters(DecStateT<KHZ>* st, DecCtrlT<KHZ>* c, RangeDec* rc, i32* q, int kDesp) {
    SB_DEC_DIMS(KHZ);
    enum { NLSF_STAGES = NlsfStages<LPC_ORDER>::N };
    DecMdT<KHZ>* md = &st->md[kDesp];
    int Ix;
    i32 GainsIndices[NB_SUBFR], NLSFIndices[NLSF_STAGES], pNLSF_Q15[LPC_ORDER], pNLSF0_Q15[LPC_ORDER];
    if (st->nFramesDecoded == 0) {
        if (st->useMDIndex == 1) rc_decode(&c->MDIndex, rc, SB_T(md_index_cdf), SB_T(md_index_offset)[0]);
        rc_decode(&Ix, rc, SB_T(sampling_rates_cdf), SB_T(sampling_rates_offset)[0]);
        if (Ix < 0 || Ix > 3) { rc->error = -7; return; }
        // the decoder's core rate only: any other would be resampled to the API rate (dec_API.c:160-177), which is not built
        if (SB_T(sampling_rates_table)[Ix] != KHZ) { rc->error = -7; return; }
        if (!st->seen_good) {
            // SKP_Silk_decoder_set_fs(KHZ) on the first decoded frame (decoder_set_fs.c:31-86)
            st->seen_good = 1;
            for (int i = 0; i < 16; i++) st->sLPC_Q14[i] = 0;
            for (int i = 0; i < 2 * FRAME; i++) st->outBuf[i] = 0;
            for (int m = 0; m < 2; m++) { for (int i = 0; i < LPC_ORDER; i++) st->md[m].prevNLSF_Q15[i] = 0; st->md[m].LastGainIndex = 1; }
            st->lagPrev = 100;
            st->prev_sigtype = 0;
            st->first_frame_after_reset = 1;
        }
    }
    if (st->nFramesDecoded == 0) rc_decode(&Ix, rc, SB_T(type_offset_cdf), SB_T(type_offset_cdf_offset)[0]);
    else rc_decode(&Ix, rc, &SB_T(type_offset_joint_cdf)[md->typeOffsetPrev * 5], SB_T(type_offset_cdf_offset)[0]);
    c->sigtype = Ix >> 1;
    c->QuantOffsetType = Ix & 1;
    md->typeOffsetPrev = Ix;
    if (st->nFramesDecoded == 0) rc_decode(&GainsIndices[0], rc, &SB_T(gain_cdf)[c->sigtype * 65], SB_T(gain_cdf_offset)[0]);
    else rc_decode(&GainsIndices[0], rc, SB_T(delta_gain_cdf), SB_T(delta_gain_cdf_offset)[0]);
    for (int i = 1; i < NB_SUBFR; i++) rc_decode(&GainsIndices[i], rc, SB_T(delta_gain_cdf), SB_T(delta_gain_cdf_offset)[0]);
    int DeltaGainIndices;
    if (st->nFramesDecoded == 0) {
        rc_decode(&DeltaGainIndices, rc, SB_T(md_delta_gain_cdf), SB_T(md_delta_gain_cdf_offset)[0]);
        md->prevDeltaGainIndex = DeltaGainIndices;
    } else DeltaGainIndices = md->prevDeltaGainIndex;
    gains_dequant(c->Gains_Q16, GainsIndices, &md->LastGainIndex, st->nFramesDecoded, DeltaGainIndices, &c->DeltaGains_Q16);
    NlsfCb cb = nlsf_cb<LPC_ORDER>(c->sigtype);
    for (int k = 0; k < NLSF_STAGES; k++) rc_decode(&NLSFIndices[k], rc, &cb.cdf[cb.cdf_start[k]], cb.cdf_mid[k]);
    nlsf_msvq_decode<LPC_ORDER>(pNLSF_Q15, cb, NLSFIndices);
    rc_decode(&c->NLSFInterpCoef_Q2, rc, SB_T(nlsf_interp_cdf), SB_T(nlsf_interp_offset)[0]);
    if (st->first_frame_after_reset == 1) c->NLSFInterpCoef_Q2 = 4;
    nlsf2a_stable(c->PredCoef_Q12[1], pNLSF_Q15, LPC_ORDER);
    if (c->NLSFInterpCoef_Q2 < 4) {
        for (int i = 0; i < LPC_ORDER; i++)
            pNLSF0_Q15[i] = md->prevNLSF_Q15[i] + (mulw(c->NLSFInterpCoef_Q2, pNLSF_Q15[i] - md->prevNLSF_Q15[i]) >> 2);
        nlsf2a_stable(c->PredCoef_Q12[0], pNLSF0_Q15, LPC_ORDER);
    } else {
        for (int i = 0; i < LPC_ORDER; i++) c->PredCoef_Q12[0][i] = c->PredCoef_Q12[1][i];
    }
    for (int i = 0; i < LPC_ORDER; i++) md->prevNLSF_Q15[i] = pNLSF_Q15[i];
    if (st->lossCnt) {
        bwexpander(c->PredCoef_Q12[0], LPC_ORDER, 63570);
        bwexpander(c->PredCoef_Q12[1], LPC_ORDER, 63570);
    }
    if (c->sigtype == 0) {
        int Ixs[2];
        if (KHZ == 8) {
            rc_decode(&Ixs[0], rc, SB_T(pitch_lag_nb_cdf), SB_T(pitch_lag_nb_offset)[0]);
            rc_decode(&Ixs[1], rc, SB_T(pitch_contour_nb_cdf), SB_T(pitch_contour_nb_offset)[0]);
        } else {
            rc_decode(&Ixs[0], rc, SB_T(pitch_lag_wb_cdf), SB_T(pitch_lag_wb_offset)[0]);
            rc_decode(&Ixs[1], rc, SB_T(pitch_contour_cdf), SB_T(pitch_contour_offset)[0]);
        }
        // SKP_Silk_decode_pitch (decode_pitch.c:34-60): minimum lag 2 ms, the stage-2 contours at 8 kHz, stage 3 above
        int lag = 2 * KHZ + Ixs[0];
        for (int i = 0; i < NB_SUBFR; i++)
            c->pitchL[i] = lag + (KHZ == 8 ? SB_T(pitch_cb_lags_stage2)[i * 11 + Ixs[1]] : SB_T(pitch_cb_lags_stage3)[i * 34 + Ixs[1]]);
        rc_decode(&c->PERIndex, rc, SB_T(ltp_per_index_cdf), SB_T(ltp_per_index_offset)[0]);
        const i16* cbk = c->PERIndex == 0 ? SB_T(ltp_vq0_q14) : (c->PERIndex == 1 ? SB_T(ltp_vq1_q14) : SB_T(ltp_vq2_q14));
        const u16* lc = c->PERIndex == 0 ? SB_T(ltp_cdf0) : (c->PERIndex == 1 ? SB_T(ltp_cdf1) : SB_T(ltp_cdf2));
        for (int k = 0; k < NB_SUBFR; k++) {
            rc_decode(&Ix, rc, lc, SB_T(ltp_cdf_offsets)[c->PERIndex]);
            for (int i = 0; i < LTP_ORDER; i++) c->LTPCoef_Q14[k * LTP_ORDER + i] = cbk[Ix * LTP_ORDER + i];
        }
        rc_decode(&Ix, rc, SB_T(ltpscale_cdf), SB_T(ltpscale_offset)[0]);
        c->LTP_scale_Q14 = SB_T(ltpscales_q14)[Ix];
    } else {
        for (int i = 0; i < NB_SUBFR; i++) c->pitchL[i] = 0;
        for (int i = 0; i < LTP_ORDER * NB_SUBFR; i++) c->LTPCoef_Q14[i] = 0;
        c->PERIndex = 0;
        c->LTP_scale_Q14 = 0;
    }
    rc_decode(&Ix, rc, SB_T(seed_cdf), SB_T(seed_offset)[0]);
    c->Seed = Ix;
    decode_pulses(rc, c, q);
    rc_decode(&st->vadFlag, rc, SB_T(vadflag_cdf), SB_T(vadflag_offset)[0]);
    rc_decode(&st->FrameTermination, rc, SB_T(frame_term_cdf), SB_T(frame_term_offset)[0]);
    int nBytesUsed = (shl(rc->bufferIx, 3) + clz32((i32)(rc->range_Q16 - 1)) - 14 + 7) >> 3;
    st->nBytesLeft[kDesp] = rc->bufLen - nBytesUsed;
    if (st->nBytesLeft[kDesp] < 0) rc->error = -6;
    if (st->nBytesLeft[kDesp] == 0) rc_check_after_decoding(rc);
}

// ---- SKP_Silk_decode_core (decode_core.c:44-213) -----------------------------------------------------------
template <int KHZ> SB_FN void decode_core(DecStateT<KHZ>* st, DecCtrlT<KHZ>* c, i16* xq) {
    SB_DEC_DIMS(KHZ);
    i16 sLTP[FRAME];
    i32 vec_Q10[SUBFR], res_Q10[SUBFR];
    i32 sLPC[16 + SUBFR];
    for (int i = 0; i < 16; i++) sLPC[i] = st->sLPC_Q14[i];
    const int NLSF_interpolation_flag = c->NLSFInterpCoef_Q2 < 4 ? 1 : 0;
    const i32* pexc_Q10 = st->exc_Q10;
    i16* pxq = &st->outBuf[FRAME];
    int sLTP_buf_idx = FRAME, lag = 0;
    for (int k = 0; k < NB_SUBFR; k++) {
        const i16* A_Q12 = c->PredCoef_Q12[k >> 1];
        i16* B_Q14 = &c->LTPCoef_Q14[k * LTP_ORDER];
        i32 Gain_Q16 = c->Gains_Q16[k];
        int sigtype = c->sigtype;
        i32 inv_gain_Q16 = imin(inverse32_varq(imax(Gain_Q16, 1), 32), 32767);
        i32 gain_adj_Q16 = 1 << 16;
        if (inv_gain_Q16 != st->prev_inv_gain_Q16) gain_adj_Q16 = div32_varq(inv_gain_Q16, st->prev_inv_gain_Q16, 16);
        if (st->lossCnt && st->prev_sigtype == 0 && c->sigtype == 1 && k < (NB_SUBFR >> 1)) {
            for (int i = 0; i < LTP_ORDER; i++) B_Q14[i] = 0;
            B_Q14[LTP_ORDER / 2] = (i16)(1 << 12);
            sigtype = 0;
            c->pitchL[k] = st->lagPrev;
        }
        if (sigtype == 0) {
            lag = c->pitchL[k];
            if ((k & (3 - shl(NLSF_interpolation_flag, 1))) == 0) {
                int start_idx = FRAME - lag - LPC_ORDER - LTP_ORDER / 2;
                ma_prediction_zero_state(&st->outBuf[start_idx + k * (FRAME >> 2)], A_Q12, sLTP + start_idx, FRAME - start_idx, LPC_ORDER);
                i32 inv_gain_Q32 = shl(inv_gain_Q16, 16);
                if (k == 0) inv_gain_Q32 = shl(smulwb(inv_gain_Q32, c->LTP_scale_Q14), 2);
                for (int i = 0; i < lag + LTP_ORDER / 2; i++) st->sLTP_Q16[sLTP_buf_idx - i - 1] = smulwb(inv_gain_Q32, sLTP[FRAME - i - 1]);
            } else if (gain_adj_Q16 != (1 << 16)) {
                for (int i = 0; i < lag + LTP_ORDER / 2; i++) st->sLTP_Q16[sLTP_buf_idx - i - 1] = smulww(gain_adj_Q16, st->sLTP_Q16[sLTP_buf_idx - i - 1]);
            }
        }
        for (int i = 0; i < 16; i++) sLPC[i] = smulww(gain_adj_Q16, sLPC[i]);
        st->prev_inv_gain_Q16 = inv_gain_Q16;
        if (sigtype == 0) {
            const i32* pred_lag_ptr = &st->sLTP_Q16[sLTP_buf_idx - lag + LTP_ORDER / 2];
            for (int i = 0; i < SUBFR; i++) {
                i32 LTP_pred_Q14 = smulwb(pred_lag_ptr[0], B_Q14[0]);
                LTP_pred_Q14 = smlawb(LTP_pred_Q14, pred_lag_ptr[-1], B_Q14[1]);
                LTP_pred_Q14 = smlawb(LTP_pred_Q14, pred_lag_ptr[-2], B_Q14[2]);
                LTP_pred_Q14 = smlawb(LTP_pred_Q14, pred_lag_ptr[-3], B_Q14[3]);
                LTP_pred_Q14 = smlawb(LTP_pred_Q14, pred_lag_ptr[-4], B_Q14[4]);
                pred_lag_ptr++;
                res_Q10[i] = addw(pexc_Q10[i], rshift_round(LTP_pred_Q14, 4));
                st->sLTP_Q16[sLTP_buf_idx] = shl(res_Q10[i], 6);
                sLTP_buf_idx++;
            }
        } else {
            for (int i = 0; i < SUBFR; i++) res_Q10[i] = pexc_Q10[i];
        }
        for (int i = 0; i < SUBFR; i++) {
            i32 LPC_pred_Q10 = 0;
            for (int j = 0; j < LPC_ORDER; j++) LPC_pred_Q10 = smlawb(LPC_pred_Q10, sLPC[16 + i - j - 1], A_Q12[j]);
            vec_Q10[i] = addw(res_Q10[i], LPC_pred_Q10);
            sLPC[16 + i] = shl(vec_Q10[i], 4);
        }
        for (int i = 0; i < SUBFR; i++) pxq[i] = (i16)sat16(rshift_round(smulww(vec_Q10[i], Gain_Q16), 10));
        for (int i = 0; i < 16; i++) sLPC[i] = sLPC[SUBFR + i];
        pexc_Q10 += SUBFR;
        pxq += SUBFR;
    }
    for (int i = 0; i < 16; i++) st->sLPC_Q14[i] = sLPC[i];
    for (int i = 0; i < FRAME; i++) xq[i] = st->outBuf[FRAME + i];
}

// ---- SKP_Silk_PLC_update (PLC.c:75-144) -------------------------------------------------------------------
template <int KHZ> SB_FN void plc_update(DecStateT<KHZ>* st, DecCtrlT<KHZ>* c) {
    SB_DEC_DIMS(KHZ);
    st->prev_sigtype = c->sigtype;
    i32 LTP_Gain_Q14 = 0;
    if (c->sigtype == 0) {
        for (int j = 0; j * SUBFR < c->pitchL[NB_SUBFR - 1]; j++) {
            i32 temp = 0;
            for (int i = 0; i < LTP_ORDER; i++) temp += c->LTPCoef_Q14[(NB_SUBFR - 1 - j) * LTP_ORDER + i];
            if (temp > LTP_Gain_Q14) {
                LTP_Gain_Q14 = temp;
                for (int i = 0; i < LTP_ORDER; i++) st->plc_LTPCoef_Q14[i] = c->LTPCoef_Q14[(NB_SUBFR - 1 - j) * LTP_ORDER + i];
                st->plc_pitchL_Q8 = shl(c->pitchL[NB_SUBFR - 1 - j], 8);
            }
        }
        for (int i = 0; i < LTP_ORDER; i++) st->plc_LTPCoef_Q14[i] = 0;
        st->plc_LTPCoef_Q14[LTP_ORDER / 2] = (i16)LTP_Gain_Q14;
        if (LTP_Gain_Q14 < 11469) {
            i32 tmp = shl(11469, 10);
            i32 scale_Q10 = tmp / imax(LTP_Gain_Q14, 1);
            for (int i = 0; i < LTP_ORDER; i++) st->plc_LTPCoef_Q14[i] = (i16)(smulbb(st->plc_LTPCoef_Q14[i], scale_Q10) >> 10);
        } else if (LTP_Gain_Q14 > 15565) {
            i32 tmp = shl(15565, 14);
            i32 scale_Q14 = tmp / imax(LTP_Gain_Q14, 1);
            for (int i = 0; i < LTP_ORDER; i++) st->plc_LTPCoef_Q14[i] = (i16)(smulbb(st->plc_LTPCoef_Q14[i], scale_Q14) >> 14);
        }
    } else {
        st->plc_pitchL_Q8 = shl(smulbb(KHZ, 18), 8);
        for (int i = 0; i < LTP_ORDER; i++) st->plc_LTPCoef_Q14[i] = 0;
    }
    for (int i = 0; i < LPC_ORDER; i++) st->plc_prevLPC_Q12[i] = c->PredCoef_Q12[1][i];
    st->plc_prevLTP_scale_Q14 = (i16)c->LTP_scale_Q14;
    for (int i = 0; i < NB_SUBFR; i++) st->plc_prevGain_Q16[i] = c->Gains_Q16[i];
}

// ---- SKP_Silk_PLC_conceal (PLC.c:146-330) -----------------------------------------------------------------
template <int KHZ> SB_FN void plc_conceal(DecStateT<KHZ>* st, DecCtrlT<KHZ>* c, i16* signal) {
    SB_DEC_DIMS(KHZ);
    const i16 HARM_ATT_Q15[2] = {32440, 31130};
    const i16 RAND_ATT_V_Q15[2] = {31130, 26214};
    const i16 RAND_ATT_UV_Q15[2] = {32440, 29491};
    i16 exc_buf[FRAME / 2];
    i32 sig_Q10[FRAME];
    i32 sLPC[16 + SUBFR];
    for (int i = 0; i < FRAME; i++) st->sLTP_Q16[i] = st->sLTP_Q16[FRAME + i];
    bwexpander(st->plc_prevLPC_Q12, LPC_ORDER, 64880);
    i16* ep = exc_buf;
    for (int k = NB_SUBFR >> 1; k < NB_SUBFR; k++) {
        for (int i = 0; i < SUBFR; i++) ep[i] = (i16)(smulww(st->exc_Q10[i + k * SUBFR], st->plc_prevGain_Q16[k]) >> 10);
        ep += SUBFR;
    }
    i32 energy1, energy2, shift1, shift2;
    sum_sqr_shift(&energy1, &shift1, exc_buf, SUBFR, 0);
    sum_sqr_shift(&energy2, &shift2, &exc_buf[SUBFR], SUBFR, 0);
    const i32* rand_ptr;
    if ((energy1 >> shift2) < (energy2 >> shift1)) rand_ptr = &st->exc_Q10[imax(0, 3 * SUBFR - 128)];
    else rand_ptr = &st->exc_Q10[imax(0, FRAME - 128)];
    i16* B_Q14 = st->plc_LTPCoef_Q14;
    i16 rand_scale_Q14 = st->plc_randScale_Q14;
    i32 harm_Gain_Q15 = HARM_ATT_Q15[imin(1, st->lossCnt)];
    i32 rand_Gain_Q15 = st->prev_sigtype == 0 ? RAND_ATT_V_Q15[imin(1, st->lossCnt)] : RAND_ATT_UV_Q15[imin(1, st->lossCnt)];
    if (st->lossCnt == 0) {
        rand_scale_Q14 = 1 << 14;
        if (st->prev_sigtype == 0) {
            for (int i = 0; i < LTP_ORDER; i++) rand_scale_Q14 = (i16)(rand_scale_Q14 - B_Q14[i]);
            rand_scale_Q14 = rand_scale_Q14 > 3277 ? rand_scale_Q14 : (i16)3277;
            rand_scale_Q14 = (i16)(smulbb(rand_scale_Q14, st->plc_prevLTP_scale_Q14) >> 14);
        }
        if (st->prev_sigtype == 1) {
            i32 invGain_Q30;
            lpc_inv_pred_gain_q12(&invGain_Q30, st->plc_prevLPC_Q12, LPC_ORDER);
            i32 down_scale_Q30 = imin((1 << 30) >> 3, invGain_Q30);
            down_scale_Q30 = imax((1 << 30) >> 8, down_scale_Q30);
            down_scale_Q30 = shl(down_scale_Q30, 3);
            rand_Gain_Q15 = smulwb(down_scale_Q30, rand_Gain_Q15) >> 14;
        }
    }
    i32 rand_seed = st->plc_rand_seed;
    int lag = rshift_round(st->plc_pitchL_Q8, 8);
    int sLTP_buf_idx = FRAME;
    i32* sp = sig_Q10;
    for (int k = 0; k < NB_SUBFR; k++) {
        const i32* pred_lag_ptr = &st->sLTP_Q16[sLTP_buf_idx - lag + LTP_ORDER / 2];
        for (int i = 0; i < SUBFR; i++) {
            rand_seed = lcg_rand(rand_seed);
            int idx = (rand_seed >> 25) & 127;
            i32 LTP_pred_Q14 = smulwb(pred_lag_ptr[0], B_Q14[0]);
            LTP_pred_Q14 = smlawb(LTP_pred_Q14, pred_lag_ptr[-1], B_Q14[1]);
            LTP_pred_Q14 = smlawb(LTP_pred_Q14, pred_lag_ptr[-2], B_Q14[2]);
            LTP_pred_Q14 = smlawb(LTP_pred_Q14, pred_lag_ptr[-3], B_Q14[3]);
            LTP_pred_Q14 = smlawb(LTP_pred_Q14, pred_lag_ptr[-4], B_Q14[4]);
            pred_lag_ptr++;
            i32 LPC_exc_Q10 = shl(smulwb(rand_ptr[idx], rand_scale_Q14), 2);
            LPC_exc_Q10 = addw(LPC_exc_Q10, rshift_round(LTP_pred_Q14, 4));
            st->sLTP_Q16[sLTP_buf_idx] = shl(LPC_exc_Q10, 6);
            sLTP_buf_idx++;
            sp[i] = LPC_exc_Q10;
        }
        sp += SUBFR;
        for (int j = 0; j < LTP_ORDER; j++) B_Q14[j] = (i16)(smulbb(harm_Gain_Q15, B_Q14[j]) >> 15);
        rand_scale_Q14 = (i16)(smulbb(rand_scale_Q14, rand_Gain_Q15) >> 15);
        st->plc_pitchL_Q8 += smulwb(st->plc_pitchL_Q8, 655);
        st->plc_pitchL_Q8 = imin(st->plc_pitchL_Q8, shl(smulbb(18, KHZ), 8));
        lag = rshift_round(st->plc_pitchL_Q8, 8);
    }
    for (int i = 0; i < 16; i++) sLPC[i] = st->sLPC_Q14[i];
    sp = sig_Q10;
    for (int k = 0; k < NB_SUBFR; k++) {
        for (int i = 0; i < SUBFR; i++) {
            i32 LPC_pred_Q10 = 0;
            for (int j = 0; j < LPC_ORDER; j++) LPC_pred_Q10 = smlawb(LPC_pred_Q10, sLPC[16 + i - j - 1], st->plc_prevLPC_Q12[j]);
            sp[i] = addw(sp[i], LPC_pred_Q10);
            sLPC[16 + i] = shl(sp[i], 4);
        }
        sp += SUBFR;
        for (int i = 0; i < 16; i++) sLPC[i] = sLPC[SUBFR + i];
    }
    for (int i = 0; i < 16; i++) st->sLPC_Q14[i] = sLPC[i];
    for (int i = 0; i < FRAME; i++) signal[i] = (i16)sat16(rshift_round(smulww(sig_Q10[i], st->plc_prevGain_Q16[NB_SUBFR - 1]), 10));
    st->plc_rand_seed = rand_seed;
    st->plc_randScale_Q14 = rand_scale_Q14;
    for (int i = 0; i < NB_SUBFR; i++) c->pitchL[i] = lag;
}

// ---- SKP_Silk_PLC_glue_frames (PLC.c:333-387) --------------------------------------------------------------
// `len_ref`: the frame length the reference divides the fade slope by.  It is FRAME except for the very first decoded frame,
// where SKP_Silk_decode_frame still holds the start-up length 480 (fs 24 kHz) it read before the range decoder switched
// the core to KHZ (decode_frame.c:277 vs decoder_set_fs); the extra 480 - FRAME samples it touches are scratch.
template <int KHZ> SB_FN void plc_glue_frames(DecStateT<KHZ>* st, i16* signal, int len_ref) {
    SB_DEC_DIMS(KHZ);
    if (st->lossCnt) {
        sum_sqr_shift(&st->plc_conc_energy, &st->plc_conc_energy_shift, signal, FRAME, 0);
        st->plc_last_frame_lost = 1;
    } else {
        if (st->plc_last_frame_lost) {
            i32 energy, energy_shift;
            sum_sqr_shift(&energy, &energy_shift, signal, FRAME, 0);
            if (energy_shift > st->plc_conc_energy_shift) st->plc_conc_energy = st->plc_conc_energy >> (energy_shift - st->plc_conc_energy_shift);
            else if (energy_shift < st->plc_conc_energy_shift) energy = energy >> (st->plc_conc_energy_shift - energy_shift);
            if (energy > st->plc_conc_energy) {
                i32 LZ = clz32(st->plc_conc_energy) - 1;
                st->plc_conc_energy = shl(st->plc_conc_energy, LZ);
                energy = energy >> imax(24 - LZ, 0);
                i32 frac_Q24 = st->plc_conc_energy / imax(energy, 1);
                i32 gain_Q12 = sqrt_approx(frac_Q24);
                i32 slope_Q12 = ((1 << 12) - gain_Q12) / len_ref;
                for (int i = 0; i < FRAME; i++) {
                    signal[i] = (i16)(mulw(gain_Q12, signal[i]) >> 12);
                    gain_Q12 += slope_Q12;
                    gain_Q12 = imin(gain_Q12, 1 << 12);
                }
            }
        }
        st->plc_last_frame_lost = 0;
    }
}

// ---- SKP_Silk_CNG (CNG.c:75-149) at the core's order; SKP_Silk_LPC_synthesis_order16 sums the same products -------
template <int KHZ> SB_FN void cng(DecStateT<KHZ>* st, const DecCtrlT<KHZ>* c, i16* signal) {
    SB_DEC_DIMS(KHZ);
    if (st->lossCnt == 0 && st->vadFlag == 0) {
        for (int i = 0; i < LPC_ORDER; i++)
            st->cng_smth_NLSF_Q15[i] += smulwb(st->md[0].prevNLSF_Q15[i] - st->cng_smth_NLSF_Q15[i], 16348);
        i32 max_Gain_Q16 = 0; int subfr = 0;
        for (int i = 0; i < NB_SUBFR; i++) if (c->Gains_Q16[i] > max_Gain_Q16) { max_Gain_Q16 = c->Gains_Q16[i]; subfr = i; }
        for (int i = FRAME - 1; i >= SUBFR; i--) st->cng_exc_buf_Q10[i] = st->cng_exc_buf_Q10[i - SUBFR];
        for (int i = 0; i < SUBFR; i++) st->cng_exc_buf_Q10[i] = st->exc_Q10[subfr * SUBFR + i];
        for (int i = 0; i < NB_SUBFR; i++) st->cng_smth_Gain_Q16 += smulwb(c->Gains_Q16[i] - st->cng_smth_Gain_Q16, 4634);
    }
    if (st->lossCnt) {
        i16 CNG_sig[FRAME], LPC_buf[LPC_ORDER];
        int exc_mask = 255;
        while (exc_mask > FRAME) exc_mask >>= 1;
        i32 seed = st->cng_rand_seed;
        for (int i = 0; i < FRAME; i++) {
            seed = lcg_rand(seed);
            int idx = (seed >> 24) & exc_mask;
            CNG_sig[i] = (i16)sat16(rshift_round(smulww(st->cng_exc_buf_Q10[idx], st->cng_smth_Gain_Q16), 10));
        }
        st->cng_rand_seed = seed;
        nlsf2a_stable(LPC_buf, st->cng_smth_NLSF_Q15, LPC_ORDER);
        // SKP_Silk_LPC_synthesis_filter (LPC_synthesis_filter.c:41-94): S[Order-1] newest
        i32* S = st->cng_synth_state;
        for (int k = 0; k < FRAME; k++) {
            i32 out32_Q10 = 0;
            for (int j = 0; j < LPC_ORDER; j++) out32_Q10 = smlawb(out32_Q10, S[LPC_ORDER - 1 - j], LPC_buf[j]);
            out32_Q10 = add_sat32(out32_Q10, smulwb(1 << 26, CNG_sig[k]));
            i32 out32 = rshift_round(out32_Q10, 10);
            for (int j = 0; j < LPC_ORDER - 1; j++) S[j] = S[j + 1];
            S[LPC_ORDER - 1] = lshift_sat32(out32_Q10, 4);
            CNG_sig[k] = (i16)sat16(out32);
        }
        for (int i = 0; i < FRAME; i++) signal[i] = (i16)sat16((i32)signal[i] + (i32)CNG_sig[i]);
    } else {
        for (int i = 0; i < LPC_ORDER; i++) st->cng_synth_state[i] = 0;
    }
}

// ---- SKP_Silk_SDK_Decode + SKP_Silk_decode_frame for one 20 ms frame ----------------------------------------
// rc[2]: range decoder states of the packet (initialised on the first frame), returns the SDK return code.
template <int KHZ> SB_FN i32 dec_silk_frame(DecStateT<KHZ>* st, DecCtrlT<KHZ>* c, RangeDec* rc, i32 (*Pulses)[DecCore<KHZ>::FRAME], const u8* pay0,
                                            int n0, const u8* pay1, int n1, int action, i16* pOut) {
    SB_DEC_DIMS(KHZ);
    i32 ret = 0;
    int used_bytes0 = 0;
    const int len_ref = st->seen_good ? FRAME : 480;
    if (st->moreInternalDecoderFrames == 0) st->nFramesDecoded = 0;
    c->LTP_scale_Q14 = 0;
    for (int i = 0; i < FRAME; i++) pOut[i] = 0;
    int do_plc = (action == 1);
    if (action != 1) {
        const int desp_type = action - 2;
        if (st->nFramesDecoded == 0) {
            rc_dec_init(&rc[0], pay0, n0);
            if (desp_type > 1) rc_dec_init(&rc[1], pay1, n1);
        }
        decode_parameters(st, c, &rc[0], Pulses[0], 0);
        if (desp_type > 1) decode_parameters(st, c, &rc[1], Pulses[1], 1);
        if (rc[0].error || (desp_type > 1 && rc[1].error)) {
            st->nBytesLeft[0] = 0;
            used_bytes0 = rc[0].bufLen;
            ret = (rc[0].error == -8) ? -11 : -12;
        } else {
            st->nFramesDecoded++;
            used_bytes0 = rc[0].bufLen - st->nBytesLeft[0];
            // inverse NSQ (decode_frame.c:104-241)
            i32 inv_gain_Q16 = inverse32_varq(imax(c->DeltaGains_Q16, 1), 32);
            i32 inv_gain_p1 = inv_gain_Q16, inv_gain_p2 = 65536 - inv_gain_Q16;
            i32 DeltaGains_p1 = inverse32_varq(imax(inv_gain_p1, 1), 32);
            i32 DeltaGains_p2 = inverse32_varq(imax(inv_gain_p2, 1), 32);
            i32 offset_Q10 = SB_T(quant_offsets_q10)[c->sigtype * 2 + c->QuantOffsetType];
            i32 offset_p1 = smulww(inv_gain_p1, offset_Q10), offset_p2 = smulww(inv_gain_p2, offset_Q10);
            i32 rand_seed = c->Seed;
            if (desp_type < 2) {
                for (int i = 0; i < FRAME; i++) {
                    int first = (i % (SUBFR << 1)) < SUBFR;
                    int use_p1 = desp_type == 0 ? first : !first;
                    rand_seed = lcg_rand(rand_seed);
                    i32 dither = rand_seed >> 31;
                    i32 q_Q10 = shl(Pulses[0][i], 10);
                    q_Q10 = addw(use_p1 ? offset_p1 : offset_p2, q_Q10);
                    i32 e = subw(q_Q10 ^ dither, dither);
                    st->exc_Q10[i] = smulww(use_p1 ? DeltaGains_p1 : DeltaGains_p2, e);
                }
            } else {
                for (int i = 0; i < FRAME; i++) {
                    rand_seed = lcg_rand(rand_seed);
                    i32 dither = rand_seed >> 31;
                    i32 q_Q10 = addw(shl(Pulses[0][i], 10), shl(Pulses[1][i], 10));
                    q_Q10 = addw(offset_p1 + offset_p2, q_Q10);
                    st->exc_Q10[i] = subw(q_Q10 ^ dither, dither);
                }
            }
            decode_core(st, c, pOut);
            plc_update(st, c);
            st->lossCnt = 0;
            st->prev_sigtype = c->sigtype;
            st->first_frame_after_reset = 0;
        }
    }
    if (do_plc) {
        plc_conceal(st, c, pOut);
        st->lossCnt++;
    }
    for (int i = 0; i < FRAME; i++) st->outBuf[i] = pOut[i];
    plc_glue_frames(st, pOut, len_ref);
    cng(st, c, pOut);
    st->lagPrev = c->pitchL[NB_SUBFR - 1];
    if (used_bytes0) {
        if (st->nBytesLeft[0] > 0 && st->FrameTermination == 1 && st->nFramesDecoded < 5) st->moreInternalDecoderFrames = 1;
        else st->moreInternalDecoderFrames = 0;
    }
    return ret;
}

// One group of four outputs of the synthesis filter bank (AGR_BWE_qmf.c:125-176) as int16 PCM, truncated and saturated
// (AGR_BWE_decode_frame_FLP.c:222-231): xx1 / xx2 = time-reversed band signals followed by the filter memories, i = even
// output-pair index.  The order of the float operations is the reference's; the groups are independent of each other,
// which is what the synthesis kernel uses (one group per lane and step).
SB_HD void qmf_synth_group(const float* xx1, const float* xx2, const float* a, int N2, int i, i16* pcm4) {
    enum { M2 = 32 };
    float y0 = 0, y1 = 0, y2 = 0, y3 = 0;
    float x10 = xx1[N2 - 2 - i], x20 = xx2[N2 - 2 - i];
    for (int j = 0; j < M2; j += 2) {
        float a0 = a[2 * j], a1 = a[2 * j + 1];
        float x11 = xx1[N2 - 1 + j - i], x21 = xx2[N2 - 1 + j - i];
        y0 = y0 + a0 * (x11 - x21);
        y1 = y1 + a1 * (x11 + x21);
        y2 = y2 + a0 * (x10 - x20);
        y3 = y3 + a1 * (x10 + x20);
        a0 = a[2 * j + 2];
        a1 = a[2 * j + 3];
        x10 = xx1[N2 + j - i];
        x20 = xx2[N2 + j - i];
        y0 = y0 + a0 * (x10 - x20);
        y1 = y1 + a1 * (x10 + x20);
        y2 = y2 + a0 * (x11 - x21);
        y3 = y3 + a1 * (x11 + x21);
    }
    const float y4[4] = {2.f * y0, 2.f * y1, 2.f * y2, 2.f * y3};
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const i32 t = trunc_i32((double)y4[q]);
        pcm4[q] = (i16)(t > 32767 ? 32767 : (t < -32768 ? -32768 : t));
    }
}

// The same group in the fixed-point build (AGR_BWE_qmf.c:134-168 with FIXED_POINT): int16 band signals, memories and
// coefficients (qmf_fix), int32 MAC16_16 sums in the reference's "multiply twice" order, PSHR32(y, 15) and
// SATURATE32(., 32767), which clamps to [-32767, 32767].  The sums wrap as the reference's int32 additions do.
SB_HD void qmf_synth_group_fix(const i16* xx1, const i16* xx2, const i16* a, int N2, int i, i16* pcm4) {
    enum { M2 = 32 };
    u32 y0 = 0, y1 = 0, y2 = 0, y3 = 0;
    i32 x10 = xx1[N2 - 2 - i], x20 = xx2[N2 - 2 - i];
    for (int j = 0; j < M2; j += 2) {
        i32 a0 = a[2 * j], a1 = a[2 * j + 1], na0 = (i16)(-a0);
        const i32 x11 = xx1[N2 - 1 + j - i], x21 = xx2[N2 - 1 + j - i];
        y0 += (u32)(a0 * x11); y0 += (u32)(na0 * x21);
        y1 += (u32)(a1 * x11); y1 += (u32)(a1 * x21);
        y2 += (u32)(a0 * x10); y2 += (u32)(na0 * x20);
        y3 += (u32)(a1 * x10); y3 += (u32)(a1 * x20);
        a0 = a[2 * j + 2]; a1 = a[2 * j + 3]; na0 = (i16)(-a0);
        x10 = xx1[N2 + j - i];
        x20 = xx2[N2 + j - i];
        y0 += (u32)(a0 * x10); y0 += (u32)(na0 * x20);
        y1 += (u32)(a1 * x10); y1 += (u32)(a1 * x20);
        y2 += (u32)(a0 * x11); y2 += (u32)(na0 * x21);
        y3 += (u32)(a1 * x11); y3 += (u32)(a1 * x21);
    }
    const u32 y4[4] = {y0, y1, y2, y3};
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const i32 t = (i32)(y4[q] + (1u << 14)) >> 15;
        pcm4[q] = (i16)(t > 32767 ? 32767 : (t < -32767 ? -32767 : t));
    }
}

// ---- scalar model of the synthesis kernel: AGR_Sate_qmf_synth (AGR_BWE_qmf.c:86-182), N = 2 * N2 = 4 * FRAME or 2 * FRAME,
// M = 64, into int16 PCM, float branch or (DEC_FIX) fixed-point branch.  low / high: the band signals dec_packet handed out.
template <int KHZ> SB_FN void dec_synth(DecStateT<KHZ>* st, const i16* low, const float* high, i16* pcm) {
    SB_DEC_DIMS(KHZ);
    enum { M2 = 32, N2MAX = 2 * FRAME };
    const int N2 = st->frames_per_packet * FRAME;
    if (st->arith == DEC_FIX) {
        i16 yy1[M2 + N2MAX], yy2[M2 + N2MAX];
        const i16* a = SB_T(qmf_fix);
        for (int i = 0; i < N2; i++) { yy1[i] = low[N2 - 1 - i]; yy2[i] = (i16)(i32)high[N2 - 1 - i]; }
        for (int i = 0; i < M2; i++) { yy1[N2 + i] = (i16)(i32)st->g0_mem[2 * i + 1]; yy2[N2 + i] = (i16)(i32)st->g1_mem[2 * i + 1]; }
        for (int i = 0; i < N2; i += 2) qmf_synth_group_fix(yy1, yy2, a, N2, i, pcm + 2 * i);
        for (int i = 0; i < M2; i++) { st->g0_mem[2 * i + 1] = (float)yy1[i]; st->g1_mem[2 * i + 1] = (float)yy2[i]; }
        return;
    }
    float xx1[M2 + N2MAX], xx2[M2 + N2MAX];
    const float* a = SB_T(qmf_flt);
    for (int i = 0; i < N2; i++) { xx1[i] = (float)low[N2 - 1 - i]; xx2[i] = high[N2 - 1 - i]; }
    for (int i = 0; i < M2; i++) { xx1[N2 + i] = st->g0_mem[2 * i + 1]; xx2[N2 + i] = st->g1_mem[2 * i + 1]; }
    for (int i = 0; i < N2; i += 2) qmf_synth_group(xx1, xx2, a, N2, i, pcm + 2 * i);
    for (int i = 0; i < M2; i++) { st->g0_mem[2 * i + 1] = xx1[i]; st->g1_mem[2 * i + 1] = xx2[i]; }
}

// ---- AGR_Bwe_decode_frame_FLP (AGR_BWE_decode_frame_FLP.c:41-130): one 20 ms high-band frame ------------------------
// hb4: the 4 coded bytes (ignored on loss); res_Q10: low-band excitation of the frame (Q10), nullptr = all zero -- the
// reference works on a float copy of (res >> 10), converted here where it is used.
template <int SF, int KHZ> SB_FN void hb_decode_frame_t(DecStateT<KHZ>* st, const u8* hb4, float* OutHigh, const i32* res_Q10, int lostflag) {
    // SF = sub-frame length: the core's SUBFR (40 or 80), or 2 * SUBFR with joint_mode 1.  The buffers hold at least
    // 80 samples, the size the 16 kHz streams' instantiations were measured with.
    enum { LEN = SF > 80 ? SF : 80 };
    float QHB_LSP[HB_ORDER], QGain[4], HB_PredCoef[HB_ORDER], HB_LPCRes[LEN];
    float sLPC[16 + LEN];
    if (lostflag == 1 || lostflag == 2) {
        for (int i = 0; i < HB_ORDER; i++) QHB_LSP[i] = st->hb_prev_NLSFq[i];
        for (int s = 0; s < 4; s++) QGain[s] = st->hb_prev_Gain;
        st->hb_lossCnt++;
    } else {
        u32 w = ((u32)hb4[0] << 24) | ((u32)hb4[1] << 16) | ((u32)hb4[2] << 8) | (u32)hb4[3];
        int hb_idx = (w >> 20) & 0xFFF;
        int idx1 = hb_idx & 0xFF, idx2 = hb_idx >> 8;
        for (int i = 0; i < HB_ORDER; i++) QHB_LSP[i] = SB_T(hb_lsp_cb1_flt)[idx1 * HB_ORDER + i] + SB_T(hb_lsp_cb2_flt)[idx2 * HB_ORDER + i];
        for (int s = 0; s < 4; s++) QGain[s] = SB_T(hb_gain_cb_flt)[(w >> (15 - 5 * s)) & 31];
        if (st->hb_first) {
            for (int i = 0; i < HB_ORDER; i++) st->hb_prev_NLSFq[i] = QHB_LSP[i];
            st->hb_prev_Gain = QGain[3];
        }
        st->hb_lossCnt = 0;
    }
    // SKP_Silk_NLSF2A_stable_FLP (wrappers_FLP.c:54-73)
    {
        i32 NLSF_fix[HB_ORDER];
        i16 a_fix_Q12[HB_ORDER];
        for (int i = 0; i < HB_ORDER; i++) NLSF_fix[i] = float2int((double)(QHB_LSP[i] * 32768.0f));
        nlsf2a_stable(a_fix_Q12, NLSF_fix, HB_ORDER);
        for (int i = 0; i < HB_ORDER; i++) HB_PredCoef[i] = (float)a_fix_Q12[i] / 4096.0f;
    }
    for (int i = 0; i < 16; i++) sLPC[i] = st->hb_sLPC[i];
    float* p_out = OutHigh;
    for (int s = 0; s < 4; s++) {
        for (int i = 0; i < SF; i++) {
            const float res_f = res_Q10 ? (float)(res_Q10[s * SF + i] >> 10) : 0.0f;
            HB_LPCRes[i] = (float)(-0.7 * (double)QGain[s] * (double)res_f);
        }
        // AGR_Sate_LPC_synthesizer (AGR_BWE_LPC_synthesizer.c:29-52)
        for (int i = 0; i < SF; i++) {
            float LPC_pred = 0.0f;
            for (int j = 0; j < HB_ORDER; j++) LPC_pred = LPC_pred + sLPC[16 + i - j - 1] * HB_PredCoef[j];
            p_out[i] = HB_LPCRes[i] + LPC_pred;
            sLPC[16 + i] = p_out[i];
        }
        for (int i = 0; i < 16; i++) sLPC[i] = sLPC[SF + i];
        p_out += SF;
    }
    for (int i = 0; i < 16; i++) st->hb_sLPC[i] = sLPC[i];
    if (lostflag == 0 || lostflag == 4 || lostflag == 3) {
        st->hb_prev_Gain = QGain[3];
        for (int i = 0; i < HB_ORDER; i++) st->hb_prev_NLSFq[i] = QHB_LSP[i];
    }
    st->hb_first = 0;
}

template <int KHZ> SB_FN void hb_decode_frame(DecStateT<KHZ>* st, const u8* hb4, float* OutHigh, const i32* res_Q10, int lostflag) {
    SB_DEC_DIMS(KHZ);
    if (st->hb_frame == FRAME) hb_decode_frame_t<SUBFR>(st, hb4, OutHigh, res_Q10, lostflag);
    else hb_decode_frame_t<2 * SUBFR>(st, hb4, OutHigh, res_Q10, lostflag);
}

// ---- AGR_Bwe_decode_frame_FIX (AGR_BWE_decode_frame_FIX.c:40-115): one 20 ms high-band frame, fixed-point build --------
// Same arguments; the int16 output goes to OutHigh as float (exact), which the synthesis stage turns back into int16.
// res_Q10 == nullptr: all-zero excitation, which is what the reference's memset of MAX_INTERNAL_FRAME_SIZE excitation words
// on a lost high band (:65) leaves for every frame of the packet.  Its AGR_Sate_PLC_interp_HB_parameters_fix and the loss
// branch at :82-88 are unreachable and have no counterpart here.
template <int SF, int KHZ> SB_FN void hb_decode_frame_fix_t(DecStateT<KHZ>* st, const u8* hb4, float* OutHigh, const i32* res_Q10, int lostflag) {
    enum { FOLDING_GAIN_FIX = 2867 };   // 0.7 in Q12
    i32 QHB_LSP_Q15[HB_ORDER];
    i16 A_Q12[HB_ORDER];
    const bool lost = lostflag == 1 || lostflag == 2;
    const u32 w = lost ? 0u : ((u32)hb4[0] << 24) | ((u32)hb4[1] << 16) | ((u32)hb4[2] << 8) | (u32)hb4[3];
    const i32 prev_gain = st->hb_prev_Gain_fix;
    // gain of sub-frame s: the previous frame's last one on loss (looked up where it is used: no array in local memory)
    auto QGain = [&](int s) -> i32 { return lost ? prev_gain : SB_T(hb_gain_cb_fix)[(w >> (15 - 5 * s)) & 31]; };
    if (lost) {
        for (int i = 0; i < HB_ORDER; i++) QHB_LSP_Q15[i] = st->hb_prev_NLSF_Q15[i];
        st->hb_lossCnt++;
    } else {
        int hb_idx = (w >> 20) & 0xFFF;
        int idx1 = hb_idx & 0xFF, idx2 = hb_idx >> 8;
        // AGR_Sate_lsp_dequant_highband (AGR_BWE_quant_highband.c:106-121)
        for (int i = 0; i < HB_ORDER; i++)
            QHB_LSP_Q15[i] = (i32)SB_T(hb_lsp_cb1_fix)[idx1 * HB_ORDER + i] + (i32)SB_T(hb_lsp_cb2_fix)[idx2 * HB_ORDER + i];
        if (st->hb_first) {
            for (int i = 0; i < HB_ORDER; i++) st->hb_prev_NLSF_Q15[i] = QHB_LSP_Q15[i];
            st->hb_prev_Gain_fix = QGain(3);
        }
        st->hb_lossCnt = 0;
    }
    // the reference converts the same LSPs once per sub-frame
    nlsf2a_stable(A_Q12, QHB_LSP_Q15, HB_ORDER);
    // AGR_Sate_LPC_synthesis_filter_fix (AGR_BWE_LPC_synthesizer.c:56-136): its little-endian branch accumulates
    // A_Q12[0] * S[7], A_Q12[1] * S[6], ... with SMLAWB / SMLAWT, i.e. smlawb in coefficient order
    i32 S[HB_ORDER];
    for (int i = 0; i < HB_ORDER; i++) S[i] = st->hb_synth_Q14[i];
    for (int s = 0; s < 4; s++) {
        const i32 Gain_Q16 = -FOLDING_GAIN_FIX * QGain(s);
        for (int k = 0; k < SF; k++) {
            i32 out32_Q10 = 0;
#pragma unroll
            for (int j = 0; j < HB_ORDER; j++) out32_Q10 = smlawb(out32_Q10, S[HB_ORDER - 1 - j], A_Q12[j]);
            out32_Q10 = add_sat32(out32_Q10, smulww(Gain_Q16, res_Q10 ? res_Q10[s * SF + k] : 0));
#pragma unroll
            for (int j = 0; j < HB_ORDER - 1; j++) S[j] = S[j + 1];
            S[HB_ORDER - 1] = lshift_sat32(out32_Q10, 4);
            OutHigh[s * SF + k] = (float)sat16(rshift_round(out32_Q10, 10));
        }
    }
    for (int i = 0; i < HB_ORDER; i++) st->hb_synth_Q14[i] = S[i];
    if (lostflag == 0 || lostflag == 4 || lostflag == 3) {
        st->hb_prev_Gain_fix = QGain(3);
        for (int i = 0; i < HB_ORDER; i++) st->hb_prev_NLSF_Q15[i] = QHB_LSP_Q15[i];
    }
    st->hb_first = 0;
}

// Out of line on the device: inlined, it tipped the float path's dec_packet out of the decode kernel (a call per packet).
template <int KHZ>
#ifdef __CUDACC__
__host__ __device__ __noinline__
#else
inline
#endif
void hb_decode_frame_fix(DecStateT<KHZ>* st, const u8* hb4, float* OutHigh, const i32* res_Q10, int lostflag) {
    SB_DEC_DIMS(KHZ);
    if (st->hb_frame == FRAME) hb_decode_frame_fix_t<SUBFR>(st, hb4, OutHigh, res_Q10, lostflag);
    else hb_decode_frame_fix_t<2 * SUBFR>(st, hb4, OutHigh, res_Q10, lostflag);
}

// A payload outliving its packet.  The reference keeps the range decoders (with their own copy of the payload) in the
// persistent state (structs.h:85-92, 295-303) and re-initialises them only when the previous packet is finished.  A
// corrupted packet whose last frame terminator decodes as "more frames" (with bytes left) therefore makes the following
// calls continue in the OLD payload, up to 5 frames, ignoring the low-band bytes they are given
// (SKP_Silk_dec_API.c:104-124, decode_frame.c:88-97).  Valid streams never get there; to behave identically on corrupted
// ones the payload copies are kept here, in storage that is only touched in that case.
struct DecStale {
    u8 pay[2][MAX_PAYLOAD + 8];
};

// ---- AGR_Sate_Decoder_Decode / AGR_Sate_decode_process (AGR_BWE_decode_frame_FLP.c:134-232) --------------------------
template <int KHZ> struct DecPacketWorkT {
    SB_DEC_DIMS(KHZ);
    DecCtrlT<KHZ> c;
    i32 Pulses[2][FRAME];
    u8 pay[2][MAX_PAYLOAD + 8];
    u8 act;                     // activity flags of the packet (sb_activity.cuh): bit f VAD flag, bit 2 + f concealed; in padding
    alignas(16) i16 lowout[2 * FRAME];
    i32 res_Q10[2 * FRAME];
    alignas(16) float OutHigh[2 * FRAME];
};
typedef DecPacketWorkT<8> DecPacketWork;
typedef DecPacketWorkT<16> DecPacketWork32;

// Band signals handed from the decoder kernel to the synthesis-filter-bank kernel: int16 low band and float high band of
// the packet (16-byte aligned on the device; a DEC_FIX stream's high band holds int16 values).
struct DecBands { i16* low; float* high; };

// bits/cap: payload row as handed in by the caller; nb: {n0, n1} (not modified); returns the reference's return code.
// Everything up to the synthesis filter bank: on 0 the band signals are in `bands`, and dec_synth (the synthesis kernel)
// turns them into PCM.
// CORE (core output): the SILK core's PCM is the result.  bands->low is the caller's PCM row (nf * FRAME samples, any
// 2-byte alignment), bands->high is unused, and the high band is not decoded: it reads the core's excitation, but nothing
// in the core reads it, so the row is the low band the reference hands to its synthesis filter bank (AGR_Sate_qmf_synth's
// first argument) for the same packets.  Checks, return codes, concealment and activity flags are the full decoder's.
template <int KHZ, bool CORE = false>
SB_FN i32 dec_packet(DecStateT<KHZ>* st, DecPacketWorkT<KHZ>* W, const u8* bits, int cap, const i16* nb_in, i32 lostflag, DecStale* stale,
                     const DecBands* bands) {
    SB_DEC_DIMS(KHZ);
    if (nb_in[0] <= 0) return -1;
    if (lostflag < 1 || lostflag > 4) return -1;
    // frame control starts from zeros: after a rejected (corrupted) frame a few of its fields are read before anything
    // has written them (the reference reads uninitialised stack there); zeros keep host and device builds deterministic
    memset(&W->c, 0, sizeof(W->c));
    i16 nb[2] = {nb_in[0], nb_in[1]};
    const int nf = st->frames_per_packet, half = nf * FRAME, F = st->hb_frame, nhb = half / F, hb_bytes = 4 * nhb;
    i32 hb_off = dec_split_lengths(nb, lostflag, hb_bytes);
    int n0 = nb[0], n1 = nb[1];
    if (n0 < 0 || n1 < 0 || n0 + n1 > cap || hb_off > cap) return -1;
    // the high-band bytes are read from the row (lostflag 3 / 4): a declared total beyond the row is rejected, never followed
    if ((lostflag == 3 || lostflag == 4) && (hb_off < 0 || hb_off + hb_bytes > cap)) return -1;
    RangeDec rc[2];
    for (int k = 0; k < 2; k++) {   // fully defined even for a description this packet does not carry
        rc[k].base_Q32 = 0; rc[k].range_Q16 = 0; rc[k].bufferIx = 0; rc[k].error = 0; rc[k].bufLen = 0; rc[k].buf = W->pay[k];
    }
    const bool cont = st->moreInternalDecoderFrames != 0;   // only after a corrupted packet, see DecStale
    if (cont) {
        for (int k = 0; k < 2; k++) {
            for (int i = 0; i < MAX_PAYLOAD + 8; i++) W->pay[k][i] = stale->pay[k][i];
            rc[k].base_Q32 = st->rc_base_Q32[k]; rc[k].range_Q16 = st->rc_range_Q16[k];
            rc[k].bufferIx = st->rc_bufferIx[k]; rc[k].error = st->rc_error[k]; rc[k].bufLen = st->rc_bufLen[k];
            rc[k].buf = W->pay[k];
        }
    }
    // zero-padded private copies of the description payloads (the range decoder may read up to 4 bytes past the end)
    if (lostflag != 1 && !cont) {
        int c0 = imin(n0, MAX_PAYLOAD), c1 = imin(n1, MAX_PAYLOAD);
        for (int i = 0; i < c0; i++) W->pay[0][i] = bits[i];
        for (int i = c0; i < c0 + 8; i++) W->pay[0][i] = 0;
        if (lostflag == 4) {
            for (int i = 0; i < c1; i++) W->pay[1][i] = bits[n0 + i];
            for (int i = c1; i < c1 + 8; i++) W->pay[1][i] = 0;
        }
    }
    for (int i = 0; i < half; i++) { if (!CORE) W->res_Q10[i] = 0; W->lowout[i] = 0; }
    W->act = 0;
    for (int f = 0; f < nf; f++) {
        i32 ret;
        // a lost packet's frames are concealed; a received frame reports the VAD flag it carried
        if (lostflag == 1) W->act |= (u8)(4 << f);
        if (!st->seen_good && lostflag == 1) {
            // Loss before any frame was decoded: the reference conceals at its start-up rate of 24 kHz from an all-zero
            // state and resamples to the API rate -> silence; only these side effects survive the later switch to the core rate.
            for (int i = 0; i < 480; i++) st->plc_rand_seed = lcg_rand(st->plc_rand_seed);
            st->lossCnt++;
            st->plc_conc_energy = 0; st->plc_conc_energy_shift = 0; st->plc_last_frame_lost = 1;
            ret = 0;
        } else {
            if (lostflag != 1 && (n0 > MAX_PAYLOAD)) { return -11; }
            ret = dec_silk_frame(st, &W->c, rc, W->Pulses, W->pay[0], n0, W->pay[1], n1, lostflag, W->lowout + f * FRAME);
        }
        if (ret < 0) return ret;
        if (lostflag != 1) W->act |= (u8)((st->vadFlag & 1) << f);
        if (!CORE) for (int i = 0; i < FRAME; i++) W->res_Q10[f * FRAME + i] = st->exc_Q10[i];
    }
    if (st->moreInternalDecoderFrames) {     // the payload outlives this call
        for (int k = 0; k < 2; k++) {
            for (int i = 0; i < MAX_PAYLOAD + 8; i++) stale->pay[k][i] = W->pay[k][i];
            st->rc_base_Q32[k] = rc[k].base_Q32; st->rc_range_Q16[k] = rc[k].range_Q16;
            st->rc_bufferIx[k] = rc[k].bufferIx; st->rc_error[k] = rc[k].error; st->rc_bufLen[k] = rc[k].bufLen;
        }
    }
    if (CORE) {
#ifdef __CUDA_ARCH__
        if ((((size_t)bands->low) & 15) == 0) {
            const int4* sl = reinterpret_cast<const int4*>(W->lowout);
            int4* dl = reinterpret_cast<int4*>(bands->low);
            for (int i = 0; i < half / 8; i++) dl[i] = sl[i];
            return 0;
        }
#endif
        for (int i = 0; i < half; i++) bands->low[i] = W->lowout[i];
        return 0;
    }
    const int hb_lost = (lostflag == 1 || lostflag == 2);
    const bool fix = st->arith == DEC_FIX;
    for (int f = 0; f < nhb; f++) {
        // App. A Q12: with the high band lost, the reference's memset after the first high-band frame wipes the excitation
        // of the rest of the packet -- later frames are synthesised from zeros.  The fixed-point build's memset comes before
        // the first frame's synthesis, so there every frame is.
        const i32* res = (hb_lost && (f > 0 || fix)) ? nullptr : W->res_Q10 + f * F;
        u8 hb4[4] = {0, 0, 0, 0};
        if (!hb_lost) for (int i = 0; i < 4; i++) hb4[i] = bits[hb_off + 4 * f + i];
        if (fix) hb_decode_frame_fix(st, hb4, W->OutHigh + f * F, res, lostflag);
        else hb_decode_frame(st, hb4, W->OutHigh + f * F, res, lostflag);
    }
    // the 64-tap synthesis filter bank has no recurrence: on the device it runs as its own kernel
#ifdef __CUDA_ARCH__
    const int4* sl = reinterpret_cast<const int4*>(W->lowout);
    int4* dl = reinterpret_cast<int4*>(bands->low);
    for (int i = 0; i < half / 8; i++) dl[i] = sl[i];
    const float4* sh = reinterpret_cast<const float4*>(W->OutHigh);
    float4* dh = reinterpret_cast<float4*>(bands->high);
    for (int i = 0; i < half / 4; i++) dh[i] = sh[i];
#else
    for (int i = 0; i < half; i++) { bands->low[i] = W->lowout[i]; bands->high[i] = W->OutHigh[i]; }
#endif
    return 0;
}

// The whole packet on one thread (host model): the decode kernel's dec_packet, then, for an accepted packet, the synthesis
// kernel's dec_synth into vout (2 * nf * FRAME samples).  A core_only stream takes the core-output decode kernel's
// dec_packet straight into vout (nf * FRAME samples).  Without DecStale storage a packet that would continue in the
// previous payload resynchronises on its own bytes instead.
template <int KHZ>
SB_FN i32 dec_packet(DecStateT<KHZ>* st, DecPacketWorkT<KHZ>* W, i16* vout, const u8* bits, int cap, const i16* nb_in, i32 lostflag,
                     DecStale* stale = nullptr) {
    SB_DEC_DIMS(KHZ);
    DecStale discard;
    if (!stale) { st->moreInternalDecoderFrames = 0; stale = &discard; }
    if (st->core_only) {
        const DecBands out = {vout, nullptr};
        return dec_packet<KHZ, true>(st, W, bits, cap, nb_in, lostflag, stale, &out);
    }
    i16 low[2 * FRAME];
    float high[2 * FRAME];
    const DecBands bands = {low, high};
    const i32 r = dec_packet(st, W, bits, cap, nb_in, lostflag, stale, &bands);
    if (r == 0) dec_synth(st, low, high, vout);
    return r;
}

}  // namespace sb
