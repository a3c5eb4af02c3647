// solo_b200 -- one SOLO packet (40 ms, 16 kHz) through the encoder: QMF split, two SILK frames with the
// MD noise-shaping quantiser, two high-band frames, payload assembly [MD1 | MD2 | HB].
// enc_packet is the scalar model of the device pipeline, stage by stage: band split, voice activity, core analysis,
// high-band analysis, shaping filters, gains, prefilter, quantiser, entropy coding.  The band split (sharing
// qmf_output_pair with its kernel), the core and high-band analysis and the quantiser have scalar forms here, the
// specification of what those kernels run (sb_coop.cuh, sb_nsq_warp.cuh); voice activity, shaping filters, gains,
// prefilter and the entropy-coding steps are the functions their kernels call.
// Reference: /root/reference/JC1_SDK_SRC_ARM/src/libBWE/AGR_BWE_encode_frame_FIX.c:8-174, AGR_BWE_qmf.c:38-80,
// AGR_BWE_find_HB_LPC_FIX.c:4-49, AGR_BWE_quant_highband.c:23-147, AGR_BWE_SDK_API.c:11-152,
// libSATECodec/SKP_Silk_enc_API.c:127-273, SKP_Silk_encode_frame_FIX.c:34-327, SKP_Silk_control_codec_FIX.c:232-389.
#pragma once
#include "sb_enc_entropy.cuh"
#include "sb_enc_front.cuh"
#include "sb_enc_pred.cuh"
#include "sb_enc_shape.cuh"
#include "sb_nsq.cuh"

namespace sb {

// ---- per-packet control: what SKP_Silk_SDK_Encode reads from the handle's encControl at the start of every packet
// (enc_API.c:161-191) and SKP_Silk_control_encoder_FIX applies (control_codec_FIX.c:56-130) -------------------------
// rate_bps >= 1: the user rate; the SILK core gets it less (1600 * 20) / bwe_framesize_ms (AGR_BWE_SDK_API.c:118),
// clamped to [5000, 100000], and both SNR targets follow (setup_rate, :319-389).  dtx 0 / 1: useDTX.  loss_perc 0-100:
// the expected packet loss of LTP_scale_ctrl.  A value outside those ranges (-1 by convention) leaves its setting as it is.
// Takes effect from the next packet; both frames of a 40 ms packet see the same settings, as in the reference.
SB_FN void enc_set_control(EncSilk* st, i32 rate_bps, i32 dtx, i32 loss_perc) {
    if (rate_bps >= 1) {
        const i32 silk_rate = limit(rate_bps - (st->hb_frame == 320 ? 800 : 1600), 5000, 100000);
        st->targetRate_bps = silk_rate;
        // setup_rate: both tables end at 100000, so each search finds its interval
        const i32* rt = SB_T(target_rate_table_nb);
        const i32* snr = SB_T(snr_table_q1);
        const i32 md_rate = silk_rate / 2;
        for (int k = 1; k < 8; k++) {
            if (md_rate < rt[k]) {
                i32 frac_Q6 = shl(md_rate - rt[k - 1], 6) / (rt[k] - rt[k - 1]);
                st->SNRPerMD_dB_Q7 = shl(snr[k - 1], 6) + mulw(frac_Q6, snr[k] - snr[k - 1]);
                break;
            }
        }
        for (int k = 1; k < 8; k++) {
            if (silk_rate <= rt[k]) {
                i32 frac_Q6 = shl(silk_rate - rt[k - 1], 6) / (rt[k] - rt[k - 1]);
                st->SNR_dB_Q7 = shl(snr[k - 1], 6) + mulw(frac_Q6, snr[k] - snr[k - 1]);
                break;
            }
        }
    }
    if (dtx == 0 || dtx == 1) st->useDTX = dtx;
    if (loss_perc >= 0 && loss_perc <= 100) st->packetLoss_perc = loss_perc;
}

// ---- Init: AGR_Sate_Encoder_Init + SKP_Silk_init_encoder_FIX + first SKP_Silk_control_encoder_FIX --------------
// enc_state_fields sets what Init sets on a zeroed state; enc_state_init zeroes the state first (the device's reset kernel
// zeroes it with word stores instead of this byte-wise memset, then calls enc_state_fields).
SB_FN void enc_state_fields(EncState* st, i32 targetRate_bps, i32 dtx_enable, i32 useMDIndex, i32 framesize_ms, i32 joint_hb) {
    st->frames_per_packet = framesize_ms == 20 ? 1 : 2;
    st->hb_frame = joint_hb ? 320 : HB_FRAME;
    // the Init settings go through the per-packet control; the reference starts with no expected loss (AGR_BWE_SDK_API.c:38)
    enc_set_control(st, targetRate_bps <= 0 ? 15600 : targetRate_bps, dtx_enable ? 1 : 0, 0);
    st->useMDIndex = useMDIndex;
    st->variable_HP_smth1_Q15 = 200844;
    st->variable_HP_smth2_Q15 = 200844;
    st->first_frame_after_reset = 1;
    vad_init(&st->vad);
    for (int i = 0; i < 3; i++) st->nsq[i].prev_inv_gain_Q16 = 65536;
    // setup_fs (control_codec_FIX.c:232-317): only the centre NSQ gets lagPrev = 100 (App. A Q5)
    st->prevLag = 100;
    st->prev_sigtype = 1;
    st->pf_lagPrev = 100;
    st->LastGainIndex = 1;
    st->nsq[0].lagPrev = 100;
    st->hb_first = 1;
}
// Returns 0, or -1 for a configuration the reference rejects / this build does not cover.
SB_FN int enc_state_init(EncState* st, i32 targetRate_bps, i32 dtx_enable, i32 useMDIndex, i32 framesize_ms = 40, i32 joint_hb = 0) {
    memset(st, 0, sizeof(EncState));
    enc_state_fields(st, targetRate_bps, dtx_enable, useMDIndex, framesize_ms, joint_hb);
    return 0;
}

// One low-band / high-band output pair of the 64-tap QMF analysis (AGR_BWE_qmf.c:66-79): x = [63 history | N new]
// samples (already >> 1), aa = the 64 coefficients.  Products are summed mod 2^32, so any order gives the same bits.
SB_HD void qmf_output_pair(const i16* x, const i16* aa, int k, i16* lo, i16* hi) {
    enum { M = 64 };
    const int i = 2 * k;
    const i16* x2 = x + M - 1;
    i32 y1k = 0, y2k = 0;
#pragma unroll 4
    for (int j = 0; j < M / 2; j += 2) {
        i32 a0 = aa[M - j - 1], a1 = aa[M - j - 2];
        i32 s0 = (i16)(x[i + j] + x2[i - j]), d0 = (i16)(x[i + j] - x2[i - j]);
        i32 s1 = (i16)(x[i + j + 1] + x2[i - j - 1]), d1 = (i16)(x[i + j + 1] - x2[i - j - 1]);
        y1k = addw(y1k, a0 * s0);
        y2k = subw(y2k, a0 * d0);
        y1k = addw(y1k, a1 * s1);
        y2k = addw(y2k, a1 * d1);
    }
    i32 v1 = addw(y1k, 16384) >> 15, v2 = addw(y2k, 16384) >> 15;
    *lo = (i16)(v1 > 32767 ? 32767 : (v1 < -32767 ? -32767 : v1));
    *hi = (i16)(v2 > 32767 ? 32767 : (v2 < -32767 ? -32767 : v2));
}

// ---- AGR_Sate_qmf_decomp (AGR_BWE_qmf.c:38-80), N = 640 or 320, M = 64, fixed point ------------------------------
// (scalar model of the band-split kernel, which computes the same output pairs with qmf_output_pair)
SB_FN void qmf_decomp(const i16* xx, i16* y1, i16* y2, i16* mem, int N) {
    enum { M = 64 };
    i16 x[PACKET + M - 1];
    const i16* aa = SB_T(qmf_fix);
    for (int i = 0; i < M - 1; i++) x[i] = mem[M - i - 2];
    for (int i = 0; i < N; i++) x[i + M - 1] = (i16)(xx[i] >> 1);
    for (int i = 0; i < M - 1; i++) mem[i] = x[N + M - 2 - i];   // == xx[N - i - 1] >> 1
    for (int k = 0; k < N / 2; k++) qmf_output_pair(x, aa, k, &y1[k], &y2[k]);
}

// ---- AGR_Sate_lsp_quant_highband (AGR_BWE_quant_highband.c:23-104) ----------------------------------------------
// Distances of lsp to first-stage code vector i (squared error) and of the first stage's residual to second-stage code
// vector i (Laroia-weighted); the high-band kernel evaluates one code vector per lane (c_hb_analyse_frame, sb_coop.cuh).
SB_HD i32 hb_lsp_dist1(const i32* lsp, int i) {
    const i16* cb1 = SB_T(hb_lsp_cb1_fix);
    i32 dist = 0;
#pragma unroll
    for (int j = 0; j < HB_ORDER; j++) { const i32 t = lsp[j] - cb1[i * HB_ORDER + j]; dist = smlabb(dist, t, t); }
    return dist;
}
SB_HD i32 hb_lsp_dist2(const i32* res, const i32* weight, int i) {
    const i16* cb2 = SB_T(hb_lsp_cb2_fix);
    i32 dist = 0;
#pragma unroll
    for (int j = 0; j < HB_ORDER; j++) { const i32 t = subw(res[j], cb2[i * HB_ORDER + j]); dist = smlawb(dist, smulbb(t, t), weight[j]); }
    return dist;
}
SB_FN i32 hb_lsp_quant(i32* lsp) {
    i32 weight[HB_ORDER];
    nlsf_vq_weights_laroia(weight, lsp, HB_ORDER);
    const i16* cb1 = SB_T(hb_lsp_cb1_fix);
    const i16* cb2 = SB_T(hb_lsp_cb2_fix);
    i32 min_dist = SB_I32_MAX; int idx1 = 0;
    for (int i = 0; i < 256; i++) {
        const i32 dist = hb_lsp_dist1(lsp, i);
        if (dist < min_dist) { min_dist = dist; idx1 = i; }
    }
    for (int i = 0; i < HB_ORDER; i++) lsp[i] -= cb1[idx1 * HB_ORDER + i];
    i32 best = SB_I32_MAX; int idx2 = 0;
    for (int i = 0; i < 16; i++) {
        const i32 dist = hb_lsp_dist2(lsp, weight, i);
        if (dist < best) { best = dist; idx2 = i; }
    }
    for (int i = 0; i < HB_ORDER; i++) lsp[i] = (i32)cb1[idx1 * HB_ORDER + i] + (i32)cb2[idx2 * HB_ORDER + i];
    return shl(idx2, 8) + idx1;
}

// ---- AGR_Bwe_encode_frame_FIX (AGR_BWE_encode_frame_FIX.c:8-82), split in two because the gain needs the low-band
// excitation produced by the noise-shaping quantiser: (1) buffer update, LPC analysis, LSP VQ, per-sub-frame residual
// energy of the high band; (2) gain = 16*sqrt(E_hb)/sqrt(E_lb_exc), 32-level VQ, bit packing (12 + 4*5 bits, MSB first).
template <int F> SB_FN void hb_analyse_frame_t(EncCore* st, const i16* high, i32* lsp_idx_out, i32* nrg0_out) {
    const int LPCF = 80, SF = F >> 2;   // LPC block and sub-frame lengths; F = frame length (compile-time: the loops unroll)
    for (int i = 0; i < F; i++) st->x_hb_buf[F + 40 + i] = high[i];
    // AGR_Sate_find_HB_LPC_FIX: 4 blocks of (80 + 8) samples, hop 80, starting 8 samples before the frame
    i16 LPC_in_pre[4 * (LPCF + HB_ORDER)];
    {
        const i16* xp = st->x_hb_buf + F - HB_ORDER;
        i16* d = LPC_in_pre;
        for (int k = 0; k < 4; k++) {
            for (int i = 0; i < LPCF + HB_ORDER; i++) d[i] = xp[i];
            d += LPCF + HB_ORDER;
            xp += LPCF;
        }
    }
    i32 NLSF_Q15[HB_ORDER], interp, prev_dummy[HB_ORDER];
    for (int i = 0; i < HB_ORDER; i++) prev_dummy[i] = 0;
    find_lpc(NLSF_Q15, &interp, prev_dummy, 0, HB_ORDER, LPC_in_pre, LPCF + HB_ORDER);
    *lsp_idx_out = hb_lsp_quant(NLSF_Q15);
    i16 coef[HB_ORDER], exc[2 * SUBFR];
    nlsf2a_stable(coef, NLSF_Q15, HB_ORDER);
    const i16* p_hb = st->x_hb_buf + F;
    for (int sub = 0; sub < 4; sub++) {
        lpc_analysis_filter_zero_state(p_hb, coef, exc, SF, HB_ORDER);
        i32 nrg0 = 0;
        for (int i = 0; i < SF; i++) nrg0 = addw(nrg0, (i32)exc[i] * (i32)exc[i]);
        nrg0_out[sub] = sqrt_approx(nrg0);
        p_hb += SF;
    }
    for (int i = 0; i < F + 40; i++) st->x_hb_buf[i] = st->x_hb_buf[F + i];
    st->hb_first = 0;
}
SB_FN void hb_analyse_frame(EncCore* st, const i16* high, i32* lsp_idx_out, i32* nrg0_out) {
    if (st->hb_frame == HB_FRAME) hb_analyse_frame_t<HB_FRAME>(st, high, lsp_idx_out, nrg0_out);
    else hb_analyse_frame_t<2 * HB_FRAME>(st, high, lsp_idx_out, nrg0_out);
}
// r16 = (int16)(low-band excitation Q10 >> 10), the only form in which AGR_BWE_encode_frame_FIX.c:56-58 uses it
// (sf = sub-frame length: 40, or 80 when one high-band frame spans both codec frames of the packet)
SB_FN void hb_pack_frame(i32 lsp_idx, const i32* nrg0, const i16* r16, u8* out4, int sf = SUBFR) {
    i32 gain_idx[4];
    for (int sub = 0; sub < 4; sub++) {
        i32 nrg1 = 0;
        for (int i = 0; i < sf; i++) nrg1 = smlabb(nrg1, r16[sub * sf + i], r16[sub * sf + i]);
        nrg1 = sqrt_approx(nrg1);
        i16 gain = (i16)(shl(nrg0[sub] + 1, 4) / (nrg1 + 1));
        i32 md = SB_I32_MAX; int gi = 0;
        for (int i = 0; i < 32; i++) {
            i16 t = (i16)(gain - SB_T(hb_gain_cb_fix)[i]);
            i32 dist = smulbb(t, t);
            if (dist < md) { md = dist; gi = i; }
        }
        gain_idx[sub] = gi;
    }
    u32 w = ((u32)lsp_idx & 0xFFF) << 20 | ((u32)gain_idx[0] << 15) | ((u32)gain_idx[1] << 10) | ((u32)gain_idx[2] << 5) | (u32)gain_idx[3];
    out4[0] = (u8)(w >> 24); out4[1] = (u8)(w >> 16); out4[2] = (u8)(w >> 8); out4[3] = (u8)w;
}

// Working set of the scalar core analysis (tests/hostsim); the analysis kernel's is CoopWork (sb_coop.cuh).
struct EncAnalysisWork {
    i16 low[PACKET / 2], high[PACKET / 2];   // band signals of the packet
    i16 pIn_HP[FRAME];
    i16 res_pitch[2 * FRAME + LA_PITCH];
};

// Start of a frame's analysis (encode_frame_FIX.c:34-75), shared with the core-analysis kernel (c_encode_frame_analysis,
// sb_coop.cuh): seed, the frame's voice activity (computed ahead by the VAD kernel: speech activity, four band qualities,
// tilt), high-pass filter of pIn into pIn_HP.
SB_HD void frame_analysis_begin(EncSilk* st, EncCtrl* c, i16* pIn_HP, const i16* pIn, i32 speech_activity_Q8, const i32* quality_Q15,
                                i32 tilt_Q15) {
    c->Seed = st->frameCounter++ & 3;
    st->speech_activity_Q8 = speech_activity_Q8;
    for (int b = 0; b < 4; b++) c->input_quality_bands_Q15[b] = quality_Q15[b];
    c->input_tilt_Q15 = tilt_Q15;
    hp_variable_cutoff(st, c, pIn_HP, pIn);
}
// what the next frame's analysis reads of this one (encode_frame_FIX.c:199-208)
SB_HD void frame_analysis_end(EncSilk* st, const EncCtrl* c) {
    st->prev_sigtype = c->sigtype;
    st->prevLag = c->pitchL[NB_SUBFR - 1];
    st->first_frame_after_reset = 0;
}

// SKP_Silk_encode_frame_FIX (encode_frame_FIX.c:34-131) up to the quantised NLSFs, for frame f of the packet: the scalar
// model of the core-analysis kernel (c_encode_frame_analysis).  Reads the frame's voice activity from scr and writes what
// the kernel writes there: c[f], x_hp[f], ar_Q24[f], shape_par[f], nlsf_Q15[f], lpc_in_pre[f], local_gains[f].
SB_FN void encode_frame_analysis(EncSilk* st, EncAnalysisWork* W, EncScratch* scr, int f) {
    EncCtrl* c = &scr->c[f];
    i16* x_frame = st->x_buf + FRAME;
    frame_analysis_begin(st, c, W->pIn_HP, W->low + f * FRAME, scr->vad_sa_Q8[f], scr->vad_quality_Q15[f], scr->vad_tilt_Q15[f]);
    for (int i = 0; i < FRAME; i++) x_frame[LA_SHAPE + i] = W->pIn_HP[i];  // LP_variable_cutoff is a copy (transition_frame_no == 0)
    find_pitch_lags(st, c, W->res_pitch, x_frame);
    noise_shape_analysis(st, c, W->res_pitch + FRAME, x_frame, scr->ar_Q24[f], scr->shape_par[f]);
    find_pred_coefs(st, c, W->res_pitch, scr, f);
    for (int i = 0; i < FRAME; i++) scr->x_hp[f][i] = x_frame[i];    // the prefilter's input: the frame as the analysis saw it
    for (int i = 0; i < FRAME + LA_SHAPE; i++) st->x_buf[i] = st->x_buf[FRAME + i];
    frame_analysis_end(st, c);
}

// scalar model of the core-analysis kernel (c_enc_packet_analysis): every frame of the packet
SB_FN void enc_packet_analysis(EncSilk* st, EncAnalysisWork* W, EncScratch* scr) {
    for (int f = 0; f < st->frames_per_packet; f++) encode_frame_analysis(st, W, scr, f);
}
// scalar model of the high-band kernel: every high-band frame of the packet
SB_FN void hb_analyse_packet(EncCore* st, const i16* high, EncScratch* scr) {
    const int nhb = st->frames_per_packet * FRAME / st->hb_frame;
    for (int f = 0; f < nhb; f++) hb_analyse_frame(st, high + f * st->hb_frame, &scr->hb_lsp_idx[f], scr->hb_nrg0[f]);
}
// the kernels between the analysis and the quantiser, which the device and the scalar model share: shaping filters,
// gain processing, prefilter
SB_FN void enc_packet_post_analysis(EncSilk* st, EncScratch* scr) {
    const int nf = st->frames_per_packet;
    for (int f = 0; f < nf; f++) for (int k = 0; k < NB_SUBFR; k++) shape_post_window(scr, f, k);
    gains_packet(st, scr, nf);
    prefilter_packet(st, scr, nf);
}

// ---- stage C: AGR_Sate_Encoder_Encode tail, in the three steps of one description k (0 or 1) that the entropy-coding
// kernel runs on thread k of a pair; all description stores come before any high-band store.  The payload row is
// [MD1 | MD2 | HB]; nBytesOut[0] = total, nBytesOut[1] = len(MD2) + high-band bytes.
// (1) range-code description k of every frame of the packet into buf (MAX_PAYLOAD bytes); rc stays live for step 2.
// Returns the byte count, *ok = 0 when the coder overflowed.
SB_HD int enc_code_description(RangeEnc* rc, u8* buf, EncCore* st, const EncScratch* scr, int k, int* ok) {
    const int nf = st->frames_per_packet;
    rc_enc_init(rc, buf, MAX_PAYLOAD);
    for (int f = 0; f < nf; f++) {
        encode_parameters(rc, st, &scr->c[f], k, f, scr->vadFlag[f], scr->q_md[f][k]);
        // frame terminator: MORE_FRAMES (1) while frames follow in this packet, LAST_FRAME (0) after the last one
        rc_encode(rc, f < nf - 1 ? 1 : 0, SB_T(frame_term_cdf));
    }
    int nb;
    rc_get_length(rc, &nb);
    *ok = rc->error ? 0 : 1;
    return nb;
}
// (2) with both descriptions' lengths and status: description 0 is kept when its own coder succeeded, description 1 when
// both did and they fit MAX_PAYLOAD (pnBytesOut[0] >= nMDBytes, encode_frame_FIX.c:245); a kept description is finished
// and copied to offset k ? nb0 : 0, bytes at or past out_cap dropped.  Returns the low-band bytes the packet carries:
// nb0 + nb1, or 0 for a rejected or DTX-dropped packet.
SB_HD int enc_store_description(RangeEnc* rc, const EncScratch* scr, int k, int nb0, int nb1, int ok0, int ok1, u8* out, i32 out_cap) {
    const int ok = ok0 && ok1 && nb0 + nb1 <= MAX_PAYLOAD;
    if (k == 0 ? ok0 : ok) {
        rc_enc_wrap_up(rc);
        const int off = k ? nb0 : 0, nb = k ? nb1 : nb0;
        for (int i = 0; i < nb; i++) if (off + i < out_cap) out[off + i] = rc->buf[i];
    }
    return (ok && !scr->dtx_drop) ? nb0 + nb1 : 0;
}
// (3) high-band frame k (if the packet has one) behind the lb low-band bytes -- so a rejected or dropped packet's
// high-band bytes land on top of its descriptions' -- and, for k = 0, the length fields.  Returns the packet's total size.
SB_HD int enc_store_high_band(const EncCore* st, const EncScratch* scr, int k, int lb, int nb1, u8* out, i32 out_cap, i16* nBytesOut) {
    const int nhb = st->frames_per_packet * FRAME / st->hb_frame, hb_bytes = 4 * nhb;
    if (k < nhb) {
        u8 hb[4];
        hb_pack_frame(scr->hb_lsp_idx[k], scr->hb_nrg0[k], &scr->r16[0][0] + k * st->hb_frame, hb, st->hb_frame >> 2);
        for (int i = 0; i < 4; i++) if (lb + 4 * k + i < out_cap) out[lb + 4 * k + i] = hb[i];
    }
    if (k == 0) {
        nBytesOut[0] = lb ? (i16)(lb + hb_bytes) : 0;
        nBytesOut[1] = lb ? (i16)(nb1 + hb_bytes) : 0;
    }
    return lb + hb_bytes;
}
// stage C on one thread: the kernel's two threads one after the other.  Returns min(out_cap, total).
SB_FN i32 enc_packet_finish(EncCore* st, const EncScratch* scr, u8 (*rcbuf)[MAX_PAYLOAD], u8* out, i32 out_cap, i16* nBytesOut) {
    RangeEnc rc[2];
    int nb[2], ok[2], lb = 0, total = 0;
    for (int k = 0; k < 2; k++) nb[k] = enc_code_description(&rc[k], rcbuf[k], st, scr, k, &ok[k]);
    for (int k = 0; k < 2; k++) lb = enc_store_description(&rc[k], scr, k, nb[0], nb[1], ok[0], ok[1], out, out_cap);
    for (int k = 0; k < 2; k++) total = enc_store_high_band(st, scr, k, lb, nb[1], out, out_cap, nBytesOut);
    return imin(out_cap, total);
}

// Whole packet on one thread: the scalar model of the device pipeline (tests/hostsim).
struct EncPacketWork {
    EncAnalysisWork a;
    EncScratch scr;
    NsqWork nsq;
    i32 r[FRAME];
    u8 rcbuf[2][MAX_PAYLOAD];   // both descriptions' coders are live at once
};
// band split and voice activity of the packet (the first two kernels)
SB_FN void enc_packet_bands(EncState* st, EncPacketWork* W, const i16* pcm) {
    const int nf = st->frames_per_packet;
    qmf_decomp(pcm, W->a.low, W->a.high, st->qmf_mem, nf * 2 * FRAME);
    vad_packet(&st->vad, W->a.low, nf, W->scr.vad_sa_Q8, W->scr.vad_quality_Q15, W->scr.vad_tilt_Q15);
}
// scalar model of the quantiser kernel, then the entropy coding
SB_FN i32 enc_packet_quantise_and_code(EncState* st, EncPacketWork* W, u8* out, i32 out_cap, i16* nBytesOut) {
    for (int f = 0; f < st->frames_per_packet; f++) {
        nsq_del_dec(st, &W->scr.c[f], &W->nsq, W->scr.xfw[f], (i8*)0, W->scr.q_md[f][0], W->scr.q_md[f][1], W->r);
        for (int i = 0; i < FRAME; i++) W->scr.r16[f][i] = (i16)(W->r[i] >> 10);
    }
    return enc_packet_finish(st, &W->scr, W->rcbuf, out, out_cap, nBytesOut);
}
// the device pipeline's stages in its order
SB_FN i32 enc_packet(EncState* st, EncPacketWork* W, const i16* pcm, u8* out, i32 out_cap, i16* nBytesOut) {
    enc_packet_bands(st, W, pcm);
    enc_packet_analysis(st, &W->a, &W->scr);
    hb_analyse_packet(st, W->a.high, &W->scr);
    enc_packet_post_analysis(st, &W->scr);
    return enc_packet_quantise_and_code(st, W, out, out_cap, nBytesOut);
}

}  // namespace sb
