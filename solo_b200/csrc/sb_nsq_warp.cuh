// solo_b200 -- MD delayed-decision noise-shaping quantiser, one stream per lane group of a warp (sm_90a device code).
//
// Same arithmetic as the scalar model in sb_nsq.cuh (which cites the reference line by line); this file only changes
// WHERE things live and WHO computes them:
//   * a warp serves two streams, one per 16-lane group (SB_NSQ_GW); lane L < 12 of a group owns one (quantiser qz = L >> 2,
//     delayed-decision state s = L & 3) recurrence: its 16-stage warped all-pass chain, its 10 newest short-term-prediction
//     taps and its scalars sit in registers;
//   * the decision history (per quantiser 2 x 32 x 4 words + output samples + pulses; centre excitation) and the two long
//     32-bit buffers (160-entry rings) sit in shared memory, 8.2 KB per stream, so that 12 one-warp blocks fit an SM (the
//     kernel's time is ~ a + b / resident warps; 168 registers allow no more than 12).  What is touched once per sample
//     with slack stays in global memory: the output ring xq (read back only by the rewhitening of voiced frames) and the
//     random-generator history (loaded at the top of a sample, used at its end).  A survivor replacing another state is
//     ~40 warp shuffles (registers + a 64-bit path word) instead of the reference's 1.5 KB memcpy;
//   * the joint rate-distortion argmin, worst/best replacement and winner emission run on shuffles; the sample loop is
//     executed by both groups in lock step with full-warp collectives and warp-uniform trip counts, everything around it
//     (rewhitening, flushes, rescaling) names its own group so the two streams may diverge there.
// Lanes 12..15 of a group execute the same instruction stream on clamped indices and never store.
#pragma once
// (tests/hostsim compiles this file for the host under SB_EMU: 32 fibres play the lanes, the warp intrinsics are shims)
#if defined(__CUDACC__) || defined(SB_EMU)
#include "sb_nsq.cuh"
#ifdef __CUDACC__
#define SB_NSQ_DEV __device__ __forceinline__
#define SB_NSQ_KFN __device__
#else
#define SB_NSQ_DEV inline
#define SB_NSQ_KFN inline
#endif

namespace sb {

// Row paddings keep the three quantisers' rows in different shared-memory banks (the 12 lanes address
// [qz][same index][state]); the pad words are never read.
// The long buffers (sLTP_Q16, sLTP_shp_Q10 here, xq in NsqState) are 160-entry rings: logical index j of the reference's
// 2*frame_length arrays (old frame [0,160), frame being written [160,320)) lives at j mod 160.  Pitch lags run from 15 to
// 146 (lag 16..144 plus a contour offset of -1..+2), and nothing older than lag + 2 <= 148 samples behind the write position
// is ever read (the rewhitening starts at FRAME - lag - LPC_ORDER - LTP_ORDER / 2 >= 2), so the ring holds exactly the
// persistent state on entry and on exit.
struct NsqSmem {
    i32 sLTP_Q16[3][FRAME + 1];
    i32 sLTP_shp_Q10[3][FRAME + 2];
    i32 tabPred[3][DD_DELAY + 1][N_DD];
    i32 tabShape[3][DD_DELAY + 1][N_DD];
    i16 tabXq[3][DD_DELAY + 1][N_DD];      // output sample as it will be emitted (gain of its own sub-frame already applied)
    i16 tabExc[DD_DELAY][N_DD];            // centre excitation >> 10
    i8 tabQ[2][DD_DELAY + 1][N_DD];        // pulses of the two descriptions (the centre's are never emitted)
};
static_assert(((2 * sizeof(NsqSmem) + 255) / 256 * 256 + 1024) * 12 <= 233472, "two streams per one-warp block, twelve blocks per SM (228 KB, 1 KB reserved per block)");

// Lane group = the SB_NSQ_GW lanes that work on one stream (16: two streams per warp, 32: one).  Every collective below
// names its own group (mask gm, width SB_NSQ_GW), so the two halves of a warp may diverge freely.
#ifndef SB_NSQ_GW
#define SB_NSQ_GW 16
#endif
SB_NSQ_DEV int cix(int j) { return j >= FRAME ? j - FRAME : j; }   // ring index, 0 <= j <= 2*FRAME
SB_NSQ_DEV i32 shfl(unsigned gm, i32 v, int src) { return __shfl_sync(gm, v, src, SB_NSQ_GW); }
SB_NSQ_DEV u64 shfl64(unsigned gm, u64 v, int src) {
    u32 lo = __shfl_sync(gm, (u32)v, src, SB_NSQ_GW), hi = __shfl_sync(gm, (u32)(v >> 32), src, SB_NSQ_GW);
    return ((u64)hi << 32) | lo;
}

struct NsqLane {            // registers of one (quantiser, state) recurrence
    i32 sAR2[SHAPE_ORDER];
    i32 lpc[LPC_ORDER];     // lpc[0] = newest sLPC_Q14 value
    i32 LF_AR, Seed, Seed2, SeedInit2, RD;
    u64 path;
};
// acc + (x * c16) >> 16 with the coefficient already moved to the high half-word (one IMAD.HI, no shift in the loop)
SB_NSQ_DEV i32 mlahi(i32 acc, i32 x, i32 c_hi) { return addw(acc, __mulhi(x, c_hi)); }
struct NsqCand { i32 Q_Q0, Q_Q10, RD, Rd_ind, xq_Q14, LF_AR, shp, exc16, exc; };

// flush `n` delayed samples of the winner of quantiser qz to the outputs, samples spread over the group's lanes (n <= 32)
SB_NSQ_DEV void nsqw_flush(NsqSmem& S, int gl, int qz_, u64 wpath, int smpl_buf_idx, int n, int sig_off, int shp_idx,
                                           int ltp_idx, i8* q, i16* r16, i16* xq, int write_pred) {
    for (int lane = gl; lane < n; lane += SB_NSQ_GW) {
        const int last = (smpl_buf_idx + n - 1 - lane) & DD_MASK;
        const int sl = (int)((wpath >> (2 * last)) & 3);
        const int o = sig_off + lane - n;
        if (q) q[o] = S.tabQ[qz_ - 1][last][sl];
        if (r16) r16[o] = S.tabExc[last][sl];
        xq[o] = S.tabXq[qz_][last][sl];
        S.sLTP_shp_Q10[qz_][cix(shp_idx - n + lane)] = S.tabShape[qz_][last][sl];
        if (write_pred) S.sLTP_Q16[qz_][cix(ltp_idx - n + lane)] = S.tabPred[qz_][last][sl];
    }
}

// One 20 ms frame.  st: persistent quantiser states (global); c: frame control from the analysis stage (global, Seed is
// updated); x: prefiltered input; outputs: pulses of the two descriptions, (int16)(centre excitation >> 10).
SB_NSQ_KFN void nsq_del_dec_warp(NsqSmem& S, NsqState* ns3, EncCtrl* c, const i16* __restrict__ x, i8* q_md0, i8* q_md1, i16* r16, i32* rand_g) {
    const int gl = threadIdx.x & (SB_NSQ_GW - 1);                 // gl inside the group
    const int gsh = (threadIdx.x & 31) & ~(SB_NSQ_GW - 1);         // first warp gl of the group
    const unsigned gm = SB_NSQ_GW == 32 ? 0xffffffffu : (0xffffu << gsh);
    const bool act = gl < 12;
    const int qz = act ? (gl >> 2) : 2;
    const int s = gl & 3;
    i8* const Qout = qz == 0 ? (i8*)0 : (qz == 1 ? q_md0 : q_md1);
    i16* const xq_out = ns3[qz].xq;     // output ring of this lane's quantiser (global state)

    const int sigtype = c->sigtype;
    const i32 offset_Q10 = SB_T(quant_offsets_q10)[sigtype * 2 + c->QuantOffsetType];
    const i32 Lambda_Q10 = c->Lambda_Q10;
    const int LSF_flag = c->NLSFInterpCoef_Q2 == 4 ? 0 : 1;
    const i32 seed0 = c->Seed;
    int lag0 = ns3[0].lagPrev;         // centre lag (gates the harmonic shaping of all three quantisers)
    int lagq = ns3[qz].lagPrev;        // this gl's quantiser lag
    int decisionDelay = imin(DD_DELAY, SUBFR);
    if (sigtype == 0) {
        for (int k = 0; k < NB_SUBFR; k++) decisionDelay = imin(decisionDelay, c->pitchL[k] - LTP_ORDER / 2 - 1);
    } else if (lag0 > 0) {
        decisionDelay = imin(decisionDelay, lag0 - LTP_ORDER / 2 - 1);
    }

    // ---- load persistent state into shared memory / registers ----
    for (int qq = 0; qq < 3; qq++) {
        const NsqState* ns = &ns3[qq];
        for (int i = gl; i < FRAME; i += SB_NSQ_GW) { S.sLTP_shp_Q10[qq][i] = ns->sLTP_shp_Q10[i]; S.sLTP_Q16[qq][i] = 0; }
        if (gl < 2) S.sLTP_shp_Q10[qq][FRAME + gl] = 0;
        if (gl == 0) S.sLTP_Q16[qq][FRAME] = 0;
        for (int i = gl; i < DD_DELAY * N_DD; i += SB_NSQ_GW) {
            rand_g[qq * (DD_DELAY * N_DD) + i] = 0; (&S.tabXq[qq][0][0])[i] = 0; (&S.tabPred[qq][0][0])[i] = 0; (&S.tabShape[qq][0][0])[i] = 0;
            if (qq) (&S.tabQ[qq - 1][0][0])[i] = 0;
            if (qq == 0) (&S.tabExc[0][0])[i] = 0;
        }
    }
    __syncwarp(gm);
    if (gl < N_DD) for (int qq = 0; qq < 3; qq++) S.tabShape[qq][0][gl] = ns3[qq].sLTP_shp_Q10[FRAME - 1];
    NsqLane L;
    {
        const NsqState* ns = &ns3[qz];
#pragma unroll
        for (int j = 0; j < SHAPE_ORDER; j++) L.sAR2[j] = ns->sAR2_Q14[j];
#pragma unroll
        for (int j = 0; j < LPC_ORDER; j++) L.lpc[j] = ns->sLPC_Q14[DD_DELAY - 1 - j];
        L.LF_AR = ns->sLF_AR_shp_Q12;
        L.Seed = (s + seed0) & 3;
        L.Seed2 = L.Seed;
        L.SeedInit2 = L.Seed;
        L.RD = 0;
        L.path = 0x5555555555555555ull * (u64)s;
    }
    i32 prev_inv_gain = ns3[qz].prev_inv_gain_Q16;
    __syncwarp(gm);

    int smpl_buf_idx = 0, shp_idx = FRAME, ltp_idx = FRAME, subfr = 0;

    for (int k = 0; k < NB_SUBFR; k++) {
        const i16* A_Q12p = c->PredCoef_Q12[(k >> 1) | (1 - LSF_flag)];
        i32 A_Q12[LPC_ORDER], AR_shp[SHAPE_ORDER], B_Q14[LTP_ORDER];
#pragma unroll
        for (int j = 0; j < LPC_ORDER; j++) A_Q12[j] = A_Q12p[j];
        // coefficients of the per-sample filters, pre-shifted into the high half-word for mlahi()
        i32 A_hi[LPC_ORDER];
#pragma unroll
        for (int j = 0; j < LPC_ORDER; j++) A_hi[j] = shl(A_Q12[j], 16);
#pragma unroll
        for (int j = 0; j < SHAPE_ORDER; j++) AR_shp[j] = shl(c->AR2_Q13[k * SHAPE_ORDER + j], 16);
#pragma unroll
        for (int j = 0; j < LTP_ORDER; j++) B_Q14[j] = shl(c->LTPCoef_Q14[k * LTP_ORDER + j], 16);
        i32 HarmShapeFIRPacked_Q14 = c->HarmShapeGain_Q14[k] >> 2;
        HarmShapeFIRPacked_Q14 |= shl(c->HarmShapeGain_Q14[k] >> 1, 16);
        const int sig_off = k * SUBFR;
        const i32 Gain_Q16 = c->Gains_Q16[k];
        i32 inv_gain_Q16 = imin(inverse32_varq(imax(Gain_Q16, 1), 32), 32767);
        int rewhite = 0;

        if (sigtype == 0) {
            lag0 = lagq = c->pitchL[k];
            if ((k & (3 - shl(LSF_flag, 1))) == 0) {
                if (k == 2) {
                    subfr = 0;
                    // reset of the delayed decisions: centre winner by its own RD, others penalised, delayed samples flushed
                    i32 rd0 = shfl(gm, L.RD, 0), rd1 = shfl(gm, L.RD, 1), rd2 = shfl(gm, L.RD, 2), rd3 = shfl(gm, L.RD, 3);
                    int Winner = 0; i32 RDmin = rd0;
                    if (rd1 < RDmin) { RDmin = rd1; Winner = 1; }
                    if (rd2 < RDmin) { RDmin = rd2; Winner = 2; }
                    if (rd3 < RDmin) { RDmin = rd3; Winner = 3; }
                    if (s != Winner) L.RD = addw(L.RD, SB_I32_MAX >> 4);
                    for (int qq = 0; qq < 3; qq++) {
                        u64 wpath = shfl64(gm, L.path, qq * 4 + Winner);
                        nsqw_flush(S, gl, qq, wpath, smpl_buf_idx, decisionDelay, sig_off, shp_idx, ltp_idx,
                                   qq == 0 ? (i8*)0 : (qq == 1 ? q_md0 : q_md1), qq == 0 ? r16 : (i16*)0, ns3[qq].xq, 0);
                    }
                    __syncwarp(gm);
                }
                // rewhitening of the LTP state with the new short-term predictor, scaled on the fly (decision of the
                // reference: MA_Prediction over [start_idx, FRAME), of which only [FRAME - lag - 2, FRAME) is kept)
                i32 inv_gain_Q32 = shl(inv_gain_Q16, 16);
                if (k == 0) inv_gain_Q32 = shl(smulwb(inv_gain_Q32, c->LTP_scale_Q14), 2);
                const int lagk = c->pitchL[k];
                const int n0 = FRAME - lagk - LTP_ORDER / 2;
                for (int qq = 0; qq < 3; qq++) {
                    const i16* in = ns3[qq].xq;   // this warp's own emissions of the frame so far, ordered by the barriers around them
                    for (int n = n0 + gl; n < FRAME; n += SB_NSQ_GW) {
                        const int j = k * SUBFR + n;   // logical position in [old frame | this frame]
                        i32 pred = 0;
#pragma unroll
                        for (int d = 0; d < LPC_ORDER; d++) pred = addw(pred, (i32)in[cix(j - 1 - d)] * A_Q12[d]);
                        i32 o = sat16(rshift_round(subw(shl((i32)in[cix(j)], 12), pred), 12));
                        S.sLTP_Q16[qq][n] = smulwb(inv_gain_Q32, o);
                    }
                }
                ltp_idx = FRAME;
                rewhite = 1;
                __syncwarp(gm);
            }
        }
        // input scaling + state rescaling for the new gain
        {
            // prev_inv_gain is per quantiser; gather the three values so that every gl can scale every buffer
            const i32 pg0 = shfl(gm, prev_inv_gain, 0), pg1 = shfl(gm, prev_inv_gain, 4), pg2 = shfl(gm, prev_inv_gain, 8);
            const int lagk = c->pitchL[k];
            for (int qq = 0; qq < 3; qq++) {
                const i32 pg = qq == 0 ? pg0 : (qq == 1 ? pg1 : pg2);
                if (inv_gain_Q16 != pg) {
                    const i32 gain_adj_Q16 = div32_varq(inv_gain_Q16, pg, 16);
                    for (int i = gl; i < FRAME; i += SB_NSQ_GW) S.sLTP_shp_Q10[qq][i] = smulww(gain_adj_Q16, S.sLTP_shp_Q10[qq][i]);  // whole ring
                    if (!rewhite)
                        for (int i = ltp_idx - lagk - LTP_ORDER / 2 + gl; i < ltp_idx; i += SB_NSQ_GW) S.sLTP_Q16[qq][cix(i)] = smulww(gain_adj_Q16, S.sLTP_Q16[qq][cix(i)]);
                    for (int i = gl; i < DD_DELAY * N_DD; i += SB_NSQ_GW) {
                        (&S.tabPred[qq][0][0])[i] = smulww(gain_adj_Q16, (&S.tabPred[qq][0][0])[i]);
                        (&S.tabShape[qq][0][0])[i] = smulww(gain_adj_Q16, (&S.tabShape[qq][0][0])[i]);
                    }
                    if (qq == qz) {
                        L.LF_AR = smulww(gain_adj_Q16, L.LF_AR);
#pragma unroll
                        for (int j = 0; j < LPC_ORDER; j++) L.lpc[j] = smulww(gain_adj_Q16, L.lpc[j]);
#pragma unroll
                        for (int j = 0; j < SHAPE_ORDER; j++) L.sAR2[j] = smulww(gain_adj_Q16, L.sAR2[j]);
                    }
                }
            }
            prev_inv_gain = inv_gain_Q16;
        }
        __syncwarp(gm);

        // ---- sub-frame constants of the description split ----
        const i32 Tilt_Q14 = c->Tilt_Q14[k], LF_shp_Q14 = c->LF_shp_Q14[k];
        const i32 invg = inverse32_varq(imax(c->DeltaGains_Q16, 1), 32);
        const i32 inv_gain_p1 = invg, inv_gain_p2 = 65536 - invg;
        const i32 DeltaGains_p1 = inverse32_varq(imax(inv_gain_p1, 1), 32);
        const i32 DeltaGains_p2 = inverse32_varq(imax(inv_gain_p2, 1), 32);
        const i32 offset_p1 = smulww(inv_gain_p1, offset_Q10), offset_p2 = smulww(inv_gain_p2, offset_Q10);
        const int swap = (subfr % 2) >= 1;
        const int role1 = (qz == 1) != (swap != 0);  // this side gl plays "p1"
        const i32 ig = role1 ? inv_gain_p1 : inv_gain_p2;
        const i32 dg = role1 ? DeltaGains_p1 : DeltaGains_p2;
        const i32 of = role1 ? offset_p1 : offset_p2;
        const i32 rdc_inv = inverse32_varq(imax(dg, 1), 32);
        const i32 offset_c = offset_p1 + offset_p2;
        int shp_lag = shp_idx - lagq + 1, pred_lag = ltp_idx - lagq + LTP_ORDER / 2;
        const i32 JL = 90000;
        const unsigned fm = 0xffffffffu;   // the sample loop is executed by both streams of the warp in lock step
        __syncwarp();

        for (int i = 0; i < SUBFR; i++) {
            // random-generator state of the sample that leaves the decision window, along this lane's path: fetched from the
            // global history now, needed only at the winner selection some 400 instructions later
            const int last_pre = (smpl_buf_idx - 1 + decisionDelay) & DD_MASK;
            const i32 rs = rand_g[(qz * DD_DELAY + last_pre) * N_DD + (int)((L.path >> (2 * last_pre)) & 3)];
            // ---- long-term prediction / harmonic shaping of this gl's quantiser ----
            i32 LTP_pred_Q14 = 0, n_LTP_Q14 = 0;
            if (sigtype == 0) {
                const i32* pl = S.sLTP_Q16[qz];
#pragma unroll
                for (int j = 0; j < LTP_ORDER; j++) LTP_pred_Q14 = mlahi(LTP_pred_Q14, pl[cix(pred_lag - j)], B_Q14[j]);
                pred_lag++;
            }
            if (lag0 > 0) {
                const i32* sl = S.sLTP_shp_Q10[qz];
                n_LTP_Q14 = smulwb(addw(sl[cix(shp_lag)], sl[cix(shp_lag - 2)]), HarmShapeFIRPacked_Q14);
                n_LTP_Q14 = smlawt(n_LTP_Q14, sl[cix(shp_lag - 1)], HarmShapeFIRPacked_Q14);
                n_LTP_Q14 = shl(n_LTP_Q14, 6);
                shp_lag++;
            }
            // ---- short-term prediction, warped noise-shape feedback, low-frequency shaping ----
            i32 LPC_pred_Q10 = 0;
#pragma unroll
            for (int j = 0; j < LPC_ORDER; j++) LPC_pred_Q10 = mlahi(LPC_pred_Q10, L.lpc[j], A_hi[j]);
            i32 tmp2 = smlawb(L.lpc[0], L.sAR2[0], WARPING_Q16);
            i32 tmp1 = smlawb(L.sAR2[0], subw(L.sAR2[1], tmp2), WARPING_Q16);
            L.sAR2[0] = tmp2;
            i32 n_AR_Q10 = __mulhi(tmp2, AR_shp[0]);
#pragma unroll
            for (int j = 2; j < SHAPE_ORDER; j += 2) {
                tmp2 = smlawb(L.sAR2[j - 1], subw(L.sAR2[j], tmp1), WARPING_Q16);
                L.sAR2[j - 1] = tmp1;
                n_AR_Q10 = mlahi(n_AR_Q10, tmp1, AR_shp[j - 1]);
                tmp1 = smlawb(L.sAR2[j], subw(L.sAR2[j + 1], tmp2), WARPING_Q16);
                L.sAR2[j] = tmp2;
                n_AR_Q10 = mlahi(n_AR_Q10, tmp2, AR_shp[j]);
            }
            L.sAR2[SHAPE_ORDER - 1] = tmp1;
            n_AR_Q10 = mlahi(n_AR_Q10, tmp1, AR_shp[SHAPE_ORDER - 1]);
            n_AR_Q10 = n_AR_Q10 >> 1;
            n_AR_Q10 = smlawb(n_AR_Q10, L.LF_AR, Tilt_Q14);
            const i32 shape_new = S.tabShape[qz][smpl_buf_idx][(int)((L.path >> (2 * smpl_buf_idx)) & 3)];
            i32 n_LF_Q10 = shl(smulwb(shape_new, LF_shp_Q14), 2);
            n_LF_Q10 = smlawt(n_LF_Q10, L.LF_AR, LF_shp_Q14);
            i32 t = subw(LTP_pred_Q14, n_LTP_Q14);
            t = t >> 4;
            t = addw(t, LPC_pred_Q10);
            t = subw(t, n_AR_Q10);
            t = subw(t, n_LF_Q10);
            i32 r_Q10 = subw(smulbb(x[sig_off + i], inv_gain_Q16) >> 6, t);   // x_sc_Q10, same address for the whole group
            L.Seed2 = lcg_rand(L.Seed2);
            L.Seed = lcg_rand(L.Seed);
            const i32 dither = L.Seed2 >> 31;
            r_Q10 = subw(r_Q10 ^ dither, dither);

            // ---- side quantisers: two candidate levels each (Agora_Silk_RDCx1), branch-free ----
            const i32 r_c = shfl(fm, r_Q10, s);   // the centre residual of this state column
            NsqCand c0, c1;
            c0.Q_Q0 = c0.Q_Q10 = c0.RD = c0.Rd_ind = 0; c1 = c0;
            {
                i32 rq = subw(smulww(ig, r_c), of);
                const i32 r_p = subw(smulww(rdc_inv, r_Q10), of);
                rq = limit(rq, -(64 << 10), 64 << 10);
                const bool lo = rq < -1536, hi = rq > 512;
                const i32 qr = shl(rshift_round(rq, 10), 10);
                const i32 q1 = (lo || hi) ? qr : -1024;
                const i32 q2 = lo ? addw(q1, 1024) : (hi ? subw(q1, 1024) : 0);
                i32 t1 = addw(q1, of), t2 = addw(q2, of);      // rate term: |level + offset| with the sign the level implies
                if (!hi) t1 = negw(t1);
                if (lo) t2 = negw(t2);
                const i32 rr1 = subw(r_p, q1), rr2 = subw(r_p, q2);
                const i32 rd1 = smlabb(mulw(t1, Lambda_Q10), rr1, rr1) >> 10;
                const i32 rd2 = smlabb(mulw(t2, Lambda_Q10), rr2, rr2) >> 10;
                {   // centre lanes compute it too and overwrite it below (no branch)
                    const bool f = rd1 < rd2;
                    const i32 qa = f ? q1 : q2, qb = f ? q2 : q1, ra = f ? rd1 : rd2, rb = f ? rd2 : rd1;
                    c0.RD = addw(L.RD, ra); c1.RD = addw(L.RD, rb);
                    c0.Q_Q0 = qa >> 10; c1.Q_Q0 = qb >> 10;
                    c0.Q_Q10 = addw(of, qa); c1.Q_Q10 = addw(of, qb);
                    c0.Rd_ind = qz != 0 ? ra : 0; c1.Rd_ind = qz != 0 ? rb : 0;
                    c0.Q_Q10 = qz != 0 ? c0.Q_Q10 : 0; c1.Q_Q10 = qz != 0 ? c1.Q_Q10 : 0;
                }
            }
            // ---- the four composites of the side candidates (Agora_Silk_CenterRD), evaluated by all three lanes of the
            //      column so that the sides know the two surviving composites without a round trip ----
            {
                const i32 a0 = shfl(fm, c0.Q_Q10, 4 + s), a1 = shfl(fm, c1.Q_Q10, 4 + s), b0 = shfl(fm, c0.Q_Q10, 8 + s), b1 = shfl(fm, c1.Q_Q10, 8 + s);
                const i32 ra0 = shfl(fm, c0.Rd_ind, 4 + s), ra1 = shfl(fm, c1.Rd_ind, 4 + s), rb0 = shfl(fm, c0.Rd_ind, 8 + s), rb1 = shfl(fm, c1.Rd_ind, 8 + s);
                i32 qx[4], rdx[4];
                qx[0] = addw(a0, b0); qx[1] = addw(a1, b1); qx[2] = addw(a0, b1); qx[3] = addw(a1, b0);
                const i32 r_temp = subw(r_c, offset_c);
#pragma unroll
                for (int m = 0; m < 4; m++) {
                    i32 rr = subw(r_temp, qx[m]);
                    i32 tt = addw(qx[m], offset_c);
                    if (qx[m] < 0) tt = negw(tt);
                    rdx[m] = smlabb(mulw(tt, Lambda_Q10), rr, rr) >> 10;
                }
                const i32 ja0 = smulww(JL, ra0), ja1 = smulww(JL, ra1), jb0 = smulww(JL, rb0), jb1 = smulww(JL, rb1);
                rdx[0] = addw(addw(rdx[0], ja0), jb0);
                rdx[1] = addw(addw(rdx[1], ja1), jb1);
                rdx[2] = addw(addw(rdx[2], ja0), jb1);
                rdx[3] = addw(addw(rdx[3], ja1), jb0);
                // best and second-best composite (strict "<": the lowest index wins ties, as in the reference's scans);
                // written with selects only -- these lines sit on every lane's critical path
                i32 mn = rdx[0], q_w1 = qx[0]; int w1 = 0;
                { const bool t = rdx[1] < mn; mn = t ? rdx[1] : mn; w1 = t ? 1 : w1; q_w1 = t ? qx[1] : q_w1; }
                { const bool t = rdx[2] < mn; mn = t ? rdx[2] : mn; w1 = t ? 2 : w1; q_w1 = t ? qx[2] : q_w1; }
                { const bool t = rdx[3] < mn; mn = t ? rdx[3] : mn; w1 = t ? 3 : w1; q_w1 = t ? qx[3] : q_w1; }
                const bool e0 = w1 == 0;
                i32 mn2 = e0 ? rdx[1] : rdx[0], q_w2 = e0 ? qx[1] : qx[0]; int w2 = e0 ? 1 : 0;
                { const bool t = (w1 != 1) & (rdx[1] < mn2); mn2 = t ? rdx[1] : mn2; w2 = t ? 1 : w2; q_w2 = t ? qx[1] : q_w2; }
                { const bool t = (w1 != 2) & (rdx[2] < mn2); mn2 = t ? rdx[2] : mn2; w2 = t ? 2 : w2; q_w2 = t ? qx[2] : q_w2; }
                { const bool t = (w1 != 3) & (rdx[3] < mn2); mn2 = t ? rdx[3] : mn2; w2 = t ? 3 : w2; q_w2 = t ? qx[3] : q_w2; }
                {
                    // centre: the two surviving composites; sides: their own candidates re-ordered to match them
                    const bool ctr = qz == 0;
                    const int sel = qz == 1 ? 0xA : 0x6;  // a(c) / b(c): candidate index inside composite c
                    const bool i1 = (sel >> w1) & 1, i2 = (sel >> w2) & 1;
                    const NsqCand o0 = c0, o1 = c1;
                    c0.Q_Q0 = ctr ? (q_w1 >> 10) : (i1 ? o1.Q_Q0 : o0.Q_Q0);
                    c1.Q_Q0 = ctr ? (q_w2 >> 10) : (i2 ? o1.Q_Q0 : o0.Q_Q0);
                    c0.Q_Q10 = ctr ? q_w1 : (i1 ? o1.Q_Q10 : o0.Q_Q10);
                    c1.Q_Q10 = ctr ? q_w2 : (i2 ? o1.Q_Q10 : o0.Q_Q10);
                    c0.RD = ctr ? addw(L.RD, mn) : (i1 ? o1.RD : o0.RD);
                    c1.RD = ctr ? addw(L.RD, mn2) : (i2 ? o1.RD : o0.RD);
                }
            }
            // ---- un-dither, description gain, simulate the decoder for both candidates ----
            {
                c0.Q_Q10 = subw(c0.Q_Q10 ^ dither, dither);
                c1.Q_Q10 = subw(c1.Q_Q10 ^ dither, dither);
                c0.exc = c0.Q_Q10; c1.exc = c1.Q_Q10;
                { const i32 g0 = smulww(dg, c0.Q_Q10), g1 = smulww(dg, c1.Q_Q10); c0.Q_Q10 = qz != 0 ? g0 : c0.Q_Q10; c1.Q_Q10 = qz != 0 ? g1 : c1.Q_Q10; }
                const i32 ltp4 = rshift_round(LTP_pred_Q14, 4);
                i32 LPC_exc_Q10 = addw(c0.Q_Q10, ltp4);
                i32 xq_Q10 = addw(LPC_exc_Q10, LPC_pred_Q10);
                i32 sLF = subw(xq_Q10, n_AR_Q10);
                c0.shp = subw(sLF, n_LF_Q10); c0.LF_AR = shl(sLF, 2); c0.xq_Q14 = shl(xq_Q10, 4); c0.exc16 = shl(LPC_exc_Q10, 6);
                LPC_exc_Q10 = addw(c1.Q_Q10, ltp4);
                xq_Q10 = addw(LPC_exc_Q10, LPC_pred_Q10);
                sLF = subw(xq_Q10, n_AR_Q10);
                c1.shp = subw(sLF, n_LF_Q10); c1.LF_AR = shl(sLF, 2); c1.xq_Q14 = shl(xq_Q10, 4); c1.exc16 = shl(LPC_exc_Q10, 6);
            }
            smpl_buf_idx = (smpl_buf_idx - 1) & DD_MASK;
            const int last_smple_idx = (smpl_buf_idx + decisionDelay) & DD_MASK;

            // ---- Agora_Silk_JudgeWinner + Agora_Silk_GetWinner.  The joint RD of every column (first and second
            //      candidates) and the centre RDs are gathered once; penalties and replacements are then tracked in
            //      registers by every lane, so the loop and the final winner need no further exchange. ----
            int Winner;
            {
                const i32 jr0 = qz == 0 ? c0.RD : smulww(c0.RD, JL);
                const i32 jr1 = qz == 0 ? c1.RD : smulww(c1.RD, JL);
                const i32 jn0 = addw(addw(jr0, __shfl_down_sync(fm, jr0, 4, SB_NSQ_GW)), __shfl_down_sync(fm, jr0, 8, SB_NSQ_GW));
                const i32 jn1 = addw(addw(jr1, __shfl_down_sync(fm, jr1, 4, SB_NSQ_GW)), __shfl_down_sync(fm, jr1, 8, SB_NSQ_GW));
                i32 j0[4], j1[4], ra[4], rb[4];   // joint RD via first / second candidate; centre RD of first / second candidate
#pragma unroll
                for (int m = 0; m < 4; m++) { j0[m] = shfl(fm, jn0, m); j1[m] = shfl(fm, jn1, m); ra[m] = shfl(fm, c0.RD, m); rb[m] = shfl(fm, c1.RD, m); }
                int W0 = 0; i32 RDmin = j0[0];
#pragma unroll
                for (int m = 1; m < 4; m++) { const bool t = j0[m] < RDmin; RDmin = t ? j0[m] : RDmin; W0 = t ? m : W0; }
                const i32 wrs = shfl(fm, rs, qz * 4 + W0);
                // De-synchronised random generators (a state whose delayed sample saw another dither sequence than the
                // winner's) are rare -- under 2 % of the samples on speech: the penalties and the extra replacement trips sit
                // behind a warp-uniform test of the ballot.
                const unsigned bal_all = __ballot_sync(fm, act && rs != wrs);
                int my_trips = 1, trips = 1;
                if (bal_all != 0) {
                    const unsigned bal = (bal_all >> gsh) & 0xffffu;
                    const unsigned mstate = (bal | (bal >> 4) | (bal >> 8)) & 0xF;
                    const int RandSyncCtl = __popc(mstate);
                    const i32 PEN = SB_I32_MAX >> 4;
#pragma unroll
                    for (int m = 0; m < 4; m++) {
                        const i32 pen = ((mstate >> m) & 1) ? PEN : 0;
                        j0[m] = addw(j0[m], pen); j1[m] = addw(j1[m], pen); ra[m] = addw(ra[m], pen); rb[m] = addw(rb[m], pen);
                    }
                    { const i32 pen = ((qz == 0) & ((mstate >> s) & 1)) ? PEN : 0; c0.RD = addw(c0.RD, pen); c1.RD = addw(c1.RD, pen); }
                    // The reference repeats the replacement once per de-synchronised state (at least once).  Both streams of
                    // the warp run the same number of trips (the larger of the two) so that the shuffles below stay
                    // warp-uniform; a stream that is done (or finds nothing to replace) shuffles every lane onto itself.
                    my_trips = RandSyncCtl > 1 ? RandSyncCtl : 1;
                    trips = __reduce_max_sync(fm, my_trips);
                }
                for (int it = 0; it < trips; it++) {
                    i32 RDmax = ra[0], RDmin2 = rb[0], j1n = j1[0]; int imx = 0, imn = 0;
#pragma unroll
                    for (int m = 1; m < 4; m++) {
                        const bool tx = ra[m] > RDmax; RDmax = tx ? ra[m] : RDmax; imx = tx ? m : imx;
                        const bool tn = rb[m] < RDmin2; RDmin2 = tn ? rb[m] : RDmin2; imn = tn ? m : imn; j1n = tn ? j1[m] : j1n;
                    }
                    const bool doit = it < my_trips && RDmin2 < RDmax;
                    if (__any_sync(fm, doit)) {   // warp-uniform: skip the 40 shuffles when neither stream replaces a state
                        const int src = qz * 4 + imn;
                        const bool tgt = doit && (s == imx);
                        const int from = tgt ? src : gl;   // everybody else reads itself: no select after the shuffle
#pragma unroll
                        for (int j = 0; j < SHAPE_ORDER; j++) L.sAR2[j] = shfl(fm, L.sAR2[j], from);
#pragma unroll
                        for (int j = 0; j < LPC_ORDER; j++) L.lpc[j] = shfl(fm, L.lpc[j], from);
                        L.LF_AR = shfl(fm, L.LF_AR, from);
                        L.Seed = shfl(fm, L.Seed, from);
                        L.Seed2 = shfl(fm, L.Seed2, from);
                        L.SeedInit2 = shfl(fm, L.SeedInit2, from);
                        L.RD = shfl(fm, L.RD, from);
                        L.path = shfl64(fm, L.path, from);
                        // first candidate of the replaced state <- second candidate of the survivor
                        i32 v;
                        v = shfl(fm, c1.Q_Q0, src); if (tgt) c0.Q_Q0 = v;
                        v = shfl(fm, c1.RD, src); if (tgt) c0.RD = v;
                        v = shfl(fm, c1.xq_Q14, src); if (tgt) c0.xq_Q14 = v;
                        v = shfl(fm, c1.LF_AR, src); if (tgt) c0.LF_AR = v;
                        v = shfl(fm, c1.shp, src); if (tgt) c0.shp = v;
                        v = shfl(fm, c1.exc16, src); if (tgt) c0.exc16 = v;
                        v = shfl(fm, c1.exc, src); if (tgt) c0.exc = v;
                        // what every lane knows about the columns afterwards
#pragma unroll
                        for (int m = 0; m < 4; m++) { const bool t = doit & (m == imx); ra[m] = t ? RDmin2 : ra[m]; j0[m] = t ? j1n : j0[m]; }
                    }
                }
                Winner = 0; RDmin = j0[0];
#pragma unroll
                for (int m = 1; m < 4; m++) { const bool t = j0[m] < RDmin; RDmin = t ? j0[m] : RDmin; Winner = t ? m : Winner; }
            }
            // ---- emit the sample that is decisionDelay old from the joint winner ----
            {
                if ((subfr > 0 || i >= decisionDelay) && act && s == Winner) {
                    const int sl = (int)((L.path >> (2 * last_smple_idx)) & 3);
                    const int o = sig_off + i - decisionDelay;
                    if (Qout) Qout[o] = S.tabQ[qz - 1][last_smple_idx][sl];
                    if (qz == 0) r16[o] = S.tabExc[last_smple_idx][sl];
                    xq_out[o] = S.tabXq[qz][last_smple_idx][sl];
                    S.sLTP_shp_Q10[qz][cix(shp_idx - decisionDelay)] = S.tabShape[qz][last_smple_idx][sl];
                    S.sLTP_Q16[qz][cix(ltp_idx - decisionDelay)] = S.tabPred[qz][last_smple_idx][sl];
                }
                shp_idx++;
                ltp_idx++;
            }
            __syncwarp();  // history reads of this sample (position last_smple_idx may alias smpl_buf_idx) before the writes below
            // ---- Agora_Silk_Update_DelDecState ----
            {
                L.LF_AR = c0.LF_AR;
#pragma unroll
                for (int j = LPC_ORDER - 1; j > 0; j--) L.lpc[j] = L.lpc[j - 1];
                L.lpc[0] = c0.xq_Q14;
                L.Seed = addw(L.Seed, c0.Q_Q0);
                L.RD = c0.RD;
                if (act) {
                    S.tabXq[qz][smpl_buf_idx][s] = (i16)sat16(rshift_round(smulww(c0.xq_Q14 >> 4, Gain_Q16), 10));
                    if (qz) S.tabQ[qz - 1][smpl_buf_idx][s] = (i8)c0.Q_Q0;
                    S.tabPred[qz][smpl_buf_idx][s] = c0.exc16;
                    S.tabShape[qz][smpl_buf_idx][s] = c0.shp;
                    rand_g[(qz * DD_DELAY + smpl_buf_idx) * N_DD + s] = L.Seed;
                    if (qz == 0) S.tabExc[smpl_buf_idx][s] = (i16)(c0.exc >> 10);
                }
                L.path = (L.path & ~((u64)3 << (2 * smpl_buf_idx))) | ((u64)s << (2 * smpl_buf_idx));
            }
            __syncwarp();
        }
        subfr++;
    }

    // ---- frame end: winner by the centre's own RD, flush, write the persistent state back ----
    {
        i32 rd0 = shfl(gm, L.RD, 0), rd1 = shfl(gm, L.RD, 1), rd2 = shfl(gm, L.RD, 2), rd3 = shfl(gm, L.RD, 3);
        int Winner = 0; i32 RDmin = rd0;
        if (rd1 < RDmin) { RDmin = rd1; Winner = 1; }
        if (rd2 < RDmin) { RDmin = rd2; Winner = 2; }
        if (rd3 < RDmin) { RDmin = rd3; Winner = 3; }
        const i32 seed_out = shfl(gm, L.SeedInit2, Winner);
        if (gl == 0) c->Seed = seed_out;
        for (int qq = 0; qq < 3; qq++) {
            u64 wpath = shfl64(gm, L.path, qq * 4 + Winner);
            nsqw_flush(S, gl, qq, wpath, smpl_buf_idx, decisionDelay, FRAME, shp_idx, ltp_idx,
                       qq == 0 ? (i8*)0 : (qq == 1 ? q_md0 : q_md1), qq == 0 ? r16 : (i16*)0, ns3[qq].xq, 1);
        }
        __syncwarp(gm);
        if (act && s == Winner) {
            NsqState* ns = &ns3[qz];
#pragma unroll
            for (int j = 0; j < LPC_ORDER; j++) ns->sLPC_Q14[DD_DELAY - 1 - j] = L.lpc[j];
#pragma unroll
            for (int j = 0; j < SHAPE_ORDER; j++) ns->sAR2_Q14[j] = L.sAR2[j];
            ns->sLF_AR_shp_Q12 = L.LF_AR;
            ns->lagPrev = c->pitchL[NB_SUBFR - 1];
            ns->prev_inv_gain_Q16 = prev_inv_gain;
        }
        for (int qq = 0; qq < 3; qq++) {
            NsqState* ns = &ns3[qq];
            for (int i = gl; i < FRAME; i += SB_NSQ_GW) ns->sLTP_shp_Q10[i] = S.sLTP_shp_Q10[qq][i];
        }
        __syncwarp(gm);
    }
}

// The nf frames of a packet for the stream of this lane group: frame controls and prefiltered input from the scratch slot,
// pulses and centre excitation back into it.
SB_NSQ_DEV void nsq_packet_warp(NsqSmem& S, NsqState* ns3, EncScratch* scr, int nf) {
    for (int f = 0; f < nf; f++)
        nsq_del_dec_warp(S, ns3, &scr->c[f], scr->xfw[f], scr->q_md[f][0], scr->q_md[f][1], scr->r16[f], &scr->nsq_rand[0][0][0]);
}

}  // namespace sb
#endif  // __CUDACC__ || SB_EMU
