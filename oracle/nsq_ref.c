/* Direct entry to the reference's multiple-description quantiser, SKP_Silk_NSQ_del_dec, one frame per call, in the
 * plain-data layout of nsq_io.h.  Compiled against the headers of the unmodified FIX tree and linked with its sources by
 * oracle/Makefile into _ref/libjc1_fix_nsq.so (and its coverage twin _ref/cov/).  Test infrastructure only.
 *
 * The encoder handle is a real one: AGR_Sate_Encoder_Init, then the settings step that SKP_Silk_SDK_Encode runs before
 * every packet (enc_API.c:161-192), so frame and sub-frame length, the number of decision states, the two filter orders,
 * the warping and the reset values of the three quantiser states (only the centre one starts with lagPrev = 100) are the
 * reference's own.  Per frame the control block is filled as SKP_Silk_encode_frame_FIX.c:63-67 leaves it (Seed_md[] =
 * Seed) and the quantiser is called with the arguments of :135-139. */
#include <string.h>
#include "SKP_Silk_main_FIX.h"
#include "AGR_BWE_main_FIX.h"
#include "AGR_JC1_SDK_API.h"
#include "nsq_io.h"

void nsq_io_sizes(int* s) { NSQ_IO_SIZES(s); }

static SKP_Silk_encoder_state_FIX* open_encoder(void** handle) {
    USER_Ctrl_enc u;
    SATEEncCtl* h;
    SKP_Silk_encoder_state_FIX* e;
    SKP_SILK_SDK_EncControlStruct* ec;
    memset(&u, 0, sizeof(u));
    u.mode = 2; u.targetRate_bps = 13600; u.samplerate = 16000; u.framesize_ms = 40;
    h = (SATEEncCtl*)AGR_Sate_Encoder_Init(&u);
    *handle = h;
    if (!h) return NULL;
    e = (SKP_Silk_encoder_state_FIX*)h->stEnc;
    ec = &h->encControl;
    e->sCmn.API_fs_Hz = ec->API_sampleRate;
    e->sCmn.maxInternal_fs_kHz = (ec->maxInternalSampleRate >> 10) + 1;
    e->sCmn.useInBandFEC = ec->useInBandFEC;
    e->sCmn.writeMDIndex = ec->useMDIndex;
    e->sCmn.md_enable = 1;
    if (SKP_Silk_control_encoder_FIX(e, 1000 * ec->packetSize / ec->API_sampleRate,
                                     SKP_LIMIT(ec->bitRate, MIN_TARGET_RATE_BPS, MAX_TARGET_RATE_BPS),
                                     ec->packetLossPercentage, ec->useDTX, ec->complexity) != 0)
        return NULL;
    if (e->sCmn.frame_length != NSQIO_FRAME || e->sCmn.subfr_length != NSQIO_FRAME / NB_SUBFR || e->sCmn.predictLPCOrder != 10 ||
        e->sCmn.shapingLPCOrder != 16 || e->sCmn.nStatesDelayedDecision != 4 || NSQ_LPC_BUF_LENGTH != 32)
        return NULL;
    return e;
}

static SKP_Silk_nsq_state* nsq_of(SKP_Silk_encoder_state_FIX* e, int qz) {
    return qz == 0 ? &e->sCmn.sNSQ : &e->sCmn.sNSQ_md[qz - 1];
}

static void state_get(NsqStateIO* o, const SKP_Silk_nsq_state* s) {
    memcpy(o->xq, s->xq, sizeof(o->xq));
    memcpy(o->sLTP_shp_Q10, s->sLTP_shp_Q10, sizeof(o->sLTP_shp_Q10));
    memcpy(o->sLPC_Q14, s->sLPC_Q14, sizeof(o->sLPC_Q14));
    memcpy(o->sAR2_Q14, s->sAR2_Q14, sizeof(o->sAR2_Q14));
    o->sLF_AR_shp_Q12 = s->sLF_AR_shp_Q12;
    o->lagPrev = s->lagPrev;
    o->prev_inv_gain_Q16 = s->prev_inv_gain_Q16;
}

static void state_set(SKP_Silk_nsq_state* s, const NsqStateIO* o) {
    memcpy(s->xq, o->xq, sizeof(o->xq));
    memcpy(s->sLTP_shp_Q10, o->sLTP_shp_Q10, sizeof(o->sLTP_shp_Q10));
    memcpy(s->sLPC_Q14, o->sLPC_Q14, sizeof(o->sLPC_Q14));
    memcpy(s->sAR2_Q14, o->sAR2_Q14, sizeof(o->sAR2_Q14));
    s->sLF_AR_shp_Q12 = o->sLF_AR_shp_Q12;
    s->lagPrev = o->lagPrev;
    s->prev_inv_gain_Q16 = o->prev_inv_gain_Q16;
}

/* the three quantiser states of a freshly initialised encoder (centre, description 1, description 2) */
int nsqref_reset_state(NsqStateIO st[3]) {
    void* h;
    SKP_Silk_encoder_state_FIX* e = open_encoder(&h);
    int qz;
    if (!e) { if (h) AGR_Sate_Encoder_Uninit(h); return -1; }
    for (qz = 0; qz < 3; qz++) state_get(&st[qz], nsq_of(e, qz));
    AGR_Sate_Encoder_Uninit(h);
    return 0;
}

/* nfr consecutive frames from the states st0[3]; out[f] and st_after[f][3] after every frame */
int nsqref_run(int nfr, const NsqStateIO st0[3], const NsqFrameIn* fr, NsqFrameOut* out, NsqStateIO* st_after) {
    void* h;
    SKP_Silk_encoder_state_FIX* e = open_encoder(&h);
    int f, k, j, qz;
    if (!e) { if (h) AGR_Sate_Encoder_Uninit(h); return -1; }
    for (qz = 0; qz < 3; qz++) state_set(nsq_of(e, qz), &st0[qz]);
    for (f = 0; f < nfr; f++) {
        const NsqFrameIn* x = &fr[f];
        SKP_Silk_encoder_control c;
        SKP_int16 pred[2 * MAX_LPC_ORDER], ltp[LTP_ORDER * NB_SUBFR], ar2[NB_SUBFR * MAX_SHAPE_LPC_ORDER];
        SKP_int harm[NB_SUBFR], tilt[NB_SUBFR];
        SKP_int32 lf[NB_SUBFR], gains[NB_SUBFR], mdgains[NB_SUBFR];
        SKP_int8 q[MAX_FRAME_LENGTH], qmd[MAX_INTERLEAVE_NUM][MAX_FRAME_LENGTH], *q_md[MAX_INTERLEAVE_NUM];
        SKP_int32 r[MAX_FRAME_LENGTH];
        memset(&c, 0, sizeof(c));
        c.sigtype = x->sigtype;
        c.QuantOffsetType = x->QuantOffsetType;
        c.NLSFInterpCoef_Q2 = x->NLSFInterpCoef_Q2;
        c.Seed = x->Seed;
        for (j = 0; j < MAX_INTERLEAVE_NUM; j++) { c.Seed_md[j] = c.Seed; q_md[j] = qmd[j]; }
        memset(pred, 0, sizeof(pred));
        memset(ar2, 0, sizeof(ar2));
        for (j = 0; j < 10; j++) { pred[j] = x->PredCoef_Q12[0][j]; pred[MAX_LPC_ORDER + j] = x->PredCoef_Q12[1][j]; }
        for (j = 0; j < LTP_ORDER * NB_SUBFR; j++) ltp[j] = x->LTPCoef_Q14[j];
        for (k = 0; k < NB_SUBFR; k++) {
            c.pitchL[k] = x->pitchL[k];
            for (j = 0; j < 16; j++) ar2[k * MAX_SHAPE_LPC_ORDER + j] = x->AR2_Q13[k * 16 + j];
            harm[k] = x->HarmShapeGain_Q14[k]; tilt[k] = x->Tilt_Q14[k]; lf[k] = x->LF_shp_Q14[k];
            gains[k] = x->Gains_Q16[k]; mdgains[k] = 0;   /* MDGains_Q16: not read by the quantiser */
        }
        memset(q, 0, sizeof(q)); memset(qmd, 0, sizeof(qmd)); memset(r, 0, sizeof(r));
        SKP_Silk_NSQ_del_dec(&e->sCmn, &c, &e->sCmn.sNSQ, e->sCmn.sNSQ_md, x->x, q, q_md, r, c.NLSFInterpCoef_Q2, pred, ltp, ar2,
                             harm, tilt, lf, gains, mdgains, x->DeltaGains_Q16, x->Lambda_Q10, x->LTP_scale_Q14);
        for (j = 0; j < NSQIO_FRAME; j++) {
            out[f].q_md[0][j] = qmd[0][j];
            out[f].q_md[1][j] = qmd[1][j];
            out[f].r16[j] = (int16_t)(r[j] >> 10);
        }
        out[f].Seed = c.Seed;
        for (qz = 0; qz < 3; qz++) state_get(&st_after[f * 3 + qz], nsq_of(e, qz));
    }
    AGR_Sate_Encoder_Uninit(h);
    return 0;
}
