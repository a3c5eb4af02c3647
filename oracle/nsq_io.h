/* One frame of the multiple-description quantiser as plain data: what the quantiser stage receives, what it returns and
 * the persistent state of one of its three quantisers.  The same layout is read and written by the reference shim
 * (oracle/nsq_ref.c), the host model (tests/hostsim) and the GPU harness (tests/gpu_ops), and mirrored by the numpy dtypes
 * in oracle/nsq_ref.py; every library exports nsq_io_sizes() so that a layout drift fails loudly.  No padding: the int32
 * fields come first and every array of narrower type has an even byte count. */
#ifndef SB_NSQ_IO_H
#define SB_NSQ_IO_H
#include <stdint.h>

#define NSQIO_FRAME 160

typedef struct {
    int32_t sigtype, QuantOffsetType, Seed, NLSFInterpCoef_Q2;
    int32_t pitchL[4], Gains_Q16[4];
    int32_t DeltaGains_Q16, Lambda_Q10, LTP_scale_Q14;
    int32_t LF_shp_Q14[4], Tilt_Q14[4], HarmShapeGain_Q14[4];
    int16_t PredCoef_Q12[2][10];
    int16_t LTPCoef_Q14[4 * 5];
    int16_t AR2_Q13[4 * 16];
    int16_t x[NSQIO_FRAME];          /* prefiltered input (xfw) */
} NsqFrameIn;

typedef struct {
    int8_t q_md[2][NSQIO_FRAME];     /* pulses of the two descriptions */
    int16_t r16[NSQIO_FRAME];        /* centre excitation as the encoder keeps it: (int16)(r_Q10 >> 10) */
    int32_t Seed;                    /* the seed the quantiser writes back into the frame control */
} NsqFrameOut;

/* what survives a frame: the last frame of output samples and of shaping state, the newest 32 short-term states */
typedef struct {
    int16_t xq[NSQIO_FRAME];
    int32_t sLTP_shp_Q10[NSQIO_FRAME];
    int32_t sLPC_Q14[32];
    int32_t sAR2_Q14[16];
    int32_t sLF_AR_shp_Q12, lagPrev, prev_inv_gain_Q16;
} NsqStateIO;

#define NSQ_IO_SIZES(s) do { (s)[0] = (int)sizeof(NsqFrameIn); (s)[1] = (int)sizeof(NsqFrameOut); (s)[2] = (int)sizeof(NsqStateIO); } while (0)

#ifdef __cplusplus
/* the kernel source's structures (sb_state.cuh must come first) */
namespace sb {
SB_HD void nsqio_ctrl(EncCtrl* c, const NsqFrameIn* f) {
    c->sigtype = f->sigtype; c->QuantOffsetType = f->QuantOffsetType; c->Seed = f->Seed; c->NLSFInterpCoef_Q2 = f->NLSFInterpCoef_Q2;
    for (int k = 0; k < NB_SUBFR; k++) {
        c->pitchL[k] = f->pitchL[k]; c->Gains_Q16[k] = f->Gains_Q16[k];
        c->LF_shp_Q14[k] = f->LF_shp_Q14[k]; c->Tilt_Q14[k] = f->Tilt_Q14[k]; c->HarmShapeGain_Q14[k] = f->HarmShapeGain_Q14[k];
    }
    c->DeltaGains_Q16 = f->DeltaGains_Q16; c->Lambda_Q10 = f->Lambda_Q10; c->LTP_scale_Q14 = f->LTP_scale_Q14;
    for (int j = 0; j < LPC_ORDER; j++) { c->PredCoef_Q12[0][j] = f->PredCoef_Q12[0][j]; c->PredCoef_Q12[1][j] = f->PredCoef_Q12[1][j]; }
    for (int j = 0; j < NB_SUBFR * LTP_ORDER; j++) c->LTPCoef_Q14[j] = f->LTPCoef_Q14[j];
    for (int j = 0; j < NB_SUBFR * SHAPE_ORDER; j++) c->AR2_Q13[j] = f->AR2_Q13[j];
}
SB_HD void nsqio_frame_from(NsqFrameIn* f, const EncCtrl* c, const i16* x) {
    f->sigtype = c->sigtype; f->QuantOffsetType = c->QuantOffsetType; f->Seed = c->Seed; f->NLSFInterpCoef_Q2 = c->NLSFInterpCoef_Q2;
    for (int k = 0; k < NB_SUBFR; k++) {
        f->pitchL[k] = c->pitchL[k]; f->Gains_Q16[k] = c->Gains_Q16[k];
        f->LF_shp_Q14[k] = c->LF_shp_Q14[k]; f->Tilt_Q14[k] = c->Tilt_Q14[k]; f->HarmShapeGain_Q14[k] = c->HarmShapeGain_Q14[k];
    }
    f->DeltaGains_Q16 = c->DeltaGains_Q16; f->Lambda_Q10 = c->Lambda_Q10; f->LTP_scale_Q14 = c->LTP_scale_Q14;
    for (int j = 0; j < LPC_ORDER; j++) { f->PredCoef_Q12[0][j] = c->PredCoef_Q12[0][j]; f->PredCoef_Q12[1][j] = c->PredCoef_Q12[1][j]; }
    for (int j = 0; j < NB_SUBFR * LTP_ORDER; j++) f->LTPCoef_Q14[j] = c->LTPCoef_Q14[j];
    for (int j = 0; j < NB_SUBFR * SHAPE_ORDER; j++) f->AR2_Q13[j] = c->AR2_Q13[j];
    for (int i = 0; i < FRAME; i++) f->x[i] = x[i];
}
// into a NsqState: the upper halves of the two long buffers are written by a frame before it reads them, except the two
// read-ahead slots, which stay zero
SB_HD void nsqio_state_to(NsqState* s, const NsqStateIO* o) {
    for (int i = 0; i < FRAME; i++) { s->xq[i] = o->xq[i]; s->xq[FRAME + i] = 0; s->sLTP_shp_Q10[i] = o->sLTP_shp_Q10[i]; s->sLTP_shp_Q10[FRAME + i] = 0; }
    s->sLTP_shp_Q10[2 * FRAME] = s->sLTP_shp_Q10[2 * FRAME + 1] = 0;
    for (int i = 0; i < DD_DELAY; i++) s->sLPC_Q14[i] = o->sLPC_Q14[i];
    for (int i = 0; i < SHAPE_ORDER; i++) s->sAR2_Q14[i] = o->sAR2_Q14[i];
    s->sLF_AR_shp_Q12 = o->sLF_AR_shp_Q12; s->lagPrev = o->lagPrev; s->prev_inv_gain_Q16 = o->prev_inv_gain_Q16;
}
SB_HD void nsqio_state_from(NsqStateIO* o, const NsqState* s) {
    for (int i = 0; i < FRAME; i++) { o->xq[i] = s->xq[i]; o->sLTP_shp_Q10[i] = s->sLTP_shp_Q10[i]; }
    for (int i = 0; i < DD_DELAY; i++) o->sLPC_Q14[i] = s->sLPC_Q14[i];
    for (int i = 0; i < SHAPE_ORDER; i++) o->sAR2_Q14[i] = s->sAR2_Q14[i];
    o->sLF_AR_shp_Q12 = s->sLF_AR_shp_Q12; o->lagPrev = s->lagPrev; o->prev_inv_gain_Q16 = s->prev_inv_gain_Q16;
}
}  // namespace sb
#endif
#endif
