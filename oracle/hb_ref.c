/* Direct entry to the reference's high-band frame analysis, AGR_Bwe_encode_frame_FIX, one frame per step, for the routine
 * tests of the high-band analysis kernel (tests/test_gpu_bands.py).  Test infrastructure only.
 *
 * oracle/Makefile compiles this file against the headers of the unmodified FIX tree and links it with its sources and three
 * linker taps (-Wl,--wrap): AGR_Sate_lsp_quant_highband (the NLSF vector going in, the index and the quantised vector coming
 * out), SKP_Silk_NLSF2A_stable (the filter of each sub-frame) and SKP_Silk_LPC_analysis_filter (the excitation of each
 * sub-frame).  The taps record only while hbref_run's own call of the frame analysis runs; otherwise they only forward.
 *
 * The encoder handle is a real one (AGR_Sate_Encoder_Init), so the frame, LPC-block and sub-frame lengths, the delay of the
 * high band behind the low band and the reset state are the reference's own.  Per frame the analysis is called on that
 * handle's high-band state with bits = NULL (nothing is packed) and a zero low-band excitation (it only feeds the gains). */
#include <stdint.h>
#include <string.h>
#include "SKP_Silk_main_FIX.h"
#include "AGR_BWE_main_FIX.h"
#include "AGR_JC1_SDK_API.h"

#define HB_ORD 8
#define HB_FMAX 320
#define HB_BUF (2 * HB_FMAX + 40)

/* one frame's record; oracle/hb_ref.py mirrors the layout (hbref_sizes checks it) */
typedef struct {
    int32_t nlsf_in[HB_ORD];       /* NLSF_Q15 handed to AGR_Sate_lsp_quant_highband */
    int32_t nlsf_q[HB_ORD];        /* the quantised vector it leaves there */
    int32_t lsp_idx;               /* its return value */
    int32_t n_quant, n_nlsf2a, n_filter;   /* tapped calls during the frame */
    int16_t coef[4][HB_ORD];       /* SKP_Silk_NLSF2A_stable output of every sub-frame */
    int16_t exc[HB_FMAX];          /* SKP_Silk_LPC_analysis_filter output, the four sub-frames back to back */
    int16_t x_hb_buf[HB_BUF];      /* high-band buffer after the frame (its first 2 * 320 + 40 samples) */
    int32_t prev_nlsfq[HB_ORD];    /* HB_prev_NLSFq_Q15 after the frame */
} HbFrameRec;

void hbref_sizes(int* s) { s[0] = (int)sizeof(HbFrameRec); }

SKP_int32 AGR_Bwe_encode_frame_FIX(AGR_Sate_HB_encoder_control_FIX* hbEncCtrl, AGR_Sate_encoder_hb_state_FIX* psHBEnc, NovaBits* bits,
                                   SKP_int16* high, SKP_int32* residue, SKP_int16* nBytesOut);

static HbFrameRec* g_rec;          /* non-NULL while hbref_run's frame analysis runs */

SKP_int32 __real_AGR_Sate_lsp_quant_highband(SKP_int32* lsp, SKP_int32 order);
SKP_int32 __wrap_AGR_Sate_lsp_quant_highband(SKP_int32* lsp, SKP_int32 order) {
    SKP_int32 idx;
    if (g_rec && order == HB_ORD) memcpy(g_rec->nlsf_in, lsp, sizeof(g_rec->nlsf_in));
    idx = __real_AGR_Sate_lsp_quant_highband(lsp, order);
    if (g_rec && order == HB_ORD) {
        memcpy(g_rec->nlsf_q, lsp, sizeof(g_rec->nlsf_q));
        g_rec->lsp_idx = idx;
        g_rec->n_quant++;
    }
    return idx;
}

void __real_SKP_Silk_NLSF2A_stable(SKP_int16* pAR_Q12, const SKP_int32* pNLSF, const SKP_int LPC_order);
void __wrap_SKP_Silk_NLSF2A_stable(SKP_int16* pAR_Q12, const SKP_int32* pNLSF, const SKP_int LPC_order) {
    __real_SKP_Silk_NLSF2A_stable(pAR_Q12, pNLSF, LPC_order);
    if (g_rec && LPC_order == HB_ORD && g_rec->n_nlsf2a < 4) memcpy(g_rec->coef[g_rec->n_nlsf2a], pAR_Q12, sizeof(g_rec->coef[0]));
    if (g_rec) g_rec->n_nlsf2a++;
}

void __real_SKP_Silk_LPC_analysis_filter(const SKP_int16* in, const SKP_int16* B, SKP_int16* S, SKP_int16* out, const SKP_int32 len,
                                         const SKP_int32 Order);
void __wrap_SKP_Silk_LPC_analysis_filter(const SKP_int16* in, const SKP_int16* B, SKP_int16* S, SKP_int16* out, const SKP_int32 len,
                                         const SKP_int32 Order) {
    __real_SKP_Silk_LPC_analysis_filter(in, B, S, out, len, Order);
    if (g_rec && (g_rec->n_filter + 1) * len <= HB_FMAX) memcpy(g_rec->exc + g_rec->n_filter * len, out, sizeof(SKP_int16) * (size_t)len);
    if (g_rec) g_rec->n_filter++;
}

/* setting: 0 = 40 ms packets, 1 = 20 ms packets (both: 20 ms high-band frames of 160 samples), 2 = joint mode 1 (one 40 ms
   frame of 320 samples per packet) */
static SATEEncCtl* open_encoder(int setting) {
    USER_Ctrl_enc u;
    memset(&u, 0, sizeof(u));
    u.mode = 2; u.targetRate_bps = 13600; u.samplerate = 16000;
    u.framesize_ms = setting == 1 ? 20 : 40;
    u.joint_enable = u.joint_mode = setting == 2;
    return (SATEEncCtl*)AGR_Sate_Encoder_Init(&u);
}

int hbref_frame_size(int setting) {
    SATEEncCtl* h = open_encoder(setting);
    int F;
    if (!h) return -1;
    F = h->HBencControl.BWE_FrameSize;
    AGR_Sate_Encoder_Uninit(h);
    return F;
}

/* nfr consecutive frames of a freshly initialised encoder: high [nfr][F] -> rec [nfr]; returns F, or -1 */
int hbref_run(int setting, int nfr, const int16_t* high, HbFrameRec* rec) {
    SATEEncCtl* h = open_encoder(setting);
    AGR_Sate_HB_encoder_control_FIX* c;
    AGR_Sate_encoder_hb_state_FIX* s;
    int F, f;
    if (!h) return -1;
    c = &h->HBencControl;
    s = (AGR_Sate_encoder_hb_state_FIX*)h->stHBEnc;
    F = c->BWE_FrameSize;
    if (F > HB_FMAX || c->BWE_LPCOrder != HB_ORD || 2 * F + c->lb_Delay * c->hb_KHz > HB_BUF) { AGR_Sate_Encoder_Uninit(h); return -1; }
    for (f = 0; f < nfr; f++) {
        SKP_int16 x[HB_FMAX], nbytes = 0;
        SKP_int32 residue[HB_FMAX];
        memcpy(x, high + (size_t)f * F, sizeof(SKP_int16) * (size_t)F);
        memset(residue, 0, sizeof(residue));
        memset(&rec[f], 0, sizeof(HbFrameRec));
        g_rec = &rec[f];
        AGR_Bwe_encode_frame_FIX(c, s, NULL, x, residue, &nbytes);
        g_rec = NULL;
        memcpy(rec[f].x_hb_buf, s->x_hb_buf_fix, sizeof(rec[f].x_hb_buf));
        memcpy(rec[f].prev_nlsfq, s->HB_prev_NLSFq_Q15, sizeof(rec[f].prev_nlsfq));
    }
    AGR_Sate_Encoder_Uninit(h);
    return F;
}
