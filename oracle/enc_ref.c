/* Whole packets through the reference encoder, AGR_Sate_Encoder_Encode, with what the voice-activity detector and the
 * high-band gain stage saw and produced in every frame, for the stage tests of the VAD and payload kernels
 * (tests/test_gpu_enc_stages.py).  Test infrastructure only.
 *
 * oracle/Makefile compiles this file against the headers of the unmodified FIX tree and links it with its sources and five
 * linker taps (-Wl,--wrap), each on a function defined in a different source file from its caller:
 *   SKP_Silk_VAD_GetSA_Q8            the 8 kHz low-band frame, the VAD state before and after, its outputs;
 *   SKP_Silk_SDK_Get_Encoder_Residue the quantiser's excitation r (Q10) of every SILK frame, which the high band's gains read;
 *   AGR_Sate_lsp_quant_highband      the high-band LSP index of every high-band frame;
 *   SKP_Silk_LPC_analysis_filter     the high-band excitation of every sub-frame (order 8 only; the SILK core's are 10);
 *   AGR_Sate_gain_quant_highband_fix the gain going in (after its int16 cast) and the index coming out, per sub-frame.
 * The taps record only while encref_run's own AGR_Sate_Encoder_Encode call runs; otherwise they only forward.
 *
 * The encoder handle is a real one (AGR_Sate_Encoder_Init) with the product's settings: rate, DTX, 20 / 40 ms packets, joint
 * mode 1 and useMDIndex, and the expected loss written into its SILK control the way Init writes it. */
#include <stdint.h>
#include <string.h>
#include "SKP_Silk_main_FIX.h"
#include "AGR_BWE_main_FIX.h"
#include "AGR_JC1_SDK_API.h"

#define FR 160                  /* SILK frame (8 kHz, 20 ms) */
#define NV 28                   /* VAD state as 28 int32: AnaState[2], AnaState1[2], AnaState2[2], XnrgSubfr[4], NrgRatioSmth_Q8[4],
                                   NL[4], inv_NL[4], NoiseLevelBias[4], counter, HPstate (the product's VadState order) */
#define HB_SF 80                /* longest high-band sub-frame (joint mode 1) */
#define MAXB 1024

/* one packet's record; oracle/enc_ref.py mirrors the layout (encref_sizes checks it) */
typedef struct {
    int16_t low[2][FR];                     /* VAD input of each SILK frame */
    int32_t vad_before[2][NV], vad_after[2][NV];
    int32_t sa_Q8[2], snr_Q7[2], quality_Q15[2][4], tilt_Q15[2];
    int32_t res_Q10[2][FR];                 /* SKP_Silk_SDK_Get_Encoder_Residue of each SILK frame */
    int32_t hb_lsp_idx[2];
    int16_t hb_exc[2][4][HB_SF];            /* high-band excitation of each sub-frame (its first BWE_SubFrameSize samples) */
    int32_t hb_gain[2][4], hb_gain_idx[2][4];
    int32_t n_vad, n_res, n_lsp, n_gain;    /* tapped calls during the packet */
    int32_t ret;                            /* AGR_Sate_Encoder_Encode's return value: bytes written */
    int32_t nbytes[2];                      /* nBytesOut[0..1] */
    int32_t no_speech_counter, in_dtx;      /* SILK state after the packet */
    uint8_t payload[MAXB];
} EncPacketRec;

void encref_sizes(int* s) { s[0] = (int)sizeof(EncPacketRec); }

static EncPacketRec* g_rec;                 /* non-NULL while encref_run's encode call runs */
static int16_t g_exc[HB_SF];                /* the last order-8 analysis filter output */

static void vad_flat(int32_t* d, const SKP_Silk_VAD_state* v) {
    int i, k = 0;
    for (i = 0; i < 2; i++) d[k++] = v->AnaState[i];
    for (i = 0; i < 2; i++) d[k++] = v->AnaState1[i];
    for (i = 0; i < 2; i++) d[k++] = v->AnaState2[i];
    for (i = 0; i < 4; i++) d[k++] = v->XnrgSubfr[i];
    for (i = 0; i < 4; i++) d[k++] = v->NrgRatioSmth_Q8[i];
    for (i = 0; i < 4; i++) d[k++] = v->NL[i];
    for (i = 0; i < 4; i++) d[k++] = v->inv_NL[i];
    for (i = 0; i < 4; i++) d[k++] = v->NoiseLevelBias[i];
    d[k++] = v->counter;
    d[k++] = v->HPstate;
}

SKP_int __real_SKP_Silk_VAD_GetSA_Q8(SKP_Silk_VAD_state* v, SKP_int* pSA_Q8, SKP_int* pSNR_dB_Q7, SKP_int pQuality_Q15[4],
                                     SKP_int* pTilt_Q15, const SKP_int16 pIn[], const SKP_int framelength);
SKP_int __wrap_SKP_Silk_VAD_GetSA_Q8(SKP_Silk_VAD_state* v, SKP_int* pSA_Q8, SKP_int* pSNR_dB_Q7, SKP_int pQuality_Q15[4],
                                     SKP_int* pTilt_Q15, const SKP_int16 pIn[], const SKP_int framelength) {
    const int f = g_rec ? g_rec->n_vad : 2;
    SKP_int ret, b;
    if (f < 2 && framelength == FR) {
        memcpy(g_rec->low[f], pIn, sizeof(g_rec->low[f]));
        vad_flat(g_rec->vad_before[f], v);
    }
    ret = __real_SKP_Silk_VAD_GetSA_Q8(v, pSA_Q8, pSNR_dB_Q7, pQuality_Q15, pTilt_Q15, pIn, framelength);
    if (f < 2 && framelength == FR) {
        vad_flat(g_rec->vad_after[f], v);
        g_rec->sa_Q8[f] = *pSA_Q8;
        g_rec->snr_Q7[f] = *pSNR_dB_Q7;
        for (b = 0; b < 4; b++) g_rec->quality_Q15[f][b] = pQuality_Q15[b];
        g_rec->tilt_Q15[f] = *pTilt_Q15;
    }
    if (g_rec) g_rec->n_vad++;
    return ret;
}

SKP_int __real_SKP_Silk_SDK_Get_Encoder_Residue(void* encState, SKP_int32* r);
SKP_int __wrap_SKP_Silk_SDK_Get_Encoder_Residue(void* encState, SKP_int32* r) {
    SKP_int ret = __real_SKP_Silk_SDK_Get_Encoder_Residue(encState, r);
    if (g_rec && g_rec->n_res < 2 && ((SKP_Silk_encoder_state_FIX*)encState)->sCmn.frame_length == FR)
        memcpy(g_rec->res_Q10[g_rec->n_res], r, sizeof(g_rec->res_Q10[0]));
    if (g_rec) g_rec->n_res++;
    return ret;
}

SKP_int32 __real_AGR_Sate_lsp_quant_highband(SKP_int32* lsp, SKP_int32 order);
SKP_int32 __wrap_AGR_Sate_lsp_quant_highband(SKP_int32* lsp, SKP_int32 order) {
    SKP_int32 idx = __real_AGR_Sate_lsp_quant_highband(lsp, order);
    if (g_rec && g_rec->n_lsp < 2) g_rec->hb_lsp_idx[g_rec->n_lsp] = idx;
    if (g_rec) g_rec->n_lsp++;
    return idx;
}

void __real_SKP_Silk_LPC_analysis_filter(const SKP_int16* in, const SKP_int16* B, SKP_int16* S, SKP_int16* out, const SKP_int32 len,
                                         const SKP_int32 Order);
void __wrap_SKP_Silk_LPC_analysis_filter(const SKP_int16* in, const SKP_int16* B, SKP_int16* S, SKP_int16* out, const SKP_int32 len,
                                         const SKP_int32 Order) {
    __real_SKP_Silk_LPC_analysis_filter(in, B, S, out, len, Order);
    if (g_rec && Order == 8 && len <= HB_SF) memcpy(g_exc, out, sizeof(SKP_int16) * (size_t)len);
}

SKP_int32 __real_AGR_Sate_gain_quant_highband_fix(SKP_int16 gain, const SKP_int16* cdbk, SKP_int32 nVect);
SKP_int32 __wrap_AGR_Sate_gain_quant_highband_fix(SKP_int16 gain, const SKP_int16* cdbk, SKP_int32 nVect) {
    SKP_int32 idx = __real_AGR_Sate_gain_quant_highband_fix(gain, cdbk, nVect);
    if (g_rec && g_rec->n_gain < 8) {
        const int f = g_rec->n_gain >> 2, sub = g_rec->n_gain & 3;
        g_rec->hb_gain[f][sub] = gain;
        g_rec->hb_gain_idx[f][sub] = idx;
        memcpy(g_rec->hb_exc[f][sub], g_exc, sizeof(g_exc));
    }
    if (g_rec) g_rec->n_gain++;
    return idx;
}

/* npk packets of a freshly initialised encoder: pcm [npk][16 * framesize_ms] -> rec [npk]; returns 0, or -1 when the
   reference refuses the settings */
int encref_run(int rate, int dtx, int framesize_ms, int joint, int mdi, int loss, int npk, const int16_t* pcm, EncPacketRec* rec) {
    USER_Ctrl_enc u;
    SATEEncCtl* h;
    SKP_Silk_encoder_state_FIX* s;
    const int L = 16 * framesize_ms;
    int p;
    memset(&u, 0, sizeof(u));
    u.mode = 2; u.targetRate_bps = rate; u.samplerate = 16000; u.dtx_enable = dtx;
    u.framesize_ms = framesize_ms; u.joint_enable = u.joint_mode = joint ? 1 : 0; u.useMDIndex = mdi;
    h = (SATEEncCtl*)AGR_Sate_Encoder_Init(&u);
    if (!h) return -1;
    h->encControl.packetLossPercentage = loss;
    s = (SKP_Silk_encoder_state_FIX*)h->stEnc;
    for (p = 0; p < npk; p++) {
        SKP_int16 nb[6] = {0, 0, 0, 0, 0, 0};
        memset(&rec[p], 0, sizeof(EncPacketRec));
        g_rec = &rec[p];
        rec[p].ret = AGR_Sate_Encoder_Encode(h, pcm + (size_t)p * L, rec[p].payload, MAXB, nb);
        g_rec = NULL;
        rec[p].nbytes[0] = nb[0];
        rec[p].nbytes[1] = nb[1];
        rec[p].no_speech_counter = s->sCmn.noSpeechCounter;
        rec[p].in_dtx = s->sCmn.inDTX;
    }
    AGR_Sate_Encoder_Uninit(h);
    return 0;
}
