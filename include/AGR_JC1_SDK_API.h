/*
 * solo_b200 -- drop-in C ABI of the SOLO codec SDK.
 *
 * The six entry points below have the same names, argument order, argument meaning, ownership rules and
 * return conventions as the reference SDK header
 *     /root/reference/JC1_SDK_SRC_{ARM,FLP}/interface/AGR_JC1_SDK_API.h:11-64
 * (implementation replaced: .../src/libBWE/AGR_BWE_SDK_API.c:11-296), so a caller written against the
 * reference links against libsolo_b200.so unchanged.  Behind them every handle owns one stream slot of a
 * device-resident state arena and each call runs the sm_90a kernels on one stream; the batched interface
 * for tens of thousands of streams per launch is in solo_b200.h.
 *
 * Contract (reference file:line in brackets):
 *   - Encode consumes exactly framesize_ms*16 int16 samples per call (640 / 320)    [test/enc_main.c:176-184]
 *   - returns the byte count of [MD1 | MD2 | HB]; nBytesOut[0] = that count,
 *     nBytesOut[1] = len(MD2) + len(HB), HB = 4 bytes per high-band frame (8 with
 *     40 ms packets, 4 with 20 ms packets or joint mode 1); nBytesOut must hold
 *     >= 3 entries                                                                  [AGR_BWE_encode_frame_FIX.c:142-171]
 *   - Init writes back targetRate_bps = 15600 when <= 0; returns NULL for an
 *     invalid joint_mode                                                            [AGR_BWE_SDK_API.c:34-36,73-76]
 *   - Decode: lostflag 1 = lost, 2 = MD1 only, 3 = MD2+HB only, 4 = both; the
 *     caller pre-trims payload / nBytes as test/dec_main.c:245-307; nBytes[] is
 *     rewritten in place; *nSamplesOut = framesize_ms * samplerate / 1000         [AGR_BWE_decode_frame_FLP.c:171-190]
 *   - Encode/Decode/Uninit return -1 on a NULL handle; Decode returns -1 when
 *     nBytes[0] <= 0                                                                [AGR_BWE_SDK_API.c:139-141,261-270]
 * Accepted configurations (the ones the reference SDK itself can run, AGR_BWE_SDK_API.c:40-110): joint_enable 0 and
 * framesize_ms 40 or 20, or joint_enable 1 / joint_mode 1 / framesize_ms 40 (one 40 ms high-band frame per packet), at
 * samplerate 16000 for both directions and at samplerate 32000 for the DECODER only (16 kHz SILK core, 8-16 kHz high band;
 * the core rates that decode are in solo_b200.h and INTEGRATION.md).  AGR_Sate_Encoder_Init with samplerate 32000 returns
 * NULL: the 32 kHz encoder is not built yet.  Anything else (joint modes 0, 2, 3 -- "Unsupport" in the reference too)
 * makes Init return NULL.
 */
#ifndef SOLO_B200_AGR_JC1_SDK_API_H
#define SOLO_B200_AGR_JC1_SDK_API_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int32_t SKP_int32;
typedef int16_t SKP_int16;
typedef uint8_t SKP_uint8;

typedef struct {
    SKP_int32 mode;            /* ignored by the reference as well */
    SKP_int32 targetRate_bps;  /* total rate incl. 1600 b/s high band; <= 0 selects 15600 (written back) */
    SKP_int32 samplerate;      /* must be 16000 (no 32 kHz encoder yet) */
    SKP_int32 dtx_enable;      /* 0 / 1 */
    SKP_int32 framesize_ms;    /* 40 or 20 */
    SKP_int32 joint_enable;    /* 0, or 1 together with joint_mode 1 and framesize_ms 40 */
    SKP_int32 joint_mode;
    SKP_int32 useMDIndex;      /* 1: each description starts with its MD index symbol */
} USER_Ctrl_enc;

typedef struct {
    SKP_int32 packetLoss_perc; /* ignored by the reference as well */
    SKP_int32 samplerate;      /* 16000 or 32000 */
    SKP_int32 framesize_ms;    /* 40 or 20 (must match the encoder) */
    SKP_int32 joint_enable;    /* as in USER_Ctrl_enc */
    SKP_int32 joint_mode;
    SKP_int32 useMDIndex;
} USER_Ctrl_dec;

void *AGR_Sate_Encoder_Init(USER_Ctrl_enc *enc_Ctrl);
SKP_int32 AGR_Sate_Encoder_Encode(void *SATEEnc_State, const SKP_int16 *AGR_Sate_PCM, SKP_uint8 *AGR_Sate_Bit,
                                  SKP_int32 AGR_Sate_Buf_Size, SKP_int16 *nBytesOut);
int AGR_Sate_Encoder_Uninit(void *SATEEnc_State);

/* Decoder arithmetic: the reference ships a float build (JC1_SDK_SRC_FLP) and a fixed-point build (JC1_SDK_SRC_ARM) whose
   decoded PCM differs.  Each Init reads the environment variable SOLO_B200_DEC_ARITH:
     unset or "flp" : PCM of the float build (the default);
     "fix"          : PCM of the fixed-point build, bit for bit (40 ms packets and joint mode 1; with 20 ms packets the
                      fixed-point build decodes every payload twice, a defect not reproduced: Init returns NULL);
     anything else  : Init prints a message and returns NULL.
   The setting stays with the handle; changing the variable later affects only later Inits. */
void *AGR_Sate_Decoder_Init(USER_Ctrl_dec *dec_Ctrl);
SKP_int32 AGR_Sate_Decoder_Decode(void *SATEDec_State, SKP_int16 *AGR_Sate_PCM, SKP_int16 *nSamplesOut,
                                  const SKP_uint8 *AGR_Sate_Bit, SKP_int16 nBytes[], SKP_int32 lostflag);
SKP_int32 AGR_Sate_Decoder_Uninit(void *SATEDec_State);

#ifdef __cplusplus
}
#endif
#endif
