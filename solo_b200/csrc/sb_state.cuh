// solo_b200 -- per-stream persistent state (device arena slot) and per-frame control block.
//
// The reference allocates ~88 KB per encoder handle (structs dimensioned for 24 kHz, four
// interleaves, LBRR, resamplers: JC1_SDK_SRC_ARM/src/libSATECodec/SKP_Silk_structs.h:142-260,
// SKP_Silk_structs_FIX.h:78-108, libBWE/AGR_BWE_structs.h:14-45).  For the only configuration the
// SOLO SDK can reach (8 kHz SILK core, order-10 LPC, complexity 2, two descriptions, LBRR off,
// resamplers bypassed -- SURVEY.md 2.2) the live state is the POD below.
#pragma once
#include "sb_common.cuh"

namespace sb {

// ---- fixed configuration (SURVEY.md 2.2) -----------------------------------------------------------
enum {
    FRAME = 160,           // 20 ms at 8 kHz
    SUBFR = 40,            // 5 ms
    NB_SUBFR = 4,
    LPC_ORDER = 10,        // predictLPCOrder (control_codec_FIX.c:278)
    SHAPE_ORDER = 16,      // shapingLPCOrder, complexity 2 (setup_complexity.h:85)
    LTP_ORDER = 5,
    LA_SHAPE = 40,         // 5 ms
    LA_PITCH = 16,         // 2 ms
    SHAPE_WIN = 120,       // shapeWinLength
    PITCH_LPC_WIN = 192,   // 24 ms
    N_DD = 4,              // delayed-decision states
    DD_DELAY = 32,         // DECISION_DELAY
    DD_MASK = 31,
    LTP_BUF = 512,
    LTP_MASK = 511,
    WARPING_Q16 = 7864,    // 8 * FIX_CONST(0.015f,16)
    PACKET = 640,          // 40 ms at 16 kHz
    HB_FRAME = 160,
    HB_ORDER = 8,
    MAX_PAYLOAD = 1024,
};

// SKP_Silk_nsq_state (structs.h:44-57) reduced to 8 kHz dimensions.
struct NsqState {
    i16 xq[2 * FRAME];
    i32 sLTP_shp_Q10[2 * FRAME + 2];  // +2: read-ahead slots that stay zero (first unvoiced frame, App. A Q5)
    i32 sLPC_Q14[DD_DELAY];
    i32 sAR2_Q14[SHAPE_ORDER];
    i32 sLF_AR_shp_Q12;
    i32 lagPrev;
    i32 prev_inv_gain_Q16;
};

// SKP_Silk_VAD_state (structs.h:69-80)
struct VadState {
    i32 AnaState[2], AnaState1[2], AnaState2[2];
    i32 XnrgSubfr[4];
    i32 NrgRatioSmth_Q8[4];
    i32 NL[4], inv_NL[4], NoiseLevelBias[4];
    i32 counter;
    i16 HPstate;
};

// Persistent encoder state, split by consumer: EncSilk is what the warp-per-stream analysis kernel stages in shared memory
// (and what the entropy-coding stage reads), EncBands belongs to the band-split and high-band kernels, NsqState x 3 to the
// quantiser kernel.  EncCore = EncSilk + EncBands is the part the scalar model (tests/hostsim) passes around as one object.
struct alignas(16) EncSilk {
    // --- per-stream settings: rate, DTX and expected loss (packetLoss_perc, last field) are set at Init and may change
    //     between packets (enc_set_control, control_codec_FIX.c:56-130,319-389); the rest are fixed at Init ---
    i32 SNR_dB_Q7;
    i32 SNRPerMD_dB_Q7;
    i32 useMDIndex;
    i32 useDTX;
    i32 targetRate_bps;  // SILK core rate (user rate - 1600, or - 800 with joint mode 1), clamped to [5000, 100000]
    i32 frames_per_packet;  // 2: 40 ms packets (the headline configuration), 1: 20 ms packets (AGR_BWE_SDK_API.c:78-81,106-110)
    i32 hb_frame;           // high-band frame length: 160 (20 ms), or 320 with joint_mode 1 (one 40 ms HB frame per packet, :63-66)
    // --- SILK encoder ---
    VadState vad;
    i32 In_HP_State[2];
    i32 variable_HP_smth1_Q15, variable_HP_smth2_Q15;
    // shape state (structs_FIX.h:44-49)
    i32 LastGainIndex, HarmBoost_smth_Q16, HarmShapeGain_smth_Q16, Tilt_smth_Q16;
    // prefilter state (structs_FIX.h:54-63)
    i16 pf_sLTP_shp[LTP_BUF];
    i32 pf_sAR_shp[SHAPE_ORDER + 1];
    i32 pf_sLTP_shp_buf_idx, pf_sLF_AR_shp_Q12, pf_sLF_MA_shp_Q12, pf_sHarmHP, pf_lagPrev;
    i32 prev_NLSFq_Q15[LPC_ORDER];
    i16 x_buf[2 * FRAME + LA_SHAPE];
    i32 LTPCorr_Q15, avgGain_Q16, speech_activity_Q8, prevLTPredCodGain_Q7, HPLTPredCodGain_Q7;
    i32 prev_sigtype, prevLag, typeOffsetPrev_md[2], frameCounter, first_frame_after_reset;
    i32 noSpeechCounter, inDTX, vadFlag;
    // expected packet loss (0-100) the LTP scaling plans for (LTP_scale_ctrl_FIX.c:61).  Last, in what was the struct's
    // alignment padding: the fields before it keep the offsets, and so the vector loads, the kernels were built around.
    i32 packetLoss_perc;
};
struct alignas(16) EncBands {
    i16 qmf_mem[64];             // QMF analysis memory (AGR_BWE_structs.h:34)
    // --- high band (AGR_BWE_structs.h:14-19) ---
    i16 x_hb_buf[2 * 320 + 40];  // ring of 2 * hb_frame + 40; with hb_frame = 160 the LPC analysis reads [360,480), which stays zero (App. A Q26)
    i32 hb_first;
};
struct EncCore : EncSilk, EncBands {};
struct EncState : EncCore {
    NsqState nsq[3];  // 0 = centre, 1 = description 1, 2 = description 2
};

// Per-frame encoder control (SKP_Silk_encoder_control{,_FIX}: structs.h:262-290, structs_FIX.h:112-153)
struct EncCtrl {
    i32 lagIndex, contourIndex, PERIndex;
    i32 LTPIndex[NB_SUBFR];
    i32 NLSFIndices[6];
    i32 NLSFInterpCoef_Q2;
    i32 GainsIndices[NB_SUBFR];
    i32 DeltaGainsIndices;
    i32 Seed;
    i32 LTP_scaleIndex;
    i32 QuantOffsetType;
    i32 sigtype;
    i32 pitchL[NB_SUBFR];
    i32 Gains_Q16[NB_SUBFR];
    i32 DeltaGains_Q16;
    i16 PredCoef_Q12[2][LPC_ORDER];
    i16 LTPCoef_Q14[LTP_ORDER * NB_SUBFR];
    i32 LTP_scale_Q14;
    i16 AR1_Q13[NB_SUBFR * SHAPE_ORDER];
    i16 AR2_Q13[NB_SUBFR * SHAPE_ORDER];
    i32 LF_shp_Q14[NB_SUBFR];
    i32 GainsPre_Q14[NB_SUBFR];
    i32 HarmBoost_Q14[NB_SUBFR];
    i32 Tilt_Q14[NB_SUBFR];
    i32 HarmShapeGain_Q14[NB_SUBFR];
    i32 Lambda_Q10;
    i32 input_quality_Q14, coding_quality_Q14;
    i32 pitch_freq_low_Hz;
    i32 current_SNR_dB_Q7, current_SNRPerMD_dB_Q7;
    float md_delta_gain_par;
    i32 sparseness_Q8;
    i32 predGain_Q16;
    i32 LTPredCodGain_Q7;
    i32 input_quality_bands_Q15[4];
    i32 input_tilt_Q15;
    i32 ResNrg[NB_SUBFR];
    i32 ResNrgQ[NB_SUBFR];
};

// ---- per-packet hand-over between the encoder stages (device: global scratch, one slot per stream) -------------------
// The scalar model (sb_enc.cuh enc_packet) fills the same fields in the same order.
//   stage A (analysis): VAD of the packet's frames           -> vad_*
//                       core analysis (warp per stream)      -> c[f], x_hp, ar_Q24, shape_par, nlsf_Q15, lpc_in_pre, local_gains
//                       high-band analysis (warp per stream) -> hb_lsp_idx, hb_nrg0
//                       shaping filters (thread per window)  -> c[f] AR1 / AR2 / GainsPre
//                       gains (thread per stream)            -> c[f] prediction filters, gains, vadFlag, dtx_drop
//                       prefilter (thread per stream)        -> xfw
//   stage B (MD noise-shaping quantiser)                     : consumes c[f], xfw[f]; produces q_md[f], r16[f], c[f].Seed
//   stage C (entropy coding + packing)                       : range-codes both descriptions, high-band gains, payload assembly
//                                                              (the same three steps per description in both builds, sb_enc.cuh)
struct EncScratch {
    EncCtrl c[2];
    i16 xfw[2][FRAME];
    i8 q_md[2][2][FRAME];  // [frame][description]
    i16 r16[2][FRAME];
    i32 vadFlag[2];
    i32 hb_lsp_idx[2];
    i32 hb_nrg0[2][4];
    i32 dtx_drop;
    // voice-activity results of the packet's frames, written by the VAD kernel and consumed by the analysis kernel
    i32 vad_sa_Q8[2], vad_quality_Q15[2][4], vad_tilt_Q15[2];
    // hand-over from the analysis kernel to the shaping-filter / prefilter kernels that run after it
    i16 x_hp[2][FRAME];                          // high-passed input, delayed by the shaping look-ahead (what the prefilter filters)
    i32 ar_Q24[2][NB_SUBFR][2][SHAPE_ORDER];     // AR2, AR1 of every shaping window after bandwidth expansion
    i32 shape_par[2][2];                         // warping_Q16, pre-gain multiplier Q16
    // ... and to the gain kernel: quantised NLSFs (interpolated first half, second half), the LPC analysis input, gains
    i32 nlsf_Q15[2][2][LPC_ORDER];
    i16 lpc_in_pre[2][NB_SUBFR * LPC_ORDER + FRAME];
    i32 local_gains[2][NB_SUBFR];
    // quantiser kernel: random-generator states of the delayed-decision window, [quantiser][position][state]
    i32 nsq_rand[3][DD_DELAY][N_DD];
};

// Range coder (SKP_Silk_range_coder_state, structs.h:85-92); the byte buffer lives with the caller.
struct RangeEnc {
    u32 base_Q32, range_Q16;
    i32 bufferIx, error;
    u8* buf;
    i32 bufLen;
};

}  // namespace sb
