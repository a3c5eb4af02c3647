// solo_b200 -- G.711 gateway (include/solo_b200.h, solo_b200_g711_*): PSTN and SIP participants in a 16 kHz room.  Written
// once for the gateway kernels (solo_b200.cu) and the host model (tests/hostsim/g711_model.cpp).
//   companding : ITU-T G.711 with the integer mapping of the classic Sun / CCITT g711.c: mu-law on x >> 2 (bias 33, clip
//                8159, complemented code), A-law on x >> 3 (code XOR 0x55); expansion gives that code's 16-bit values
//   uplink     : 8 kHz G.711 -> the codec's 16 kHz rows: expansion (lost 20 ms frames are silence), the encoder's VAD on
//                every 160-sample frame, the fixed-point synthesis filter bank over (low = the 8 kHz signal, high = 0)
//   downlink   : 16 kHz rows -> 8 kHz G.711: the low band of the fixed-point QMF analysis (the band split), compressed
// No resampler is involved: the filter bank that splits and joins the codec's bands is the 2:1 rate change.
#pragma once
#include "sb_activity.cuh"
#include "sb_dec.cuh"
#include "sb_enc.cuh"

namespace sb {

enum { G711_ULAW = 0, G711_ALAW = 1 };
#define SB_G711_VAD_THR SB_FIXC(0.1f, 8)    // vad_flag_and_dtx: the encoder codes a frame's VAD flag from speech_activity_Q8 >= this

// Per-stream state of the gateway
struct alignas(16) G711State {
    VadState vad;               // uplink voice activity: the encoder's detector, on the 8 kHz signal
    i16 syn_mem[32];            // uplink synthesis memory of the low band (the high band's stays zero)
    i16 ana_mem[64];            // downlink analysis memory: the band split's qmf_mem layout (63 used)
    i32 law;                    // G711_ULAW or G711_ALAW
};

SB_FN void g711_state_init(G711State* st, int law) {
    memset(st, 0, sizeof(G711State));
    vad_init(&st->vad);
    st->law = law;
}

// linear16 -> code
SB_HD u8 g711_compress(int law, i16 x) {
    if (law == G711_ALAW) {
        i32 v = x >> 3;
        int mask = 0xD5;
        if (v < 0) { mask = 0x55; v = -v - 1; }                       // 0 .. 4095
        const int seg = v < 32 ? 0 : 27 - clz32(v);                    // segment ends 0x1F, 0x3F, ... 0xFFF
        const int q = (v >> (seg < 2 ? 1 : seg)) & 0xF;
        return (u8)(((seg << 4) | q) ^ mask);
    }
    i32 v = x >> 2;
    int mask = 0xFF;
    if (v < 0) { v = -v; mask = 0x7F; }
    v = (v > 8159 ? 8159 : v) + 33;                                    // 33 .. 8192
    const int seg = 26 - clz32(v);                                     // segment ends 0x3F, 0x7F, ... 0x1FFF
    if (seg >= 8) return (u8)(0x7F ^ mask);
    return (u8)(((seg << 4) | ((v >> (seg + 1)) & 0xF)) ^ mask);
}

// code -> linear16
SB_HD i16 g711_expand(int law, u8 c) {
    if (law == G711_ALAW) {
        const int a = c ^ 0x55, seg = (a & 0x70) >> 4;
        i32 t = (a & 0xF) << 4;
        t += seg == 0 ? 8 : 0x108;
        if (seg > 1) t <<= seg - 1;
        return (i16)((a & 0x80) ? t : -t);
    }
    const int u = ~c & 0xFF;
    const i32 t = (((u & 0xF) << 3) + 0x84) << ((u & 0x70) >> 4);
    return (i16)((u & 0x80) ? 0x84 - t : t - 0x84);
}

// uplink sample i of a packet: the expansion of its code, 0 in a lost frame (bit i / FRAME of `lost`)
SB_HD i16 g711_up_sample(int law, u8 c, i32 lost, int i) { return ((lost >> (i / FRAME)) & 1) ? (i16)0 : g711_expand(law, c); }

// the uplink's activity flags from the frames' speech activity: bit f = VAD flag of a received frame, bit 2 + f = frame f
// was lost (concealed), as the decoder reports them
SB_HD int g711_flags(const i32* sa_Q8, i32 lost, int nf) {
    int fl = 0;
    for (int f = 0; f < nf; f++) fl |= ((lost >> f) & 1) ? 4 << f : (sa_Q8[f] >= SB_G711_VAD_THR ? 1 << f : 0);
    return fl;
}

// the uplink's voice activity: the encoder's VAD stage over the nf frames of the 8 kHz signal x8, lost frames included
SB_FN int g711_vad(VadState* v, const i16* x8, int nf, i32 lost, i32* sa_Q8) {
    i32 quality_Q15[2][4], tilt_Q15[2];
    vad_packet(v, x8, nf, sa_Q8, quality_Q15, tilt_Q15);
    return g711_flags(sa_Q8, lost, nf);
}

// ---- scalar model of the uplink kernels: one packet of nf frames, codes [nf * FRAME] -> pcm [2 * nf * FRAME], flags ----
SB_FN int g711_uplink(G711State* st, const u8* codes, i32 lost, int nf, i16* pcm, i32* sa_Q8) {
    enum { M2 = 32 };
    const int N2 = nf * FRAME;
    i16 x8[2 * FRAME], yy1[M2 + 2 * FRAME], yy2[M2 + 2 * FRAME];
    for (int i = 0; i < N2; i++) x8[i] = g711_up_sample(st->law, codes[i], lost, i);
    const int fl = g711_vad(&st->vad, x8, nf, lost, sa_Q8);
    // the decoder's fixed-point synthesis (dec_synth) with a zero high band
    for (int i = 0; i < N2; i++) { yy1[i] = x8[N2 - 1 - i]; yy2[i] = 0; }
    for (int i = 0; i < M2; i++) { yy1[N2 + i] = st->syn_mem[i]; yy2[N2 + i] = 0; }
    for (int i = 0; i < N2; i += 2) qmf_synth_group_fix(yy1, yy2, SB_T(qmf_fix), N2, i, pcm + 2 * i);
    for (int i = 0; i < M2; i++) st->syn_mem[i] = yy1[i];
    return fl;
}

// ---- scalar model of the downlink kernel: one row of N = 2 * nf * FRAME samples -> low band lo [N / 2] -> codes [N / 2] --
SB_FN void g711_downlink(G711State* st, const i16* pcm, int N, i16* lo, u8* codes) {
    i16 hi[PACKET / 2];
    qmf_decomp(pcm, lo, hi, st->ana_mem, N);
    for (int k = 0; k < N / 2; k++) codes[k] = g711_compress(st->law, lo[k]);
}

}  // namespace sb
