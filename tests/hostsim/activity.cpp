// Host build of the activity reports (solo_b200/csrc/sb_activity.cuh compiled by g++) with the encoder and decoder source
// they report on: the level function, the activity kernel's arithmetic on one row, and codec streams that return each
// packet's flags beside its payload or PCM.  TEST INFRASTRUCTURE ONLY; compiled by tests/test_activity.py, never linked
// into libsolo_b200.so.
//   g++ -O2 -ffp-contract=off -std=c++17 -shared -fPIC -w activity.cpp -o libactivity.so
#include <stdlib.h>

#include "../../solo_b200/csrc/sb_activity.cuh"
#include "../../solo_b200/csrc/sb_dec.cuh"
#include "../../solo_b200/csrc/sb_enc.cuh"

struct Enc { sb::EncState st; sb::EncPacketWork w; };
template <int KHZ> struct Dec { sb::DecStateT<KHZ> st; sb::DecPacketWorkT<KHZ> w; sb::DecStale stale; };
template <int KHZ> static int decode(void* p, short* pcm, const unsigned char* bits, int cap, const short* nb, int lostflag, unsigned char* flags) {
    Dec<KHZ>* h = (Dec<KHZ>*)p;
    const int r = sb::dec_packet(&h->st, &h->w, pcm, bits, cap, nb, lostflag, &h->stale);
    *flags = r < 0 ? 0 : h->w.act;      // what the decode kernel stores for the activity kernel
    return r;
}

extern "C" {
int act_level(long long E, int n) { return sb::rfc6464_level(E, n); }
// the activity kernel's level of one row of n samples
int act_row_level(const short* pcm, int n) {
    long long e = 0;
    for (int i = 0; i < n; i++) e += (long long)pcm[i] * pcm[i];
    return sb::rfc6464_level(e, n);
}

void* act_enc_create(int rate, int dtx, int mdi, int framesize_ms, int joint_hb) {
    Enc* h = (Enc*)calloc(1, sizeof(Enc));
    sb::enc_state_init(&h->st, rate, dtx, mdi, framesize_ms, joint_hb);
    return h;
}
// one packet (the scalar model of the encoder kernels); *flags = the activity kernel's flags of that packet
int act_enc_encode(void* p, const short* pcm, unsigned char* out, int cap, short* nb, unsigned char* flags) {
    Enc* h = (Enc*)p;
    const int n = sb::enc_packet(&h->st, &h->w, pcm, out, cap, nb);
    *flags = (unsigned char)sb::enc_activity_flags(&h->w.scr, h->st.frames_per_packet);
    return n;
}
void act_enc_destroy(void* p) { free(p); }

// samplerate 16000 (8 kHz core) or 32000 (16 kHz core); decode calls take the same samplerate as create
void* act_dec_create(int mdi, int framesize_ms, int joint_hb, int arith, int samplerate) {
    if (samplerate == 32000) {
        Dec<16>* h = (Dec<16>*)calloc(1, sizeof(Dec<16>));
        sb::dec_state_init(&h->st, mdi, framesize_ms, joint_hb, arith);
        return h;
    }
    Dec<8>* h = (Dec<8>*)calloc(1, sizeof(Dec<8>));
    sb::dec_state_init(&h->st, mdi, framesize_ms, joint_hb, arith);
    return h;
}
// same calling convention as AGR_Sate_Decoder_Decode (payload pre-trimmed by the caller); *flags = the packet's flags
int act_dec_decode(void* p, int samplerate, short* pcm, const unsigned char* bits, int cap, const short* nb, int lostflag, unsigned char* flags) {
    return samplerate == 32000 ? decode<16>(p, pcm, bits, cap, nb, lostflag, flags) : decode<8>(p, pcm, bits, cap, nb, lostflag, flags);
}
void act_dec_destroy(void* p) { free(p); }
}
