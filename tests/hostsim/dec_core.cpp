// Host build of the core-output decoder of 32 kHz streams: the per-stream body of sb_decode_kernel<16, true>
// (dec_packet<16, true> of solo_b200/csrc/sb_dec.cuh) compiled by g++.
// TEST INFRASTRUCTURE ONLY: lets the CPU-only container check the core rows bit for bit against the low band of the
// compiled reference (oracle/lowband.mk).  Never linked into libsolo_b200.so.
#include <stdlib.h>
#include "../../solo_b200/csrc/sb_dec.cuh"

extern "C" {
// one 32 kHz stream decoded to its 16 kHz core
struct HsDecCore { sb::DecState32 st; sb::DecPacketWork32 w; sb::DecStale stale; };
// arith: sb::DEC_FLP or sb::DEC_FIX
void* hs_dec_core_create(int mdi, int framesize_ms, int joint_hb, int arith) {
    HsDecCore* h = (HsDecCore*)calloc(1, sizeof(HsDecCore));
    sb::dec_state_init(&h->st, mdi, framesize_ms, joint_hb, arith, 1);
    return h;
}
// same calling convention as AGR_Sate_Decoder_Decode (payload pre-trimmed by the caller), 16 * framesize_ms samples into
// pcm; nb is not modified.  flags (may be NULL): the packet's activity flags, 0 for a rejected packet
int hs_dec_core_decode(void* p, short* pcm, const unsigned char* bits, int cap, const short* nb, int lostflag, unsigned char* flags) {
    HsDecCore* h = (HsDecCore*)p;
    const int r = sb::dec_packet(&h->st, &h->w, pcm, bits, cap, nb, lostflag, &h->stale);   // core_only: dec_packet<16, true>
    if (flags) *flags = r < 0 ? 0 : h->w.act;
    return r;
}
void hs_dec_core_destroy(void* p) { free(p); }
}
