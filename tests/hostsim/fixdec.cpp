// Host build of the decoder source (solo_b200/csrc/sb_dec.cuh compiled by g++) with a chosen arithmetic per stream:
// sb::DEC_FLP (the reference's float build) or sb::DEC_FIX (its fixed-point build).  TEST INFRASTRUCTURE ONLY; compiled by
// tests/test_fix_decoder.py, never linked into libsolo_b200.so.
//   shared library : g++ -O2 -ffp-contract=off -std=c++17 -shared -fPIC -w fixdec.cpp -o libfixdec.so
//   fuzzer         : g++ -O1 -g -std=c++17 -fsanitize=address,undefined -fno-sanitize-recover=all -w -DSB_FIXDEC_FUZZ fixdec.cpp
//                    -o fuzz_fixdec && ./fuzz_fixdec [iterations] [seed]
// The fuzzer feeds fixed-point decoders (40 ms packets and joint mode 1, the configurations that mode supports)
// bit-flipped, random, truncated and mislabelled payloads, rows shorter than the declared total and arbitrary lost flags,
// so that an out-of-bounds table or buffer access on malformed input shows up here rather than as a faulting kernel.
#include <stdlib.h>

#include "../../solo_b200/csrc/sb_dec.cuh"

extern "C" {
struct FxDec { sb::DecState st; sb::DecPacketWork w; sb::DecStale stale; };
void* fx_dec_create(int mdi, int framesize_ms, int joint_hb, int arith) {
    FxDec* h = (FxDec*)calloc(1, sizeof(FxDec));
    sb::dec_state_init(&h->st, mdi, framesize_ms, joint_hb, arith);
    return h;
}
// same calling convention as AGR_Sate_Decoder_Decode (payload pre-trimmed by the caller); nb is not modified
int fx_dec_decode(void* p, short* pcm, const unsigned char* bits, int cap, const short* nb, int lostflag) {
    FxDec* h = (FxDec*)p;
    return sb::dec_packet(&h->st, &h->w, pcm, bits, cap, nb, lostflag, &h->stale);
}
void fx_dec_destroy(void* p) { free(p); }
}

#ifdef SB_FIXDEC_FUZZ
#include <math.h>
#include <stdio.h>
#include <vector>

#include "../../solo_b200/csrc/sb_enc.cuh"

static unsigned long long rs = 88172645463325252ull;
static unsigned rnd() { rs ^= rs << 13; rs ^= rs >> 7; rs ^= rs << 17; return (unsigned)(rs >> 11); }

int main(int argc, char** argv) {
    const int iters = argc > 1 ? atoi(argv[1]) : 20000;
    if (argc > 2) rs ^= (unsigned long long)atoll(argv[2]) * 0x9E3779B97F4A7C15ull;
    auto* est = (sb::EncState*)calloc(1, sizeof(sb::EncState));
    auto* ew = (sb::EncPacketWork*)calloc(1, sizeof(sb::EncPacketWork));
    auto* dst = (sb::DecState*)calloc(1, sizeof(sb::DecState));
    auto* dw = (sb::DecPacketWork*)calloc(1, sizeof(sb::DecPacketWork));
    auto* stale = (sb::DecStale*)calloc(1, sizeof(sb::DecStale));
    long errs = 0, oks = 0;
    for (int mode = 0; mode < 2; mode++) {          // 40 ms packets, joint mode 1
        const int joint = mode == 1, spp = 640;
        sb::enc_state_init(est, 13600 + 6000 * mode, 0, mode, 40, joint);
        sb::dec_state_init(dst, mode, 40, joint, sb::DEC_FIX);
        double ph = 0;
        for (int it = 0; it < iters; it++) {
            short pcm[640], nb[2] = {0, 0}, out[640];
            const int sig = (it / 50) % 6;     // tonal + noise, full-scale noise, rails, silence, impulses, DC steps
            for (int i = 0; i < spp; i++) {
                ph += 0.05 + 0.04 * sin(it * 0.01);
                if (sig == 0) pcm[i] = (short)(6000 * sin(ph) + (int)(rnd() % 2000) - 1000);
                else if (sig == 1) pcm[i] = (short)rnd();
                else if (sig == 2) pcm[i] = (rnd() & 64) ? 32767 : -32768;
                else if (sig == 3) pcm[i] = 0;
                else if (sig == 4) pcm[i] = (rnd() % 97 == 0) ? (short)((rnd() & 1) ? 32767 : -32768) : 0;
                else pcm[i] = (short)(((it >> 2) & 1) ? 30000 : -30000);
            }
            std::vector<unsigned char> row(1100, 0);        // exact-size heap buffers so that ASan sees overruns
            sb::enc_packet(est, ew, pcm, row.data(), 1024, nb);
            int kind = rnd() % 8, flag = 1 + rnd() % 4;
            int n0 = nb[0], n1 = nb[1];
            if (n0 <= 0) { n0 = 16; n1 = 8; flag = 1; }
            if (kind == 1) for (int k = 0; k < 1 + (int)(rnd() % 4); k++) row[rnd() % n0] ^= (unsigned char)(1u << (rnd() % 8));
            if (kind == 2) for (int i = 0; i < n0; i++) row[i] = (unsigned char)rnd();
            if (kind == 3) { n0 = 1 + rnd() % 1024; n1 = rnd() % (n0 + 1); }
            if (kind == 4) { n0 = 1 + rnd() % 12; n1 = rnd() % 16; }
            if (kind == 5) flag = (int)(rnd() % 9) - 2;
            int capx = 1024;
            if (kind == 6) { capx = 4 + rnd() % 124; n0 = capx + 1 + rnd() % 8; n1 = rnd() % (n0 + 1); }   // short rows
            if (kind == 7) { capx = 4 + rnd() % 60; n0 = sb::imin(capx, n0); n1 = rnd() % (n0 + 1); }        // short, consistent
            short nbb[2] = {(short)n0, (short)n1};
            if (flag == 2 && kind < 3) { nbb[0] = (short)(n0 - n1); nbb[1] = 0; }
            if (flag == 3 && kind < 3) { for (int i = 0; i < n1; i++) row[i] = row[n0 - n1 + i]; nbb[0] = (short)n1; nbb[1] = 0; }
            std::vector<unsigned char> arg(row.begin(), row.begin() + capx);
            int r = sb::dec_packet(dst, dw, out, arg.data(), capx, nbb, flag, (rnd() & 1) ? stale : nullptr);
            (r < 0 ? errs : oks)++;
        }
    }
    free(est); free(ew); free(dst); free(dw); free(stale);
    printf("fuzz_fixdec: %ld decoded, %ld rejected, no memory errors\n", oks, errs);
    return 0;
}
#endif
