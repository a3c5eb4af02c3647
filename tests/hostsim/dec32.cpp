// Host build of the decoder source (solo_b200/csrc/sb_dec.cuh compiled by g++) for 32 kHz streams: the DecState32
// instantiation (16 kHz SILK core), in either arithmetic (sb::DEC_FLP / sb::DEC_FIX), beside the 16 kHz one (DecState) for
// tests that feed one rate's packets to the other.  TEST INFRASTRUCTURE ONLY; compiled by tests/test_dec32.py, never linked
// into libsolo_b200.so.
//   shared library : g++ -O2 -ffp-contract=off -std=c++17 -shared -fPIC -w dec32.cpp -o libdec32.so
//   fuzzer         : g++ -O1 -g -std=c++17 -fsanitize=address,undefined -fno-sanitize-recover=all -w -DSB_DEC32_FUZZ dec32.cpp
//                    -o fuzz_dec32 && ./fuzz_dec32 corpus32 [iterations] [seed]
// The fuzzer feeds the 32 kHz decoders (40 ms, 20 ms and joint-mode-1 packets in float arithmetic, 40 ms and joint mode 1
// in fixed point) bit-flipped, random, truncated and mislabelled versions of the packets in `corpus32` (records of the
// reference's .bit format: int16 total, int16 len(MD2)+8, payload; the library has no 32 kHz encoder to make them), rows
// shorter than the declared total and arbitrary lost flags, so that an out-of-bounds table or buffer access on malformed
// input shows up here rather than as a faulting kernel.
#include <stdlib.h>

#include "../../solo_b200/csrc/sb_dec.cuh"

template <int KHZ> struct Dec { sb::DecStateT<KHZ> st; sb::DecPacketWorkT<KHZ> w; sb::DecStale stale; };
template <int KHZ> static void* create(int mdi, int framesize_ms, int joint_hb, int arith) {
    Dec<KHZ>* h = (Dec<KHZ>*)calloc(1, sizeof(Dec<KHZ>));
    sb::dec_state_init(&h->st, mdi, framesize_ms, joint_hb, arith);
    return h;
}
template <int KHZ> static int decode(void* p, short* pcm, const unsigned char* bits, int cap, const short* nb, int lostflag) {
    Dec<KHZ>* h = (Dec<KHZ>*)p;
    return sb::dec_packet(&h->st, &h->w, pcm, bits, cap, nb, lostflag, &h->stale);
}

extern "C" {
// samplerate 32000 (16 kHz core) or 16000 (8 kHz core); decode calls take the same samplerate as create
void* d32_create(int mdi, int framesize_ms, int joint_hb, int arith, int samplerate) {
    return samplerate == 32000 ? create<16>(mdi, framesize_ms, joint_hb, arith) : create<8>(mdi, framesize_ms, joint_hb, arith);
}
// same calling convention as AGR_Sate_Decoder_Decode (payload pre-trimmed by the caller); nb is not modified
int d32_decode(void* p, int samplerate, short* pcm, const unsigned char* bits, int cap, const short* nb, int lostflag) {
    return samplerate == 32000 ? decode<16>(p, pcm, bits, cap, nb, lostflag) : decode<8>(p, pcm, bits, cap, nb, lostflag);
}
void d32_destroy(void* p) { free(p); }
}

#ifdef SB_DEC32_FUZZ
#include <stdio.h>
#include <vector>

static unsigned long long rs = 88172645463325252ull;
static unsigned rnd() { rs ^= rs << 13; rs ^= rs >> 7; rs ^= rs << 17; return (unsigned)(rs >> 11); }

int main(int argc, char** argv) {
    if (argc < 2) { fprintf(stderr, "usage: fuzz_dec32 corpus32 [iterations] [seed]\n"); return 2; }
    const int iters = argc > 2 ? atoi(argv[2]) : 2000;
    if (argc > 3) rs ^= (unsigned long long)atoll(argv[3]) * 0x9E3779B97F4A7C15ull;
    std::vector<std::vector<unsigned char>> corpus;
    std::vector<std::pair<short, short>> lens;
    FILE* f = fopen(argv[1], "rb");
    if (!f) { fprintf(stderr, "fuzz_dec32: cannot open %s\n", argv[1]); return 2; }
    short h[2];
    while (fread(h, 2, 2, f) == 2 && h[0] <= 1024) {
        std::vector<unsigned char> pk(h[0] > 0 ? h[0] : 0);
        if (!pk.empty() && fread(pk.data(), 1, pk.size(), f) != pk.size()) break;
        corpus.push_back(pk);
        lens.push_back({h[0], h[1]});
    }
    fclose(f);
    if (corpus.empty()) { fprintf(stderr, "fuzz_dec32: empty corpus\n"); return 2; }
    auto* dst = (sb::DecState32*)calloc(1, sizeof(sb::DecState32));
    auto* dw = (sb::DecPacketWork32*)calloc(1, sizeof(sb::DecPacketWork32));
    auto* stale = (sb::DecStale*)calloc(1, sizeof(sb::DecStale));
    long errs = 0, oks = 0;
    for (int mode = 0; mode < 5; mode++) {      // 40 ms, 20 ms, joint mode 1 (float); 40 ms, joint mode 1 (fixed point)
        const int fs_ms = mode == 1 ? 20 : 40, joint = mode == 2 || mode == 4, arith = mode >= 3 ? sb::DEC_FIX : sb::DEC_FLP;
        sb::dec_state_init(dst, mode & 1, fs_ms, joint, arith);
        for (int it = 0; it < iters; it++) {
            const size_t k = rnd() % corpus.size();
            std::vector<unsigned char> row(1100, 0);        // exact-size heap buffers so that ASan sees overruns
            for (size_t i = 0; i < corpus[k].size(); i++) row[i] = corpus[k][i];
            int n0 = lens[k].first, n1 = lens[k].second, kind = rnd() % 8, flag = 1 + rnd() % 4;
            if (n0 <= 0) { n0 = 16; n1 = 8; flag = 1; }
            if (kind == 1) for (int j = 0; j < 1 + (int)(rnd() % 4); j++) row[rnd() % n0] ^= (unsigned char)(1u << (rnd() % 8));   // bit flips
            if (kind == 2) for (int i = 0; i < n0; i++) row[i] = (unsigned char)rnd();                                        // garbage
            if (kind == 3) { n0 = 1 + rnd() % 1024; n1 = rnd() % (n0 + 1); }                                                  // lying lengths
            if (kind == 4) { n0 = 1 + rnd() % 12; n1 = rnd() % 16; }                                                         // tiny / inconsistent
            if (kind == 5) flag = (int)(rnd() % 9) - 2;                                                                       // invalid flags
            int capx = 1024;
            if (kind == 6) { capx = 4 + rnd() % 124; n0 = capx + 1 + rnd() % 8; n1 = rnd() % (n0 + 1); }                      // declared total beyond a short row
            if (kind == 7) { capx = 4 + rnd() % 60; n0 = sb::imin(capx, n0); n1 = rnd() % (n0 + 1); }                        // short, consistent
            short nbb[2] = {(short)n0, (short)n1};
            if (flag == 2 && kind < 3) { nbb[0] = (short)(n0 - n1); nbb[1] = 0; }
            if (flag == 3 && kind < 3) { for (int i = 0; i < n1; i++) row[i] = row[n0 - n1 + i]; nbb[0] = (short)n1; nbb[1] = 0; }
            std::vector<unsigned char> arg(row.begin(), row.begin() + capx);
            short out[1280];
            const int r = sb::dec_packet(dst, dw, out, arg.data(), capx, nbb, flag, (rnd() & 1) ? stale : nullptr);
            (r < 0 ? errs : oks)++;
        }
    }
    free(dst); free(dw); free(stale);
    printf("fuzz_dec32: %ld decoded, %ld rejected, no memory errors\n", oks, errs);
    return 0;
}
#endif
