// Robustness fuzzer of the decoder arithmetic (host build of solo_b200/csrc, test infrastructure only), built with
// -fsanitize=address,undefined so that an out-of-bounds table or buffer access on malformed input shows up here instead of
// as a faulting CUDA kernel that takes the whole batch down.
//   fuzz_dec <iterations> <seed>            16 kHz streams, packets from the host encoder over six signal classes
//   fuzz_dec <iterations> <seed> corpus32   32 kHz streams, packets from corpus32: records of the reference's .bit format
//                                           (int16 total, int16 len(MD2) + 8, payload), as there is no 32 kHz encoder here
// Every mode of the rate decodes `iterations` packets, each possibly bit-flipped, random, truncated or mislabelled, in a row
// that may be shorter than its declared total, under an arbitrary lost flag; it prints how many it decoded and rejected.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

#include "../../solo_b200/csrc/sb_dec.cuh"
#include "../../solo_b200/csrc/sb_enc.cuh"

static unsigned long long rs = 88172645463325252ull;
static unsigned rnd() { rs ^= rs << 13; rs ^= rs >> 7; rs ^= rs << 17; return (unsigned)(rs >> 11); }

struct Mode { const char* name; int khz, fs_ms, joint, mdi, arith, enc_rate; };
static const Mode MODES[] = {
    {"16k flp 40ms", 8, 40, 0, 0, sb::DEC_FLP, 13600},
    {"16k flp 20ms", 8, 20, 0, 1, sb::DEC_FLP, 17600},
    {"16k flp joint", 8, 40, 1, 0, sb::DEC_FLP, 21600},
    {"16k fix 40ms", 8, 40, 0, 0, sb::DEC_FIX, 13600},     // the fixed-point decoder has no 20 ms mode
    {"16k fix joint", 8, 40, 1, 1, sb::DEC_FIX, 19600},
    {"32k flp 40ms", 16, 40, 0, 0, sb::DEC_FLP, 0},
    {"32k flp 20ms", 16, 20, 0, 1, sb::DEC_FLP, 0},
    {"32k flp joint", 16, 40, 1, 0, sb::DEC_FLP, 0},
    {"32k fix 40ms", 16, 40, 0, 1, sb::DEC_FIX, 0},
    {"32k fix joint", 16, 40, 1, 0, sb::DEC_FIX, 0},
};
struct Packet { std::vector<unsigned char> b; short n0, n1; };

// one packet of the host encoder into row; sig cycles through tonal + noise, full-scale noise, rails, silence, impulses, DC steps
static void encode_one(sb::EncState* est, sb::EncPacketWork* ew, int spp, int it, double& ph, unsigned char* row, short* nb) {
    short pcm[640];
    const int sig = (it / 50) % 6;
    for (int i = 0; i < spp; i++) {
        ph += 0.05 + 0.04 * sin(it * 0.01);
        if (sig == 0) pcm[i] = (short)(6000 * sin(ph) + (int)(rnd() % 2000) - 1000);
        else if (sig == 1) pcm[i] = (short)rnd();
        else if (sig == 2) pcm[i] = (rnd() & 64) ? 32767 : -32768;
        else if (sig == 3) pcm[i] = 0;
        else if (sig == 4) pcm[i] = (rnd() % 97 == 0) ? (short)((rnd() & 1) ? 32767 : -32768) : 0;
        else pcm[i] = (short)(((it >> 2) & 1) ? 30000 : -30000);
    }
    sb::enc_packet(est, ew, pcm, row, 1024, nb);
}

template <int KHZ> static void run(const Mode& m, int iters, const std::vector<Packet>& corpus) {
    auto* dst = (sb::DecStateT<KHZ>*)calloc(1, sizeof(sb::DecStateT<KHZ>));
    auto* dw = (sb::DecPacketWorkT<KHZ>*)calloc(1, sizeof(sb::DecPacketWorkT<KHZ>));
    auto* stale = (sb::DecStale*)calloc(1, sizeof(sb::DecStale));
    auto* est = (sb::EncState*)calloc(1, sizeof(sb::EncState));
    auto* ew = (sb::EncPacketWork*)calloc(1, sizeof(sb::EncPacketWork));
    sb::dec_state_init(dst, m.mdi, m.fs_ms, m.joint, m.arith);
    if (m.enc_rate) sb::enc_state_init(est, m.enc_rate, 0, m.mdi, m.fs_ms, m.joint);
    double ph = 0;
    long errs = 0, oks = 0;
    for (int it = 0; it < iters; it++) {
        std::vector<unsigned char> row(1100, 0);        // exact-size heap buffers so that ASan sees overruns
        int n0, n1;
        if (m.enc_rate) {
            short nb[2] = {0, 0};
            encode_one(est, ew, 16 * m.fs_ms, it, ph, row.data(), nb);
            n0 = nb[0], n1 = nb[1];
        } else {
            const Packet& p = corpus[rnd() % corpus.size()];
            for (size_t i = 0; i < p.b.size(); i++) row[i] = p.b[i];
            n0 = p.n0, n1 = p.n1;
        }
        int kind = rnd() % 8, flag = 1 + rnd() % 4;
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
        std::vector<short> out(80 * KHZ);               // one 40 ms packet of PCM
        const int r = sb::dec_packet(dst, dw, out.data(), arg.data(), capx, nbb, flag, (rnd() & 1) ? stale : nullptr);
        (r < 0 ? errs : oks)++;
    }
    free(dst); free(dw); free(stale); free(est); free(ew);
    printf("%s: %ld decoded, %ld rejected\n", m.name, oks, errs);
}

int main(int argc, char** argv) {
    if (argc < 3) { fprintf(stderr, "usage: fuzz_dec iterations seed [corpus32]\n"); return 2; }
    const int iters = atoi(argv[1]);
    rs ^= (unsigned long long)atoll(argv[2]) * 0x9E3779B97F4A7C15ull;
    std::vector<Packet> corpus;
    if (argc > 3) {
        FILE* f = fopen(argv[3], "rb");
        if (!f) { fprintf(stderr, "fuzz_dec: cannot open %s\n", argv[3]); return 2; }
        short h[2];
        while (fread(h, 2, 2, f) == 2 && h[0] <= 1024) {
            Packet p{std::vector<unsigned char>(h[0] > 0 ? h[0] : 0), h[0], h[1]};
            if (!p.b.empty() && fread(p.b.data(), 1, p.b.size(), f) != p.b.size()) break;
            corpus.push_back(p);
        }
        fclose(f);
        if (corpus.empty()) { fprintf(stderr, "fuzz_dec: empty corpus\n"); return 2; }
    }
    for (const Mode& m : MODES) {
        if ((m.khz == 16) != !corpus.empty()) continue;
        if (m.khz == 16) run<16>(m, iters, corpus);
        else run<8>(m, iters, corpus);
    }
    printf("fuzz_dec: no memory errors\n");
    return 0;
}
