// Host build of the conference mixer (solo_b200/csrc/sb_mix.cuh compiled by g++): the two mix kernels' arithmetic in their
// order -- 32 lanes' top-8 lists over strided slices of each room, merged one smallest head per round, and every member's
// row found by the kernel's room search and summed from the talkers it hears.  TEST INFRASTRUCTURE ONLY; compiled by
// tests/test_mix.py, never linked into libsolo_b200.so.  Expects valid input (solo_b200_mix_host's checks).
//   g++ -O2 -std=c++17 -shared -fPIC -w mix.cpp -o libmix.so
#include "../../solo_b200/csrc/sb_mix.cuh"

extern "C" {
void mix_model(const short* in, short* out, int spp, int n, const unsigned char* level, const unsigned char* flags,
               const int* room_start, const int* members, int R, int k, int* talkers) {
    using namespace sb;
    for (int r = 0; r < R; r++) {               // sb_mix_select_kernel: lane l takes members lo + l, lo + l + 32, ...
        u64 L[32][SB_MIX_KMAX];
        for (int l = 0; l < 32; l++)
            for (int i = 0; i < SB_MIX_KMAX; i++) L[l][i] = SB_MIX_NONE;
        for (int m = room_start[r]; m < room_start[r + 1]; m++) {
            const int j = members[m];
            if (mix_eligible(flags[j])) mix_topk_insert(L[(m - room_start[r]) & 31], mix_key(level[j], j));
        }
        for (int t = 0; t < k; t++) {
            u64 best = SB_MIX_NONE;
            for (int l = 0; l < 32; l++) best = L[l][0] < best ? L[l][0] : best;
            for (int l = 0; l < 32; l++) mix_topk_pop(L[l], best);
            talkers[r * k + t] = mix_key_stream(best);
        }
    }
    for (int m = 0; m < (R ? room_start[R] : 0); m++) {   // sb_mix_kernel: one member row
        const int i = members[m], r = mix_room_of(room_start, R, m);
        for (int t = 0; t < spp; t++) {
            i32 sum = 0;
            for (int q = 0; q < k; q++) {
                const int j = talkers[r * k + q];
                if (mix_hears(i, j)) sum += in[(long)j * spp + t];
            }
            out[(long)i * spp + t] = mix_out(sum);
        }
    }
}
}
