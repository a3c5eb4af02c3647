// solo_b200 -- per-room mix-minus of the loudest talkers (include/solo_b200.h, solo_b200_mix_*).  Written once for the mix
// kernels (solo_b200.cu) and the host model (tests/hostsim/server.cpp).
//   selection : a room's talkers are its up-to-k eligible members ((flags & 3) != 0, RFC 6464's V bit) with the smallest
//               (level, stream index) -- lower level is louder, ties go to the lower index
//   mixing    : out[i][t] = clamp(sum over talkers j != i of in[j][t], -32768, 32767), summed in int32 (k <= 8 rows of
//               int16 cannot overflow it, so the order of the sum does not matter)
#pragma once
#include "sb_common.cuh"

namespace sb {

#define SB_MIX_KMAX 8
#define SB_MIX_NONE (~(u64)0)   // an empty slot of a top-k list: after every real key

SB_HD bool mix_eligible(u8 flags) { return (flags & 3) != 0; }
// selection key of stream j: the talker with the smaller key wins; keys of distinct streams are distinct
SB_HD u64 mix_key(u8 level, i32 j) { return ((u64)level << 32) | (u32)j; }
SB_HD i32 mix_key_stream(u64 key) { return key == SB_MIX_NONE ? -1 : (i32)(u32)key; }

// L[0..8) ascending: insert x, dropping the largest (branch-free, fixed indices, so L stays in registers)
SB_HD void mix_topk_insert(u64 L[SB_MIX_KMAX], u64 x) {
#pragma unroll
    for (int i = SB_MIX_KMAX - 1; i > 0; i--) L[i] = x < L[i - 1] ? L[i - 1] : (x < L[i] ? x : L[i]);
    L[0] = x < L[0] ? x : L[0];
}
// the merge of the lanes' lists takes the smallest head of all lanes each round: a lane whose head it was drops it
SB_HD void mix_topk_pop(u64 L[SB_MIX_KMAX], u64 taken) {
    if (L[0] != taken) return;
#pragma unroll
    for (int i = 0; i < SB_MIX_KMAX - 1; i++) L[i] = L[i + 1];
    L[SB_MIX_KMAX - 1] = SB_MIX_NONE;
}

// does listener i hear talker j (a talkers[] entry, -1 = none)
SB_HD bool mix_hears(i32 i, i32 j) { return j >= 0 && j != i; }
// one output sample from its int32 sum
SB_HD i16 mix_out(i32 sum) { return (i16)sat16(sum); }

// The room of member position m: the last r in [0, R) with room_start[r] <= m, by a 33-ary search that a warp runs with one
// probe per lane (3 rounds for 16 384 rooms).  A round over the candidates [lo, lo + span) probes p = lo + l * step for
// l = 0..31 (p < lo + span); the last probe with room_start[p] <= m keeps its step.  Only room_start[0..R) is read, so
// contents that are not monotone still give an r in range.
SB_HD int mix_search_step(int span) { return (span + 31) >> 5; }
SB_HD void mix_search_narrow(int* lo, int* span, int step, u32 le_mask) {
    const int l = le_mask ? 31 - clz32((i32)le_mask) : 0, end = *lo + *span;
    *lo += l * step;
    *span = imin(step, end - *lo);
}
// the same search, probes in turn (the host model's form of the kernel's ballot)
SB_HD int mix_room_of(const i32* room_start, int R, i32 m) {
    int lo = 0, span = R;
    while (span > 1) {
        const int step = mix_search_step(span);
        u32 le = 0;
        for (int l = 0; l < 32; l++) {
            const int p = lo + l * step;
            if (p < lo + span && room_start[p] <= m) le |= 1u << l;
        }
        mix_search_narrow(&lo, &span, step, le);
    }
    return lo;
}

}  // namespace sb
