// solo_b200 -- per-packet activity reports: the RFC 6464 audio level of a PCM row and the SILK voice-activity /
// concealment flags of the packet's frames.  Written once for the activity kernel (solo_b200.cu) and the host model.
//   level : clamp(round(10 * log10(n * 32768^2 / E)), 0, 127) of the row's energy E = sum(x^2) over its n samples, as
//           the number of thresholds T_n[k] (sb_level_tables.inc, tools/gen_level_tables.py) above E: exact integers,
//           127 for digital silence
//   flags : bit f = frame f's VAD flag; bit 2 + f (decoder) = frame f was concealed
#pragma once
#include "sb_common.cuh"
#include "sb_state.cuh"
#include "sb_tables.cuh"

namespace sb {
namespace tab {
#define SB_TAB(T, name, N, ...) static const T name##_h[N] = {__VA_ARGS__};
#include "sb_level_tables.inc"
#undef SB_TAB
#ifdef __CUDACC__
#define SB_TAB(T, name, N, ...) static __device__ const T name##_d[N] = {__VA_ARGS__};
#include "sb_level_tables.inc"
#undef SB_TAB
#endif
}  // namespace tab

// RFC 6464 level (0-127, -dBov) of a row of n = 320, 640 or 1280 samples whose sum of squares is E
SB_HD int rfc6464_level(i64 E, int n) {
    const i64* T = n == 320 ? SB_T(level_thr_320) : n == 640 ? SB_T(level_thr_640) : SB_T(level_thr_1280);
    int lo = 0, hi = 127;               // T is non-increasing: E < T[k] holds for k < level and fails from there on
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (E < T[mid]) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// the encoder's flags of the packet the last wave coded: each frame's coded VAD flag, none for a DTX-dropped packet
SB_HD int enc_activity_flags(const EncScratch* scr, int nf) {
    if (scr->dtx_drop) return 0;
    return (scr->vadFlag[0] & 1) | (nf > 1 ? (scr->vadFlag[1] & 1) << 1 : 0);
}

}  // namespace sb
