// solo_b200 -- send queue of descriptions (include/solo_b200.h, solo_b200_tx_*) and the downlink contributor lists
// (solo_b200_mix_contributors_*).  The per-row and per-member rules, written once for the kernels (solo_b200.cu) and the
// host model (tests/hostsim/server.cpp).
//   row     : an encoded row {bits, nbytes[2]} is DTX (nbytes[0] <= 0), bad (what solo_b200_split_packet refuses, or
//             nbytes[0] > cap) or sent: description 1 = bits[0, n0 - n1), description 2 = bits[n0 - n1, n0); a description
//             of 0 bytes is not emitted.  The two descriptions are the row's first n0 bytes in order, so a sent row's
//             datagrams are those bytes copied verbatim.
//   pack    : three passes -- sizes (thread per stream: datagrams and bytes, a block-wide exclusive scan of both), scan (the
//             block totals, one block), pack (warp per stream: the datagram entries, the index and counters, the bytes).
//   contrib : member i of room r lists the entries j of talkers[r][0..k) with 0 <= j < n and j != i, in order, with
//             level[j] & 0x7f beside each, padded with -1 / 127.
#pragma once
#include "sb_common.cuh"

namespace sb {

// the four per-stream counters, in the order solo_b200_tx_stats reports them
enum { TX_SENT = 0, TX_OCTETS, TX_DTX, TX_BAD, TX_NCOUNT };
#define SB_TX_BLOCK 256     // streams per block of the sizes pass, and so per block total of the scan
#define SB_TX_LVL_NONE 127  // csrc_level of a padding entry (RFC 6464's digital silence)

// The row's counter (TX_SENT, TX_DTX or TX_BAD) and, when sent, its description lengths l1 >= 0 and l2 >= 4
SB_HD int tx_row(int n0, int n1, int cap, int* l1, int* l2) {
    *l1 = *l2 = 0;
    if (n0 <= 0) return TX_DTX;
    if (n1 < 4 || n1 > n0 || n0 > cap) return TX_BAD;
    *l1 = n0 - n1;
    *l2 = n1;
    return TX_SENT;
}
// datagrams of a row with description lengths l1, l2: one per non-empty description
SB_HD int tx_datagrams(int l1, int l2) { return (l1 > 0) + (l2 > 0); }
// what the scan carries per stream: bytes in the high word, datagrams in the low word (a block's datagrams, at most
// 2 * SB_TX_BLOCK, and a call's, at most 2 * N, never carry into the high word)
SB_HD u64 tx_scan_word(int l1, int l2) { return ((u64)(u32)(l1 + l2) << 32) | (u32)tx_datagrams(l1, l2); }
SB_HD i32 tx_word_datagrams(u64 w) { return (i32)(u32)w; }
SB_HD i64 tx_word_bytes(u64 w) { return (i64)(w >> 32); }

// per-stream state after row s's pack: the index advances for every row, the row's counter once (octets by the payload)
SB_HD void tx_count(u32* cnt, int cls, int l1, int l2) {
    cnt[cls]++;
    if (cls == TX_SENT) cnt[TX_OCTETS] += (u32)(l1 + l2);
}

// Contributor list of member i of a room with talkers tk[0..k): writes csrc[0..k) and lvl[0..k)
SB_HD void tx_contributors(i32 i, const i32* tk, int k, const u8* level, int n, i32* csrc, u8* lvl) {
    int c = 0;
    for (int t = 0; t < k; t++) {
        const i32 j = tk[t];
        if ((u32)j >= (u32)n || j == i) continue;
        csrc[c] = j;
        lvl[c++] = (u8)(level[j] & 0x7f);
    }
    for (; c < k; c++) { csrc[c] = -1; lvl[c] = SB_TX_LVL_NONE; }
}

// The room of member position m: the last r in [0, R) with room_start[r] <= m, by binary search (R >= 1).  Only
// room_start[0..R) is read, so contents that are not monotone still give an r in range.
SB_HD int tx_room_of(const i32* room_start, int R, i32 m) {
    int lo = 0, hi = R;                         // room_start[lo] <= m is assumed; the answer is in [lo, hi)
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (room_start[mid] <= m) lo = mid; else hi = mid;
    }
    return lo;
}

}  // namespace sb
