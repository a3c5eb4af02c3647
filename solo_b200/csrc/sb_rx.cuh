// solo_b200 -- receive queue of descriptions (include/solo_b200.h, solo_b200_rx_*).  The per-arrival and per-slot rules,
// written once for the queue's kernels (solo_b200.cu) and the host model (tests/hostsim/server.cpp), and
// the per-row merge rule that solo_b200_merge_packets and the pull kernel share.
//   current : packet index p is current for a stream whose last played index is `last` when (p - last) mod 2^32 lies in
//             [1, 2^31); "newer" is a larger distance p - last.  A slot keeps the newest current index among its held one
//             and the call's valid arrivals; per description of it a held one stays, otherwise the first arrival in array
//             order is stored.
//   insert  : three passes over the arrivals -- elect (per (slot, desc) a 64-bit atomic max of distance << 32 | ~position,
//             so the newest index and, for it, the first arrival win; per slot an atomic min of position picks the one
//             arrival that commits the slot), classify (count every arrival, copy the stored ones), commit (the slot's new
//             index and lengths, the held descriptions it discards, and the election words back to empty).
//   timing  : (solo_b200_rx_enable_timing, solo_b200_rx_insert_timed_*) per stream transit, RFC 3550 A.8 jitter, the
//             extended highest index, the count of valid arrivals and a playout-margin histogram, from each arrival's
//             receive time.  Jitter and highest follow the stream's valid arrivals in array order (rx_timing_step); the
//             margin bin of an arrival depends only on it and `last` (rx_margin_bin).
#pragma once
#include "sb_common.cuh"

namespace sb {

// the eight per-stream counters, in the order solo_b200_rx_stats reports them
enum { RX_STORED = 0, RX_DUPLICATE, RX_LATE, RX_DROPPED, RX_MALFORMED, RX_PLAYED_BOTH, RX_PLAYED_ONE, RX_PLAYED_NONE, RX_NCOUNT };
#define RX_NO_REP 0xFFFFFFFFu   // the per-slot commit word when no arrival of the call is for the slot

SB_HD bool rx_current(u32 p, u32 last) { return p - last - 1u < 0x7FFFFFFFu; }
SB_HD u32 rx_slot(u32 p, int depth) { return p & (u32)(depth - 1); }

// desc in {1, 2}, len in [1, desc_cap], bytes inside payload[0, payload_bytes)
SB_HD bool rx_malformed(int desc, i32 off, i32 len, int desc_cap, i64 payload_bytes) {
    return (desc != 1 && desc != 2) || len < 1 || len > desc_cap || off < 0 || (i64)off + len > payload_bytes;
}

// slot s * depth + (p mod depth) of an arrival for stream s, index p, when it is valid and current (and its distance
// p - last[s]), else -1
SB_HD long long rx_arrival_slot(int n, int depth, int desc_cap, const u32* last, i32 s, int desc, i32 off, i32 len, u32 p,
                                i64 payload_bytes, u32* dist) {
    if ((u32)s >= (u32)n || rx_malformed(desc, off, len, desc_cap, payload_bytes) || !rx_current(p, last[s])) return -1;
    *dist = p - last[s];
    return (long long)s * depth + rx_slot(p, depth);
}

// election word of arrival `pos` at distance `dist` (0 = no candidate): the larger word is the newer index, then the
// earlier arrival
SB_HD u64 rx_key(u32 dist, i32 pos) { return ((u64)dist << 32) | (u32)~(u32)pos; }
SB_HD u32 rx_key_dist(u64 key) { return (u32)(key >> 32); }
SB_HD i32 rx_key_pos(u64 key) { return (i32)~(u32)key; }

// distance of the slot's held index when it holds a description of a current index, else 0 (it does not compete)
SB_HD u32 rx_held_dist(u32 idx, const u16* len, u32 last) {
    return (len[0] | len[1]) && rx_current(idx, last) ? idx - last : 0u;
}
// distance of the index the slot keeps: the newest of the held one and the two descriptions' elected arrivals
SB_HD u32 rx_winner(const u64* e, u32 held_dist) {
    const u32 a = rx_key_dist(e[0]), b = rx_key_dist(e[1]);
    const u32 m = a > b ? a : b;
    return m > held_dist ? m : held_dist;
}

// outcome of a valid, current arrival at distance `dist`, position `pos`, description d (0 or 1) of its slot
SB_HD int rx_classify(u32 dist, int d, i32 pos, const u64* e, u32 idx, const u16* len, u32 last) {
    const u32 hd = rx_held_dist(idx, len, last), w = rx_winner(e, hd);
    if (dist != w) return RX_DROPPED;
    if (w == hd && (d ? len[1] : len[0])) return RX_DUPLICATE;       // selects, not an index: the arrays stay in registers
    return rx_key_pos(d ? e[1] : e[0]) == pos ? RX_STORED : RX_DUPLICATE;
}

// the slot after a call with at least one valid, current arrival for it: updates idx / len from the election words e and
// the arrivals' lengths alen; returns the number of held descriptions it discards (counted as dropped)
SB_HD int rx_commit(u32 last, u32* idx, u16* len, const u64* e, const i32* alen) {
    const u32 hd = rx_held_dist(*idx, len, last), w = rx_winner(e, hd);
    int discarded = 0;
    if (w != hd) {
        discarded = (len[0] != 0) + (len[1] != 0);
        len[0] = len[1] = 0;
        *idx = last + w;
    }
    for (int d = 0; d < 2; d++)
        if (rx_key_dist(e[d]) == w && !len[d]) len[d] = (u16)alen[rx_key_pos(e[d])];
    return discarded;
}

// The decoder's row from the descriptions of one packet, n1 / n2 bytes (0 = that one did not arrive): description 1, then
// description 2.  Sets nbytes[2] and the lostflag (4 both, 2 only description 1, 3 only description 2, 1 neither) and
// returns the row's length; with neither the row is 16 zero bytes (the decoder conceals, but wants nBytes[0] > 0,
// AGR_BWE_SDK_API.c:268-270, and does not read them).
SB_HD int rx_merge(int n1, int n2, i16* nbytes, i32* lostflag) {
    if (n1 > 0 && n2 > 0) { nbytes[0] = (i16)(n1 + n2); nbytes[1] = (i16)n2; *lostflag = 4; return n1 + n2; }
    if (n1 > 0) { nbytes[0] = (i16)n1; nbytes[1] = 0; *lostflag = 2; return n1; }
    if (n2 > 0) { nbytes[0] = (i16)n2; nbytes[1] = 0; *lostflag = 3; return n2; }
    nbytes[0] = 16; nbytes[1] = 8; *lostflag = 1;
    return 16;
}

// pull of index t from its slot: the lengths of the descriptions of t the slot holds
SB_HD void rx_play(u32 t, u32 idx, const u16* len, int* n1, int* n2) {
    *n1 = idx == t ? len[0] : 0;
    *n2 = idx == t ? len[1] : 0;
}
SB_HD int rx_played_counter(int n1, int n2) {
    return n1 > 0 && n2 > 0 ? RX_PLAYED_BOTH : (n1 > 0 || n2 > 0 ? RX_PLAYED_ONE : RX_PLAYED_NONE);
}
// after last = t: a slot that holds an index that is no longer current is emptied; returns the descriptions it discards
// that were not the ones just played (counted as dropped)
SB_HD int rx_after_play(u32 t, u32 idx, u16* len) {
    if (!(len[0] | len[1]) || rx_current(idx, t)) return 0;
    const int stale = idx != t ? (len[0] != 0) + (len[1] != 0) : 0;
    len[0] = len[1] = 0;
    return stale;
}

// ---- timing ------------------------------------------------------------------------------------------------------------
#define RX_MARGIN_BINS 8

// an arrival the timing counts: its stream is in range and it is not malformed (late and duplicate arrivals count, as
// RFC 3550 updates the jitter for every packet received)
SB_HD bool rx_timed(int n, int desc_cap, i32 s, int desc, i32 off, i32 len, i64 payload_bytes) {
    return (u32)s < (u32)n && !rx_malformed(desc, off, len, desc_cap, payload_bytes);
}

// margin bin of a valid arrival of index p for a stream whose last played index is `last`: min(p - last - 1, 7) when p is
// current (bin 0 plays at the next pull), -1 when it is late
SB_HD int rx_margin_bin(u32 p, u32 last) {
    if (!rx_current(p, last)) return -1;
    const u32 m = p - last - 1u;
    return m < RX_MARGIN_BINS - 1 ? (int)m : RX_MARGIN_BINS - 1;
}

// One valid arrival of index p at receive time `arrival` (RTP timestamp units, mod 2^32) into its stream's timing state.
// Transit t = arrival - p * ts_per_index.  From the second valid arrival since the reset on, RFC 3550 A.8:
// d = |(int32)(t - transit)| (2^31 for INT_MIN), jitter += d - ((jitter + 8) >> 4), all in uint32; and highest
// (cycles << 32 | index) moves to p when p is ahead of its low word by [1, 2^31), one cycle up when p wrapped below it.
// The first valid arrival sets highest = p.
SB_HD void rx_timing_step(u32 p, u32 arrival, u32 ts_per_index, u32* transit, u32* jitter, u64* highest, u32* received) {
    const u32 t = arrival - p * ts_per_index;
    if (*received) {
        const u32 diff = t - *transit;
        const u32 d = (diff & 0x80000000u) ? 0u - diff : diff;
        *jitter += d - ((*jitter + 8u) >> 4);
        const u32 lo = (u32)*highest;
        if (p - lo - 1u < 0x7FFFFFFFu) *highest = (((*highest >> 32) + (p < lo ? 1u : 0u)) << 32) | p;
    } else {
        *highest = p;
    }
    *transit = t;
    (*received)++;
}

}  // namespace sb
