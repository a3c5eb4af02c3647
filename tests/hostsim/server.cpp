// Host build of the server-side kernels (solo_b200/csrc/sb_mix.cuh, sb_rx.cuh and sb_tx.cuh compiled by g++): the
// conference mixer, the receive queue with its timing, the send queue and the downlink contributor lists, each in its
// kernels' order.  TEST INFRASTRUCTURE ONLY; built into tests/_hostsim/libsb_hostsim.so by build_hostsim.py and driven by
// sim.py, never linked into libsolo_b200.so.  The state arrays have the device layout of solo_b200.cu's RxDev, RxTiming
// and TxDev.  Expects valid input where the host entry points check it (solo_b200_mix_host's checks).
#include <string.h>

#include <vector>

#include "../../solo_b200/csrc/sb_mix.cuh"
#include "../../solo_b200/csrc/sb_rx.cuh"
#include "../../solo_b200/csrc/sb_tx.cuh"

using namespace sb;

extern "C" {
// the two mix kernels' arithmetic in their order: 32 lanes' top-8 lists over strided slices of each room, merged one
// smallest head per round, and every member's row found by the kernel's room search and summed from the talkers it hears
void mix_model(const short* in, short* out, int spp, int n, const unsigned char* level, const unsigned char* flags,
               const int* room_start, const int* members, int R, int k, int* talkers) {
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

// the receive queue's insert kernels' three passes in their order over the arrivals (elect, classify and copy, commit),
// with the atomics as plain read-modify-writes
void rx_model_insert(int n, int depth, int desc_cap, const u32* last, u32* idx, u16* len, u64* elect, u32* rep, u32* cnt,
                     u64* bad, u8* store, const i32* stream, const u32* index, const u8* desc, const i32* off, const i32* alen,
                     int na, const u8* payload, i64 payload_bytes) {
    for (int a = 0; a < na; a++) {              // sb_rx_elect_kernel
        u32 dist;
        const long long sl = rx_arrival_slot(n, depth, desc_cap, last, stream[a], desc[a], off[a], alen[a], index[a], payload_bytes, &dist);
        if (sl < 0) continue;
        u64& e = elect[2 * sl + desc[a] - 1];
        const u64 k = rx_key(dist, a);
        if (k > e) e = k;
        if ((u32)a < rep[sl]) rep[sl] = (u32)a;
    }
    for (int a = 0; a < na; a++) {              // sb_rx_classify_kernel
        const i32 s = stream[a];
        if ((u32)s >= (u32)n) { (*bad)++; continue; }
        const int d = desc[a];
        int cls;
        long long sl = -1;
        if (rx_malformed(d, off[a], alen[a], desc_cap, payload_bytes)) cls = RX_MALFORMED;
        else if (!rx_current(index[a], last[s])) cls = RX_LATE;
        else {
            sl = (long long)s * depth + rx_slot(index[a], depth);
            cls = rx_classify(index[a] - last[s], d - 1, a, elect + 2 * sl, idx[sl], len + 2 * sl, last[s]);
        }
        cnt[(size_t)s * RX_NCOUNT + cls]++;
        if (cls == RX_STORED) memcpy(store + (size_t)(2 * sl + d - 1) * desc_cap, payload + off[a], (size_t)alen[a]);
    }
    for (int a = 0; a < na; a++) {              // sb_rx_commit_kernel
        u32 dist;
        const long long sl = rx_arrival_slot(n, depth, desc_cap, last, stream[a], desc[a], off[a], alen[a], index[a], payload_bytes, &dist);
        if (sl < 0 || rep[sl] != (u32)a) continue;
        cnt[(size_t)stream[a] * RX_NCOUNT + RX_DROPPED] += rx_commit(last[stream[a]], idx + sl, len + 2 * sl, elect + 2 * sl, alen);
        elect[2 * sl] = elect[2 * sl + 1] = 0;
        rep[sl] = RX_NO_REP;
    }
}

// sb_rx_pull_kernel for every stream (play = NULL: last + 1)
void rx_model_pull(int n, int depth, int desc_cap, u32* last, u32* idx, u16* len, u32* cnt, const u8* store, const u32* play,
                   u8* bits, int cap, i16* nbytes, i32* lostflag) {
    for (int s = 0; s < n; s++) {
        const u32 t = play ? play[s] : last[s] + 1u;
        const size_t sl = (size_t)s * depth + rx_slot(t, depth);
        int n1, n2;
        rx_play(t, idx[sl], len + 2 * sl, &n1, &n2);
        const int nrow = rx_merge(n1, n2, nbytes + 2 * s, lostflag + s);
        u8* row = bits + (size_t)s * cap;
        if (lostflag[s] == 1) memset(row, 0, (size_t)nrow);
        memcpy(row, store + 2 * sl * desc_cap, (size_t)n1);
        memcpy(row + n1, store + (2 * sl + 1) * desc_cap, (size_t)n2);
        last[s] = t;
        cnt[(size_t)s * RX_NCOUNT + rx_played_counter(n1, n2)]++;
        cnt[(size_t)s * RX_NCOUNT + RX_DROPPED] += rx_after_play(t, idx[sl], len + 2 * sl);
    }
}

// the shared merge rule alone: the row length, nbytes and lostflag of descriptions of n1 / n2 bytes (0 = missing)
int rx_model_merge(int n1, int n2, i16* nbytes, i32* lostflag) { return rx_merge(n1, n2, nbytes, lostflag); }

// the timing of a timed insert (solo_b200_rx_insert_timed_*), sequentially in array order: what the keys kernel's margin
// atomics and the sort + walk kernels' per-stream recurrence compute.  `last` is read only (an insert does not change it),
// so it may run before or after rx_model_insert of the same arrays.
void rx_model_timing(int n, int desc_cap, u32 ts_per_index, const u32* last, u32* transit, u32* jitter, u64* highest,
                     u32* received, u32* margin, const i32* stream, const u32* index, const u8* desc, const i32* off,
                     const i32* alen, const u32* arrival, int na, i64 payload_bytes) {
    for (int a = 0; a < na; a++) {
        const i32 s = stream[a];
        if (!rx_timed(n, desc_cap, s, desc[a], off[a], alen[a], payload_bytes)) continue;
        const int b = rx_margin_bin(index[a], last[s]);
        if (b >= 0) margin[(size_t)s * RX_MARGIN_BINS + b]++;
        rx_timing_step(index[a], arrival[a], ts_per_index, transit + s, jitter + s, highest + s, received + s);
    }
}

// one pack of n rows, the send queue's pack kernels' three passes in their order (sizes with per-block prefixes and
// totals, the scan of the block totals, the pack of every stream); returns the datagram count and writes the byte total
int tx_model_pack(int n, const u8* bits, int cap, const i16* nbytes, u32* next, u32* cnt, u8* payload, i32* stream, u32* index,
                  u8* desc, i32* off, i32* len, i64* total) {
    const int nblk = (n + SB_TX_BLOCK - 1) / SB_TX_BLOCK;
    std::vector<u64> pre(n), blk(nblk, 0);
    for (int s = 0; s < n; s++) {               // sb_tx_sizes_kernel
        int l1, l2;
        tx_row(nbytes[2 * s], nbytes[2 * s + 1], cap, &l1, &l2);
        pre[s] = blk[s / SB_TX_BLOCK];
        blk[s / SB_TX_BLOCK] += tx_scan_word(l1, l2);
    }
    u64 carry = 0;                              // sb_tx_scan_kernel
    for (int b = 0; b < nblk; b++) {
        const u64 t = blk[b];
        blk[b] = carry;
        carry += t;
    }
    for (int s = 0; s < n; s++) {               // sb_tx_pack_kernel
        int l1, l2;
        const int cls = tx_row(nbytes[2 * s], nbytes[2 * s + 1], cap, &l1, &l2);
        const u32 idx = next[s]++;
        tx_count(cnt + (size_t)s * TX_NCOUNT, cls, l1, l2);
        if (cls != TX_SENT) continue;
        const u64 at = blk[s / SB_TX_BLOCK] + pre[s];
        i32 k = tx_word_datagrams(at);
        const i64 b0 = tx_word_bytes(at);
        for (int d = 1; d <= 2; d++) {
            const int ln = d == 1 ? l1 : l2;
            if (ln <= 0) continue;
            stream[k] = s; index[k] = idx; desc[k] = (u8)d; off[k] = (i32)(b0 + (d == 2 ? l1 : 0)); len[k] = ln;
            k++;
        }
        memcpy(payload + b0, bits + (size_t)s * cap, (size_t)(l1 + l2));
    }
    *total = tx_word_bytes(carry);
    return tx_word_datagrams(carry);
}

// sb_mix_contributors_kernel over every member position, after the rows were set to -1 / 127
void tx_model_contributors(const i32* room_start, const i32* members, int R, int k, const i32* talkers, const u8* level,
                           int n, i32* csrc, u8* csrc_level) {
    for (size_t e = 0; e < (size_t)n * k; e++) { csrc[e] = -1; csrc_level[e] = SB_TX_LVL_NONE; }
    if (R == 0) return;
    for (i32 m = 0; m < room_start[R]; m++) {
        const i32 i = members[m];
        if ((u32)i >= (u32)n) continue;
        const int r = tx_room_of(room_start, R, m);
        tx_contributors(i, talkers + (size_t)r * k, k, level, n, csrc + (size_t)i * k, csrc_level + (size_t)i * k);
    }
}
}
