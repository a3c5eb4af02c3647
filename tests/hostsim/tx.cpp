// Host build of the send queue and the downlink contributor lists (solo_b200/csrc/sb_tx.cuh compiled by g++): the pack
// kernels' three passes in their order (sizes with per-block prefixes and totals, the scan of the block totals, the pack of
// every stream) and the contributor kernel's per-member rule.  TEST INFRASTRUCTURE ONLY; compiled by tests/test_tx.py,
// never linked into libsolo_b200.so.  The state arrays have the device layout of solo_b200.cu's TxDev.
//   g++ -O2 -std=c++17 -shared -fPIC -w tx.cpp -o libtx.so
#include <string.h>

#include <vector>

#include "../../solo_b200/csrc/sb_tx.cuh"

using namespace sb;

extern "C" {
// one pack of n rows; returns the datagram count and writes the byte total
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
