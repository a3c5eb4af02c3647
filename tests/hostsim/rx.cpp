// Host build of the receive queue (solo_b200/csrc/sb_rx.cuh compiled by g++): the insert kernels' three passes in their
// order over the arrivals (elect, classify and copy, commit), with the atomics as plain read-modify-writes, and the pull
// kernel's per-stream rule.  TEST INFRASTRUCTURE ONLY; compiled by tests/test_rx.py, never linked into libsolo_b200.so.
// The state arrays have the device layout of solo_b200.cu's RxDev.
//   g++ -O2 -std=c++17 -shared -fPIC -w rx.cpp -o librx.so
#include "../../solo_b200/csrc/sb_rx.cuh"

using namespace sb;

extern "C" {
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
}
