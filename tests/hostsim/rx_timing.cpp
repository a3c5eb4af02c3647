// Host build of the receive queue's timing (solo_b200/csrc/sb_rx.cuh compiled by g++): what a timed insert
// (solo_b200_rx_insert_timed_*) adds to the queue's state, the kernels' per-arrival rules applied one arrival at a time in
// array order.  TEST INFRASTRUCTURE ONLY; built by tests/hostsim/rx_timing.py into tests/_hostsim/librx_timing.so, never
// linked into libsolo_b200.so.  The state arrays have the device layout of solo_b200.cu's RxTiming.
#include "../../solo_b200/csrc/sb_rx.cuh"

using namespace sb;

extern "C" {
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
}
