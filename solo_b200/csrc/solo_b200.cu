// solo_b200 -- sm_90a (H100) kernels and the C ABI of libsolo_b200.so.
//
// One packet wave of the encoder = eight launches, of the decoder = two (DESIGN.md section 4):
//   sb_enc_qmf_kernel            warp per stream       QMF band split, PCM rows fetched by the TMA engine (cp.async.bulk)
//   sb_enc_vad_kernel            thread per stream     voice-activity detection of both frames (pure recurrences)
//   sb_enc_hb_warp_kernel        warp per stream       high-band LPC / LSP analysis            (sb_analysis.cu, sb_coop.cuh)
//   sb_enc_analysis_warp_kernel  warp per stream       pitch, noise shaping, LTP / LPC / NLSF analysis, state in shared memory
//   sb_enc_shape_post_kernel     thread per window     shaping-filter post-processing (inverse gains, coefficient limiting)
//   sb_enc_prefilter_kernel      thread per stream     prefilter recurrence | gain processing (grid.y)
//   sb_enc_nsq_kernel            two streams per warp  MD delayed-decision noise-shaping quantiser, history in shared memory
//   sb_enc_finish_kernel         2 threads per stream  range coding of one description each, high-band gains, payload assembly
//   sb_decode_kernel             thread per stream     range decoding, synthesis, concealment, comfort noise, high band
//   sb_dec_synth_kernel          warp per stream       QMF synthesis filter bank + float -> int16
// The two decoder kernels exist once per SILK core rate (template argument KHZ): 8 for 16 kHz streams, 16 for 32 kHz
// streams.  A batch holds one configuration, so it picks its instantiation when it is created.
// Between packets, sb_enc_control_kernel (thread per stream) changes the rate / DTX / expected-loss settings of streams;
// sb_enc_reset_kernel / sb_dec_reset_kernel (thread per listed stream) give listed streams a fresh state, and
// sb_state_copy_kernel (warp per listed stream, after sb_dec_blob_check_kernel for a 32 kHz decoder import) moves listed
// streams' states to or from device blobs.
// After a wave, and only when the caller asks for it, sb_activity_kernel (warp per stream) reports every stream's audio level
// and voice-activity / concealment flags of that wave (sb_activity.cuh).
// The conference mixer (solo_b200_mix_*, sb_mix.cuh) is two launches of its own: sb_mix_select_kernel (warp per room) picks
// each room's loudest talkers, sb_mix_kernel (warp per member) writes each member's mix-minus row.
// The receive queue (solo_b200_rx_*, sb_rx.cuh) pairs, reorders and screens the two descriptions of each stream's packets:
// an insert is sb_rx_elect_kernel, sb_rx_classify_kernel and sb_rx_commit_kernel over the arrivals, a pull is
// sb_rx_pull_kernel (warp per stream), which writes the decoder's input rows.  A timed insert of a queue with timing
// enabled adds sb_rx_timing_keys_kernel, a stable radix sort of the arrivals by stream (sb_rx_sort_hist / scan / scatter
// per 8-bit digit) and sb_rx_timing_walk_kernel, which runs each stream's jitter recurrence in array order.
// The send queue (solo_b200_tx_*, sb_tx.cuh) turns the encoder's rows into numbered datagrams packed back to back: a pack
// is sb_tx_sizes_kernel (thread per stream), sb_tx_scan_kernel (one block) and sb_tx_pack_kernel (warp per stream).
// sb_mix_contributors_kernel (thread per member) writes each downlink's CSRC list and RFC 6465 levels.
// The G.711 gateway (solo_b200_g711_*, sb_g711.cuh) puts PSTN / SIP participants in 16 kHz rooms: an uplink is
// sb_g711_vad_kernel (thread per stream) and sb_g711_synth_kernel (warp per stream), a downlink sb_g711_downlink_kernel
// (warp per stream), create and reset sb_g711_reset_kernel.
// Persistent per-stream state lives in device arrays (EncState / DecState) that never leave the GPU between packets;
// the *_host entry points process a wave as a few chunks of streams on the batch's CUDA streams.  The host code below is the C ABI:
// the batched entry points of include/solo_b200.h and the reference's six functions of include/AGR_JC1_SDK_API.h.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <mutex>
#include <vector>

#include "../../include/solo_b200.h"
#include "sb_activity.cuh"
#include "sb_dec.cuh"
#include "sb_enc.cuh"
#include "sb_g711.cuh"
#include "sb_mix.cuh"
#include "sb_nsq_warp.cuh"
#include "sb_rx.cuh"
#include "sb_tx.cuh"

using namespace sb;

// ---------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------
#define SB_TPB 64
#define SB_DEC_TPB 64
// the warp-per-stream analysis kernels live in sb_analysis.cu
extern "C" int sb_enc_analysis_setup(void);
extern "C" void sb_launch_enc_analysis_warp(void* states, void* scratch, const void* bands, int spp, int n, void* stream);
extern "C" void sb_launch_enc_hb_warp(void* states, void* scratch, const void* bands, int spp, int n, void* stream);
#define SB_FINISH_MINB 8     // 128 registers: every stream of a chunk resident
#define SB_DECODE_MINB 8

__global__ void __launch_bounds__(SB_TPB) sb_enc_init_kernel(EncState* states, int n, int rate, int dtx, int mdi, int framesize_ms, int joint_hb) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) enc_state_init(&states[s], rate, dtx, mdi, framesize_ms, joint_hb);
}
// rate / DTX / expected loss of each stream from the next packet on; a NULL array leaves that setting alone for every stream,
// an entry outside its range (-1 by convention) for that stream
__global__ void __launch_bounds__(SB_TPB) sb_enc_control_kernel(EncState* states, int n, const i32* __restrict__ rate, const i32* __restrict__ dtx,
                                                                const i32* __restrict__ loss) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) enc_set_control(&states[s], rate ? rate[s] : -1, dtx ? dtx[s] : -1, loss ? loss[s] : -1);
}

// ---- stage A0: QMF band split, one warp per stream, PCM tile fetched by the TMA engine ----------------------------------
// The split is the one part of the analysis without a recurrence: 320 (160) output pairs of a 64-tap symmetric FIR per
// packet.  A block takes SB_QMF_SPB consecutive streams; their PCM rows are contiguous in HBM, so ONE bulk asynchronous copy
// (cp.async.bulk -> UBLKCP, completion on an mbarrier) brings the whole tile into shared memory while the warps load their
// filter memories; each lane then produces output pairs k = lane, lane + 32, ... (products summed mod 2^32: order-free).
// Against the split inside kernel A this raised end-to-end throughput and left device-resident throughput unchanged;
// larger blocks (8 streams) were slower device-resident because they cannot start while kernel B holds the shared memory.
#define SB_QMF_SPB 1        // one-warp blocks of 2.8 KB: they fit in the shared memory the quantiser kernel leaves free on an SM
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__global__ void __launch_bounds__(SB_QMF_SPB * 32) sb_enc_qmf_kernel(EncState* states, const i16* __restrict__ pcm, i16* __restrict__ bands, int spp, int n, int bulk_ok) {
    __shared__ __align__(16) i16 tile[SB_QMF_SPB][PACKET];
    __shared__ __align__(16) i16 xs[SB_QMF_SPB][PACKET + 64];
    __shared__ i16 coef[64];
    __shared__ __align__(8) unsigned long long mbar;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int s0 = blockIdx.x * SB_QMF_SPB;
    const int rows = min(SB_QMF_SPB, n - s0);
    const i16* src = pcm + (size_t)s0 * spp;
    const unsigned bytes = (unsigned)(rows * spp * 2);
    const bool bulk = bulk_ok && (((size_t)src) & 15) == 0;  // 16-byte aligned source in this GPU's memory: use the copy engine
    const unsigned mb = smem_u32(&mbar);
    if (threadIdx.x == 0 && bulk) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mb));
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    for (int i = threadIdx.x; i < 64; i += blockDim.x) coef[i] = SB_T(qmf_fix)[i];
    __syncthreads();
    if (threadIdx.x == 0 && bulk) {
        // rows of `spp` samples land back to back: tile is addressed as a flat [rows * spp] array below
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mb), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(&tile[0][0])), "l"(src),
                     "r"(bytes), "r"(mb)
                     : "memory");
    }
    const int s = s0 + w;
    const bool live = w < rows;
    EncState* st = live ? &states[s] : nullptr;
    i16* x = xs[w];
    if (live) for (int i = lane; i < 63; i += 32) x[i] = st->qmf_mem[62 - i];      // x[i] = mem[M - i - 2]
    const i16* flat = &tile[0][0];
    if (bulk) {
        asm volatile("{\n .reg .pred p;\n WAIT_%=:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @p bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}" ::"r"(mb), "r"(0u)
                     : "memory");
    } else {
        for (int i = threadIdx.x; i < rows * spp; i += blockDim.x) tile[0][i] = src[i];
        __syncthreads();
    }
    if (!live) return;
    for (int i = lane; i < spp; i += 32) x[63 + i] = (i16)(flat[w * spp + i] >> 1);
    __syncwarp();
    i16* out = bands + (size_t)s * spp;
    const int half = spp >> 1;
    for (int k = lane; k < half; k += 32) {
        i16 lo, hi;
        qmf_output_pair(x, coef, k, &lo, &hi);
        out[k] = lo; out[half + k] = hi;
    }
    for (int i = lane; i < 63; i += 32) st->qmf_mem[i] = x[spp + 62 - i];          // mem[i] = x[N + M - 2 - i]
}

// ---- stage A1: voice-activity detector of both frames, one thread per stream (pure recurrence, full lane efficiency) ----
__global__ void __launch_bounds__(SB_TPB) sb_enc_vad_kernel(EncState* states, EncScratch* scratch, const i16* __restrict__ bands, int spp, int n) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    VadState v = states[s].vad;
    __align__(16) i16 low[2 * FRAME];
    const int nf = states[s].frames_per_packet;
    const int4* src = reinterpret_cast<const int4*>(bands + (size_t)s * spp);     // low band = first half of the row
    int4* dst = reinterpret_cast<int4*>(low);
    for (int i = 0; i < nf * FRAME / 8; i++) dst[i] = src[i];
    EncScratch* scr = &scratch[s];
    vad_packet(&v, low, nf, scr->vad_sa_Q8, scr->vad_quality_Q15, scr->vad_tilt_Q15);
    states[s].vad = v;
}

// ---- after the analysis kernel: scalar recursions whose results only the quantiser reads, one thread per instance ----
__global__ void __launch_bounds__(128) sb_enc_shape_post_kernel(const EncState* states, EncScratch* scratch, int n) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;       // (stream, frame, window)
    const int s = t >> 3;
    if (s >= n) return;
    const int f = (t >> 2) & 1, k = t & 3;
    if (f >= states[s].frames_per_packet) return;
    shape_post_window(&scratch[s], f, k);
}
__global__ void __launch_bounds__(SB_TPB) sb_enc_prefilter_kernel(EncState* states, EncScratch* scratch, int n) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const int nf = states[s].frames_per_packet;
    // two independent recursions per stream, one thread each (blockIdx.y): gain processing and the prefilter touch different
    // fields of the control blocks and of the state, so the two halves of the grid run side by side
    if (blockIdx.y == 0) prefilter_packet(&states[s], &scratch[s], nf);
    else gains_packet(&states[s], &scratch[s], nf);
}

#define SB_NSQ_WARPS 1      // one warp = two streams = 2 x 8.2 KB of shared memory; 12 blocks (24 streams) per SM
#define SB_NSQ_MINB 12     // <= 170 registers per thread
#define SB_NSQ_SPB (SB_NSQ_WARPS * (32 / SB_NSQ_GW))   // streams per block
__global__ void __launch_bounds__(SB_NSQ_WARPS * 32, SB_NSQ_MINB) sb_enc_nsq_kernel(EncState* states, EncScratch* scratch, int n) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int g = threadIdx.x / SB_NSQ_GW;                  // lane group inside the block = stream slot
    NsqSmem* S = reinterpret_cast<NsqSmem*>(smem_raw) + g;
    int s = blockIdx.x * SB_NSQ_SPB + g;
    const int warp_first = blockIdx.x * SB_NSQ_SPB + (threadIdx.x >> 5) * (32 / SB_NSQ_GW);
    if (warp_first >= n) return;                            // whole warps leave
    // A lane group without a stream of its own (odd batch size) shadows the warp's last valid stream: same inputs, same
    // arithmetic in its own shared-memory slot, identical values stored twice.  This keeps the sample loop's full-warp
    // collectives valid for every warp.
    if (s >= n) s = n - 1;
    nsq_packet_warp(*S, states[s].nsq, &scratch[s], states[s].frames_per_packet);
}

// Entropy coding and payload assembly, TWO threads per stream: thread k runs the stage-C steps of description k
// (sb_enc.cuh; the two coders share nothing but read-only frame parameters) and exchanges lengths and status with its
// partner by shuffle between coding and storing.  enc_packet_finish runs the same steps for both k on one thread.
__global__ void __launch_bounds__(SB_TPB, SB_FINISH_MINB) sb_enc_finish_kernel(EncState* states, const EncScratch* scratch, u8* __restrict__ bits, int cap,
                                                               i16* __restrict__ nbytes, int n) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int s = t >> 1, k = t & 1;
    const unsigned m = __ballot_sync(0xffffffffu, s < n);     // whole pairs
    if (s >= n) return;
    EncCore* st = &states[s];
    const EncScratch* scr = &scratch[s];
    u8* out = bits + (size_t)s * cap;
    u8 rcbuf[MAX_PAYLOAD];
    RangeEnc rc;
    int ok_k;
    const int nb_k = enc_code_description(&rc, rcbuf, st, scr, k, &ok_k);
    const int nb_o = __shfl_xor_sync(m, nb_k, 1), ok_o = __shfl_xor_sync(m, ok_k, 1);
    const int nb0 = k ? nb_o : nb_k, nb1 = k ? nb_k : nb_o, ok0 = k ? ok_o : ok_k, ok1 = k ? ok_k : ok_o;
    const int lb = enc_store_description(&rc, scr, k, nb0, nb1, ok0, ok1, out, cap);
    __syncwarp(m);      // a rejected or dropped packet's high-band bytes land on top of description 1's
    enc_store_high_band(st, scr, k, lb, nb1, out, cap, &nbytes[2 * s]);
}

static_assert(SOLO_B200_DEC_FLP == DEC_FLP && SOLO_B200_DEC_FIX == DEC_FIX, "decoder arithmetic codes");
template <int KHZ>
__global__ void __launch_bounds__(SB_TPB) sb_dec_init_kernel(DecStateT<KHZ>* states, int n, int mdi, int framesize_ms, int joint_hb, int arith,
                                                             int core_only) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) dec_state_init(&states[s], mdi, framesize_ms, joint_hb, arith, core_only);
}

// ---- stream membership: reset, export and import of a list of streams (solo_b200_{enc,dec}_batch_reset / *_states) -----
// Reset, one thread per listed stream: the stream as create made it (the batch's create settings), then its own settings
// through the per-packet control -- create followed by set_control is create with those settings.  An entry of -1, or a
// NULL array, keeps the create value.  The state is zeroed with word stores (16 bytes for EncState, 4 for the decoder's
// 4-byte aligned states) where the init bodies' memset stores byte by byte, then the init bodies set their fields.
template <class W, class S> __device__ __forceinline__ void zero_state(S* st) {
    static_assert(sizeof(S) % sizeof(W) == 0 && alignof(S) >= alignof(W), "zero_state word");
    W* w = reinterpret_cast<W*>(st);
#pragma unroll 8
    for (int k = 0; k < (int)(sizeof(S) / sizeof(W)); k++) w[k] = W{};
}
__global__ void __launch_bounds__(SB_TPB) sb_enc_reset_kernel(EncState* states, const i32* __restrict__ streams, int n, const i32* __restrict__ rate,
                                                              const i32* __restrict__ dtx, const i32* __restrict__ loss, int rate0, int dtx0,
                                                              int mdi, int framesize_ms, int joint_hb) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    EncState* st = &states[streams[i]];
    zero_state<uint4>(st);
    enc_state_fields(st, rate0, dtx0, mdi, framesize_ms, joint_hb);
    enc_set_control(st, rate ? rate[i] : -1, dtx ? dtx[i] : -1, loss ? loss[i] : -1);
}
template <int KHZ>
__global__ void __launch_bounds__(SB_TPB) sb_dec_reset_kernel(DecStateT<KHZ>* states, const i32* __restrict__ streams, int n, const i32* __restrict__ arith,
                                                              int arith0, int mdi, int framesize_ms, int joint_hb, int core_only) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    DecStateT<KHZ>* st = &states[streams[i]];
    zero_state<u32>(st);
    dec_state_fields(st, mdi, framesize_ms, joint_hb, arith && arith[i] != -1 ? arith[i] : arith0, core_only);
}
// 32 kHz import: a blob of the other output mode than the batch's sets *bad, and then the copy kernel copies nothing
__global__ void __launch_bounds__(SB_TPB) sb_dec_blob_check_kernel(const DecState32* blobs, int n, int core_only, int* bad) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && blobs[i].core_only != core_only) *bad = 1;
}
// One warp per listed stream moves its state between the batch's array and row i of `blobs` (to_blobs: export) in words of
// W: 8 bytes (256 contiguous bytes per warp instruction) for the encoder's and the 32 kHz decoder's states, 4 bytes for the
// 16 kHz decoder's, whose 4 252-byte stride keeps only 4-byte alignment; four loads in flight per lane.  Blobs in another
// GPU's memory are read and written with ordinary loads and stores over NVLink, as the ingest path's kernels do with peer
// rows.  skip != NULL and *skip != 0: the import check found a blob of the other mode, nothing is copied.
#define SB_COPY_WARPS 8
template <class W>
__global__ void __launch_bounds__(SB_COPY_WARPS * 32) sb_state_copy_kernel(W* states, int words, const i32* __restrict__ streams, int n,
                                                                           W* blobs, int to_blobs, const int* __restrict__ skip) {
    const int i = blockIdx.x * SB_COPY_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (i >= n || (skip && *skip)) return;
    W* s = states + (size_t)streams[i] * words;
    W* b = blobs + (size_t)i * words;
    W* dst = to_blobs ? b : s;
    const W* src = to_blobs ? s : b;
    int k = lane;
    for (; k + 96 < words; k += 128) {
        const W w0 = src[k], w1 = src[k + 32], w2 = src[k + 64], w3 = src[k + 96];
        dst[k] = w0; dst[k + 32] = w1; dst[k + 64] = w2; dst[k + 96] = w3;
    }
    for (; k < words; k += 32) dst[k] = src[k];
}

// CORE = false: band signals of `spp`-sample packets into band_low / band_high, rows of spp / 2 samples, for the synthesis
// kernel.  CORE = true (core output): the SILK core's PCM straight into band_low = the caller's PCM rows of spp / 2 samples;
// band_high is not used and there is no synthesis launch.
template <int KHZ, bool CORE = false>
__global__ void __launch_bounds__(SB_DEC_TPB, SB_DECODE_MINB) sb_decode_kernel(DecStateT<KHZ>* states, const u8* __restrict__ bits, int cap,
                                                           const i16* __restrict__ nbytes, const i32* __restrict__ lostflag,
                                                           i32* __restrict__ ret, i32* __restrict__ ret_int, u8* __restrict__ act, DecStale* stale,
                                                           i16* __restrict__ band_low, float* __restrict__ band_high, int spp, int n) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    DecPacketWorkT<KHZ> W;
    i16 nb[2] = {nbytes[2 * s], nbytes[2 * s + 1]};
    const DecBands bands = {band_low + (size_t)s * (spp / 2), CORE ? nullptr : band_high + (size_t)s * (spp / 2)};
    i32 r = dec_packet<KHZ, CORE>(&states[s], &W, bits + (size_t)s * cap, cap, nb, lostflag[s], &stale[s], &bands);
    if (ret) ret[s] = r;
    ret_int[s] = r;
    act[s] = r < 0 ? (u8)0 : W.act;
}

// ---- synthesis filter bank + float -> int16, one warp per stream (AGR_BWE_qmf.c:86-182, AGR_BWE_decode_frame_FLP.c:222-231) ----
// N2 / 2 independent groups of four outputs per packet (160 or 80 for 16 kHz streams, twice that for 32 kHz): lanes over
// groups, band signals and filter memories staged in shared memory; the PCM row is written with 8-byte stores, 256 contiguous bytes per warp instruction.  A DEC_FIX stream
// takes the integer filter bank in the same layout, its band signals staged as int16 in the first half of each row.
#define SB_SYN_WARPS 4
__device__ __forceinline__ void store_pcm4(i16* out, int g, const i16* y) {
    int2 pk;
    pk.x = (int)((u16)y[0] | ((u32)(u16)y[1] << 16));
    pk.y = (int)((u16)y[2] | ((u32)(u16)y[3] << 16));
    reinterpret_cast<int2*>(out)[g] = pk;
}
template <int KHZ>
__global__ void __launch_bounds__(SB_SYN_WARPS * 32) sb_dec_synth_kernel(DecStateT<KHZ>* states, const i16* __restrict__ band_low, const float* __restrict__ band_high,
                                                                        const i32* __restrict__ ret_int, i16* __restrict__ pcm, int spp, int n) {
    __shared__ float xx[SB_SYN_WARPS][2][32 + 2 * DecCore<KHZ>::FRAME];
    __shared__ float coef[64];
    __shared__ i16 coef_fix[64];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < 64; i += blockDim.x) { coef[i] = SB_T(qmf_flt)[i]; coef_fix[i] = SB_T(qmf_fix)[i]; }
    __syncthreads();
    const int s = blockIdx.x * SB_SYN_WARPS + w;
    if (s >= n || ret_int[s] < 0) return;         // a rejected packet leaves its PCM row and the filter memories alone
    const int N2 = spp >> 1;
    float* xx1 = xx[w][0];
    float* xx2 = xx[w][1];
    DecStateT<KHZ>* st = &states[s];
    const i16* lo = band_low + (size_t)s * N2;
    const float* hi = band_high + (size_t)s * N2;
    i16* out = pcm + (size_t)s * spp;
    if (st->arith == DEC_FIX) {                   // warp-uniform: one stream per warp
        i16* yy1 = reinterpret_cast<i16*>(xx1);
        i16* yy2 = reinterpret_cast<i16*>(xx2);
        for (int i = lane; i < N2; i += 32) { yy1[i] = lo[N2 - 1 - i]; yy2[i] = (i16)__float2int_rz(hi[N2 - 1 - i]); }
        yy1[N2 + lane] = (i16)__float2int_rz(st->g0_mem[2 * lane + 1]);
        yy2[N2 + lane] = (i16)__float2int_rz(st->g1_mem[2 * lane + 1]);
        __syncwarp();
        for (int g = lane; g < N2 / 2; g += 32) {
            i16 y[4];
            qmf_synth_group_fix(yy1, yy2, coef_fix, N2, 2 * g, y);
            store_pcm4(out, g, y);
        }
        __syncwarp();
        st->g0_mem[2 * lane + 1] = (float)yy1[lane];
        st->g1_mem[2 * lane + 1] = (float)yy2[lane];
        return;
    }
    for (int i = lane; i < N2; i += 32) { xx1[i] = (float)lo[N2 - 1 - i]; xx2[i] = hi[N2 - 1 - i]; }
    xx1[N2 + lane] = st->g0_mem[2 * lane + 1];
    xx2[N2 + lane] = st->g1_mem[2 * lane + 1];
    __syncwarp();
    for (int g = lane; g < N2 / 2; g += 32) {
        i16 y[4];
        qmf_synth_group(xx1, xx2, coef, N2, 2 * g, y);
        store_pcm4(out, g, y);
    }
    __syncwarp();
    st->g0_mem[2 * lane + 1] = xx1[lane];
    st->g1_mem[2 * lane + 1] = xx2[lane];
}

// ---- activity report of the last wave (sb_activity.cuh), one warp per row ----------------------------------------------
// The row's sum of squares from 16-byte loads (2-byte loads when the caller's rows are not 16-byte aligned), reduced over
// the warp in int64, then lane 0 looks up the level and copies the flags: the encoder's from its scratch (enc), the
// decoder's from the bytes the decode kernel stored (dec_act).  A decoder row whose packet was rejected (dec_ret < 0)
// reports 127 / 0 without reading its PCM row, which that packet did not write.
#define SB_ACT_WARPS 8
__global__ void __launch_bounds__(SB_ACT_WARPS * 32) sb_activity_kernel(const i16* __restrict__ pcm, int spp, int nf, const EncScratch* __restrict__ enc,
                                                                         const u8* __restrict__ dec_act, const i32* __restrict__ dec_ret,
                                                                         u8* __restrict__ level, u8* __restrict__ flags, int n) {
    const int s = blockIdx.x * SB_ACT_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (s >= n) return;                           // whole warps
    if (dec_ret && dec_ret[s] < 0) {
        if (lane == 0) { level[s] = 127; flags[s] = 0; }
        return;
    }
    const i16* row = pcm + (size_t)s * spp;       // rows are multiples of 16 bytes: every row is aligned as the first
    i64 e = 0;
    if ((((size_t)row) & 15) == 0) {
        const int4* v = reinterpret_cast<const int4*>(row);
        for (int i = lane; i < spp / 8; i += 32) {
            const int4 q = v[i];
            const int w[4] = {q.x, q.y, q.z, q.w};
            for (int j = 0; j < 4; j++) {
                const i32 lo = (i16)(w[j] & 0xffff), hi = w[j] >> 16;
                e += (i64)((u32)(lo * lo) + (u32)(hi * hi));     // <= 2^31: exact in u32
            }
        }
    } else {
        for (int i = lane; i < spp; i += 32) { const i32 x = row[i]; e += x * x; }
    }
    for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
    if (lane == 0) {
        level[s] = (u8)rfc6464_level(e, spp);
        flags[s] = enc ? (u8)enc_activity_flags(&enc[s], nf) : dec_act[s];
    }
}

// ---- conference mixer (sb_mix.cuh): talker selection, one warp per room -------------------------------------------------
// Lane l keeps the top 8 keys of members lo + l, lo + l + 32, ...; then k rounds each take the smallest head of the 32 lists
// (a shuffle reduction) and the lane that held it drops it.  Members are fetched SB_MIX_UNROLL per lane at a time so that the
// gathers of flags / level of a large room overlap.  Room bounds are clamped to [0, M] (M = room_start[R]) and members outside
// [0, n) are skipped, so no contents of the arrays lead to an access out of bounds.
#define SB_MIX_WARPS 8
#define SB_MIX_UNROLL 16
__global__ void __launch_bounds__(SB_MIX_WARPS * 32) sb_mix_select_kernel(const u8* __restrict__ level, const u8* __restrict__ flags,
                                                                           const i32* __restrict__ room_start, const i32* __restrict__ members,
                                                                           int n, int R, int k, i32* __restrict__ talkers) {
    const int r = blockIdx.x * SB_MIX_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= R) return;                           // whole warps
    const i32 M = imax(room_start[R], 0);
    const i32 lo = imin(imax(room_start[r], 0), M), hi = imin(imax(room_start[r + 1], lo), M);
    u64 L[SB_MIX_KMAX];
#pragma unroll
    for (int i = 0; i < SB_MIX_KMAX; i++) L[i] = SB_MIX_NONE;
    for (i32 base = lo; base < hi; base += 32 * SB_MIX_UNROLL) {
        i32 j[SB_MIX_UNROLL];
        u8 f[SB_MIX_UNROLL], lv[SB_MIX_UNROLL];
#pragma unroll
        for (int u = 0; u < SB_MIX_UNROLL; u++) {
            const i32 m = base + u * 32 + lane;
            j[u] = m < hi ? members[m] : -1;
        }
#pragma unroll
        for (int u = 0; u < SB_MIX_UNROLL; u++) {
            const bool ok = (u32)j[u] < (u32)n;
            f[u] = ok ? flags[j[u]] : (u8)0;
            lv[u] = ok ? level[j[u]] : (u8)0;
        }
#pragma unroll
        for (int u = 0; u < SB_MIX_UNROLL; u++) {
            const u64 key = mix_key(lv[u], j[u]);
            if (mix_eligible(f[u]) && key < L[SB_MIX_KMAX - 1]) mix_topk_insert(L, key);
        }
    }
    for (int t = 0; t < k; t++) {
        u64 best = L[0];
        for (int o = 16; o > 0; o >>= 1) {
            const u64 v = __shfl_xor_sync(0xffffffffu, best, o);
            best = v < best ? v : best;
        }
        mix_topk_pop(L, best);
        if (lane == 0) talkers[(size_t)r * k + t] = mix_key_stream(best);
    }
}

// ---- conference mixer: one warp per member row ---------------------------------------------------------------------------
// Member position m (grid-stride over M = room_start[R], which the host cannot read without a synchronise) finds its room by
// the warp's 33-ary search (one probe per lane and round), lanes 0..k-1 read the room's talkers and the warp keeps those the
// listener hears.  Then each lane sums 16-byte chunks c = lane, lane + 32, ... of those rows in int32 and stores the
// saturated chunk with one 16-byte store.  The talker rows are read by every member of the room: after the first they come
// from L2 (or L1, for members in one block).  The kernel is a chain of dependent loads per member (bounds, member, search,
// talkers, rows), so it is sized for 6 resident blocks per SM (40 registers, 36 bytes of spill stores): the more members in flight, the more
// of the chain overlaps.
__global__ void __launch_bounds__(SB_MIX_WARPS * 32, 6) sb_mix_kernel(const i16* __restrict__ in, i16* __restrict__ out, int spp, int n,
                                                                       const i32* __restrict__ room_start, const i32* __restrict__ members,
                                                                       int R, int k, const i32* __restrict__ talkers) {
    const int lane = threadIdx.x & 31, nv = spp / 8;
    const i32 M = room_start[R];
    for (i32 m = blockIdx.x * SB_MIX_WARPS + (threadIdx.x >> 5); m < M; m += gridDim.x * SB_MIX_WARPS) {
        const i32 i = members[m];
        if ((u32)i >= (u32)n) continue;           // whole warps
        int r = 0, span = R;
        while (span > 1) {
            const int step = mix_search_step(span), p = r + lane * step;
            mix_search_narrow(&r, &span, step, __ballot_sync(0xffffffffu, p < r + span && room_start[p] <= m));
        }
        const i32 tj = lane < k ? talkers[(size_t)r * k + lane] : -1;
        unsigned hear = __ballot_sync(0xffffffffu, (u32)tj < (u32)n && mix_hears(i, tj));
        const int nt = __popc(hear);
        i32 src[SB_MIX_KMAX];                     // the talker rows heard, as stream indices
#pragma unroll
        for (int t = 0; t < SB_MIX_KMAX; t++) {
            src[t] = 0;
            if (t < nt) {
                const int l = __ffs(hear) - 1;
                hear &= hear - 1;
                src[t] = __shfl_sync(0xffffffffu, tj, l);
            }
        }
        const int4* rows = reinterpret_cast<const int4*>(in);
        int4* dst = reinterpret_cast<int4*>(out + (size_t)i * spp);
        for (int c = lane; c < nv; c += 32) {
            i32 acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
            for (int t = 0; t < SB_MIX_KMAX; t++) {
                if (t < nt) {
                    const int4 q = __ldg(rows + (size_t)src[t] * nv + c);
                    const int w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                    for (int h = 0; h < 4; h++) { acc[2 * h] += (i16)(w[h] & 0xffff); acc[2 * h + 1] += w[h] >> 16; }
                }
            }
            int w[4];
#pragma unroll
            for (int h = 0; h < 4; h++) w[h] = (i32)((u32)(u16)mix_out(acc[2 * h]) | ((u32)(u16)mix_out(acc[2 * h + 1]) << 16));
            dst[c] = make_int4(w[0], w[1], w[2], w[3]);
        }
    }
}

// ---- G.711 gateway (sb_g711.cuh) -------------------------------------------------------------------------------------------
// Create and reset, one thread per stream: the listed streams (streams = NULL: every stream) as create makes them, each with
// its law (-1 or a NULL array: law0).
__global__ void __launch_bounds__(SB_TPB) sb_g711_reset_kernel(G711State* states, const i32* __restrict__ streams, int n,
                                                               const i32* __restrict__ law, int law0) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    g711_state_init(&states[streams ? streams[i] : i], law && law[i] != -1 ? law[i] : law0);
}

// Uplink, voice activity: one thread per stream, as sb_enc_vad_kernel (the detector is a pure recurrence).  The thread
// expands its row from 16-byte loads into a local frame buffer and writes the flags byte.
__global__ void __launch_bounds__(SB_TPB) sb_g711_vad_kernel(G711State* states, const u8* __restrict__ codes, const i32* __restrict__ lost,
                                                             u8* __restrict__ flags, int nf, int n) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    const int law = states[s].law;
    const i32 ls = lost ? lost[s] : 0;
    __align__(16) i16 x8[2 * FRAME];
    const uint4* src = reinterpret_cast<const uint4*>(codes + (size_t)s * nf * FRAME);
    for (int c = 0; c < nf * FRAME / 16; c++) {
        const uint4 q = src[c];
        const u32 w[4] = {q.x, q.y, q.z, q.w};
        for (int b = 0; b < 16; b++) x8[16 * c + b] = g711_up_sample(law, (u8)(w[b >> 2] >> (8 * (b & 3))), ls, 16 * c + b);
    }
    VadState v = states[s].vad;
    i32 sa_Q8[2];
    flags[s] = (u8)g711_vad(&v, x8, nf, ls, sa_Q8);
    states[s].vad = v;
}

// Uplink, synthesis and level: one warp per stream.  Lanes expand 16 codes each (one 16-byte load) into the time-reversed
// low band in shared memory, then run the decoder's fixed-point synthesis groups over it against a shared zero high band
// (sb_dec_synth_kernel's DEC_FIX layout), store the row with 8-byte stores and reduce the row's energy for its level.
#define SB_G711_WARPS 8
__global__ void __launch_bounds__(SB_G711_WARPS * 32) sb_g711_synth_kernel(G711State* states, const u8* __restrict__ codes, const i32* __restrict__ lost,
                                                                           i16* __restrict__ pcm, u8* __restrict__ level, int nf, int n) {
    __shared__ i16 yy[SB_G711_WARPS][32 + 2 * FRAME];
    __shared__ i16 zero[32 + 2 * FRAME];
    __shared__ i16 coef[64];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < 32 + 2 * FRAME; i += blockDim.x) zero[i] = 0;
    for (int i = threadIdx.x; i < 64; i += blockDim.x) coef[i] = SB_T(qmf_fix)[i];
    __syncthreads();
    const int s = blockIdx.x * SB_G711_WARPS + w;
    if (s >= n) return;                           // whole warps
    const int N2 = nf * FRAME;
    G711State* st = &states[s];
    const int law = st->law;
    const i32 ls = lost ? lost[s] : 0;
    i16* yy1 = yy[w];
    if (lane < N2 / 16) {
        const uint4 q = reinterpret_cast<const uint4*>(codes + (size_t)s * N2)[lane];
        const u32 c4[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int b = 0; b < 16; b++) {
            const int i = 16 * lane + b;
            yy1[N2 - 1 - i] = g711_up_sample(law, (u8)(c4[b >> 2] >> (8 * (b & 3))), ls, i);
        }
    }
    yy1[N2 + lane] = st->syn_mem[lane];
    __syncwarp();
    i16* out = pcm + (size_t)s * 2 * N2;
    i64 e = 0;
    for (int g = lane; g < N2 / 2; g += 32) {
        i16 y[4];
        qmf_synth_group_fix(yy1, zero, coef, N2, 2 * g, y);
        store_pcm4(out, g, y);
        e += (i64)((u32)(y[0] * y[0]) + (u32)(y[1] * y[1])) + (i64)((u32)(y[2] * y[2]) + (u32)(y[3] * y[3]));
    }
    st->syn_mem[lane] = yy1[lane];
    for (int o = 16; o > 0; o >>= 1) e += __shfl_xor_sync(0xffffffffu, e, o);
    if (lane == 0) level[s] = (u8)rfc6464_level(e, 2 * N2);
}

// Downlink: one warp per stream, sb_enc_qmf_kernel's band split (history and row in shared memory, output pairs k = lane,
// lane + 32, ...) with the low band compressed in lane and stored as one coalesced byte per lane; the high band is dropped.
__global__ void __launch_bounds__(SB_G711_WARPS * 32) sb_g711_downlink_kernel(G711State* states, const i16* __restrict__ pcm, u8* __restrict__ codes,
                                                                              int spp, int n) {
    __shared__ i16 xs[SB_G711_WARPS][PACKET + 64];
    __shared__ i16 coef[64];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < 64; i += blockDim.x) coef[i] = SB_T(qmf_fix)[i];
    __syncthreads();
    const int s = blockIdx.x * SB_G711_WARPS + w;
    if (s >= n) return;
    G711State* st = &states[s];
    const int law = st->law;
    i16* x = xs[w];
    for (int i = lane; i < 63; i += 32) x[i] = st->ana_mem[62 - i];      // x[i] = mem[M - i - 2]
    const int4* row = reinterpret_cast<const int4*>(pcm + (size_t)s * spp);
    for (int c = lane; c < spp / 8; c += 32) {
        const int4 q = row[c];
        const int v[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int h = 0; h < 4; h++) {
            x[63 + 8 * c + 2 * h] = (i16)((i16)(v[h] & 0xffff) >> 1);
            x[64 + 8 * c + 2 * h] = (i16)(v[h] >> 17);
        }
    }
    __syncwarp();
    const int half = spp >> 1;
    u8* out = codes + (size_t)s * half;
    for (int k = lane; k < half; k += 32) {
        i16 lo, hi;
        qmf_output_pair(x, coef, k, &lo, &hi);
        out[k] = g711_compress(law, lo);
    }
    for (int i = lane; i < 63; i += 32) st->ana_mem[i] = x[spp + 62 - i];    // mem[i] = x[N + M - 2 - i]
}

// ---- receive queue (sb_rx.cuh) -------------------------------------------------------------------------------------------
// The queue's device arrays.  Slot metadata (index, the two lengths, the election words) is kept apart from the payload
// store, so the election and classify passes touch a few bytes per slot.  Slot sl = s * depth + j; description d of it is
// store[(2 * sl + d) * desc_cap ...], 16-byte aligned (desc_cap is a multiple of 16); the store has 16 bytes of padding
// after the last slot for the pull kernel's second aligned load.
struct RxDev {
    int n, depth, desc_cap;
    u32* last;                  // [n] last played index
    u32* idx;                   // [n][depth] held index
    u16* len;                   // [n][depth][2] held description lengths, 0 = not held
    unsigned long long* elect;  // [n][depth][2] election words of the running insert, 0 between calls
    u32* rep;                   // [n][depth] position of the arrival that commits the slot, RX_NO_REP between calls
    u32* cnt;                   // [n][RX_NCOUNT]
    unsigned long long* bad;    // arrivals for streams outside [0, n)
    u8* store;                  // [n][depth][2][desc_cap] + 16
};
struct RxArrivals {
    const i32* stream; const u32* index; const u8* desc; const i32* off; const i32* len;
    int n; const u8* payload; i64 payload_bytes;
};
__device__ __forceinline__ long long rx_arrival_slot_of(const RxDev& q, const RxArrivals& A, int a, u32* dist) {
    return rx_arrival_slot(q.n, q.depth, q.desc_cap, q.last, A.stream[a], A.desc[a], A.off[a], A.len[a], A.index[a],
                           A.payload_bytes, dist);
}

#define SB_RX_THREADS 256
#define SB_RX_TEAM 8            // lanes per arrival in the classify pass: 16 bytes each, 128 bytes per round
// insert, pass 1 (thread per arrival): per (slot, desc) the newest index and its first arrival; per slot the first arrival
__global__ void __launch_bounds__(SB_RX_THREADS) sb_rx_elect_kernel(RxDev q, RxArrivals A) {
    const int a = blockIdx.x * SB_RX_THREADS + threadIdx.x;
    if (a >= A.n) return;
    u32 dist;
    const long long sl = rx_arrival_slot_of(q, A, a, &dist);
    if (sl < 0) return;
    atomicMax(&q.elect[2 * sl + A.desc[a] - 1], (unsigned long long)rx_key(dist, a));
    atomicMin(&q.rep[sl], (u32)a);
}

// insert, pass 2 (SB_RX_TEAM lanes per arrival): count every arrival once and copy the stored ones to their slot, 16-byte
// stores from byte loads of the unaligned source.  Reads the slots' metadata and election words, writes neither.
__global__ void __launch_bounds__(SB_RX_THREADS) sb_rx_classify_kernel(RxDev q, RxArrivals A) {
    const long long g = (long long)blockIdx.x * SB_RX_THREADS + threadIdx.x;
    const int a = (int)(g / SB_RX_TEAM), t = (int)(g % SB_RX_TEAM);
    if (a >= A.n) return;
    const i32 s = A.stream[a];
    if ((u32)s >= (u32)q.n) {
        if (t == 0) atomicAdd(q.bad, 1ull);
        return;
    }
    const int d = A.desc[a];
    const i32 o = A.off[a], l = A.len[a];
    int cls;
    long long sl = -1;
    if (rx_malformed(d, o, l, q.desc_cap, A.payload_bytes)) cls = RX_MALFORMED;
    else if (!rx_current(A.index[a], q.last[s])) cls = RX_LATE;
    else {
        const u32 p = A.index[a], last = q.last[s];
        sl = (long long)s * q.depth + rx_slot(p, q.depth);
        const u64 e[2] = {q.elect[2 * sl], q.elect[2 * sl + 1]};
        const u16 ln[2] = {q.len[2 * sl], q.len[2 * sl + 1]};
        cls = rx_classify(p - last, d - 1, a, e, q.idx[sl], ln, last);
    }
    if (t == 0) atomicAdd(&q.cnt[(size_t)s * RX_NCOUNT + cls], 1u);
    if (cls != RX_STORED) return;
    const u8* src = A.payload + o;
    uint4* dst = reinterpret_cast<uint4*>(q.store + (size_t)(2 * sl + d - 1) * q.desc_cap);
    for (int c = t; 16 * c < l; c += SB_RX_TEAM) {
        u32 w[4] = {0, 0, 0, 0};
#pragma unroll
        for (int i = 0; i < 16; i++)
            if (16 * c + i < l) w[i >> 2] |= (u32)src[16 * c + i] << (8 * (i & 3));
        dst[c] = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

// insert, pass 3 (thread per arrival): the slot's committing arrival writes its new index and lengths, counts the held
// descriptions it discards and empties the election words
__global__ void __launch_bounds__(SB_RX_THREADS) sb_rx_commit_kernel(RxDev q, RxArrivals A) {
    const int a = blockIdx.x * SB_RX_THREADS + threadIdx.x;
    if (a >= A.n) return;
    u32 dist;
    const long long sl = rx_arrival_slot_of(q, A, a, &dist);
    if (sl < 0 || q.rep[sl] != (u32)a) return;
    const i32 s = A.stream[a];
    const u64 e[2] = {q.elect[2 * sl], q.elect[2 * sl + 1]};
    u32 id = q.idx[sl];
    u16 ln[2] = {q.len[2 * sl], q.len[2 * sl + 1]};
    const int discarded = rx_commit(q.last[s], &id, ln, e, A.len);
    q.idx[sl] = id;
    q.len[2 * sl] = ln[0];
    q.len[2 * sl + 1] = ln[1];
    if (discarded) atomicAdd(&q.cnt[(size_t)s * RX_NCOUNT + RX_DROPPED], (u32)discarded);
    q.elect[2 * sl] = 0;
    q.elect[2 * sl + 1] = 0;
    q.rep[sl] = RX_NO_REP;
}

// 16 bytes of the merged row [description 1 (n1 bytes) | description 2] starting at row byte 16c, from the slot's two
// descriptions at S (16-byte aligned) and S + desc_cap.  Row bytes below n1 come from the aligned chunk c of description 1,
// the others from description 2 at byte desc_cap + 16c - n1: two aligned loads, a word select and a funnel shift.
__device__ __forceinline__ void rx_row_chunk(const u8* S, int desc_cap, int n1, int c, u32 w[4]) {
    const int base = 16 * c;
    u32 wa[4] = {0, 0, 0, 0}, wb[4] = {0, 0, 0, 0};
    if (base < n1) {
        const uint4 x = reinterpret_cast<const uint4*>(S)[c];
        wa[0] = x.x; wa[1] = x.y; wa[2] = x.z; wa[3] = x.w;
    }
    if (base + 16 > n1) {
        const int b = desc_cap + base - n1;
        const uint4* src = reinterpret_cast<const uint4*>(S + (b & ~15));
        const uint4 x = src[0], y = (b & 15) ? src[1] : make_uint4(0, 0, 0, 0);
        const u32 v[8] = {x.x, x.y, x.z, x.w, y.x, y.y, y.z, y.w};
        const int sh = (b & 15) >> 2, bs = (b & 3) * 8;
        u32 r[5];
#pragma unroll
        for (int k = 0; k < 5; k++) r[k] = sh == 0 ? v[k] : sh == 1 ? v[k + 1] : sh == 2 ? v[k + 2] : v[k + 3];
#pragma unroll
        for (int k = 0; k < 4; k++) wb[k] = __funnelshift_r(r[k], r[k + 1], bs);
    }
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int m = imin(imax(n1 - (base + 4 * k), 0), 4);      // bytes of word k that come from description 1
        const u32 mask = m >= 4 ? 0xFFFFFFFFu : (1u << (8 * m)) - 1u;
        w[k] = (wa[k] & mask) | (wb[k] & ~mask);
    }
}

// pull (warp per stream): the row, nbytes and lostflag of index t = play[s] (or last + 1), then last = t and the slot
// emptied when its index is no longer current.  Only bytes below nbytes[0] of the row are written: 16-byte stores when the
// row is 16-byte aligned, byte stores for the tail.
#define SB_RX_PULL_WARPS 8
__global__ void __launch_bounds__(SB_RX_PULL_WARPS * 32) sb_rx_pull_kernel(RxDev q, const u32* __restrict__ play, u8* __restrict__ bits,
                                                                            int cap, i16* __restrict__ nbytes, i32* __restrict__ lostflag) {
    const int s = blockIdx.x * SB_RX_PULL_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (s >= q.n) return;                         // whole warps
    const u32 t = play ? play[s] : q.last[s] + 1u;
    const size_t sl = (size_t)s * q.depth + rx_slot(t, q.depth);
    const u32 id = q.idx[sl];
    u16 ln[2] = {q.len[2 * sl], q.len[2 * sl + 1]};
    int n1, n2;
    rx_play(t, id, ln, &n1, &n2);
    i16 nb[2];
    i32 lf;
    const int nrow = rx_merge(n1, n2, nb, &lf);
    const u8* S = q.store + 2 * sl * (size_t)q.desc_cap;
    u8* row = bits + (size_t)s * cap;
    const bool aligned = (cap & 15) == 0;
    for (int c = lane; 16 * c < nrow; c += 32) {
        u32 w[4] = {0, 0, 0, 0};
        if (lf != 1) rx_row_chunk(S, q.desc_cap, n1, c, w);
        if (aligned && 16 * c + 16 <= nrow) {
            *reinterpret_cast<uint4*>(row + 16 * c) = make_uint4(w[0], w[1], w[2], w[3]);
        } else {
            for (int i = 0; i < 16 && 16 * c + i < nrow; i++) row[16 * c + i] = (u8)(w[i >> 2] >> (8 * (i & 3)));
        }
    }
    if (lane == 0) {
        nbytes[2 * s] = nb[0];
        nbytes[2 * s + 1] = nb[1];
        lostflag[s] = lf;
        q.last[s] = t;
        u32* cnt = q.cnt + (size_t)s * RX_NCOUNT;
        cnt[rx_played_counter(n1, n2)]++;
        if (const int stale = rx_after_play(t, id, ln)) cnt[RX_DROPPED] += stale;
        q.len[2 * sl] = ln[0];
        q.len[2 * sl + 1] = ln[1];
    }
}

// reset (thread per listed stream; the host has checked the list): empty slots, zero counters, last = start - 1
__global__ void __launch_bounds__(SB_RX_THREADS) sb_rx_reset_kernel(RxDev q, const i32* __restrict__ streams, const u32* __restrict__ start, int n) {
    const int i = blockIdx.x * SB_RX_THREADS + threadIdx.x;
    if (i >= n) return;
    const i32 s = streams[i];
    q.last[s] = start[i] - 1u;
    for (int k = 0; k < RX_NCOUNT; k++) q.cnt[(size_t)s * RX_NCOUNT + k] = 0;
    for (int j = 0; j < 2 * q.depth; j++) q.len[(size_t)s * 2 * q.depth + j] = 0;
}

// ---- receive queue timing (sb_rx.cuh, solo_b200_rx_insert_timed_*) ------------------------------------------------------
// A timed insert runs the three insert passes unchanged, then its own kernels.  The margin histogram is order-free (an
// atomicAdd per arrival; it reads `last`, which no insert changes).  Jitter and highest are a recurrence over each stream's
// valid arrivals in array order: the call's arrivals are grouped by stream with a stable LSD radix sort of their positions
// (8-bit digits of the stream, ceil(log2 N / 8) passes of histogram, scan and scatter), then one thread per stream runs the
// recurrence over its group.  Arrivals the timing does not count are keyed to stream 0 with RX_KEY_SKIP set and skipped
// there.  Every step's result is fixed by the arrays alone, so nothing depends on scheduling.
struct RxTiming {
    u32 ts_per_index;
    int max_arrivals, passes;   // passes: 8-bit digits of the largest stream index
    u32* transit;               // [n] transit of the last valid arrival
    u32* jitter;                // [n] RFC 3550 jitter, 1/16 units
    unsigned long long* highest;// [n] cycles << 32 | highest index
    u32* received;              // [n] valid arrivals since the reset
    u32* margin;                // [n][RX_MARGIN_BINS]
    u32* key[2];                // [max_arrivals] sort keys (stream, or RX_KEY_SKIP), double-buffered
    u32* pos[2];                // [max_arrivals] arrival positions, double-buffered
    u32* hist;                  // [256][tiles] per tile digit counts, then their exclusive prefix in digit-major order
};
#define RX_KEY_SKIP 0x80000000u
#define SB_RX_SORT_THREADS 256  // one thread per digit value in the histogram and rank bookkeeping
#define SB_RX_SORT_ITEMS 8      // rounds of 256 arrivals per tile
#define SB_RX_SORT_TILE (SB_RX_SORT_THREADS * SB_RX_SORT_ITEMS)
__device__ __forceinline__ u32 rx_sort_digit(u32 key, int shift) { return ((key & ~RX_KEY_SKIP) >> shift) & 255u; }
__device__ __forceinline__ unsigned long long tx_warp_scan(unsigned long long v, int lane);   // send queue, below

// timed insert, pass 1 (thread per arrival): the sort key and position of each arrival, and its margin bin
__global__ void __launch_bounds__(SB_RX_THREADS) sb_rx_timing_keys_kernel(RxDev q, RxTiming T, RxArrivals A) {
    const int a = blockIdx.x * SB_RX_THREADS + threadIdx.x;
    if (a >= A.n) return;
    const i32 s = A.stream[a];
    const bool ok = rx_timed(q.n, q.desc_cap, s, A.desc[a], A.off[a], A.len[a], A.payload_bytes);
    T.key[0][a] = ok ? (u32)s : RX_KEY_SKIP;
    T.pos[0][a] = (u32)a;
    if (!ok) return;
    const int b = rx_margin_bin(A.index[a], q.last[s]);
    if (b >= 0) atomicAdd(&T.margin[(size_t)s * RX_MARGIN_BINS + b], 1u);
}

// sort pass, step 1 (block per tile): the tile's count of each digit, stored digit-major
__global__ void __launch_bounds__(SB_RX_SORT_THREADS) sb_rx_sort_hist_kernel(const u32* __restrict__ key, u32* __restrict__ hist, int n, int shift) {
    __shared__ u32 h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int base = blockIdx.x * SB_RX_SORT_TILE + threadIdx.x;
    for (int r = 0; r < SB_RX_SORT_ITEMS; r++) {
        const int i = base + r * SB_RX_SORT_THREADS;
        if (i < n) atomicAdd(&h[rx_sort_digit(key[i], shift)], 1u);
    }
    __syncthreads();
    hist[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = h[threadIdx.x];
}

// sort pass, step 2 (one block): the exclusive prefix of the `total` digit-major counts, in place.  Each thread sums a
// contiguous run of counts; the runs' sums are scanned as the send queue scans its block totals.
#define SB_RX_SCAN_THREADS 1024
__global__ void __launch_bounds__(SB_RX_SCAN_THREADS) sb_rx_sort_scan_kernel(u32* __restrict__ hist, int total) {
    __shared__ unsigned long long warp_total[SB_RX_SCAN_THREADS / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int per = (total + SB_RX_SCAN_THREADS - 1) / SB_RX_SCAN_THREADS;
    const int lo = imin((int)threadIdx.x * per, total), hi = imin(lo + per, total);
    unsigned long long x = 0;
    for (int i = lo; i < hi; i++) x += hist[i];
    const unsigned long long v = tx_warp_scan(x, lane);
    if (lane == 31) warp_total[w] = v;
    __syncthreads();
    unsigned long long base = 0;
    for (int i = 0; i < w; i++) base += warp_total[i];
    u32 run = (u32)(base + v - x);
    for (int i = lo; i < hi; i++) {
        const u32 c = hist[i];
        hist[i] = run;
        run += c;
    }
}

// sort pass, step 3 (block per tile): stable scatter of the tile's keys and positions to their digit's place.  Within a
// round of 256 arrivals, an arrival's rank among equal digits is the count in the warps before its own plus, from
// __match_any_sync, the count of lower lanes; the rounds run in order and carry each digit's running place.
__global__ void __launch_bounds__(SB_RX_SORT_THREADS) sb_rx_sort_scatter_kernel(const u32* __restrict__ kin, const u32* __restrict__ pin,
                                                                            u32* __restrict__ kout, u32* __restrict__ pout,
                                                                            const u32* __restrict__ hist, int n, int shift) {
    __shared__ u32 place[256];
    __shared__ u32 wcount[SB_RX_SORT_THREADS / 32][256];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    place[threadIdx.x] = hist[(size_t)threadIdx.x * gridDim.x + blockIdx.x];
    for (int k = 0; k < SB_RX_SORT_THREADS / 32; k++) wcount[k][threadIdx.x] = 0;
    __syncthreads();
    for (int r = 0; r < SB_RX_SORT_ITEMS; r++) {
        const int r0 = blockIdx.x * SB_RX_SORT_TILE + r * SB_RX_SORT_THREADS;
        if (r0 >= n) break;                       // uniform over the block
        const int i = r0 + threadIdx.x;
        const bool ok = i < n;
        const u32 key = ok ? kin[i] : 0u, p = ok ? pin[i] : 0u;
        const u32 dig = ok ? rx_sort_digit(key, shift) : 256u;
        const u32 peers = __match_any_sync(0xffffffffu, dig);
        const u32 below = __popc(peers & ((1u << lane) - 1u));
        if (ok && below == 0) wcount[w][dig] = __popc(peers);
        __syncthreads();
        if (ok) {
            u32 dst = place[dig] + below;
            for (int k = 0; k < w; k++) dst += wcount[k][dig];
            kout[dst] = key;
            pout[dst] = p;
        }
        __syncthreads();
        u32 t = 0;
        for (int k = 0; k < SB_RX_SORT_THREADS / 32; k++) {
            t += wcount[k][threadIdx.x];
            wcount[k][threadIdx.x] = 0;
        }
        place[threadIdx.x] += t;
        __syncthreads();
    }
}

// timed insert, last pass (thread per sorted arrival; the first of each stream's group works): the stream's valid
// arrivals in array order through rx_timing_step
__global__ void __launch_bounds__(SB_RX_THREADS) sb_rx_timing_walk_kernel(RxTiming T, const u32* __restrict__ K, const u32* __restrict__ P,
                                                                           RxArrivals A, const u32* __restrict__ arrival) {
    const int i = blockIdx.x * SB_RX_THREADS + threadIdx.x;
    if (i >= A.n) return;
    const u32 s = K[i] & ~RX_KEY_SKIP;
    if (i > 0 && (K[i - 1] & ~RX_KEY_SKIP) == s) return;
    u32 transit = T.transit[s], jitter = T.jitter[s], received = T.received[s];
    u64 highest = T.highest[s];
    bool any = false;
    for (int j = i; j < A.n; j++) {
        const u32 k = K[j];
        if ((k & ~RX_KEY_SKIP) != s) break;
        if (k & RX_KEY_SKIP) continue;
        const u32 a = P[j];
        rx_timing_step(A.index[a], arrival[a], T.ts_per_index, &transit, &jitter, &highest, &received);
        any = true;
    }
    if (!any) return;
    T.transit[s] = transit;
    T.jitter[s] = jitter;
    T.highest[s] = highest;
    T.received[s] = received;
}

// reset of the timing state (thread per listed stream; the host has checked the list)
__global__ void __launch_bounds__(SB_RX_THREADS) sb_rx_timing_reset_kernel(RxTiming T, const i32* __restrict__ streams, int n) {
    const int i = blockIdx.x * SB_RX_THREADS + threadIdx.x;
    if (i >= n) return;
    const i32 s = streams[i];
    T.transit[s] = 0;
    T.jitter[s] = 0;
    T.highest[s] = 0;
    T.received[s] = 0;
    for (int k = 0; k < RX_MARGIN_BINS; k++) T.margin[(size_t)s * RX_MARGIN_BINS + k] = 0;
}

// ---- send queue (sb_tx.cuh) ----------------------------------------------------------------------------------------------
// The queue's device arrays.  The scan words (bytes << 32 | datagrams) are scratch of the running pack: the sizes pass
// writes each stream's prefix within its block and each block's total, the scan pass turns the totals into the blocks'
// prefixes, the pack pass adds the two.
struct TxDev {
    int n;
    u32* next;                  // [n] index of the stream's next row
    u32* cnt;                   // [n][TX_NCOUNT]
    unsigned long long* pre;    // [n] scan word of the streams before s in its block
    unsigned long long* blk;    // [ceil(n / SB_TX_BLOCK)] block totals, then their exclusive prefix
};
struct TxOut {
    u8* payload; i32* stream; u32* index; u8* desc; i32* off; i32* len; i32* count; i64* total;
};

// inclusive scan of v over the warp
__device__ __forceinline__ unsigned long long tx_warp_scan(unsigned long long v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += y;
    }
    return v;
}

// pack, pass 1 (thread per stream): each row's datagrams and bytes, their exclusive prefix within the block (warp scans
// and the warps' totals in shared memory) and the block's total
__global__ void __launch_bounds__(SB_TX_BLOCK) sb_tx_sizes_kernel(TxDev q, const i16* __restrict__ nbytes, int cap) {
    __shared__ unsigned long long warp_total[SB_TX_BLOCK / 32];
    const int s = blockIdx.x * SB_TX_BLOCK + threadIdx.x, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int l1 = 0, l2 = 0;
    if (s < q.n) tx_row(nbytes[2 * s], nbytes[2 * s + 1], cap, &l1, &l2);
    const unsigned long long x = tx_scan_word(l1, l2), v = tx_warp_scan(x, lane);
    if (lane == 31) warp_total[w] = v;
    __syncthreads();
    unsigned long long base = 0, tot = 0;
#pragma unroll
    for (int i = 0; i < SB_TX_BLOCK / 32; i++) {
        const unsigned long long t = warp_total[i];
        base += i < w ? t : 0ull;
        tot += t;
    }
    if (s < q.n) q.pre[s] = base + v - x;
    if (threadIdx.x == 0) q.blk[blockIdx.x] = tot;
}

// pack, pass 2 (one block): the exclusive prefix of the block totals, SB_TX_SCAN_THREADS at a time in order, and the
// call's datagram count and byte total
#define SB_TX_SCAN_THREADS 1024
__global__ void __launch_bounds__(SB_TX_SCAN_THREADS) sb_tx_scan_kernel(TxDev q, int nblk, i32* __restrict__ count, i64* __restrict__ total) {
    __shared__ unsigned long long warp_total[SB_TX_SCAN_THREADS / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    unsigned long long carry = 0;
    for (int b0 = 0; b0 < nblk; b0 += SB_TX_SCAN_THREADS) {
        const int b = b0 + threadIdx.x;
        const unsigned long long x = b < nblk ? q.blk[b] : 0ull, v = tx_warp_scan(x, lane);
        if (lane == 31) warp_total[w] = v;
        __syncthreads();
        unsigned long long base = carry, tot = 0;
        for (int i = 0; i < SB_TX_SCAN_THREADS / 32; i++) {
            const unsigned long long t = warp_total[i];
            base += i < w ? t : 0ull;
            tot += t;
        }
        if (b < nblk) q.blk[b] = base + v - x;
        carry += tot;
        __syncthreads();                          // warp_total is rewritten by the next round
    }
    if (threadIdx.x == 0) {
        *count = tx_word_datagrams(carry);
        *total = tx_word_bytes(carry);
    }
}

// pack, pass 3 (warp per stream): the row's index and counters, its datagram entries, and its n0 bytes at payload offset
// b0.  The 16-byte words of payload that lie inside [b0, b0 + n0) get one 16-byte store each, built from two aligned
// 16-byte loads of the row (aligned: d_bits is, and cap is a multiple of 16) funnel-shifted by the stream's constant
// misalignment.  The partial words at both ends are shared with the neighbouring streams' datagrams: byte stores only.
#define SB_TX_PACK_WARPS 8
__global__ void __launch_bounds__(SB_TX_PACK_WARPS * 32) sb_tx_pack_kernel(TxDev q, const u8* __restrict__ bits, int cap,
                                                                            const i16* __restrict__ nbytes, TxOut o) {
    const int s = blockIdx.x * SB_TX_PACK_WARPS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (s >= q.n) return;                         // whole warps
    int l1, l2;
    const int cls = tx_row(nbytes[2 * s], nbytes[2 * s + 1], cap, &l1, &l2);
    const u32 idx = q.next[s];
    if (lane == 0) {
        q.next[s] = idx + 1u;
        tx_count(q.cnt + (size_t)s * TX_NCOUNT, cls, l1, l2);
    }
    if (cls != TX_SENT) return;
    const unsigned long long at = q.blk[s / SB_TX_BLOCK] + q.pre[s];
    const i32 k0 = tx_word_datagrams(at);
    const i64 b0 = tx_word_bytes(at), end = b0 + l1 + l2;
    if (lane < 2) {                               // lane d - 1: the entry of description d, when it is not empty
        const int len = lane ? l2 : l1;
        if (len > 0) {
            const i32 k = k0 + (lane && l1 > 0);
            o.stream[k] = s;
            o.index[k] = idx;
            o.desc[k] = (u8)(lane + 1);
            o.off[k] = (i32)(b0 + (lane ? l1 : 0));
            o.len[k] = len;
        }
    }
    const u8* row = bits + (size_t)s * cap;       // payload byte x is row byte x - b0
    const i64 h_end = end < ((b0 + 15) & ~15ll) ? end : ((b0 + 15) & ~15ll);
    const i64 t_beg = (end & ~15ll) > h_end ? (end & ~15ll) : h_end;
    {
        const i64 x = lane < 16 ? b0 + lane : t_beg + (lane - 16);
        if (x < (lane < 16 ? h_end : end)) o.payload[x] = row[x - b0];
    }
    const int mis = (int)((h_end - b0) & 15);     // the row offset of every full payload word, mod 16
    const int ws = mis >> 2, bs = (mis & 3) * 8;
    for (i64 x = h_end + 16 * lane; x < t_beg; x += 16 * 32) {
        const uint4* src = reinterpret_cast<const uint4*>(row + (x - b0 - mis));
        const uint4 a = src[0], b = mis ? src[1] : make_uint4(0, 0, 0, 0);
        const u32 v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        u32 r[5], w[4];
#pragma unroll
        for (int k = 0; k < 5; k++) r[k] = ws == 0 ? v[k] : ws == 1 ? v[k + 1] : ws == 2 ? v[k + 2] : v[k + 3];
#pragma unroll
        for (int k = 0; k < 4; k++) w[k] = __funnelshift_r(r[k], r[k + 1], bs);
        *reinterpret_cast<uint4*>(o.payload + x) = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

// reset (thread per listed stream; the host has checked the list): next = start, counters zero
__global__ void __launch_bounds__(SB_TX_BLOCK) sb_tx_reset_kernel(TxDev q, const i32* __restrict__ streams, const u32* __restrict__ start, int n) {
    const int i = blockIdx.x * SB_TX_BLOCK + threadIdx.x;
    if (i >= n) return;
    const i32 s = streams[i];
    q.next[s] = start[i];
    for (int k = 0; k < TX_NCOUNT; k++) q.cnt[(size_t)s * TX_NCOUNT + k] = 0;
}

// ---- downlink contributor lists (sb_tx.cuh), thread per member --------------------------------------------------------------
// Member position m (grid-stride over M = room_start[R]) finds its room by binary search and writes its stream's row.
// Rows of streams in no room were set to -1 / 127 by the caller's memsets; members outside [0, n) are skipped.
#define SB_CONTRIB_THREADS 256
__global__ void __launch_bounds__(SB_CONTRIB_THREADS) sb_mix_contributors_kernel(const i32* __restrict__ room_start, const i32* __restrict__ members,
                                                                                  int R, int k, const i32* __restrict__ talkers,
                                                                                  const u8* __restrict__ level, int n, i32* __restrict__ csrc,
                                                                                  u8* __restrict__ csrc_level) {
    const i32 M = room_start[R];
    for (i32 m = blockIdx.x * SB_CONTRIB_THREADS + threadIdx.x; m < M; m += gridDim.x * SB_CONTRIB_THREADS) {
        const i32 i = members[m];
        if ((u32)i >= (u32)n) continue;
        const int r = tx_room_of(room_start, R, m);
        tx_contributors(i, talkers + (size_t)r * k, k, level, n, csrc + (size_t)i * k, csrc_level + (size_t)i * k);
    }
}

// ---------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------
static thread_local char g_err[256] = "";
static std::mutex g_mu;
static long long g_launches = 0;
static int g_profile = 0;
// ---- sender / receiver glue around the payload row [MD1 | MD2 | HB] (SURVEY.md 8(f) rank 1) -----------------------------
// What the reference's decoder driver does between the network and AGR_Sate_Decoder_Decode (dec_main.c:245-307), for a whole
// batch on the device: lostflag 2 keeps MD1 only, 3 moves MD2 + HB to the front, 4 passes the row through, 1 (lost) leaves
// the row alone (the decoder does not read it).  One warp per row, 16-byte aligned rows when cap is a multiple of 16.
__global__ void __launch_bounds__(256) sb_apply_loss_kernel(const u8* __restrict__ bits_in, const i16* __restrict__ nb_in, const i32* __restrict__ flag,
                                                           u8* __restrict__ bits_out, i16* __restrict__ nb_out, int cap, int n) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (row >= n) return;
    const int n0 = nb_in[2 * row], n1 = nb_in[2 * row + 1], f = flag[row];
    int off = 0, len = n0, o0 = n0, o1 = n1;
    if (f == 2) { len = n0 - n1; o0 = len; o1 = 0; }
    else if (f == 3) { off = n0 - n1; len = n1; o0 = n1; o1 = 0; }
    // wire-supplied lengths: anything outside 0 <= n1 <= n0, off + len <= cap yields an empty row (the decoder rejects it)
    if (n0 < 0 || n1 < 0 || n1 > n0 || off < 0 || off > cap) { off = 0; len = 0; o0 = 0; o1 = 0; }
    if (len < 0) len = 0;
    if (len > cap) len = cap;
    if (len > cap - off) len = cap - off;
    const u8* src = bits_in + (size_t)row * cap + off;
    u8* dst = bits_out + (size_t)row * cap;
    for (int i = lane; i < len; i += 32) dst[i] = src[i];
    if (lane == 0) { nb_out[2 * row] = (i16)o0; nb_out[2 * row + 1] = (i16)o1; }
}

struct EvPair { cudaEvent_t a, b; int kind; };
static std::vector<EvPair> g_events;

static int fail(const char* what, cudaError_t e) {
    snprintf(g_err, sizeof g_err, "%s: %s", what, cudaGetErrorString(e));
    return -2;
}
#define CK(call)                                  \
    do {                                          \
        cudaError_t e_ = (call);                  \
        if (e_ != cudaSuccess) return fail(#call, e_); \
    } while (0)

static void prof_begin(cudaStream_t st, int kind, EvPair* p) {
    p->kind = -1;
    if (!g_profile) return;
    if (cudaEventCreate(&p->a) != cudaSuccess || cudaEventCreate(&p->b) != cudaSuccess) return;
    p->kind = kind;
    cudaEventRecord(p->a, st);
}
static void prof_end(cudaStream_t st, EvPair* p) {
    if (p->kind < 0) return;
    cudaEventRecord(p->b, st);
    std::lock_guard<std::mutex> lk(g_mu);
    g_events.push_back(*p);
}
// right after one kernel launch: count it and report a launch error under the kernel's name
static int launched(const char* kernel) {
    {
        std::lock_guard<std::mutex> lk(g_mu);
        g_launches++;
    }
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail(kernel, e);
}

// The stream list of a reset, export or import (the queues' and the codec batches'): true when its n entries are distinct
// streams of [0, N); otherwise false with g_err naming the first bad entry.
static bool streams_ok(const i32* streams, int n, int N, const char* who) {
    std::vector<u8> seen((size_t)N, 0);
    for (int i = 0; i < n; i++) {
        if (streams[i] < 0 || streams[i] >= N) { snprintf(g_err, sizeof g_err, "%s: stream %d outside [0, %d)", who, streams[i], N); return false; }
        if (seen[streams[i]]++) { snprintf(g_err, sizeof g_err, "%s: stream %d is listed twice", who, streams[i]); return false; }
    }
    return true;
}

// The device staging of one call of the mixer, queue, stream-membership, activity and set_control entry points, on the call's
// stream.  span() lays out the call's arrays: each gets a 16-byte-aligned place in one allocation, is copied in from `in`
// and back to `out` where those are not NULL, and its device address is written to `dev` when run() has allocated.  Copies back happen only when every
// earlier step succeeded, the launch's execution included.  finish() always frees, synchronises and returns the first error.
// With `kept`, the allocation is that buffer instead, grown when too small and never freed here: an object whose calls
// each end with a synchronise of their stream keeps one, so that its calls do not pay for an allocation from a memory
// pool that returns its memory at every synchronise.
struct DevBuf { u8* d = nullptr; size_t bytes = 0; };
struct Staging {
    struct Span { void** dev; const void* in; void* out; size_t bytes, off; };
    cudaStream_t st;
    const char* who;            // names the entry point in errors
    DevBuf* keep;
    std::vector<Span> spans;
    size_t size = 0;
    u8* d = nullptr;
    int r = 0;

    Staging(cudaStream_t stream, const char* name, DevBuf* kept = nullptr) : st(stream), who(name), keep(kept) {}
    bool alloc() {
        if (!keep) return ok(cudaMallocAsync(&d, size, st), who);
        if (keep->bytes < size) {
            if (keep->d) cudaFreeAsync(keep->d, st);
            *keep = DevBuf();
            if (!ok(cudaMallocAsync(&keep->d, size, st), who)) return false;
            keep->bytes = size;
        }
        d = keep->d;
        return true;
    }
    bool ok(cudaError_t e, const char* what) { if (!r && e != cudaSuccess) r = fail(what, e); return !r; }
    template <class T> void span(T*& dev, const void* in, void* out, size_t bytes) {
        spans.push_back({(void**)&dev, in, out, bytes, size});
        size += (bytes + 15) / 16 * 16;
    }
    bool sync() { return ok(cudaStreamSynchronize(st), who); }
    bool back(void* host, const void* dev, size_t bytes) { return !bytes || ok(cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, st), who); }
    // allocate, copy in, launch() (0 or the error it reported), then wait and copy back; false after any failure
    template <class F> bool run(F launch) {
        if (!alloc()) return false;
        for (Span& p : spans) *p.dev = d + p.off;
        for (Span& p : spans)
            if (p.in && p.bytes && !ok(cudaMemcpyAsync(d + p.off, p.in, p.bytes, cudaMemcpyHostToDevice, st), who)) return false;
        if ((r = launch())) return false;
        if (std::none_of(spans.begin(), spans.end(), [](const Span& p) { return p.out; })) return true;
        if (!sync()) return false;
        for (Span& p : spans)
            if (p.out && !back(p.out, d + p.off, p.bytes)) return false;
        return true;
    }
    int finish() {
        if (d && !keep) cudaFreeAsync(d, st);
        sync();
        return r;
    }
};

// A packet wave of a *_host call is cut into chunks of streams that run on the batch's CUDA streams: the copies of one chunk
// overlap the kernels of another, and the blocks of one chunk's kernel fill the SMs that the tail of another chunk's kernel
// leaves idle (all four kernels are latency-bound at a fixed number of resident warps per SM).  The *_device entry points
// launch every kernel once for the whole batch on the caller's stream.
#define SB_PIPE_STREAMS 4
static int g_chunks = -1;   // -1: SOLO_B200_CHUNKS or the default below
// Default: three chunks (the copies of one chunk hide behind the kernels of its neighbours; three beat two, four and six in
// an earlier comparison, not repeated on H100).
static int pipe_chunks(int n) {
    if (g_chunks < 0) {
        const char* e = getenv("SOLO_B200_CHUNKS");
        g_chunks = e ? atoi(e) : 0;
        if (g_chunks < 0) g_chunks = 0;
        if (g_chunks > 64) g_chunks = 64;
    }
    int c = g_chunks ? g_chunks : 3;
    while (c > 1 && n / c < 2048) c--;   // small batches: fewer, larger chunks
    return c;
}
// chunk c of C over n streams, boundaries on multiples of 64 streams (block size of the thread-per-stream kernels)
static void chunk_bounds(int n, int C, int c, int* lo, int* hi) {
    long long per = ((long long)n + C - 1) / C;
    per = (per + 63) / 64 * 64;
    long long a = per * c, b = per * (c + 1);
    *lo = (int)(a > n ? n : a);
    *hi = (int)(b > n ? n : b);
}

// What encoder and decoder batches share.  Batches are created value-initialised (every member zero), so the destructors
// also clean up after a partial create.
enum { WAVE_NONE = 0, WAVE_HOST, WAVE_DEVICE };
struct Batch {
    int n, device;
    int spp;                    // samples per packet and stream: 16 kHz 640 (40 ms) or 320 (20 ms), 32 kHz twice that
    int nf;                     // codec frames per packet: 2 (40 ms) or 1 (20 ms)
    int hb_bytes;               // high-band bytes per packet: 4 per high-band frame
    int wave;                   // entry point of the last packet wave of the batched API: WAVE_NONE, WAVE_HOST or WAVE_DEVICE
    int nst;                    // CUDA streams in st[]: SB_PIPE_STREAMS for a batch of the batched API, 1 for an arena segment
    cudaStream_t st[SB_PIPE_STREAMS];
    // staging for the *_host entry points and the arena
    i16* d_pcm; u8* d_bits; i16* d_nbytes; int bits_cap;
    DevBuf d_list;              // the Staging of reset / export / import, activity and set_control host calls (grown on use)
    ~Batch() {
        for (int i = 0; i < nst; i++) cudaStreamDestroy(st[i]);
        cudaFree(d_pcm); cudaFree(d_bits); cudaFree(d_nbytes); cudaFree(d_list.d);
    }
};
struct solo_b200_enc_batch : Batch {
    EncState* d_states;
    EncScratch* d_scratch;
    i16* d_bands;               // [n][spp]: low band | high band of the packet, written by the QMF kernel
    USER_Ctrl_enc ctrl;         // the create settings (targetRate_bps after the <= 0 -> 15600 rule), what a reset restores
    ~solo_b200_enc_batch() { cudaFree(d_states); cudaFree(d_scratch); cudaFree(d_bands); }
};
struct solo_b200_dec_batch : Batch {
    int khz;                    // SILK core rate: 8 (16 kHz streams, DecState) or 16 (32 kHz streams, DecState32)
    int core_only;              // 1: 32 kHz streams decoded to their 16 kHz core (spp = the core's rows, no band buffers)
    USER_Ctrl_dec ctrl;         // the create settings and arithmetic, what a reset restores
    int arith;
    void* d_states;             // DecStateT<khz>[n]
    DecStale* d_stale;          // payload copies that outlive a packet call (only touched after a corrupted packet, see sb_dec.cuh)
    i32* d_flags; i32* d_ret;   // staging for the *_host entry points and the arena
    i16* d_band_low; float* d_band_high; i32* d_ret_int;   // decoder kernel -> synthesis kernel (and activity kernel)
    u8* d_act_flags;            // [n]: decoder kernel -> activity kernel, the flags of each stream's last packet
    ~solo_b200_dec_batch() {
        cudaFree(d_states); cudaFree(d_stale); cudaFree(d_flags); cudaFree(d_ret);
        cudaFree(d_band_low); cudaFree(d_band_high); cudaFree(d_ret_int); cudaFree(d_act_flags);
    }
};

// Supported configurations (AGR_BWE_SDK_API.c:40-81): no joint coding with 40 or 20 ms packets ("40ms 2MD", "20ms 2MD");
// joint mode 1 (one 40 ms high-band frame per 40 ms packet).  Joint modes 0, 2, 3 are "Unsupport" in the reference as
// well.  16 kHz streams encode and decode; 32 kHz streams (AGR_BWE_SDK_API.c:86-94,196-200) only decode so far.
static int check_modes(int samplerate, int framesize_ms, int joint_enable, int joint_mode) {
    if (samplerate != 16000 && samplerate != 32000) return -1;
    if (!joint_enable) return (framesize_ms == 40 || framesize_ms == 20) ? 0 : -1;
    return (joint_mode == 1 && framesize_ms == 40) ? 0 : -1;
}
static int check_enc_ctrl(const USER_Ctrl_enc* c) {
    if (c && c->samplerate == 32000) { snprintf(g_err, sizeof g_err, "the 32 kHz encoder is not built yet (32 kHz streams can only be decoded)"); return -1; }
    if (!c || check_modes(c->samplerate, c->framesize_ms, c->joint_enable, c->joint_mode)) { snprintf(g_err, sizeof g_err, "bad encoder configuration"); return -1; }
    return 0;
}
static int check_dec_ctrl(const USER_Ctrl_dec* c) { return c ? check_modes(c->samplerate, c->framesize_ms, c->joint_enable, c->joint_mode) : -1; }
static int hb_bytes_of(int framesize_ms, int joint_enable) { return joint_enable ? 4 : 4 * (framesize_ms / 20); }

static int require_gpu(int device) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count <= 0) {
        snprintf(g_err, sizeof g_err, "no CUDA device available (%s): libsolo_b200 has no CPU fallback",
                 e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
        return -2;
    }
    if (device < 0 || device >= count) { snprintf(g_err, sizeof g_err, "bad device ordinal %d", device); return -1; }
    CK(cudaSetDevice(device));
    return 0;
}

// the packet layout and `nst` CUDA streams of a new batch; false when a stream cannot be created
static bool batch_setup(Batch* b, int n, int device, int samplerate, int framesize_ms, int joint_enable, int nst) {
    b->n = n; b->device = device; b->spp = samplerate / 1000 * framesize_ms; b->nf = framesize_ms / 20; b->hb_bytes = hb_bytes_of(framesize_ms, joint_enable);
    for (; b->nst < nst; b->nst++)
        if (cudaStreamCreateWithFlags(&b->st[b->nst], cudaStreamNonBlocking) != cudaSuccess) return false;
    return true;
}
template <class B> static B* batch_destroy(B* b) {
    if (!b) return nullptr;
    cudaSetDevice(b->device);
    for (int i = 0; i < b->nst; i++) cudaStreamSynchronize(b->st[i]);
    delete b;
    return nullptr;
}

// staging allocated on first use; the payload rows grow with `cap`.  The *_host calls copy whole rows back, so the payload
// rows start zeroed: bytes past a packet are then a function of the stream's history, never of what the memory held before.
static int staging(Batch* b, int cap) {
    if (!b->d_pcm) CK(cudaMalloc(&b->d_pcm, sizeof(i16) * b->spp * (size_t)b->n));
    if (!b->d_nbytes) CK(cudaMalloc(&b->d_nbytes, sizeof(i16) * 2 * (size_t)b->n));
    if (!b->d_bits || b->bits_cap < cap) {
        if (b->d_bits) cudaFree(b->d_bits);
        b->d_bits = nullptr;
        CK(cudaMalloc(&b->d_bits, (size_t)cap * b->n));
        b->bits_cap = cap;
        CK(cudaMemsetAsync(b->d_bits, 0, (size_t)cap * b->n, b->st[0]));
        CK(cudaStreamSynchronize(b->st[0]));    // the batch's other streams do not wait for st[0]
    }
    return 0;
}
static int dec_staging(solo_b200_dec_batch* b, int cap) {
    if (!b->d_flags) CK(cudaMalloc(&b->d_flags, sizeof(i32) * (size_t)b->n));
    if (!b->d_ret) CK(cudaMalloc(&b->d_ret, sizeof(i32) * (size_t)b->n));
    return staging(b, cap);
}

// The wave of a *_host call: f(lo, hi, stream) enqueues the copies and kernels of streams [lo, hi).  Chunks alternate over
// the batch's CUDA streams; the call returns when all of them are done.
template <class F> static int host_chunks(Batch* b, F f) {
    const int C = pipe_chunks(b->n);
    const int S = C < b->nst ? C : b->nst;
    for (int c = 0; c < C; c++) {
        int lo, hi;
        chunk_bounds(b->n, C, c, &lo, &hi);
        if (hi <= lo) continue;
        int r = f(lo, hi, b->st[c % S]);
        if (r) return r;
    }
    for (int i = 0; i < S; i++) CK(cudaStreamSynchronize(b->st[i]));
    return 0;
}

// ---- stream state hand-over (checkpoint / migration, SURVEY.md 8(f) rank 3) ----------------------------------------------
static size_t state_stride(const solo_b200_enc_batch*) { return sizeof(EncState); }
static size_t state_stride(const solo_b200_dec_batch* b) { return b->khz == 16 ? sizeof(DecState32) : sizeof(DecState); }
// blob_bytes: the caller's blob size, or -1 when the caller did not say (the unsized entry points)
template <class B> static int state_copy(B* b, int idx, void* host, int to_host, long long blob_bytes = -1) {
    if (!b || !host || idx < 0 || idx >= b->n) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    const size_t stride = state_stride(b);
    if (blob_bytes >= 0 && (size_t)blob_bytes != stride) {
        snprintf(g_err, sizeof g_err, "state blob of %lld bytes, this batch's streams have %zu (a stream of another sample rate?)", blob_bytes, stride);
        return -1;
    }
    CK(cudaSetDevice(b->device));
    CK(cudaDeviceSynchronize());    // packet waves run on the batch's streams and on caller streams: wait for all of them
    char* p = (char*)b->d_states + stride * (size_t)idx;
    if (to_host) CK(cudaMemcpy(host, p, stride, cudaMemcpyDeviceToHost));
    else CK(cudaMemcpy(p, host, stride, cudaMemcpyHostToDevice));
    return 0;
}

// ---- activity reports of the last packet wave (sb_activity.cuh) -------------------------------------------------------
// the activity kernel over streams [lo, lo + n) on st: `pcm` is the wave's PCM matrix (row 0 = stream 0); the encoder's
// flags come from its scratch, the decoder's from the bytes and return codes its decode kernel left
static int activity_launch(const solo_b200_enc_batch* b, int lo, int n, const i16* pcm, u8* level, u8* flags, cudaStream_t st) {
    sb_activity_kernel<<<(n + SB_ACT_WARPS - 1) / SB_ACT_WARPS, SB_ACT_WARPS * 32, 0, st>>>(pcm + (size_t)lo * b->spp, b->spp, b->nf, b->d_scratch + lo,
                                                                                         nullptr, nullptr, level, flags, n);
    return launched("sb_activity_kernel");
}
static int activity_launch(const solo_b200_dec_batch* b, int lo, int n, const i16* pcm, u8* level, u8* flags, cudaStream_t st) {
    sb_activity_kernel<<<(n + SB_ACT_WARPS - 1) / SB_ACT_WARPS, SB_ACT_WARPS * 32, 0, st>>>(pcm + (size_t)lo * b->spp, b->spp, b->nf, nullptr,
                                                                                         b->d_act_flags + lo, b->d_ret_int + lo, level, flags, n);
    return launched("sb_activity_kernel");
}
// the report of streams [lo, lo + n) from the staged PCM rows into host arrays of n entries, on the batch's first CUDA
// stream; returns when the arrays are filled
template <class B> static int activity_host(B* b, int lo, int n, u8* level, u8* flags) {
    cudaStream_t st = b->st[0];
    u8 *d_level, *d_flags;
    Staging s(st, "activity_host", &b->d_list);
    s.span(d_level, nullptr, level, (size_t)n);
    s.span(d_flags, nullptr, flags, (size_t)n);
    s.run([&] { return activity_launch(b, lo, n, b->d_pcm, d_level, d_flags, st); });
    return s.finish();
}
// the activity entry point of kind `want` (WAVE_HOST / WAVE_DEVICE) reports on a last wave of the same kind only: the
// other kind's PCM rows are not where it looks
static int activity_wave_check(const Batch* b, int want) {
    if (b->wave == want) return 0;
    snprintf(g_err, sizeof g_err, "%s", b->wave == WAVE_NONE ? "activity: the batch has not run a packet wave yet"
                                        : want == WAVE_HOST ? "activity_host: the last packet wave was a *_device call"
                                                            : "activity_device: the last packet wave was a *_host call");
    return -1;
}
// solo_b200_{enc,dec}_batch_activity_host / _device
template <class B> static int batch_activity_host(B* b, u8* level, u8* flags) {
    if (!b || !level || !flags) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    if (activity_wave_check(b, WAVE_HOST)) return -1;
    CK(cudaSetDevice(b->device));
    return activity_host(b, 0, b->n, level, flags);
}
template <class B> static int batch_activity_device(B* b, const i16* d_pcm, u8* d_level, u8* d_flags, void* cuda_stream) {
    if (!b || !d_pcm || !d_level || !d_flags) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    if (activity_wave_check(b, WAVE_DEVICE)) return -1;
    CK(cudaSetDevice(b->device));
    return activity_launch(b, 0, b->n, d_pcm, d_level, d_flags, (cudaStream_t)cuda_stream);
}

extern "C" {

const char* solo_b200_last_error(void) { return g_err; }
long long solo_b200_kernel_launches(void) { std::lock_guard<std::mutex> lk(g_mu); return g_launches; }
int solo_b200_enc_state_bytes(void) { return (int)sizeof(EncState); }
int solo_b200_dec_state_bytes(void) { return (int)sizeof(DecState); }
int solo_b200_dec_state_bytes_rate(int samplerate) {
    return samplerate == 16000 ? (int)sizeof(DecState) : samplerate == 32000 ? (int)sizeof(DecState32) : -1;
}
void solo_b200_set_chunks(int chunks) { g_chunks = chunks < 0 ? 0 : (chunks > 64 ? 64 : chunks); }   // 0: the default
void solo_b200_profile_enable(int on) {
    std::lock_guard<std::mutex> lk(g_mu);
    g_profile = on;
    for (auto& p : g_events) { cudaEventDestroy(p.a); cudaEventDestroy(p.b); }
    g_events.clear();
}
int solo_b200_profile_read(double* ms_total, long long* launches) {
    // index 0 = encoder analysis kernel, 1 = encoder NSQ kernel, 2 = encoder finish kernel, 3 = decode kernel
    std::lock_guard<std::mutex> lk(g_mu);
    double t[4] = {0, 0, 0, 0}; long long c[4] = {0, 0, 0, 0};
    for (auto& p : g_events) {
        if (cudaEventSynchronize(p.b) != cudaSuccess) continue;
        float ms = 0;
        if (cudaEventElapsedTime(&ms, p.a, p.b) == cudaSuccess) { t[p.kind] += ms; c[p.kind]++; }
        cudaEventDestroy(p.a); cudaEventDestroy(p.b);
    }
    g_events.clear();
    for (int i = 0; i < 4; i++) { if (ms_total) ms_total[i] = t[i]; if (launches) launches[i] = c[i]; }
    return 0;
}

// ---- encoder batch --------------------------------------------------------------------------------
// (re)initialise streams [lo, lo + n) of an encoder batch on its first CUDA stream, with ctrl's rate (> 0), DTX and MD index
static int enc_init_launch(solo_b200_enc_batch* b, int lo, int n, const USER_Ctrl_enc* ctrl) {
    sb_enc_init_kernel<<<(n + SB_TPB - 1) / SB_TPB, SB_TPB, 0, b->st[0]>>>(b->d_states + lo, n, ctrl->targetRate_bps, ctrl->dtx_enable, ctrl->useMDIndex,
                                                                          ctrl->framesize_ms, ctrl->joint_enable ? 1 : 0);
    return launched("sb_enc_init_kernel");
}
static solo_b200_enc_batch* enc_batch_create_impl(int n_streams, const USER_Ctrl_enc* ctrl, int device, int nst) {
    if (n_streams <= 0) { snprintf(g_err, sizeof g_err, "bad encoder configuration"); return nullptr; }
    if (check_enc_ctrl(ctrl)) return nullptr;
    if (require_gpu(device)) return nullptr;
    solo_b200_enc_batch* b = new solo_b200_enc_batch();
    // the kernels' shared-memory limits are attributes of the device that require_gpu selected
    if (!batch_setup(b, n_streams, device, ctrl->samplerate, ctrl->framesize_ms, ctrl->joint_enable, nst) ||
        cudaMalloc(&b->d_states, sizeof(EncState) * (size_t)n_streams) != cudaSuccess ||
        cudaMalloc(&b->d_scratch, sizeof(EncScratch) * (size_t)n_streams) != cudaSuccess ||
        cudaMalloc(&b->d_bands, sizeof(i16) * (size_t)b->spp * (size_t)n_streams) != cudaSuccess ||
        cudaFuncSetAttribute(sb_enc_nsq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(SB_NSQ_SPB * sizeof(NsqSmem))) != cudaSuccess ||
        sb_enc_analysis_setup() != cudaSuccess) {
        fail("enc_batch_create", cudaGetLastError());
        return batch_destroy(b);
    }
    b->ctrl = *ctrl;
    if (b->ctrl.targetRate_bps <= 0) b->ctrl.targetRate_bps = 15600;
    if (enc_init_launch(b, 0, n_streams, &b->ctrl)) return batch_destroy(b);
    cudaError_t e = cudaStreamSynchronize(b->st[0]);
    if (e != cudaSuccess) { fail("enc init kernel", e); return batch_destroy(b); }
    return b;
}
solo_b200_enc_batch* solo_b200_enc_batch_create(int n_streams, const USER_Ctrl_enc* ctrl, int device) { return enc_batch_create_impl(n_streams, ctrl, device, SB_PIPE_STREAMS); }

// PCM rows in another GPU's memory (peer ingest) are read with ordinary loads over NVLink; the bulk-copy engine path is for
// rows in this GPU's HBM
static int pcm_is_local(int device, const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return 1; }
    return (a.type == cudaMemoryTypeDevice && a.device != device) ? 0 : 1;
}

// the encoder kernels (A0, A, B, C) for streams [lo, lo + n) on one CUDA stream
static int enc_launch(solo_b200_enc_batch* b, int lo, int n, const i16* d_pcm, u8* d_bits, int cap, i16* d_nbytes, cudaStream_t st) {
    if (n <= 0) return 0;
    EncState* states = b->d_states + lo;
    EncScratch* scratch = b->d_scratch + lo;
    const i16* pcm = d_pcm + (size_t)lo * b->spp;
    EvPair ev;
    prof_begin(st, 0, &ev);
    i16* bands = b->d_bands + (size_t)lo * b->spp;
    sb_enc_qmf_kernel<<<(n + SB_QMF_SPB - 1) / SB_QMF_SPB, SB_QMF_SPB * 32, 0, st>>>(states, pcm, bands, b->spp, n, pcm_is_local(b->device, pcm));
    if (int e = launched("sb_enc_qmf_kernel")) return e;
    sb_enc_vad_kernel<<<(n + SB_TPB - 1) / SB_TPB, SB_TPB, 0, st>>>(states, scratch, bands, b->spp, n);
    if (int e = launched("sb_enc_vad_kernel")) return e;
    sb_launch_enc_hb_warp(states, scratch, bands, b->spp, n, st);
    if (int e = launched("sb_enc_hb_warp_kernel")) return e;
    sb_launch_enc_analysis_warp(states, scratch, bands, b->spp, n, st);
    if (int e = launched("sb_enc_analysis_warp_kernel")) return e;
    sb_enc_shape_post_kernel<<<(8 * n + 127) / 128, 128, 0, st>>>(states, scratch, n);
    if (int e = launched("sb_enc_shape_post_kernel")) return e;
    sb_enc_prefilter_kernel<<<dim3((n + SB_TPB - 1) / SB_TPB, 2), SB_TPB, 0, st>>>(states, scratch, n);
    if (int e = launched("sb_enc_prefilter_kernel")) return e;
    prof_end(st, &ev);
    prof_begin(st, 1, &ev);
    sb_enc_nsq_kernel<<<(n + SB_NSQ_SPB - 1) / SB_NSQ_SPB, SB_NSQ_WARPS * 32, SB_NSQ_SPB * sizeof(NsqSmem), st>>>(states, scratch, n);
    if (int e = launched("sb_enc_nsq_kernel")) return e;
    prof_end(st, &ev);
    prof_begin(st, 2, &ev);
    sb_enc_finish_kernel<<<(2 * n + SB_TPB - 1) / SB_TPB, SB_TPB, 0, st>>>(states, scratch, d_bits + (size_t)lo * cap, cap, d_nbytes + 2 * (size_t)lo, n);
    if (int e = launched("sb_enc_finish_kernel")) return e;
    prof_end(st, &ev);
    return 0;
}

int solo_b200_enc_batch_encode_device(solo_b200_enc_batch* b, const int16_t* d_pcm, uint8_t* d_bits, int cap, int16_t* d_nbytes, void* cuda_stream) {
    if (!b || !d_pcm || !d_bits || !d_nbytes || cap < 16) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    CK(cudaSetDevice(b->device));
    b->wave = WAVE_DEVICE;
    return enc_launch(b, 0, b->n, d_pcm, d_bits, cap, d_nbytes, (cudaStream_t)cuda_stream);
}

// streams [lo, lo + m) through the batch's staging on st: PCM rows in, the encoder kernels, payload rows and lengths out.
// The host arrays start at row lo; the caller waits for st.
static int enc_host_range(solo_b200_enc_batch* b, int lo, int m, const i16* pcm, u8* bits, int cap, i16* nbytes, cudaStream_t st) {
    CK(cudaMemcpyAsync(b->d_pcm + (size_t)lo * b->spp, pcm, sizeof(i16) * b->spp * (size_t)m, cudaMemcpyHostToDevice, st));
    if (int e = enc_launch(b, lo, m, b->d_pcm, b->d_bits, cap, b->d_nbytes, st)) return e;
    CK(cudaMemcpyAsync(bits, b->d_bits + (size_t)lo * cap, (size_t)cap * m, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(nbytes, b->d_nbytes + 2 * (size_t)lo, sizeof(i16) * 2 * (size_t)m, cudaMemcpyDeviceToHost, st));
    return 0;
}

int solo_b200_enc_batch_encode_host(solo_b200_enc_batch* b, const int16_t* pcm, uint8_t* bits, int cap, int16_t* nbytes) {
    if (!b || !pcm || !bits || !nbytes || cap < 16) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    CK(cudaSetDevice(b->device));
    int r = staging(b, cap);
    if (r) return r;
    b->wave = WAVE_HOST;
    return host_chunks(b, [&](int lo, int hi, cudaStream_t st) {
        return enc_host_range(b, lo, hi - lo, pcm + (size_t)lo * b->spp, bits + (size_t)lo * cap, cap, nbytes + 2 * (size_t)lo, st);
    });
}

// ---- per-stream rate / DTX / expected loss between packets (enc_set_control) ----------------------------------------------
// What the host entry points accept: -1 (leave the setting alone), rate >= 1, dtx 0 or 1, loss 0-100.  A NULL array is fine.
static bool control_in_range(const i32* rate, const i32* dtx, const i32* loss, int n) {
    for (int i = 0; i < n; i++) {
        if (rate && rate[i] != -1 && rate[i] < 1) return false;
        if (dtx && dtx[i] != -1 && dtx[i] != 0 && dtx[i] != 1) return false;
        if (loss && loss[i] != -1 && (loss[i] < 0 || loss[i] > 100)) return false;
    }
    return true;
}
// the control kernel for streams [lo, lo + n); the arrays hold those n streams' entries
static int enc_control_launch(solo_b200_enc_batch* b, int lo, int n, const i32* d_rate, const i32* d_dtx, const i32* d_loss, cudaStream_t st) {
    sb_enc_control_kernel<<<(n + SB_TPB - 1) / SB_TPB, SB_TPB, 0, st>>>(b->d_states + lo, n, d_rate, d_dtx, d_loss);
    return launched("sb_enc_control_kernel");
}
// host arrays of streams [lo, lo + n) through the batch's staging into the control kernel on st; returns when it is done
static int enc_control_host(solo_b200_enc_batch* b, int lo, int n, const i32* rate, const i32* dtx, const i32* loss, cudaStream_t st) {
    const i32 *d_rate = nullptr, *d_dtx = nullptr, *d_loss = nullptr;
    Staging s(st, "set_control", &b->d_list);
    if (rate) s.span(d_rate, rate, nullptr, 4 * (size_t)n);
    if (dtx) s.span(d_dtx, dtx, nullptr, 4 * (size_t)n);
    if (loss) s.span(d_loss, loss, nullptr, 4 * (size_t)n);
    s.run([&] { return enc_control_launch(b, lo, n, d_rate, d_dtx, d_loss, st); });
    return s.finish();
}

int solo_b200_enc_batch_set_control_device(solo_b200_enc_batch* b, const int32_t* d_rate_bps, const int32_t* d_dtx, const int32_t* d_loss_perc, void* cuda_stream) {
    if (!b) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    CK(cudaSetDevice(b->device));
    if (!d_rate_bps && !d_dtx && !d_loss_perc) return 0;
    return enc_control_launch(b, 0, b->n, d_rate_bps, d_dtx, d_loss_perc, (cudaStream_t)cuda_stream);
}

int solo_b200_enc_batch_set_control_host(solo_b200_enc_batch* b, const int32_t* rate_bps, const int32_t* dtx, const int32_t* loss_perc) {
    if (!b) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    if (!control_in_range(rate_bps, dtx, loss_perc, b->n)) { snprintf(g_err, sizeof g_err, "set_control: a setting is out of range"); return -1; }
    CK(cudaSetDevice(b->device));
    CK(cudaDeviceSynchronize());    // after the packet waves already enqueued, on the batch's streams and on caller streams
    return enc_control_host(b, 0, b->n, rate_bps, dtx, loss_perc, b->st[0]);
}

void solo_b200_enc_batch_destroy(solo_b200_enc_batch* b) { batch_destroy(b); }

// ---- decoder batch --------------------------------------------------------------------------------
// The fixed-point build decodes two SILK frames per call whatever the packet length (AGR_BWE_decode_frame_FIX.c:173,
// HB2LB_NUM = 2), so with 20 ms packets it decodes every payload twice: that defect is not reproduced, 20 ms is refused.
static int check_dec_arith(const USER_Ctrl_dec* c, int arith) {
    if (arith != SOLO_B200_DEC_FLP && arith != SOLO_B200_DEC_FIX) { snprintf(g_err, sizeof g_err, "bad decoder arithmetic %d", arith); return -1; }
    if (arith == SOLO_B200_DEC_FIX && c && c->framesize_ms == 20) {
        snprintf(g_err, sizeof g_err, "fixed-point decoding of 20 ms packets is not supported");
        return -1;
    }
    return 0;
}
// (re)initialise streams [lo, lo + n) of a decoder batch on its first CUDA stream
static int dec_init_launch(solo_b200_dec_batch* b, int lo, int n, int mdi, int framesize_ms, int joint_enable, int arith) {
    const int g = (n + SB_TPB - 1) / SB_TPB, joint = joint_enable ? 1 : 0;
    if (b->khz == 16) sb_dec_init_kernel<16><<<g, SB_TPB, 0, b->st[0]>>>((DecState32*)b->d_states + lo, n, mdi, framesize_ms, joint, arith, b->core_only);
    else sb_dec_init_kernel<8><<<g, SB_TPB, 0, b->st[0]>>>((DecState*)b->d_states + lo, n, mdi, framesize_ms, joint, arith, 0);
    return launched("sb_dec_init_kernel");
}
// out_samplerate: ctrl->samplerate, or 16000 for 32 kHz streams decoded to their 16 kHz core
static solo_b200_dec_batch* dec_batch_create_impl(int n_streams, const USER_Ctrl_dec* ctrl, int device, int nst, int arith, int out_samplerate) {
    if (n_streams <= 0 || check_dec_ctrl(ctrl)) { snprintf(g_err, sizeof g_err, "bad decoder configuration"); return nullptr; }
    if (check_dec_arith(ctrl, arith)) return nullptr;
    const int core_only = ctrl->samplerate == 32000 && out_samplerate == 16000;
    if (out_samplerate != ctrl->samplerate && !core_only) {
        snprintf(g_err, sizeof g_err, "bad decoder output rate %d for %d Hz streams (the stream's rate, or 16000 for 32000)", out_samplerate, ctrl->samplerate);
        return nullptr;
    }
    if (require_gpu(device)) return nullptr;
    solo_b200_dec_batch* b = new solo_b200_dec_batch();
    b->khz = ctrl->samplerate == 32000 ? 16 : 8;
    b->core_only = core_only;
    b->ctrl = *ctrl;
    b->arith = arith;
    const size_t band = core_only ? 0 : (size_t)ctrl->samplerate / 2000 * ctrl->framesize_ms;   // samples per band and packet
    if (!batch_setup(b, n_streams, device, out_samplerate, ctrl->framesize_ms, ctrl->joint_enable, nst) ||
        cudaMalloc(&b->d_states, state_stride(b) * (size_t)n_streams) != cudaSuccess ||
        cudaMalloc(&b->d_stale, sizeof(DecStale) * (size_t)n_streams) != cudaSuccess ||
        (band && cudaMalloc(&b->d_band_low, sizeof(i16) * band * (size_t)n_streams) != cudaSuccess) ||
        (band && cudaMalloc(&b->d_band_high, sizeof(float) * band * (size_t)n_streams) != cudaSuccess) ||
        cudaMalloc(&b->d_ret_int, sizeof(i32) * (size_t)n_streams) != cudaSuccess ||
        cudaMalloc(&b->d_act_flags, (size_t)n_streams) != cudaSuccess) {
        fail("dec_batch_create", cudaGetLastError());
        return batch_destroy(b);
    }
    if (dec_init_launch(b, 0, n_streams, ctrl->useMDIndex, ctrl->framesize_ms, ctrl->joint_enable, arith)) return batch_destroy(b);
    cudaError_t e = cudaStreamSynchronize(b->st[0]);
    if (e != cudaSuccess) { fail("dec init kernel", e); return batch_destroy(b); }
    return b;
}
solo_b200_dec_batch* solo_b200_dec_batch_create(int n_streams, const USER_Ctrl_dec* ctrl, int device) {
    return dec_batch_create_impl(n_streams, ctrl, device, SB_PIPE_STREAMS, SOLO_B200_DEC_FLP, ctrl ? ctrl->samplerate : 0);
}
solo_b200_dec_batch* solo_b200_dec_batch_create_arith(int n_streams, const USER_Ctrl_dec* ctrl, int device, int arith) {
    return dec_batch_create_impl(n_streams, ctrl, device, SB_PIPE_STREAMS, arith, ctrl ? ctrl->samplerate : 0);
}
solo_b200_dec_batch* solo_b200_dec_batch_create_out(int n_streams, const USER_Ctrl_dec* ctrl, int device, int arith, int out_samplerate) {
    return dec_batch_create_impl(n_streams, ctrl, device, SB_PIPE_STREAMS, arith, out_samplerate);
}

// the decoder kernels of core rate KHZ for streams [lo, lo + n) of b: decode and synthesis, or the core-output decode alone;
// the first launch error
extern "C++" {
template <int KHZ>
static int dec_kernels(solo_b200_dec_batch* b, int lo, int n, i16* d_pcm, const u8* d_bits, int cap, const i16* d_nbytes, const i32* d_lostflag,
                       i32* d_ret, cudaStream_t st) {
    DecStateT<KHZ>* states = (DecStateT<KHZ>*)b->d_states + lo;
    // core output: the PCM rows (b->spp samples) are the low band of 2 * b->spp-sample packets
    if constexpr (KHZ == 16) if (b->core_only) {
        sb_decode_kernel<KHZ, true><<<(n + SB_DEC_TPB - 1) / SB_DEC_TPB, SB_DEC_TPB, 0, st>>>(states, d_bits + (size_t)lo * cap, cap, d_nbytes + 2 * (size_t)lo,
                                                                                    d_lostflag + lo, d_ret ? d_ret + lo : nullptr, b->d_ret_int + lo,
                                                                                    b->d_act_flags + lo, b->d_stale + lo, d_pcm + (size_t)lo * b->spp,
                                                                                    nullptr, 2 * b->spp, n);
        return launched("sb_decode_kernel");
    }
    const size_t half = (size_t)(b->spp / 2);
    sb_decode_kernel<KHZ><<<(n + SB_DEC_TPB - 1) / SB_DEC_TPB, SB_DEC_TPB, 0, st>>>(states, d_bits + (size_t)lo * cap, cap, d_nbytes + 2 * (size_t)lo, d_lostflag + lo,
                                                                       d_ret ? d_ret + lo : nullptr, b->d_ret_int + lo, b->d_act_flags + lo, b->d_stale + lo,
                                                                       b->d_band_low + (size_t)lo * half, b->d_band_high + (size_t)lo * half, b->spp, n);
    if (int e = launched("sb_decode_kernel")) return e;
    sb_dec_synth_kernel<KHZ><<<(n + SB_SYN_WARPS - 1) / SB_SYN_WARPS, SB_SYN_WARPS * 32, 0, st>>>(states, b->d_band_low + (size_t)lo * half, b->d_band_high + (size_t)lo * half,
                                                                                               b->d_ret_int + lo, d_pcm + (size_t)lo * b->spp, b->spp, n);
    return launched("sb_dec_synth_kernel");
}
}  // extern "C++"
static int dec_launch(solo_b200_dec_batch* b, int lo, int n, i16* d_pcm, const u8* d_bits, int cap, const i16* d_nbytes, const i32* d_lostflag,
                      i32* d_ret, cudaStream_t st) {
    if (n <= 0) return 0;
    EvPair ev; prof_begin(st, 3, &ev);
    const int r = b->khz == 16 ? dec_kernels<16>(b, lo, n, d_pcm, d_bits, cap, d_nbytes, d_lostflag, d_ret, st)
                               : dec_kernels<8>(b, lo, n, d_pcm, d_bits, cap, d_nbytes, d_lostflag, d_ret, st);
    prof_end(st, &ev);
    return r;
}

int solo_b200_dec_batch_decode_device(solo_b200_dec_batch* b, int16_t* d_pcm, const uint8_t* d_bits, int cap, const int16_t* d_nbytes,
                                      const int32_t* d_lostflag, int32_t* d_ret, void* cuda_stream) {
    if (!b || !d_pcm || !d_bits || !d_nbytes || !d_lostflag || cap < 16) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    // full-band rows are written by the synthesis kernel's 8-byte stores; core-output rows take any 2-byte alignment
    const uintptr_t align = b->core_only ? 2 : 8;
    if ((uintptr_t)d_pcm % align) {
        snprintf(g_err, sizeof g_err, "decode_device: d_pcm must be %d-byte aligned (%s rows)", (int)align, b->core_only ? "core-output" : "full-band");
        return -1;
    }
    CK(cudaSetDevice(b->device));
    b->wave = WAVE_DEVICE;
    return dec_launch(b, 0, b->n, d_pcm, d_bits, cap, d_nbytes, d_lostflag, d_ret, (cudaStream_t)cuda_stream);
}

// streams [lo, lo + m) through the batch's staging on st: payload rows, lengths and loss flags in, the decoder kernels, PCM
// rows and (ret != NULL) return codes out.  The host arrays start at row lo; the caller waits for st.
static int dec_host_range(solo_b200_dec_batch* b, int lo, int m, i16* pcm, const u8* bits, int cap, const i16* nbytes, const i32* lostflag,
                          i32* ret, cudaStream_t st) {
    const size_t r = (size_t)m;
    CK(cudaMemcpyAsync(b->d_bits + (size_t)lo * cap, bits, (size_t)cap * r, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(b->d_nbytes + 2 * (size_t)lo, nbytes, sizeof(i16) * 2 * r, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(b->d_flags + lo, lostflag, sizeof(i32) * r, cudaMemcpyHostToDevice, st));
    if (int e = dec_launch(b, lo, m, b->d_pcm, b->d_bits, cap, b->d_nbytes, b->d_flags, b->d_ret, st)) return e;
    CK(cudaMemcpyAsync(pcm, b->d_pcm + (size_t)lo * b->spp, sizeof(i16) * b->spp * r, cudaMemcpyDeviceToHost, st));
    if (ret) CK(cudaMemcpyAsync(ret, b->d_ret + lo, sizeof(i32) * r, cudaMemcpyDeviceToHost, st));
    return 0;
}

int solo_b200_dec_batch_decode_host(solo_b200_dec_batch* b, int16_t* pcm, const uint8_t* bits, int cap, const int16_t* nbytes,
                                    const int32_t* lostflag, int32_t* ret) {
    if (!b || !pcm || !bits || !nbytes || !lostflag || cap < 16) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    CK(cudaSetDevice(b->device));
    int r = dec_staging(b, cap);
    if (r) return r;
    b->wave = WAVE_HOST;
    return host_chunks(b, [&](int lo, int hi, cudaStream_t st) {
        return dec_host_range(b, lo, hi - lo, pcm + (size_t)lo * b->spp, bits + (size_t)lo * cap, cap, nbytes + 2 * (size_t)lo, lostflag + lo,
                              ret ? ret + lo : nullptr, st);
    });
}

void solo_b200_dec_batch_destroy(solo_b200_dec_batch* b) { batch_destroy(b); }

int solo_b200_enc_batch_export_state(solo_b200_enc_batch* b, int idx, void* blob) { return state_copy(b, idx, blob, 1); }
int solo_b200_enc_batch_import_state(solo_b200_enc_batch* b, int idx, const void* blob) { return state_copy(b, idx, (void*)blob, 0); }
int solo_b200_dec_batch_export_state(solo_b200_dec_batch* b, int idx, void* blob) { return state_copy(b, idx, blob, 1); }
int solo_b200_dec_batch_import_state(solo_b200_dec_batch* b, int idx, const void* blob) { return state_copy(b, idx, (void*)blob, 0); }
int solo_b200_dec_batch_export_state_sized(solo_b200_dec_batch* b, int idx, void* blob, int blob_bytes) {
    return state_copy(b, idx, blob, 1, blob_bytes < 0 ? 0 : blob_bytes);
}
int solo_b200_dec_batch_import_state_sized(solo_b200_dec_batch* b, int idx, const void* blob, int blob_bytes) {
    // a blob of the batch's size but of the other output mode: a core-output stream's high-band and filter-bank memories
    // have not followed its packets
    if (b && blob && b->khz == 16 && blob_bytes == (int)sizeof(DecState32) && ((const DecState32*)blob)->core_only != b->core_only) {
        snprintf(g_err, sizeof g_err, "state blob of a %s stream, this batch decodes %s", b->core_only ? "full-band 32 kHz" : "core-output (16 kHz)",
                 b->core_only ? "to the 16 kHz core" : "the full 32 kHz band");
        return -1;
    }
    return state_copy(b, idx, (void*)blob, 0, blob_bytes < 0 ? 0 : blob_bytes);
}

// ---- stream membership on the device: reset, export and import of a list of streams -----------------------------------
// The list and the settings are checked on the host first; then one or two kernels on the caller's stream, which the call
// synchronises (the Staging of the host arrays ends with it).  The device is never synchronised: other tenants' work and
// the waves on other CUDA streams keep running.
static int list_args_ok(const void* b, const i32* streams, int n, const char* who) {
    if (b && n >= 0 && (n == 0 || streams)) return 1;
    snprintf(g_err, sizeof g_err, "%s: bad argument", who);
    return 0;
}

int solo_b200_enc_batch_reset(solo_b200_enc_batch* b, const int32_t* streams, int n, const int32_t* rate_bps, const int32_t* dtx,
                              const int32_t* loss_perc, void* cuda_stream) {
    if (!list_args_ok(b, streams, n, "enc_reset") || !streams_ok(streams, n, b->n, "enc_reset")) return -1;
    if (!control_in_range(rate_bps, dtx, loss_perc, n)) { snprintf(g_err, sizeof g_err, "enc_reset: a setting is out of range"); return -1; }
    if (n == 0) return 0;
    CK(cudaSetDevice(b->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    const i32 *d_streams, *d_rate = nullptr, *d_dtx = nullptr, *d_loss = nullptr;
    Staging s(st, "enc_reset", &b->d_list);
    s.span(d_streams, streams, nullptr, 4 * (size_t)n);
    if (rate_bps) s.span(d_rate, rate_bps, nullptr, 4 * (size_t)n);
    if (dtx) s.span(d_dtx, dtx, nullptr, 4 * (size_t)n);
    if (loss_perc) s.span(d_loss, loss_perc, nullptr, 4 * (size_t)n);
    const USER_Ctrl_enc& c = b->ctrl;
    s.run([&] {
        sb_enc_reset_kernel<<<(n + SB_TPB - 1) / SB_TPB, SB_TPB, 0, st>>>(b->d_states, d_streams, n, d_rate, d_dtx, d_loss, c.targetRate_bps,
                                                                        c.dtx_enable ? 1 : 0, c.useMDIndex, c.framesize_ms, c.joint_enable ? 1 : 0);
        return launched("sb_enc_reset_kernel");
    });
    return s.finish();
}

int solo_b200_dec_batch_reset(solo_b200_dec_batch* b, const int32_t* streams, int n, const int32_t* arith, void* cuda_stream) {
    if (!list_args_ok(b, streams, n, "dec_reset") || !streams_ok(streams, n, b->n, "dec_reset")) return -1;
    for (int i = 0; arith && i < n; i++)
        if (arith[i] != -1 && check_dec_arith(&b->ctrl, arith[i])) return -1;     // g_err names the arithmetic
    if (n == 0) return 0;
    CK(cudaSetDevice(b->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    const i32 *d_streams, *d_arith = nullptr;
    Staging s(st, "dec_reset", &b->d_list);
    s.span(d_streams, streams, nullptr, 4 * (size_t)n);
    if (arith) s.span(d_arith, arith, nullptr, 4 * (size_t)n);
    const USER_Ctrl_dec& c = b->ctrl;
    const int g = (n + SB_TPB - 1) / SB_TPB, joint = c.joint_enable ? 1 : 0;
    s.run([&] {
        if (b->khz == 16)
            sb_dec_reset_kernel<16><<<g, SB_TPB, 0, st>>>((DecState32*)b->d_states, d_streams, n, d_arith, b->arith, c.useMDIndex, c.framesize_ms, joint, b->core_only);
        else sb_dec_reset_kernel<8><<<g, SB_TPB, 0, st>>>((DecState*)b->d_states, d_streams, n, d_arith, b->arith, c.useMDIndex, c.framesize_ms, joint, 0);
        return launched("sb_dec_reset_kernel");
    });
    return s.finish();
}

static_assert(sizeof(EncState) % 8 == 0 && sizeof(DecState) % 4 == 0 && sizeof(DecState32) % 8 == 0, "the copy kernel's words");
// export (to_blobs = 1) or import of the listed streams' states through d_blobs [n][stride]; check_mode >= 0 (a 32 kHz decoder
// import): blobs whose core_only differs from check_mode refuse the whole import
static int states_move(Batch* b, void* d_states, size_t stride, const i32* streams, int n, void* d_blobs, int to_blobs, int check_mode,
                       void* cuda_stream, const char* who) {
    if (!list_args_ok(b, streams, n, who) || !streams_ok(streams, n, b->n, who)) return -1;
    if (n == 0) return 0;
    if (!d_blobs || (uintptr_t)d_blobs % 8) { snprintf(g_err, sizeof g_err, "%s: d_blobs must be a non-NULL, 8-byte aligned device address", who); return -1; }
    CK(cudaSetDevice(b->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    const i32* d_streams;
    int* d_bad = nullptr;
    int bad = 0;
    Staging s(st, who, &b->d_list);
    s.span(d_streams, streams, nullptr, 4 * (size_t)n);
    if (check_mode >= 0) s.span(d_bad, &bad, &bad, sizeof bad);
    s.run([&] {
        if (d_bad) {
            sb_dec_blob_check_kernel<<<(n + SB_TPB - 1) / SB_TPB, SB_TPB, 0, st>>>((const DecState32*)d_blobs, n, check_mode, d_bad);
            if (int e = launched("sb_dec_blob_check_kernel")) return e;
        }
        const int g = (n + SB_COPY_WARPS - 1) / SB_COPY_WARPS;
        if (stride % 8 == 0)
            sb_state_copy_kernel<u64><<<g, SB_COPY_WARPS * 32, 0, st>>>((u64*)d_states, (int)(stride / 8), d_streams, n, (u64*)d_blobs, to_blobs, d_bad);
        else sb_state_copy_kernel<u32><<<g, SB_COPY_WARPS * 32, 0, st>>>((u32*)d_states, (int)(stride / 4), d_streams, n, (u32*)d_blobs, to_blobs, d_bad);
        return launched("sb_state_copy_kernel");
    });
    if (int r = s.finish()) return r;
    if (bad) {
        snprintf(g_err, sizeof g_err, "%s: a state blob of a %s stream, this batch decodes %s: nothing imported", who,
                 check_mode ? "full-band 32 kHz" : "core-output (16 kHz)", check_mode ? "to the 16 kHz core" : "the full 32 kHz band");
        return -1;
    }
    return 0;
}
int solo_b200_enc_batch_export_states(solo_b200_enc_batch* b, const int32_t* streams, int n, void* d_blobs, void* cuda_stream) {
    return states_move(b, b ? b->d_states : nullptr, sizeof(EncState), streams, n, d_blobs, 1, -1, cuda_stream, "enc_export_states");
}
int solo_b200_enc_batch_import_states(solo_b200_enc_batch* b, const int32_t* streams, int n, const void* d_blobs, void* cuda_stream) {
    return states_move(b, b ? b->d_states : nullptr, sizeof(EncState), streams, n, (void*)d_blobs, 0, -1, cuda_stream, "enc_import_states");
}
int solo_b200_dec_batch_export_states(solo_b200_dec_batch* b, const int32_t* streams, int n, void* d_blobs, void* cuda_stream) {
    return states_move(b, b ? b->d_states : nullptr, b ? state_stride(b) : 0, streams, n, d_blobs, 1, -1, cuda_stream, "dec_export_states");
}
int solo_b200_dec_batch_import_states(solo_b200_dec_batch* b, const int32_t* streams, int n, const void* d_blobs, void* cuda_stream) {
    const int check = b && b->khz == 16 ? b->core_only : -1;
    return states_move(b, b ? b->d_states : nullptr, b ? state_stride(b) : 0, streams, n, (void*)d_blobs, 0, check, cuda_stream, "dec_import_states");
}

int solo_b200_enc_batch_activity_host(solo_b200_enc_batch* b, uint8_t* level, uint8_t* flags) { return batch_activity_host(b, level, flags); }
int solo_b200_enc_batch_activity_device(solo_b200_enc_batch* b, const int16_t* d_pcm, uint8_t* d_level, uint8_t* d_flags, void* cuda_stream) {
    return batch_activity_device(b, d_pcm, d_level, d_flags, cuda_stream);
}
int solo_b200_dec_batch_activity_host(solo_b200_dec_batch* b, uint8_t* level, uint8_t* flags) { return batch_activity_host(b, level, flags); }
int solo_b200_dec_batch_activity_device(solo_b200_dec_batch* b, const int16_t* d_pcm, uint8_t* d_level, uint8_t* d_flags, void* cuda_stream) {
    return batch_activity_device(b, d_pcm, d_level, d_flags, cuda_stream);
}

// ---- packet framing (host, no GPU involved): enc_main.c:212-234 / dec_main.c:196-307 / README "Bitstream sending" --------
int solo_b200_split_packet(const uint8_t* bits, const int16_t* nbytes, const uint8_t** p1, int* n1, const uint8_t** p2, int* n2) {
    if (!bits || !nbytes || !p1 || !n1 || !p2 || !n2) return -1;
    const int t = nbytes[0], m2 = nbytes[1];
    if (t <= 0) { *p1 = *p2 = bits; *n1 = *n2 = 0; return 0; }    // DTX: nothing to send (enc_API.c:260-265)
    if (m2 < 4 || m2 > t) return -1;   // description 2 carries the high-band bytes: 8 (40 ms packets) or 4 (20 ms, joint mode 1)
    *p1 = bits; *n1 = t - m2;          // description 1: low band only
    *p2 = bits + (t - m2); *n2 = m2;   // description 2: low band + the 8 high-band bytes
    return 0;
}
int solo_b200_merge_packets(const uint8_t* p1, int n1, const uint8_t* p2, int n2, uint8_t* bits, int cap, int16_t* nbytes, int32_t* lostflag) {
    if (!bits || !nbytes || !lostflag || n1 < 0 || n2 < 0) return -1;
    const int m1 = p1 && n1 > 0 ? n1 : 0, m2 = p2 && n2 > 0 ? n2 : 0;   // the descriptions that arrived
    const long long total = (long long)m1 + m2;
    if (total > 0 && total > cap) return -1;
    rx_merge(m1, m2, nbytes, lostflag);
    if (total == 0) {
        if (cap >= 16) memset(bits, 0, 16);
    } else {
        if (m1) memmove(bits, p1, (size_t)m1);
        if (m2) memmove(bits + m1, p2, (size_t)m2);
    }
    return 0;
}
// one record of the reference's .bit file: int16 total, int16 len(MD2)+8, payload (little endian as written by fwrite on x86)
int solo_b200_bitfile_pack(const uint8_t* bits, const int16_t* nbytes, uint8_t* out, int out_cap) {
    if (!bits || !nbytes || !out) return -1;
    const int t = nbytes[0] > 0 ? nbytes[0] : 0;
    if (out_cap < 4 + t) return -1;
    out[0] = (uint8_t)(nbytes[0] & 0xff); out[1] = (uint8_t)((nbytes[0] >> 8) & 0xff);
    out[2] = (uint8_t)(nbytes[1] & 0xff); out[3] = (uint8_t)((nbytes[1] >> 8) & 0xff);
    memcpy(out + 4, bits, (size_t)t);
    return 4 + t;
}
int solo_b200_bitfile_unpack(const uint8_t* in, int in_len, const uint8_t** payload, int16_t* nbytes) {
    if (!in || !payload || !nbytes || in_len < 4) return -1;
    nbytes[0] = (int16_t)(in[0] | (in[1] << 8)); nbytes[1] = (int16_t)(in[2] | (in[3] << 8));
    if (nbytes[0] < 0 || nbytes[1] < 0 || 4 + nbytes[0] > in_len) return -1;
    *payload = in + 4;
    return 4 + nbytes[0];
}
int solo_b200_apply_loss_device(const uint8_t* d_bits_in, const int16_t* d_nbytes_in, const int32_t* d_lostflag, uint8_t* d_bits_out,
                                int16_t* d_nbytes_out, int cap, int n, void* cuda_stream) {
    if (!d_bits_in || !d_nbytes_in || !d_lostflag || !d_bits_out || !d_nbytes_out || cap < 16 || n <= 0) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    sb_apply_loss_kernel<<<(n + 7) / 8, 256, 0, (cudaStream_t)cuda_stream>>>(d_bits_in, d_nbytes_in, d_lostflag, d_bits_out, d_nbytes_out, cap, n);
    return launched("sb_apply_loss_kernel");
}

// ---- conference mixer (sb_mix.cuh) ---------------------------------------------------------------------------------------
static int mix_scalars_ok(int spp, int n, int n_rooms, int k) {
    if ((spp == 320 || spp == 640 || spp == 1280) && n > 0 && n_rooms >= 0 && k >= 1 && k <= SB_MIX_KMAX) return 1;
    snprintf(g_err, sizeof g_err, "mix: bad argument (spp %d, n %d, n_rooms %d, k %d)", spp, n, n_rooms, k);
    return 0;
}
// the two kernels of one mix call on st; nothing when there are no rooms
static int mix_launch(const i16* in, i16* out, int spp, int n, const u8* level, const u8* flags, const i32* room_start,
                      const i32* members, int R, int k, i32* talkers, cudaStream_t st) {
    if (R == 0) return 0;
    sb_mix_select_kernel<<<(R + SB_MIX_WARPS - 1) / SB_MIX_WARPS, SB_MIX_WARPS * 32, 0, st>>>(level, flags, room_start, members, n, R, k, talkers);
    if (int e = launched("sb_mix_select_kernel")) return e;
    sb_mix_kernel<<<(n + SB_MIX_WARPS - 1) / SB_MIX_WARPS, SB_MIX_WARPS * 32, 0, st>>>(in, out, spp, n, room_start, members, R, k, talkers);
    return launched("sb_mix_kernel");
}
// the room layout a *_host call of the mixer or the contributor lists takes: room_start[0] == 0 and non-decreasing,
// members in [0, n), no stream listed twice; `who` prefixes the error text
static int rooms_ok(const i32* room_start, const i32* members, int n_rooms, int n, const char* who) {
    if (room_start[0] != 0) { snprintf(g_err, sizeof g_err, "%s: room_start[0] is %d, not 0", who, room_start[0]); return 0; }
    for (int r = 0; r < n_rooms; r++)
        if (room_start[r + 1] < room_start[r]) { snprintf(g_err, sizeof g_err, "%s: room_start decreases at room %d", who, r); return 0; }
    const i32 M = room_start[n_rooms];
    if (M > 0 && !members) { snprintf(g_err, sizeof g_err, "%s: bad argument (members NULL)", who); return 0; }
    std::vector<u8> seen((size_t)n, 0);
    for (i32 m = 0; m < M; m++) {
        const i32 j = members[m];
        if (j < 0 || j >= n) { snprintf(g_err, sizeof g_err, "%s: member %d is stream %d, outside [0, %d)", who, m, j, n); return 0; }
        if (seen[j]++) { snprintf(g_err, sizeof g_err, "%s: stream %d is listed twice", who, j); return 0; }
    }
    return 1;
}

int solo_b200_mix_device(const int16_t* d_in, int16_t* d_out, int spp, int n, const uint8_t* d_level, const uint8_t* d_flags,
                         const int32_t* d_room_start, const int32_t* d_members, int n_rooms, int k, int32_t* d_talkers, void* cuda_stream) {
    if (!d_in || !d_out || !d_level || !d_flags || !d_room_start || !d_members || !d_talkers) { snprintf(g_err, sizeof g_err, "mix: bad argument"); return -1; }
    if (!mix_scalars_ok(spp, n, n_rooms, k)) return -1;
    const size_t bytes = sizeof(i16) * (size_t)spp * (size_t)n;
    const uintptr_t a = (uintptr_t)d_in, b = (uintptr_t)d_out;
    if (((a | b) & 15) != 0) { snprintf(g_err, sizeof g_err, "mix_device: d_in and d_out must be 16-byte aligned"); return -1; }
    if (a < b + bytes && b < a + bytes) { snprintf(g_err, sizeof g_err, "mix_device: d_in and d_out overlap"); return -1; }
    return mix_launch(d_in, d_out, spp, n, d_level, d_flags, d_room_start, d_members, n_rooms, k, d_talkers, (cudaStream_t)cuda_stream);
}

int solo_b200_mix_host(const int16_t* in, int16_t* out, int spp, int n, const uint8_t* level, const uint8_t* flags,
                       const int32_t* room_start, const int32_t* members, int n_rooms, int k, int32_t* talkers) {
    if (!in || !out || !level || !flags || !room_start || !talkers) { snprintf(g_err, sizeof g_err, "mix: bad argument"); return -1; }
    if (!mix_scalars_ok(spp, n, n_rooms, k)) return -1;
    if (!rooms_ok(room_start, members, n_rooms, n, "mix")) return -1;
    if (n_rooms == 0) return 0;
    int dev = 0;
    CK(cudaGetDevice(&dev));
    if (int e = require_gpu(dev)) return e;
    cudaStream_t st;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    const size_t bytes = sizeof(i16) * (size_t)spp * (size_t)n;
    const i16* d_in; i16* d_out; const u8 *d_level, *d_flags; const i32 *d_rs, *d_members; i32* d_tk;
    Staging s(st, "mix");
    s.span(d_in, in, nullptr, bytes);
    s.span(d_out, out, out, bytes);     // `out` goes in too: rows of streams in no room come back as they were
    s.span(d_level, level, nullptr, (size_t)n);
    s.span(d_flags, flags, nullptr, (size_t)n);
    s.span(d_rs, room_start, nullptr, sizeof(i32) * ((size_t)n_rooms + 1));
    s.span(d_members, members, nullptr, sizeof(i32) * (size_t)room_start[n_rooms]);
    s.span(d_tk, nullptr, talkers, sizeof(i32) * (size_t)n_rooms * (size_t)k);
    s.run([&] { return mix_launch(d_in, d_out, spp, n, d_level, d_flags, d_rs, d_members, n_rooms, k, d_tk, st); });
    const int r = s.finish();
    cudaStreamDestroy(st);
    return r;
}

// ---- receive queue (sb_rx.cuh) -------------------------------------------------------------------------------------------
struct solo_b200_rx {
    int device;
    cudaStream_t st;            // the _host forms' stream
    RxDev q;
    RxTiming t;                 // all zero until solo_b200_rx_enable_timing
    ~solo_b200_rx() {
        if (st) cudaStreamDestroy(st);
        cudaFree(q.last); cudaFree(q.idx); cudaFree(q.len); cudaFree(q.elect); cudaFree(q.rep); cudaFree(q.cnt);
        cudaFree(q.bad); cudaFree(q.store);
        cudaFree(t.transit); cudaFree(t.jitter); cudaFree(t.highest); cudaFree(t.received); cudaFree(t.margin);
        cudaFree(t.key[0]); cudaFree(t.key[1]); cudaFree(t.pos[0]); cudaFree(t.pos[1]); cudaFree(t.hist);
    }
};

solo_b200_rx* solo_b200_rx_create(int n_streams, int depth, int desc_cap, int device) {
    if (n_streams <= 0 || depth < 2 || depth > 32 || (depth & (depth - 1)) || desc_cap < 16 || desc_cap > 1024 || desc_cap % 16) {
        snprintf(g_err, sizeof g_err, "rx_create: bad argument (n %d, depth %d, desc_cap %d)", n_streams, depth, desc_cap);
        return nullptr;
    }
    if (require_gpu(device)) return nullptr;
    solo_b200_rx* r = new solo_b200_rx();
    r->device = device;
    RxDev& q = r->q;
    q.n = n_streams; q.depth = depth; q.desc_cap = desc_cap;
    const size_t n = (size_t)n_streams, slots = n * depth, store = slots * 2 * desc_cap + 16;
    bool ok = cudaStreamCreateWithFlags(&r->st, cudaStreamNonBlocking) == cudaSuccess &&
              cudaMalloc(&q.last, 4 * n) == cudaSuccess && cudaMalloc(&q.idx, 4 * slots) == cudaSuccess &&
              cudaMalloc(&q.len, 4 * slots) == cudaSuccess && cudaMalloc(&q.elect, 16 * slots) == cudaSuccess &&
              cudaMalloc(&q.rep, 4 * slots) == cudaSuccess && cudaMalloc(&q.cnt, 4 * RX_NCOUNT * n) == cudaSuccess &&
              cudaMalloc(&q.bad, 8) == cudaSuccess && cudaMalloc(&q.store, store) == cudaSuccess;
    // last = 0xFFFFFFFF (index 0 plays first), slots empty, election words empty, counters zero
    ok = ok && cudaMemsetAsync(q.last, 0xFF, 4 * n, r->st) == cudaSuccess && cudaMemsetAsync(q.idx, 0, 4 * slots, r->st) == cudaSuccess &&
         cudaMemsetAsync(q.len, 0, 4 * slots, r->st) == cudaSuccess && cudaMemsetAsync(q.elect, 0, 16 * slots, r->st) == cudaSuccess &&
         cudaMemsetAsync(q.rep, 0xFF, 4 * slots, r->st) == cudaSuccess && cudaMemsetAsync(q.cnt, 0, 4 * RX_NCOUNT * n, r->st) == cudaSuccess &&
         cudaMemsetAsync(q.bad, 0, 8, r->st) == cudaSuccess && cudaMemsetAsync(q.store, 0, store, r->st) == cudaSuccess &&
         cudaStreamSynchronize(r->st) == cudaSuccess;
    if (!ok) {
        snprintf(g_err, sizeof g_err, "rx_create: %s", cudaGetErrorString(cudaGetLastError()));
        delete r;
        return nullptr;
    }
    return r;
}

void solo_b200_rx_destroy(solo_b200_rx* q) {
    if (!q) return;
    cudaSetDevice(q->device);
    delete q;
}

// the three insert passes on st; nothing for no arrivals
static int rx_insert_launch(solo_b200_rx* r, const RxArrivals& A, cudaStream_t st) {
    if (A.n == 0) return 0;
    const unsigned g = (unsigned)(((long long)A.n + SB_RX_THREADS - 1) / SB_RX_THREADS);
    const unsigned g2 = (unsigned)(((long long)A.n * SB_RX_TEAM + SB_RX_THREADS - 1) / SB_RX_THREADS);
    sb_rx_elect_kernel<<<g, SB_RX_THREADS, 0, st>>>(r->q, A);
    if (int e = launched("sb_rx_elect_kernel")) return e;
    sb_rx_classify_kernel<<<g2, SB_RX_THREADS, 0, st>>>(r->q, A);
    if (int e = launched("sb_rx_classify_kernel")) return e;
    sb_rx_commit_kernel<<<g, SB_RX_THREADS, 0, st>>>(r->q, A);
    return launched("sb_rx_commit_kernel");
}
static int rx_insert_args_ok(solo_b200_rx* q, const void* stream, const void* index, const void* desc, const void* off,
                             const void* len, int n_arrivals, const void* payload, int64_t payload_bytes) {
    if (q && n_arrivals >= 0 && payload_bytes >= 0 && (n_arrivals == 0 || (stream && index && desc && off && len)) &&
        (payload || payload_bytes == 0))
        return 1;
    snprintf(g_err, sizeof g_err, "rx_insert: bad argument (n_arrivals %d, payload_bytes %lld)", n_arrivals, (long long)payload_bytes);
    return 0;
}

int solo_b200_rx_insert_device(solo_b200_rx* q, const int32_t* d_stream, const uint32_t* d_index, const uint8_t* d_desc,
                               const int32_t* d_off, const int32_t* d_len, int n_arrivals, const uint8_t* d_payload,
                               int64_t payload_bytes, void* cuda_stream) {
    if (!rx_insert_args_ok(q, d_stream, d_index, d_desc, d_off, d_len, n_arrivals, d_payload, payload_bytes)) return -1;
    if (n_arrivals == 0) return 0;
    CK(cudaSetDevice(q->device));
    const RxArrivals A = {d_stream, d_index, d_desc, d_off, d_len, n_arrivals, d_payload, payload_bytes};
    return rx_insert_launch(q, A, (cudaStream_t)cuda_stream);
}

int solo_b200_rx_insert_host(solo_b200_rx* q, const int32_t* stream, const uint32_t* index, const uint8_t* desc,
                             const int32_t* off, const int32_t* len, int n_arrivals, const uint8_t* payload, int64_t payload_bytes) {
    if (!rx_insert_args_ok(q, stream, index, desc, off, len, n_arrivals, payload, payload_bytes)) return -1;
    if (n_arrivals == 0) return 0;
    CK(cudaSetDevice(q->device));
    const size_t na = (size_t)n_arrivals;
    RxArrivals A = {nullptr, nullptr, nullptr, nullptr, nullptr, n_arrivals, nullptr, payload_bytes};
    Staging s(q->st, "rx_insert");
    s.span(A.stream, stream, nullptr, 4 * na);
    s.span(A.index, index, nullptr, 4 * na);
    s.span(A.desc, desc, nullptr, na);
    s.span(A.off, off, nullptr, 4 * na);
    s.span(A.len, len, nullptr, 4 * na);
    s.span(A.payload, payload, nullptr, (size_t)payload_bytes);
    s.run([&] { return rx_insert_launch(q, A, q->st); });
    return s.finish();
}

static int rx_sort_tiles(int n_arrivals) { return (n_arrivals + SB_RX_SORT_TILE - 1) / SB_RX_SORT_TILE; }

int solo_b200_rx_enable_timing(solo_b200_rx* q, uint32_t ts_per_index, int max_arrivals) {
    if (!q || ts_per_index == 0 || max_arrivals < 1 || q->t.transit) {
        snprintf(g_err, sizeof g_err, "rx_enable_timing: bad argument (ts_per_index %u, max_arrivals %d%s)", ts_per_index,
                 max_arrivals, q && q->t.transit ? ", timing already enabled" : "");
        return -1;
    }
    CK(cudaSetDevice(q->device));
    RxTiming t = {};
    t.ts_per_index = ts_per_index;
    t.max_arrivals = max_arrivals;
    for (u32 top = (u32)(q->q.n - 1); top; top >>= 8) t.passes++;
    const size_t n = (size_t)q->q.n, na = (size_t)max_arrivals, nh = 256 * (size_t)rx_sort_tiles(max_arrivals);
    bool ok = cudaMalloc(&t.transit, 4 * n) == cudaSuccess && cudaMalloc(&t.jitter, 4 * n) == cudaSuccess &&
              cudaMalloc(&t.highest, 8 * n) == cudaSuccess && cudaMalloc(&t.received, 4 * n) == cudaSuccess &&
              cudaMalloc(&t.margin, 4 * RX_MARGIN_BINS * n) == cudaSuccess;
    for (int b = 0; b < 2; b++) ok = ok && cudaMalloc(&t.key[b], 4 * na) == cudaSuccess && cudaMalloc(&t.pos[b], 4 * na) == cudaSuccess;
    ok = ok && cudaMalloc(&t.hist, 4 * nh) == cudaSuccess;
    ok = ok && cudaMemsetAsync(t.transit, 0, 4 * n, q->st) == cudaSuccess && cudaMemsetAsync(t.jitter, 0, 4 * n, q->st) == cudaSuccess &&
         cudaMemsetAsync(t.highest, 0, 8 * n, q->st) == cudaSuccess && cudaMemsetAsync(t.received, 0, 4 * n, q->st) == cudaSuccess &&
         cudaMemsetAsync(t.margin, 0, 4 * RX_MARGIN_BINS * n, q->st) == cudaSuccess && cudaStreamSynchronize(q->st) == cudaSuccess;
    if (!ok) {
        snprintf(g_err, sizeof g_err, "rx_enable_timing: %s", cudaGetErrorString(cudaGetLastError()));
        cudaFree(t.transit); cudaFree(t.jitter); cudaFree(t.highest); cudaFree(t.received); cudaFree(t.margin);
        cudaFree(t.key[0]); cudaFree(t.key[1]); cudaFree(t.pos[0]); cudaFree(t.pos[1]); cudaFree(t.hist);
        return -1;
    }
    q->t = t;
    return 0;
}

// the timed insert on st: the three insert passes, the keys pass, the sort passes and the walk; nothing for no arrivals
static int rx_insert_timed_launch(solo_b200_rx* r, const RxArrivals& A, const u32* arrival, cudaStream_t st) {
    if (A.n == 0) return 0;
    if (int e = rx_insert_launch(r, A, st)) return e;
    RxTiming& T = r->t;
    const unsigned g = (unsigned)(((long long)A.n + SB_RX_THREADS - 1) / SB_RX_THREADS), tiles = (unsigned)rx_sort_tiles(A.n);
    sb_rx_timing_keys_kernel<<<g, SB_RX_THREADS, 0, st>>>(r->q, T, A);
    if (int e = launched("sb_rx_timing_keys_kernel")) return e;
    int src = 0;
    for (int p = 0; p < T.passes; p++, src ^= 1) {
        sb_rx_sort_hist_kernel<<<tiles, SB_RX_SORT_THREADS, 0, st>>>(T.key[src], T.hist, A.n, 8 * p);
        if (int e = launched("sb_rx_sort_hist_kernel")) return e;
        sb_rx_sort_scan_kernel<<<1, SB_RX_SCAN_THREADS, 0, st>>>(T.hist, 256 * (int)tiles);
        if (int e = launched("sb_rx_sort_scan_kernel")) return e;
        sb_rx_sort_scatter_kernel<<<tiles, SB_RX_SORT_THREADS, 0, st>>>(T.key[src], T.pos[src], T.key[src ^ 1], T.pos[src ^ 1],
                                                                         T.hist, A.n, 8 * p);
        if (int e = launched("sb_rx_sort_scatter_kernel")) return e;
    }
    sb_rx_timing_walk_kernel<<<g, SB_RX_THREADS, 0, st>>>(T, T.key[src], T.pos[src], A, arrival);
    return launched("sb_rx_timing_walk_kernel");
}
static int rx_insert_timed_args_ok(solo_b200_rx* q, const void* arrival, int n_arrivals) {
    if (!q->t.transit) { snprintf(g_err, sizeof g_err, "rx_insert_timed: timing is not enabled"); return 0; }
    if (n_arrivals > q->t.max_arrivals || (n_arrivals > 0 && !arrival)) {
        snprintf(g_err, sizeof g_err, "rx_insert_timed: bad argument (n_arrivals %d, max_arrivals %d)", n_arrivals, q->t.max_arrivals);
        return 0;
    }
    return 1;
}

int solo_b200_rx_insert_timed_device(solo_b200_rx* q, const int32_t* d_stream, const uint32_t* d_index, const uint8_t* d_desc,
                                     const int32_t* d_off, const int32_t* d_len, const uint32_t* d_arrival, int n_arrivals,
                                     const uint8_t* d_payload, int64_t payload_bytes, void* cuda_stream) {
    if (!rx_insert_args_ok(q, d_stream, d_index, d_desc, d_off, d_len, n_arrivals, d_payload, payload_bytes) ||
        !rx_insert_timed_args_ok(q, d_arrival, n_arrivals))
        return -1;
    if (n_arrivals == 0) return 0;
    CK(cudaSetDevice(q->device));
    const RxArrivals A = {d_stream, d_index, d_desc, d_off, d_len, n_arrivals, d_payload, payload_bytes};
    return rx_insert_timed_launch(q, A, d_arrival, (cudaStream_t)cuda_stream);
}

int solo_b200_rx_insert_timed_host(solo_b200_rx* q, const int32_t* stream, const uint32_t* index, const uint8_t* desc,
                                   const int32_t* off, const int32_t* len, const uint32_t* arrival, int n_arrivals,
                                   const uint8_t* payload, int64_t payload_bytes) {
    if (!rx_insert_args_ok(q, stream, index, desc, off, len, n_arrivals, payload, payload_bytes) ||
        !rx_insert_timed_args_ok(q, arrival, n_arrivals))
        return -1;
    if (n_arrivals == 0) return 0;
    CK(cudaSetDevice(q->device));
    const size_t na = (size_t)n_arrivals;
    RxArrivals A = {nullptr, nullptr, nullptr, nullptr, nullptr, n_arrivals, nullptr, payload_bytes};
    const u32* d_arrival;
    Staging s(q->st, "rx_insert_timed");
    s.span(A.stream, stream, nullptr, 4 * na);
    s.span(A.index, index, nullptr, 4 * na);
    s.span(A.desc, desc, nullptr, na);
    s.span(A.off, off, nullptr, 4 * na);
    s.span(A.len, len, nullptr, 4 * na);
    s.span(d_arrival, arrival, nullptr, 4 * na);
    s.span(A.payload, payload, nullptr, (size_t)payload_bytes);
    s.run([&] { return rx_insert_timed_launch(q, A, d_arrival, q->st); });
    return s.finish();
}

int solo_b200_rx_timing(solo_b200_rx* q, uint32_t* jitter, uint64_t* highest, uint32_t* received, uint32_t* margin,
                        void* cuda_stream) {
    if (!q || !q->t.transit) { snprintf(g_err, sizeof g_err, "rx_timing: %s", q ? "timing is not enabled" : "bad argument"); return -1; }
    CK(cudaSetDevice(q->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    const size_t n = (size_t)q->q.n;
    if (jitter) CK(cudaMemcpyAsync(jitter, q->t.jitter, 4 * n, cudaMemcpyDeviceToHost, st));
    if (highest) CK(cudaMemcpyAsync(highest, q->t.highest, 8 * n, cudaMemcpyDeviceToHost, st));
    if (received) CK(cudaMemcpyAsync(received, q->t.received, 4 * n, cudaMemcpyDeviceToHost, st));
    if (margin) CK(cudaMemcpyAsync(margin, q->t.margin, 4 * RX_MARGIN_BINS * n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (jitter)
        for (size_t s = 0; s < n; s++) jitter[s] >>= 4;     // the state keeps 1/16 units (RFC 3550 A.8)
    return 0;
}

static int rx_pull_args_ok(solo_b200_rx* q, const void* bits, int cap, const void* nbytes, const void* lostflag) {
    if (!q || !bits || !nbytes || !lostflag) { snprintf(g_err, sizeof g_err, "rx_pull: bad argument"); return 0; }
    if (cap < 2 * q->q.desc_cap) { snprintf(g_err, sizeof g_err, "rx_pull: cap %d is below 2 * desc_cap = %d", cap, 2 * q->q.desc_cap); return 0; }
    return 1;
}
static int rx_pull_launch(solo_b200_rx* r, const u32* play, u8* bits, int cap, i16* nbytes, i32* lostflag, cudaStream_t st) {
    sb_rx_pull_kernel<<<(r->q.n + SB_RX_PULL_WARPS - 1) / SB_RX_PULL_WARPS, SB_RX_PULL_WARPS * 32, 0, st>>>(r->q, play, bits, cap, nbytes, lostflag);
    return launched("sb_rx_pull_kernel");
}

int solo_b200_rx_pull_device(solo_b200_rx* q, const uint32_t* d_play, uint8_t* d_bits, int cap, int16_t* d_nbytes,
                             int32_t* d_lostflag, void* cuda_stream) {
    if (!rx_pull_args_ok(q, d_bits, cap, d_nbytes, d_lostflag)) return -1;
    if ((uintptr_t)d_bits & 15) { snprintf(g_err, sizeof g_err, "rx_pull_device: d_bits must be 16-byte aligned"); return -1; }
    CK(cudaSetDevice(q->device));
    return rx_pull_launch(q, d_play, d_bits, cap, d_nbytes, d_lostflag, (cudaStream_t)cuda_stream);
}

int solo_b200_rx_pull_host(solo_b200_rx* q, const uint32_t* play, uint8_t* bits, int cap, int16_t* nbytes, int32_t* lostflag) {
    if (!rx_pull_args_ok(q, bits, cap, nbytes, lostflag)) return -1;
    CK(cudaSetDevice(q->device));
    const size_t n = (size_t)q->q.n;
    u8* d_bits; i16* d_nbytes; i32* d_lostflag; const u32* d_play;
    Staging s(q->st, "rx_pull");
    s.span(d_bits, bits, bits, n * (size_t)cap);    // the caller's rows go in too: bytes past nbytes[0] come back unchanged
    s.span(d_nbytes, nullptr, nbytes, 4 * n);
    s.span(d_lostflag, nullptr, lostflag, 4 * n);
    s.span(d_play, play, nullptr, 4 * n);
    s.run([&] { return rx_pull_launch(q, play ? d_play : nullptr, d_bits, cap, d_nbytes, d_lostflag, q->st); });
    return s.finish();
}

// The reset of either queue (Q solo_b200_rx or solo_b200_tx): a list of distinct streams of the queue, nothing done when it
// is refused, then `kernel` (block threads per block) on the caller's stream, which the call synchronises.  `also`, when
// given, launches more work on the same device list of streams after it.
extern "C++" {
template <class Q, class D>
static int queue_reset(Q* q, const i32* streams, const u32* start, int n, cudaStream_t st,
                       void (*kernel)(D, const i32*, const u32*, int), int block, const char* who,
                       int (*also)(Q*, const i32*, int, cudaStream_t) = nullptr) {
    if (!q || n < 0 || (n > 0 && (!streams || !start))) { snprintf(g_err, sizeof g_err, "%s: bad argument", who); return -1; }
    if (!streams_ok(streams, n, q->q.n, who)) return -1;
    if (n == 0) return 0;
    CK(cudaSetDevice(q->device));
    const i32* d_streams; const u32* d_start;
    Staging s(st, who);
    s.span(d_streams, streams, nullptr, 4 * (size_t)n);
    s.span(d_start, start, nullptr, 4 * (size_t)n);
    s.run([&] {
        kernel<<<(n + block - 1) / block, block, 0, st>>>(q->q, d_streams, d_start, n);
        if (int e = launched(who)) return e;
        return also ? also(q, d_streams, n, st) : 0;
    });
    return s.finish();
}
}  // extern "C++"

// a timed queue's reset also clears the listed streams' timing state: one more launch
static int rx_reset_timing(solo_b200_rx* q, const i32* d_streams, int n, cudaStream_t st) {
    if (!q->t.transit) return 0;
    sb_rx_timing_reset_kernel<<<(n + SB_RX_THREADS - 1) / SB_RX_THREADS, SB_RX_THREADS, 0, st>>>(q->t, d_streams, n);
    return launched("sb_rx_timing_reset_kernel");
}

int solo_b200_rx_reset(solo_b200_rx* q, const int32_t* streams, const uint32_t* start, int n, void* cuda_stream) {
    return queue_reset(q, streams, start, n, (cudaStream_t)cuda_stream, sb_rx_reset_kernel, SB_RX_THREADS, "rx_reset",
                       rx_reset_timing);
}

int solo_b200_rx_stats(solo_b200_rx* q, uint32_t* counters, uint64_t* bad_stream, void* cuda_stream) {
    if (!q) { snprintf(g_err, sizeof g_err, "rx_stats: bad argument"); return -1; }
    CK(cudaSetDevice(q->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    if (counters) CK(cudaMemcpyAsync(counters, q->q.cnt, 4 * RX_NCOUNT * (size_t)q->q.n, cudaMemcpyDeviceToHost, st));
    if (bad_stream) CK(cudaMemcpyAsync(bad_stream, q->q.bad, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return 0;
}

// ---- send queue (sb_tx.cuh) ----------------------------------------------------------------------------------------------
struct solo_b200_tx {
    int device;
    cudaStream_t st;            // the _host form's stream
    TxDev q;
    ~solo_b200_tx() {
        if (st) cudaStreamDestroy(st);
        cudaFree(q.next); cudaFree(q.cnt); cudaFree(q.pre); cudaFree(q.blk);
    }
};
static int tx_blocks(int n) { return (n + SB_TX_BLOCK - 1) / SB_TX_BLOCK; }

solo_b200_tx* solo_b200_tx_create(int n_streams, int device) {
    if (n_streams <= 0) { snprintf(g_err, sizeof g_err, "tx_create: bad argument (n %d)", n_streams); return nullptr; }
    if (require_gpu(device)) return nullptr;
    solo_b200_tx* t = new solo_b200_tx();
    t->device = device;
    TxDev& q = t->q;
    q.n = n_streams;
    const size_t n = (size_t)n_streams;
    bool ok = cudaStreamCreateWithFlags(&t->st, cudaStreamNonBlocking) == cudaSuccess &&
              cudaMalloc(&q.next, 4 * n) == cudaSuccess && cudaMalloc(&q.cnt, 4 * TX_NCOUNT * n) == cudaSuccess &&
              cudaMalloc(&q.pre, 8 * n) == cudaSuccess && cudaMalloc(&q.blk, 8 * (size_t)tx_blocks(n_streams)) == cudaSuccess;
    ok = ok && cudaMemsetAsync(q.next, 0, 4 * n, t->st) == cudaSuccess &&
         cudaMemsetAsync(q.cnt, 0, 4 * TX_NCOUNT * n, t->st) == cudaSuccess && cudaStreamSynchronize(t->st) == cudaSuccess;
    if (!ok) {
        snprintf(g_err, sizeof g_err, "tx_create: %s", cudaGetErrorString(cudaGetLastError()));
        delete t;
        return nullptr;
    }
    return t;
}

void solo_b200_tx_destroy(solo_b200_tx* q) {
    if (!q) return;
    cudaSetDevice(q->device);
    delete q;
}

// the scalars of a pack: cap a multiple of 16 (aligned rows), every offset within int32, room for the worst case
static int tx_pack_args_ok(solo_b200_tx* q, const void* bits, int cap, const void* nbytes, const TxOut& o, int64_t payload_cap) {
    if (!q || !bits || !nbytes || !o.payload || !o.stream || !o.index || !o.desc || !o.off || !o.len || !o.count || !o.total) {
        snprintf(g_err, sizeof g_err, "tx_pack: bad argument");
        return 0;
    }
    const long long worst = (long long)q->q.n * cap;
    if (cap < 16 || cap % 16 || worst > 0x7FFFFFFFll) {
        snprintf(g_err, sizeof g_err, "tx_pack: cap %d must be a multiple of 16 with n * cap <= 2^31 - 1 (n %d)", cap, q->q.n);
        return 0;
    }
    if (payload_cap < worst) {
        snprintf(g_err, sizeof g_err, "tx_pack: payload_cap %lld is below n * cap = %lld", (long long)payload_cap, worst);
        return 0;
    }
    return 1;
}
static int tx_pack_launch(solo_b200_tx* t, const u8* bits, int cap, const i16* nbytes, const TxOut& o, cudaStream_t st) {
    const int nblk = tx_blocks(t->q.n);
    sb_tx_sizes_kernel<<<nblk, SB_TX_BLOCK, 0, st>>>(t->q, nbytes, cap);
    if (int e = launched("sb_tx_sizes_kernel")) return e;
    sb_tx_scan_kernel<<<1, SB_TX_SCAN_THREADS, 0, st>>>(t->q, nblk, o.count, o.total);
    if (int e = launched("sb_tx_scan_kernel")) return e;
    sb_tx_pack_kernel<<<(t->q.n + SB_TX_PACK_WARPS - 1) / SB_TX_PACK_WARPS, SB_TX_PACK_WARPS * 32, 0, st>>>(t->q, bits, cap, nbytes, o);
    return launched("sb_tx_pack_kernel");
}

int solo_b200_tx_pack_device(solo_b200_tx* q, const uint8_t* d_bits, int cap, const int16_t* d_nbytes, uint8_t* d_payload,
                             int64_t payload_cap, int32_t* d_stream, uint32_t* d_index, uint8_t* d_desc, int32_t* d_off,
                             int32_t* d_len, int32_t* d_count, int64_t* d_total, void* cuda_stream) {
    const TxOut o = {d_payload, d_stream, d_index, d_desc, d_off, d_len, d_count, d_total};
    if (!tx_pack_args_ok(q, d_bits, cap, d_nbytes, o, payload_cap)) return -1;
    if (((uintptr_t)d_bits | (uintptr_t)d_payload) & 15) {
        snprintf(g_err, sizeof g_err, "tx_pack_device: d_bits and d_payload must be 16-byte aligned");
        return -1;
    }
    CK(cudaSetDevice(q->device));
    return tx_pack_launch(q, d_bits, cap, d_nbytes, o, (cudaStream_t)cuda_stream);
}

int solo_b200_tx_pack_host(solo_b200_tx* q, const uint8_t* bits, int cap, const int16_t* nbytes, uint8_t* payload,
                           int64_t payload_cap, int32_t* stream, uint32_t* index, uint8_t* desc, int32_t* off, int32_t* len,
                           int64_t* total) {
    i32 count = 0;              // host copies of the call's datagram count and byte total
    i64 tot = 0;
    const TxOut h = {payload, stream, index, desc, off, len, &count, total};
    if (!tx_pack_args_ok(q, bits, cap, nbytes, h, payload_cap)) return -1;
    CK(cudaSetDevice(q->device));
    const size_t n = (size_t)q->q.n, rows = n * (size_t)cap, e = 2 * n;
    const u8* d_bits; const i16* d_nbytes; TxOut o;
    Staging s(q->st, "tx_pack");
    s.span(d_bits, bits, nullptr, rows);
    s.span(d_nbytes, nbytes, nullptr, 4 * n);
    s.span(o.payload, nullptr, nullptr, rows);
    s.span(o.stream, nullptr, nullptr, 4 * e);
    s.span(o.index, nullptr, nullptr, 4 * e);
    s.span(o.desc, nullptr, nullptr, e);
    s.span(o.off, nullptr, nullptr, 4 * e);
    s.span(o.len, nullptr, nullptr, 4 * e);
    s.span(o.count, nullptr, &count, 4);
    s.span(o.total, nullptr, &tot, 8);
    // the count and the total first, then only the datagrams they cover
    if (s.run([&] { return tx_pack_launch(q, d_bits, cap, d_nbytes, o, q->st); }) && s.sync()) {
        const size_t c = (size_t)count;
        s.back(payload, o.payload, (size_t)tot) && s.back(stream, o.stream, 4 * c) && s.back(index, o.index, 4 * c) &&
            s.back(desc, o.desc, c) && s.back(off, o.off, 4 * c) && s.back(len, o.len, 4 * c);
    }
    if (int r = s.finish()) return r;
    *total = tot;
    return count;
}

int solo_b200_tx_reset(solo_b200_tx* q, const int32_t* streams, const uint32_t* start, int n, void* cuda_stream) {
    return queue_reset(q, streams, start, n, (cudaStream_t)cuda_stream, sb_tx_reset_kernel, SB_TX_BLOCK, "tx_reset");
}

int solo_b200_tx_stats(solo_b200_tx* q, uint32_t* counters, void* cuda_stream) {
    if (!q || !counters) { snprintf(g_err, sizeof g_err, "tx_stats: bad argument"); return -1; }
    CK(cudaSetDevice(q->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    CK(cudaMemcpyAsync(counters, q->q.cnt, 4 * TX_NCOUNT * (size_t)q->q.n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return 0;
}

// ---- downlink contributor lists (sb_tx.cuh) ----------------------------------------------------------------------------------
static int contributors_scalars_ok(int n, int n_rooms, int k) {
    if (n > 0 && n_rooms >= 0 && k >= 1 && k <= SB_MIX_KMAX) return 1;
    snprintf(g_err, sizeof g_err, "mix_contributors: bad argument (n %d, n_rooms %d, k %d)", n, n_rooms, k);
    return 0;
}
// every row -1 / 127 (the rows of streams in no room keep that), then one kernel for the members' rows; no kernel without rooms
static int contributors_launch(const i32* room_start, const i32* members, int R, int k, const i32* talkers, const u8* level,
                               int n, i32* csrc, u8* csrc_level, cudaStream_t st) {
    const size_t e = (size_t)n * (size_t)k;
    CK(cudaMemsetAsync(csrc, 0xFF, 4 * e, st));
    CK(cudaMemsetAsync(csrc_level, SB_TX_LVL_NONE, e, st));
    if (R == 0) return 0;
    sb_mix_contributors_kernel<<<(n + SB_CONTRIB_THREADS - 1) / SB_CONTRIB_THREADS, SB_CONTRIB_THREADS, 0, st>>>(
        room_start, members, R, k, talkers, level, n, csrc, csrc_level);
    return launched("sb_mix_contributors_kernel");
}

int solo_b200_mix_contributors_device(const int32_t* d_room_start, const int32_t* d_members, int n_rooms, int k,
                                      const int32_t* d_talkers, const uint8_t* d_level, int n, int32_t* d_csrc,
                                      uint8_t* d_csrc_level, void* cuda_stream) {
    if (!d_room_start || !d_members || !d_talkers || !d_level || !d_csrc || !d_csrc_level) { snprintf(g_err, sizeof g_err, "mix_contributors: bad argument"); return -1; }
    if (!contributors_scalars_ok(n, n_rooms, k)) return -1;
    return contributors_launch(d_room_start, d_members, n_rooms, k, d_talkers, d_level, n, d_csrc, d_csrc_level, (cudaStream_t)cuda_stream);
}

int solo_b200_mix_contributors_host(const int32_t* room_start, const int32_t* members, int n_rooms, int k, const int32_t* talkers,
                                    const uint8_t* level, int n, int32_t* csrc, uint8_t* csrc_level) {
    if (!room_start || !level || !csrc || !csrc_level || (n_rooms > 0 && !talkers)) { snprintf(g_err, sizeof g_err, "mix_contributors: bad argument"); return -1; }
    if (!contributors_scalars_ok(n, n_rooms, k)) return -1;
    if (!rooms_ok(room_start, members, n_rooms, n, "mix_contributors")) return -1;
    int dev = 0;
    CK(cudaGetDevice(&dev));
    if (int e = require_gpu(dev)) return e;
    cudaStream_t st;
    CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    const size_t e = (size_t)n * (size_t)k;
    const i32 *d_rs, *d_members, *d_talkers; const u8* d_level; i32* d_csrc; u8* d_csrc_level;
    Staging s(st, "mix_contributors");
    s.span(d_rs, room_start, nullptr, 4 * ((size_t)n_rooms + 1));
    s.span(d_members, members, nullptr, 4 * (size_t)room_start[n_rooms]);
    s.span(d_talkers, talkers, nullptr, 4 * (size_t)n_rooms * (size_t)k);
    s.span(d_level, level, nullptr, (size_t)n);
    s.span(d_csrc, nullptr, csrc, 4 * e);
    s.span(d_csrc_level, nullptr, csrc_level, e);
    s.run([&] { return contributors_launch(d_rs, d_members, n_rooms, k, d_talkers, d_level, n, d_csrc, d_csrc_level, st); });
    const int r = s.finish();
    cudaStreamDestroy(st);
    return r;
}

// ---- G.711 gateway (sb_g711.cuh) ---------------------------------------------------------------------------------------------
struct solo_b200_g711 {
    int n, device, nf, law;     // nf: 20 ms frames per row (framesize_ms / 20); law: the create default
    cudaStream_t st;            // the _host forms' stream
    G711State* d_states;
    DevBuf d_list;              // the Staging of the host calls (grown on use)
    ~solo_b200_g711() {
        if (st) cudaStreamDestroy(st);
        cudaFree(d_states); cudaFree(d_list.d);
    }
};
static int g711_reset_launch(solo_b200_g711* g, const i32* streams, int n, const i32* law, cudaStream_t st) {
    sb_g711_reset_kernel<<<(n + SB_TPB - 1) / SB_TPB, SB_TPB, 0, st>>>(g->d_states, streams, n, law, g->law);
    return launched("sb_g711_reset_kernel");
}

solo_b200_g711* solo_b200_g711_create(int n_streams, int framesize_ms, int law, int device) {
    if (n_streams <= 0 || (framesize_ms != 40 && framesize_ms != 20) || (law != G711_ULAW && law != G711_ALAW)) {
        snprintf(g_err, sizeof g_err, "g711_create: bad argument (n %d, framesize_ms %d, law %d)", n_streams, framesize_ms, law);
        return nullptr;
    }
    if (require_gpu(device)) return nullptr;
    solo_b200_g711* g = new solo_b200_g711();
    g->n = n_streams; g->device = device; g->nf = framesize_ms / 20; g->law = law;
    const bool ok = cudaStreamCreateWithFlags(&g->st, cudaStreamNonBlocking) == cudaSuccess &&
                    cudaMalloc(&g->d_states, sizeof(G711State) * (size_t)n_streams) == cudaSuccess &&
                    g711_reset_launch(g, nullptr, n_streams, nullptr, g->st) == 0 && cudaStreamSynchronize(g->st) == cudaSuccess;
    if (!ok) {
        snprintf(g_err, sizeof g_err, "g711_create: %s", cudaGetErrorString(cudaGetLastError()));
        delete g;
        return nullptr;
    }
    return g;
}

void solo_b200_g711_destroy(solo_b200_g711* g) {
    if (!g) return;
    cudaSetDevice(g->device);
    cudaStreamSynchronize(g->st);
    delete g;
}

int solo_b200_g711_state_bytes(void) { return (int)sizeof(G711State); }

static int g711_uplink_launch(solo_b200_g711* g, const u8* codes, const i32* lost, i16* pcm, u8* level, u8* flags, cudaStream_t st) {
    sb_g711_vad_kernel<<<(g->n + SB_TPB - 1) / SB_TPB, SB_TPB, 0, st>>>(g->d_states, codes, lost, flags, g->nf, g->n);
    if (int e = launched("sb_g711_vad_kernel")) return e;
    sb_g711_synth_kernel<<<(g->n + SB_G711_WARPS - 1) / SB_G711_WARPS, SB_G711_WARPS * 32, 0, st>>>(g->d_states, codes, lost, pcm, level, g->nf, g->n);
    return launched("sb_g711_synth_kernel");
}
static int g711_downlink_launch(solo_b200_g711* g, const i16* pcm, u8* codes, cudaStream_t st) {
    sb_g711_downlink_kernel<<<(g->n + SB_G711_WARPS - 1) / SB_G711_WARPS, SB_G711_WARPS * 32, 0, st>>>(g->d_states, pcm, codes, 2 * FRAME * g->nf, g->n);
    return launched("sb_g711_downlink_kernel");
}
// the device forms' pointers: the rows 16-byte aligned (16-byte loads of the codes and of the downlink's PCM, 8-byte stores of
// the uplink's PCM), lost 4-byte aligned or NULL
static int g711_device_args_ok(const solo_b200_g711* g, const void* codes, const void* pcm, const void* lost, const char* who) {
    if (!g || !codes || !pcm) { snprintf(g_err, sizeof g_err, "%s: bad argument", who); return 0; }
    if ((((uintptr_t)codes | (uintptr_t)pcm) & 15) || ((uintptr_t)lost & 3)) {
        snprintf(g_err, sizeof g_err, "%s: the G.711 and PCM rows must be 16-byte aligned and lost 4-byte aligned", who);
        return 0;
    }
    return 1;
}

int solo_b200_g711_uplink_device(solo_b200_g711* g, const uint8_t* d_g711, const int32_t* d_lost, int16_t* d_pcm, uint8_t* d_level,
                                 uint8_t* d_flags, void* cuda_stream) {
    if (!g711_device_args_ok(g, d_g711, d_pcm, d_lost, "g711_uplink_device")) return -1;
    if (!d_level || !d_flags) { snprintf(g_err, sizeof g_err, "g711_uplink_device: bad argument"); return -1; }
    CK(cudaSetDevice(g->device));
    return g711_uplink_launch(g, d_g711, d_lost, d_pcm, d_level, d_flags, (cudaStream_t)cuda_stream);
}

int solo_b200_g711_uplink_host(solo_b200_g711* g, const uint8_t* g711, const int32_t* lost, int16_t* pcm, uint8_t* level, uint8_t* flags) {
    if (!g || !g711 || !pcm || !level || !flags) { snprintf(g_err, sizeof g_err, "g711_uplink_host: bad argument"); return -1; }
    CK(cudaSetDevice(g->device));
    const size_t n = (size_t)g->n, spp8 = (size_t)FRAME * g->nf;
    const u8* d_codes; const i32* d_lost = nullptr; i16* d_pcm; u8 *d_level, *d_flags;
    Staging s(g->st, "g711_uplink", &g->d_list);
    s.span(d_codes, g711, nullptr, n * spp8);
    if (lost) s.span(d_lost, lost, nullptr, 4 * n);
    s.span(d_pcm, nullptr, pcm, 2 * n * 2 * spp8);
    s.span(d_level, nullptr, level, n);
    s.span(d_flags, nullptr, flags, n);
    s.run([&] { return g711_uplink_launch(g, d_codes, d_lost, d_pcm, d_level, d_flags, g->st); });
    return s.finish();
}

int solo_b200_g711_downlink_device(solo_b200_g711* g, const int16_t* d_pcm, uint8_t* d_g711, void* cuda_stream) {
    if (!g711_device_args_ok(g, d_g711, d_pcm, nullptr, "g711_downlink_device")) return -1;
    CK(cudaSetDevice(g->device));
    return g711_downlink_launch(g, d_pcm, d_g711, (cudaStream_t)cuda_stream);
}

int solo_b200_g711_downlink_host(solo_b200_g711* g, const int16_t* pcm, uint8_t* g711) {
    if (!g || !pcm || !g711) { snprintf(g_err, sizeof g_err, "g711_downlink_host: bad argument"); return -1; }
    CK(cudaSetDevice(g->device));
    const size_t n = (size_t)g->n, spp8 = (size_t)FRAME * g->nf;
    const i16* d_pcm; u8* d_codes;
    Staging s(g->st, "g711_downlink", &g->d_list);
    s.span(d_pcm, pcm, nullptr, 2 * n * 2 * spp8);
    s.span(d_codes, nullptr, g711, n * spp8);
    s.run([&] { return g711_downlink_launch(g, d_pcm, d_codes, g->st); });
    return s.finish();
}

int solo_b200_g711_reset(solo_b200_g711* g, const int32_t* streams, int n, const int32_t* law, void* cuda_stream) {
    if (!list_args_ok(g, streams, n, "g711_reset") || !streams_ok(streams, n, g->n, "g711_reset")) return -1;
    for (int i = 0; law && i < n; i++)
        if (law[i] != -1 && law[i] != G711_ULAW && law[i] != G711_ALAW) {
            snprintf(g_err, sizeof g_err, "g711_reset: law %d of stream %d is not 0 (mu-law) or 1 (A-law)", law[i], streams[i]);
            return -1;
        }
    if (n == 0) return 0;
    CK(cudaSetDevice(g->device));
    cudaStream_t st = (cudaStream_t)cuda_stream;
    const i32 *d_streams, *d_law = nullptr;
    Staging s(st, "g711_reset", &g->d_list);
    s.span(d_streams, streams, nullptr, 4 * (size_t)n);
    if (law) s.span(d_law, law, nullptr, 4 * (size_t)n);
    s.run([&] { return g711_reset_launch(g, d_streams, n, d_law, st); });
    return s.finish();
}

// ---- multi-GPU ingest through peer memory --------------------------------------------------------------------------------
// The *_device entry points take any device-visible address.  With peer access enabled, a rank passes rows of a buffer that
// lives in ANOTHER GPU's HBM (mapped through CUDA IPC by the caller): the band-split kernel then pulls its PCM rows over
// NVLink / NVSwitch (bulk copies) and the entropy-coding / decoder kernels push their result rows back -- the "scatter" and
// "gather" of a single-ingest deployment happen inside the kernels that consume / produce the data.
int solo_b200_enable_peer_access(int device, int peer_device) {
    if (device == peer_device) return 0;
    if (require_gpu(device)) return -2;
    int can = 0;
    CK(cudaDeviceCanAccessPeer(&can, device, peer_device));
    if (!can) { snprintf(g_err, sizeof g_err, "device %d cannot access device %d", device, peer_device); return -1; }
    cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return 0; }
    if (e != cudaSuccess) return fail("cudaDeviceEnablePeerAccess", e);
    return 0;
}

// ---- single-stream drop-in entry points (AGR_JC1_SDK_API.h) -------------------------------------------------------
// A handle is a SLOT of a process-wide, lazily grown arena: segments of SB_ARENA_SEG streams (ordinary batch objects with a
// single CUDA stream instead of SB_PIPE_STREAMS, and one set of staging buffers per segment, shared by its slots).  Init
// takes a free slot of a segment with the same packet layout and (re)initialises that one stream on the device; Uninit gives
// it back.  10 000 handles are 40 segments = 40 CUDA streams and 240 device allocations, not 10 000 batches.  Calls on
// handles of the same segment are serialised by the segment's mutex; different segments run concurrently.
// Same names / return conventions as AGR_BWE_SDK_API.c:11-296 and libBWE/AGR_BWE_init.c:6-76.
extern "C++" {
static constexpr int SB_ARENA_SEG = 256;
struct ArenaKey { int device, samplerate, framesize_ms, joint; };
template <class B> struct ArenaSeg {
    ArenaKey key;
    B* b;
    std::vector<char> used;
    int n_used;
    std::mutex mu;
};
template <class B> struct Handle { unsigned magic; ArenaSeg<B>* seg; int slot; int coded; };   // coded: a packet went through
typedef Handle<solo_b200_enc_batch> EncHandle;
typedef Handle<solo_b200_dec_batch> DecHandle;
static const unsigned ENC_MAGIC = 0x53424531u, DEC_MAGIC = 0x53424431u;   // "SBE1", "SBD1"
static std::mutex g_arena_mu;
static std::vector<ArenaSeg<solo_b200_enc_batch>*> g_enc_segs;
static std::vector<ArenaSeg<solo_b200_dec_batch>*> g_dec_segs;

template <class B> static ArenaSeg<B>* arena_take(std::vector<ArenaSeg<B>*>& segs, ArenaKey k, int* slot) {
    for (auto* sg : segs)
        if (sg->key.device == k.device && sg->key.samplerate == k.samplerate && sg->key.framesize_ms == k.framesize_ms && sg->key.joint == k.joint &&
            sg->n_used < SB_ARENA_SEG)
            for (int i = 0; i < SB_ARENA_SEG; i++)
                if (!sg->used[i]) { sg->used[i] = 1; sg->n_used++; *slot = i; return sg; }
    return nullptr;
}
template <class B> static void arena_release(ArenaSeg<B>* sg, int slot) {   // under g_arena_mu
    sg->used[slot] = 0;
    sg->n_used--;
}
// A slot on the current device: a free one of a segment with this packet layout, or the first one of a new segment made by
// create(device).  init(batch, slot) enqueues the (re)initialisation of that one stream with the caller's settings and
// returns its launch error.
template <class B, class Create, class Init>
static Handle<B>* arena_open(std::vector<ArenaSeg<B>*>& segs, unsigned magic, int samplerate, int framesize_ms, int joint_enable, const char* who,
                             const char* what, Create create, Init init) {
    int dev = 0;
    cudaGetDevice(&dev);
    const ArenaKey k = {dev, samplerate, framesize_ms, joint_enable ? 1 : 0};
    std::lock_guard<std::mutex> lk(g_arena_mu);
    int slot = -1;
    auto* sg = arena_take(segs, k, &slot);
    if (!sg) {
        B* b = create(dev);
        if (!b) { fprintf(stderr, "solo_b200: %s failed: %s\n", who, g_err); return nullptr; }
        sg = new ArenaSeg<B>();
        sg->key = k; sg->b = b; sg->used.assign(SB_ARENA_SEG, 0); sg->n_used = 0;
        segs.push_back(sg);
        sg->used[0] = 1; sg->n_used = 1; slot = 0;
    }
    {
        std::lock_guard<std::mutex> lk2(sg->mu);
        cudaSetDevice(dev);
        if (init(sg->b, slot) || cudaStreamSynchronize(sg->b->st[0]) != cudaSuccess) { arena_release(sg, slot); fprintf(stderr, "solo_b200: %s slot init failed\n", what); return nullptr; }
    }
    return new Handle<B>{magic, sg, slot};
}
template <class B> static int arena_close(void* handle, unsigned magic) {
    Handle<B>* h = (Handle<B>*)handle;
    if (!h || h->magic != magic) return -1;
    {
        std::lock_guard<std::mutex> lk(g_arena_mu);
        arena_release(h->seg, h->slot);
    }
    h->magic = 0;
    delete h;
    return 0;
}
// the activity report of a handle's last packet, from its slot of the segment
template <class B> static int handle_activity(void* handle, unsigned magic, u8* level, u8* flags) {
    Handle<B>* h = (Handle<B>*)handle;
    if (!h || h->magic != magic || !level || !flags) { snprintf(g_err, sizeof g_err, "bad argument (NULL or foreign handle)"); return -1; }
    if (!h->coded) { snprintf(g_err, sizeof g_err, "activity: the handle has not coded a packet yet"); return -1; }
    B* b = h->seg->b;
    std::lock_guard<std::mutex> lk(h->seg->mu);
    CK(cudaSetDevice(b->device));
    return activity_host(b, h->slot, 1, level, flags);
}
}  // extern "C++"

void* AGR_Sate_Encoder_Init(USER_Ctrl_enc* enc_Ctrl) {
    if (!enc_Ctrl) return nullptr;
    if (enc_Ctrl->targetRate_bps <= 0) enc_Ctrl->targetRate_bps = 15600;  // written back (AGR_BWE_SDK_API.c:34-36)
    if (enc_Ctrl->joint_enable && (enc_Ctrl->joint_mode < 0 || enc_Ctrl->joint_mode > 3)) {
        printf("Error in setting joint mode! It must be 0, 1, 2, 3\n");
        return nullptr;
    }
    if (check_enc_ctrl(enc_Ctrl)) { fprintf(stderr, "solo_b200: AGR_Sate_Encoder_Init: unsupported configuration: %s\n", g_err); return nullptr; }
    return arena_open(g_enc_segs, ENC_MAGIC, enc_Ctrl->samplerate, enc_Ctrl->framesize_ms, enc_Ctrl->joint_enable, "AGR_Sate_Encoder_Init", "encoder",
                      [&](int dev) { return enc_batch_create_impl(SB_ARENA_SEG, enc_Ctrl, dev, 1); },
                      [&](solo_b200_enc_batch* b, int slot) { return enc_init_launch(b, slot, 1, enc_Ctrl); });   // the caller's settings
}
SKP_int32 AGR_Sate_Encoder_Encode(void* SATEEnc_State, const SKP_int16* AGR_Sate_PCM, SKP_uint8* AGR_Sate_Bit, SKP_int32 AGR_Sate_Buf_Size,
                                  SKP_int16* nBytesOut) {
    EncHandle* h = (EncHandle*)SATEEnc_State;
    if (!h || h->magic != ENC_MAGIC) return -1;
    solo_b200_enc_batch* b = h->seg->b;
    const int cap = MAX_PAYLOAD + 8;
    uint8_t tmp[MAX_PAYLOAD + 8];
    int16_t nb[2] = {0, 0};
    {
        std::lock_guard<std::mutex> lk(h->seg->mu);
        if (cudaSetDevice(b->device) != cudaSuccess || staging(b, cap) || enc_host_range(b, h->slot, 1, AGR_Sate_PCM, tmp, cap, nb, b->st[0]) ||
            cudaStreamSynchronize(b->st[0]) != cudaSuccess) {
            fprintf(stderr, "solo_b200: encode failed: %s\n", g_err[0] ? g_err : cudaGetErrorString(cudaGetLastError()));
            return -1;
        }
        h->coded = 1;
    }
    // DTX packets return the high-band bytes (4 per 20 ms frame) with nBytesOut[0] == 0 (App. A Q16)
    int total = nb[0] ? nb[0] : b->hb_bytes;
    int n = total < AGR_Sate_Buf_Size ? total : AGR_Sate_Buf_Size;
    if (n < 0) n = 0;
    memcpy(AGR_Sate_Bit, tmp, n);
    nBytesOut[0] = nb[0];
    nBytesOut[1] = nb[1];
    return n;
}
int AGR_Sate_Encoder_Uninit(void* SATEEnc_State) { return arena_close<solo_b200_enc_batch>(SATEEnc_State, ENC_MAGIC); }
// the handle's slot gets the settings of the batched call (-1 leaves one alone); encodes of the handle are synchronous, so
// the next one sees them
int solo_b200_encoder_set_control(void* SATEEnc_State, int32_t rate_bps, int32_t dtx, int32_t loss_perc) {
    EncHandle* h = (EncHandle*)SATEEnc_State;
    if (!h || h->magic != ENC_MAGIC) return -1;
    const i32 v[3] = {rate_bps, dtx, loss_perc};
    if (!control_in_range(&v[0], &v[1], &v[2], 1)) return -1;
    solo_b200_enc_batch* b = h->seg->b;
    std::lock_guard<std::mutex> lk(h->seg->mu);
    CK(cudaSetDevice(b->device));
    return enc_control_host(b, h->slot, 1, v[0] != -1 ? &v[0] : nullptr, v[1] != -1 ? &v[1] : nullptr, v[2] != -1 ? &v[2] : nullptr, b->st[0]);
}

void* AGR_Sate_Decoder_Init(USER_Ctrl_dec* dec_Ctrl) {
    if (!dec_Ctrl) return nullptr;
    if (dec_Ctrl->joint_enable && (dec_Ctrl->joint_mode < 0 || dec_Ctrl->joint_mode > 3)) {
        fprintf(stderr, "Error in setting joint mode! It must be 0, 1, 2, 3\n");
        return nullptr;
    }
    if (check_dec_ctrl(dec_Ctrl)) {
        snprintf(g_err, sizeof g_err, "bad decoder configuration");
        fprintf(stderr, "solo_b200: AGR_Sate_Decoder_Init: unsupported configuration\n");
        return nullptr;
    }
    // SOLO_B200_DEC_ARITH, read at every Init: unset or "flp" = the float build's PCM, "fix" = the fixed-point build's
    const char* e = getenv("SOLO_B200_DEC_ARITH");
    int arith;
    if (!e || !strcmp(e, "flp")) arith = SOLO_B200_DEC_FLP;
    else if (!strcmp(e, "fix")) arith = SOLO_B200_DEC_FIX;
    else { fprintf(stderr, "solo_b200: AGR_Sate_Decoder_Init: SOLO_B200_DEC_ARITH must be \"flp\" or \"fix\", not \"%s\"\n", e); return nullptr; }
    if (check_dec_arith(dec_Ctrl, arith)) { fprintf(stderr, "solo_b200: AGR_Sate_Decoder_Init: %s\n", g_err); return nullptr; }
    // the arithmetic is a property of the slot, not of the segment: one segment holds handles of both kinds
    return arena_open(g_dec_segs, DEC_MAGIC, dec_Ctrl->samplerate, dec_Ctrl->framesize_ms, dec_Ctrl->joint_enable, "AGR_Sate_Decoder_Init", "decoder",
                      [&](int dev) { return dec_batch_create_impl(SB_ARENA_SEG, dec_Ctrl, dev, 1, SOLO_B200_DEC_FLP, dec_Ctrl->samplerate); },
                      [&](solo_b200_dec_batch* b, int slot) {
                          return dec_init_launch(b, slot, 1, dec_Ctrl->useMDIndex, dec_Ctrl->framesize_ms, dec_Ctrl->joint_enable, arith);
                      });
}
SKP_int32 AGR_Sate_Decoder_Decode(void* SATEDec_State, SKP_int16* AGR_Sate_PCM, SKP_int16* nSamplesOut, const SKP_uint8* AGR_Sate_Bit,
                                  SKP_int16 nBytes[], SKP_int32 lostflag) {
    DecHandle* h = (DecHandle*)SATEDec_State;
    if (!h || h->magic != DEC_MAGIC) return -1;
    if (nBytes[0] <= 0) return -1;
    solo_b200_dec_batch* b = h->seg->b;
    const int cap = MAX_PAYLOAD + 8;
    uint8_t tmp[MAX_PAYLOAD + 8];
    memset(tmp, 0, sizeof tmp);
    int n0 = nBytes[0] > cap ? cap : nBytes[0];
    memcpy(tmp, AGR_Sate_Bit, n0);
    int16_t nb[2] = {nBytes[0], nBytes[1]};
    int32_t flag = lostflag, ret = 0;
    {
        std::lock_guard<std::mutex> lk(h->seg->mu);
        if (cudaSetDevice(b->device) != cudaSuccess || dec_staging(b, cap) ||
            dec_host_range(b, h->slot, 1, AGR_Sate_PCM, tmp, cap, nb, &flag, &ret, b->st[0]) || cudaStreamSynchronize(b->st[0]) != cudaSuccess) {
            fprintf(stderr, "solo_b200: decode failed: %s\n", g_err[0] ? g_err : cudaGetErrorString(cudaGetLastError()));
            return -1;
        }
        h->coded = 1;
    }
    // the reference rewrites the caller's nBytes[] while splitting the payload (AGR_BWE_decode_frame_FLP.c:171-190)
    dec_split_lengths(nb, lostflag, b->hb_bytes);
    nBytes[0] = nb[0];
    nBytes[1] = nb[1];
    *nSamplesOut = (SKP_int16)b->spp;
    return ret;
}
SKP_int32 AGR_Sate_Decoder_Uninit(void* SATEDec_State) { return arena_close<solo_b200_dec_batch>(SATEDec_State, DEC_MAGIC); }
int solo_b200_encoder_last_activity(void* SATEEnc_State, uint8_t* level, uint8_t* flags) {
    return handle_activity<solo_b200_enc_batch>(SATEEnc_State, ENC_MAGIC, level, flags);
}
int solo_b200_decoder_last_activity(void* SATEDec_State, uint8_t* level, uint8_t* flags) {
    return handle_activity<solo_b200_dec_batch>(SATEDec_State, DEC_MAGIC, level, flags);
}
/* arena bookkeeping for tests: segments and slots in use (encoder, decoder) */
int solo_b200_arena_stats(int out[4]) {
    std::lock_guard<std::mutex> lk(g_arena_mu);
    int eu = 0, du = 0;
    for (auto* sg : g_enc_segs) eu += sg->n_used;
    for (auto* sg : g_dec_segs) du += sg->n_used;
    if (out) { out[0] = (int)g_enc_segs.size(); out[1] = eu; out[2] = (int)g_dec_segs.size(); out[3] = du; }
    return 0;
}

}  // extern "C"
