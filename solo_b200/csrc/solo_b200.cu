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
// Persistent per-stream state lives in device arrays (EncState / DecState) that never leave the GPU between packets;
// a wave is processed as a few chunks of streams on internal CUDA streams (Pipe).  The host code below is the C ABI:
// the batched entry points of include/solo_b200.h and the reference's six functions of include/AGR_JC1_SDK_API.h.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <mutex>
#include <vector>

#include "../../include/solo_b200.h"
#include "sb_dec.cuh"
#include "sb_enc.cuh"
#include "sb_nsq_warp.cuh"

using namespace sb;

// ---------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------
#define SB_TPB 64
#ifndef SB_DEC_TPB
#define SB_DEC_TPB 64
#endif
#ifndef SB_DECODE_LOCAL_STATE
#define SB_DECODE_LOCAL_STATE 0
#endif
// the warp-per-stream analysis kernels live in sb_analysis.cu
extern "C" int sb_launch_enc_analysis_warp(void* states, void* scratch, const void* bands, int spp, int n, void* stream);
extern "C" int sb_launch_enc_hb_warp(void* states, void* scratch, const void* bands, int spp, int n, void* stream);
#ifndef SB_FINISH_MINB
#define SB_FINISH_MINB 8     // 128 registers: every stream of a chunk resident
#endif
#ifndef SB_DECODE_MINB
#define SB_DECODE_MINB 8
#endif

__global__ void __launch_bounds__(SB_TPB) sb_enc_init_kernel(EncState* states, int n, int rate, int dtx, int mdi, int framesize_ms, int joint_hb) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) enc_state_init(&states[s], rate, dtx, mdi, framesize_ms, joint_hb);
}

// ---- stage A0: QMF band split, one warp per stream, PCM tile fetched by the TMA engine ----------------------------------
// The split is the one part of the analysis without a recurrence: 320 (160) output pairs of a 64-tap symmetric FIR per
// packet.  A block takes SB_QMF_SPB consecutive streams; their PCM rows are contiguous in HBM, so ONE bulk asynchronous copy
// (cp.async.bulk -> UBLKCP, completion on an mbarrier) brings the whole tile into shared memory while the warps load their
// filter memories; each lane then produces output pairs k = lane, lane + 32, ... (products summed mod 2^32: order-free).
// Against the split inside kernel A this raised end-to-end throughput and left device-resident throughput unchanged;
// larger blocks (8 streams) were slower device-resident because they cannot start while kernel B holds the shared memory.
#ifndef SB_QMF_SPB
#define SB_QMF_SPB 1        // one-warp blocks of 2.8 KB: they fit in the shared memory the quantiser kernel leaves free on an SM
#endif
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

#ifndef SB_NSQ_WARPS
#define SB_NSQ_WARPS 1      // one warp = two streams = 2 x 8.2 KB of shared memory; 12 blocks (24 streams) per SM
#endif
#ifndef SB_NSQ_MINB
#define SB_NSQ_MINB 12     // <= 170 registers per thread
#endif
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
    EncScratch* scr = &scratch[s];
    const int nf = states[s].frames_per_packet;
    for (int f = 0; f < nf; f++)
        nsq_del_dec_warp(*S, states[s].nsq, &scr->c[f], scr->xfw[f], scr->q_md[f][0], scr->q_md[f][1], scr->r16[f], &scr->nsq_rand[0][0][0]);
}

// Entropy coding and payload assembly, TWO threads per stream: thread k range-codes description k of both frames (the two
// coders share nothing but read-only frame parameters) and packs high-band frame k; the pair exchanges lengths and status
// by shuffle and writes the row [MD1 | MD2 | HB].  Same result as the one-thread model enc_packet_finish() (sb_enc.cuh).
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
    const int nf = st->frames_per_packet, nhb = nf * FRAME / st->hb_frame, hb_bytes = 4 * nhb;
    RangeEnc rc;
    rc_enc_init(&rc, rcbuf, MAX_PAYLOAD);
    for (int f = 0; f < nf; f++) {
        encode_parameters(&rc, st, &scr->c[f], k, f, scr->vadFlag[f], scr->q_md[f][k]);
        // frame terminator: MORE_FRAMES (1) while frames follow in this packet, LAST_FRAME (0) after the last one
        rc_encode(&rc, f < nf - 1 ? 1 : 0, SB_T(frame_term_cdf));
    }
    int nb_k;
    rc_get_length(&rc, &nb_k);
    const int ok_k = rc.error ? 0 : 1;
    const int nb_o = __shfl_xor_sync(m, nb_k, 1), ok_o = __shfl_xor_sync(m, ok_k, 1);
    const int nb0 = k ? nb_o : nb_k, nb1 = k ? nb_k : nb_o, ok0 = k ? ok_o : ok_k, ok1 = k ? ok_k : ok_o;
    const int ok = ok0 && ok1 && nb0 + nb1 <= MAX_PAYLOAD;        // pnBytesOut[0] >= nMDBytes (encode_frame_FIX.c:245)
    const int dtx = scr->dtx_drop;
    if (k == 0 ? ok0 : ok) {
        rc_enc_wrap_up(&rc);
        const int off = k ? nb0 : 0;
        for (int i = 0; i < nb_k; i++) if (off + i < cap) out[off + i] = rcbuf[i];
    }
    u8 hb[4];
    const int my_hb = k < nhb;
    if (my_hb) hb_pack_frame(scr->hb_lsp_idx[k], scr->hb_nrg0[k], &scr->r16[0][0] + k * st->hb_frame, hb, st->hb_frame >> 2);
    __syncwarp(m);      // a rejected or dropped packet's high-band bytes land on top of description 1's
    const int lb = (ok && !dtx) ? nb0 + nb1 : 0;
    if (my_hb) for (int i = 0; i < 4; i++) if (lb + 4 * k + i < cap) out[lb + 4 * k + i] = hb[i];
    if (k == 0) {
        nbytes[2 * s] = lb ? (i16)(lb + hb_bytes) : 0;
        nbytes[2 * s + 1] = lb ? (i16)(nb1 + hb_bytes) : 0;
    }
}

__global__ void __launch_bounds__(SB_TPB) sb_dec_init_kernel(DecState* states, int n, int mdi, int framesize_ms, int joint_hb) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s < n) dec_state_init(&states[s], mdi, framesize_ms, joint_hb);
}

__global__ void __launch_bounds__(SB_DEC_TPB, SB_DECODE_MINB) sb_decode_kernel(DecState* states, const u8* __restrict__ bits, int cap,
                                                           const i16* __restrict__ nbytes, const i32* __restrict__ lostflag,
                                                           i32* __restrict__ ret, i32* __restrict__ ret_int, DecStale* stale,
                                                           i16* __restrict__ band_low, float* __restrict__ band_high, int spp, int n) {
    int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    DecPacketWork W;
    i16 nb[2] = {nbytes[2 * s], nbytes[2 * s + 1]};
    const DecBands bands = {band_low + (size_t)s * (spp / 2), band_high + (size_t)s * (spp / 2)};
#if SB_DECODE_LOCAL_STATE
    DecState st = states[s];
    i32 r = dec_packet(&st, &W, nullptr, bits + (size_t)s * cap, cap, nb, lostflag[s], &stale[s], &bands);
    states[s] = st;
#else
    i32 r = dec_packet(&states[s], &W, nullptr, bits + (size_t)s * cap, cap, nb, lostflag[s], &stale[s], &bands);
#endif
    if (ret) ret[s] = r;
    ret_int[s] = r;
}

// ---- synthesis filter bank + float -> int16, one warp per stream (AGR_BWE_qmf.c:86-182, AGR_BWE_decode_frame_FLP.c:222-231) ----
// 160 (80) independent groups of four outputs per packet: lanes over groups, band signals and filter memories staged in
// shared memory; the PCM row is written with 8-byte stores, 256 contiguous bytes per warp instruction.
#ifndef SB_SYN_WARPS
#define SB_SYN_WARPS 4
#endif
__global__ void __launch_bounds__(SB_SYN_WARPS * 32) sb_dec_synth_kernel(DecState* states, const i16* __restrict__ band_low, const float* __restrict__ band_high,
                                                                        const i32* __restrict__ ret_int, i16* __restrict__ pcm, int spp, int n) {
    __shared__ float xx[SB_SYN_WARPS][2][32 + PACKET / 2];
    __shared__ float coef[64];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < 64; i += blockDim.x) coef[i] = SB_T(qmf_flt)[i];
    __syncthreads();
    const int s = blockIdx.x * SB_SYN_WARPS + w;
    if (s >= n || ret_int[s] < 0) return;         // a rejected packet leaves its PCM row and the filter memories alone
    const int N2 = spp >> 1;
    float* xx1 = xx[w][0];
    float* xx2 = xx[w][1];
    DecState* st = &states[s];
    const i16* lo = band_low + (size_t)s * N2;
    const float* hi = band_high + (size_t)s * N2;
    for (int i = lane; i < N2; i += 32) { xx1[i] = (float)lo[N2 - 1 - i]; xx2[i] = hi[N2 - 1 - i]; }
    xx1[N2 + lane] = st->g0_mem[2 * lane + 1];
    xx2[N2 + lane] = st->g1_mem[2 * lane + 1];
    __syncwarp();
    i16* out = pcm + (size_t)s * spp;
    for (int g = lane; g < N2 / 2; g += 32) {
        float y4[4];
        qmf_synth_group(xx1, xx2, coef, N2, 2 * g, y4);
        i32 t[4];
#pragma unroll
        for (int q = 0; q < 4; q++) { i32 v = trunc_i32((double)y4[q]); t[q] = v > 32767 ? 32767 : (v < -32768 ? -32768 : v); }
        int2 pk;
        pk.x = (t[0] & 0xffff) | (t[1] << 16);
        pk.y = (t[2] & 0xffff) | (t[3] << 16);
        reinterpret_cast<int2*>(out)[g] = pk;
    }
    __syncwarp();
    st->g0_mem[2 * lane + 1] = xx1[lane];
    st->g1_mem[2 * lane + 1] = xx2[lane];
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
static void count_launch() {
    std::lock_guard<std::mutex> lk(g_mu);
    g_launches++;
}

// A packet wave is cut into chunks of streams that run on a few internal CUDA streams: the copies of one chunk overlap
// the kernels of another (host entry points), and the blocks of one chunk's kernel fill the SMs that the tail of another
// chunk's kernel leaves idle (all four kernels are latency-bound at a fixed number of resident warps per SM).
#define SB_PIPE_STREAMS 4
struct Pipe {
    cudaStream_t st[SB_PIPE_STREAMS];
    cudaEvent_t fork, join[SB_PIPE_STREAMS];
    bool ok;
};
static int g_chunks = -1;   // -1: SOLO_B200_CHUNKS or the defaults below
// Default: the host entry points cut a wave in three (the copies of one chunk hide behind the kernels of its neighbours;
// three beat two, four and six in an earlier comparison, not repeated on H100); the device entry points launch every
// kernel once for the whole batch.
static int pipe_chunks(int n, bool host_copies) {
    if (g_chunks < 0) {
        const char* e = getenv("SOLO_B200_CHUNKS");
        g_chunks = e ? atoi(e) : 0;
        if (g_chunks < 0) g_chunks = 0;
        if (g_chunks > 64) g_chunks = 64;
    }
    int c = g_chunks ? g_chunks : (host_copies ? 3 : 1);
    while (c > 1 && n / c < 2048) c--;   // small batches: fewer, larger chunks
    return c;
}
static int pipe_create(Pipe* p) {
    p->ok = false;
    for (int i = 0; i < SB_PIPE_STREAMS; i++) {
        if (cudaStreamCreateWithFlags(&p->st[i], cudaStreamNonBlocking) != cudaSuccess) return -2;
        if (cudaEventCreateWithFlags(&p->join[i], cudaEventDisableTiming) != cudaSuccess) return -2;
    }
    if (cudaEventCreateWithFlags(&p->fork, cudaEventDisableTiming) != cudaSuccess) return -2;
    p->ok = true;
    return 0;
}
static void pipe_destroy(Pipe* p) {   // also after a partial pipe_create: members are zero until created
    for (int i = 0; i < SB_PIPE_STREAMS; i++) {
        if (p->st[i]) { cudaStreamSynchronize(p->st[i]); cudaStreamDestroy(p->st[i]); p->st[i] = nullptr; }
        if (p->join[i]) { cudaEventDestroy(p->join[i]); p->join[i] = nullptr; }
    }
    if (p->fork) { cudaEventDestroy(p->fork); p->fork = nullptr; }
    p->ok = false;
}
// chunk c of C over n streams, boundaries on multiples of 64 streams (block size of the thread-per-stream kernels)
static void chunk_bounds(int n, int C, int c, int* lo, int* hi) {
    long long per = ((long long)n + C - 1) / C;
    per = (per + 63) / 64 * 64;
    long long a = per * c, b = per * (c + 1);
    *lo = (int)(a > n ? n : a);
    *hi = (int)(b > n ? n : b);
}

struct solo_b200_enc_batch {
    int n, device;
    int spp;                    // samples per packet and stream: 640 (40 ms) or 320 (20 ms)
    int hb_bytes;               // high-band bytes per packet: 4 per high-band frame
    EncState* d_states;
    EncScratch* d_scratch;
    i16* d_bands;               // [n][spp]: low band | high band of the packet, written by the QMF kernel
    // staging for the *_host entry points
    i16* d_pcm; u8* d_bits; i16* d_nbytes; int bits_cap;
    cudaStream_t stream;
    Pipe pipe;
};
struct solo_b200_dec_batch {
    int n, device;
    int spp, hb_bytes;
    DecState* d_states;
    DecStale* d_stale;          // payload copies that outlive a packet call (only touched after a corrupted packet, see sb_dec.cuh)
    i16* d_pcm; u8* d_bits; i16* d_nbytes; i32* d_flags; i32* d_ret; int bits_cap;
    i16* d_band_low; float* d_band_high; i32* d_ret_int;   // decoder kernel -> synthesis kernel
    cudaStream_t stream;
    Pipe pipe;
};

// Supported configurations (AGR_BWE_SDK_API.c:40-81): 16 kHz input; no joint coding with 40 or 20 ms packets ("40ms 2MD",
// "20ms 2MD"); joint mode 1 (one 40 ms high-band frame per 40 ms packet).  Joint modes 0, 2, 3 are "Unsupport" in the
// reference as well; 32 kHz input is out of scope here.
static int check_modes(int samplerate, int framesize_ms, int joint_enable, int joint_mode) {
    if (samplerate != 16000) return -1;
    if (!joint_enable) return (framesize_ms == 40 || framesize_ms == 20) ? 0 : -1;
    return (joint_mode == 1 && framesize_ms == 40) ? 0 : -1;
}
static int check_enc_ctrl(const USER_Ctrl_enc* c) { return c ? check_modes(c->samplerate, c->framesize_ms, c->joint_enable, c->joint_mode) : -1; }
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

extern "C" {

const char* solo_b200_last_error(void) { return g_err; }
long long solo_b200_kernel_launches(void) { std::lock_guard<std::mutex> lk(g_mu); return g_launches; }
int solo_b200_enc_state_bytes(void) { return (int)sizeof(EncState); }
int solo_b200_dec_state_bytes(void) { return (int)sizeof(DecState); }
void solo_b200_set_chunks(int chunks) { g_chunks = chunks < 0 ? 0 : (chunks > 64 ? 64 : chunks); }   // 0: the defaults
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
static solo_b200_enc_batch* enc_batch_create_impl(int n_streams, const USER_Ctrl_enc* ctrl, int device, bool with_pipe);
solo_b200_enc_batch* solo_b200_enc_batch_create(int n_streams, const USER_Ctrl_enc* ctrl, int device) { return enc_batch_create_impl(n_streams, ctrl, device, true); }
static solo_b200_enc_batch* enc_batch_create_impl(int n_streams, const USER_Ctrl_enc* ctrl, int device, bool with_pipe) {
    if (n_streams <= 0 || check_enc_ctrl(ctrl)) { snprintf(g_err, sizeof g_err, "bad encoder configuration"); return nullptr; }
    if (require_gpu(device)) return nullptr;
    solo_b200_enc_batch* b = new solo_b200_enc_batch();
    memset(b, 0, sizeof *b);
    b->n = n_streams; b->device = device; b->spp = 16 * ctrl->framesize_ms; b->hb_bytes = hb_bytes_of(ctrl->framesize_ms, ctrl->joint_enable);
    if (cudaMalloc(&b->d_states, sizeof(EncState) * (size_t)n_streams) != cudaSuccess ||
        cudaMalloc(&b->d_scratch, sizeof(EncScratch) * (size_t)n_streams) != cudaSuccess ||
        cudaMalloc(&b->d_bands, sizeof(i16) * (size_t)b->spp * (size_t)n_streams) != cudaSuccess ||
        cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking) != cudaSuccess || (with_pipe && pipe_create(&b->pipe) != 0) ||
        cudaFuncSetAttribute(sb_enc_nsq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(SB_NSQ_SPB * sizeof(NsqSmem))) != cudaSuccess) {
        fail("enc_batch_create", cudaGetLastError());
        solo_b200_enc_batch_destroy(b); return nullptr;
    }
    int rate = ctrl->targetRate_bps <= 0 ? 15600 : ctrl->targetRate_bps;
    sb_enc_init_kernel<<<(n_streams + SB_TPB - 1) / SB_TPB, SB_TPB, 0, b->stream>>>(b->d_states, n_streams, rate, ctrl->dtx_enable, ctrl->useMDIndex, ctrl->framesize_ms, ctrl->joint_enable ? 1 : 0);
    count_launch();
    cudaError_t e = cudaStreamSynchronize(b->stream);
    if (e != cudaSuccess) { fail("enc init kernel", e); solo_b200_enc_batch_destroy(b); return nullptr; }
    return b;
}

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
    sb_enc_vad_kernel<<<(n + SB_TPB - 1) / SB_TPB, SB_TPB, 0, st>>>(states, scratch, bands, b->spp, n);
    { int e = sb_launch_enc_hb_warp(states, scratch, bands, b->spp, n, st); if (e) return fail("high-band analysis launch", (cudaError_t)e); }
    { int e = sb_launch_enc_analysis_warp(states, scratch, bands, b->spp, n, st); if (e) return fail("analysis launch", (cudaError_t)e); }
    sb_enc_shape_post_kernel<<<(8 * n + 127) / 128, 128, 0, st>>>(states, scratch, n);
    sb_enc_prefilter_kernel<<<dim3((n + SB_TPB - 1) / SB_TPB, 2), SB_TPB, 0, st>>>(states, scratch, n);
    for (int i = 0; i < 6; i++) count_launch();
    prof_end(st, &ev);
    prof_begin(st, 1, &ev);
    sb_enc_nsq_kernel<<<(n + SB_NSQ_SPB - 1) / SB_NSQ_SPB, SB_NSQ_WARPS * 32, SB_NSQ_SPB * sizeof(NsqSmem), st>>>(states, scratch, n);
    prof_end(st, &ev);
    prof_begin(st, 2, &ev);
    sb_enc_finish_kernel<<<(2 * n + SB_TPB - 1) / SB_TPB, SB_TPB, 0, st>>>(states, scratch, d_bits + (size_t)lo * cap, cap, d_nbytes + 2 * (size_t)lo, n);
    prof_end(st, &ev);
    count_launch(); count_launch();
    CK(cudaGetLastError());
    return 0;
}

int solo_b200_enc_batch_encode_device(solo_b200_enc_batch* b, const int16_t* d_pcm, uint8_t* d_bits, int cap, int16_t* d_nbytes, void* cuda_stream) {
    if (!b || !d_pcm || !d_bits || !d_nbytes || cap < 16) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    CK(cudaSetDevice(b->device));
    cudaStream_t user = (cudaStream_t)cuda_stream;
    const int C = pipe_chunks(b->n, false);
    if (C == 1) return enc_launch(b, 0, b->n, d_pcm, d_bits, cap, d_nbytes, user);
    // fork from the caller's stream onto the internal ones, join back: the caller sees ordinary stream semantics
    CK(cudaEventRecord(b->pipe.fork, user));
    const int S = C < SB_PIPE_STREAMS ? C : SB_PIPE_STREAMS;
    for (int i = 0; i < S; i++) CK(cudaStreamWaitEvent(b->pipe.st[i], b->pipe.fork, 0));
    for (int c = 0; c < C; c++) {
        int lo, hi;
        chunk_bounds(b->n, C, c, &lo, &hi);
        int r = enc_launch(b, lo, hi - lo, d_pcm, d_bits, cap, d_nbytes, b->pipe.st[c % S]);
        if (r) return r;
    }
    for (int i = 0; i < S; i++) {
        CK(cudaEventRecord(b->pipe.join[i], b->pipe.st[i]));
        CK(cudaStreamWaitEvent(user, b->pipe.join[i], 0));
    }
    return 0;
}

static int enc_staging(solo_b200_enc_batch* b, int cap) {
    if (!b->d_pcm) CK(cudaMalloc(&b->d_pcm, sizeof(i16) * b->spp * (size_t)b->n));
    if (!b->d_nbytes) CK(cudaMalloc(&b->d_nbytes, sizeof(i16) * 2 * (size_t)b->n));
    if (!b->d_bits || b->bits_cap < cap) {
        if (b->d_bits) cudaFree(b->d_bits);
        b->d_bits = nullptr;
        CK(cudaMalloc(&b->d_bits, (size_t)cap * b->n));
        b->bits_cap = cap;
    }
    return 0;
}

int solo_b200_enc_batch_encode_host(solo_b200_enc_batch* b, const int16_t* pcm, uint8_t* bits, int cap, int16_t* nbytes) {
    if (!b || !pcm || !bits || !nbytes || cap < 16) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    CK(cudaSetDevice(b->device));
    int r = enc_staging(b, cap);
    if (r) return r;
    const int C = pipe_chunks(b->n, true);
    const int S = C < SB_PIPE_STREAMS ? C : SB_PIPE_STREAMS;
    for (int c = 0; c < C; c++) {   // per chunk: H2D, encoder kernels, D2H -- chunks alternate over the internal streams
        int lo, hi;
        chunk_bounds(b->n, C, c, &lo, &hi);
        if (hi <= lo) continue;
        cudaStream_t st = b->pipe.st[c % S];
        const size_t m = (size_t)(hi - lo);
        CK(cudaMemcpyAsync(b->d_pcm + (size_t)lo * b->spp, pcm + (size_t)lo * b->spp, sizeof(i16) * b->spp * m, cudaMemcpyHostToDevice, st));
        r = enc_launch(b, lo, hi - lo, b->d_pcm, b->d_bits, cap, b->d_nbytes, st);
        if (r) return r;
        CK(cudaMemcpyAsync(bits + (size_t)lo * cap, b->d_bits + (size_t)lo * cap, (size_t)cap * m, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(nbytes + 2 * (size_t)lo, b->d_nbytes + 2 * (size_t)lo, sizeof(i16) * 2 * m, cudaMemcpyDeviceToHost, st));
    }
    for (int i = 0; i < S; i++) CK(cudaStreamSynchronize(b->pipe.st[i]));
    return 0;
}

void solo_b200_enc_batch_destroy(solo_b200_enc_batch* b) {
    if (!b) return;
    cudaSetDevice(b->device);
    if (b->stream) cudaStreamSynchronize(b->stream);
    pipe_destroy(&b->pipe);
    cudaFree(b->d_states); cudaFree(b->d_scratch); cudaFree(b->d_bands); cudaFree(b->d_pcm); cudaFree(b->d_bits); cudaFree(b->d_nbytes);
    cudaStreamDestroy(b->stream);
    delete b;
}

// ---- decoder batch --------------------------------------------------------------------------------
static solo_b200_dec_batch* dec_batch_create_impl(int n_streams, const USER_Ctrl_dec* ctrl, int device, bool with_pipe);
solo_b200_dec_batch* solo_b200_dec_batch_create(int n_streams, const USER_Ctrl_dec* ctrl, int device) { return dec_batch_create_impl(n_streams, ctrl, device, true); }
static solo_b200_dec_batch* dec_batch_create_impl(int n_streams, const USER_Ctrl_dec* ctrl, int device, bool with_pipe) {
    if (n_streams <= 0 || check_dec_ctrl(ctrl)) { snprintf(g_err, sizeof g_err, "bad decoder configuration"); return nullptr; }
    if (require_gpu(device)) return nullptr;
    solo_b200_dec_batch* b = new solo_b200_dec_batch();
    memset(b, 0, sizeof *b);
    b->n = n_streams; b->device = device; b->spp = 16 * ctrl->framesize_ms; b->hb_bytes = hb_bytes_of(ctrl->framesize_ms, ctrl->joint_enable);
    if (cudaMalloc(&b->d_states, sizeof(DecState) * (size_t)n_streams) != cudaSuccess ||
        cudaMalloc(&b->d_stale, sizeof(DecStale) * (size_t)n_streams) != cudaSuccess ||
        cudaMalloc(&b->d_band_low, sizeof(i16) * (size_t)(b->spp / 2) * (size_t)n_streams) != cudaSuccess ||
        cudaMalloc(&b->d_band_high, sizeof(float) * (size_t)(b->spp / 2) * (size_t)n_streams) != cudaSuccess ||
        cudaMalloc(&b->d_ret_int, sizeof(i32) * (size_t)n_streams) != cudaSuccess ||
        cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking) != cudaSuccess || (with_pipe && pipe_create(&b->pipe) != 0)) {
        fail("dec_batch_create", cudaGetLastError());
        solo_b200_dec_batch_destroy(b); return nullptr;
    }
    sb_dec_init_kernel<<<(n_streams + SB_TPB - 1) / SB_TPB, SB_TPB, 0, b->stream>>>(b->d_states, n_streams, ctrl->useMDIndex, ctrl->framesize_ms, ctrl->joint_enable ? 1 : 0);
    count_launch();
    cudaError_t e = cudaStreamSynchronize(b->stream);
    if (e != cudaSuccess) { fail("dec init kernel", e); solo_b200_dec_batch_destroy(b); return nullptr; }
    return b;
}

static int dec_launch(solo_b200_dec_batch* b, int lo, int n, i16* d_pcm, const u8* d_bits, int cap, const i16* d_nbytes, const i32* d_lostflag,
                      i32* d_ret, cudaStream_t st) {
    if (n <= 0) return 0;
    EvPair ev; prof_begin(st, 3, &ev);
    const size_t half = (size_t)(b->spp / 2);
    sb_decode_kernel<<<(n + SB_DEC_TPB - 1) / SB_DEC_TPB, SB_DEC_TPB, 0, st>>>(b->d_states + lo, d_bits + (size_t)lo * cap, cap, d_nbytes + 2 * (size_t)lo, d_lostflag + lo,
                                                                  d_ret ? d_ret + lo : nullptr, b->d_ret_int + lo, b->d_stale + lo,
                                                                  b->d_band_low + (size_t)lo * half, b->d_band_high + (size_t)lo * half, b->spp, n);
    sb_dec_synth_kernel<<<(n + SB_SYN_WARPS - 1) / SB_SYN_WARPS, SB_SYN_WARPS * 32, 0, st>>>(b->d_states + lo, b->d_band_low + (size_t)lo * half, b->d_band_high + (size_t)lo * half,
                                                                                          b->d_ret_int + lo, d_pcm + (size_t)lo * b->spp, b->spp, n);
    prof_end(st, &ev);
    count_launch(); count_launch();
    CK(cudaGetLastError());
    return 0;
}

int solo_b200_dec_batch_decode_device(solo_b200_dec_batch* b, int16_t* d_pcm, const uint8_t* d_bits, int cap, const int16_t* d_nbytes,
                                      const int32_t* d_lostflag, int32_t* d_ret, void* cuda_stream) {
    if (!b || !d_pcm || !d_bits || !d_nbytes || !d_lostflag || cap < 16) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    CK(cudaSetDevice(b->device));
    cudaStream_t user = (cudaStream_t)cuda_stream;
    const int C = pipe_chunks(b->n, false);
    if (C == 1) return dec_launch(b, 0, b->n, d_pcm, d_bits, cap, d_nbytes, d_lostflag, d_ret, user);
    CK(cudaEventRecord(b->pipe.fork, user));
    const int S = C < SB_PIPE_STREAMS ? C : SB_PIPE_STREAMS;
    for (int i = 0; i < S; i++) CK(cudaStreamWaitEvent(b->pipe.st[i], b->pipe.fork, 0));
    for (int c = 0; c < C; c++) {
        int lo, hi;
        chunk_bounds(b->n, C, c, &lo, &hi);
        int r = dec_launch(b, lo, hi - lo, d_pcm, d_bits, cap, d_nbytes, d_lostflag, d_ret, b->pipe.st[c % S]);
        if (r) return r;
    }
    for (int i = 0; i < S; i++) {
        CK(cudaEventRecord(b->pipe.join[i], b->pipe.st[i]));
        CK(cudaStreamWaitEvent(user, b->pipe.join[i], 0));
    }
    return 0;
}

static int dec_staging(solo_b200_dec_batch* b, int cap) {
    if (!b->d_pcm) CK(cudaMalloc(&b->d_pcm, sizeof(i16) * b->spp * (size_t)b->n));
    if (!b->d_nbytes) CK(cudaMalloc(&b->d_nbytes, sizeof(i16) * 2 * (size_t)b->n));
    if (!b->d_flags) CK(cudaMalloc(&b->d_flags, sizeof(i32) * (size_t)b->n));
    if (!b->d_ret) CK(cudaMalloc(&b->d_ret, sizeof(i32) * (size_t)b->n));
    if (!b->d_bits || b->bits_cap < cap) {
        if (b->d_bits) cudaFree(b->d_bits);
        b->d_bits = nullptr;
        CK(cudaMalloc(&b->d_bits, (size_t)cap * b->n));
        b->bits_cap = cap;
    }
    return 0;
}

int solo_b200_dec_batch_decode_host(solo_b200_dec_batch* b, int16_t* pcm, const uint8_t* bits, int cap, const int16_t* nbytes,
                                    const int32_t* lostflag, int32_t* ret) {
    if (!b || !pcm || !bits || !nbytes || !lostflag || cap < 16) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    CK(cudaSetDevice(b->device));
    int r = dec_staging(b, cap);
    if (r) return r;
    const int C = pipe_chunks(b->n, true);
    const int S = C < SB_PIPE_STREAMS ? C : SB_PIPE_STREAMS;
    for (int c = 0; c < C; c++) {
        int lo, hi;
        chunk_bounds(b->n, C, c, &lo, &hi);
        if (hi <= lo) continue;
        cudaStream_t st = b->pipe.st[c % S];
        const size_t m = (size_t)(hi - lo);
        CK(cudaMemcpyAsync(b->d_bits + (size_t)lo * cap, bits + (size_t)lo * cap, (size_t)cap * m, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(b->d_nbytes + 2 * (size_t)lo, nbytes + 2 * (size_t)lo, sizeof(i16) * 2 * m, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(b->d_flags + lo, lostflag + lo, sizeof(i32) * m, cudaMemcpyHostToDevice, st));
        r = dec_launch(b, lo, hi - lo, b->d_pcm, b->d_bits, cap, b->d_nbytes, b->d_flags, b->d_ret, st);
        if (r) return r;
        CK(cudaMemcpyAsync(pcm + (size_t)lo * b->spp, b->d_pcm + (size_t)lo * b->spp, sizeof(i16) * b->spp * m, cudaMemcpyDeviceToHost, st));
        if (ret) CK(cudaMemcpyAsync(ret + lo, b->d_ret + lo, sizeof(i32) * m, cudaMemcpyDeviceToHost, st));
    }
    for (int i = 0; i < S; i++) CK(cudaStreamSynchronize(b->pipe.st[i]));
    return 0;
}

void solo_b200_dec_batch_destroy(solo_b200_dec_batch* b) {
    if (!b) return;
    cudaSetDevice(b->device);
    if (b->stream) cudaStreamSynchronize(b->stream);
    pipe_destroy(&b->pipe);
    cudaFree(b->d_states); cudaFree(b->d_stale); cudaFree(b->d_pcm); cudaFree(b->d_bits); cudaFree(b->d_nbytes); cudaFree(b->d_flags); cudaFree(b->d_ret);
    cudaFree(b->d_band_low); cudaFree(b->d_band_high); cudaFree(b->d_ret_int);
    if (b->stream) cudaStreamDestroy(b->stream);
    delete b;
}

// ---- stream state hand-over (checkpoint / migration, SURVEY.md 8(f) rank 3) ----------------------------------------------
static int state_copy(void* dev_base, size_t stride, int n, int idx, void* host, int to_host, int device, cudaStream_t st) {
    if (!dev_base || !host || idx < 0 || idx >= n) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    CK(cudaSetDevice(device));
    (void)st;
    CK(cudaDeviceSynchronize());    // packet waves run on the internal pipeline streams and on caller streams: wait for all of them
    char* p = (char*)dev_base + stride * (size_t)idx;
    if (to_host) CK(cudaMemcpy(host, p, stride, cudaMemcpyDeviceToHost));
    else CK(cudaMemcpy(p, host, stride, cudaMemcpyHostToDevice));
    return 0;
}
int solo_b200_enc_batch_export_state(solo_b200_enc_batch* b, int idx, void* blob) {
    if (!b) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    return state_copy(b->d_states, sizeof(EncState), b->n, idx, blob, 1, b->device, b->stream);
}
int solo_b200_enc_batch_import_state(solo_b200_enc_batch* b, int idx, const void* blob) {
    if (!b) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    return state_copy(b->d_states, sizeof(EncState), b->n, idx, (void*)blob, 0, b->device, b->stream);
}
int solo_b200_dec_batch_export_state(solo_b200_dec_batch* b, int idx, void* blob) {
    if (!b) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    return state_copy(b->d_states, sizeof(DecState), b->n, idx, blob, 1, b->device, b->stream);
}
int solo_b200_dec_batch_import_state(solo_b200_dec_batch* b, int idx, const void* blob) {
    if (!b) { snprintf(g_err, sizeof g_err, "bad argument"); return -1; }
    return state_copy(b->d_states, sizeof(DecState), b->n, idx, (void*)blob, 0, b->device, b->stream);
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
    const int have1 = p1 && n1 > 0, have2 = p2 && n2 > 0;
    if (have1 && have2) {
        if (n1 + n2 > cap) return -1;
        memmove(bits, p1, (size_t)n1); memmove(bits + n1, p2, (size_t)n2);
        nbytes[0] = (int16_t)(n1 + n2); nbytes[1] = (int16_t)n2; *lostflag = 4;
    } else if (have1) {
        if (n1 > cap) return -1;
        memmove(bits, p1, (size_t)n1); nbytes[0] = (int16_t)n1; nbytes[1] = 0; *lostflag = 2;
    } else if (have2) {
        if (n2 > cap) return -1;
        memmove(bits, p2, (size_t)n2); nbytes[0] = (int16_t)n2; nbytes[1] = 0; *lostflag = 3;
    } else {
        // nothing arrived: the decoder conceals; it still wants nBytes[0] > 0 (AGR_BWE_SDK_API.c:268-270), the bytes are not read
        nbytes[0] = 16; nbytes[1] = 8; *lostflag = 1;
        if (cap >= 16) memset(bits, 0, 16);
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
    count_launch();
    CK(cudaGetLastError());
    return 0;
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
// A handle is a SLOT of a process-wide, lazily grown arena: segments of SB_ARENA_SEG streams (ordinary batch objects without
// the chunk pipeline: one CUDA stream and one set of staging buffers per segment, shared by its slots).  Init takes a free
// slot of a segment with the same packet layout and (re)initialises that one stream on the device; Uninit gives it back.
// 10 000 handles are 40 segments = 40 CUDA streams and 240 device allocations, not 10 000 batches.  Calls on handles of the
// same segment are serialised by the segment's mutex; different segments run concurrently.
// Same names / return conventions as AGR_BWE_SDK_API.c:11-296 and libBWE/AGR_BWE_init.c:6-76.
#ifndef SB_ARENA_SEG
#define SB_ARENA_SEG 256
#endif
extern "C++" {
struct ArenaKey { int device, framesize_ms, joint; };
template <class Batch> struct ArenaSeg {
    ArenaKey key;
    Batch* b;
    std::vector<char> used;
    int n_used;
    std::mutex mu;
};
struct EncHandle { unsigned magic; ArenaSeg<solo_b200_enc_batch>* seg; int slot; };
struct DecHandle { unsigned magic; ArenaSeg<solo_b200_dec_batch>* seg; int slot; };
static const unsigned ENC_MAGIC = 0x53424531u, DEC_MAGIC = 0x53424431u;   // "SBE1", "SBD1"
static std::mutex g_arena_mu;
static std::vector<ArenaSeg<solo_b200_enc_batch>*> g_enc_segs;
static std::vector<ArenaSeg<solo_b200_dec_batch>*> g_dec_segs;

template <class Batch> static ArenaSeg<Batch>* arena_take(std::vector<ArenaSeg<Batch>*>& segs, ArenaKey k, int* slot) {
    for (auto* sg : segs)
        if (sg->key.device == k.device && sg->key.framesize_ms == k.framesize_ms && sg->key.joint == k.joint && sg->n_used < SB_ARENA_SEG)
            for (int i = 0; i < SB_ARENA_SEG; i++)
                if (!sg->used[i]) { sg->used[i] = 1; sg->n_used++; *slot = i; return sg; }
    return nullptr;
}
}  // extern "C++"

void* AGR_Sate_Encoder_Init(USER_Ctrl_enc* enc_Ctrl) {
    if (!enc_Ctrl) return nullptr;
    if (enc_Ctrl->targetRate_bps <= 0) enc_Ctrl->targetRate_bps = 15600;  // written back (AGR_BWE_SDK_API.c:34-36)
    if (enc_Ctrl->joint_enable && (enc_Ctrl->joint_mode < 0 || enc_Ctrl->joint_mode > 3)) {
        printf("Error in setting joint mode! It must be 0, 1, 2, 3\n");
        return nullptr;
    }
    if (check_enc_ctrl(enc_Ctrl)) { fprintf(stderr, "solo_b200: AGR_Sate_Encoder_Init: unsupported configuration\n"); return nullptr; }
    int dev = 0;
    cudaGetDevice(&dev);
    const ArenaKey k = {dev, enc_Ctrl->framesize_ms, enc_Ctrl->joint_enable ? 1 : 0};
    std::lock_guard<std::mutex> lk(g_arena_mu);
    int slot = -1;
    auto* sg = arena_take(g_enc_segs, k, &slot);
    if (!sg) {
        solo_b200_enc_batch* b = enc_batch_create_impl(SB_ARENA_SEG, enc_Ctrl, dev, false);
        if (!b) { fprintf(stderr, "solo_b200: AGR_Sate_Encoder_Init failed: %s\n", g_err); return nullptr; }
        sg = new ArenaSeg<solo_b200_enc_batch>();
        sg->key = k; sg->b = b; sg->used.assign(SB_ARENA_SEG, 0); sg->n_used = 0;
        g_enc_segs.push_back(sg);
        sg->used[0] = 1; sg->n_used = 1; slot = 0;
    }
    {   // (re)initialise this one stream with the caller's rate / DTX / MD-index settings
        std::lock_guard<std::mutex> lk2(sg->mu);
        cudaSetDevice(dev);
        sb_enc_init_kernel<<<1, SB_TPB, 0, sg->b->stream>>>(sg->b->d_states + slot, 1, enc_Ctrl->targetRate_bps, enc_Ctrl->dtx_enable, enc_Ctrl->useMDIndex,
                                                          enc_Ctrl->framesize_ms, enc_Ctrl->joint_enable ? 1 : 0);
        count_launch();
        if (cudaStreamSynchronize(sg->b->stream) != cudaSuccess) { sg->used[slot] = 0; sg->n_used--; fprintf(stderr, "solo_b200: encoder slot init failed\n"); return nullptr; }
    }
    EncHandle* h = new EncHandle{ENC_MAGIC, sg, slot};
    return h;
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
        if (cudaSetDevice(b->device) != cudaSuccess || enc_staging(b, cap)) { fprintf(stderr, "solo_b200: encode failed: %s\n", g_err); return -1; }
        const size_t s = (size_t)h->slot;
        cudaStream_t st = b->stream;
        bool ok = cudaMemcpyAsync(b->d_pcm + s * b->spp, AGR_Sate_PCM, sizeof(i16) * b->spp, cudaMemcpyHostToDevice, st) == cudaSuccess;
        ok = ok && enc_launch(b, h->slot, 1, b->d_pcm, b->d_bits, cap, b->d_nbytes, st) == 0;
        ok = ok && cudaMemcpyAsync(tmp, b->d_bits + s * cap, cap, cudaMemcpyDeviceToHost, st) == cudaSuccess;
        ok = ok && cudaMemcpyAsync(nb, b->d_nbytes + 2 * s, sizeof nb, cudaMemcpyDeviceToHost, st) == cudaSuccess;
        ok = ok && cudaStreamSynchronize(st) == cudaSuccess;
        if (!ok) { fprintf(stderr, "solo_b200: encode failed: %s\n", g_err[0] ? g_err : cudaGetErrorString(cudaGetLastError())); return -1; }
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
int AGR_Sate_Encoder_Uninit(void* SATEEnc_State) {
    EncHandle* h = (EncHandle*)SATEEnc_State;
    if (!h || h->magic != ENC_MAGIC) return -1;
    {
        std::lock_guard<std::mutex> lk(g_arena_mu);
        h->seg->used[h->slot] = 0;
        h->seg->n_used--;
    }
    h->magic = 0;
    delete h;
    return 0;
}

void* AGR_Sate_Decoder_Init(USER_Ctrl_dec* dec_Ctrl) {
    if (!dec_Ctrl) return nullptr;
    if (dec_Ctrl->joint_enable && (dec_Ctrl->joint_mode < 0 || dec_Ctrl->joint_mode > 3)) {
        fprintf(stderr, "Error in setting joint mode! It must be 0, 1, 2, 3\n");
        return nullptr;
    }
    if (check_dec_ctrl(dec_Ctrl)) { fprintf(stderr, "solo_b200: AGR_Sate_Decoder_Init: unsupported configuration\n"); return nullptr; }
    int dev = 0;
    cudaGetDevice(&dev);
    const ArenaKey k = {dev, dec_Ctrl->framesize_ms, dec_Ctrl->joint_enable ? 1 : 0};
    std::lock_guard<std::mutex> lk(g_arena_mu);
    int slot = -1;
    auto* sg = arena_take(g_dec_segs, k, &slot);
    if (!sg) {
        solo_b200_dec_batch* b = dec_batch_create_impl(SB_ARENA_SEG, dec_Ctrl, dev, false);
        if (!b) { fprintf(stderr, "solo_b200: AGR_Sate_Decoder_Init failed: %s\n", g_err); return nullptr; }
        sg = new ArenaSeg<solo_b200_dec_batch>();
        sg->key = k; sg->b = b; sg->used.assign(SB_ARENA_SEG, 0); sg->n_used = 0;
        g_dec_segs.push_back(sg);
        sg->used[0] = 1; sg->n_used = 1; slot = 0;
    }
    {
        std::lock_guard<std::mutex> lk2(sg->mu);
        cudaSetDevice(dev);
        sb_dec_init_kernel<<<1, SB_TPB, 0, sg->b->stream>>>(sg->b->d_states + slot, 1, dec_Ctrl->useMDIndex, dec_Ctrl->framesize_ms, dec_Ctrl->joint_enable ? 1 : 0);
        count_launch();
        if (cudaStreamSynchronize(sg->b->stream) != cudaSuccess) { sg->used[slot] = 0; sg->n_used--; fprintf(stderr, "solo_b200: decoder slot init failed\n"); return nullptr; }
    }
    DecHandle* h = new DecHandle{DEC_MAGIC, sg, slot};
    return h;
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
        if (cudaSetDevice(b->device) != cudaSuccess || dec_staging(b, cap)) { fprintf(stderr, "solo_b200: decode failed: %s\n", g_err); return -1; }
        const size_t s = (size_t)h->slot;
        cudaStream_t st = b->stream;
        bool ok = cudaMemcpyAsync(b->d_bits + s * cap, tmp, cap, cudaMemcpyHostToDevice, st) == cudaSuccess;
        ok = ok && cudaMemcpyAsync(b->d_nbytes + 2 * s, nb, sizeof nb, cudaMemcpyHostToDevice, st) == cudaSuccess;
        ok = ok && cudaMemcpyAsync(b->d_flags + s, &flag, sizeof flag, cudaMemcpyHostToDevice, st) == cudaSuccess;
        ok = ok && dec_launch(b, h->slot, 1, b->d_pcm, b->d_bits, cap, b->d_nbytes, b->d_flags, b->d_ret, st) == 0;
        ok = ok && cudaMemcpyAsync(AGR_Sate_PCM, b->d_pcm + s * b->spp, sizeof(i16) * b->spp, cudaMemcpyDeviceToHost, st) == cudaSuccess;
        ok = ok && cudaMemcpyAsync(&ret, b->d_ret + s, sizeof ret, cudaMemcpyDeviceToHost, st) == cudaSuccess;
        ok = ok && cudaStreamSynchronize(st) == cudaSuccess;
        if (!ok) { fprintf(stderr, "solo_b200: decode failed: %s\n", g_err[0] ? g_err : cudaGetErrorString(cudaGetLastError())); return -1; }
    }
    // the reference rewrites the caller's nBytes[] while splitting the payload (AGR_BWE_decode_frame_FLP.c:171-190)
    dec_split_lengths(nb, lostflag, b->hb_bytes);
    nBytes[0] = nb[0];
    nBytes[1] = nb[1];
    *nSamplesOut = (SKP_int16)b->spp;
    return ret;
}
SKP_int32 AGR_Sate_Decoder_Uninit(void* SATEDec_State) {
    DecHandle* h = (DecHandle*)SATEDec_State;
    if (!h || h->magic != DEC_MAGIC) return -1;
    {
        std::lock_guard<std::mutex> lk(g_arena_mu);
        h->seg->used[h->slot] = 0;
        h->seg->n_used--;
    }
    h->magic = 0;
    delete h;
    return 0;
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
