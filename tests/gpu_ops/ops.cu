// Test-only harness: single routines of the analysis kernel's warp-cooperative form (sb_coop.cuh) and of the level-0 kit
// (sb_common.cuh), compiled for sm_90a exactly as sb_analysis.cu compiles them, one warp per case.  Each kernel reads its
// case from global memory, stages the routine's scratch struct and arrays in shared memory as the analysis kernel does,
// calls the routine and writes every output back.  tests/test_gpu_ops.py compares the results with the reference.
// The quantiser kernel's device code runs here too, whole packets in the production kernel's layout (sb_ops_nsq,
// tests/test_gpu_nsq.py), and so does the device code of the band-split, high-band analysis and synthesis filter-bank
// kernels (sb_ops_qmf_split, sb_ops_hb, sb_ops_hb_vq, sb_ops_synth; tests/test_gpu_bands.py), and that of the voice-activity
// kernel and the high-band store of the entropy-coding kernel (sb_ops_vad, sb_ops_hb_store; tests/test_gpu_enc_stages.py).
// Every launcher takes host arrays, copies them to the device and back, and returns a CUDA error code (0 = success).
#define SB_COOP 1
#define SB_DIV_OUTLINE 1
#define SB_BLOCK_STREAMS 8
#include <cuda_runtime.h>
#include <string.h>
#include <vector>
#include "sb_coop.cuh"
#include "sb_dec.cuh"
#include "sb_nsq_warp.cuh"
#include "../../oracle/nsq_io.h"
#include "../../oracle/vad_io.h"

using namespace sb;

namespace {

// ---- level-0 primitives, one thread per element -------------------------------------------------------------------------
enum PrimOp {
    OP_SMULWB, OP_SMULWT, OP_SMMUL, OP_ADD_SAT32, OP_SUB_SAT32, OP_CLZ32, OP_CLZ64, OP_DIV_Q29, OP_DIV32_VARQ,
    OP_INVERSE32_VARQ, OP_SQRT_APPROX, OP_LIN2LOG, OP_LOG2LIN, OP_SIGM_Q15, OP_LSHIFT_SAT32, OP_POPC32, OP_CTZ32,
    OP_FLOAT2INT, OP_TRUNC_I32, OP_SMULWW,
};

__global__ void prim_kernel(int op, const long long* a, const long long* b, const long long* c, const double* f, long long* out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const i32 x = (i32)a[i], y = (i32)b[i];
    long long r = 0;
    switch (op) {
        case OP_SMULWB: r = smulwb(x, y); break;
        case OP_SMULWT: r = smulwt(x, y); break;
        case OP_SMMUL: r = smmul(x, y); break;
        case OP_ADD_SAT32: r = add_sat32(x, y); break;
        case OP_SUB_SAT32: r = sub_sat32(x, y); break;
        case OP_CLZ32: r = clz32(x); break;
        case OP_CLZ64: r = clz64((i64)a[i]); break;
        case OP_DIV_Q29: r = div_q29(x); break;
        case OP_DIV32_VARQ: r = div32_varq(x, y, (int)c[i]); break;
        case OP_INVERSE32_VARQ: r = inverse32_varq(x, (int)c[i]); break;
        case OP_SQRT_APPROX: r = sqrt_approx(x); break;
        case OP_LIN2LOG: r = lin2log(x); break;
        case OP_LOG2LIN: r = log2lin(x); break;
        case OP_SIGM_Q15: r = sigm_q15(x); break;
        case OP_LSHIFT_SAT32: r = lshift_sat32(x, y); break;
        case OP_POPC32: r = popc32((u32)x); break;
        case OP_CTZ32: r = ctz32((u32)x); break;
        case OP_FLOAT2INT: r = float2int(f[i]); break;
        case OP_TRUNC_I32: r = trunc_i32(f[i]); break;
        case OP_SMULWW: r = smulww(x, y); break;
        default: r = 0x7fffffffffffffffLL;
    }
    out[i] = r;
}

// ---- c_schur (order <= 16) and c_k2a: c [17] and rc_in [16] per case -> rc_Q15 [16], residual energy, A_Q24 [16] -----
__global__ void schur_kernel(const i32* c, const i16* rc_in, int order, i16* rc_out, i32* nrg_out, i32* A_out) {
    __shared__ i32 cs[32];
    __shared__ i16 rc[32], rk[32];
    const int lane = threadIdx.x, cse = blockIdx.x;
    cs[lane] = lane <= 16 ? c[cse * 17 + lane] : 0;
    rc[lane] = 0;
    rk[lane] = lane < 16 ? rc_in[cse * 16 + lane] : 0;
    __syncwarp();
    const i32 nrg = c_schur(rc, cs, order);
    __syncwarp();
    const i32 A = c_k2a(rk, order);
    if (lane < 16) { rc_out[cse * 16 + lane] = rc[lane]; A_out[cse * 16 + lane] = lane < order ? A : 0; }
    if (lane == 0) nrg_out[cse] = nrg;
}

// ---- schur64_r / k2a_q16_r at the shaping order, one thread per case: c [17] -> rc_Q16 [16], energy; rc_in -> A_Q24 ------
__global__ void schur64_kernel(const i32* c, const i32* rc_in, i32* rc_out, i32* nrg_out, i32* A_out, int n) {
    const int cse = blockIdx.x * blockDim.x + threadIdx.x;
    if (cse >= n) return;
    i32 cc[SHAPE_ORDER + 1], rc[SHAPE_ORDER], rk[SHAPE_ORDER], A[SHAPE_ORDER];
#pragma unroll
    for (int i = 0; i <= SHAPE_ORDER; i++) cc[i] = c[cse * 17 + i];
#pragma unroll
    for (int i = 0; i < SHAPE_ORDER; i++) rk[i] = rc_in[cse * 16 + i];
    nrg_out[cse] = schur64_r<SHAPE_ORDER>(rc, cc);
    k2a_q16_r<SHAPE_ORDER>(A, rk);
#pragma unroll
    for (int i = 0; i < SHAPE_ORDER; i++) { rc_out[cse * 16 + i] = rc[i]; A_out[cse * 16 + i] = A[i]; }
}

// ---- c_burg2<D>: two analyses per case, x [2][XMAX] (one signal per half of the warp) -----------------------------------
enum { XMAX = NB_SUBFR * (80 + HB_ORDER) };
struct BurgCase { i32 nb[2], L, wnf; };
template <int D> __global__ void burg_kernel(const BurgCase* cases, const i16* x, i32* nrg_out, i32* q_out, i32* A_out) {
    __shared__ __align__(16) i16 xs[2][XMAX];
    __shared__ i32 A[2][16];
    __shared__ BurgScr B;
    const int lane = threadIdx.x, cse = blockIdx.x;
    const BurgCase k = cases[cse];
    for (int i = lane; i < 2 * XMAX; i += 32) xs[i / XMAX][i % XMAX] = x[(size_t)cse * 2 * XMAX + i];
    A[lane >> 4][lane & 15] = 0;
    __syncwarp();
    i32 rn, rq;
    c_burg2<D>(&rn, &rq, A, &B, xs[0], k.nb[0], xs[1], k.nb[1], k.L, k.wnf);
    __syncwarp();
    if ((lane & 15) == 0) { nrg_out[cse * 2 + (lane >> 4)] = rn; q_out[cse * 2 + (lane >> 4)] = rq; }
    A_out[cse * 32 + lane] = A[lane >> 4][lane & 15];
}

// ---- c_a2nlsf<D>: a_Q16 [16] in / out (widened in place), NLSF [16] ----------------------------------------------------
template <int D> __global__ void a2nlsf_kernel(i32* a, i32* nlsf_out) {
    __shared__ i32 as[16], nl[16];
    __shared__ A2nlsfScr Z;
    const int lane = threadIdx.x, cse = blockIdx.x;
    if (lane < 16) { as[lane] = a[cse * 16 + lane]; nl[lane] = -1; }
    __syncwarp();
    c_a2nlsf<D>(nl, as, &Z);
    __syncwarp();
    if (lane < 16) { a[cse * 16 + lane] = as[lane]; nlsf_out[cse * 16 + lane] = nl[lane]; }
}

// ---- c_warped_autocorr4: four windows [4][SHAPE_WIN] per case -> corr [4][17], scale [4] --------------------------------
__global__ void warped_kernel(const i16* x, const i32* warping, i32* corr_out, i32* scale_out) {
    __shared__ ShapeScr S;
    const int lane = threadIdx.x, cse = blockIdx.x;
    for (int i = lane; i < NB_SUBFR * SHAPE_WIN; i += 32) S.xw[i / SHAPE_WIN][i % SHAPE_WIN] = x[(size_t)cse * NB_SUBFR * SHAPE_WIN + i];
    for (int i = lane; i < NB_SUBFR * (SHAPE_ORDER + 1); i += 32) S.acorr[i / (SHAPE_ORDER + 1)][i % (SHAPE_ORDER + 1)] = 0x5a5a5a5a;
    __syncwarp();
    c_warped_autocorr4(&S, warping[cse]);
    __syncwarp();
    for (int i = lane; i < NB_SUBFR * (SHAPE_ORDER + 1); i += 32) corr_out[cse * NB_SUBFR * (SHAPE_ORDER + 1) + i] = S.acorr[i / (SHAPE_ORDER + 1)][i % (SHAPE_ORDER + 1)];
    if (lane < NB_SUBFR) scale_out[cse * NB_SUBFR + lane] = S.scale[lane];
}

// ---- c_quant_ltp_gains: B_Q14 [20] in / out, W_Q18 [100] -> cbk_index [4], periodicity index ---------------------------
__global__ void ltp_kernel(i16* B, const i32* W, const i32* mu, i32* cbk_out, i32* per_out) {
    __shared__ i16 Bs[NB_SUBFR * LTP_ORDER];
    __shared__ i32 Ws[NB_SUBFR * LTP_ORDER * LTP_ORDER];
    __shared__ i32 cbk[NB_SUBFR], per;
    const int lane = threadIdx.x, cse = blockIdx.x;
    if (lane < NB_SUBFR * LTP_ORDER) Bs[lane] = B[cse * NB_SUBFR * LTP_ORDER + lane];
    for (int i = lane; i < NB_SUBFR * LTP_ORDER * LTP_ORDER; i += 32) Ws[i] = W[cse * NB_SUBFR * LTP_ORDER * LTP_ORDER + i];
    if (lane < NB_SUBFR) cbk[lane] = -1;
    if (lane == 0) per = -1;
    __syncwarp();
    c_quant_ltp_gains(Bs, cbk, &per, Ws, mu[cse]);
    __syncwarp();
    if (lane < NB_SUBFR * LTP_ORDER) B[cse * NB_SUBFR * LTP_ORDER + lane] = Bs[lane];
    if (lane < NB_SUBFR) cbk_out[cse * NB_SUBFR + lane] = cbk[lane];
    if (lane == 0) per_out[cse] = per;
}

// ---- routines with scalar instances (c_instances): the analysis kernel's block layout ----------------------------------
// SB_BLOCK_STREAMS warps per block, one case each, every warp with an AnaSmem slot (sb_slot_bytes() apart) in dynamic shared
// memory behind the NLSF codebook copy, as sb_enc_analysis_warp_kernel lays them out.  The instances of a block run on
// consecutive threads and reach the other warps' slots, so every warp takes part: a warp beyond the last case repeats it
// and writes nothing back.
#define SB_OPS_TABS_BYTES ((sizeof(NlsfFastTabs) + 15) & ~15)
constexpr int kSlotSmem = (int)SB_OPS_TABS_BYTES + SB_BLOCK_STREAMS * (int)sizeof(AnaSmem);
__device__ __forceinline__ AnaSmem* ops_slot(unsigned char* smem_raw, int w) {
    return reinterpret_cast<AnaSmem*>(smem_raw + SB_OPS_TABS_BYTES) + w;
}

// c_pitch_analysis_core on a 320-sample 8 kHz signal.  case: prevLag, search_thres1_Q16, search_thres2_Q15, LTPCorr_Q15 in.
// out [8]: pitch lags [4], lagIndex, contourIndex, LTPCorr_Q15, returned signal type
struct PitchCase { i32 prevLag, thres1_Q16, thres2_Q15, ltpcorr_Q15; };
enum { PITCH_LEN = 320 };
__global__ void __launch_bounds__(SB_BLOCK_STREAMS * 32) pitch_kernel(const PitchCase* cases, const i16* sig, int n, i32* out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ i32 res[SB_BLOCK_STREAMS][8];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int s = blockIdx.x * SB_BLOCK_STREAMS + w;
    const bool live = s < n;
    if (!live) s = n - 1;
    AnaSmem* S = ops_slot(smem_raw, w);
    PitchScr* P = &S->W.u.pitch;
    i16* signal = S->W.res_pitch;
    static_assert(sizeof(S->W.res_pitch) >= PITCH_LEN * sizeof(i16), "pitch signal fits the residual buffer");
    for (int i = lane; i < PITCH_LEN; i += 32) signal[i] = sig[(size_t)s * PITCH_LEN + i];
    const PitchCase k = cases[s];
    if (lane < 8) res[w][lane] = -1;
    __syncwarp();
    if (lane == 0) res[w][6] = k.ltpcorr_Q15;
    __syncwarp();
    const int sigtype = c_pitch_analysis_core(P, signal, &res[w][0], &res[w][4], &res[w][5], &res[w][6], k.prevLag, k.thres1_Q16, k.thres2_Q15);
    __syncwarp();
    if (lane == 0) res[w][7] = sigtype;
    __syncwarp();
    if (live && lane < 8) out[(size_t)s * 8 + lane] = res[w][lane];
}

// c_nlsf_msvq_encode, order 10.  case: NLSF_mu_Q15, NLSF_mu_fluc_red_Q16, deactivate_fluc_red, sigtype; nlsf / prev / w [10].
// out: indices [6], quantised NLSF [10].  The target, the previous quantised vector, the weights and the results live where
// c_process_nlsfs keeps them: PredScr, EncSilk and EncCtrl of the slot.
struct MsvqCase { i32 mu_Q15, fluc_red_Q16, deactivate, sigtype; };
__global__ void __launch_bounds__(SB_BLOCK_STREAMS * 32) msvq_kernel(const MsvqCase* cases, const i32* nlsf, const i32* prev, const i32* wts, int n,
                                                                     i32* idx_out, i32* nlsf_out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    NlsfFastTabs* tabs = reinterpret_cast<NlsfFastTabs*>(smem_raw);
    nlsf_fast_tabs_fill(tabs, threadIdx.x, blockDim.x);
    __syncthreads();
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int s = blockIdx.x * SB_BLOCK_STREAMS + w;
    const bool live = s < n;
    if (!live) s = n - 1;
    AnaSmem* S = ops_slot(smem_raw, w);
    PredScr* Q = &S->W.u.pred;
    const MsvqCase k = cases[s];
    if (lane < LPC_ORDER) {
        Q->NLSF_Q15[lane] = nlsf[s * LPC_ORDER + lane];
        S->st.prev_NLSFq_Q15[lane] = prev[s * LPC_ORDER + lane];
        Q->NLSFW_Q6[lane] = wts[s * LPC_ORDER + lane];
    }
    if (lane < 6) S->W.c.NLSFIndices[lane] = -1;
    __syncwarp();
    NlsfCb cb = nlsf_cb(k.sigtype);
    cb.cb_q15 = k.sigtype == 0 ? tabs->cb0 : tabs->cb1;
    cb.rates_q5 = k.sigtype == 0 ? tabs->rates0 : tabs->rates1;
    c_nlsf_msvq_encode(S->W.c.NLSFIndices, Q->NLSF_Q15, cb, S->st.prev_NLSFq_Q15, Q->NLSFW_Q6, k.mu_Q15, k.fluc_red_Q16, k.deactivate,
                       k.sigtype, Q);
    __syncthreads();
    if (live && lane < 6) idx_out[s * 6 + lane] = S->W.c.NLSFIndices[lane];
    if (live && lane < LPC_ORDER) nlsf_out[s * LPC_ORDER + lane] = Q->NLSF_Q15[lane];
}

// ---- the quantiser kernel's device code (nsq_packet_warp) in sb_enc_nsq_kernel's layout: one-warp blocks, a stream per
//      16-lane group, a group without a case of its own shadowing the last one, the same dynamic shared memory and bounds ----
constexpr int kNsqSpb = 32 / SB_NSQ_GW;
__global__ void __launch_bounds__(32, 12) nsq_kernel(NsqState* ns, EncScratch* scratch, int nf, int n) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int g = threadIdx.x / SB_NSQ_GW;
    NsqSmem* S = reinterpret_cast<NsqSmem*>(smem_raw) + g;
    int s = blockIdx.x * kNsqSpb + g;
    if (s >= n) s = n - 1;
    nsq_packet_warp(*S, &ns[3 * s], &scratch[s], nf);
}

// ---- the band-split kernel's device code (qmf_output_pair) in sb_enc_qmf_kernel's staging: one-warp blocks, history
//      reversed from the filter memory, the packet's samples >> 1, the memory written back from the staged row -------------
__global__ void __launch_bounds__(32) qmf_split_kernel(const i32* spp_of, i16* mems, const i16* pcm, i16* bands) {
    __shared__ __align__(16) i16 xs[PACKET + 64];
    __shared__ i16 coef[64];
    const int lane = threadIdx.x, s = blockIdx.x;
    const int spp = spp_of[s];
    for (int i = lane; i < 64; i += 32) coef[i] = SB_T(qmf_fix)[i];
    i16* mem = mems + (size_t)s * 64;
    for (int i = lane; i < 63; i += 32) xs[i] = mem[62 - i];                     // x[i] = mem[M - i - 2]
    for (int i = lane; i < spp; i += 32) xs[63 + i] = (i16)(pcm[(size_t)s * PACKET + i] >> 1);
    __syncwarp();
    i16* out = bands + (size_t)s * PACKET;
    const int half = spp >> 1;
    for (int k = lane; k < half; k += 32) {
        i16 lo, hi;
        qmf_output_pair(xs, coef, k, &lo, &hi);
        out[k] = lo; out[half + k] = hi;
    }
    for (int i = lane; i < 63; i += 32) mem[i] = xs[spp + 62 - i];               // mem[i] = x[N + M - 2 - i]
}

// ---- the high-band analysis kernel's device code (c_hb_analyse_packet, c_hb_lsp_quant) in sb_enc_hb_warp_kernel's layout:
//      kHbWarps warps per block (SB_HB_WARPS of sb_analysis.cu), one HbSmem slot each, a warp beyond the last case returns ----
constexpr int kHbWarps = 4;
struct HbSmem {
    EncBands hb;
    HbScr H;
    alignas(16) i16 high[PACKET / 2];
};
constexpr int kHbSmem = kHbWarps * (int)sizeof(HbSmem);
struct HbCase { i32 F, n; };      // frame length (160 or 320), high-band samples per packet (160 or 320)
struct HbFrameOut {
    i32 lsp_idx, nrg0[4];
    i32 nlsf_pre[HB_ORDER], nlsf_q[HB_ORDER], weight[HB_ORDER];
    i16 coef[HB_ORDER];
    i16 x_hb_buf[2 * 320 + 40];
    i32 hb_first;
};
__device__ __forceinline__ void ops_copy16(void* dst, const void* src, int bytes, int lane) {
    const int4* s = reinterpret_cast<const int4*>(src);
    int4* d = reinterpret_cast<int4*>(dst);
    for (int i = lane; i < bytes / 16; i += 32) d[i] = s[i];
}
// One packet of every case: high [n][PACKET / 2] (the case's first k.n samples); the state moves between global and shared
// memory as in the product kernel.
// per_frame = 0: one c_hb_analyse_packet call over the whole packet, as the product kernel makes it (its loop over the
//   packet's frames, scr->hb_lsp_idx[f] / hb_nrg0[f]); out[f] gets those and the state after the packet.
// per_frame = 1: one c_hb_analyse_packet call per frame, so that each frame's working set is read before the next frame
//   overwrites it; the packet loop itself is not run in this mode.  The NLSF vector the LSP search started from is
//   recovered by running c_a2nlsf once more on the polynomial the frame's c_a2nlsf left behind (widened in place): its root
//   search succeeds on that polynomial at the first attempt.  (A frame that ended in A2NLSF's white-spectrum fallback would
//   not be recovered this way; Burg's filters do not reach that fallback, see tests/test_gpu_bands.py.)
__global__ void __launch_bounds__(kHbWarps * 32) hb_kernel(const HbCase* cases, EncBands* states, EncScratch* scratch, const i16* high, int n,
                                                           int per_frame, HbFrameOut* out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int s = blockIdx.x * kHbWarps + w;
    if (s >= n) return;
    HbSmem* S = reinterpret_cast<HbSmem*>(smem_raw) + w;
    const HbCase k = cases[s];
    const int nf = k.n / k.F;
    EncScratch* scr = &scratch[s];
    ops_copy16(&S->hb, &states[s], (int)sizeof(EncBands), lane);
    ops_copy16(S->high, high + (size_t)s * (PACKET / 2), k.n * 2, lane);
    if (lane < 2) scr->hb_lsp_idx[lane] = 0x5a5a5a5a;
    if (lane < 8) scr->hb_nrg0[lane >> 2][lane & 3] = 0x5a5a5a5a;
    __syncwarp();
    if (!per_frame) {
        c_hb_analyse_packet(&S->hb, &S->H, S->high, k.n, k.F, scr);
        __syncwarp();
        for (int f = 0; f < nf; f++) {
            HbFrameOut* o = &out[(size_t)s * 2 + f];
            if (lane == 0) { o->lsp_idx = scr->hb_lsp_idx[f]; o->hb_first = S->hb.hb_first; }
            if (lane < 4) o->nrg0[lane] = scr->hb_nrg0[f][lane];
            for (int i = lane; i < 2 * 320 + 40; i += 32) o->x_hb_buf[i] = S->hb.x_hb_buf[i];
        }
    }
    for (int f = 0; per_frame && f < nf; f++) {
        c_hb_analyse_packet(&S->hb, &S->H, S->high + f * k.F, k.F, k.F, scr);
        __syncwarp();
        HbFrameOut* o = &out[(size_t)s * 2 + f];
        if (lane == 0) { o->lsp_idx = scr->hb_lsp_idx[0]; o->hb_first = S->hb.hb_first; }
        if (lane < 4) o->nrg0[lane] = scr->hb_nrg0[0][lane];
        if (lane < HB_ORDER) {
            o->nlsf_q[lane] = S->H.NLSF_Q15[lane];
            o->weight[lane] = S->H.weight[lane];
            o->coef[lane] = S->H.coef[lane];
            S->H.A_Q16[1][lane] = S->H.A_Q16[0][lane];
        }
        for (int i = lane; i < 2 * 320 + 40; i += 32) o->x_hb_buf[i] = S->hb.x_hb_buf[i];
        if (lane == 0) scr->hb_lsp_idx[0] = 0x5a5a5a5a;
        if (lane < 4) scr->hb_nrg0[0][lane] = 0x5a5a5a5a;
        __syncwarp();
        c_a2nlsf<HB_ORDER>(S->H.NLSF_Q15, S->H.A_Q16[1], &S->H.u.a2n);
        __syncwarp();
        if (lane < HB_ORDER) o->nlsf_pre[lane] = S->H.NLSF_Q15[lane];
        __syncwarp();
    }
    ops_copy16(&states[s], &S->hb, (int)sizeof(EncBands), lane);
}
// c_hb_lsp_quant alone: nlsf [n][8] -> index, quantised vector, Laroia weights
__global__ void __launch_bounds__(kHbWarps * 32) hb_vq_kernel(const i32* nlsf, int n, i32* idx, i32* nlsf_q, i32* weight) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int s = blockIdx.x * kHbWarps + w;
    if (s >= n) return;
    HbScr* H = &(reinterpret_cast<HbSmem*>(smem_raw) + w)->H;
    if (lane < HB_ORDER) { H->NLSF_Q15[lane] = nlsf[s * HB_ORDER + lane]; H->weight[lane] = -1; }
    __syncwarp();
    c_hb_lsp_quant(H, &idx[s]);
    __syncwarp();
    if (lane < HB_ORDER) { nlsf_q[s * HB_ORDER + lane] = H->NLSF_Q15[lane]; weight[s * HB_ORDER + lane] = H->weight[lane]; }
}

// ---- the synthesis kernel's device code (qmf_synth_group, qmf_synth_group_fix) in sb_dec_synth_kernel's layout: kSynWarps
//      warps per block (SB_SYN_WARPS of solo_b200.cu), band signals and memories staged in shared memory, a fixed-point stream
//      staged as int16 in the first half of its rows, PCM written with 8-byte stores ---------------------------------------------
constexpr int kSynWarps = 4;
enum { SYN_N2MAX = 640 };         // 40 ms of a 32 kHz stream's bands
struct SynMem { float g0[64], g1[64]; };
__global__ void __launch_bounds__(kSynWarps * 32) synth_kernel(const i32* fix_of, const i32* n2_of, SynMem* mem, const i16* band_low,
                                                               const float* band_high, i16* pcm, int n) {
    __shared__ float xx[kSynWarps][2][32 + SYN_N2MAX];
    __shared__ float coef[64];
    __shared__ i16 coef_fix[64];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < 64; i += blockDim.x) { coef[i] = SB_T(qmf_flt)[i]; coef_fix[i] = SB_T(qmf_fix)[i]; }
    __syncthreads();
    const int s = blockIdx.x * kSynWarps + w;
    if (s >= n) return;
    const int N2 = n2_of[s];
    float* xx1 = xx[w][0];
    float* xx2 = xx[w][1];
    SynMem* st = &mem[s];
    const i16* lo = band_low + (size_t)s * SYN_N2MAX;
    const float* hi = band_high + (size_t)s * SYN_N2MAX;
    int2* out = reinterpret_cast<int2*>(pcm + (size_t)s * 2 * SYN_N2MAX);
    if (fix_of[s]) {
        i16* yy1 = reinterpret_cast<i16*>(xx1);
        i16* yy2 = reinterpret_cast<i16*>(xx2);
        for (int i = lane; i < N2; i += 32) { yy1[i] = lo[N2 - 1 - i]; yy2[i] = (i16)__float2int_rz(hi[N2 - 1 - i]); }
        yy1[N2 + lane] = (i16)__float2int_rz(st->g0[2 * lane + 1]);
        yy2[N2 + lane] = (i16)__float2int_rz(st->g1[2 * lane + 1]);
        __syncwarp();
        for (int g = lane; g < N2 / 2; g += 32) {
            i16 y[4];
            qmf_synth_group_fix(yy1, yy2, coef_fix, N2, 2 * g, y);
            out[g] = make_int2((int)((u16)y[0] | ((u32)(u16)y[1] << 16)), (int)((u16)y[2] | ((u32)(u16)y[3] << 16)));
        }
        __syncwarp();
        st->g0[2 * lane + 1] = (float)yy1[lane];
        st->g1[2 * lane + 1] = (float)yy2[lane];
        return;
    }
    for (int i = lane; i < N2; i += 32) { xx1[i] = (float)lo[N2 - 1 - i]; xx2[i] = hi[N2 - 1 - i]; }
    xx1[N2 + lane] = st->g0[2 * lane + 1];
    xx2[N2 + lane] = st->g1[2 * lane + 1];
    __syncwarp();
    for (int g = lane; g < N2 / 2; g += 32) {
        i16 y[4];
        qmf_synth_group(xx1, xx2, coef, N2, 2 * g, y);
        out[g] = make_int2((int)((u16)y[0] | ((u32)(u16)y[1] << 16)), (int)((u16)y[2] | ((u32)(u16)y[3] << 16)));
    }
    __syncwarp();
    st->g0[2 * lane + 1] = xx1[lane];
    st->g1[2 * lane + 1] = xx2[lane];
}

// ---- the voice-activity kernel's body (vad_packet) in sb_enc_vad_kernel's layout: one thread per stream, kTpb threads per
//      block (SB_TPB of solo_b200.cu), the state copied to registers / local memory and back, the low band through 16-byte
//      loads.  out [n][2][6]: speech activity, four band qualities, tilt of each frame ---------------------------------------
constexpr int kTpb = 64;
__global__ void __launch_bounds__(kTpb) vad_kernel(VadState* states, const i32* nf_of, const i16* __restrict__ bands, int n, i32* out) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    VadState v = states[s];
    __align__(16) i16 low[2 * FRAME];
    const int nf = nf_of[s];
    const int4* src = reinterpret_cast<const int4*>(bands + (size_t)s * 2 * FRAME);
    int4* dst = reinterpret_cast<int4*>(low);
    for (int i = 0; i < nf * FRAME / 8; i++) dst[i] = src[i];
    i32 sa[2], q[2][4], tilt[2];
    vad_packet(&v, low, nf, sa, q, tilt);
    for (int f = 0; f < nf; f++) {
        i32* o = out + ((size_t)s * 2 + f) * 6;
        o[0] = sa[f];
        for (int b = 0; b < 4; b++) o[1 + b] = q[f][b];
        o[5] = tilt[f];
    }
    states[s] = v;
}

// ---- the last step of the entropy-coding kernel (enc_store_high_band: gains, their 32-level VQ, bit packing, length
//      fields) in sb_enc_finish_kernel's thread mapping: two threads per stream, thread k packing high-band frame k, kTpb
//      threads per block with SB_FINISH_MINB's register budget.  The kernel's earlier steps (description coding, the
//      partners' shuffles and the barrier before this store) do not run here.  lb_nb1 [n][2]: the low-band bytes and description 1's length; total [n][2]:
//      what each thread returned -----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTpb, 8) hb_store_kernel(const EncCore* states, const EncScratch* scratch, const i32* lb_nb1, u8* bits, int cap,
                                                         i16* nbytes, i32* total, int n) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int s = t >> 1, k = t & 1;
    if (s >= n) return;
    total[t] = enc_store_high_band(&states[s], &scratch[s], k, lb_nb1[2 * s], lb_nb1[2 * s + 1], bits + (size_t)s * cap, cap, &nbytes[2 * s]);
}

template <class T> struct Dev {
    T* p = nullptr;
    size_t n = 0;
    cudaError_t err = cudaSuccess;
    Dev(const T* h, size_t count) : n(count) {
        err = cudaMalloc(&p, sizeof(T) * (n ? n : 1));
        if (err == cudaSuccess && h && n) err = cudaMemcpy(p, h, sizeof(T) * n, cudaMemcpyHostToDevice);
    }
    cudaError_t back(T* h) const { return cudaMemcpy(h, p, sizeof(T) * n, cudaMemcpyDeviceToHost); }
    ~Dev() { if (p) cudaFree(p); }
};

#define SB_CHECK(e) do { const cudaError_t e_ = (e); if (e_ != cudaSuccess) return (int)e_; } while (0)
cudaError_t finish() {
    const cudaError_t e = cudaGetLastError();
    return e != cudaSuccess ? e : cudaDeviceSynchronize();
}

}  // namespace

extern "C" int sb_ops_prim(int op, const long long* a, const long long* b, const long long* c, const double* f, long long* out, int n) {
    if (n <= 0) return 0;
    Dev<long long> da(a, n), db(b, n), dc(c, n), dout(nullptr, n);
    Dev<double> df(f, n);
    SB_CHECK(da.err); SB_CHECK(db.err); SB_CHECK(dc.err); SB_CHECK(dout.err); SB_CHECK(df.err);
    prim_kernel<<<(n + 255) / 256, 256>>>(op, da.p, db.p, dc.p, df.p, dout.p, n);
    SB_CHECK(finish());
    return (int)dout.back(out);
}

extern "C" int sb_ops_schur(const int32_t* c, const int16_t* rc_in, int order, int n, int16_t* rc, int32_t* nrg, int32_t* A) {
    if (order < 1 || order > 16) return -1;
    Dev<i32> dc(c, 17 * (size_t)n), dA(nullptr, 16 * (size_t)n), dn(nullptr, n);
    Dev<i16> dri(rc_in, 16 * (size_t)n), drc(nullptr, 16 * (size_t)n);
    SB_CHECK(dc.err); SB_CHECK(dA.err); SB_CHECK(dn.err); SB_CHECK(dri.err); SB_CHECK(drc.err);
    schur_kernel<<<n, 32>>>(dc.p, dri.p, order, drc.p, dn.p, dA.p);
    SB_CHECK(finish());
    SB_CHECK(drc.back(rc)); SB_CHECK(dn.back(nrg));
    return (int)dA.back(A);
}

extern "C" int sb_ops_schur64(const int32_t* c, const int32_t* rc_in, int n, int32_t* rc, int32_t* nrg, int32_t* A) {
    Dev<i32> dc(c, 17 * (size_t)n), dri(rc_in, 16 * (size_t)n), drc(nullptr, 16 * (size_t)n), dn(nullptr, n), dA(nullptr, 16 * (size_t)n);
    SB_CHECK(dc.err); SB_CHECK(dri.err); SB_CHECK(drc.err); SB_CHECK(dn.err); SB_CHECK(dA.err);
    schur64_kernel<<<(n + 63) / 64, 64>>>(dc.p, dri.p, drc.p, dn.p, dA.p, n);
    SB_CHECK(finish());
    SB_CHECK(drc.back(rc)); SB_CHECK(dn.back(nrg));
    return (int)dA.back(A);
}

extern "C" int sb_ops_burg_xmax() { return XMAX; }

// cases: int32 [n][4] = nb0, nb1, L, WhiteNoiseFrac_Q32; x: int16 [n][2][XMAX]; outputs per half
extern "C" int sb_ops_burg(int D, const int32_t* cases, const int16_t* x, int n, int32_t* nrg, int32_t* q, int32_t* A) {
    if (D != 10 && D != 8) return -1;
    for (int i = 0; i < n; i++) {
        const int32_t* k = cases + 4 * i;
        if (k[0] < 1 || k[0] > NB_SUBFR || k[1] < 1 || k[1] > NB_SUBFR || k[2] <= D || k[0] * k[2] > XMAX || k[1] * k[2] > XMAX) return -1;
    }
    Dev<BurgCase> dk(reinterpret_cast<const BurgCase*>(cases), n);
    Dev<i16> dx(x, (size_t)n * 2 * XMAX);
    Dev<i32> dn(nullptr, 2 * (size_t)n), dq(nullptr, 2 * (size_t)n), dA(nullptr, 32 * (size_t)n);
    SB_CHECK(dk.err); SB_CHECK(dx.err); SB_CHECK(dn.err); SB_CHECK(dq.err); SB_CHECK(dA.err);
    if (D == 10) burg_kernel<10><<<n, 32>>>(dk.p, dx.p, dn.p, dq.p, dA.p);
    else burg_kernel<8><<<n, 32>>>(dk.p, dx.p, dn.p, dq.p, dA.p);
    SB_CHECK(finish());
    SB_CHECK(dn.back(nrg)); SB_CHECK(dq.back(q));
    return (int)dA.back(A);
}

// a: int32 [n][16] in / out; nlsf: int32 [n][16]
extern "C" int sb_ops_a2nlsf(int D, int32_t* a, int n, int32_t* nlsf) {
    if (D != 10 && D != 8) return -1;
    Dev<i32> da(a, 16 * (size_t)n), dn(nullptr, 16 * (size_t)n);
    SB_CHECK(da.err); SB_CHECK(dn.err);
    if (D == 10) a2nlsf_kernel<10><<<n, 32>>>(da.p, dn.p);
    else a2nlsf_kernel<8><<<n, 32>>>(da.p, dn.p);
    SB_CHECK(finish());
    SB_CHECK(da.back(a));
    return (int)dn.back(nlsf);
}

// x: int16 [n][4][SHAPE_WIN]; warping: int32 [n]; corr: int32 [n][4][17]; scale: int32 [n][4]
extern "C" int sb_ops_warped_autocorr(const int16_t* x, const int32_t* warping, int n, int32_t* corr, int32_t* scale) {
    Dev<i16> dx(x, (size_t)n * NB_SUBFR * SHAPE_WIN);
    Dev<i32> dw(warping, n), dc(nullptr, (size_t)n * NB_SUBFR * (SHAPE_ORDER + 1)), ds(nullptr, (size_t)n * NB_SUBFR);
    SB_CHECK(dx.err); SB_CHECK(dw.err); SB_CHECK(dc.err); SB_CHECK(ds.err);
    warped_kernel<<<n, 32>>>(dx.p, dw.p, dc.p, ds.p);
    SB_CHECK(finish());
    SB_CHECK(dc.back(corr));
    return (int)ds.back(scale);
}

// B: int16 [n][20] in / out; W: int32 [n][100]; mu: int32 [n]; cbk: int32 [n][4]; per: int32 [n]
extern "C" int sb_ops_quant_ltp_gains(int16_t* B, const int32_t* W, const int32_t* mu, int n, int32_t* cbk, int32_t* per) {
    Dev<i16> dB(B, (size_t)n * NB_SUBFR * LTP_ORDER);
    Dev<i32> dW(W, (size_t)n * NB_SUBFR * LTP_ORDER * LTP_ORDER), dm(mu, n), dc(nullptr, (size_t)n * NB_SUBFR), dp(nullptr, n);
    SB_CHECK(dB.err); SB_CHECK(dW.err); SB_CHECK(dm.err); SB_CHECK(dc.err); SB_CHECK(dp.err);
    ltp_kernel<<<n, 32>>>(dB.p, dW.p, dm.p, dc.p, dp.p);
    SB_CHECK(finish());
    SB_CHECK(dB.back(B)); SB_CHECK(dc.back(cbk));
    return (int)dp.back(per);
}

// cases: int32 [n][4] (PitchCase); sig: int16 [n][320]; out: int32 [n][8]
extern "C" int sb_ops_pitch(const int32_t* cases, const int16_t* sig, int n, int32_t* out) {
    if (n <= 0) return 0;
    SB_CHECK(cudaFuncSetAttribute(pitch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSlotSmem));
    Dev<PitchCase> dk(reinterpret_cast<const PitchCase*>(cases), n);
    Dev<i16> ds(sig, (size_t)n * PITCH_LEN);
    Dev<i32> dout(nullptr, (size_t)n * 8);
    SB_CHECK(dk.err); SB_CHECK(ds.err); SB_CHECK(dout.err);
    pitch_kernel<<<(n + SB_BLOCK_STREAMS - 1) / SB_BLOCK_STREAMS, SB_BLOCK_STREAMS * 32, kSlotSmem>>>(dk.p, ds.p, n, dout.p);
    SB_CHECK(finish());
    return (int)dout.back(out);
}

// cases: int32 [n][4] (MsvqCase); nlsf, prev, w: int32 [n][10]; idx: int32 [n][6]; nlsf_q: int32 [n][10]
extern "C" int sb_ops_msvq(const int32_t* cases, const int32_t* nlsf, const int32_t* prev, const int32_t* w, int n, int32_t* idx, int32_t* nlsf_q) {
    if (n <= 0) return 0;
    for (int i = 0; i < n; i++) if (cases[4 * i + 3] != 0 && cases[4 * i + 3] != 1) return -1;
    SB_CHECK(cudaFuncSetAttribute(msvq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSlotSmem));
    Dev<MsvqCase> dk(reinterpret_cast<const MsvqCase*>(cases), n);
    Dev<i32> dn(nlsf, (size_t)n * LPC_ORDER), dp(prev, (size_t)n * LPC_ORDER), dw(w, (size_t)n * LPC_ORDER);
    Dev<i32> di(nullptr, (size_t)n * 6), dq(nullptr, (size_t)n * LPC_ORDER);
    SB_CHECK(dk.err); SB_CHECK(dn.err); SB_CHECK(dp.err); SB_CHECK(dw.err); SB_CHECK(di.err); SB_CHECK(dq.err);
    msvq_kernel<<<(n + SB_BLOCK_STREAMS - 1) / SB_BLOCK_STREAMS, SB_BLOCK_STREAMS * 32, kSlotSmem>>>(dk.p, dn.p, dp.p, dw.p, n, di.p, dq.p);
    SB_CHECK(finish());
    SB_CHECK(di.back(idx));
    return (int)dq.back(nlsf_q);
}

extern "C" void nsq_io_sizes(int* s) { NSQ_IO_SIZES(s); }

// n cases of npk packets of nf frames (oracle/nsq_io.h): st0 [n][3], fr [n][npk * nf] -> out [n][npk * nf] after every
// frame, st_after [n][npk][3] after every packet.  One launch per packet; the states stay on the device between packets and
// the scratch outputs (pulses, centre excitation, random-generator history) are poisoned with 0xA5 before every launch.
extern "C" int sb_ops_nsq(int n, int npk, int nf, const NsqStateIO* st0, const NsqFrameIn* fr, NsqFrameOut* out, NsqStateIO* st_after) {
    if (n <= 0 || npk <= 0 || (nf != 1 && nf != 2)) return -1;
    const int nfr = npk * nf;
    const int smem = kNsqSpb * (int)sizeof(NsqSmem);
    SB_CHECK(cudaFuncSetAttribute(nsq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    std::vector<NsqState> ns((size_t)n * 3);
    std::vector<EncScratch> scr(n);
    for (int i = 0; i < n * 3; i++) nsqio_state_to(&ns[i], &st0[i]);
    Dev<NsqState> dns(ns.data(), ns.size());
    Dev<EncScratch> dscr(nullptr, scr.size());
    SB_CHECK(dns.err); SB_CHECK(dscr.err);
    for (int p = 0; p < npk; p++) {
        for (int s = 0; s < n; s++) {
            memset(&scr[s], 0, sizeof(EncScratch));
            memset(scr[s].q_md, 0xA5, sizeof(scr[s].q_md));
            memset(scr[s].r16, 0xA5, sizeof(scr[s].r16));
            memset(scr[s].nsq_rand, 0xA5, sizeof(scr[s].nsq_rand));
            for (int f = 0; f < nf; f++) {
                const NsqFrameIn* x = &fr[(size_t)s * nfr + p * nf + f];
                nsqio_ctrl(&scr[s].c[f], x);
                memcpy(scr[s].xfw[f], x->x, sizeof(scr[s].xfw[f]));
            }
        }
        SB_CHECK(cudaMemcpy(dscr.p, scr.data(), sizeof(EncScratch) * scr.size(), cudaMemcpyHostToDevice));
        nsq_kernel<<<(n + kNsqSpb - 1) / kNsqSpb, 32, smem>>>(dns.p, dscr.p, nf, n);
        SB_CHECK(finish());
        SB_CHECK(dscr.back(scr.data()));
        SB_CHECK(dns.back(ns.data()));
        for (int s = 0; s < n; s++) {
            for (int f = 0; f < nf; f++) {
                NsqFrameOut* o = &out[(size_t)s * nfr + p * nf + f];
                memcpy(o->q_md, scr[s].q_md[f], sizeof(o->q_md));
                memcpy(o->r16, scr[s].r16[f], sizeof(o->r16));
                o->Seed = scr[s].c[f].Seed;
            }
            for (int qz = 0; qz < 3; qz++) nsqio_state_from(&st_after[((size_t)s * npk + p) * 3 + qz], &ns[s * 3 + qz]);
        }
    }
    return 0;
}

// n cases of npk packets: spp [n] (640 or 320 samples per packet), mem0 [n][64], pcm [n][npk][PACKET] -> bands [n][npk][PACKET]
// ([low | high], spp samples), mem_after [n][npk][64].  One launch per packet; the memories stay on the device between them.
extern "C" int sb_ops_qmf_split(int n, int npk, const int32_t* spp, const int16_t* mem0, const int16_t* pcm, int16_t* bands, int16_t* mem_after) {
    if (n <= 0 || npk <= 0) return -1;
    for (int i = 0; i < n; i++) if (spp[i] != PACKET && spp[i] != PACKET / 2) return -1;
    Dev<i32> dspp(spp, n);
    Dev<i16> dmem(mem0, (size_t)n * 64), dpcm(nullptr, (size_t)n * PACKET), dout(nullptr, (size_t)n * PACKET);
    SB_CHECK(dspp.err); SB_CHECK(dmem.err); SB_CHECK(dpcm.err); SB_CHECK(dout.err);
    std::vector<i16> h((size_t)n * PACKET);
    for (int p = 0; p < npk; p++) {
        for (int s = 0; s < n; s++) memcpy(&h[(size_t)s * PACKET], pcm + ((size_t)s * npk + p) * PACKET, sizeof(i16) * PACKET);
        SB_CHECK(cudaMemcpy(dpcm.p, h.data(), sizeof(i16) * h.size(), cudaMemcpyHostToDevice));
        SB_CHECK(cudaMemset(dout.p, 0xA5, sizeof(i16) * h.size()));
        qmf_split_kernel<<<n, 32>>>(dspp.p, dmem.p, dpcm.p, dout.p);
        SB_CHECK(finish());
        SB_CHECK(dout.back(h.data()));
        for (int s = 0; s < n; s++) memcpy(bands + ((size_t)s * npk + p) * PACKET, &h[(size_t)s * PACKET], sizeof(i16) * PACKET);
        std::vector<i16> m((size_t)n * 64);
        SB_CHECK(dmem.back(m.data()));
        for (int s = 0; s < n; s++) memcpy(mem_after + ((size_t)s * npk + p) * 64, &m[(size_t)s * 64], sizeof(i16) * 64);
    }
    return 0;
}

extern "C" int sb_ops_hb_out_bytes() { return (int)sizeof(HbFrameOut); }

// n cases of npk packets from the reset state (zero buffer, hb_first = 1 as enc_state_fields sets it): cases [n] (F, samples
// per packet), high [n][npk][PACKET / 2] -> out [n][npk][2] (HbFrameOut; a packet of one frame leaves its second record
// zero).  per_frame: see hb_kernel.  One launch per packet.
// (out is untyped here: a parameter of the harness's internal record type would give the entry point internal linkage)
extern "C" int sb_ops_hb(int n, int npk, int per_frame, const int32_t* cases, const int16_t* high, void* out_) {
    HbFrameOut* out = static_cast<HbFrameOut*>(out_);
    if (n <= 0 || npk <= 0) return -1;
    for (int i = 0; i < n; i++) {
        const int F = cases[2 * i], m = cases[2 * i + 1];
        if ((F != HB_FRAME && F != 2 * HB_FRAME) || (m != HB_FRAME && m != 2 * HB_FRAME) || m % F) return -1;
    }
    SB_CHECK(cudaFuncSetAttribute(hb_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kHbSmem));
    Dev<HbCase> dk(reinterpret_cast<const HbCase*>(cases), n);
    std::vector<EncBands> reset(n);
    memset(reset.data(), 0, sizeof(EncBands) * n);
    for (int i = 0; i < n; i++) reset[i].hb_first = 1;
    Dev<EncBands> dst(reset.data(), n);
    Dev<EncScratch> dscr(nullptr, n);
    Dev<i16> dhigh(nullptr, (size_t)n * (PACKET / 2));
    Dev<HbFrameOut> dout(nullptr, (size_t)n * 2);
    SB_CHECK(dk.err); SB_CHECK(dst.err); SB_CHECK(dscr.err); SB_CHECK(dhigh.err); SB_CHECK(dout.err);
    std::vector<i16> h((size_t)n * (PACKET / 2));
    std::vector<HbFrameOut> o((size_t)n * 2);
    for (int p = 0; p < npk; p++) {
        for (int s = 0; s < n; s++) memcpy(&h[(size_t)s * (PACKET / 2)], high + ((size_t)s * npk + p) * (PACKET / 2), sizeof(i16) * (PACKET / 2));
        SB_CHECK(cudaMemcpy(dhigh.p, h.data(), sizeof(i16) * h.size(), cudaMemcpyHostToDevice));
        SB_CHECK(cudaMemset(dout.p, 0, sizeof(HbFrameOut) * o.size()));
        hb_kernel<<<(n + kHbWarps - 1) / kHbWarps, kHbWarps * 32, kHbSmem>>>(dk.p, dst.p, dscr.p, dhigh.p, n, per_frame, dout.p);
        SB_CHECK(finish());
        SB_CHECK(dout.back(o.data()));
        for (int s = 0; s < n; s++) memcpy(out + ((size_t)s * npk + p) * 2, &o[(size_t)s * 2], sizeof(HbFrameOut) * 2);
    }
    return 0;
}

// nlsf [n][8] -> idx [n], nlsf_q [n][8], weight [n][8]
extern "C" int sb_ops_hb_vq(int n, const int32_t* nlsf, int32_t* idx, int32_t* nlsf_q, int32_t* weight) {
    if (n <= 0) return -1;
    SB_CHECK(cudaFuncSetAttribute(hb_vq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kHbSmem));
    Dev<i32> dn(nlsf, (size_t)n * HB_ORDER), di(nullptr, n), dq(nullptr, (size_t)n * HB_ORDER), dw(nullptr, (size_t)n * HB_ORDER);
    SB_CHECK(dn.err); SB_CHECK(di.err); SB_CHECK(dq.err); SB_CHECK(dw.err);
    hb_vq_kernel<<<(n + kHbWarps - 1) / kHbWarps, kHbWarps * 32, kHbSmem>>>(dn.p, n, di.p, dq.p, dw.p);
    SB_CHECK(finish());
    SB_CHECK(di.back(idx)); SB_CHECK(dq.back(nlsf_q));
    return (int)dw.back(weight);
}

// n streams of npk packets: fix [n] (0 = float, 1 = fixed point), n2 [n] (160, 320 or 640 band samples per packet), mem0 [n]
// (g0_mem, g1_mem), low [n][npk][640] int16, high [n][npk][640] float -> pcm [n][npk][1280], mem_after [n][npk].  One launch
// per packet; the memories stay on the device between them.
extern "C" int sb_ops_synth(int n, int npk, const int32_t* fix, const int32_t* n2, const float* mem0, const int16_t* low, const float* high,
                            int16_t* pcm, float* mem_after) {
    if (n <= 0 || npk <= 0) return -1;
    for (int i = 0; i < n; i++) if (n2[i] != 160 && n2[i] != 320 && n2[i] != 640) return -1;
    const size_t B = SYN_N2MAX;
    Dev<i32> dfix(fix, n), dn2(n2, n);
    Dev<SynMem> dmem(reinterpret_cast<const SynMem*>(mem0), n);
    Dev<i16> dlow(nullptr, n * B), dpcm(nullptr, n * 2 * B);
    Dev<float> dhigh(nullptr, n * B);
    SB_CHECK(dfix.err); SB_CHECK(dn2.err); SB_CHECK(dmem.err); SB_CHECK(dlow.err); SB_CHECK(dpcm.err); SB_CHECK(dhigh.err);
    std::vector<i16> hl(n * B), hp(n * 2 * B);
    std::vector<float> hh(n * B);
    std::vector<SynMem> m(n);
    for (int p = 0; p < npk; p++) {
        for (int s = 0; s < n; s++) {
            memcpy(&hl[s * B], low + ((size_t)s * npk + p) * B, sizeof(i16) * B);
            memcpy(&hh[s * B], high + ((size_t)s * npk + p) * B, sizeof(float) * B);
        }
        SB_CHECK(cudaMemcpy(dlow.p, hl.data(), sizeof(i16) * hl.size(), cudaMemcpyHostToDevice));
        SB_CHECK(cudaMemcpy(dhigh.p, hh.data(), sizeof(float) * hh.size(), cudaMemcpyHostToDevice));
        SB_CHECK(cudaMemset(dpcm.p, 0xA5, sizeof(i16) * hp.size()));
        synth_kernel<<<(n + kSynWarps - 1) / kSynWarps, kSynWarps * 32>>>(dfix.p, dn2.p, dmem.p, dlow.p, dhigh.p, dpcm.p, n);
        SB_CHECK(finish());
        SB_CHECK(dpcm.back(hp.data()));
        SB_CHECK(dmem.back(m.data()));
        for (int s = 0; s < n; s++) {
            memcpy(pcm + ((size_t)s * npk + p) * 2 * B, &hp[s * 2 * B], sizeof(i16) * 2 * B);
            memcpy(mem_after + ((size_t)s * npk + p) * 128, &m[s], sizeof(SynMem));
        }
    }
    return 0;
}

// n streams of npk packets of nf [n] frames: st0 [n][28], low [n][npk][2][FRAME] -> out [n][npk][2][6] (see vad_kernel; a
// 20 ms stream's second row stays zero), st_after [n][npk][28].  One launch per packet; the states stay on the device.
extern "C" int sb_ops_vad(int n, int npk, const int32_t* nf, const int32_t* st0, const int16_t* low, int32_t* out, int32_t* st_after) {
    if (n <= 0 || npk <= 0) return -1;
    for (int i = 0; i < n; i++) if (nf[i] != 1 && nf[i] != 2) return -1;
    std::vector<VadState> v(n);
    for (int s = 0; s < n; s++) vadio_to(&v[s], st0 + (size_t)s * VADIO_WORDS);
    Dev<VadState> dv(v.data(), n);
    Dev<i32> dnf(nf, n), dout(nullptr, (size_t)n * 12);
    Dev<i16> dlow(nullptr, (size_t)n * 2 * FRAME);
    SB_CHECK(dv.err); SB_CHECK(dnf.err); SB_CHECK(dout.err); SB_CHECK(dlow.err);
    std::vector<i16> h((size_t)n * 2 * FRAME);
    std::vector<i32> o((size_t)n * 12);
    for (int p = 0; p < npk; p++) {
        for (int s = 0; s < n; s++) memcpy(&h[(size_t)s * 2 * FRAME], low + ((size_t)s * npk + p) * 2 * FRAME, sizeof(i16) * 2 * FRAME);
        SB_CHECK(cudaMemcpy(dlow.p, h.data(), sizeof(i16) * h.size(), cudaMemcpyHostToDevice));
        SB_CHECK(cudaMemset(dout.p, 0, sizeof(i32) * o.size()));
        vad_kernel<<<(n + kTpb - 1) / kTpb, kTpb>>>(dv.p, dnf.p, dlow.p, n, dout.p);
        SB_CHECK(finish());
        SB_CHECK(dout.back(o.data()));
        SB_CHECK(dv.back(v.data()));
        for (int s = 0; s < n; s++) {
            memcpy(out + ((size_t)s * npk + p) * 12, &o[(size_t)s * 12], sizeof(i32) * 12);
            vadio_from(st_after + ((size_t)s * npk + p) * VADIO_WORDS, &v[s]);
        }
    }
    return 0;
}

// n packets, one per stream: cfg [n][4] = frames per packet, high-band frame length, low-band bytes lb, description 1's
// length nb1; lsp_idx [n][2], nrg0 [n][2][4], r16 [n][2][FRAME] (the high-band frames' inputs) -> bits [n][cap] (poisoned
// with 0xA5 first), nbytes [n][2], total [n][2] (each thread's return value).  One launch.
extern "C" int sb_ops_hb_store(int n, int cap, const int32_t* cfg, const int32_t* lsp_idx, const int32_t* nrg0, const int16_t* r16,
                               uint8_t* bits, int16_t* nbytes, int32_t* total) {
    if (n <= 0 || cap <= 0) return -1;
    std::vector<EncCore> st(n);
    std::vector<EncScratch> scr(n);
    std::vector<i32> lb(2 * (size_t)n);
    for (int s = 0; s < n; s++) {
        const int32_t* c = cfg + 4 * (size_t)s;
        if ((c[0] != 1 && c[0] != 2) || (c[1] != HB_FRAME && c[1] != 2 * HB_FRAME) || c[0] * FRAME < c[1]) return -1;
        memset(&st[s], 0, sizeof(EncCore));
        memset(&scr[s], 0, sizeof(EncScratch));
        st[s].frames_per_packet = c[0];
        st[s].hb_frame = c[1];
        lb[2 * s] = c[2];
        lb[2 * s + 1] = c[3];
        memcpy(scr[s].hb_lsp_idx, lsp_idx + 2 * (size_t)s, sizeof(scr[s].hb_lsp_idx));
        memcpy(scr[s].hb_nrg0, nrg0 + 8 * (size_t)s, sizeof(scr[s].hb_nrg0));
        memcpy(scr[s].r16, r16 + 2 * FRAME * (size_t)s, sizeof(scr[s].r16));
    }
    Dev<EncCore> dst(st.data(), n);
    Dev<EncScratch> dscr(scr.data(), n);
    Dev<i32> dlb(lb.data(), lb.size()), dtot(nullptr, 2 * (size_t)n);
    Dev<u8> dbits(nullptr, (size_t)n * cap);
    Dev<i16> dnb(nullptr, 2 * (size_t)n);
    SB_CHECK(dst.err); SB_CHECK(dscr.err); SB_CHECK(dlb.err); SB_CHECK(dtot.err); SB_CHECK(dbits.err); SB_CHECK(dnb.err);
    SB_CHECK(cudaMemset(dbits.p, 0xA5, (size_t)n * cap));
    SB_CHECK(cudaMemset(dnb.p, 0xA5, sizeof(i16) * 2 * (size_t)n));
    hb_store_kernel<<<(2 * n + kTpb - 1) / kTpb, kTpb>>>(dst.p, dscr.p, dlb.p, dbits.p, cap, dnb.p, dtot.p, n);
    SB_CHECK(finish());
    SB_CHECK(dbits.back(bits)); SB_CHECK(dnb.back(nbytes));
    return (int)dtot.back(total);
}
