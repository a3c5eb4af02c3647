// solo_b200 -- encoder stage A as warp-per-stream kernels (sm_90a).
//
// This translation unit compiles the analysis routines in their cooperative form (sb_coop.cuh): the 32 lanes of a warp work on
// ONE stream, whose persistent analysis state and per-packet working set live in shared memory for the duration of the packet.
//   sb_enc_analysis_warp_kernel : SILK core analysis of both 20 ms frames (VAD .. gain processing) -> EncScratch
//   sb_enc_hb_warp_kernel       : high-band analysis (order-8 LPC, LSP VQ, sub-frame energies)     -> EncScratch
// State moves between HBM and shared memory with 128-bit accesses, 512 contiguous bytes per warp instruction; both kernels
// read the band-split rows [low | high] that the QMF kernel (solo_b200.cu) wrote.
#define SB_COOP 1
// Code size is a first-order cost here: a warp executes most of its instructions once per packet, so the kernel streams its
// code through the 32 KB instruction cache.  Routines with many call sites are kept out of line in this translation unit.
#ifndef SB_ANA_INLINE_ALL
#define SB_DIV_OUTLINE 1
#endif
#ifndef SB_NO_PHASE_ALIGN
#define SB_PHASE_ALIGN 1
#endif
#ifndef SB_ANA_WARPS
#define SB_ANA_WARPS 8      // streams per block of the core-analysis kernel; its warps pass the phases together, two blocks per SM
#endif
#ifndef SB_NO_XPOSE
#define SB_XPOSE 1          // scalar recursions of all streams of a block run side by side on consecutive threads (sb_par.cuh)
#define SB_BLOCK_STREAMS SB_ANA_WARPS
#endif
#include <cuda_runtime.h>
#include "sb_coop.cuh"

using namespace sb;

#ifndef SB_HB_WARPS
#define SB_HB_WARPS 4
#endif

namespace {

struct HbSmem {
    EncBands hb;
    HbScr H;
    alignas(16) i16 high[PACKET / 2];
};
static_assert(sizeof(EncSilk) % 16 == 0 && sizeof(EncBands) % 16 == 0, "state parts are moved with 128-bit accesses");
static_assert(sizeof(EncState) % 16 == 0, "stream stride keeps the parts 16-byte aligned");
static_assert(sizeof(AnaSmem) % 16 == 0 && sizeof(HbSmem) % 16 == 0, "per-warp shared-memory slots stay 16-byte aligned");

__device__ __forceinline__ void copy16(void* dst, const void* src, int bytes, int lane) {
    const int4* s = reinterpret_cast<const int4*>(src);
    int4* d = reinterpret_cast<int4*>(dst);
    for (int i = lane; i < bytes / 16; i += 32) d[i] = s[i];
}

#ifndef SB_ANA_SMEM_TABS
#define SB_ANA_SMEM_TABS 1  // a copy of the NLSF codebooks (4.2 KB) per block in shared memory
#endif
#define SB_ANA_TABS_BYTES (SB_ANA_SMEM_TABS ? ((sizeof(NlsfFastTabs) + 15) & ~15) : 0)
#ifndef SB_ANA_MINB
#define SB_ANA_MINB 2      // resident blocks per SM the register budget is sized for
#endif
__global__ void __launch_bounds__(SB_ANA_WARPS * 32, SB_ANA_MINB) sb_enc_analysis_warp_kernel(EncState* states, EncScratch* scratch, const i16* __restrict__ bands, int spp, int n) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
#if SB_ANA_SMEM_TABS
    NlsfFastTabs* tabs = reinterpret_cast<NlsfFastTabs*>(smem_raw);
    nlsf_fast_tabs_fill(tabs, threadIdx.x, blockDim.x);
    __syncthreads();
#else
    NlsfFastTabs* tabs = nullptr;        // code vectors come from the global tables (L1 / L2 resident)
#endif
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int s = blockIdx.x * SB_ANA_WARPS + w;
    // every warp of the block takes part in the phase barriers: a warp beyond the batch shadows the last stream (same inputs,
    // same values stored to the same scratch slot) and does not write state back
    const bool live = s < n;
    if (!live) s = n - 1;
    // the slot address as an opaque 32-bit shared-window offset: kept in a register instead of being recomputed from threadIdx
    // at every use (the compiler otherwise rematerialises it ~130 times)
    unsigned slot = (unsigned)__cvta_generic_to_shared(smem_raw + SB_ANA_TABS_BYTES) + (unsigned)w * (unsigned)sizeof(AnaSmem);
    asm volatile("" : "+r"(slot));
    AnaSmem* S = reinterpret_cast<AnaSmem*>(__cvta_shared_to_generic(slot));
    copy16(&S->st, static_cast<EncSilk*>(&states[s]), (int)sizeof(EncSilk), lane);
    copy16(S->W.low, bands + (size_t)s * spp, spp, lane);          // low band = first half of the row (spp / 2 samples)
    __syncwarp();
    c_enc_packet_analysis(&S->st, &S->W, &scratch[s], tabs);
    __syncwarp();
    if (live) copy16(static_cast<EncSilk*>(&states[s]), &S->st, (int)sizeof(EncSilk), lane);
}

__global__ void __launch_bounds__(SB_HB_WARPS * 32) sb_enc_hb_warp_kernel(EncState* states, EncScratch* scratch, const i16* __restrict__ bands, int spp, int n) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int s = blockIdx.x * SB_HB_WARPS + w;
    if (s >= n) return;
    HbSmem* S = reinterpret_cast<HbSmem*>(smem_raw) + w;
    copy16(&S->hb, static_cast<EncBands*>(&states[s]), (int)sizeof(EncBands), lane);
    copy16(S->high, bands + (size_t)s * spp + spp / 2, spp, lane);  // high band = second half of the row
    __syncwarp();
    const int F = states[s].hb_frame, nhb = (spp / 2) / F;
    EncScratch* scr = &scratch[s];
    for (int f = 0; f < nhb; f++) {
        if (F == HB_FRAME) c_hb_analyse_frame<HB_FRAME>(&S->hb, &S->H, S->high + f * F, &scr->hb_lsp_idx[f], scr->hb_nrg0[f]);
        else c_hb_analyse_frame<2 * HB_FRAME>(&S->hb, &S->H, S->high + f * F, &scr->hb_lsp_idx[f], scr->hb_nrg0[f]);
    }
    __syncwarp();
    // qmf_mem belongs to the band-split kernel: only the high-band ring and its flag go back
    copy16(static_cast<EncBands*>(&states[s])->x_hb_buf, S->hb.x_hb_buf, (int)(sizeof(EncBands) - offsetof(EncBands, x_hb_buf)), lane);
}

}  // namespace

// called from the host code in solo_b200.cu; return a CUDA error code
extern "C" int sb_launch_enc_analysis_warp(void* states, void* scratch, const void* bands, int spp, int n, void* stream) {
    static bool configured = false;
    const int smem = (int)SB_ANA_TABS_BYTES + SB_ANA_WARPS * (int)sizeof(AnaSmem);
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(sb_enc_analysis_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return (int)e;
        configured = true;
    }
    sb_enc_analysis_warp_kernel<<<(n + SB_ANA_WARPS - 1) / SB_ANA_WARPS, SB_ANA_WARPS * 32, smem, (cudaStream_t)stream>>>(
        (EncState*)states, (EncScratch*)scratch, (const i16*)bands, spp, n);
    return (int)cudaGetLastError();
}
extern "C" int sb_launch_enc_hb_warp(void* states, void* scratch, const void* bands, int spp, int n, void* stream) {
    static bool configured = false;
    const int smem = SB_HB_WARPS * (int)sizeof(HbSmem);
    if (!configured) {
        cudaError_t e = cudaFuncSetAttribute(sb_enc_hb_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) return (int)e;
        configured = true;
    }
    sb_enc_hb_warp_kernel<<<(n + SB_HB_WARPS - 1) / SB_HB_WARPS, SB_HB_WARPS * 32, smem, (cudaStream_t)stream>>>(
        (EncState*)states, (EncScratch*)scratch, (const i16*)bands, spp, n);
    return (int)cudaGetLastError();
}
#ifdef SB_PHASE_TIMING
extern "C" int sb_phase_times_read(long long* stamps, int* lines, int cap) {
    int n = 0;
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(&n, sb_phase_count, sizeof(int));
    if (n > cap) n = cap;
    cudaMemcpyFromSymbol(stamps, sb_phase_stamp, sizeof(long long) * n);
    cudaMemcpyFromSymbol(lines, sb_phase_line, sizeof(int) * n);
    int zero = 0;
    cudaMemcpyToSymbol(sb_phase_count, &zero, sizeof(int));
    return n;
}
#endif
extern "C" int sb_analysis_smem_bytes(int which) { return which == 0 ? (int)sizeof(AnaSmem) : (int)sizeof(HbSmem); }
