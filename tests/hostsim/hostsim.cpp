// Host build of the per-stream kernel source (solo_b200/csrc/*.cuh compiled by g++).
// TEST INFRASTRUCTURE ONLY: lets the CPU-only container check the kernel logic bit-for-bit against the
// compiled reference (oracle/_ref).  Never linked into libsolo_b200.so.
// With -DSB_EMU the analysis stage runs in its cooperative form on 32 OS threads per stream (sb_par.cuh), so that
// races / missing barriers of the warp-per-stream kernel can be caught without a GPU.
#ifdef SB_EMU
// 32 lanes of one stream as 32 fibers on one OS thread, run round-robin between barriers: lane 0 runs to its next barrier,
// then lane 1, ... so a lane that reads what another lane has not written yet (missing SB_SYNC) or that takes a different
// number of barriers (divergent collective) shows up deterministically.
#include <ucontext.h>
#include <stdio.h>
#include <stdlib.h>
#include <functional>
#include "../../solo_b200/csrc/sb_common.cuh"
namespace sb { namespace emu {
int lane = 0;
static ucontext_t ctx[32], main_ctx;
static char* stacks[32];
static long long scr[32];
static long nbar[32];
static std::function<void()> body;
void barrier() {
    const int me = lane;
    nbar[me]++;
    lane = (me + 1) & 31;
    swapcontext(&ctx[me], &ctx[lane]);
    lane = me;
    if (me == 0)      // a full round has passed: every lane must have arrived at its barrier number nbar[0]
        for (int i = 1; i < 32; i++)
            if (nbar[i] != nbar[0]) { fprintf(stderr, "emu: divergent collective -- lane %d is at barrier %ld, lane 0 at %ld\n", i, nbar[i], nbar[0]); abort(); }
}
long long* scratch() { return scr; }
static void entry() { body(); }
// run f on 32 lanes (f reads sb::emu::lane)
static void run32(const std::function<void()>& f) {
    body = f;
    for (int i = 0; i < 32; i++) {
        if (!stacks[i]) stacks[i] = (char*)malloc(1 << 20);
        getcontext(&ctx[i]);
        ctx[i].uc_stack.ss_sp = stacks[i];
        ctx[i].uc_stack.ss_size = 1 << 20;
        ctx[i].uc_link = i < 31 ? &ctx[i + 1] : &main_ctx;
        makecontext(&ctx[i], (void (*)())entry, 0);
        nbar[i] = 0;
    }
    // a lane that returns falls through (uc_link) into the next lane's saved context; `lane` is restored inside barrier()
    lane = 0;
    swapcontext(&main_ctx, &ctx[0]);
    for (int i = 1; i < 32; i++)
        if (nbar[i] != nbar[0]) { fprintf(stderr, "emu: lane %d took %ld barriers, lane 0 took %ld (divergent collective)\n", i, nbar[i], nbar[0]); abort(); }
    lane = 0;
}

// ---- a second scheduler for code whose collectives name a lane mask (the quantiser kernel: two 16-lane groups that may take
//      different paths between the full-warp sections).  barrier_mask(m) really waits: a lane spins (yielding round-robin to
//      the other lanes) until every lane of m has arrived at a barrier with the same mask.  Lanes finish at different times. ----
static bool done_[32];
static struct MaskBar { unsigned mask, arrived; unsigned long phase; } mbar[8];
static int n_mbar;
static long spins;
static void yield_next() {
    const int me = lane;
    for (int k = 1; k <= 32; k++) {
        const int nx = (me + k) & 31;
        if (!done_[nx]) { if (nx == me) return; lane = nx; swapcontext(&ctx[me], &ctx[nx]); lane = me; return; }
    }
}
void barrier_mask(unsigned m) {
    const int me = lane;
    MaskBar* e = nullptr;
    for (int i = 0; i < n_mbar; i++) if (mbar[i].mask == m) e = &mbar[i];
    if (!e) { if (n_mbar == 8) { fprintf(stderr, "emu: too many distinct lane masks\n"); abort(); } e = &mbar[n_mbar++]; e->mask = m; e->arrived = 0; e->phase = 0; }
    if (!((m >> me) & 1)) { fprintf(stderr, "emu: lane %d at a barrier whose mask %08x does not name it\n", me, m); abort(); }
    const unsigned long my_phase = e->phase;
    e->arrived |= 1u << me;
    if (e->arrived == m) { e->arrived = 0; e->phase++; spins = 0; }
    while (e->phase == my_phase) {
        if (++spins > 100000000L) { fprintf(stderr, "emu: deadlock -- lanes %08x of mask %08x never arrived (divergent collective)\n", m & ~e->arrived, m); abort(); }
        yield_next();
    }
}
static void entry_m() {
    body();
    const int me = lane;
    done_[me] = true;
    for (int k = 1; k < 32; k++) { const int nx = (me + k) & 31; if (!done_[nx]) { lane = nx; setcontext(&ctx[nx]); } }
    setcontext(&main_ctx);
}
static void run32m(const std::function<void()>& f) {
    body = f;
    n_mbar = 0; spins = 0;
    for (int i = 0; i < 32; i++) {
        if (!stacks[i]) stacks[i] = (char*)malloc(1 << 20);
        getcontext(&ctx[i]);
        ctx[i].uc_stack.ss_sp = stacks[i];
        ctx[i].uc_stack.ss_size = 1 << 20;
        ctx[i].uc_link = &main_ctx;
        makecontext(&ctx[i], (void (*)())entry_m, 0);
        done_[i] = false;
    }
    lane = 0;
    swapcontext(&main_ctx, &ctx[0]);
    lane = 0;
}
} }
#endif
#include "../../solo_b200/csrc/sb_enc.cuh"
#include "../../solo_b200/csrc/sb_dec.cuh"
#include "../../solo_b200/csrc/sb_activity.cuh"
#include "../../oracle/nsq_io.h"
#include "../../oracle/vad_io.h"
#ifdef SB_EMU
#include "../../solo_b200/csrc/sb_coop.cuh"
// ---- the quantiser kernel's device code (sb_nsq_warp.cuh) under the same 32-fibre emulation: one stream per "warp"
//      (SB_NSQ_GW = 32), the CUDA warp intrinsics it uses as shims over the emulation's exchange buffer ----
namespace {
struct EmuThreadIdx { struct X { operator int() const { return sb::emu::lane; } } x; } threadIdx;
static long long xbuf[32];     // exchange line of the shims (one slot per lane)
template <class T> inline T emu_xchg(unsigned m, T v, int src) {
    xbuf[sb::emu::lane] = (long long)v;
    sb::emu::barrier_mask(m);
    const T r = (T)xbuf[src & 31];
    sb::emu::barrier_mask(m);
    return r;
}
template <class T> inline T __shfl_sync(unsigned m, T v, int src, int w = 32) { return emu_xchg<T>(m, v, (sb::emu::lane & ~(w - 1)) | (src & (w - 1))); }
template <class T> inline T __shfl_down_sync(unsigned m, T v, int d, int w = 32) {
    const int l = sb::emu::lane;
    return emu_xchg<T>(m, v, ((l & (w - 1)) + d < w) ? l + d : l);
}
inline unsigned __ballot_sync(unsigned m, bool p) {
    xbuf[sb::emu::lane] = p ? 1 : 0;
    sb::emu::barrier_mask(m);
    unsigned r = 0;
    for (int i = 0; i < 32; i++) if ((m >> i) & 1) r |= (unsigned)xbuf[i] << i;
    sb::emu::barrier_mask(m);
    return r;
}
inline bool __any_sync(unsigned m, bool p) { return __ballot_sync(m, p) != 0; }
inline int __reduce_max_sync(unsigned m, int v) {
    xbuf[sb::emu::lane] = v;
    sb::emu::barrier_mask(m);
    int r = v;
    for (int i = 0; i < 32; i++) if (((m >> i) & 1) && (int)xbuf[i] > r) r = (int)xbuf[i];
    sb::emu::barrier_mask(m);
    return r;
}
inline void __syncwarp(unsigned m = 0xffffffffu) { sb::emu::barrier_mask(m); }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __mulhi(int a, int b) { return (int)(((long long)a * (long long)b) >> 32); }
}
#ifdef SB_EMU_GW16
#define SB_NSQ_GW 16     // the kernel's packing: two lane groups per warp; here the second group shadows the first one's stream
#else                    // (what the kernel does with the last stream of an odd batch), so both take the same path
#define SB_NSQ_GW 32
#endif
#include "../../solo_b200/csrc/sb_nsq_warp.cuh"
static int g_emu_nsq = 0;
extern "C" void hs_set_emu_nsq(int on) { g_emu_nsq = on; }
#endif
#include <stdlib.h>

extern "C" {
struct HsEnc { sb::EncState st; sb::EncPacketWork w; };
void* hs_enc_create3(int rate, int dtx, int mdi, int framesize_ms, int joint_hb) {
    HsEnc* h = (HsEnc*)calloc(1, sizeof(HsEnc));
    sb::enc_state_init(&h->st, rate, dtx, mdi, framesize_ms, joint_hb);
    return h;
}
#ifdef SB_EMU
// the core and high-band analysis kernels' code (sb_coop.cuh) on emulated lanes
static void emu_analysis(HsEnc* h) {
    static sb::CoopWork cw;
    static sb::HbScr hs;
    const int nf = h->st.frames_per_packet;
    for (int i = 0; i < nf * sb::FRAME; i++) cw.low[i] = h->w.a.low[i];
    sb::emu::run32([=]() { sb::c_enc_packet_analysis(&h->st, &cw, &h->w.scr); });
    sb::emu::run32([=]() { sb::c_hb_analyse_packet(&h->st, &hs, h->w.a.high, nf * sb::FRAME, h->st.hb_frame, &h->w.scr); });
}
// the quantiser kernel's code for one warp: lane group g works on stream hh[g] (one group with SB_NSQ_GW = 32)
static void emu_nsq(HsEnc* const* hh) {
    static sb::NsqSmem S[2];
    sb::emu::run32m([=]() {
        const int g = sb::emu::lane / SB_NSQ_GW;
        sb::nsq_packet_warp(S[g], hh[g]->st.nsq, &hh[g]->w.scr, hh[g]->st.frames_per_packet);
    });
}
#endif
// the stages of sb::enc_packet up to the quantiser; the emulated build swaps in the cooperative analysis
static void enc_front(HsEnc* h, const short* pcm) {
    sb::enc_packet_bands(&h->st, &h->w, pcm);
#ifdef SB_EMU
    emu_analysis(h);
#else
    sb::enc_packet_analysis(&h->st, &h->w.a, &h->w.scr);
    sb::hb_analyse_packet(&h->st, h->w.a.high, &h->w.scr);
#endif
    sb::enc_packet_post_analysis(&h->st, &h->w.scr);
}
int hs_enc_encode(void* p, const short* pcm, unsigned char* out, int cap, short* nb) {
    HsEnc* h = (HsEnc*)p;
    enc_front(h, pcm);
#ifdef SB_EMU
    if (g_emu_nsq) {      // second lane group (SB_NSQ_GW = 16): shadows the same stream, as the kernel does for an odd batch
        HsEnc* hh[2] = {h, h};
        emu_nsq(hh);
        return sb::enc_packet_finish(&h->st, &h->w.scr, h->w.rcbuf, out, cap, nb);
    }
#endif
    return sb::enc_packet_quantise_and_code(&h->st, &h->w, out, cap, nb);
}
// two DIFFERENT streams through one emulated quantiser warp (SB_NSQ_GW = 16 build): the lane groups take their own paths
// between the full-warp sample loops.  Both encoders must have the same packet length.  ret[g] = bytes of stream g.
int hs_enc_encode_pair(void* pa, void* pb, const short* pcm_a, const short* pcm_b, unsigned char* out_a, unsigned char* out_b, int cap,
                       short* nb_a, short* nb_b, int* ret) {
#if defined(SB_EMU) && defined(SB_EMU_GW16)
    HsEnc* hh[2] = {(HsEnc*)pa, (HsEnc*)pb};
    if (hh[0]->st.frames_per_packet != hh[1]->st.frames_per_packet) return -1;
    enc_front(hh[0], pcm_a);
    enc_front(hh[1], pcm_b);
    emu_nsq(hh);
    ret[0] = sb::enc_packet_finish(&hh[0]->st, &hh[0]->w.scr, hh[0]->w.rcbuf, out_a, cap, nb_a);
    ret[1] = sb::enc_packet_finish(&hh[1]->st, &hh[1]->w.scr, hh[1]->w.rcbuf, out_b, cap, nb_b);
    return 0;
#else
    return -1;
#endif
}
// ---- the quantiser stage on its own (tests/test_gpu_nsq.py), frames and states in the layout of oracle/nsq_io.h ----
void nsq_io_sizes(int* s) { NSQ_IO_SIZES(s); }
// one packet: what the quantiser stage receives -- fr[f] (frame control and prefiltered input of every frame) and st[3]
// (the three quantiser states before it runs) -- then the rest of the packet as hs_enc_encode runs it
int hs_enc_capture(void* p, const short* pcm, NsqFrameIn* fr, NsqStateIO* st, unsigned char* out, int cap, short* nb) {
    HsEnc* h = (HsEnc*)p;
    enc_front(h, pcm);
    for (int f = 0; f < h->st.frames_per_packet; f++) sb::nsqio_frame_from(&fr[f], &h->w.scr.c[f], h->w.scr.xfw[f]);
    for (int qz = 0; qz < 3; qz++) sb::nsqio_state_from(&st[qz], &h->st.nsq[qz]);
    return sb::enc_packet_quantise_and_code(&h->st, &h->w, out, cap, nb);
}
// n cases of npk packets of nf frames each, from the states st0[n][3]: out[n][npk * nf] after every frame, st_after[n][npk][3]
// after every packet.  kernel_code = 0: the scalar model (sb_nsq.cuh, one frame at a time); 1 (emulated builds): the device
// code, nsq_packet_warp, on emulated warps with the kernel's packing -- lane group g of warp w takes case w * G + g (G = 32 /
// SB_NSQ_GW), a group without a case of its own shadows the last one -- and its scratch outputs poisoned before every packet.
int hs_nsq_run(int kernel_code, int n, int npk, int nf, const NsqStateIO* st0, const NsqFrameIn* fr, NsqFrameOut* out, NsqStateIO* st_after) {
    if (n <= 0 || npk <= 0 || (nf != 1 && nf != 2)) return -1;
    const int nfr = npk * nf;
    if (kernel_code == 0) {
        sb::EncState* st = (sb::EncState*)calloc(1, sizeof(sb::EncState));
        sb::NsqWork* W = (sb::NsqWork*)calloc(1, sizeof(sb::NsqWork));
        static sb::EncCtrl c;
        sb::i32 r[sb::FRAME];
        for (int s = 0; s < n; s++) {
            for (int qz = 0; qz < 3; qz++) sb::nsqio_state_to(&st->nsq[qz], &st0[s * 3 + qz]);
            for (int f = 0; f < nfr; f++) {
                const NsqFrameIn* x = &fr[(size_t)s * nfr + f];
                NsqFrameOut* o = &out[(size_t)s * nfr + f];
                sb::nsqio_ctrl(&c, x);
                sb::nsq_del_dec(st, &c, W, x->x, (sb::i8*)0, o->q_md[0], o->q_md[1], r);
                for (int i = 0; i < sb::FRAME; i++) o->r16[i] = (sb::i16)(r[i] >> 10);
                o->Seed = c.Seed;
                if (f % nf == nf - 1)
                    for (int qz = 0; qz < 3; qz++) sb::nsqio_state_from(&st_after[((size_t)s * npk + f / nf) * 3 + qz], &st->nsq[qz]);
            }
        }
        free(st); free(W);
        return 0;
    }
#ifdef SB_EMU
    const int G = 32 / SB_NSQ_GW;
    sb::NsqState* ns = (sb::NsqState*)calloc((size_t)n * 3, sizeof(sb::NsqState));
    sb::EncScratch* scr = (sb::EncScratch*)calloc(n, sizeof(sb::EncScratch));
    static sb::NsqSmem S[2];
    for (int s = 0; s < n; s++) for (int qz = 0; qz < 3; qz++) sb::nsqio_state_to(&ns[s * 3 + qz], &st0[s * 3 + qz]);
    for (int p = 0; p < npk; p++) {
        for (int s = 0; s < n; s++) {
            memset(scr[s].q_md, 0xA5, sizeof(scr[s].q_md)); memset(scr[s].r16, 0xA5, sizeof(scr[s].r16));
            memset(scr[s].nsq_rand, 0xA5, sizeof(scr[s].nsq_rand));
            for (int f = 0; f < nf; f++) {
                const NsqFrameIn* x = &fr[(size_t)s * nfr + p * nf + f];
                sb::nsqio_ctrl(&scr[s].c[f], x);
                for (int i = 0; i < sb::FRAME; i++) scr[s].xfw[f][i] = x->x[i];
            }
        }
        for (int w = 0; w * G < n; w++)
            sb::emu::run32m([=]() {
                const int g = sb::emu::lane / SB_NSQ_GW;
                const int s = w * G + g < n ? w * G + g : n - 1;
                sb::nsq_packet_warp(S[g], &ns[s * 3], &scr[s], nf);
            });
        for (int s = 0; s < n; s++) {
            for (int f = 0; f < nf; f++) {
                NsqFrameOut* o = &out[(size_t)s * nfr + p * nf + f];
                memcpy(o->q_md, scr[s].q_md[f], sizeof(o->q_md));
                memcpy(o->r16, scr[s].r16[f], sizeof(o->r16));
                o->Seed = scr[s].c[f].Seed;
            }
            for (int qz = 0; qz < 3; qz++) sb::nsqio_state_from(&st_after[((size_t)s * npk + p) * 3 + qz], &ns[s * 3 + qz]);
        }
    }
    free(ns); free(scr);
    return 0;
#else
    return -1;
#endif
}
// the voice-activity stage of one packet (vad_packet) from a state given as oracle/vad_io.h's words: low [nf][FRAME] ->
// out [nf][6] (speech activity, four band qualities, tilt), st [VADIO_WORDS] in / out
void hs_vad_packet(int* st, int nf, const short* low, int* out) {
    sb::VadState v;
    vadio_to(&v, st);
    int sa[2], q[2][4], tilt[2];
    sb::vad_packet(&v, low, nf, sa, q, tilt);
    for (int f = 0; f < nf; f++) {
        out[6 * f] = sa[f];
        for (int b = 0; b < 4; b++) out[6 * f + 1 + b] = q[f][b];
        out[6 * f + 5] = tilt[f];
    }
    vadio_from(st, &v);
}
// the high-band half of the entropy coding (enc_store_high_band) on one packet: cfg = frames per packet, high-band frame
// length, low-band bytes, description 1's length; lsp_idx [2], nrg0 [2][4], r16 [2][FRAME] -> out [cap], nb [2]; returns
// the packet's total size
int hs_hb_store(const int* cfg, const int* lsp_idx, const int* nrg0, const short* r16, unsigned char* out, int cap, short* nb) {
    static sb::EncCore st;
    static sb::EncScratch scr;
    memset(&st, 0, sizeof(st));
    memset(&scr, 0, sizeof(scr));
    st.frames_per_packet = cfg[0];
    st.hb_frame = cfg[1];
    memcpy(scr.hb_lsp_idx, lsp_idx, sizeof(scr.hb_lsp_idx));
    memcpy(scr.hb_nrg0, nrg0, sizeof(scr.hb_nrg0));
    memcpy(scr.r16, r16, sizeof(scr.r16));
    int total = 0;
    for (int k = 0; k < 2; k++) total = sb::enc_store_high_band(&st, &scr, k, cfg[2], cfg[3], out, cap, nb);
    return total;
}
// rate (b/s), DTX, expected loss (%) from the next packet on: the body of the device's control kernel on the host model's
// state; -1 or any other out-of-range value leaves a setting alone
void hs_enc_set_control(void* p, int rate, int dtx, int loss) { sb::enc_set_control(&((HsEnc*)p)->st, rate, dtx, loss); }
// the activity kernel's flags of the last packet this encoder coded
int hs_enc_flags(void* p) {
    HsEnc* h = (HsEnc*)p;
    return sb::enc_activity_flags(&h->w.scr, h->st.frames_per_packet);
}
void hs_enc_destroy(void* p) { free(p); }
int hs_is_emu() {
#ifdef SB_EMU
    return 1;
#else
    return 0;
#endif
}
// the RFC 6464 level of a row whose sum of squares is E, and the activity kernel's level of one row of n samples
int hs_level(long long E, int n) { return sb::rfc6464_level(E, n); }
int hs_row_level(const short* pcm, int n) {
    long long e = 0;
    for (int i = 0; i < n; i++) e += (long long)pcm[i] * pcm[i];
    return sb::rfc6464_level(e, n);
}
}

// one decoder stream; samplerate (first, so that hs_dec_decode can read it) picks the core rate: 16000 -> KHZ 8, 32000 -> 16
template <int KHZ> struct HsDec { int samplerate; sb::DecStateT<KHZ> st; sb::DecPacketWorkT<KHZ> w; sb::DecStale stale; };
template <int KHZ> static void* dec_create(int mdi, int framesize_ms, int joint_hb, int arith, int samplerate, int core_only) {
    HsDec<KHZ>* h = (HsDec<KHZ>*)calloc(1, sizeof(HsDec<KHZ>));
    h->samplerate = samplerate;
    sb::dec_state_init(&h->st, mdi, framesize_ms, joint_hb, arith, core_only);
    return h;
}
template <int KHZ> static int dec_decode(void* p, short* pcm, const unsigned char* bits, int cap, const short* nb, int lostflag, unsigned char* flags) {
    HsDec<KHZ>* h = (HsDec<KHZ>*)p;
    const int r = sb::dec_packet(&h->st, &h->w, pcm, bits, cap, nb, lostflag, &h->stale);
    if (flags) *flags = r < 0 ? 0 : h->w.act;      // what the decode kernel stores for the activity kernel
    return r;
}

extern "C" {
// arith: sb::DEC_FLP or sb::DEC_FIX; samplerate 16000 or 32000; out_samplerate the stream's own rate, or 16000 for a 32 kHz
// stream decoded to its 16 kHz core (the core-output decode kernel's dec_packet<16, true>).  NULL for any other pair, as
// solo_b200_dec_batch_create_out refuses them.
void* hs_dec_create(int mdi, int framesize_ms, int joint_hb, int arith, int samplerate, int out_samplerate) {
    if (samplerate == 16000 && out_samplerate == 16000) return dec_create<8>(mdi, framesize_ms, joint_hb, arith, samplerate, 0);
    if (samplerate == 32000 && (out_samplerate == 32000 || out_samplerate == 16000))
        return dec_create<16>(mdi, framesize_ms, joint_hb, arith, samplerate, out_samplerate == 16000);
    return nullptr;
}
// same calling convention as AGR_Sate_Decoder_Decode (payload pre-trimmed by the caller); nb is not modified.  flags (may be
// NULL): the packet's activity flags, 0 for a rejected packet
int hs_dec_decode(void* p, short* pcm, const unsigned char* bits, int cap, const short* nb, int lostflag, unsigned char* flags) {
    return *(const int*)p == 32000 ? dec_decode<16>(p, pcm, bits, cap, nb, lostflag, flags) : dec_decode<8>(p, pcm, bits, cap, nb, lostflag, flags);
}
void hs_dec_destroy(void* p) { free(p); }
}
