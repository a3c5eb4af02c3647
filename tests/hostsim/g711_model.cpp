// Host build of the G.711 gateway's per-stream code (solo_b200/csrc/sb_g711.cuh compiled by g++), in its kernels' order.
// TEST INFRASTRUCTURE ONLY; built into tests/_hostsim/libsb_g711.so by g711_sim.py, never linked into libsolo_b200.so.
// The state array has the device layout of G711State.
#include <string.h>

#include "../../solo_b200/csrc/sb_g711.cuh"

using namespace sb;

extern "C" {
int g711_model_state_bytes() { return (int)sizeof(G711State); }
// sb_g711_reset_kernel for the listed streams (streams = NULL: all n), law entry -1 or law = NULL: law0
void g711_model_reset(G711State* st, const i32* streams, int n, const i32* law, int law0) {
    for (int i = 0; i < n; i++) g711_state_init(&st[streams ? streams[i] : i], law && law[i] != -1 ? law[i] : law0);
}
// one uplink of n streams (lost = NULL: nothing lost); sa_Q8 [n][nf] receives each frame's speech activity
void g711_model_uplink(G711State* st, int n, int nf, const u8* codes, const i32* lost, i16* pcm, u8* level, u8* flags, i32* sa_Q8) {
    const int N2 = nf * FRAME;
    for (int s = 0; s < n; s++) {
        i16* row = pcm + (size_t)s * 2 * N2;
        flags[s] = (u8)g711_uplink(&st[s], codes + (size_t)s * N2, lost ? lost[s] : 0, nf, row, sa_Q8 + (size_t)s * nf);
        i64 e = 0;
        for (int i = 0; i < 2 * N2; i++) e += (i32)row[i] * row[i];
        level[s] = (u8)rfc6464_level(e, 2 * N2);
    }
}
// one downlink of n rows of 2 * nf * FRAME samples; low [n][nf * FRAME] receives the low band before companding
void g711_model_downlink(G711State* st, int n, int nf, const i16* pcm, i16* low, u8* codes) {
    const int N2 = nf * FRAME;
    for (int s = 0; s < n; s++) g711_downlink(&st[s], pcm + (size_t)s * 2 * N2, 2 * N2, low + (size_t)s * N2, codes + (size_t)s * N2);
}
// the companding alone over a whole array
void g711_model_compress(int law, const i16* x, int n, u8* c) { for (int i = 0; i < n; i++) c[i] = g711_compress(law, x[i]); }
void g711_model_expand(int law, const u8* c, int n, i16* x) { for (int i = 0; i < n; i++) x[i] = g711_expand(law, c[i]); }
}
