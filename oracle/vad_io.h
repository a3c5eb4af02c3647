/* The voice-activity detector's state as 28 plain int32, in the order oracle/enc_ref.c records the reference's
 * SKP_Silk_VAD_state: AnaState[2], AnaState1[2], AnaState2[2], XnrgSubfr[4], NrgRatioSmth_Q8[4], NL[4], inv_NL[4],
 * NoiseLevelBias[4], counter, HPstate.  The host model (tests/hostsim) and the GPU harness (tests/gpu_ops) convert the
 * product's VadState (sb_state.cuh) with these, so tests can start either from any state the reference passed through. */
#ifndef SB_VAD_IO_H
#define SB_VAD_IO_H
#include <stdint.h>
#include <string.h>

#define VADIO_WORDS 28

static inline void vadio_to(sb::VadState* v, const int32_t* d) {
    int32_t* w[] = {v->AnaState, v->AnaState1, v->AnaState2, v->XnrgSubfr, v->NrgRatioSmth_Q8, v->NL, v->inv_NL, v->NoiseLevelBias};
    const int len[] = {2, 2, 2, 4, 4, 4, 4, 4};
    memset(v, 0, sizeof(*v));
    for (int a = 0; a < 8; a++) for (int i = 0; i < len[a]; i++) w[a][i] = *d++;
    v->counter = d[0];
    v->HPstate = (int16_t)d[1];
}

static inline void vadio_from(int32_t* d, const sb::VadState* v) {
    const int32_t* w[] = {v->AnaState, v->AnaState1, v->AnaState2, v->XnrgSubfr, v->NrgRatioSmth_Q8, v->NL, v->inv_NL, v->NoiseLevelBias};
    const int len[] = {2, 2, 2, 4, 4, 4, 4, 4};
    for (int a = 0; a < 8; a++) for (int i = 0; i < len[a]; i++) *d++ = w[a][i];
    d[0] = v->counter;
    d[1] = v->HPstate;
}

#endif
