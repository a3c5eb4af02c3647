/* A tap on the reference decoder's low band, for the core-output decoder's parity tests (test infrastructure only).
 *
 * lowband.mk links each reference library, unmodified, with -Wl,--wrap=AGR_Sate_qmf_synth, so that the decoder's call of
 * its synthesis filter bank (AGR_BWE_decode_frame_FLP.c:220, AGR_BWE_decode_frame_FIX.c:194) lands here first.  The
 * wrapper records the first argument, the low band of the packet: N / 2 samples for N = JC1_FrameSize output samples.
 * The float build holds it as floats converted from int16 (OutLow[i] = (float)lowout[i]), so the conversion back is exact;
 * the fixed-point build passes int16 (OutLow).  Then the real filter bank runs, so the library's PCM is unchanged.
 * Build with -DLOWBAND_FLOAT for the float tree. */
#include <stdint.h>
#include <string.h>

#ifdef LOWBAND_FLOAT
typedef float band_t;
#else
typedef int16_t band_t;
#endif

#define LOWBAND_MAX 640     /* 40 ms of the 16 kHz core of a 32 kHz stream */

static int16_t g_low[LOWBAND_MAX];
static int g_n;

void __real_AGR_Sate_qmf_synth(const band_t *x1, const band_t *x2, const band_t *a, band_t *y, int32_t N, int32_t M, band_t *mem1,
                               band_t *mem2, int8_t *stack);

void __wrap_AGR_Sate_qmf_synth(const band_t *x1, const band_t *x2, const band_t *a, band_t *y, int32_t N, int32_t M, band_t *mem1,
                               band_t *mem2, int8_t *stack) {
    int n = N / 2;
    if (n > LOWBAND_MAX) n = LOWBAND_MAX;
    for (int i = 0; i < n; i++) g_low[i] = (int16_t)x1[i];
    g_n = n;
    __real_AGR_Sate_qmf_synth(x1, x2, a, y, N, M, mem1, mem2, stack);
}

/* The low band of the last synthesis since the previous call into out[cap]; returns its length, 0 when the decoder has not
   run its filter bank since then (a rejected packet returns before it). */
int lowband_take(int16_t *out, int cap) {
    const int n = g_n < cap ? g_n : cap;
    memcpy(out, g_low, sizeof(int16_t) * (size_t)n);
    g_n = 0;
    return n;
}
