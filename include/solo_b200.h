/*
 * solo_b200 -- batched extension of the SOLO SDK ABI (plain C, no CUDA or torch types in the signatures).
 *
 * One batch object owns N independent codec streams whose state stays resident in GPU memory between
 * calls; one call advances every stream by one 40 ms packet.  Semantics per stream are exactly those of
 * AGR_Sate_Encoder_Encode / AGR_Sate_Decoder_Decode (AGR_JC1_SDK_API.h; reference
 * /root/reference/JC1_SDK_SRC_ARM/src/libBWE/AGR_BWE_SDK_API.c:129-152, JC1_SDK_SRC_FLP/.../AGR_BWE_SDK_API.c:249-279).
 *
 * Two flavours of every call:
 *   *_host    : buffers are host memory (pinned or pageable); host<->device copies happen inside the call
 *   *_device  : buffers are device pointers; the call only enqueues kernels on `cuda_stream`
 *               (a cudaStream_t passed as void*; NULL = legacy default stream) and does not synchronise.
 *
 * Packet size: ctrl->framesize_ms = 40 (two 20 ms codec frames per packet, 8 high-band bytes, 640 samples per row) or 20
 * (one frame, 4 high-band bytes, 320 samples per row) -- the two packet sizes of the reference (AGR_BWE_SDK_API.c:78-110);
 * with joint_enable = 1, joint_mode = 1 (40 ms packets only) the high band is coded as one 40 ms frame (4 bytes, :63-66).
 *
 * Sample rate: ctrl->samplerate = 16000 (8 kHz SILK core, 4-8 kHz parametric high band) or, for the DECODER only, 32000
 * (the reference's 32 kHz API, AGR_BWE_SDK_API.c:86-94,196-200: 16 kHz SILK core with order-16 LPC, 8-16 kHz high band).
 *   - 32 kHz decoding covers every packet configuration above, in both decoder arithmetics (the fixed-point one with 40 ms
 *     packets and joint mode 1, as at 16 kHz).  PCM rows are 32 * framesize_ms samples (1280 or 640); the drop-in
 *     AGR_Sate_Decoder_Decode reports *nSamplesOut = 1280 / 640.
 *   - Core rate: a 32 kHz stream decodes when its SILK core is 16 kHz.  The reference encoder chooses its core from the core
 *     bitrate (user rate - 1600, or - 800 with joint mode 1; SKP_Silk_control_audio_bandwidth.c:38-114): see INTEGRATION.md
 *     for the user rates that keep the 16 kHz core.  A frame that codes another core rate (8 or 12 kHz, which the reference
 *     would resample to 16 kHz) is that stream's error, ret = -12, exactly like a corrupted packet; the other streams of the
 *     batch are not affected.
 *   - A decoder batch of 32 kHz streams may instead output their 16 kHz core (solo_b200_dec_batch_create_out): rows of
 *     16 * framesize_ms samples, which mix with 16 kHz streams' rows.
 *   - There is no 32 kHz ENCODER yet: solo_b200_enc_batch_create and AGR_Sate_Encoder_Init return NULL for samplerate 32000,
 *     with solo_b200_last_error() saying so.
 *
 * Layouts (row = stream):  pcm  int16 [N][samplerate / 1000 * framesize_ms]   bits uint8 [N][cap]
 *                          nbytes int16 [N][2]        ({total, len(MD2)+8} as the single-stream API)
 *                          lostflag int32 [N]         (1 lost, 2 MD1 only, 3 MD2+HB only, 4 both)
 * For decode, row i of `bits` holds the payload exactly as the caller would hand it to
 * AGR_Sate_Decoder_Decode (already trimmed for lostflag 2 / 3) and nbytes[i] the matching {n0, n1};
 * nbytes is NOT modified (the single-stream call rewrites its nBytes[], SURVEY.md App. A Q15).
 * ret[i] receives the per-stream return code of the reference call (0 ok, negative SILK error codes).
 *
 * All functions return 0 on success, a negative value on error (-1 bad argument, -2 CUDA failure;
 * solo_b200_last_error() gives a text).  A missing GPU is an error: there is no CPU fallback.
 */
#ifndef SOLO_B200_H
#define SOLO_B200_H

#include <stdint.h>
#include "AGR_JC1_SDK_API.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct solo_b200_enc_batch solo_b200_enc_batch;
typedef struct solo_b200_dec_batch solo_b200_dec_batch;

/* device = CUDA device ordinal; ctrl is applied to every stream (same checks as AGR_Sate_Encoder_Init). */
solo_b200_enc_batch *solo_b200_enc_batch_create(int n_streams, const USER_Ctrl_enc *ctrl, int device);
int solo_b200_enc_batch_encode_host(solo_b200_enc_batch *b, const int16_t *pcm, uint8_t *bits, int cap, int16_t *nbytes);
int solo_b200_enc_batch_encode_device(solo_b200_enc_batch *b, const int16_t *d_pcm, uint8_t *d_bits, int cap,
                                      int16_t *d_nbytes, void *cuda_stream);
void solo_b200_enc_batch_destroy(solo_b200_enc_batch *b);

/* Per-stream encoder settings that may change between packets, as the reference's SILK core re-reads them from the
   handle at the start of every packet (SKP_Silk_enc_API.c:161-191):
     rate_bps  : target rate as USER_Ctrl_enc.targetRate_bps (>= 1; the core gets it less 1600 b/s, or less 800 b/s with
                 joint mode 1, clamped to [5000, 100000])
     dtx       : 0 or 1, as USER_Ctrl_enc.dtx_enable
     loss_perc : expected packet loss in percent, 0-100 (Init starts at 0).  The encoder then trades long-term prediction
                 gain for robustness (SKP_Silk_LTP_scale_ctrl_FIX.c:39-81); the decoder needs no change.
   Arrays are int32 [N].  A NULL array leaves that setting unchanged for every stream, an entry of -1 for that stream.  New
   settings apply from the next packet; both frames of a 40 ms packet use the same settings.
     set_control_host   : host arrays.  Returns -1 and applies nothing if any entry is out of range; otherwise returns once
                          the settings are in place, after every packet wave already enqueued for the batch.
     set_control_device : device arrays; only enqueues a kernel on `cuda_stream`, in order with the encode_device calls
                          on that stream.  The arrays are not checked on the host: an out-of-range entry leaves that
                          stream's setting unchanged, like -1.
   Create followed by set_control before the first packet is the same as creating the stream with those settings. */
int solo_b200_enc_batch_set_control_host(solo_b200_enc_batch *b, const int32_t *rate_bps, const int32_t *dtx,
                                         const int32_t *loss_perc);
int solo_b200_enc_batch_set_control_device(solo_b200_enc_batch *b, const int32_t *d_rate_bps, const int32_t *d_dtx,
                                           const int32_t *d_loss_perc, void *cuda_stream);
/* The same for one AGR_Sate_Encoder_Init handle (scalars, -1 = unchanged): 0, or -1 for a NULL or foreign handle or an
   out-of-range value (nothing applied). */
int solo_b200_encoder_set_control(void *SATEEnc_State, int32_t rate_bps, int32_t dtx, int32_t loss_perc);

/* Decoder arithmetic of a batch's streams.  The reference ships two builds whose decoded PCM differs (by up to ~1 800 LSB on
   speech); the low band is the same integer decoder in both, the high-band synthesis and the synthesis filter bank are not.
     SOLO_B200_DEC_FLP : PCM of the float build (JC1_SDK_SRC_FLP), what solo_b200_dec_batch_create gives.
     SOLO_B200_DEC_FIX : PCM of the fixed-point build (JC1_SDK_SRC_ARM), bit for bit; 40 ms packets and joint mode 1 only.
                         With 20 ms packets the fixed-point build decodes every payload twice (it always decodes two SILK
                         frames per call), which is its defect, not a mode worth reproducing: create returns NULL.
   The arithmetic is part of each stream's state, so exported blobs carry it. */
#define SOLO_B200_DEC_FLP 0
#define SOLO_B200_DEC_FIX 1
solo_b200_dec_batch *solo_b200_dec_batch_create(int n_streams, const USER_Ctrl_dec *ctrl, int device);
/* The same with the arithmetic: NULL, with solo_b200_last_error() set, for an unknown value or SOLO_B200_DEC_FIX with 20 ms
   packets. */
solo_b200_dec_batch *solo_b200_dec_batch_create_arith(int n_streams, const USER_Ctrl_dec *ctrl, int device, int arith);
/* The same with the output rate of the batch's PCM rows.  out_samplerate = ctrl->samplerate gives the batch of
   solo_b200_dec_batch_create_arith.  out_samplerate = 16000 with ctrl->samplerate = 32000 is core output: every packet of a
   32 kHz stream is decoded to its 16 kHz SILK core (0-8 kHz) only, rows of 16 * framesize_ms samples (640 or 320), the
   layout of a 16 kHz batch, so that a 32 kHz uplink is an ordinary row of a 16 kHz room (mixer, downlink encoder).
     - The row is exactly the int16 low band the reference hands to its synthesis filter bank (AGR_Sate_qmf_synth) for the
       same packets: band-limited to what a 16 kHz stream carries, with no resampling.  The 8-16 kHz band is not decoded
       and the synthesis filter bank does not run: a wave is one launch instead of two.
     - Return codes (including -12 for frames coded at an 8 or 12 kHz core), concealment, DTX / comfort noise, lostflag 2 / 3
       and the activity flags are those of a full 32 kHz batch fed the same packets; the activity level is that of the
       640- or 320-sample row.
     - State blobs record the mode: the sized import refuses a blob of the other mode (a core-output stream's high-band and
       filter-bank memories have not followed its packets, so it cannot continue as a full-band stream, nor the reverse).
   Any other out_samplerate returns NULL with solo_b200_last_error() set. */
solo_b200_dec_batch *solo_b200_dec_batch_create_out(int n_streams, const USER_Ctrl_dec *ctrl, int device, int arith,
                                                    int out_samplerate);
int solo_b200_dec_batch_decode_host(solo_b200_dec_batch *b, int16_t *pcm, const uint8_t *bits, int cap,
                                    const int16_t *nbytes, const int32_t *lostflag, int32_t *ret);
/* d_pcm's alignment: a full-band batch (16 kHz, or 32 kHz at its own rate) writes its rows with 8-byte stores, so d_pcm
   must be 8-byte aligned; a core-output batch accepts any 2-byte alignment (16-byte aligned rows are stored 16 bytes at a
   time, others sample by sample).  Otherwise -1 with solo_b200_last_error() naming the alignment, before anything is
   enqueued. */
int solo_b200_dec_batch_decode_device(solo_b200_dec_batch *b, int16_t *d_pcm, const uint8_t *d_bits, int cap,
                                      const int16_t *d_nbytes, const int32_t *d_lostflag, int32_t *d_ret, void *cuda_stream);
void solo_b200_dec_batch_destroy(solo_b200_dec_batch *b);

/* Stream state hand-over (checkpoint, migration between batches / GPUs, streams joining and leaving a batch): the complete
   codec state of stream `idx` as an opaque blob of solo_b200_{enc,dec}_state_bytes() bytes.  Synchronous; a blob is only
   meaningful to the same build of the library. */
int solo_b200_enc_batch_export_state(solo_b200_enc_batch *b, int idx, void *blob);
int solo_b200_enc_batch_import_state(solo_b200_enc_batch *b, int idx, const void *blob);
int solo_b200_dec_batch_export_state(solo_b200_dec_batch *b, int idx, void *blob);
int solo_b200_dec_batch_import_state(solo_b200_dec_batch *b, int idx, const void *blob);
/* The decoder forms with the blob's size: -1 (nothing copied, solo_b200_last_error() set) when blob_bytes is not the batch's
   solo_b200_dec_state_bytes_rate(samplerate), i.e. for a blob of a stream of the other sample rate, and on import when a
   32 kHz blob is of the other output mode (core output or full band, see solo_b200_dec_batch_create_out).  The unsized
   forms above trust the caller's blob to be of the batch's rate and mode. */
int solo_b200_dec_batch_export_state_sized(solo_b200_dec_batch *b, int idx, void *blob, int blob_bytes);
int solo_b200_dec_batch_import_state_sized(solo_b200_dec_batch *b, int idx, const void *blob, int blob_bytes);

/* Stream membership on the device, for participants joining, leaving and moving between batches or GPUs without stopping
   the GPU.  The calls follow the queues' reset (solo_b200_rx_reset / solo_b200_tx_reset):
     - `streams` is a host array of n stream indices; n = 0 does nothing;
     - the list is checked first: -1 with nothing done (solo_b200_last_error() set) for a stream outside [0, N), a stream
       listed twice, and for the bad settings and d_blobs described below;
     - the work is one kernel (two for a 32 kHz decoder import) ordered on `cuda_stream`, after the packet waves already
       enqueued there; the call then synchronises that CUDA stream only, never the device, so other tenants' work and the
       batch's other streams keep running.
   reset: re-initialises the listed streams exactly as create would.  From the next wave a reset stream produces exactly
     what a stream of a newly created batch with the same ctrl and settings produces on the same input: encoder payload
     bytes and nbytes, decoder PCM, return codes and activity flags.  Settings are host arrays of n entries, one per listed
     stream; an entry of -1, or a NULL array, takes the batch's create value.
       encoder: rate_bps, dtx, loss_perc with the ranges and checks of set_control_host (-1 and nothing done for an entry
                out of range).  A reset stream is create followed by set_control with those settings.
       decoder: arith SOLO_B200_DEC_FLP or SOLO_B200_DEC_FIX (FIX refused with 20 ms packets, as create refuses it).  A
                core-output batch resets its streams into core output.  Packet size, joint mode and useMDIndex are the
                batch's.
   export_states / import_states: copy the listed streams' states to / from d_blobs [n][state_bytes] in device memory --
     this GPU's HBM, a peer GPU's HBM after solo_b200_enable_peer_access, or mapped pinned host memory.  d_blobs must be
     8-byte aligned (-1 before anything is enqueued otherwise).  state_bytes is solo_b200_enc_state_bytes() or
     solo_b200_dec_state_bytes_rate(samplerate).  Bytes [i * state_bytes, (i + 1) * state_bytes) are exactly the blob of
     export_state(streams[i]), and import_state accepts them; import_states accepts export_state's blobs likewise.
     A 32 kHz decoder import refuses blobs of the other output mode, as import_state_sized does, all or nothing: a check
     kernel runs first, and if any blob is of the other mode nothing is imported and the call returns -1 after its
     synchronise.
   Like the per-stream hand-over, blobs leave out the payload copies a decoder stream reads only while it continues a
   corrupted packet (see DecStale in solo_b200/csrc/sb_dec.cuh): a reset stream never reads them; an imported stream reads
   the destination slot's copy, as after import_state.
   Streams that left are still coded by every wave; reset them when the slot is reused.
   Launches: a reset or an export is one kernel; an import two for a 32 kHz decoder batch, one otherwise. */
int solo_b200_enc_batch_reset(solo_b200_enc_batch *b, const int32_t *streams, int n, const int32_t *rate_bps, const int32_t *dtx,
                              const int32_t *loss_perc, void *cuda_stream);
int solo_b200_dec_batch_reset(solo_b200_dec_batch *b, const int32_t *streams, int n, const int32_t *arith, void *cuda_stream);
int solo_b200_enc_batch_export_states(solo_b200_enc_batch *b, const int32_t *streams, int n, void *d_blobs, void *cuda_stream);
int solo_b200_enc_batch_import_states(solo_b200_enc_batch *b, const int32_t *streams, int n, const void *d_blobs, void *cuda_stream);
int solo_b200_dec_batch_export_states(solo_b200_dec_batch *b, const int32_t *streams, int n, void *d_blobs, void *cuda_stream);
int solo_b200_dec_batch_import_states(solo_b200_dec_batch *b, const int32_t *streams, int n, const void *d_blobs, void *cuda_stream);

/* Packet framing around one payload row [MD1 | MD2 | HB] (reference drivers enc_main.c:212-234, dec_main.c:196-307, README
   "Bitstream sending" / "Bitstream screening and synthesis at receiver").  Host functions, no GPU involved.
     split : the two network packets of a row -- description 1 = MD1, description 2 = MD2 + 8 high-band bytes (pointers into
             `bits`); both empty for a DTX row (nbytes[0] == 0)
     merge : from whichever packets arrived (pass NULL / 0 for a missing one) build the decoder's row, nbytes[2] and lostflag
             (4 both, 2 only description 1, 3 only description 2, 1 none)
     bitfile_pack / unpack : one record of the reference's .bit file (int16 total, int16 len(MD2)+8, payload); return the
             record size, or -1
     apply_loss_device : the receiver-side trimming for a whole batch on the GPU (rows of `cap` bytes): lostflag 2 keeps MD1,
             3 moves MD2 + HB to the front, 4 / 1 pass through -- feeds solo_b200_dec_batch_decode_device directly */
int solo_b200_split_packet(const uint8_t *bits, const int16_t *nbytes, const uint8_t **p1, int *n1, const uint8_t **p2, int *n2);
int solo_b200_merge_packets(const uint8_t *p1, int n1, const uint8_t *p2, int n2, uint8_t *bits, int cap, int16_t *nbytes,
                            int32_t *lostflag);
int solo_b200_bitfile_pack(const uint8_t *bits, const int16_t *nbytes, uint8_t *out, int out_cap);
int solo_b200_bitfile_unpack(const uint8_t *in, int in_len, const uint8_t **payload, int16_t *nbytes);
int solo_b200_apply_loss_device(const uint8_t *d_bits_in, const int16_t *d_nbytes_in, const int32_t *d_lostflag, uint8_t *d_bits_out,
                                int16_t *d_nbytes_out, int cap, int n, void *cuda_stream);

/* Activity reports: the audio level and voice activity of every stream's last packet, for the RFC 6464 header extension
   (client-to-mixer audio level), dominant-speaker detection and receive statistics.  Per stream, one byte each:
     level : the RFC 6464 level (0-127, -dBov) of the packet's PCM row -- the encoder's input row, the decoder's output row.
             With E = sum of x^2 over the row (int64) and n = the row length (320, 640 or 1280 samples), level = the number
             of k in 0..126 with E < T_n[k], T_n[k] = ceil(n * 2^30 * 10^(-(k + 0.5) / 10)).  That is
             clamp(round(10 * log10(n * 32768^2 / E)), 0, 127), 127 for digital silence, in exact integers: the tables
             (solo_b200/csrc/sb_level_tables.inc) are generated by tools/gen_level_tables.py in exact decimal arithmetic.
     flags : bit f (f = 0, 1) = SILK VAD flag of frame f of the packet.  Encoder: the flag coded into that frame (0 for both
             frames of a DTX-dropped packet).  Decoder: the flag decoded from that frame, 0 when it was concealed.
             bit 2 + f (decoder only) = frame f was concealed (lost packet, including loss before the first good frame).
             With 20 ms packets bits 1 and 3 are 0.  RFC 6464's V bit is (flags & 3) != 0.
   A decoder stream whose packet was rejected (ret < 0) reports level 127 and flags 0.
     *_activity_host   : after a *_host packet wave, from the PCM that wave staged on the device; fills the host arrays
                         level[N] and flags[N] and returns when they are filled.
     *_activity_device : after a *_device packet wave; d_pcm = the device PCM rows passed to that wave (the encoder's input,
                         the decoder's output).  Only enqueues one kernel on `cuda_stream` that writes d_level[N], d_flags[N].
   The report is of the last wave: call it before the batch's next wave.  Returns -1 (solo_b200_last_error() set) for a
   batch that has not run a wave yet, and for *_host after a *_device wave or the reverse.  The packet calls launch exactly
   the kernels they did without these calls; each activity call adds one launch. */
int solo_b200_enc_batch_activity_host(solo_b200_enc_batch *b, uint8_t *level, uint8_t *flags);
int solo_b200_enc_batch_activity_device(solo_b200_enc_batch *b, const int16_t *d_pcm, uint8_t *d_level, uint8_t *d_flags,
                                        void *cuda_stream);
int solo_b200_dec_batch_activity_host(solo_b200_dec_batch *b, uint8_t *level, uint8_t *flags);
int solo_b200_dec_batch_activity_device(solo_b200_dec_batch *b, const int16_t *d_pcm, uint8_t *d_level, uint8_t *d_flags,
                                        void *cuda_stream);
/* The same for the last packet of one AGR_Sate_*_Init handle (one byte each): 0, or -1 for a NULL or foreign handle or a
   handle that has not coded a packet yet. */
int solo_b200_encoder_last_activity(void *SATEEnc_State, uint8_t *level, uint8_t *flags);
int solo_b200_decoder_last_activity(void *SATEDec_State, uint8_t *level, uint8_t *flags);

/* Conference mixer (MCU): per room, the mix-minus of its loudest talkers, from the decoder's PCM rows to the downlink
   encoder's input rows, for top-N mixing with an RFC 6465 (mixer-to-client audio level) header.
   Inputs:
     in          : int16 [n][spp], the decoder's output rows, spp = 320, 640 or 1280.
     level, flags: uint8 [n] each, in the activity report's format: exactly what solo_b200_dec_batch_activity_{host,device}
                   writes.
     rooms, CSR  : room_start int32 [R+1] with room_start[0] = 0, non-decreasing, room_start[R] = M; members int32 [M],
                   stream indices in any order.  Room r is members[room_start[r] .. room_start[r+1]).
     k           : 1 to 8.
   Selection:
     A member j of a room is eligible when (flags[j] & 3) != 0, i.e. RFC 6464's V bit; concealed and rejected packets
     report flags 0, so they are never mixed.  The room's talkers are its up-to-k eligible members with the smallest
     (level[j], j): lower level is louder, ties go to the lower index.  They are written to talkers int32 [R][k] in that
     order, padded with -1: the CSRC list (and, with level[], the levels) of an RFC 6465 header.
   Mixing:
     For every member i of room r and every sample t:
       out[i][t] = clamp(sum over talkers j of r with j != i of in[j][t], -32768, 32767).
     A listener hears all the talkers, a talker hears the others, a room without talkers gives zeros.  The sum is in int32;
     with k <= 8 it cannot overflow, so the result does not depend on the order of summation.  No floating point is used.
     Rows of streams that are in no room are not written.
   Policy stays with the caller, in the two byte arrays: mute a participant with flags 0, pin a moderator with level 0,
   apply hysteresis by rewriting the bytes before the call.
     mix_host   : host arrays.  Checks everything first and returns -1, writing nothing (solo_b200_last_error() set), for a
                  bad spp, n or k, offsets that do not start at 0 or decrease, a member outside [0, n), or a stream listed
                  twice (in one room or in two).  Runs on the calling thread's current CUDA device and returns when out[]
                  and talkers[] are filled.
     mix_device : device arrays; only enqueues work on `cuda_stream` (at most two kernel launches).  It checks the scalars
                  (-1 for a bad spp, n or k, for d_in / d_out not 16-byte aligned, and for d_in and d_out overlapping:
                  they must not), not the arrays' contents, and never reads or writes out of bounds whatever they hold:
                  room bounds are clamped to [0, room_start[R]], a member outside [0, n) is skipped (neither a talker nor
                  written), and a stream listed twice gives unspecified rows but no fault.
   n_rooms = 0 is a call that does nothing. */
int solo_b200_mix_host(const int16_t *in, int16_t *out, int spp, int n, const uint8_t *level, const uint8_t *flags,
                       const int32_t *room_start, const int32_t *members, int n_rooms, int k, int32_t *talkers);
int solo_b200_mix_device(const int16_t *d_in, int16_t *d_out, int spp, int n, const uint8_t *d_level,
                         const uint8_t *d_flags, const int32_t *d_room_start, const int32_t *d_members, int n_rooms,
                         int k, int32_t *d_talkers, void *cuda_stream);
/* Downlink contributor lists: for every member i of room r (rooms, n and k as for solo_b200_mix_*, talkers int32 [R][k]
   as the mix writes them, level uint8 [n] as the activity report writes it):
     csrc int32 [n][k]      : the entries j of talkers[r] with 0 <= j < n and j != i, in the mixer's order (loudest first),
                              padded with -1: the CSRC list of i's downlink packet (as stream indices);
     csrc_level uint8 [n][k]: level[j] & 0x7f beside each entry, 127 in the padding: its RFC 6465 levels.
   Rows of streams in no room are all -1 and 127.
     mix_contributors_host   : host arrays, the checks of mix_host (-1, nothing written, for a bad n or k, bad offsets, a
                               member outside [0, n) or a stream listed twice); returns when the rows are written.
     mix_contributors_device : device arrays; only enqueues two memsets and, for n_rooms > 0, one kernel launch (a thread
                               per member) on `cuda_stream`.  It checks the scalars, and clamps as mix_device does: a member
                               outside [0, n) is skipped, a stream listed twice gives an unspecified row but no fault. */
int solo_b200_mix_contributors_host(const int32_t *room_start, const int32_t *members, int n_rooms, int k,
                                    const int32_t *talkers, const uint8_t *level, int n, int32_t *csrc, uint8_t *csrc_level);
int solo_b200_mix_contributors_device(const int32_t *d_room_start, const int32_t *d_members, int n_rooms, int k,
                                      const int32_t *d_talkers, const uint8_t *d_level, int n, int32_t *d_csrc,
                                      uint8_t *d_csrc_level, void *cuda_stream);

/* Receive queue: per stream, holds the two descriptions of each packet (solo_b200_split_packet) as they arrive early, out
   of order or twice, pairs them and hands the decoder one row per tick, for N streams on the device.  It is independent
   of the codec batches: a pull writes rows for any decoder batch with the same N and cap.
   Created with depth D (a power of two, 2 to 32) and desc_cap (the largest description in bytes, 16 to 1024, a multiple
   of 16).  Per stream it keeps:
     last     : the last played packet index (uint32), 0xFFFFFFFF at create, so packet 0 plays first;
     D slots  : slot j holds at most one packet index t with t = j (mod D), and for it description 1 and / or 2;
     counters : 8 uint32, in this order: stored, duplicate, late, dropped, malformed, played_both, played_one,
                played_none.
   Packet index: the caller derives it from the RTP timestamp (timestamp / samples per packet); it wraps at 2^32.  Index p
   is CURRENT for a stream when (p - last) mod 2^32 lies in [1, 2^31), otherwise LATE; among current indices the newer one
   has the larger distance (p - last) mod 2^32.
   insert: arrival a is (stream[a], index[a], desc[a], len[a] bytes at payload + off[a]).
     - An arrival whose stream is outside [0, N) only counts in the queue-wide bad_stream counter.
     - It is malformed when desc is not 1 or 2, len is outside [1, desc_cap], or its bytes are not inside
       payload[0, payload_bytes).
     - Per slot, from its held packet and the call's valid, current arrivals for it: the slot keeps the NEWEST of those
       indices (a held index that is no longer current does not compete).  If that is not the held index, the held
       descriptions are discarded.  For each description of the kept index a held one stays, otherwise the FIRST arrival
       in array order is stored.
     - Every arrival counts exactly once, as stored; duplicate (its (index, desc) was already held or stored); late;
       dropped (its slot keeps a newer index); or malformed.  Held descriptions that are discarded count as dropped too.
     The result does not depend on thread scheduling: the same calls give the same state and counters.
   pull: for each stream s, with t = play[s] (play = NULL: last + 1), writes row s of bits [N][cap], nbytes[s][2] and
     lostflag[s] exactly as solo_b200_merge_packets does for the descriptions of t its slot holds (4 both, 2 only
     description 1, 3 only description 2, 1 neither: 16 zero bytes and {16, 8}).  Row bytes after nbytes[0] are not
     written.  cap must be at least 2 * desc_cap (else -1), so a merge always fits.  Then last = t, and the slot is
     emptied when it held t or an index that is no longer current (counted as dropped); one of played_both, played_one
     or played_none is incremented.
   reset: for a participant joining or rejoining a stream: empties the listed streams' slots, zeroes their counters and
     sets last = start - 1.  Host arrays; -1 (nothing done) for a stream outside [0, N) or listed twice.
   stats: counters uint32 [N][8] and the bad_stream count (either may be NULL).
   Entry points:
     *_host   : host arrays; run on the queue's own CUDA stream and return when done.
     *_device : device arrays; only enqueue work on `cuda_stream`.  They check the scalars (-1 for n_arrivals < 0,
                payload_bytes < 0, a cap below 2 * desc_cap, d_bits not 16-byte aligned), not the arrays' contents, and
                never read or write out of bounds whatever those hold: bad entries are classified and counted as above.
     reset, stats : host arrays, ordered on `cuda_stream`; return after synchronising it.
   Launches: an insert of n_arrivals = 0 launches nothing, any other insert three kernels; a pull one kernel. */
typedef struct solo_b200_rx solo_b200_rx;
/* NULL (solo_b200_last_error() set) for a bad n_streams, depth, desc_cap or device. */
solo_b200_rx *solo_b200_rx_create(int n_streams, int depth, int desc_cap, int device);
void solo_b200_rx_destroy(solo_b200_rx *q);
int solo_b200_rx_insert_host(solo_b200_rx *q, const int32_t *stream, const uint32_t *index, const uint8_t *desc,
                             const int32_t *off, const int32_t *len, int n_arrivals, const uint8_t *payload,
                             int64_t payload_bytes);
int solo_b200_rx_insert_device(solo_b200_rx *q, const int32_t *d_stream, const uint32_t *d_index, const uint8_t *d_desc,
                               const int32_t *d_off, const int32_t *d_len, int n_arrivals, const uint8_t *d_payload,
                               int64_t payload_bytes, void *cuda_stream);
int solo_b200_rx_pull_host(solo_b200_rx *q, const uint32_t *play, uint8_t *bits, int cap, int16_t *nbytes,
                           int32_t *lostflag);
int solo_b200_rx_pull_device(solo_b200_rx *q, const uint32_t *d_play, uint8_t *d_bits, int cap, int16_t *d_nbytes,
                             int32_t *d_lostflag, void *cuda_stream);
int solo_b200_rx_reset(solo_b200_rx *q, const int32_t *streams, const uint32_t *start, int n, void *cuda_stream);
int solo_b200_rx_stats(solo_b200_rx *q, uint32_t *counters, uint64_t *bad_stream, void *cuda_stream);

/* Receive queue timing: what an RTCP receiver report (RFC 3550 6.4.1) needs beyond the counters, and how early packets
   arrive, from each datagram's arrival time.  Opt-in per queue; the calls above keep their behaviour and kernels.
   enable_timing: ts_per_index is the number of RTP timestamp units per packet index (640 for 16 kHz streams with 40 ms
     packets); max_arrivals bounds n_arrivals of a timed insert.  Allocates 52 B per stream plus 16.5 B per arrival of
     scratch.  -1 for ts_per_index = 0, max_arrivals < 1, or when timing is already enabled.  Per stream it keeps:
       transit  : uint32, transit time of the previous valid arrival;
       jitter   : uint32, RFC 3550 A.8 interarrival jitter in 1/16 timestamp units;
       highest  : uint64, extended highest index received, cycles << 32 | index;
       received : uint32, valid arrivals since the last reset (mod 2^32);
       margin   : 8 uint32, the playout-margin histogram.
   insert_timed: the insert's arrays plus arrival[a], arrival a's receive time in RTP timestamp units of the receiver's
     clock (mod 2^32).  It leaves exactly the slots, stored payload, counters and bad_stream count that insert leaves
     for the same arrays, and also:
     - A VALID arrival has its stream in [0, N) and is not malformed; late and duplicate arrivals are valid.  Only valid
       arrivals touch the timing state.
     - Over a stream's valid arrivals in ARRAY ORDER (the arrival order), with uint32 arithmetic: transit
       t = arrival - index * ts_per_index.  If received > 0: d = |(int32)(t - transit)| (2^31 for INT_MIN) and
       jitter += d - ((jitter + 8) >> 4); highest moves to index p when (p - (uint32)highest) mod 2^32 lies in [1, 2^31),
       with one more cycle when p < (uint32)highest.  If received = 0, highest = p (cycle 0).  Then transit = t and
       received += 1.
     - Each valid arrival whose index is current adds one to margin bin min(index - last - 1, 7): bin 0 plays at the
       next pull, bin 7 seven or more pulls later.  Late arrivals count in `late` only.
     The result does not depend on thread scheduling.  The running time is linear in n_arrivals whatever the arrays hold,
     including every arrival on one stream.
   timing: jitter (reported as jitter >> 4, RFC 3550), highest and received [N], margin [N][8]; any may be NULL.  Ordered
     on `cuda_stream`; returns after synchronising it.  -1 when timing is not enabled.
   reset also zeroes the listed streams' timing state (highest restarts from the next valid arrival).  insert never
   touches it.
   Entry points: *_host and *_device as for insert; the device form checks the scalars (-1 also when timing is not
   enabled or n_arrivals > max_arrivals) and never reads or writes out of bounds whatever the arrays hold.
   Launches: a timed insert of n_arrivals > 0 launches insert's three kernels, then 2 + 3 * ceil(log2(N) / 8); a reset
   of a timed queue two kernels. */
int solo_b200_rx_enable_timing(solo_b200_rx *q, uint32_t ts_per_index, int max_arrivals);
int solo_b200_rx_insert_timed_host(solo_b200_rx *q, const int32_t *stream, const uint32_t *index, const uint8_t *desc,
                                   const int32_t *off, const int32_t *len, const uint32_t *arrival, int n_arrivals,
                                   const uint8_t *payload, int64_t payload_bytes);
int solo_b200_rx_insert_timed_device(solo_b200_rx *q, const int32_t *d_stream, const uint32_t *d_index,
                                     const uint8_t *d_desc, const int32_t *d_off, const int32_t *d_len,
                                     const uint32_t *d_arrival, int n_arrivals, const uint8_t *d_payload,
                                     int64_t payload_bytes, void *cuda_stream);
int solo_b200_rx_timing(solo_b200_rx *q, uint32_t *jitter, uint64_t *highest, uint32_t *received, uint32_t *margin,
                        void *cuda_stream);

/* Send queue: turns a wave of the encoder's rows into numbered datagrams, two per row (solo_b200_split_packet), packed
   back to back in one buffer in the receive queue's arrival format, for N streams on the device.  It is independent of
   the codec batches: a pack takes the rows of any encoder batch with the same N.
   Per stream it keeps:
     next     : the packet index of the stream's next row (uint32), 0 at create; it wraps at 2^32;
     counters : 4 uint32, in this order: sent (rows that produced datagrams), octets (payload bytes sent, mod 2^32: the RTCP
                SR sender's octet count), dtx (rows with nbytes[0] <= 0), bad (rows solo_b200_split_packet refuses, i.e.
                nbytes[1] < 4 or nbytes[1] > nbytes[0], and rows with nbytes[0] > cap).
   pack: takes the encoder's output as it is, bits [N][cap] and nbytes [N][2].  For each stream s, in stream order:
     - the row's index is next[s]; then next[s] is incremented, for every stream on every call: the index follows the RTP
       clock, so it advances through DTX and bad rows too;
     - a DTX or bad row emits nothing, only its counter changes;
     - otherwise (n0 = nbytes[s][0], n1 = nbytes[s][1]) the row emits description 1 = bits[s][0, n0 - n1) and description
       2 = bits[s][n0 - n1, n0), what solo_b200_split_packet returns, and counts sent and n0 octets.  A description of 0
       bytes is not emitted (the receive queue would count it malformed).  The high-band tail is 8 bytes for 40 ms packets
       and 4 for 20 ms packets and joint mode 1; the rule does not depend on it.
     Datagram a of the call: stream[a] int32, index[a] uint32, desc[a] uint8 (1 or 2), off[a] int32, len[a] int32 -- the
     types solo_b200_rx_insert_* takes -- and its len[a] bytes at payload + off[a].  Datagrams are in the order stream 0
     description 1, stream 0 description 2, stream 1 description 1, ...; off[a] is the sum of the lengths before a, so
     the payloads lie back to back from payload[0].  Each entry array has room for 2N entries; the call writes the
     datagram count (int32) and the byte total (int64).  The result depends only on the inputs and the queue's state.
   reset: for a participant joining or rejoining a stream: sets next = start for the listed streams and zeroes their
     counters.  Host arrays; -1 (nothing done) for a stream outside [0, N) or listed twice.
   stats: counters uint32 [N][4].
   Entry points:
     pack_host   : host arrays; runs on the queue's own CUDA stream; returns the datagram count (>= 0) and writes the byte
                   total to *total, once the arrays are filled (only the first count entries and total bytes are written).
     pack_device : device arrays; only enqueues work on `cuda_stream`.  It checks the scalars (-1 for cap not a multiple
                   of 16 or below 16, N * cap above 2^31 - 1, payload_cap below N * cap -- the worst case, so the payload
                   always fits -- and d_bits or d_payload not 16-byte aligned), not the arrays' contents, and never reads or
                   writes out of bounds whatever nbytes holds.  The caller copies back the byte total, then that many bytes.
     reset, stats : host arrays, ordered on `cuda_stream`; return after synchronising it.
   Launches: a pack is exactly three kernels; a reset one. */
typedef struct solo_b200_tx solo_b200_tx;
/* NULL (solo_b200_last_error() set) for a bad n_streams or device. */
solo_b200_tx *solo_b200_tx_create(int n_streams, int device);
void solo_b200_tx_destroy(solo_b200_tx *q);
int solo_b200_tx_pack_host(solo_b200_tx *q, const uint8_t *bits, int cap, const int16_t *nbytes, uint8_t *payload,
                           int64_t payload_cap, int32_t *stream, uint32_t *index, uint8_t *desc, int32_t *off, int32_t *len,
                           int64_t *total);
int solo_b200_tx_pack_device(solo_b200_tx *q, const uint8_t *d_bits, int cap, const int16_t *d_nbytes, uint8_t *d_payload,
                             int64_t payload_cap, int32_t *d_stream, uint32_t *d_index, uint8_t *d_desc, int32_t *d_off,
                             int32_t *d_len, int32_t *d_count, int64_t *d_total, void *cuda_stream);
int solo_b200_tx_reset(solo_b200_tx *q, const int32_t *streams, const uint32_t *start, int n, void *cuda_stream);
int solo_b200_tx_stats(solo_b200_tx *q, uint32_t *counters, void *cuda_stream);

/* G.711 gateway: PSTN and SIP participants (PCMU / PCMA, 8 kHz) in 16 kHz rooms, for N streams on the device.  It is
   independent of the codec batches: its uplink rows go into the mixer's input matrix beside the decoder's rows, its
   downlink takes the mixer's output rows.  Created with framesize_ms 40 or 20 for the whole gateway, so that its rows line
   up with the room's: spp16 = 16 * framesize_ms (640 or 320) samples of 16 kHz PCM, spp8 = 8 * framesize_ms (320 or 160)
   G.711 bytes.  Each stream has a law, 0 = mu-law (PCMU) or 1 = A-law (PCMA): create sets it for every stream, reset per
   stream.
   Companding is ITU-T G.711 with exactly this integer mapping (that of the classic Sun / CCITT g711.c):
     mu-law: v = x >> 2 (arithmetic); sign mask 0xFF for v >= 0, else 0x7F with v = -v; v = min(v, 8159) + 33; seg = the
             first s in 0..7 with v < 0x40 << s (8 if none: code 0x7F ^ mask); code = ((seg << 4) | ((v >> (seg + 1)) & 0xF)) ^ mask.
             Expansion of code c: u = ~c, t = (((u & 0xF) << 3) + 0x84) << ((u & 0x70) >> 4); x = u & 0x80 ? 0x84 - t : t - 0x84.
     A-law : v = x >> 3; mask 0xD5 for v >= 0, else 0x55 with v = -v - 1; seg = the first s in 0..7 with v < 0x20 << s;
             code = ((seg << 4) | ((v >> (seg < 2 ? 1 : seg)) & 0xF)) ^ mask.
             Expansion: a = c ^ 0x55, seg = (a & 0x70) >> 4, t = ((a & 0xF) << 4) + (seg ? 0x108 : 8), t <<= seg - 1 for
             seg > 1; x = a & 0x80 ? t : -t.
   Any byte is a valid code, so no input can fault a kernel.
   uplink (PSTN -> room): g711 uint8 [N][spp8] and lost int32 [N] (bit f: 20 ms frame f, bytes [160 f, 160 f + 160), did
     not arrive; NULL: nothing lost) -> pcm int16 [N][spp16], level uint8 [N], flags uint8 [N].  Per stream:
       1. x8 = the expansion of each byte under the stream's law; the 160 samples of a lost frame are 0;
       2. the encoder's voice-activity detector runs on each 160-sample frame of x8 with the stream's detector state; flag
          bit f = speech_activity_Q8 >= SKP_FIX_CONST(0.1, 8), the comparison the encoder codes its VAD flag from.  It runs
          on lost frames too, but their bit f is 0 and bit 2 + f is set (concealed, as the decoder reports it);
       3. pcm = the fixed-point synthesis filter bank of the codec (AGR_Sate_qmf_synth of the fixed-point build) over
          (low band = x8, high band = 0) with the stream's memories: the 0-4 kHz signal at 16 kHz;
       4. level = the RFC 6464 level of the pcm row (n = spp16), as the activity reports define it.
     level and flags have the activity reports' format: they drop into the arrays solo_b200_mix_* reads, so a speaking
     PSTN participant is ranked and picked as a talker like any other, and a lost frame is never mixed.
   downlink (room -> PSTN): pcm int16 [N][spp16] (e.g. the mixer's output rows) -> g711 uint8 [N][spp8]: the low band of the
     fixed-point QMF analysis (AGR_Sate_qmf_decomp of the fixed-point build, the encoder's band split) with the stream's
     63-sample memory, compressed under the stream's law.  The high band (4-8 kHz) is dropped.
   reset: for a participant joining or rejoining a stream: the listed streams (host array of n) become fresh streams with
     law[i] (a host array of n; NULL or an entry of -1 takes the create law).  -1 with nothing done (solo_b200_last_error()
     set) for a stream outside [0, N), one listed twice, or a law other than 0 / 1.  One kernel ordered on `cuda_stream`,
     which the call then synchronises (that stream only).  From the next call a reset stream gives, in both directions,
     exactly what a stream of a newly created gateway with that law gives.
   Entry points:
     *_host   : host arrays; run on the gateway's own CUDA stream and return when done.
     *_device : device arrays; only enqueue work on `cuda_stream`.  They check the pointers: -1 before any launch for a
                NULL row pointer, d_g711 or d_pcm not 16-byte aligned, or d_lost not 4-byte aligned.
   Launches: an uplink is two kernels, a downlink one, a reset one (create one).
   state_bytes: device bytes per stream. */
typedef struct solo_b200_g711 solo_b200_g711;
#define SOLO_B200_G711_ULAW 0
#define SOLO_B200_G711_ALAW 1
/* NULL (solo_b200_last_error() set) for a bad n_streams, framesize_ms, law or device. */
solo_b200_g711 *solo_b200_g711_create(int n_streams, int framesize_ms, int law, int device);
void solo_b200_g711_destroy(solo_b200_g711 *g);
int solo_b200_g711_uplink_host(solo_b200_g711 *g, const uint8_t *g711, const int32_t *lost, int16_t *pcm, uint8_t *level,
                               uint8_t *flags);
int solo_b200_g711_uplink_device(solo_b200_g711 *g, const uint8_t *d_g711, const int32_t *d_lost, int16_t *d_pcm,
                                 uint8_t *d_level, uint8_t *d_flags, void *cuda_stream);
int solo_b200_g711_downlink_host(solo_b200_g711 *g, const int16_t *pcm, uint8_t *g711);
int solo_b200_g711_downlink_device(solo_b200_g711 *g, const int16_t *d_pcm, uint8_t *d_g711, void *cuda_stream);
int solo_b200_g711_reset(solo_b200_g711 *g, const int32_t *streams, int n, const int32_t *law, void *cuda_stream);
int solo_b200_g711_state_bytes(void);

/* Multi-GPU ingest through peer memory:after this call kernels launched on `device` may read and write buffers that live in
   `peer_device`'s memory (same process, or another process's allocation mapped with CUDA IPC).  The *_device entry points
   then accept such addresses for pcm / bits / nbytes / lostflag: the band-split kernel pulls its PCM rows over NVLink and
   the entropy-coding and decoder kernels push their result rows back, so a single-ingest deployment needs no separate
   scatter / gather step (solo_b200/shard.py shows the plumbing with torch.distributed). */
int solo_b200_enable_peer_access(int device, int peer_device);

/* The six AGR_Sate_* functions (AGR_JC1_SDK_API.h) hand out slots of a process-wide arena: segments of 256 streams that are
   created on demand and shared by the handles.  out[4] = {encoder segments, encoder slots in use, decoder segments, decoder
   slots in use}. */
int solo_b200_arena_stats(int out[4]);

/* Bytes of device state held per stream (encoder / 16 kHz decoder; decoder of a sample rate, 16000 or 32000, -1 for any
   other). */
int solo_b200_enc_state_bytes(void);
int solo_b200_dec_state_bytes(void);
int solo_b200_dec_state_bytes_rate(int samplerate);
/* Number of kernels this library has launched in this process (for benchmark bookkeeping). */
long long solo_b200_kernel_launches(void);
/* Kernel timing with CUDA events recorded on the launching stream (only while enabled).  profile_read fills two arrays
   of 4: total ms and launch count since the last read for {encoder analysis, encoder NSQ, encoder finish, decode}. */
void solo_b200_profile_enable(int on);
int solo_b200_profile_read(double ms_total[4], long long launches[4]);
/* The *_host entry points process a packet wave as `chunks` groups of streams on the batch's CUDA streams so that the copies
   of one group overlap the kernels of another.  Default (0, or env SOLO_B200_CHUNKS unset): 3.  The *_device entry points
   always launch each kernel once for the whole batch on the caller's stream.  Results do not depend on it. */
void solo_b200_set_chunks(int chunks);
const char *solo_b200_last_error(void);

#ifdef __cplusplus
}
#endif
#endif
