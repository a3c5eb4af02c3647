"""ctypes binding of libsolo_b200.so.

Mirrors the reference interface for the hot path:
  * ``SoloEncoder`` / ``SoloDecoder``  -- the six ``AGR_Sate_*`` entry points (one stream per handle), same argument
    meaning and return conventions as /root/reference/JC1_SDK_SRC_ARM/interface/AGR_JC1_SDK_API.h:33-64;
  * ``EncoderBatch`` / ``DecoderBatch`` -- the batched extension (``include/solo_b200.h``), N streams per call.
Buffers are numpy arrays (host entry points) or raw device pointers (ints) for the ``*_device`` entry points.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# SOLO_B200_LIB: load another build of the same CUDA library (kernel-variant experiments); never a CPU path
LIB_PATH = os.environ.get("SOLO_B200_LIB") or os.path.join(_HERE, "libsolo_b200.so")
PACKET = 640


class SoloError(RuntimeError):
    pass


class EncCtrl(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("mode", "targetRate_bps", "samplerate", "dtx_enable", "framesize_ms",
                                         "joint_enable", "joint_mode", "useMDIndex")]


class DecCtrl(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("packetLoss_perc", "samplerate", "framesize_ms", "joint_enable",
                                         "joint_mode", "useMDIndex")]


_lib = None


def lib():
    """Load libsolo_b200.so (fails loudly when it has not been built: there is no CPU implementation)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SoloError("%s missing: run `python -m solo_b200.build` (needs nvcc); no CPU fallback exists" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        vp, i32p = C.c_void_p, C.c_void_p
        L.solo_b200_last_error.restype = C.c_char_p
        L.solo_b200_set_chunks.argtypes = [C.c_int]
        L.solo_b200_kernel_launches.restype = C.c_longlong
        L.solo_b200_enc_batch_create.restype = vp
        L.solo_b200_enc_batch_create.argtypes = [C.c_int, C.POINTER(EncCtrl), C.c_int]
        L.solo_b200_enc_batch_encode_host.argtypes = [vp, vp, vp, C.c_int, vp]
        L.solo_b200_enc_batch_encode_device.argtypes = [vp, vp, vp, C.c_int, vp, vp]
        L.solo_b200_enc_batch_destroy.argtypes = [vp]
        L.solo_b200_enc_batch_set_control_host.argtypes = [vp, vp, vp, vp]
        L.solo_b200_enc_batch_set_control_device.argtypes = [vp, vp, vp, vp, vp]
        L.solo_b200_encoder_set_control.argtypes = [vp, C.c_int32, C.c_int32, C.c_int32]
        L.solo_b200_dec_batch_create.restype = vp
        L.solo_b200_dec_batch_create.argtypes = [C.c_int, C.POINTER(DecCtrl), C.c_int]
        L.solo_b200_dec_batch_create_arith.restype = vp
        L.solo_b200_dec_batch_create_arith.argtypes = [C.c_int, C.POINTER(DecCtrl), C.c_int, C.c_int]
        L.solo_b200_dec_batch_create_out.restype = vp
        L.solo_b200_dec_batch_create_out.argtypes = [C.c_int, C.POINTER(DecCtrl), C.c_int, C.c_int, C.c_int]
        L.solo_b200_dec_batch_decode_host.argtypes = [vp, vp, vp, C.c_int, vp, vp, vp]
        L.solo_b200_dec_batch_decode_device.argtypes = [vp, vp, vp, C.c_int, vp, vp, vp, vp]
        L.solo_b200_dec_batch_destroy.argtypes = [vp]
        for f in ("solo_b200_enc_batch_export_state", "solo_b200_enc_batch_import_state", "solo_b200_dec_batch_export_state",
                  "solo_b200_dec_batch_import_state"):
            getattr(L, f).argtypes = [vp, C.c_int, vp]
        for f in ("solo_b200_dec_batch_export_state_sized", "solo_b200_dec_batch_import_state_sized"):
            getattr(L, f).argtypes = [vp, C.c_int, vp, C.c_int]
        L.solo_b200_enc_batch_reset.argtypes = [vp, vp, C.c_int, vp, vp, vp, vp]
        L.solo_b200_dec_batch_reset.argtypes = [vp, vp, C.c_int, vp, vp]
        for f in ("solo_b200_enc_batch_export_states", "solo_b200_enc_batch_import_states", "solo_b200_dec_batch_export_states",
                  "solo_b200_dec_batch_import_states"):
            getattr(L, f).argtypes = [vp, vp, C.c_int, vp, vp]
        pp, ip = C.POINTER(vp), C.POINTER(C.c_int)
        L.solo_b200_split_packet.argtypes = [vp, vp, pp, ip, pp, ip]
        L.solo_b200_merge_packets.argtypes = [vp, C.c_int, vp, C.c_int, vp, C.c_int, vp, vp]
        L.solo_b200_bitfile_pack.argtypes = [vp, vp, vp, C.c_int]
        L.solo_b200_bitfile_unpack.argtypes = [vp, C.c_int, pp, vp]
        L.solo_b200_apply_loss_device.argtypes = [vp, vp, vp, vp, vp, C.c_int, C.c_int, vp]
        L.solo_b200_enable_peer_access.argtypes = [C.c_int, C.c_int]
        L.solo_b200_enc_state_bytes.restype = C.c_int
        L.solo_b200_dec_state_bytes.restype = C.c_int
        L.solo_b200_dec_state_bytes_rate.restype = C.c_int
        L.solo_b200_dec_state_bytes_rate.argtypes = [C.c_int]
        L.solo_b200_profile_enable.argtypes = [C.c_int]
        L.solo_b200_profile_read.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_longlong)]
        L.AGR_Sate_Encoder_Init.restype = vp
        L.AGR_Sate_Encoder_Init.argtypes = [C.POINTER(EncCtrl)]
        L.AGR_Sate_Encoder_Encode.restype = C.c_int32
        L.AGR_Sate_Encoder_Encode.argtypes = [vp, vp, vp, C.c_int32, vp]
        L.AGR_Sate_Encoder_Uninit.argtypes = [vp]
        L.AGR_Sate_Decoder_Init.restype = vp
        L.AGR_Sate_Decoder_Init.argtypes = [C.POINTER(DecCtrl)]
        L.AGR_Sate_Decoder_Decode.restype = C.c_int32
        L.AGR_Sate_Decoder_Decode.argtypes = [vp, vp, vp, vp, vp, C.c_int32]
        L.AGR_Sate_Decoder_Uninit.argtypes = [vp]
        for f in ("solo_b200_enc_batch_activity_host", "solo_b200_dec_batch_activity_host", "solo_b200_encoder_last_activity",
                  "solo_b200_decoder_last_activity"):
            getattr(L, f).argtypes = [vp, vp, vp]
        for f in ("solo_b200_enc_batch_activity_device", "solo_b200_dec_batch_activity_device"):
            getattr(L, f).argtypes = [vp, vp, vp, vp, vp]
        L.solo_b200_mix_host.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int, vp]
        L.solo_b200_mix_device.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int, C.c_int, vp, vp]
        L.solo_b200_rx_create.restype = vp
        L.solo_b200_rx_create.argtypes = [C.c_int] * 4
        L.solo_b200_rx_destroy.argtypes = [vp]
        L.solo_b200_rx_insert_host.argtypes = [vp] * 6 + [C.c_int, vp, C.c_int64]
        L.solo_b200_rx_insert_device.argtypes = [vp] * 6 + [C.c_int, vp, C.c_int64, vp]
        L.solo_b200_rx_pull_host.argtypes = [vp, vp, vp, C.c_int, vp, vp]
        L.solo_b200_rx_pull_device.argtypes = [vp, vp, vp, C.c_int, vp, vp, vp]
        L.solo_b200_rx_reset.argtypes = [vp, vp, vp, C.c_int, vp]
        L.solo_b200_rx_stats.argtypes = [vp, vp, vp, vp]
        L.solo_b200_rx_enable_timing.argtypes = [vp, C.c_uint32, C.c_int]
        L.solo_b200_rx_insert_timed_host.argtypes = [vp] * 7 + [C.c_int, vp, C.c_int64]
        L.solo_b200_rx_insert_timed_device.argtypes = [vp] * 7 + [C.c_int, vp, C.c_int64, vp]
        L.solo_b200_rx_timing.argtypes = [vp] * 6
        L.solo_b200_tx_create.restype = vp
        L.solo_b200_tx_create.argtypes = [C.c_int, C.c_int]
        L.solo_b200_tx_destroy.argtypes = [vp]
        L.solo_b200_tx_pack_host.argtypes = [vp, vp, C.c_int, vp, vp, C.c_int64] + [vp] * 6
        L.solo_b200_tx_pack_device.argtypes = [vp, vp, C.c_int, vp, vp, C.c_int64] + [vp] * 8
        L.solo_b200_tx_reset.argtypes = [vp, vp, vp, C.c_int, vp]
        L.solo_b200_tx_stats.argtypes = [vp, vp, vp]
        L.solo_b200_mix_contributors_host.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp]
        L.solo_b200_mix_contributors_device.argtypes = [vp, vp, C.c_int, C.c_int, vp, vp, C.c_int, vp, vp, vp]
        L.solo_b200_g711_create.restype = vp
        L.solo_b200_g711_create.argtypes = [C.c_int] * 4
        L.solo_b200_g711_destroy.argtypes = [vp]
        L.solo_b200_g711_uplink_host.argtypes = [vp] * 6
        L.solo_b200_g711_uplink_device.argtypes = [vp] * 7
        L.solo_b200_g711_downlink_host.argtypes = [vp] * 3
        L.solo_b200_g711_downlink_device.argtypes = [vp] * 4
        L.solo_b200_g711_reset.argtypes = [vp, vp, C.c_int, vp, vp]
        L.solo_b200_g711_state_bytes.restype = C.c_int
        _lib = L
    return _lib


def _err():
    return lib().solo_b200_last_error().decode("utf-8", "replace")


def kernel_launches():
    return int(lib().solo_b200_kernel_launches())


def state_bytes():
    return int(lib().solo_b200_enc_state_bytes()), int(lib().solo_b200_dec_state_bytes())


def dec_state_bytes(samplerate=16000):
    """Bytes of device state per decoder stream of a sample rate (16000 or 32000)."""
    n = int(lib().solo_b200_dec_state_bytes_rate(int(samplerate)))
    if n < 0:
        raise SoloError("no decoder for sample rate %r" % (samplerate,))
    return n


def _activity_host(fn, h, n):
    level = np.empty(n, np.uint8)
    flags = np.empty(n, np.uint8)
    r = fn(h, level.ctypes.data, flags.ctypes.data)
    if r:
        raise SoloError("activity failed (%d): %s" % (r, _err()))
    return level, flags


def _activity_device(fn, h, d_pcm, d_level, d_flags, stream):
    r = fn(h, d_pcm, d_level, d_flags, stream)
    if r:
        raise SoloError("activity_device failed (%d): %s" % (r, _err()))


def _queue_reset(fn, name, h, streams, start, stream):
    streams = np.ascontiguousarray(streams, np.int32).ravel()
    start = np.ascontiguousarray(np.broadcast_to(np.asarray(start, np.int64) & 0xFFFFFFFF, streams.shape), np.uint32)
    r = fn(h, streams.ctypes.data, start.ctypes.data, len(streams), stream)
    if r:
        raise SoloError("%s failed (%d): %s" % (name, r, _err()))


def _stream_list(streams):
    s = np.asarray(streams, np.int64).ravel()
    if (s < 0).any() or (s > np.iinfo(np.int32).max).any():
        raise SoloError("a stream index is outside the batch")
    return np.ascontiguousarray(s.astype(np.int32))


def _settings(name, v, n, keep):
    """A reset setting as an int32 [n] host array (None: NULL, a scalar: the same for every listed stream)."""
    if v is None:
        return None
    a = np.ascontiguousarray(np.broadcast_to(np.asarray(v, np.int64), (n,)))
    if (a < np.iinfo(np.int32).min).any() or (a > np.iinfo(np.int32).max).any():
        raise SoloError("%s: a setting is out of range" % name)
    keep.append(a.astype(np.int32))
    return keep[-1].ctypes.data


def _move_states(fn, name, h, streams, d_blobs, stream):
    s = _stream_list(streams)
    r = fn(h, s.ctypes.data, len(s), d_blobs, stream)
    if r:
        raise SoloError("%s failed (%d): %s" % (name, r, _err()))


def profile_enable(on=True):
    lib().solo_b200_profile_enable(1 if on else 0)


def profile_read():
    """{kernel: (total_ms, launches)} since the last read."""
    t = (C.c_double * 4)()
    n = (C.c_longlong * 4)()
    lib().solo_b200_profile_read(t, n)
    names = ("enc_analysis", "enc_nsq", "enc_finish", "decode")
    return {k: (t[i], n[i]) for i, k in enumerate(names)}


class SoloEncoder:
    """One stream through AGR_Sate_Encoder_Init / Encode / Uninit."""

    def __init__(self, rate=13600, dtx=0, use_md_index=0, samplerate=16000, framesize_ms=40, joint_enable=0, joint_mode=0):
        self.ctrl = EncCtrl(2, rate, samplerate, dtx, framesize_ms, joint_enable, joint_mode, use_md_index)
        self.h = lib().AGR_Sate_Encoder_Init(C.byref(self.ctrl))
        if not self.h:
            raise SoloError("AGR_Sate_Encoder_Init returned NULL: " + _err())
        self._bits = np.zeros(1024, np.uint8)
        self._nb = np.zeros(6, np.int16)
        self.samples = 16 * framesize_ms

    def encode(self, pcm640, bufsize=1024):
        pcm = np.ascontiguousarray(pcm640, dtype=np.int16)
        assert pcm.size == self.samples
        self._nb[:] = 0
        n = lib().AGR_Sate_Encoder_Encode(self.h, pcm.ctypes.data, self._bits.ctypes.data, bufsize, self._nb.ctypes.data)
        return bytes(self._bits[:max(n, 0)]), (int(self._nb[0]), int(self._nb[1])), n

    def last_activity(self):
        """(level, flags) of the last packet: RFC 6464 level of its input and the VAD flags coded into its frames (see
        solo_b200_encoder_last_activity in include/solo_b200.h)."""
        level, flags = _activity_host(lib().solo_b200_encoder_last_activity, self.h, 1)
        return int(level[0]), int(flags[0])

    def set_control(self, rate=None, dtx=None, loss=None):
        """Target rate (b/s), DTX on / off and expected packet loss (%) from the next packet on; None leaves a setting as
        it is (see solo_b200_encoder_set_control in include/solo_b200.h)."""
        r = lib().solo_b200_encoder_set_control(self.h, *(-1 if v is None else int(v) for v in (rate, dtx, loss)))
        if r:
            raise SoloError("set_control failed (%d): %s" % (r, "setting out of range" if r == -1 else _err()))

    def close(self):
        if getattr(self, "h", None):
            lib().AGR_Sate_Encoder_Uninit(self.h)
            self.h = None

    __del__ = close


class SoloDecoder:
    """One stream through AGR_Sate_Decoder_Init / Decode / Uninit (payload pre-trimmed by the caller).  samplerate 16000
    or 32000 (the latter: decoder only, a 16 kHz SILK core; see include/solo_b200.h)."""

    def __init__(self, use_md_index=0, samplerate=16000, framesize_ms=40, joint_enable=0, joint_mode=0):
        self.ctrl = DecCtrl(0, samplerate, framesize_ms, joint_enable, joint_mode, use_md_index)
        self.h = lib().AGR_Sate_Decoder_Init(C.byref(self.ctrl))
        if not self.h:
            raise SoloError("AGR_Sate_Decoder_Init returned NULL: " + _err())
        self._out = np.zeros(1920, np.int16)
        self._ns = C.c_int16(0)
        self.samples = samplerate // 1000 * framesize_ms

    def decode(self, payload, nbytes, lostflag):
        buf = np.zeros(1040, np.uint8)
        buf[:len(payload)] = np.frombuffer(bytes(payload), np.uint8)
        nb = np.array([nbytes[0], nbytes[1], 0, 0, 0, 0], np.int16)
        ret = lib().AGR_Sate_Decoder_Decode(self.h, self._out.ctypes.data, C.byref(self._ns), buf.ctypes.data, nb.ctypes.data, int(lostflag))
        self.last_nbytes = (int(nb[0]), int(nb[1]))
        self.last_nsamples = int(self._ns.value)
        return self._out[:self.samples].copy(), ret

    def last_activity(self):
        """(level, flags) of the last packet: RFC 6464 level of its output, VAD and concealment flags of its frames (see
        solo_b200_decoder_last_activity in include/solo_b200.h)."""
        level, flags = _activity_host(lib().solo_b200_decoder_last_activity, self.h, 1)
        return int(level[0]), int(flags[0])

    def close(self):
        if getattr(self, "h", None):
            lib().AGR_Sate_Decoder_Uninit(self.h)
            self.h = None

    __del__ = close


class EncoderBatch:
    """N encoder streams resident on one GPU; one call = one 40 ms packet for every stream."""

    def __init__(self, n, rate=13600, dtx=0, use_md_index=0, device=0, framesize_ms=40, joint_hb=0):
        """joint_hb=1: the reference's joint mode 1 (one 40 ms high-band frame per packet)."""
        self.n = int(n)
        self.samples = 16 * framesize_ms          # samples per packet and stream (row length of the PCM matrix)
        self.ctrl = EncCtrl(2, rate, 16000, dtx, framesize_ms, 1 if joint_hb else 0, 1 if joint_hb else 0, use_md_index)
        self.h = lib().solo_b200_enc_batch_create(self.n, C.byref(self.ctrl), device)
        if not self.h:
            raise SoloError("solo_b200_enc_batch_create failed: " + _err())

    def encode(self, pcm, cap=256, bits=None, nbytes=None):
        """pcm: int16 [N, 640] host array -> (bits uint8 [N, cap], nbytes int16 [N, 2])."""
        pcm = np.ascontiguousarray(pcm, dtype=np.int16)
        assert pcm.shape == (self.n, self.samples)
        if bits is None:
            bits = np.empty((self.n, cap), np.uint8)
        if nbytes is None:
            nbytes = np.empty((self.n, 2), np.int16)
        r = lib().solo_b200_enc_batch_encode_host(self.h, pcm.ctypes.data, bits.ctypes.data, cap, nbytes.ctypes.data)
        if r:
            raise SoloError("encode_host failed (%d): %s" % (r, _err()))
        return bits, nbytes

    def encode_ptr(self, pcm_ptr, bits_ptr, cap, nbytes_ptr):
        """Host entry point on raw addresses (e.g. pinned torch tensors' data_ptr())."""
        r = lib().solo_b200_enc_batch_encode_host(self.h, pcm_ptr, bits_ptr, cap, nbytes_ptr)
        if r:
            raise SoloError("encode_host failed (%d): %s" % (r, _err()))

    def export_state(self, idx):
        """Opaque blob with the complete state of stream idx (checkpoint / migration)."""
        blob = np.zeros(lib().solo_b200_enc_state_bytes(), np.uint8)
        if lib().solo_b200_enc_batch_export_state(self.h, int(idx), blob.ctypes.data):
            raise SoloError(_err())
        return blob

    def import_state(self, idx, blob):
        blob = np.ascontiguousarray(blob, np.uint8)
        if blob.size != lib().solo_b200_enc_state_bytes() or lib().solo_b200_enc_batch_import_state(self.h, int(idx), blob.ctypes.data):
            raise SoloError("import_state: " + _err())

    def encode_device(self, d_pcm, d_bits, cap, d_nbytes, stream=0):
        r = lib().solo_b200_enc_batch_encode_device(self.h, d_pcm, d_bits, cap, d_nbytes, stream)
        if r:
            raise SoloError("encode_device failed (%d): %s" % (r, _err()))

    def activity(self):
        """(level uint8 [N], flags uint8 [N]) of the last encode() wave: the RFC 6464 level of every input row and the VAD
        flags coded into its frames (bit f = frame f; see include/solo_b200.h)."""
        return _activity_host(lib().solo_b200_enc_batch_activity_host, self.h, self.n)

    def activity_device(self, d_pcm, d_level, d_flags, stream=0):
        """The same after an encode_device() wave: d_pcm = that wave's input rows, d_level / d_flags = device uint8 [N]
        outputs; enqueued on `stream`."""
        _activity_device(lib().solo_b200_enc_batch_activity_device, self.h, d_pcm, d_level, d_flags, stream)

    def set_control(self, rate=None, dtx=None, loss=None):
        """Per-stream target rate (b/s), DTX (0 / 1) and expected packet loss (0-100 %) from the next packet on.  Each is
        None (unchanged), a scalar for every stream or an int array [N] whose -1 entries leave that stream alone.  Raises
        SoloError, with nothing applied, if a value is out of range."""
        keep = []

        def arg(v):
            if v is None:
                return None
            a = np.ascontiguousarray(np.broadcast_to(np.asarray(v, np.int64), (self.n,)))
            if (a < np.iinfo(np.int32).min).any() or (a > np.iinfo(np.int32).max).any():
                raise SoloError("set_control: a setting is out of range")
            keep.append(a.astype(np.int32))
            return keep[-1].ctypes.data

        r = lib().solo_b200_enc_batch_set_control_host(self.h, arg(rate), arg(dtx), arg(loss))
        if r:
            raise SoloError("set_control failed (%d): %s" % (r, _err()))

    def set_control_device(self, d_rate=None, d_dtx=None, d_loss=None, stream=0):
        """Device int32 arrays [N] (addresses, None = unchanged), enqueued on `stream` in order with encode_device; an
        out-of-range entry leaves that stream's setting unchanged."""
        r = lib().solo_b200_enc_batch_set_control_device(self.h, d_rate, d_dtx, d_loss, stream)
        if r:
            raise SoloError("set_control_device failed (%d): %s" % (r, _err()))

    def reset(self, streams, rate=None, dtx=None, loss=None, stream=0):
        """Re-initialise the listed streams as a new batch's, then give them rate / dtx / loss: None or -1 keeps the create
        value, a scalar applies to every listed stream, an array has one entry per listed stream.  Ordered on `stream`;
        returns once that stream is done.  Raises SoloError, with nothing done, for a stream outside [0, N), one listed
        twice or a setting out of range (see solo_b200_enc_batch_reset)."""
        s, keep = _stream_list(streams), []
        args = [_settings("enc_reset", v, len(s), keep) for v in (rate, dtx, loss)]
        r = lib().solo_b200_enc_batch_reset(self.h, s.ctypes.data, len(s), *args, stream)
        if r:
            raise SoloError("enc_reset failed (%d): %s" % (r, _err()))

    def export_states(self, streams, d_blobs, stream=0):
        """The listed streams' states into d_blobs (a device address: uint8 [len(streams), enc_state_bytes], 8-byte
        aligned; this GPU's, a peer GPU's or mapped host memory), ordered on `stream`."""
        _move_states(lib().solo_b200_enc_batch_export_states, "enc_export_states", self.h, streams, d_blobs, stream)

    def import_states(self, streams, d_blobs, stream=0):
        """The listed streams' states from d_blobs (laid out as export_states writes them), ordered on `stream`."""
        _move_states(lib().solo_b200_enc_batch_import_states, "enc_import_states", self.h, streams, d_blobs, stream)

    def close(self):
        if getattr(self, "h", None):
            lib().solo_b200_enc_batch_destroy(self.h)
            self.h = None

    __del__ = close


DEC_ARITH = {"flp": 0, "fix": 1}   # SOLO_B200_DEC_FLP / SOLO_B200_DEC_FIX


class DecoderBatch:
    """N decoder streams resident on one GPU."""

    def __init__(self, n, use_md_index=0, device=0, framesize_ms=40, joint_hb=0, arith="flp", samplerate=16000, out_samplerate=None):
        """arith: "flp" decodes to the reference float build's PCM, "fix" to its fixed-point build's (40 ms packets and
        joint mode 1 only; see solo_b200_dec_batch_create_arith in include/solo_b200.h).  samplerate: 16000, or 32000 for
        streams of the reference's 32 kHz API (16 kHz SILK core; PCM rows of 32 * framesize_ms samples).
        out_samplerate: the rate of the PCM rows, samplerate by default; 16000 with samplerate 32000 decodes the streams to
        their 16 kHz core only (rows of 16 * framesize_ms samples that mix with 16 kHz streams' rows; see
        solo_b200_dec_batch_create_out)."""
        if arith not in DEC_ARITH:
            raise SoloError("arith must be one of %s, not %r" % (sorted(DEC_ARITH), arith))
        self.n = int(n)
        self.samplerate = int(samplerate)
        self.out_samplerate = self.samplerate if out_samplerate is None else int(out_samplerate)
        self.samples = self.out_samplerate // 1000 * framesize_ms
        self.arith = arith
        self.ctrl = DecCtrl(0, self.samplerate, framesize_ms, 1 if joint_hb else 0, 1 if joint_hb else 0, use_md_index)
        self.h = lib().solo_b200_dec_batch_create_out(self.n, C.byref(self.ctrl), device, DEC_ARITH[arith], self.out_samplerate)
        if not self.h:
            raise SoloError("solo_b200_dec_batch_create failed: " + _err())

    def decode(self, bits, nbytes, lostflag, pcm=None, ret=None):
        """bits uint8 [N, cap], nbytes int16 [N, 2], lostflag int32 [N] -> (pcm int16 [N, samples], ret int32 [N])."""
        bits = np.ascontiguousarray(bits, dtype=np.uint8)
        nbytes = np.ascontiguousarray(nbytes, dtype=np.int16)
        lostflag = np.ascontiguousarray(lostflag, dtype=np.int32)
        assert bits.shape[0] == self.n and nbytes.shape == (self.n, 2) and lostflag.shape == (self.n,)
        if pcm is None:
            pcm = np.zeros((self.n, self.samples), np.int16)
        if ret is None:
            ret = np.zeros(self.n, np.int32)
        r = lib().solo_b200_dec_batch_decode_host(self.h, pcm.ctypes.data, bits.ctypes.data, bits.shape[1], nbytes.ctypes.data,
                                                  lostflag.ctypes.data, ret.ctypes.data)
        if r:
            raise SoloError("decode_host failed (%d): %s" % (r, _err()))
        return pcm, ret

    def decode_ptr(self, pcm_ptr, bits_ptr, cap, nbytes_ptr, flags_ptr, ret_ptr):
        r = lib().solo_b200_dec_batch_decode_host(self.h, pcm_ptr, bits_ptr, cap, nbytes_ptr, flags_ptr, ret_ptr)
        if r:
            raise SoloError("decode_host failed (%d): %s" % (r, _err()))

    def export_state(self, idx):
        blob = np.zeros(lib().solo_b200_dec_state_bytes_rate(self.samplerate), np.uint8)
        if lib().solo_b200_dec_batch_export_state_sized(self.h, int(idx), blob.ctypes.data, blob.size):
            raise SoloError(_err())
        return blob

    def import_state(self, idx, blob):
        """A blob of export_state from a batch of the same sample rate and output rate (a blob of another rate, or of a
        32 kHz batch of the other output rate, is refused)."""
        blob = np.ascontiguousarray(blob, np.uint8)
        if lib().solo_b200_dec_batch_import_state_sized(self.h, int(idx), blob.ctypes.data, blob.size):
            raise SoloError("import_state: " + _err())

    def decode_device(self, d_pcm, d_bits, cap, d_nbytes, d_flags, d_ret=0, stream=0):
        r = lib().solo_b200_dec_batch_decode_device(self.h, d_pcm, d_bits, cap, d_nbytes, d_flags, d_ret, stream)
        if r:
            raise SoloError("decode_device failed (%d): %s" % (r, _err()))

    def reset(self, streams, arith=None, stream=0):
        """Re-initialise the listed streams as a new batch's.  arith: None or -1 keeps the create arithmetic, "flp" / "fix"
        (or 0 / 1) for every listed stream, or an array with one entry per listed stream.  Ordered on `stream`; returns
        once that stream is done.  Raises SoloError, with nothing done, for a stream outside [0, N), one listed twice or
        a bad arithmetic (see solo_b200_dec_batch_reset)."""
        s, keep = _stream_list(streams), []
        if isinstance(arith, str):
            if arith not in DEC_ARITH:
                raise SoloError("arith must be one of %s, not %r" % (sorted(DEC_ARITH), arith))
            arith = DEC_ARITH[arith]
        r = lib().solo_b200_dec_batch_reset(self.h, s.ctypes.data, len(s), _settings("dec_reset", arith, len(s), keep), stream)
        if r:
            raise SoloError("dec_reset failed (%d): %s" % (r, _err()))

    def export_states(self, streams, d_blobs, stream=0):
        """The listed streams' states into d_blobs (a device address: uint8 [len(streams), dec_state_bytes(samplerate)],
        8-byte aligned; this GPU's, a peer GPU's or mapped host memory), ordered on `stream`."""
        _move_states(lib().solo_b200_dec_batch_export_states, "dec_export_states", self.h, streams, d_blobs, stream)

    def import_states(self, streams, d_blobs, stream=0):
        """The listed streams' states from d_blobs (laid out as export_states writes them), ordered on `stream`; a 32 kHz
        batch refuses the whole list if any blob is of the other output mode."""
        _move_states(lib().solo_b200_dec_batch_import_states, "dec_import_states", self.h, streams, d_blobs, stream)

    def activity(self):
        """(level uint8 [N], flags uint8 [N]) of the last decode() wave: the RFC 6464 level of every output row, the VAD
        flags decoded from its frames (bit f) and which frames were concealed (bit 2 + f); a rejected packet gives 127 / 0."""
        return _activity_host(lib().solo_b200_dec_batch_activity_host, self.h, self.n)

    def activity_device(self, d_pcm, d_level, d_flags, stream=0):
        """The same after a decode_device() wave: d_pcm = that wave's output rows, d_level / d_flags = device uint8 [N]
        outputs; enqueued on `stream`."""
        _activity_device(lib().solo_b200_dec_batch_activity_device, self.h, d_pcm, d_level, d_flags, stream)

    def close(self):
        if getattr(self, "h", None):
            lib().solo_b200_dec_batch_destroy(self.h)
            self.h = None

    __del__ = close


def set_chunks(n):
    """Number of stream groups a packet wave is pipelined as (see include/solo_b200.h); 1 = plain single launches."""
    lib().solo_b200_set_chunks(int(n))


# ---- packet framing (host functions of the library; no GPU involved) --------------------------------------------------
def split_packet(bits, nbytes):
    """(description 1, description 2) = (MD1, MD2 + 8 high-band bytes) of one payload row; (b"", b"") for a DTX row."""
    buf = np.ascontiguousarray(np.frombuffer(bytes(bits), np.uint8))
    nb = np.array([nbytes[0], nbytes[1]], np.int16)
    p1, p2, n1, n2 = C.c_void_p(), C.c_void_p(), C.c_int(), C.c_int()
    if lib().solo_b200_split_packet(buf.ctypes.data, nb.ctypes.data, C.byref(p1), C.byref(n1), C.byref(p2), C.byref(n2)):
        raise SoloError("split_packet: inconsistent length fields")
    o1 = (p1.value or buf.ctypes.data) - buf.ctypes.data
    o2 = (p2.value or buf.ctypes.data) - buf.ctypes.data
    return bytes(buf[o1:o1 + n1.value]), bytes(buf[o2:o2 + n2.value])


def merge_packets(p1, p2, cap=1024):
    """(payload row, (n0, n1), lostflag) for the decoder from whichever descriptions arrived (None / b"" = lost)."""
    a = np.frombuffer(p1, np.uint8).copy() if p1 else None
    b = np.frombuffer(p2, np.uint8).copy() if p2 else None
    out = np.zeros(cap, np.uint8)
    nb = np.zeros(2, np.int16)
    flag = C.c_int32()
    r = lib().solo_b200_merge_packets(a.ctypes.data if a is not None else None, len(a) if a is not None else 0,
                                      b.ctypes.data if b is not None else None, len(b) if b is not None else 0,
                                      out.ctypes.data, cap, nb.ctypes.data, C.byref(flag))
    if r:
        raise SoloError("merge_packets: packets do not fit")
    return bytes(out[:max(int(nb[0]), 0)]), (int(nb[0]), int(nb[1])), int(flag.value)


def bitfile_pack(bits, nbytes):
    """One record of the reference CLI's .bit file."""
    buf = np.frombuffer(bytes(bits) + b"\0", np.uint8).copy()
    nb = np.array([nbytes[0], nbytes[1]], np.int16)
    out = np.zeros(4 + max(int(nbytes[0]), 0), np.uint8)
    n = lib().solo_b200_bitfile_pack(buf.ctypes.data, nb.ctypes.data, out.ctypes.data, out.size)
    if n < 0:
        raise SoloError("bitfile_pack")
    return bytes(out[:n])


def bitfile_unpack(data, offset=0):
    """(payload, (n0, n1), next offset) of the record starting at `offset`."""
    buf = np.frombuffer(data, np.uint8)
    view = np.ascontiguousarray(buf[offset:])
    nb = np.zeros(2, np.int16)
    p = C.c_void_p()
    n = lib().solo_b200_bitfile_unpack(view.ctypes.data, view.size, C.byref(p), nb.ctypes.data)
    if n < 0:
        raise SoloError("bitfile_unpack: truncated record")
    return bytes(view[4:n]), (int(nb[0]), int(nb[1])), offset + n


def enable_peer_access(device, peer_device):
    if lib().solo_b200_enable_peer_access(int(device), int(peer_device)):
        raise SoloError(_err())


def apply_loss_device(d_bits_in, d_nbytes_in, d_lostflag, d_bits_out, d_nbytes_out, cap, n, stream=0):
    if lib().solo_b200_apply_loss_device(d_bits_in, d_nbytes_in, d_lostflag, d_bits_out, d_nbytes_out, cap, n, stream):
        raise SoloError(_err())


# ---- conference mixer (include/solo_b200.h, solo_b200_mix_*) ----------------------------------------------------------
def rooms_csr(rooms):
    """(room_start int32 [R+1], members int32 [M]) of a list of index arrays, one per room."""
    sizes = [len(r) for r in rooms]
    room_start = np.zeros(len(rooms) + 1, np.int32)
    room_start[1:] = np.cumsum(sizes, dtype=np.int64)
    members = np.concatenate([np.asarray(r, np.int32).ravel() for r in rooms]) if rooms else np.zeros(0, np.int32)
    return room_start, np.ascontiguousarray(members, np.int32)


def mix(pcm, level, flags, rooms, k, out=None):
    """Mix-minus of each room's up-to-k loudest talkers: pcm int16 [n, spp] (the decoder's rows), level / flags uint8 [n]
    (DecoderBatch.activity()), rooms = a list of index arrays -> (out int16 [n, spp], talkers int32 [R, k]).  Rows of streams
    in no room keep what `out` held (zeros when it is None).  Raises SoloError, with `out` untouched, for a bad argument,
    a member outside [0, n) or a stream listed twice."""
    pcm = np.ascontiguousarray(pcm, np.int16)
    n, spp = pcm.shape
    level = np.ascontiguousarray(level, np.uint8)
    flags = np.ascontiguousarray(flags, np.uint8)
    if level.shape != (n,) or flags.shape != (n,):
        raise SoloError("mix: level and flags must be uint8 [%d]" % n)
    if out is None:
        out = np.zeros((n, spp), np.int16)
    if out.shape != (n, spp) or out.dtype != np.int16 or not out.flags.c_contiguous:
        raise SoloError("mix: out must be a C-contiguous int16 [%d, %d] array" % (n, spp))
    room_start, members = rooms_csr(rooms)
    talkers = np.empty((len(rooms), max(int(k), 0)), np.int32)
    r = lib().solo_b200_mix_host(pcm.ctypes.data, out.ctypes.data, spp, n, level.ctypes.data, flags.ctypes.data,
                                 room_start.ctypes.data, members.ctypes.data, len(rooms), int(k), talkers.ctypes.data)
    if r:
        raise SoloError("mix failed (%d): %s" % (r, _err()))
    return out, talkers


def mix_contributors(rooms, talkers, level, n):
    """Every downlink's CSRC list and RFC 6465 levels: rooms = a list of index arrays, talkers int32 [R, k] (what mix
    returns), level uint8 [n] -> (csrc int32 [n, k], csrc_level uint8 [n, k]).  Member i of room r lists r's talkers
    except i, loudest first, padded with -1 / 127; rows of streams in no room are all -1 / 127 (see
    solo_b200_mix_contributors_host).  Raises SoloError for a bad argument, a member outside [0, n) or a stream listed
    twice."""
    talkers = np.ascontiguousarray(talkers, np.int32)
    if talkers.ndim != 2 or talkers.shape[0] != len(rooms):
        raise SoloError("mix_contributors: talkers must be int32 [%d, k]" % len(rooms))
    level = np.ascontiguousarray(level, np.uint8)
    if level.shape != (int(n),):
        raise SoloError("mix_contributors: level must be uint8 [%d]" % int(n))
    k = talkers.shape[1]
    room_start, members = rooms_csr(rooms)
    csrc = np.empty((int(n), k), np.int32)
    csrc_level = np.empty((int(n), k), np.uint8)
    r = lib().solo_b200_mix_contributors_host(room_start.ctypes.data, members.ctypes.data, len(rooms), k, talkers.ctypes.data,
                                              level.ctypes.data, int(n), csrc.ctypes.data, csrc_level.ctypes.data)
    if r:
        raise SoloError("mix_contributors failed (%d): %s" % (r, _err()))
    return csrc, csrc_level


def mix_contributors_device(d_room_start, d_members, n_rooms, k, d_talkers, d_level, n, d_csrc, d_csrc_level, stream=0):
    """The same on device arrays (addresses): enqueued on `stream`; contents are not checked."""
    r = lib().solo_b200_mix_contributors_device(d_room_start, d_members, int(n_rooms), int(k), d_talkers, d_level, int(n),
                                                d_csrc, d_csrc_level, stream)
    if r:
        raise SoloError("mix_contributors_device failed (%d): %s" % (r, _err()))


def mix_device(d_in, d_out, spp, n, d_level, d_flags, d_room_start, d_members, n_rooms, k, d_talkers, stream=0):
    """The same on device arrays (addresses): enqueued on `stream`; contents are not checked (see solo_b200_mix_device)."""
    r = lib().solo_b200_mix_device(d_in, d_out, int(spp), int(n), d_level, d_flags, d_room_start, d_members, int(n_rooms),
                                   int(k), d_talkers, stream)
    if r:
        raise SoloError("mix_device failed (%d): %s" % (r, _err()))


# ---- receive queue (include/solo_b200.h, solo_b200_rx_*) --------------------------------------------------------------
RX_COUNTERS = ("stored", "duplicate", "late", "dropped", "malformed", "played_both", "played_one", "played_none")


class RxQueue:
    """Receive queue of N streams on one GPU: holds each packet's two descriptions as they arrive (early, out of order,
    twice), pairs them and hands the decoder one row per stream and tick (see solo_b200_rx_* in include/solo_b200.h)."""

    def __init__(self, n, depth=8, desc_cap=128, device=0):
        self.n, self.depth, self.desc_cap = int(n), int(depth), int(desc_cap)
        self.h = lib().solo_b200_rx_create(self.n, self.depth, self.desc_cap, int(device))
        if not self.h:
            raise SoloError("solo_b200_rx_create failed: " + _err())

    def enable_timing(self, ts_per_index, max_arrivals):
        """Keep per-stream arrival timing from now on (RFC 3550 jitter, extended highest index, valid arrivals and the
        playout-margin histogram; see solo_b200_rx_enable_timing): ts_per_index RTP timestamp units per packet index,
        at most max_arrivals arrivals per timed insert."""
        r = lib().solo_b200_rx_enable_timing(self.h, int(ts_per_index), int(max_arrivals))
        if r:
            raise SoloError("rx_enable_timing failed (%d): %s" % (r, _err()))

    def insert(self, streams, index, desc, payloads, arrival=None):
        """Arrival a is description desc[a] (1 or 2) of packet index[a] of stream streams[a], bytes payloads[a]; the
        payloads are laid out back to back for the call.  arrival (uint32 receive times in RTP timestamp units, one
        per arrival) makes it a timed insert, which needs enable_timing first; None is the untimed insert."""
        streams = np.ascontiguousarray(streams, np.int32)
        index = np.ascontiguousarray(np.asarray(index, np.int64) & 0xFFFFFFFF, np.uint32)
        desc = np.ascontiguousarray(desc, np.uint8)
        lens = np.array([len(p) for p in payloads], np.int32)
        off = np.zeros(len(lens), np.int32)
        if len(lens):
            off[1:] = np.cumsum(lens[:-1], dtype=np.int64)
        flat = np.frombuffer(b"".join(bytes(p) for p in payloads), np.uint8).copy()
        if not (len(streams) == len(index) == len(desc) == len(lens)):
            raise SoloError("RxQueue.insert: streams, index, desc and payloads differ in length")
        if arrival is None:
            r = lib().solo_b200_rx_insert_host(self.h, streams.ctypes.data, index.ctypes.data, desc.ctypes.data,
                                               off.ctypes.data, lens.ctypes.data, len(streams), flat.ctypes.data, flat.size)
            if r:
                raise SoloError("rx_insert_host failed (%d): %s" % (r, _err()))
            return
        arrival = np.ascontiguousarray(np.asarray(arrival, np.int64) & 0xFFFFFFFF, np.uint32)
        if arrival.shape != (len(streams),):
            raise SoloError("RxQueue.insert: arrival must have one entry per arrival")
        r = lib().solo_b200_rx_insert_timed_host(self.h, streams.ctypes.data, index.ctypes.data, desc.ctypes.data,
                                                 off.ctypes.data, lens.ctypes.data, arrival.ctypes.data, len(streams),
                                                 flat.ctypes.data, flat.size)
        if r:
            raise SoloError("rx_insert_timed_host failed (%d): %s" % (r, _err()))

    def insert_device(self, d_stream, d_index, d_desc, d_off, d_len, n_arrivals, d_payload, payload_bytes, stream=0,
                      d_arrival=None):
        """insert on device arrays (addresses), enqueued on `stream`: three kernel launches, none for n_arrivals = 0.
        d_arrival (uint32 receive times) makes it a timed insert: 2 + 3 * ceil(log2(N) / 8) launches more."""
        if d_arrival is None:
            r = lib().solo_b200_rx_insert_device(self.h, d_stream, d_index, d_desc, d_off, d_len, int(n_arrivals), d_payload,
                                                 int(payload_bytes), stream)
            if r:
                raise SoloError("rx_insert_device failed (%d): %s" % (r, _err()))
            return
        r = lib().solo_b200_rx_insert_timed_device(self.h, d_stream, d_index, d_desc, d_off, d_len, d_arrival,
                                                   int(n_arrivals), d_payload, int(payload_bytes), stream)
        if r:
            raise SoloError("rx_insert_timed_device failed (%d): %s" % (r, _err()))

    def pull(self, play=None, cap=256):
        """One tick: -> (bits uint8 [N, cap], nbytes int16 [N, 2], lostflag int32 [N]) of packet play[s] (None: each
        stream's last + 1), ready for DecoderBatch.decode.  Row bytes after nbytes[s, 0] are zero."""
        p = None
        if play is not None:
            p = np.ascontiguousarray(np.asarray(play, np.int64) & 0xFFFFFFFF, np.uint32)
            if p.shape != (self.n,):
                raise SoloError("RxQueue.pull: play must have %d entries" % self.n)
        bits = np.zeros((self.n, int(cap)), np.uint8)
        nbytes = np.zeros((self.n, 2), np.int16)
        lostflag = np.zeros(self.n, np.int32)
        r = lib().solo_b200_rx_pull_host(self.h, p.ctypes.data if p is not None else None, bits.ctypes.data, int(cap),
                                         nbytes.ctypes.data, lostflag.ctypes.data)
        if r:
            raise SoloError("rx_pull_host failed (%d): %s" % (r, _err()))
        return bits, nbytes, lostflag

    def pull_device(self, d_play, d_bits, cap, d_nbytes, d_lostflag, stream=0):
        """pull on device arrays (d_play = 0 for last + 1), enqueued on `stream`: one kernel launch."""
        r = lib().solo_b200_rx_pull_device(self.h, d_play or None, d_bits, int(cap), d_nbytes, d_lostflag, stream)
        if r:
            raise SoloError("rx_pull_device failed (%d): %s" % (r, _err()))

    def reset(self, streams, start, stream=0):
        """Empty the listed streams' slots, zero their counters, and play packet start[i] next on stream streams[i]."""
        _queue_reset(lib().solo_b200_rx_reset, "rx_reset", self.h, streams, start, stream)

    def stats(self, stream=0):
        """(counters uint32 [N, 8] in the order of RX_COUNTERS, arrivals for streams outside [0, N))."""
        cnt = np.zeros((self.n, 8), np.uint32)
        bad = C.c_uint64()
        r = lib().solo_b200_rx_stats(self.h, cnt.ctypes.data, C.byref(bad), stream)
        if r:
            raise SoloError("rx_stats failed (%d): %s" % (r, _err()))
        return cnt, int(bad.value)

    def timing(self, stream=0):
        """(jitter uint32 [N] in RTP timestamp units (RFC 3550: the kept value >> 4), highest uint64 [N] (cycles << 32 |
        index), received uint32 [N], margin uint32 [N, 8]) of a timed queue."""
        jitter, received = np.zeros(self.n, np.uint32), np.zeros(self.n, np.uint32)
        highest, margin = np.zeros(self.n, np.uint64), np.zeros((self.n, 8), np.uint32)
        r = lib().solo_b200_rx_timing(self.h, jitter.ctypes.data, highest.ctypes.data, received.ctypes.data,
                                      margin.ctypes.data, stream)
        if r:
            raise SoloError("rx_timing failed (%d): %s" % (r, _err()))
        return jitter, highest, received, margin

    def close(self):
        if getattr(self, "h", None):
            lib().solo_b200_rx_destroy(self.h)
            self.h = None

    __del__ = close


# ---- send queue (include/solo_b200.h, solo_b200_tx_*) -----------------------------------------------------------------
TX_COUNTERS = ("sent", "octets", "dtx", "bad")


class TxQueue:
    """Send queue of N streams on one GPU: turns each wave of encoded rows into numbered datagrams, two per row, packed
    back to back in RxQueue's arrival format (see solo_b200_tx_* in include/solo_b200.h)."""

    def __init__(self, n, device=0):
        self.n = int(n)
        self.h = lib().solo_b200_tx_create(self.n, int(device))
        if not self.h:
            raise SoloError("solo_b200_tx_create failed: " + _err())

    def pack(self, bits, nbytes):
        """bits uint8 [N, cap], nbytes int16 [N, 2] (an encoder wave) -> (payload uint8 [total], stream int32, index uint32,
        desc uint8, off int32, len int32 [count])."""
        bits = np.ascontiguousarray(bits, np.uint8)
        nbytes = np.ascontiguousarray(nbytes, np.int16)
        if bits.ndim != 2 or bits.shape[0] != self.n or nbytes.shape != (self.n, 2):
            raise SoloError("TxQueue.pack: bits must be [%d, cap] and nbytes [%d, 2]" % (self.n, self.n))
        cap = bits.shape[1]
        payload = np.empty(self.n * cap, np.uint8)
        e = 2 * self.n
        stream, index, desc = np.empty(e, np.int32), np.empty(e, np.uint32), np.empty(e, np.uint8)
        off, lens = np.empty(e, np.int32), np.empty(e, np.int32)
        total = C.c_int64()
        c = lib().solo_b200_tx_pack_host(self.h, bits.ctypes.data, cap, nbytes.ctypes.data, payload.ctypes.data, payload.size,
                                         stream.ctypes.data, index.ctypes.data, desc.ctypes.data, off.ctypes.data,
                                         lens.ctypes.data, C.byref(total))
        if c < 0:
            raise SoloError("tx_pack_host failed (%d): %s" % (c, _err()))
        return payload[:total.value], stream[:c], index[:c], desc[:c], off[:c], lens[:c]

    def pack_device(self, d_bits, cap, d_nbytes, d_payload, payload_cap, d_stream, d_index, d_desc, d_off, d_len, d_count,
                    d_total, stream=0):
        """pack on device arrays (addresses), enqueued on `stream`: three kernel launches.  d_count int32 [1] and d_total
        int64 [1] receive the datagram count and byte total."""
        r = lib().solo_b200_tx_pack_device(self.h, d_bits, int(cap), d_nbytes, d_payload, int(payload_cap), d_stream, d_index,
                                           d_desc, d_off, d_len, d_count, d_total, stream)
        if r:
            raise SoloError("tx_pack_device failed (%d): %s" % (r, _err()))

    def reset(self, streams, start, stream=0):
        """Give the listed streams' next rows index start[i] and zero their counters."""
        _queue_reset(lib().solo_b200_tx_reset, "tx_reset", self.h, streams, start, stream)

    def stats(self, stream=0):
        """counters uint32 [N, 4] in the order of TX_COUNTERS."""
        cnt = np.zeros((self.n, 4), np.uint32)
        r = lib().solo_b200_tx_stats(self.h, cnt.ctypes.data, stream)
        if r:
            raise SoloError("tx_stats failed (%d): %s" % (r, _err()))
        return cnt

    def close(self):
        if getattr(self, "h", None):
            lib().solo_b200_tx_destroy(self.h)
            self.h = None

    __del__ = close


# ---- G.711 gateway (include/solo_b200.h, solo_b200_g711_*) ------------------------------------------------------------
G711_LAWS = {"pcmu": 0, "pcma": 1}    # SOLO_B200_G711_ULAW / SOLO_B200_G711_ALAW


def _law(v):
    if isinstance(v, str):
        if v not in G711_LAWS:
            raise SoloError("law must be one of %s, not %r" % (sorted(G711_LAWS), v))
        return G711_LAWS[v]
    return v


class G711Gateway:
    """PSTN and SIP participants (G.711 PCMU / PCMA at 8 kHz) in 16 kHz rooms, N streams on one GPU: the uplink turns
    G.711 payloads into 16 kHz rows with level and VAD flags for the mixer, the downlink turns the mixer's rows into G.711
    payloads (see solo_b200_g711_* in include/solo_b200.h)."""

    def __init__(self, n, framesize_ms=40, law="pcmu", device=0):
        self.n, self.framesize_ms = int(n), int(framesize_ms)
        self.spp8, self.spp16 = 8 * self.framesize_ms, 16 * self.framesize_ms
        self.h = lib().solo_b200_g711_create(self.n, self.framesize_ms, int(_law(law)), int(device))
        if not self.h:
            raise SoloError("solo_b200_g711_create failed: " + _err())

    def uplink(self, payload, lost=None):
        """payload uint8 [N, spp8] (G.711 bytes; 160 per 20 ms frame), lost int32 [N] (bit f: frame f did not arrive) or
        None -> (pcm int16 [N, spp16], level uint8 [N], flags uint8 [N]) in the activity reports' format."""
        g = np.ascontiguousarray(payload, np.uint8)
        if g.shape != (self.n, self.spp8):
            raise SoloError("G711Gateway.uplink: payload must be [%d, %d]" % (self.n, self.spp8))
        lo = None
        if lost is not None:
            lo = np.ascontiguousarray(lost, np.int32)
            if lo.shape != (self.n,):
                raise SoloError("G711Gateway.uplink: lost must have %d entries" % self.n)
        pcm = np.zeros((self.n, self.spp16), np.int16)
        level, flags = np.zeros(self.n, np.uint8), np.zeros(self.n, np.uint8)
        r = lib().solo_b200_g711_uplink_host(self.h, g.ctypes.data, None if lo is None else lo.ctypes.data, pcm.ctypes.data,
                                             level.ctypes.data, flags.ctypes.data)
        if r:
            raise SoloError("g711_uplink_host failed (%d): %s" % (r, _err()))
        return pcm, level, flags

    def uplink_device(self, d_payload, d_lost, d_pcm, d_level, d_flags, stream=0):
        """uplink on device arrays (addresses; d_lost = 0 for nothing lost), enqueued on `stream`: two kernel launches."""
        r = lib().solo_b200_g711_uplink_device(self.h, d_payload, d_lost or None, d_pcm, d_level, d_flags, stream)
        if r:
            raise SoloError("g711_uplink_device failed (%d): %s" % (r, _err()))

    def downlink(self, pcm):
        """pcm int16 [N, spp16] (e.g. the mixer's output rows) -> payload uint8 [N, spp8]."""
        x = np.ascontiguousarray(pcm, np.int16)
        if x.shape != (self.n, self.spp16):
            raise SoloError("G711Gateway.downlink: pcm must be [%d, %d]" % (self.n, self.spp16))
        out = np.zeros((self.n, self.spp8), np.uint8)
        r = lib().solo_b200_g711_downlink_host(self.h, x.ctypes.data, out.ctypes.data)
        if r:
            raise SoloError("g711_downlink_host failed (%d): %s" % (r, _err()))
        return out

    def downlink_device(self, d_pcm, d_payload, stream=0):
        """downlink on device arrays (addresses), enqueued on `stream`: one kernel launch."""
        r = lib().solo_b200_g711_downlink_device(self.h, d_pcm, d_payload, stream)
        if r:
            raise SoloError("g711_downlink_device failed (%d): %s" % (r, _err()))

    def reset(self, streams, law=None, stream=0):
        """Make the listed streams fresh streams with `law` ("pcmu" / "pcma", 0 / 1, -1 or None for the create law, or an
        array with one entry per listed stream).  Ordered on `stream`; returns once that stream is done.  Raises
        SoloError, with nothing done, for a stream outside [0, N), one listed twice or a bad law."""
        s, keep = _stream_list(streams), []
        if law is not None and not isinstance(law, str):
            law = [_law(v) for v in np.broadcast_to(np.asarray(law, object), (len(s),))]
        r = lib().solo_b200_g711_reset(self.h, s.ctypes.data, len(s), _settings("g711_reset", _law(law), len(s), keep), stream)
        if r:
            raise SoloError("g711_reset failed (%d): %s" % (r, _err()))

    @staticmethod
    def state_bytes():
        return int(lib().solo_b200_g711_state_bytes())

    def close(self):
        if getattr(self, "h", None):
            lib().solo_b200_g711_destroy(self.h)
            self.h = None

    __del__ = close
