"""On-device checks of the pieces around the hot path: pipelining invariance, ragged batch sizes, stream state hand-over
(SURVEY.md 8(f) rank 3) and receiver-side loss trimming for a whole batch on the GPU (rank 1)."""
import numpy as np
import pytest

from tests.parity import DevicePath, RefRows, batch_packets, received, ref, sb  # noqa: F401  (fixtures)
from tests.util import load_clip, load_golden, loss_flags, speech_replay, trim_payload

pytestmark = pytest.mark.gpu


def run_streams(sb, N, T, cap=128, flags=None, rate=13600):
    x = speech_replay(load_clip(), N, T)
    eb, db = sb.EncoderBatch(N, rate=rate), sb.DecoderBatch(N)
    out = []
    for p in range(T):
        bits, nb = eb.encode(x[p], cap=cap)
        f = np.full(N, 4, np.int32) if flags is None else flags[:, p].copy()
        pcm, ret = db.decode(bits, nb, f)
        out.append((bits.copy(), nb.copy(), pcm.copy(), ret.copy()))
    eb.close(); db.close()
    return out


def test_results_do_not_depend_on_the_number_of_pipeline_chunks(sb):
    N, T = 8192 + 64 + 5, 3          # ragged: not a multiple of the chunk granularity, odd (a shadowed lane group in the NSQ kernel)
    ref = None
    for chunks in (1, 2, 3, 8):
        sb.set_chunks(chunks)
        got = run_streams(sb, N, T)
        if ref is None:
            ref = got
            g = load_golden()            # stream 0 of the speech-replay batch reads the clip from offset 0 at gain 1
            for p in range(T):
                n0 = int(g["fix_nbytes"][p, 0])
                assert tuple(got[p][1][0]) == tuple(g["fix_nbytes"][p])
                assert bytes(got[p][0][0, :n0]) == bytes(g["fix_bits"][p, :n0])
        else:
            for a, b in zip(ref, got):
                for u, v in zip(a, b):
                    assert np.array_equal(u, v), chunks
    sb.set_chunks(0)           # back to the defaults


@pytest.mark.parametrize("N", [1, 2, 3, 63, 65])
def test_small_and_odd_batches_match_the_single_stream_result(sb, N):
    T = 4
    got = run_streams(sb, N, T, cap=256)
    x = speech_replay(load_clip(), N, T)
    for s in sorted({0, N // 2, N - 1}):
        e, d = sb.SoloEncoder(rate=13600), sb.SoloDecoder()
        for p in range(T):
            b, nb, n = e.encode(x[p, s])
            assert nb == tuple(got[p][1][s]) and b == bytes(got[p][0][s, :n])
            pcm, r = d.decode(b, nb, 4)
            assert np.array_equal(pcm, got[p][2][s])
        e.close(); d.close()


def test_state_export_import_continues_bit_exactly(sb):
    """A stream leaves one batch (slot 5 of 16) after 6 packets and joins another one (slot 2 of 4, other streams at a
    different point of their lives): its payloads and decoded PCM continue as if nothing had happened."""
    T0, T1, cap = 6, 6, 256
    x = speech_replay(load_clip(), 16, T0 + T1)
    eb, db = sb.EncoderBatch(16), sb.DecoderBatch(16)
    want = []
    for p in range(T0 + T1):
        bits, nb = eb.encode(x[p], cap=cap)
        pcm, ret = db.decode(bits, nb, np.full(16, 4, np.int32))
        want.append((bytes(bits[5, :nb[5, 0]]), tuple(nb[5]), pcm[5].copy()))
        if p == T0 - 1:
            enc_blob, dec_blob = eb.export_state(5), db.export_state(5)
    eb.close(); db.close()
    assert enc_blob.size == sb.lib().solo_b200_enc_state_bytes() and dec_blob.size == sb.lib().solo_b200_dec_state_bytes()
    eb2, db2 = sb.EncoderBatch(4), sb.DecoderBatch(4)
    y = speech_replay(load_clip(), 4, 3, first_packet=40)
    for p in range(3):                                   # the new batch already has a history
        bits, nb = eb2.encode(y[p], cap=cap)
        db2.decode(bits, nb, np.full(4, 4, np.int32))
    eb2.import_state(2, enc_blob); db2.import_state(2, dec_blob)
    for p in range(T0, T0 + T1):
        xin = speech_replay(load_clip(), 4, 1, first_packet=50 + p)[0]
        xin[2] = x[p, 5]
        bits, nb = eb2.encode(xin, cap=cap)
        pcm, ret = db2.decode(bits, nb, np.full(4, 4, np.int32))
        assert (bytes(bits[2, :nb[2, 0]]), tuple(nb[2])) == want[p][:2], p
        assert np.array_equal(pcm[2], want[p][2]), p
    with pytest.raises(sb.SoloError):
        eb2.import_state(7, enc_blob)                    # no such slot
    eb2.close(); db2.close()


def test_loss_trimming_on_device_matches_the_receiver_restatement(sb):
    import torch
    N, cap, T = 4096, 128, 3
    x = speech_replay(load_clip(), N, T)
    eb, db, db_ref = sb.EncoderBatch(N), sb.DecoderBatch(N), sb.DecoderBatch(N)
    flags = np.array([loss_flags(T, 50, seed=1 + s) for s in range(N)], np.int32)
    dev = torch.device("cuda", 0)
    for p in range(T):
        bits, nb = eb.encode(x[p], cap=cap)
        f = flags[:, p].copy()
        # host restatement of dec_main.c:245-307, row by row
        hb, hn = np.zeros((N, cap), np.uint8), np.zeros((N, 2), np.int16)
        for s in range(N):
            pb, pnb = trim_payload(bytes(bits[s, :nb[s, 0]]), nb[s], f[s])
            hb[s, :len(pb)] = np.frombuffer(pb, np.uint8)
            hn[s] = pnb
        want, wret = db_ref.decode(hb, hn, f)
        # the same on the device, feeding the device decode entry point
        d_in, d_nb, d_f = torch.from_numpy(bits).to(dev), torch.from_numpy(nb).to(dev), torch.from_numpy(f).to(dev)
        d_out, d_onb = torch.zeros_like(d_in), torch.zeros_like(d_nb)
        d_pcm, d_ret = torch.zeros((N, 640), dtype=torch.int16, device=dev), torch.zeros(N, dtype=torch.int32, device=dev)
        st = torch.cuda.current_stream().cuda_stream
        sb.apply_loss_device(d_in.data_ptr(), d_nb.data_ptr(), d_f.data_ptr(), d_out.data_ptr(), d_onb.data_ptr(), cap, N, st)
        db.decode_device(d_pcm.data_ptr(), d_out.data_ptr(), cap, d_onb.data_ptr(), d_f.data_ptr(), d_ret.data_ptr(), st)
        torch.cuda.synchronize()
        assert np.array_equal(d_onb.cpu().numpy(), hn)
        keep = f != 1
        got_rows, want_rows = d_out.cpu().numpy(), hb
        for s in np.nonzero(keep)[0][:512]:
            assert bytes(got_rows[s, :hn[s, 0]]) == bytes(want_rows[s, :hn[s, 0]])
        assert np.array_equal(d_pcm.cpu().numpy(), want) and np.array_equal(d_ret.cpu().numpy(), wret)
    eb.close(); db.close(); db_ref.close()


def test_config2_batch_4096_streams_50_packets_sampled_against_reference(sb, ref):
    """BASELINE config 2: 4 096 concurrent streams, encode only, 50 packets (2 s).  Every stream runs on the GPU; 64 of
    them (spread over the batch, all four input gains) are replayed through libjc1_fix.so and must match byte for byte."""
    N, T, cap = 4096, 50, 160
    clip = load_clip()
    sample = sorted(set(list(range(0, N, 67)) + [1, 2, 3, N - 1]))[:64]
    eb, rr = sb.EncoderBatch(N, rate=13600), RefRows(ref, sample, rate=13600)
    for p in range(T):
        x = speech_replay(clip, N, 1, first_packet=p)[0]
        bits, nb = eb.encode(x, cap=cap)
        assert (nb[:, 0] <= cap).all()
        rr.step(x[sample], bits[sample], nb[sample])
    rr.close()
    eb.close()


def test_config5_full_batch_with_per_stream_loss_sampled_against_reference(sb, ref):
    """BASELINE configs 3 + 5 at full size: 65 536 streams, encode -> receiver-side trimming on the device -> decode with
    a 50 % loss process per stream (seed 1 + stream id, dec_main.c:229-241); 48 sampled streams against libjc1_fix.so and
    against libjc1_flp.so fed the same payloads and flags (PCM identical; the north star allows +-1 LSB)."""
    N, T, cap = 65536, 8, 128
    clip = load_clip()
    sample = [0, 1, 2, 3] + list(range(997, N, 1489))[:44]
    flags = np.full((N, T), 4, np.int32)
    for s in sample:
        flags[s] = loss_flags(T, 50, seed=1 + s)
    rng = np.random.Generator(np.random.PCG64(7))
    other = rng.integers(1, 5, size=(N, T)).astype(np.int32)       # everybody else: arbitrary flags
    mask = np.ones(N, bool); mask[sample] = False
    flags[mask] = other[mask]
    eb, db = sb.EncoderBatch(N), sb.DecoderBatch(N)
    dp, rr = DevicePath(sb, eb, db, cap=cap), RefRows(ref, sample, decode="gpu")
    for p in range(T):
        x = speech_replay(clip, N, 1, first_packet=p)[0]
        dp.encode(x)
        dp.decode(flags[:, p])
        bits, nb, pcm = dp.rows(sample)
        rr.step(x[sample], bits, nb, flags[sample, p])
        rr.check_pcm(pcm)
    rr.close()
    eb.close(); db.close()


def test_single_stream_small_output_buffer(sb):
    """Same contract through the drop-in ABI on the GPU (the caller's buffer may be smaller than the packet)."""
    g = load_golden()
    clip = load_clip()
    for cap in (64, 9):
        e = sb.SoloEncoder(rate=13600)
        for p in range(6):
            b, nb, n = e.encode(clip[p * 640:(p + 1) * 640], bufsize=cap)
            n0 = int(g["fix_nbytes"][p, 0])
            assert nb == tuple(g["fix_nbytes"][p]) and n == min(cap, n0) and b == bytes(g["fix_bits"][p, :n])
        e.close()


def test_20ms_packets_on_device(sb, ref):
    """framesize_ms = 20 through the batched ABI and the drop-in ABI against the reference (FIX bytes, FLP PCM)."""
    N, T, cap = 130, 40, 128
    clip = load_clip()
    eb, db = sb.EncoderBatch(N, rate=13600, framesize_ms=20), sb.DecoderBatch(N, framesize_ms=20)
    sample = [0, 1, 64, 65, 129]
    rr = RefRows(ref, sample, decode="gpu", rate=13600, framesize_ms=20)
    off = (np.arange(N) * 7919 * 320) % (len(clip) - 320 * (T + 1))
    flags = np.array([loss_flags(T, 40, seed=3 + s) for s in range(N)], np.int32)
    for p in range(T):
        x = np.stack([clip[o + p * 320:o + (p + 1) * 320] for o in off]).astype(np.int16)
        bits, nb = eb.encode(x, cap=cap)
        pcm, ret = db.decode(*received(batch_packets(bits, nb), flags[:, p], cap))
        assert pcm.shape == (N, 320) and (ret == 0).all()
        rr.step(x[sample], bits[sample], nb[sample], flags[sample, p])
        rr.check_pcm(pcm[sample])
    rr.close()
    eb.close(); db.close()
    e, d = sb.SoloEncoder(rate=13600, framesize_ms=20), sb.SoloDecoder(framesize_ms=20)
    r0 = ref.RefEncoder("fix", rate=13600, framesize_ms=20)
    for p in range(10):
        b, nb2, n = e.encode(clip[p * 320:(p + 1) * 320])
        assert (b, nb2, n) == r0.encode(clip[p * 320:(p + 1) * 320])
        y, r = d.decode(b, nb2, 4)
        assert r == 0 and y.size == 320 and d.last_nsamples == 320
    e.close(); d.close()


def test_example_file_codec_reproduces_the_reference_cli_files(sb, tmp_path):
    """examples/jc1_file_codec.c (plain C on the six-function API + framing helpers) writes the same .bit file and the
    same decoded PCM files as the reference's enc_main / dec_main: both descriptions, 50 % loss (seed 1), MD1 only, MD2 only."""
    import hashlib
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = tmp_path / "jc1_file_codec"
    subprocess.check_call(["gcc", "-O2", "-Wall", "-Werror", "-I", os.path.join(root, "include"), os.path.join(root, "examples", "jc1_file_codec.c"),
                           "-L", os.path.join(root, "solo_b200"), "-lsolo_b200", "-Wl,-rpath," + os.path.join(root, "solo_b200"), "-o", str(exe)])
    g = load_golden()
    pcm, bit = tmp_path / "in.pcm", tmp_path / "out.bit"
    load_clip().tofile(pcm)
    subprocess.check_call([str(exe), "enc", str(pcm), str(bit), "13600"])
    assert hashlib.md5(bit.read_bytes()).hexdigest() == str(g["fix_bitfile_md5"])
    for args, key in ((["0", "0"], "flp_pcm_mode4_md5"), (["50", "0"], "flp_pcm_loss50_md5"), (["0", "1"], "flp_pcm_mode2_md5"), (["0", "2"], "flp_pcm_mode3_md5")):
        out = tmp_path / ("out_%s_%s.pcm" % tuple(args))
        subprocess.check_call([str(exe), "dec", str(bit), str(out)] + args)
        assert hashlib.md5(out.read_bytes()).hexdigest() == str(g[key]), key


def test_joint_mode1_on_device(sb, ref):
    """The reference's joint mode 1 through the batched ABI and the drop-in ABI (unsupported modes are refused)."""
    N, T, cap = 67, 20, 192
    x = speech_replay(load_clip(), N, T)
    eb, db = sb.EncoderBatch(N, rate=13600, joint_hb=1), sb.DecoderBatch(N, joint_hb=1)
    sample = [0, 1, 33, 66]
    rr = RefRows(ref, sample, decode="gpu", rate=13600, joint_hb=1)
    flags = np.array([loss_flags(T, 40, seed=11 + s) for s in range(N)], np.int32)
    for p in range(T):
        bits, nb = eb.encode(x[p], cap=cap)
        pcm, ret = db.decode(*received(batch_packets(bits, nb), flags[:, p], cap))
        assert (ret == 0).all()
        rr.step(x[p, sample], bits[sample], nb[sample], flags[sample, p])
        rr.check_pcm(pcm[sample])
    rr.close()
    eb.close(); db.close()
    e = sb.SoloEncoder(rate=13600, joint_enable=1, joint_mode=1)
    b, nb2, n = e.encode(x[0, 0])
    assert (b, nb2, n) == ref.RefEncoder("fix", rate=13600, joint_hb=1).encode(x[0, 0])
    e.close()
    for bad in (dict(joint_enable=1, joint_mode=0), dict(joint_enable=1, joint_mode=2), dict(samplerate=32000), dict(framesize_ms=60)):
        with pytest.raises(sb.SoloError):
            sb.SoloEncoder(**bad)


def test_malformed_payloads_do_not_fault_and_match_the_host_build(sb):
    """Bit-flipped / random / mislabelled payloads on the device: the kernel must survive (a fault would kill the whole
    batch) and, the arithmetic being deterministic, produce exactly what the host build of the same source produces --
    including the reference's 'stale payload' continuation after a corrupted frame terminator."""
    from tests.hostsim import sim
    N, T, cap = 96, 24, 128
    rng = np.random.Generator(np.random.PCG64(21))
    x = speech_replay(load_clip(), N, T)
    eb, db = sb.EncoderBatch(N), sb.DecoderBatch(N)
    hdec = [sim.SimDecoder() for _ in range(N)]
    for p in range(T):
        bits, nb = eb.encode(x[p], cap=cap)
        bits, nb = bits.copy(), nb.copy()
        flags = rng.integers(1, 5, size=N).astype(np.int32)
        for s in range(N):
            kind = int(rng.integers(0, 6))
            n0 = int(nb[s, 0])
            if kind == 1:
                for _ in range(int(rng.integers(1, 4))):
                    bits[s, int(rng.integers(0, n0))] ^= np.uint8(1 << int(rng.integers(0, 8)))
            elif kind == 2:
                bits[s] = rng.integers(0, 256, size=cap).astype(np.uint8)
            elif kind == 3:
                nb[s] = (int(rng.integers(1, cap + 1)), 0)
                nb[s, 1] = int(rng.integers(0, int(nb[s, 0]) + 1))
            elif kind == 4:
                flags[s] = int(rng.integers(-2, 8))
        pcm, ret = db.decode(bits, nb, flags)
        for s in range(N):
            want, r = hdec[s].decode(bytes(bits[s]), (int(nb[s, 0]), int(nb[s, 1])), int(flags[s]))
            assert r == ret[s], (p, s, r, ret[s])
            if r == 0:
                assert np.array_equal(want, pcm[s]), (p, s)
    eb.close(); db.close()


def test_ten_thousand_drop_in_handles_share_the_arena(sb):
    """AGR_Sate_Encoder_Init / Decoder_Init hand out slots of the process-wide arena (segments of 256 streams): 10 000 encoder
    handles come up in well under a second each thousand, occupy 40 segments (not 10 000 batches / 50 000 CUDA streams), still
    produce the golden bitstream, and a released slot is reused."""
    import ctypes as C
    import time
    L = sb.lib()
    L.solo_b200_arena_stats.argtypes = [C.POINTER(C.c_int)]
    st = (C.c_int * 4)()
    L.solo_b200_arena_stats(st)
    seg0, used0 = st[0], st[1]
    g, clip = load_golden(), load_clip()
    t0 = time.perf_counter()
    hs = [sb.SoloEncoder(rate=13600) for _ in range(10000)]
    dt = time.perf_counter() - t0
    L.solo_b200_arena_stats(st)
    assert st[1] - used0 == 10000 and st[0] - seg0 <= 40, list(st)
    assert dt < 10.0, dt                     # ~0.1 ms per handle including the Python wrapper; round 1 needed ~1 ms and 5 CUDA streams each
    for k in (0, 255, 256, 5000, 9999):      # slots of different segments, first packets of the clip
        for p in range(3):
            b, nb, n = hs[k].encode(clip[p * 640:(p + 1) * 640])
            assert nb == tuple(g["fix_nbytes"][p]) and b[:n] == bytes(g["fix_bits"][p, :n]), (k, p)
    for h in hs[:3000]:
        h.close()
    L.solo_b200_arena_stats(st)
    assert st[1] - used0 == 7000
    again = [sb.SoloEncoder(rate=13600) for _ in range(3000)]      # reuses the released slots: no new segment
    L.solo_b200_arena_stats(st)
    assert st[1] - used0 == 10000 and st[0] - seg0 <= 40
    b, nb, n = again[0].encode(clip[:640])                          # a recycled slot starts from a fresh state
    assert nb == tuple(g["fix_nbytes"][0]) and b[:n] == bytes(g["fix_bits"][0, :n])
    for h in hs[3000:] + again:
        h.close()
    d = [sb.SoloDecoder() for _ in range(1000)]
    L.solo_b200_arena_stats(st)
    assert st[3] >= 1000 and st[2] <= 8
    for h in d:
        h.close()
    print("10000 encoder handles in %.3f s" % dt)
