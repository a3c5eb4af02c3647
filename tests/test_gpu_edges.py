"""Near-silence end to end, and device configurations no other batched test runs.

Real calls spend much of their time in near-silence: a quiet room's noise floor of a few LSB, a +-1 DC offset, clicks.
That input drives Burg's small-energy arithmetic with non-zero data, the VAD and the gain quantiser at the bottom of their
ranges, and DTX with comfort noise.  Here it runs in neighbouring streams with speech, in an odd-sized batch, through
encode_device / decode_device with DTX, 20 ms packets, joint mode 1 and use_md_index = 1, under a per-stream loss process
with bursts of 10 or more packets.  Every row is compared with the unmodified reference given the same configuration:
payloads byte-exact, PCM 0 LSB.  A CPU test runs the same class through the host model of the kernels.

Batched encodes with a cap below the packet size check the kernels' cap guards: bytes [0, min(cap, total)) of each row
equal the reference's, the length fields describe the whole packet, and nothing is written outside the row."""
import numpy as np
import pytest

from tests.parity import DevicePath, RefRows, lockstep, ref, ref_and_model, sb, sim  # noqa: F401  (fixtures)
from tests.util import load_clip, loss_with_bursts, near_silent_classes


def test_host_model_near_silence_matches_reference(sim, ref):
    T, N = 40, 16
    x = near_silent_classes(load_clip(), N, T)
    flags = loss_with_bursts(T, N)
    for s in range(N):
        kw = dict(dtx=1) if s % 2 else dict(use_md_index=1)
        lockstep(*ref_and_model(ref, sim, **kw), x[:, s], flags[s], tag=(s, s % 8))


def run_device_against_reference(sb, ref, x, **cfg):
    """x: [T, N, samples].  encode_device / decode_device vs one reference encoder + decoder per row; the device decoder
    gets the host-trimmed payloads and a DTX row as a lost packet, exactly as the reference decoder does.  Returns the
    number of (row, packet) pairs that DTX dropped."""
    T, N, _ = x.shape
    eb = sb.EncoderBatch(N, **cfg)
    db = sb.DecoderBatch(N, **{k: v for k, v in cfg.items() if k not in ("rate", "dtx")})
    dp, rr = DevicePath(sb, eb, db, cap=256), RefRows(ref, range(N), decode="ref", **cfg)
    flags = loss_with_bursts(T, N)
    for p in range(T):
        dp.encode(x[p])
        bits, nb, _ = dp.rows()
        rx = rr.step(x[p], bits, nb, flags[:, p])
        dp.decode(rx[2], rx)
        rr.check_pcm(dp.rows()[2])
    rr.close()
    eb.close(); db.close()
    return rr.dtx_rows


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", [
    dict(dtx=1),
    dict(dtx=1, use_md_index=1, framesize_ms=20),
    dict(dtx=1, joint_hb=1),
    dict(use_md_index=1),
], ids=["40ms_dtx", "20ms_dtx_mdi", "joint1_dtx", "40ms_mdi"])
def test_near_silence_next_to_speech_on_the_device(sb, ref, cfg):
    S = 16 * cfg.get("framesize_ms", 40)
    x = near_silent_classes(load_clip(), 37, 60, samples=S)
    dtx_rows = run_device_against_reference(sb, ref, x, **cfg)
    if cfg.get("dtx"):
        assert dtx_rows > 0, "no stream entered DTX: the near-silent rows did not reach comfort-noise coding"


def _cap_inputs(N, T, seed=21):
    clip = load_clip()
    x = near_silent_classes(clip, N, T, seed=seed)
    # loud, noisy rows produce the largest packets at high rates
    rng = np.random.Generator(np.random.PCG64(seed))
    for s in range(0, N, 3):
        x[:, s] = np.clip(rng.normal(0, 12000, (T, 640)), -32768, 32767).astype(np.int16)
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["host", "device"])
def test_batched_encode_below_the_packet_size(sb, ref, entry):
    import torch
    N, T = 29, 6
    rates = np.array([6000, 10000, 13600, 24000, 40000, 64000, 100000] * 5)[:N]
    dtx = (np.arange(N) % 4 == 3).astype(np.int32)           # every fourth row with DTX (silent classes go quiet)
    x = _cap_inputs(N, T)
    # the largest packet of this input, from the reference
    want = []
    for s in range(N):
        e = ref.RefEncoder("fix", rate=int(rates[s]), dtx=int(dtx[s]))
        want.append([e.encode(x[p, s]) for p in range(T)])
        e.close()
    biggest = max(n for row in want for (_, _, n) in row)
    assert biggest > 64
    assert sum(rnb[0] <= 0 for row in want for (_, rnb, _) in row) > 0, "no DTX row dropped a packet: the DTX case is not run"
    for cap in sorted({16, 17, 31, 64, biggest - 1, biggest}):
        eb = sb.EncoderBatch(N)
        eb.set_control(rate=rates, dtx=dtx)
        dev = torch.device("cuda", 0)
        canary = 0xA5
        for p in range(T):
            if entry == "host":
                bits = np.full((N + 1, cap), canary, np.uint8)      # a canary row after the batch
                nb = np.zeros((N, 2), np.int16)
                eb.encode(x[p], cap=cap, bits=bits[:N], nbytes=nb)
                tail = bits[N]
            else:
                d_bits = torch.full((N + 1, cap), canary, dtype=torch.uint8, device=dev)
                d_nb = torch.zeros((N, 2), dtype=torch.int16, device=dev)
                d_pcm = torch.from_numpy(np.ascontiguousarray(x[p])).to(dev)
                eb.encode_device(d_pcm.data_ptr(), d_bits.data_ptr(), cap, d_nb.data_ptr(), torch.cuda.current_stream().cuda_stream)
                torch.cuda.synchronize()
                bits, nb = d_bits.cpu().numpy(), d_nb.cpu().numpy()
                tail = bits[N]
            assert (tail == canary).all(), ("bytes written past the last row", cap, p)
            for s in range(N):
                b, rnb, n = want[s][p]
                assert tuple(nb[s]) == rnb, ("length fields", cap, p, s)
                k = min(cap, max(n, 0))
                assert bytes(bits[s, :k]) == b[:k], ("payload prefix", cap, p, s)
        eb.close()
