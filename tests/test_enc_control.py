"""Encoder settings changed between packets -- target rate, DTX and expected packet loss per stream (enc_set_control) --
on the CPU: the host model of the kernel source (tests/hostsim) against the unmodified FIX reference fed the same settings
schedule through its handle (oracle.ref.RefEncoder.set_control).  Bar: payloads and both length fields byte-identical."""
import numpy as np
import pytest

from tests.parity import ref, sim  # noqa: F401  (fixtures)
from tests.util import load_clip, signal_classes

MODES = {"40ms": dict(), "20ms": dict(framesize_ms=20), "joint1": dict(joint_hb=1)}
P = 48                      # packets per schedule
SILENCE = (12, 26)          # packets [12, 26) of every input are silent, so DTX is switched while there is nothing to code


def inputs(spp):
    """(name, int16 signal of P packets): the speech clip and the eight signal classes of the hetero batch tests, each with
    the silent stretch SILENCE."""
    clip = load_clip()
    rows = signal_classes(clip, 8, (P * spp + 639) // 640).transpose(1, 0, 2).reshape(8, -1)[:, :P * spp]
    names = ["noise2000", "noise20000", "zeros", "dc1000", "square", "sine200", "clip4x"]
    out = [("speech", clip[:P * spp].copy())] + [(n, rows[k + 1].copy()) for k, n in enumerate(names)] + [("speech_off", rows[0].copy())]
    for _, x in out:
        x[SILENCE[0] * spp:SILENCE[1] * spp] = 0
    return out


def schedule(seed):
    """Per packet, the settings to change before it ({} = no call).  Rates are log-uniform in [3 000, 120 000] b/s and
    reach both clamps, loss is uniform in 0-100, DTX is switched on at the start of the silence and toggled inside it."""
    rng = np.random.Generator(np.random.PCG64(seed))
    out = [{} for _ in range(P)]
    for p in range(P):
        if p == 0 or rng.random() < 0.3:
            out[p]["rate"] = int(np.exp(rng.uniform(np.log(3000), np.log(120000))))
        if rng.random() < 0.3:
            out[p]["loss"] = int(rng.integers(0, 101))
    out[5]["rate"], out[9]["rate"] = 3000, 120000                   # below and above the SILK core's [5000, 100000]
    for p, v in ((SILENCE[0], 1), (17, 0), (20, 1), (24, 0), (30, 1)):
        out[p]["dtx"] = v
    return out


def run(enc, x, sched, without=()):
    spp = enc.samples
    pk = []
    for p in range(P):
        c = {k: v for k, v in sched[p].items() if k not in without}
        if c:
            enc.set_control(**c)
        b, nb, n = enc.encode(x[p * spp:(p + 1) * spp])
        pk.append((b[:max(n, 0)], nb, n))
    enc.close()
    return pk


@pytest.mark.parametrize("mode", list(MODES))
def test_random_schedules_match_the_reference(sim, ref, mode):
    kw = MODES[mode]
    spp = 16 * kw.get("framesize_ms", 40)
    moved_by_loss = zero_length = 0
    size_by_rate = []
    for i, (name, x) in enumerate(inputs(spp)):
        sched = schedule(1000 * i + len(mode))
        want = run(ref.RefEncoder(**kw), x, sched)
        got = run(sim.SimEncoder(**kw), x, sched)
        for p in range(P):
            assert got[p] == want[p], (mode, name, p, sched[p])
        # the schedule did something: loss changes packets against loss 0, DTX drops packets, rate moves payload sizes
        moved_by_loss += sum(a != b for a, b in zip(want, run(ref.RefEncoder(**kw), x, sched, without=("loss",))))
        zero_length += sum(nb[0] == 0 for _, nb, _ in want)
        rate = None
        for p in range(P):
            rate = sched[p].get("rate", rate)
            if want[p][1][0] > 0 and name.startswith("speech"):
                size_by_rate.append((rate, want[p][1][0]))
    assert moved_by_loss > 0 and zero_length > 0, (moved_by_loss, zero_length)
    r, n = np.array(size_by_rate).T
    assert n[r >= 40000].mean() > 1.5 * n[r <= 10000].mean(), (n[r >= 40000].mean(), n[r <= 10000].mean())


def test_reference_handle_layout(ref):
    """The handle fields set_control writes are where the library keeps them: the SILK control block reads back what Init
    put there, and after one packet the SILK core reports the written rate (clamped), loss and DTX as its own state."""
    import ctypes as C
    for kw, sub in ((dict(), 1600), (dict(joint_hb=1), 800), (dict(framesize_ms=20), 1600)):
        e = ref.RefEncoder(rate=13600, dtx=1, use_md_index=1, **kw)
        c = e.head().encControl
        assert (c.API_sampleRate, c.maxInternalSampleRate, c.bitRate, c.packetLossPercentage, c.complexity, c.useInBandFEC,
                c.useDTX, c.useMDIndex) == (8000, 8000, 13600 - sub, 0, 2, 0, 1, 1)
        assert c.packetSize == 8 * kw.get("framesize_ms", 40)
        q = ref.SilkEncControl()
        e.L.SKP_Silk_SDK_QueryEncoder.argtypes = [C.c_void_p, C.c_void_p]
        for rate, dtx, loss, want_rate in ((30000, 0, 37, 30000 - sub), (3000, 1, 100, 5000), (150000, 0, 0, 100000)):
            e.set_control(rate=rate, dtx=dtx, loss=loss)
            e.encode(np.zeros(e.samples, np.int16))
            e.L.SKP_Silk_SDK_QueryEncoder(e.head().stEnc, C.byref(q))
            assert (q.bitRate, q.packetLossPercentage, q.useDTX) == (want_rate, loss, dtx), kw
        e.close()
    with pytest.raises(ValueError):                     # the FLP build's layout is not described
        ref.RefEncoder("flp").set_control(rate=13600)


def test_loss_schedule_through_the_32_lane_analysis(sim, ref):
    """The warp kernel's call of ltp_scale_ctrl (sb_coop.cuh) reads the stream's expected loss from the state it stages in
    shared memory: the emulated-lane build follows a loss schedule bit-exactly, and the schedule changes packets."""
    clip = load_clip()
    x = clip[640 * 10:640 * (10 + P)]
    sched = [{} for _ in range(P)]
    for p, v in ((0, 0), (6, 20), (14, 100), (22, 5), (30, 50), (38, 0), (42, 75)):
        sched[p]["loss"] = v
    want = run(ref.RefEncoder(), x, sched)
    got = run(sim.SimEncoder(emu=True), x, sched)
    assert sim.lib(True).hs_is_emu() == 1
    assert got == want
    assert sum(a != b for a, b in zip(want, run(ref.RefEncoder(), x, sched, without=("loss",)))) > 0


@pytest.mark.parametrize("mode", list(MODES))
def test_set_control_before_the_first_packet_equals_init(sim, ref, mode):
    """Create with rate A, then set_control(B) before packet 0: the same packets as the reference created with B -- for
    the rate, for DTX and for both."""
    kw = MODES[mode]
    spp = 16 * kw.get("framesize_ms", 40)
    x = dict(inputs(spp))["speech"]
    first = [{} for _ in range(P)]
    for a, b in (((13600, 0), (24000, 0)), ((13600, 0), (13600, 1)), ((30000, 1), (7000, 0))):
        first[0] = {"rate": b[0], "dtx": b[1]}
        got = run(sim.SimEncoder(rate=a[0], dtx=a[1], **kw), x, first)
        want = run(ref.RefEncoder(rate=b[0], dtx=b[1], **kw), x, [{}] * P)
        assert got == want, (mode, a, b)
        assert got != run(sim.SimEncoder(rate=a[0], dtx=a[1], **kw), x, [{}] * P)     # the call mattered


def test_current_values_and_out_of_range_values_change_nothing(sim, ref):
    """Writing the settings a stream already has before every packet is byte-identical to never calling, in the host model
    and in the reference.  Values outside rate >= 1, dtx 0 / 1, loss 0-100 -- which the device call leaves alone -- do
    not change the stream either."""
    x = dict(inputs(640))["speech"]
    plain = run(ref.RefEncoder(rate=13600, dtx=1), x, [{}] * P)
    same = [{"rate": 13600, "dtx": 1, "loss": 0}] * P
    assert run(ref.RefEncoder(rate=13600, dtx=1), x, same) == plain
    assert run(sim.SimEncoder(rate=13600, dtx=1), x, same) == plain
    bad = [{"rate": r, "dtx": d, "loss": l} for r, d, l in ((0, 2, 101), (-5, -2, -3), (-1, 7, 1000))] * (P // 3)
    assert run(sim.SimEncoder(rate=13600, dtx=1), x, bad) == plain
