"""The G.711 gateway (solo_b200_g711_*) on the GPU against its host model (tests/hostsim, the host build of sb_g711.cuh),
byte for byte and sample for sample: signal classes, every loss mask, both laws in one batch, batch sizes 1, 33 and 4 099,
more than 500 packets of continuity, the host and device entry points, reset, the argument checks and the launch budget, a
room of SOLO and G.711 participants through the mixer, and the round trip of the speech clip."""
import numpy as np
import pytest

import solo_b200
from tests.hostsim import g711_sim, sim
from tests.test_g711 import ref_compress
from tests.util import load_clip

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


def uplink_payloads(N, npk, spp8, seed):
    """uint8 [npk, N, spp8] by stream class s % 6: the clip's 8 kHz low band (compressed under the stream's law), a sine of
    a stream-dependent frequency across 0-4 kHz, a full-scale square, the codes of silence, random bytes, quiet noise."""
    rng = np.random.Generator(np.random.PCG64(seed))
    clip = load_clip()
    T = npk * spp8
    t = np.arange(T)
    out = np.zeros((N, T), np.uint8)
    for s in range(N):
        law, c = s % 2, s % 6
        if c == 0:
            x = np.resize(np.roll(clip[::2], -997 * s), T)
        elif c == 1:
            x = np.round(20000 * np.sin(2 * np.pi * (50 + 3950 * ((s * 0.37) % 1)) * t / 8000))
        elif c == 2:
            x = np.where((t // (4 + s % 9)) % 2, 32767, -32768)
        elif c == 3:
            x = np.zeros(T)
        elif c == 5:
            x = rng.normal(0, 30, T)
        if c == 4:
            out[s] = rng.integers(0, 256, T)
        else:
            out[s] = ref_compress(law, np.clip(x, -32768, 32767).astype(np.int16))
    return out.reshape(N, npk, spp8).transpose(1, 0, 2).copy()


def downlink_rows(N, npk, spp16, seed):
    """int16 [npk, N, spp16] by class s % 5: the clip, a sine across 0-8 kHz (the QMF transition band included), a
    full-scale square, silence, white noise."""
    rng = np.random.Generator(np.random.PCG64(seed))
    clip = load_clip()
    T = npk * spp16
    t = np.arange(T)
    out = np.zeros((N, T), np.int16)
    for s in range(N):
        c = s % 5
        if c == 0:
            x = np.resize(np.roll(clip, -1999 * s), T)
        elif c == 1:
            x = np.round(25000 * np.sin(2 * np.pi * (8000 * ((s * 0.61) % 1)) * t / 16000))
        elif c == 2:
            x = np.where((t // (3 + s % 7)) % 2, 32767, -32768)
        elif c == 3:
            x = np.zeros(T)
        else:
            x = rng.normal(0, 8000, T)
        out[s] = np.clip(x, -32768, 32767).astype(np.int16)
    return out.reshape(N, npk, spp16).transpose(1, 0, 2).copy()


def loss_masks(N, npk, nf, seed):
    """int32 [npk, N]: every mask of nf frames on every stream over the packets, with bits above nf set at random (they
    mean nothing and must change nothing)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    m = (np.arange(npk)[:, None] + np.arange(N)[None, :]) % (1 << nf)
    return (m | (rng.integers(0, 2, (npk, N)) << 5)).astype(np.int32)


class Dev:
    """A gateway driven through its device entry points with torch buffers on one CUDA stream."""

    def __init__(self, N, fs, mixed_laws=True):
        self.g = solo_b200.G711Gateway(N, fs, "pcmu")
        self.N, self.spp8, self.spp16 = N, 8 * fs, 16 * fs
        self.st = torch.cuda.Stream()
        d = "cuda"
        self.pay = torch.zeros((N, self.spp8), dtype=torch.uint8, device=d)
        self.lost = torch.zeros(N, dtype=torch.int32, device=d)
        self.pcm = torch.zeros((N, self.spp16), dtype=torch.int16, device=d)
        self.level = torch.zeros(N, dtype=torch.uint8, device=d)
        self.flags = torch.zeros(N, dtype=torch.uint8, device=d)
        self.x = torch.zeros((N, self.spp16), dtype=torch.int16, device=d)
        self.out = torch.zeros((N, self.spp8), dtype=torch.uint8, device=d)
        if mixed_laws:
            self.g.reset(np.arange(1, N, 2), "pcma", stream=self.st.cuda_stream)

    def uplink(self, pay, lost):
        with torch.cuda.stream(self.st):
            self.pay.copy_(torch.from_numpy(pay))
            if lost is not None:
                self.lost.copy_(torch.from_numpy(lost))
            self.g.uplink_device(self.pay.data_ptr(), 0 if lost is None else self.lost.data_ptr(), self.pcm.data_ptr(),
                                 self.level.data_ptr(), self.flags.data_ptr(), self.st.cuda_stream)
        self.st.synchronize()
        return self.pcm.cpu().numpy(), self.level.cpu().numpy(), self.flags.cpu().numpy()

    def downlink(self, rows):
        with torch.cuda.stream(self.st):
            self.x.copy_(torch.from_numpy(rows))
            self.g.downlink_device(self.x.data_ptr(), self.out.data_ptr(), self.st.cuda_stream)
        self.st.synchronize()
        return self.out.cpu().numpy()


def model(N, fs, mixed_laws=True):
    m = g711_sim.SimG711(N, fs, 0)
    if mixed_laws:
        m.reset(np.arange(1, N, 2), 1)
    return m


def same(what, got, want):
    if not np.array_equal(got, want):
        bad = np.argwhere(np.asarray(got) != np.asarray(want))
        raise AssertionError("%s differs at %d places, first %s: %r != %r" % (what, len(bad), bad[0].tolist(),
                                                                             got[tuple(bad[0])], want[tuple(bad[0])]))


@pytest.mark.parametrize("N,fs,npk", [(1, 40, 24), (1, 20, 24), (33, 40, 520), (33, 20, 40), (4099, 40, 8), (4099, 20, 8)])
def test_device_equals_host_model(N, fs, npk):
    nf = fs // 20
    pay = uplink_payloads(N, npk, 8 * fs, seed=N + fs)
    rows = downlink_rows(N, npk, 16 * fs, seed=2 * N + fs)
    lost = loss_masks(N, npk, nf, seed=N)
    dev, ref = Dev(N, fs), model(N, fs)
    host = solo_b200.G711Gateway(N, fs, "pcmu") if N == 33 else None      # the host entry points, on the same inputs
    if host is not None:
        host.reset(np.arange(1, N, 2), "pcma")
    seen = set()
    for p in range(npk):
        lp = None if p % 5 == 4 else lost[p]
        got, want = dev.uplink(pay[p], lp), ref.uplink(pay[p], lp)
        for name, a, b in zip(("pcm", "level", "flags"), got, want):
            same("packet %d uplink %s" % (p, name), a, b)
        seen.update(int(f) for f in want[2])
        same("packet %d downlink" % p, dev.downlink(rows[p]), ref.downlink(rows[p]))
        if host is not None:
            for name, a, b in zip(("pcm", "level", "flags"), host.uplink(pay[p], lp), want):
                same("packet %d uplink_host %s" % (p, name), a, b)
            same("packet %d downlink_host" % p, host.downlink(rows[p]), dev.out.cpu().numpy())
    if N > 1:
        # speech and no speech, and concealment, in every frame position
        for f in range(nf):
            assert any(v & (1 << f) for v in seen) and any(v & (4 << f) for v in seen), sorted(seen)


def test_reset_equals_fresh_and_checks():
    N, fs, npk = 40, 40, 30
    pay = uplink_payloads(N, 2 * npk, 320, seed=21)
    rows = downlink_rows(N, 2 * npk, 640, seed=22)
    lost = loss_masks(N, 2 * npk, 2, seed=23)
    dev, ref = Dev(N, fs), model(N, fs)
    for p in range(npk):
        dev.uplink(pay[p], lost[p]), dev.downlink(rows[p])
        ref.uplink(pay[p], lost[p]), ref.downlink(rows[p])
    L0 = solo_b200.kernel_launches()
    st = dev.st.cuda_stream
    for bad in (dict(streams=[0, N]), dict(streams=[-1]), dict(streams=[3, 5, 3]), dict(streams=[1, 2], law=[0, 2]),
                dict(streams=[1], law=[-2])):
        with pytest.raises(solo_b200.SoloError):
            dev.g.reset(bad["streams"], bad.get("law"), stream=st)
    with pytest.raises(solo_b200.SoloError):
        dev.g.uplink_device(dev.pay.data_ptr() + 1, 0, dev.pcm.data_ptr(), dev.level.data_ptr(), dev.flags.data_ptr(), st)
    with pytest.raises(solo_b200.SoloError):
        dev.g.uplink_device(dev.pay.data_ptr(), dev.lost.data_ptr() + 2, dev.pcm.data_ptr(), dev.level.data_ptr(),
                            dev.flags.data_ptr(), st)
    with pytest.raises(solo_b200.SoloError):
        dev.g.downlink_device(dev.x.data_ptr() + 8, dev.out.data_ptr(), st)
    with pytest.raises(solo_b200.SoloError):
        dev.g.downlink_device(dev.x.data_ptr(), dev.out.data_ptr() + 4, st)
    with pytest.raises(solo_b200.SoloError):
        solo_b200.G711Gateway(4, 30)
    with pytest.raises(solo_b200.SoloError):
        solo_b200.G711Gateway(4, 40, 2)
    assert solo_b200.kernel_launches() == L0, "a refused call launched work"
    # reset a few streams to both laws; they must then equal the streams of new gateways with those laws
    streams, laws = np.array([0, 7, 8, 21, 39]), np.array([1, 0, -1, 1, 0])
    dev.g.reset(streams, laws, stream=st)
    assert solo_b200.kernel_launches() == L0 + 1
    ref.reset(streams, np.where(laws == -1, 0, laws))
    fresh = {law: (Dev(N, fs, mixed_laws=False), model(N, fs, mixed_laws=False)) for law in (0, 1)}
    for law, (fd, _) in fresh.items():
        if law == 1:
            fd.g.reset(np.arange(N), "pcma", stream=fd.st.cuda_stream)
    eff = np.where(laws == -1, 0, laws)
    for p in range(npk, 2 * npk):
        L1 = solo_b200.kernel_launches()
        up, dn = dev.uplink(pay[p], lost[p]), dev.downlink(rows[p])
        assert solo_b200.kernel_launches() == L1 + 3, "an uplink is two launches, a downlink one"
        for name, a, b in zip(("pcm", "level", "flags"), up, ref.uplink(pay[p], lost[p])):
            same("packet %d uplink %s after reset" % (p, name), a, b)
        same("packet %d downlink after reset" % p, dn, ref.downlink(rows[p]))
        for law, (fd, _) in fresh.items():
            fu, fdn = fd.uplink(pay[p], lost[p]), fd.downlink(rows[p])
            sel = streams[eff == law]
            for name, a, b in zip(("pcm", "level", "flags"), up, fu):
                same("packet %d reset vs fresh %s" % (p, name), a[sel], b[sel])
            same("packet %d reset vs fresh downlink" % p, dn[sel], fdn[sel])


def test_room_of_solo_and_g711_participants():
    """Three SOLO participants (encoder -> decoder at 16 kHz) and three G.711 ones in one room, k = 2: gateway rows after
    the SOLO rows of the [N][640] matrix, one mix on the device, SOLO downlinks through an encoder batch and G.711
    downlinks through the gateway.  G.711 participant 0 speaks (the clip at full level), participant 1 is louder still but
    loses both frames of every odd packet, participant 2 is silent."""
    Ns, Ng, npk, k, fs = 3, 3, 30, 2, 40
    N = Ns + Ng
    clip = load_clip()
    enc = solo_b200.EncoderBatch(Ns, rate=13600)
    dec = solo_b200.DecoderBatch(Ns)
    down = solo_b200.EncoderBatch(Ns, rate=13600)
    dev = Dev(Ng, fs, mixed_laws=False)
    dev.g.reset([1], "pcma", stream=dev.st.cuda_stream)
    gm = g711_sim.SimG711(Ng, fs, 0)
    gm.reset([1], 1)
    room_start, members = np.array([0, N], np.int32), np.arange(N, dtype=np.int32)[::-1].copy()
    d = "cuda"
    d_in, d_out = torch.zeros((N, 640), dtype=torch.int16, device=d), torch.zeros((N, 640), dtype=torch.int16, device=d)
    d_level, d_flags = torch.zeros(N, dtype=torch.uint8, device=d), torch.zeros(N, dtype=torch.uint8, device=d)
    d_rs, d_mb = torch.from_numpy(room_start).to(d), torch.from_numpy(members).to(d)
    d_tk = torch.zeros(k, dtype=torch.int32, device=d)
    d_lost = torch.zeros(Ng, dtype=torch.int32, device=d)
    d_pay = torch.zeros((Ng, 320), dtype=torch.uint8, device=d)
    d_g711 = torch.zeros((Ng, 320), dtype=torch.uint8, device=d)
    x8 = np.resize(clip[::2], npk * 320).reshape(npk, 320)
    picked, picked_lost = 0, 0
    for p in range(npk):
        x = np.stack([(np.resize(np.roll(clip, -3001 * (s + 1)), 640 * (p + 1))[640 * p:] >> (3 + s)) for s in range(Ns)])
        bits, nb = enc.encode(x.astype(np.int16))
        pcm_s, ret = dec.decode(bits, nb, np.full(Ns, 4, np.int32))
        assert (ret == 0).all()
        lv_s, fl_s = dec.activity()
        pay = np.stack([ref_compress(0, x8[p]), ref_compress(1, np.clip(x8[p].astype(np.int32) * 4, -32768, 32767)),
                        np.full(320, 0xFF)]).astype(np.uint8)
        lost = np.array([0, 3 if p % 2 else 0, 0], np.int32)
        with torch.cuda.stream(dev.st):
            d_in[:Ns].copy_(torch.from_numpy(pcm_s))
            d_level[:Ns].copy_(torch.from_numpy(lv_s))
            d_flags[:Ns].copy_(torch.from_numpy(fl_s))
            d_pay.copy_(torch.from_numpy(pay))
            d_lost.copy_(torch.from_numpy(lost))
            dev.g.uplink_device(d_pay.data_ptr(), d_lost.data_ptr(), d_in[Ns:].data_ptr(), d_level[Ns:].data_ptr(),
                                d_flags[Ns:].data_ptr(), dev.st.cuda_stream)
            solo_b200.mix_device(d_in.data_ptr(), d_out.data_ptr(), 640, N, d_level.data_ptr(), d_flags.data_ptr(),
                                 d_rs.data_ptr(), d_mb.data_ptr(), 1, k, d_tk.data_ptr(), stream=dev.st.cuda_stream)
            dev.g.downlink_device(d_out[Ns:].data_ptr(), d_g711.data_ptr(), dev.st.cuda_stream)
        dev.st.synchronize()
        g_pcm, g_lv, g_fl = gm.uplink(pay, lost)
        same("packet %d gateway rows" % p, d_in[Ns:].cpu().numpy(), g_pcm)
        same("packet %d gateway levels" % p, d_level[Ns:].cpu().numpy(), g_lv)
        same("packet %d gateway flags" % p, d_flags[Ns:].cpu().numpy(), g_fl)
        rows_in = np.concatenate([pcm_s, g_pcm])
        want_out, want_tk = sim.mix_model(rows_in, np.concatenate([lv_s, g_lv]), np.concatenate([fl_s, g_fl]), room_start,
                                          members, k, np.zeros((N, 640), np.int16))
        tk = d_tk.cpu().numpy()
        same("packet %d talkers" % p, tk, want_tk[0])
        same("packet %d mixed rows" % p, d_out.cpu().numpy(), want_out)
        same("packet %d G.711 downlinks" % p, d_g711.cpu().numpy(), gm.downlink(want_out[Ns:]))
        bits_d, nb_d = down.encode(d_out[:Ns].cpu().numpy())
        assert (nb_d[:, 0] > 0).all()
        if Ns in tk:
            picked += 1
            for i in range(N):      # everyone else hears G.711 participant 0
                if i != Ns:
                    others = [j for j in tk if j >= 0 and j != i and j != Ns]
                    assert np.array_equal(want_out[i].astype(np.int32),
                                          np.clip(rows_in[Ns].astype(np.int32) + sum(rows_in[j].astype(np.int32) for j in others),
                                                  -32768, 32767))
        if p % 2 and Ns + 1 in tk:
            picked_lost += 1
    assert picked >= npk // 3, "the speaking PSTN participant was rarely picked (%d of %d packets)" % (picked, npk)
    assert picked_lost == 0, "a participant whose frames were lost was mixed"


def test_round_trip_of_the_clip():
    """Uplink then downlink of the clip's band-limited 8 kHz signal gives it back delayed by the two filter banks: 63
    samples at 16 kHz, 31.5 at 8 kHz.  The SNR against that delay is the host model's and at least 30 dB."""
    clip = load_clip()
    npk = len(clip) // 640
    for law in (0, 1):
        lawname = ("pcmu", "pcma")[law]
        band = solo_b200.G711Gateway(1, 40, lawname)
        codes = np.concatenate([band.downlink(clip[None, 640 * p:640 * (p + 1)]) for p in range(npk)])
        dev, m = solo_b200.G711Gateway(1, 40, lawname), g711_sim.SimG711(1, 40, law)
        got, want = [], []
        for p in range(npk):
            pcm, _, _ = dev.uplink(codes[p:p + 1])
            got.append(dev.downlink(pcm))
            pm, _, _ = m.uplink(codes[p:p + 1])
            want.append(m.downlink(pm))
        same("round trip law %d" % law, np.concatenate(got), np.concatenate(want))
        x = g711_sim.g711_expand(law, codes.ravel()).astype(np.float64)
        y = g711_sim.g711_expand(law, np.concatenate(got).ravel()).astype(np.float64)
        n = len(x)
        F = np.fft.rfftfreq(2 * n)
        xd = np.fft.irfft(np.fft.rfft(x, 2 * n) * np.exp(-2j * np.pi * F * 31.5), 2 * n)[:n]
        snr = 10 * np.log10((xd[100:] ** 2).sum() / ((y[100:] - xd[100:]) ** 2).sum())
        assert snr >= 30.0, snr
