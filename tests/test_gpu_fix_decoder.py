"""The decoder's fixed-point arithmetic (SOLO_B200_DEC_FIX) on the GPU, at 0 LSB against the reference's fixed-point build
(oracle/_ref/libjc1_fix.so): batched host and device entry points, the drop-in ABI selected by SOLO_B200_DEC_ARITH, the
refusal of 20 ms packets, state hand-over into a float-mode batch, and the example program."""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from tests.parity import DeviceDecoder, DevicePath, batch_packets, received, ref, sb  # noqa: F401  (fixtures)
from tests.util import load_clip, load_golden, loss_flags, signal_classes, speech_replay, trim_payload

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI_MD5 = "149ad62fe193f19d6c80aacc7336ebce"


def load_fixdec():
    return np.load(os.path.join(ROOT, "tests", "golden", "golden_fixdec.npz"))


class RefFixRows:
    """A fixed-point reference decoder per checked row, fed what the batch decoder is fed."""

    def __init__(self, ref, rows, **cfg):
        self.rows = list(rows)
        self.dec = [ref.RefDecoder("fix", **cfg) for _ in self.rows]
        self.pool = ThreadPoolExecutor(32)

    def check(self, tb, tnb, tf, pcm):
        """tb / tnb / tf: the batch's received rows; pcm: its decoded rows, all indexed by batch row."""
        def one(k):
            s = self.rows[k]
            return self.dec[k].decode(bytes(tb[s, :tnb[s, 0]]), tuple(tnb[s]), int(tf[s]))
        want = list(self.pool.map(one, range(len(self.rows))))
        assert all(r == 0 for _, r in want)
        for k, s in enumerate(self.rows):
            assert np.array_equal(pcm[s], want[k][0]), (s, int(np.abs(pcm[s].astype(np.int32) - want[k][0]).max()))

    def close(self):
        for d in self.dec:
            d.close()
        self.pool.shutdown()


@pytest.mark.parametrize("joint", [0, 1])
@pytest.mark.parametrize("signal", ["speech", "classes"])
def test_odd_batch_with_per_stream_loss_matches_fixed_point_reference(sb, ref, joint, signal):
    """N = 257 streams (speech replay, or the eight signal classes in neighbouring streams), each with its own 50 % loss
    process; every row of decode_host and of decode_device against the fixed-point reference."""
    N, cap = 257, 320            # the 200 Hz sine class reaches 205 bytes per packet
    T = 40 if signal == "speech" else 25
    x = speech_replay(load_clip(), N, T) if signal == "speech" else signal_classes(load_clip(), N, T)
    flags = np.array([loss_flags(T, 50, seed=21 + s) for s in range(N)], np.int32)
    eb = sb.EncoderBatch(N, rate=13600, joint_hb=joint)
    dh = sb.DecoderBatch(N, joint_hb=joint, arith="fix")
    dd = sb.DecoderBatch(N, joint_hb=joint, arith="fix")
    rr = RefFixRows(ref, range(N), joint_hb=joint)
    dev = DeviceDecoder(dd, cap)
    for p in range(T):
        bits, nb = eb.encode(x[p], cap=cap)
        tb, tnb, tf = received(batch_packets(bits, nb), flags[:, p], cap)
        pcm, ret = dh.decode(tb, tnb, tf)
        assert (ret == 0).all(), p
        rr.check(tb, tnb, tf, pcm)
        assert np.array_equal(dev.decode(tb, tnb, tf)[0], pcm), p
    rr.close()
    eb.close(); dh.close(); dd.close()


def test_sample_of_a_full_batch_matches_fixed_point_reference(sb, ref):
    """65 536 streams through the device entry points for 4 packets, 20 % loss on the device (apply_loss_device); a
    1 024-row sample against the fixed-point reference."""
    N, T, cap = 65536, 4, 128
    rng = np.random.Generator(np.random.PCG64(7))
    rows = sorted(rng.choice(N, 1024, replace=False).tolist())
    eb, db = sb.EncoderBatch(N, rate=13600), sb.DecoderBatch(N, arith="fix")
    path = DevicePath(sb, eb, db, cap=cap)
    rr = RefFixRows(ref, range(len(rows)))
    flags = np.array([loss_flags(T, 20, seed=1 + s) for s in range(N)], np.int32)
    for p in range(T):
        x = speech_replay(load_clip(), N, 1, first_packet=p)[0]
        path.encode(x)
        path.decode(flags[:, p])
        bits, nb, pcm = path.rows(rows)
        tb, tnb, tf = received(batch_packets(bits, nb), flags[rows, p], cap)
        rr.check(tb, tnb, tf, pcm)
    rr.close()
    eb.close(); db.close()


def test_fixed_point_with_20ms_packets_is_refused(sb):
    with pytest.raises(sb.SoloError) as e:
        sb.DecoderBatch(8, framesize_ms=20, arith="fix")
    assert "20 ms" in str(e.value)
    with pytest.raises(sb.SoloError):
        sb.DecoderBatch(8, arith="fixed")
    d = sb.DecoderBatch(8, framesize_ms=20, arith="flp")
    d.close()


def test_fixed_point_state_continues_in_a_float_batch(sb, ref):
    """A fixed-point stream's blob, exported after 6 packets and imported into a batch created for float decoding, goes on
    decoding as the fixed-point build, bit for bit; the float streams around it stay float."""
    T0, T1, cap = 6, 8, 192
    x = speech_replay(load_clip(), 8, T0 + T1)
    flags = np.array([loss_flags(T0 + T1, 30, seed=4 + s) for s in range(8)], np.int32)
    eb, db = sb.EncoderBatch(8, rate=13600), sb.DecoderBatch(8, arith="fix")
    db2 = sb.DecoderBatch(8, arith="flp")
    fix_ref, flp_ref = ref.RefDecoder("fix"), ref.RefDecoder("flp")
    for p in range(T0 + T1):
        bits, nb = eb.encode(x[p], cap=cap)
        tb, tnb, tf = received(batch_packets(bits, nb), flags[:, p], cap)
        want_fix = fix_ref.decode(bytes(tb[3, :tnb[3, 0]]), tuple(tnb[3]), int(tf[3]))[0]
        if p < T0:
            pcm, ret = db.decode(tb, tnb, tf)
            assert (ret == 0).all() and np.array_equal(pcm[3], want_fix), p
            if p == T0 - 1:
                blob = db.export_state(3)
        else:
            if p == T0:
                db2.import_state(5, blob)
            tb2, tnb2, tf2 = tb.copy(), tnb.copy(), tf.copy()
            tb2[5], tnb2[5], tf2[5] = tb[3], tnb[3], tf[3]
            pcm, ret = db2.decode(tb2, tnb2, tf2)
            assert (ret == 0).all()
            assert np.array_equal(pcm[5], want_fix), p
            want_flp = flp_ref.decode(bytes(tb2[1, :tnb2[1, 0]]), tuple(tnb2[1]), int(tf2[1]))[0]
            assert np.array_equal(pcm[1], want_flp), p    # a neighbour in the float batch stays float
    fix_ref.close(); flp_ref.close()
    eb.close(); db.close(); db2.close()


DROPIN = r"""
import os, sys
sys.path.insert(0, %(root)r)
import numpy as np
import solo_b200 as sb
from oracle import ref
from tests.util import load_golden, loss_flags, trim_payload
g = load_golden()
pk = [(bytes(g["fix_bits"][i, :int(g["fix_nbytes"][i, 0])]), tuple(int(v) for v in g["fix_nbytes"][i])) for i in range(60)]
os.environ["SOLO_B200_DEC_ARITH"] = "fix"
dfix = sb.SoloDecoder()
os.environ["SOLO_B200_DEC_ARITH"] = "flp"
dflp = sb.SoloDecoder()
del os.environ["SOLO_B200_DEC_ARITH"]
ddef = sb.SoloDecoder()
st = (sb.api.C.c_int * 4)()
sb.lib().solo_b200_arena_stats(st)
assert st[2] == 1 and st[3] == 3, list(st)          # one decoder segment holds all three handles
rfix, rflp, rdef = ref.RefDecoder("fix"), ref.RefDecoder("flp"), ref.RefDecoder("flp")
flags = loss_flags(len(pk), 30, seed=8)
for p, ((b, nb), f) in enumerate(zip(pk, flags)):
    pb, pnb = trim_payload(b, nb, f)
    for d, r in ((dfix, rfix), (dflp, rflp), (ddef, rdef)):
        y, ret = d.decode(pb, pnb, f)
        want, rret = r.decode(pb, pnb, f)
        assert ret == rret == 0 and np.array_equal(y, want), p
for bad in ("FIX", "float", ""):
    os.environ["SOLO_B200_DEC_ARITH"] = bad
    try:
        sb.SoloDecoder()
        raise AssertionError("accepted " + repr(bad))
    except sb.SoloError:
        pass
os.environ["SOLO_B200_DEC_ARITH"] = "fix"
try:
    sb.SoloDecoder(framesize_ms=20)
    raise AssertionError("accepted fix with 20 ms")
except sb.SoloError:
    pass
j = sb.SoloDecoder(joint_enable=1, joint_mode=1)
j.close()
for d in (dfix, dflp, ddef):
    d.close()
print("dropin ok")
"""


def test_drop_in_handles_select_the_arithmetic_from_the_environment(sb, ref):
    """In a fresh process (an empty handle arena): a handle made with SOLO_B200_DEC_ARITH=fix, one with "flp" and one with
    the variable unset share one arena segment and each matches its own reference build packet for packet under loss;
    an unknown value and "fix" with 20 ms packets make Init return NULL."""
    p = subprocess.run([sys.executable, "-c", DROPIN % {"root": ROOT}], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert p.returncode == 0 and "dropin ok" in p.stdout, p.stdout[-2000:] + p.stderr[-4000:]


def test_example_file_codec_decodes_like_the_fixed_point_cli(sb, tmp_path):
    """examples/jc1_file_codec.c with SOLO_B200_DEC_ARITH=fix: the clip's .bit file decodes to the reference CLI's md5 at
    loss 0, and to the fixed-point reference's PCM under the driver's 50 % loss process, MD1 only and MD2 only."""
    exe = tmp_path / "jc1_file_codec"
    subprocess.check_call(["gcc", "-O2", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "jc1_file_codec.c"),
                           "-L", os.path.join(ROOT, "solo_b200"), "-lsolo_b200", "-Wl,-rpath," + os.path.join(ROOT, "solo_b200"), "-o", str(exe)])
    f = load_fixdec()
    pcm, bit = tmp_path / "in.pcm", tmp_path / "out.bit"
    load_clip().tofile(pcm)
    subprocess.check_call([str(exe), "enc", str(pcm), str(bit), "13600"])
    assert hashlib.md5(bit.read_bytes()).hexdigest() == str(load_golden()["fix_bitfile_md5"])
    env = dict(os.environ, SOLO_B200_DEC_ARITH="fix")
    for args, key in ((["0", "0"], "fix_pcm_mode4_md5"), (["50", "0"], "fix_pcm_loss50_md5"), (["0", "1"], "fix_pcm_mode2_md5"), (["0", "2"], "fix_pcm_mode3_md5")):
        out = tmp_path / ("out_%s_%s.pcm" % tuple(args))
        subprocess.check_call([str(exe), "dec", str(bit), str(out)] + args, env=env)
        assert hashlib.md5(out.read_bytes()).hexdigest() == str(f[key]), key
        if args == ["0", "0"]:
            assert hashlib.md5(out.read_bytes()).hexdigest() == CLI_MD5
