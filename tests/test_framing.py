"""Packet framing around the payload row [MD1 | MD2 | HB] (SURVEY.md 8(f) rank 1): host functions of libsolo_b200.so,
checked against the reference drivers' conventions (enc_main.c:212-234 file records, dec_main.c:245-307 receiver trimming)
as restated in tests/util.py and against the golden bit file.  No GPU needed."""
import hashlib

import numpy as np
import pytest

from tests.parity import sb  # noqa: F401  (fixture)
from tests.util import load_golden, trim_payload


def rows():
    g = load_golden()
    for i in range(g["fix_nbytes"].shape[0]):
        nb = tuple(int(v) for v in g["fix_nbytes"][i])
        yield bytes(g["fix_bits"][i, :nb[0]]), nb


def test_bitfile_records_reproduce_the_reference_bit_file(sb):
    g = load_golden()
    blob = b"".join(sb.bitfile_pack(b, nb) for b, nb in rows())
    assert hashlib.md5(blob).hexdigest() == str(g["fix_bitfile_md5"])
    off, out = 0, []
    while off < len(blob):
        p, nb, off = sb.bitfile_unpack(blob, off)
        out.append((p, nb))
    assert out == list(rows())
    with pytest.raises(sb.SoloError):
        sb.bitfile_unpack(blob[:-1], len(blob) - len(out[-1][0]) - 4)     # truncated last record


def test_split_then_merge_is_what_the_reference_receiver_feeds_its_decoder(sb):
    for b, nb in rows():
        p1, p2 = sb.split_packet(b, nb)
        assert p1 + p2 == b and len(p2) == nb[1] and len(p2) >= 8
        for keep1, keep2, flag in ((1, 1, 4), (1, 0, 2), (0, 1, 3)):
            row, mnb, f = sb.merge_packets(p1 if keep1 else None, p2 if keep2 else None)
            assert f == flag
            want_row, want_nb = trim_payload(b, nb, flag)
            assert (row, mnb) == (want_row, want_nb)
        row, mnb, f = sb.merge_packets(None, None)
        assert f == 1 and mnb[0] > 0            # the decoder rejects nBytes[0] <= 0 even for a lost packet


def test_dtx_row_and_bad_lengths(sb):
    assert sb.split_packet(b"\0" * 8, (0, 0)) == (b"", b"")
    p1, p2 = sb.split_packet(bytes(range(20)), (20, 4))   # 20 ms packets / joint mode 1: description 2 may be just the 4 high-band bytes
    assert p1 == bytes(range(16)) and p2 == bytes(range(16, 20))
    with pytest.raises(sb.SoloError):
        sb.split_packet(b"\0" * 20, (20, 3))        # description 2 always carries the high-band bytes (at least 4)
    with pytest.raises(sb.SoloError):
        sb.split_packet(b"\0" * 20, (20, 30))
    with pytest.raises(sb.SoloError):
        sb.merge_packets(b"\1" * 100, b"\2" * 100, cap=128)
