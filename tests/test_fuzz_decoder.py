"""Memory safety of the decoder arithmetic on malformed input: the host build of the kernel source under AddressSanitizer
and UBSan, fed bit-flipped, random, truncated and mislabelled payloads with arbitrary lost flags (tests/hostsim/fuzz_dec.cpp).
A decoder that reads outside its tables on a bad packet would, on the GPU, fault the kernel and take the whole batch down."""
from tests.util import fuzz_decoder


def test_decoder_survives_malformed_packets_under_asan():
    """The 16 kHz decoders, from the host encoder's packets of six signal classes: float 40 ms, 20 ms and joint mode 1, and
    fixed point 40 ms and joint mode 1 (the configurations that arithmetic supports), including rows shorter than the
    declared total.  Every mode both decodes and rejects some of them."""
    counts = fuzz_decoder(1500, 7)
    assert sorted(counts) == ["16k fix 40ms", "16k fix joint", "16k flp 20ms", "16k flp 40ms", "16k flp joint"], counts
    assert all(ok > 0 and bad > 0 and ok + bad == 1500 for ok, bad in counts.values()), counts
