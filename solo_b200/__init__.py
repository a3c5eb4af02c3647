"""solo_b200 -- H100-native batched SOLO speech codec (host-side Python mirror of the C ABI).

The product is ``libsolo_b200.so`` (hand-written sm_90a CUDA behind the reference's C ABI, see
``include/AGR_JC1_SDK_API.h`` and ``include/solo_b200.h``).  This package only binds it with ctypes for tests
and benchmarks; it contains no codec arithmetic and no CPU fallback: importing the binding without the built
library, or creating a codec without a GPU, raises.
"""
from .api import (DecoderBatch, EncoderBatch, SoloDecoder, SoloEncoder, SoloError, kernel_launches, lib, set_chunks,  # noqa: F401
                  profile_enable, profile_read, state_bytes, split_packet, merge_packets, bitfile_pack,
                  bitfile_unpack, apply_loss_device, enable_peer_access)
