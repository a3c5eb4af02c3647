"""Run-time control of a reference encoder handle, for the tests of the encoder's per-packet settings.

The reference SDK sets bitRate, useDTX and packetLossPercentage of its handle once, in AGR_Sate_Encoder_Init
(AGR_BWE_SDK_API.c:38-119), but its SILK core re-reads all three from the handle's encControl at the start of every packet
(SKP_Silk_enc_API.c:161-191).  set_control writes them into a live handle of the unmodified FIX library the way Init does,
so the reference also follows a settings schedule.  Only the leading fields of the handle are described here;
tests/test_enc_control.py checks the description against what the library itself reports."""
import ctypes as C

from oracle import ref


class SilkEncControl(C.Structure):
    # SKP_SILK_SDK_EncControlStruct (interface/SKP_Silk_control.h:41-69): nine ints
    _fields_ = [(n, C.c_int32) for n in ("API_sampleRate", "maxInternalSampleRate", "packetSize", "bitRate", "packetLossPercentage",
                                         "complexity", "useInBandFEC", "useDTX", "useMDIndex")]


class SateEncHead(C.Structure):
    # the leading fields of SATEEncCtl (libBWE/AGR_BWE_structs.h:61-67): SILK state, high-band state, SILK control
    _fields_ = [("stEnc", C.c_void_p), ("stHBEnc", C.c_void_p), ("encControl", SilkEncControl)]


class RefEncoder(ref.RefEncoder):
    """oracle.ref.RefEncoder of the FIX build, plus set_control."""

    def __init__(self, **kw):
        super().__init__("fix", **kw)

    def head(self):
        return C.cast(C.c_void_p(self.h), C.POINTER(SateEncHead)).contents

    def set_control(self, rate=None, dtx=None, loss=None):
        """From the next packet on: target rate (b/s, less 1600 -- or 800 with joint mode 1 -- as Init computes bitRate,
        AGR_BWE_SDK_API.c:118), useDTX, packetLossPercentage.  None leaves a field as it is."""
        c = self.head().encControl
        if rate is not None:
            c.bitRate = int(rate) - (800 if self.ctrl.joint_enable and self.ctrl.joint_mode == 1 else 1600)
        if dtx is not None:
            c.useDTX = int(dtx)
        if loss is not None:
            c.packetLossPercentage = int(loss)
