// The host model (hostsim.cpp) plus the per-packet control of a stream: the body of the device's control kernel,
// sb::enc_set_control, on the host model's state.  TEST INFRASTRUCTURE ONLY, built on first use by enc_control.py
// (with -DSB_EMU for the emulated-lane build of the analysis stage).
#include "hostsim.cpp"

// rate (b/s), DTX, expected loss (%) from the next packet on; -1 or any other out-of-range value leaves a setting alone
extern "C" void hs_enc_set_control(void* p, int rate, int dtx, int loss) { sb::enc_set_control(&((HsEnc*)p)->st, rate, dtx, loss); }
