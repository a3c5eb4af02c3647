# The reference's two libraries again, each linked with lowband_tap.c and -Wl,--wrap=AGR_Sate_qmf_synth: the decoder's call
# of its synthesis filter bank first records the low band it passes (the parity target of the core-output decoder), then
# runs the real one.  The sources are the untouched reference trees, compiled with the flags of Makefile (included below).
#   libjc1_flp_lowband.so : JC1_SDK_SRC_FLP + the tap (float low band, converted back to int16 exactly)
#   libjc1_fix_lowband.so : JC1_SDK_SRC_ARM + the tap (int16 low band)
#     make -C oracle -f lowband.mk
include Makefile
.DEFAULT_GOAL := lowband

WRAP := -Wl,--wrap=AGR_Sate_qmf_synth

define build_tap
	@mkdir -p $(OUT)
	$(CC) $(CFLAGS) $(3) -I$(1)/interface -I$(1)/src/libBWE -I$(1)/src/libSATECodec \
	    lowband_tap.c $(1)/src/libBWE/*.c $(1)/src/libSATECodec/*.c $(LDFLAGS) $(WRAP) -o $(2)
endef

lowband: $(OUT)/libjc1_flp_lowband.so $(OUT)/libjc1_fix_lowband.so

$(OUT)/libjc1_flp_lowband.so: lowband_tap.c lowband.mk
	$(call build_tap,$(REF)/JC1_SDK_SRC_FLP,$@,-DLOWBAND_FLOAT)

$(OUT)/libjc1_fix_lowband.so: lowband_tap.c lowband.mk
	$(call build_tap,$(REF)/JC1_SDK_SRC_ARM,$@,)

.PHONY: lowband
