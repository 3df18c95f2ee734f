# TEST INFRASTRUCTURE ONLY. Builds oracle/_ref/libsatref_fengyun.so, the checker of the FengYun-3 AHRPT decoder (fengyun_ahrpt_decoder):
# Viterbi3_4 (fymode) with its CCDecoder / CCEncoder, rotate_soft, FengyunDiff, BPSK_CCSDS_Deframer, the derandomiser and Reed-Solomon,
# compiled unmodified where they lie, + fengyun_harness.cpp (our wiring / C ABI). It uses oracle/Makefile's settings and checker rule:
#   make -C oracle -f fengyun.mk
# Where the reference is absent the prebuilt library is kept and the tests read tests/golden/fengyun_pins.json.
include Makefile

fengyun_SRC := $(addprefix src-core/common/codings/,viterbi/viterbi_3_4.cpp viterbi/cc_decoder.cpp viterbi/cc_encoder.cpp viterbi/utils.cpp \
  rotation.cpp deframing/bpsk_ccsds_deframer.cpp randomization.cpp reedsolomon/reedsolomon.cpp) plugins/fengyun3_support/fengyun3/diff.cpp $(RS_C)
fengyun_CXX := $(CXXFLAGS) -I$(PLUG)/fengyun3_support
fengyun_CC := $(CFLAGS)
$(eval $(call checker,fengyun))

ifneq ($(wildcard $(SRC)),)
fengyun: $(OUT)/libsatref_fengyun.so
else
fengyun:
	@echo "oracle: $(REF) absent - keeping the prebuilt $(OUT)/libsatref_fengyun.so"
endif
.DEFAULT_GOAL := fengyun
.PHONY: fengyun
