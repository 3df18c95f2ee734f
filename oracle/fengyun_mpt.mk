# TEST INFRASTRUCTURE ONLY. Builds oracle/_ref/libsatref_fengyun_mpt.so, the checker of the FengYun-3 MPT decoder (fengyun_mpt_decoder):
# Viterbi1_2 with its CCDecoder / CCEncoder, rotate_soft, FengyunDiff, BPSK_CCSDS_Deframer, the derandomiser and Reed-Solomon, compiled
# unmodified where they lie, + fengyun_mpt_harness.cpp (our wiring / C ABI). It uses oracle/Makefile's settings and checker rule:
#   make -C oracle -f fengyun_mpt.mk
# Where the reference is absent the prebuilt library is kept and the tests read tests/golden/fengyun_mpt_pins.json.
include Makefile

fengyun_mpt_SRC := $(addprefix src-core/common/codings/,viterbi/viterbi_1_2.cpp viterbi/cc_decoder.cpp viterbi/cc_encoder.cpp \
  viterbi/utils.cpp rotation.cpp deframing/bpsk_ccsds_deframer.cpp randomization.cpp reedsolomon/reedsolomon.cpp) \
  plugins/fengyun3_support/fengyun3/diff.cpp $(RS_C)
fengyun_mpt_CXX := $(CXXFLAGS) -I$(PLUG)/fengyun3_support
fengyun_mpt_CC := $(CFLAGS)
$(eval $(call checker,fengyun_mpt))

ifneq ($(wildcard $(SRC)),)
fengyun_mpt: $(OUT)/libsatref_fengyun_mpt.so
else
fengyun_mpt:
	@echo "oracle: $(REF) absent - keeping the prebuilt $(OUT)/libsatref_fengyun_mpt.so"
endif
.DEFAULT_GOAL := fengyun_mpt
.PHONY: fengyun_mpt
