# TEST INFRASTRUCTURE ONLY. The checker of the METEOR-M LRPT decoder (meteor_lrpt_decoder), built beside the rest of the oracle
# (oracle/Makefile) with the same compiler flags:
#   oracle/_ref/libsatref_meteor.so  the UNMODIFIED reference translation units of Correlator, Viterbi27 (CCDecoder, CCEncoder), Viterbi1_2,
#                                    NRZ-M, rotate_soft, the derandomiser, BPSK_CCSDS_Deframer and the Reed-Solomon decoder (+ libcorrect),
#                                    compiled where they lie under $(REF) (never copied), + meteor_harness.cpp (our wiring / C ABI)
# Where the reference is absent the tests read tests/golden/meteor_lrpt_pins.json (written by tests/golden/make_meteor_lrpt_pins.py).
REF ?= /root/reference
SRC := $(REF)/src-core
OUT := _ref
CXX := $(shell [ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
CC  := $(shell [ -x /usr/bin/gcc ] && echo /usr/bin/gcc || echo gcc)
CXXFLAGS := -std=c++17 -O2 -fPIC -DSOURCE_PATH_SIZE=0 -Ishim -I$(REF)/volk_includes -I$(SRC) -w
CFLAGS := -O2 -fPIC -I$(SRC)/libs/correct -I$(SRC) -w

REF_CXX := common/codings/correlator.cpp common/codings/rotation.cpp common/codings/randomization.cpp common/codings/reedsolomon/reedsolomon.cpp \
  common/codings/viterbi/viterbi27.cpp common/codings/viterbi/cc_decoder.cpp common/codings/viterbi/cc_encoder.cpp \
  common/codings/viterbi/viterbi_1_2.cpp common/codings/viterbi/utils.cpp common/codings/differential/nrzm.cpp \
  common/codings/deframing/bpsk_ccsds_deframer.cpp
REF_C := libs/correct/reed-solomon/decode.c libs/correct/reed-solomon/encode.c libs/correct/reed-solomon/polynomial.c \
  libs/correct/reed-solomon/reed-solomon.c
SHIM := shim/volk/volk.h shim/volk/volk_typedefs.h shim/logger.h
OBJ := $(patsubst %.cpp,$(OUT)/obj_meteor/%.o,$(REF_CXX)) $(patsubst %.c,$(OUT)/obj_meteor/%.o,$(REF_C))

all: ref

ref:
	@if [ -d "$(REF)/src-core" ]; then $(MAKE) --no-print-directory -f meteor.mk $(OUT)/libsatref_meteor.so; \
	 else echo "oracle: $(REF) absent - keeping prebuilt $(OUT)/libsatref_meteor.so"; fi

$(OUT)/obj_meteor/%.o: $(SRC)/%.cpp $(SHIM)
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/obj_meteor/%.o: $(SRC)/%.c
	@mkdir -p $(dir $@)
	$(CC) $(CFLAGS) -c $< -o $@
$(OUT)/obj_meteor/meteor_harness.o: meteor_harness.cpp $(SHIM)
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/libsatref_meteor.so: $(OBJ) $(OUT)/obj_meteor/meteor_harness.o
	$(CXX) -shared -Wl,-Bsymbolic -o $@ $^ -lstdc++ -lm

clean:
	rm -rf $(OUT)/obj_meteor $(OUT)/libsatref_meteor.so
.PHONY: all ref clean
