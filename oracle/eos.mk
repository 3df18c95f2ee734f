# TEST INFRASTRUCTURE ONLY. The checker of the Aqua / Aura DB decoder (aqua_db_decoder), built beside the rest of the oracle
# (oracle/Makefile) with the same compiler flags:
#   oracle/_ref/libsatref_eos.so  the UNMODIFIED reference translation units of constellation_t, NRZMDiff, BPSK_CCSDS_Deframer, the
#                                 derandomiser and the Reed-Solomon decoder (+ libcorrect), compiled where they lie under $(REF) (never
#                                 copied), + eos_harness.cpp (our wiring / C ABI)
# Where the reference is absent the tests read tests/golden/eos_pins.json (written by tests/golden/make_eos_pins.py).
REF ?= /root/reference
SRC := $(REF)/src-core
OUT := _ref
CXX := $(shell [ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
CC  := $(shell [ -x /usr/bin/gcc ] && echo /usr/bin/gcc || echo gcc)
CXXFLAGS := -std=c++17 -O2 -fPIC -DSOURCE_PATH_SIZE=0 -Ishim -I$(REF)/volk_includes -I$(SRC) -w
CFLAGS := -O2 -fPIC -I$(SRC)/libs/correct -I$(SRC) -w

REF_CXX := common/dsp/demod/constellation.cpp common/codings/differential/nrzm.cpp common/codings/deframing/bpsk_ccsds_deframer.cpp \
  common/codings/randomization.cpp common/codings/reedsolomon/reedsolomon.cpp
REF_C := libs/correct/reed-solomon/decode.c libs/correct/reed-solomon/encode.c libs/correct/reed-solomon/polynomial.c \
  libs/correct/reed-solomon/reed-solomon.c
SHIM := shim/volk/volk.h shim/volk/volk_typedefs.h shim/logger.h
OBJ := $(patsubst %.cpp,$(OUT)/obj_eos/%.o,$(REF_CXX)) $(patsubst %.c,$(OUT)/obj_eos/%.o,$(REF_C))

all: ref

ref:
	@if [ -d "$(REF)/src-core" ]; then $(MAKE) --no-print-directory -f eos.mk $(OUT)/libsatref_eos.so; \
	 else echo "oracle: $(REF) absent - keeping prebuilt $(OUT)/libsatref_eos.so"; fi

$(OUT)/obj_eos/%.o: $(SRC)/%.cpp $(SHIM)
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/obj_eos/%.o: $(SRC)/%.c
	@mkdir -p $(dir $@)
	$(CC) $(CFLAGS) -c $< -o $@
$(OUT)/obj_eos/eos_harness.o: eos_harness.cpp $(SHIM)
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/libsatref_eos.so: $(OBJ) $(OUT)/obj_eos/eos_harness.o
	$(CXX) -shared -Wl,-Bsymbolic -o $@ $^ -lstdc++ -lm

clean:
	rm -rf $(OUT)/obj_eos $(OUT)/libsatref_eos.so
.PHONY: all ref clean
