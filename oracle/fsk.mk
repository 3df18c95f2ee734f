# TEST INFRASTRUCTURE ONLY. The checker of the FSK demodulator (fsk_demod), built beside the rest of the oracle (oracle/Makefile) with
# the same compiler flags:
#   oracle/_ref/libsatref_fsk.so  the UNMODIFIED reference translation units of the complex AGC, QuadratureDemodBlock, CorrectIQBlock,
#                                 AGCBlock, FIRBlock + firdes, MMClockRecoveryBlock (+ its polyphase bank and window) and the M2M4 SNR
#                                 estimator, compiled where they lie under $(REF) (never copied), + fsk_harness.cpp (our wiring / C ABI).
#                                 Linked with --wrap=atan2f: the harness chooses glibc's atan2f or the correctly rounded one.
# Where the reference is absent the tests read tests/golden/fsk_pins.json (written by tests/golden/make_fsk_pins.py).
REF ?= /root/reference
SRC := $(REF)/src-core
OUT := _ref
CXX := $(shell [ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
CXXFLAGS := -std=c++17 -O2 -fPIC -DSOURCE_PATH_SIZE=0 -Ishim -I$(REF)/volk_includes -I$(SRC) -w

REF_CXX := common/dsp/block.cpp common/dsp/buffer.cpp common/dsp/utils/agc.cpp common/dsp/utils/correct_iq.cpp common/dsp/utils/snr_estimator.cpp \
  common/dsp/demod/quadrature_demod.cpp common/dsp/utils/fast_trig.cpp common/dsp/filter/fir.cpp common/dsp/filter/firdes.cpp \
  common/dsp/clock_recovery/clock_recovery_mm.cpp common/dsp/resamp/polyphase_bank.cpp common/dsp/window/window.cpp
SHIM := shim/volk/volk.h shim/volk/volk_typedefs.h shim/logger.h
OBJ := $(patsubst %.cpp,$(OUT)/obj_fsk/%.o,$(REF_CXX))

all: ref

ref:
	@if [ -d "$(REF)/src-core" ]; then $(MAKE) --no-print-directory -f fsk.mk $(OUT)/libsatref_fsk.so; \
	 else echo "oracle: $(REF) absent - keeping prebuilt $(OUT)/libsatref_fsk.so"; fi

$(OUT)/obj_fsk/%.o: $(SRC)/%.cpp $(SHIM)
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/obj_fsk/fsk_harness.o: fsk_harness.cpp $(SHIM)
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/libsatref_fsk.so: $(OBJ) $(OUT)/obj_fsk/fsk_harness.o
	$(CXX) -shared -Wl,-Bsymbolic -Wl,--wrap=atan2f -o $@ $^ -lstdc++ -lm -lpthread

clean:
	rm -rf $(OUT)/obj_fsk $(OUT)/libsatref_fsk.so
.PHONY: all ref clean
