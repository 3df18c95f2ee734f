# TEST INFRASTRUCTURE ONLY. The checker of the METEOR-M X-band dump decoder (meteor_xband_decoder), built beside the rest of the oracle
# (oracle/Makefile) with the same compiler flags:
#   oracle/_ref/libsatref_xband.so  the UNMODIFIED reference translation units meteor/meteor_rec_deframer.cpp (with the record deframers
#                                   of its header), common/codings/differential/nrzm.cpp and common/repack_bits_byte.cpp, compiled where
#                                   they lie under $(REF) (never copied), + xband_harness.cpp (our wiring / C ABI), which includes the
#                                   reference's header-only SimpleDeframer
# Where the reference is absent the tests read tests/golden/meteor_xband_pins.json (written by tests/golden/make_meteor_xband_pins.py).
REF ?= /root/reference
PLUG := $(REF)/plugins
CORE := $(REF)/src-core
OUT := _ref
CXX := $(shell [ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
CXXFLAGS := -std=c++17 -O2 -fPIC -w -I$(CORE) -I$(PLUG)/meteor_support

OBJ := $(OUT)/obj_xband/meteor_rec_deframer.o $(OUT)/obj_xband/nrzm.o $(OUT)/obj_xband/repack_bits_byte.o $(OUT)/obj_xband/xband_harness.o

all: ref

ref:
	@if [ -d "$(PLUG)" ]; then $(MAKE) --no-print-directory -f xband.mk $(OUT)/libsatref_xband.so; \
	 else echo "oracle: $(REF) absent - keeping prebuilt $(OUT)/libsatref_xband.so"; fi

$(OUT)/obj_xband/meteor_rec_deframer.o: $(PLUG)/meteor_support/meteor/meteor_rec_deframer.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/obj_xband/nrzm.o: $(CORE)/common/codings/differential/nrzm.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/obj_xband/repack_bits_byte.o: $(CORE)/common/repack_bits_byte.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/obj_xband/xband_harness.o: xband_harness.cpp $(PLUG)/meteor_support/meteor/meteor_rec_deframer.h $(CORE)/common/simple_deframer.h
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/libsatref_xband.so: $(OBJ)
	$(CXX) -shared -Wl,-Bsymbolic -o $@ $^ -lstdc++ -lm

clean:
	rm -rf $(OUT)/obj_xband $(OUT)/libsatref_xband.so
.PHONY: all ref clean
