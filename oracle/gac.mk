# TEST INFRASTRUCTURE ONLY. The checker of the NOAA GAC and DMSP RTD decoders (noaa_gac_decoder, dmsp_rtd_decoder), built beside the rest
# of the oracle (oracle/Makefile) with the same compiler flags:
#   oracle/_ref/libsatref_gac.so  the UNMODIFIED reference translation units common/codings/deframing/bpsk_ccsds_deframer.cpp and
#                                 dmsp/dmsp_deframer.cpp, compiled where they lie under $(REF) (never copied), + gac_harness.cpp (our
#                                 wiring / C ABI), which includes the reference's noaa/gac_pn.h at compile time
# Where the reference is absent the tests read tests/golden/gac_pins.json (written by tests/golden/make_gac_pins.py).
REF ?= /root/reference
PLUG := $(REF)/plugins
CORE := $(REF)/src-core
OUT := _ref
CXX := $(shell [ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
CXXFLAGS := -std=c++17 -O2 -fPIC -w -I$(CORE) -I$(PLUG)/dmsp_support -I$(PLUG)/noaa_metop_support

OBJ := $(OUT)/obj_gac/bpsk_ccsds_deframer.o $(OUT)/obj_gac/dmsp_deframer.o $(OUT)/obj_gac/gac_harness.o

all: ref

ref:
	@if [ -d "$(PLUG)" ]; then $(MAKE) --no-print-directory -f gac.mk $(OUT)/libsatref_gac.so; \
	 else echo "oracle: $(REF) absent - keeping prebuilt $(OUT)/libsatref_gac.so"; fi

$(OUT)/obj_gac/bpsk_ccsds_deframer.o: $(CORE)/common/codings/deframing/bpsk_ccsds_deframer.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/obj_gac/dmsp_deframer.o: $(PLUG)/dmsp_support/dmsp/dmsp_deframer.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/obj_gac/gac_harness.o: gac_harness.cpp $(PLUG)/noaa_metop_support/noaa/gac_pn.h
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/libsatref_gac.so: $(OBJ)
	$(CXX) -shared -Wl,-Bsymbolic -o $@ $^ -lstdc++ -lm

clean:
	rm -rf $(OUT)/obj_gac $(OUT)/libsatref_gac.so
.PHONY: all ref clean
