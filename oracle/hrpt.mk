# TEST INFRASTRUCTURE ONLY. The checker of the NOAA and METEOR HRPT decoders (noaa_hrpt_decoder, meteor_hrpt_decoder), built beside the
# rest of the oracle (oracle/Makefile) with the same compiler flags:
#   oracle/_ref/libsatref_hrpt.so  the UNMODIFIED reference translation units noaa/noaa_deframer.cpp and meteor/deframer.cpp, compiled
#                                  where they lie under $(REF) (never copied), + hrpt_harness.cpp (our wiring / C ABI)
# Where the reference is absent the tests read tests/golden/hrpt_pins.json (written by tests/golden/make_hrpt_pins.py).
REF ?= /root/reference
PLUG := $(REF)/plugins
OUT := _ref
CXX := $(shell [ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
CXXFLAGS := -std=c++17 -O2 -fPIC -w -I$(PLUG)/noaa_metop_support -I$(PLUG)/meteor_support

REF_CXX := noaa_metop_support/noaa/noaa_deframer.cpp meteor_support/meteor/deframer.cpp
OBJ := $(patsubst %.cpp,$(OUT)/obj_hrpt/%.o,$(REF_CXX))

all: ref

ref:
	@if [ -d "$(PLUG)" ]; then $(MAKE) --no-print-directory -f hrpt.mk $(OUT)/libsatref_hrpt.so; \
	 else echo "oracle: $(REF) absent - keeping prebuilt $(OUT)/libsatref_hrpt.so"; fi

$(OUT)/obj_hrpt/%.o: $(PLUG)/%.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/obj_hrpt/hrpt_harness.o: hrpt_harness.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/libsatref_hrpt.so: $(OBJ) $(OUT)/obj_hrpt/hrpt_harness.o
	$(CXX) -shared -Wl,-Bsymbolic -o $@ $^ -lstdc++ -lm

clean:
	rm -rf $(OUT)/obj_hrpt $(OUT)/libsatref_hrpt.so
.PHONY: all ref clean
