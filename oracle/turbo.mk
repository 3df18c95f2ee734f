# TEST INFRASTRUCTURE ONLY. The checker of the CCSDS turbo decoder (ccsds_turbo_decoder), built beside the rest of the oracle
# (oracle/Makefile) with the same compiler flags:
#   oracle/_ref/libsatref_turbo.so  the UNMODIFIED reference translation units of CCSDSTurbo, the deepspace-turbo library, the CRC and the
#                                   derandomiser, compiled where they lie under $(REF) (never copied), + turbo_harness.cpp (our wiring / C ABI)
#   oracle/libturbo_port.so         our own C restatement of the same path (turbo_port.c)
# Where the reference is absent the tests read tests/golden/turbo_pins.json (written by tests/golden/make_turbo_pins.py).
REF ?= /root/reference
SRC := $(REF)/src-core
OUT := _ref
CXX := $(shell [ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
CC  := $(shell [ -x /usr/bin/gcc ] && echo /usr/bin/gcc || echo gcc)
# -O2 without -march: no FMA contraction (the correlator's dot products and the BCJR are plain IEEE operations)
CXXFLAGS := -std=c++17 -O2 -fPIC -DSOURCE_PATH_SIZE=0 -Ildpc_shim -Ishim -I$(REF)/volk_includes -I$(SRC) -w
CFLAGS := -std=gnu11 -O2 -fPIC -I$(SRC) -w

REF_CXX := common/codings/turbo/ccsds_turbo.cpp common/codings/crc/crc_generic.cpp common/codings/randomization.cpp
REF_C := libs/deepspace-turbo/libconvcodes.c libs/deepspace-turbo/libturbocodes.c
SHIM := ldpc_shim/volk/volk.h shim/volk/volk.h shim/volk/volk_typedefs.h
OBJ := $(patsubst %.cpp,$(OUT)/obj_turbo/%.o,$(REF_CXX)) $(patsubst %.c,$(OUT)/obj_turbo/%.o,$(REF_C))

all: libturbo_port.so ref

ref:
	@if [ -d "$(REF)/src-core" ]; then $(MAKE) --no-print-directory -f turbo.mk $(OUT)/libsatref_turbo.so; \
	 else echo "oracle: $(REF) absent - keeping prebuilt $(OUT)/libsatref_turbo.so"; fi

$(OUT)/obj_turbo/%.o: $(SRC)/%.cpp $(SHIM)
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/obj_turbo/%.o: $(SRC)/%.c
	@mkdir -p $(dir $@)
	$(CC) $(CFLAGS) -c $< -o $@
$(OUT)/obj_turbo/turbo_harness.o: turbo_harness.cpp $(SHIM)
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/libsatref_turbo.so: $(OBJ) $(OUT)/obj_turbo/turbo_harness.o
	$(CXX) -shared -Wl,-Bsymbolic -o $@ $^ -lstdc++ -lm

libturbo_port.so: turbo_port.c
	$(CC) -O2 -ffp-contract=off -fPIC -std=gnu11 -shared -o $@ turbo_port.c -lm

clean:
	rm -rf $(OUT)/obj_turbo $(OUT)/libsatref_turbo.so libturbo_port.so
.PHONY: all ref clean
