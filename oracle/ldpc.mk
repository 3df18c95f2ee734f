# TEST INFRASTRUCTURE ONLY. The checker of the CCSDS LDPC decoder (ccsds_ldpc_decoder, rate 7/8 C2 code), built beside the rest of the
# oracle (oracle/Makefile) with the same compiler flags:
#   oracle/_ref/libsatref_ldpc.so  the UNMODIFIED reference translation units of the correlator and the generic LDPC decoder, compiled
#                                  where they lie under $(REF) (never copied), + ldpc_harness.cpp (our wiring / C ABI)
#   oracle/libldpc_port.so         our own C restatement of the same algorithms (ldpc_port.c)
REF ?= /root/reference
SRC := $(REF)/src-core
OUT := _ref
CXX := $(shell [ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
CC  := $(shell [ -x /usr/bin/gcc ] && echo /usr/bin/gcc || echo gcc)
# -O2 without -march: no FMA contraction (the correlator's dot products are plain IEEE left-to-right sums)
CXXFLAGS := -std=c++17 -O2 -fPIC -DSOURCE_PATH_SIZE=0 -Ildpc_shim -Ishim -I$(REF)/volk_includes -I$(SRC) -w

REF_CXX := common/codings/ldpc/ccsds_ldpc.cpp common/codings/ldpc/ldpc_decoder_generic.cpp common/codings/ldpc/make_ccsds.cpp \
  common/codings/ldpc/ldpc_decoder.cpp common/cpu_features.cpp \
  common/codings/ldpc/matrix/sparse_matrix.cpp common/codings/ldpc/matrix/matrix.cpp common/codings/ldpc/matrix/alist.cpp \
  common/codings/ldpc/matrix/general_utils.cpp common/codings/generic_correlator.cpp common/codings/rotation.cpp \
  common/codings/randomization.cpp common/codings/deframing/bpsk_ccsds_deframer.cpp
SHIM := ldpc_shim/volk/volk.h shim/volk/volk.h shim/volk/volk_typedefs.h shim/logger.h
OBJ := $(patsubst %.cpp,$(OUT)/obj_ldpc/%.o,$(REF_CXX))

all: libldpc_port.so ref

ref:
	@if [ -d "$(REF)/src-core" ]; then $(MAKE) --no-print-directory -f ldpc.mk $(OUT)/libsatref_ldpc.so; \
	 else echo "oracle: $(REF) absent - keeping prebuilt $(OUT)/libsatref_ldpc.so"; fi

$(OUT)/obj_ldpc/%.o: $(SRC)/%.cpp $(SHIM)
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/obj_ldpc/ldpc_harness.o: ldpc_harness.cpp $(SHIM)
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/libsatref_ldpc.so: $(OBJ) $(OUT)/obj_ldpc/ldpc_harness.o
	$(CXX) -shared -Wl,-Bsymbolic -o $@ $^ -lstdc++ -lm -lpthread

libldpc_port.so: ldpc_port.c
	$(CC) -O2 -ffp-contract=off -fPIC -std=gnu11 -shared -o $@ ldpc_port.c -lm

clean:
	rm -rf $(OUT)/obj_ldpc $(OUT)/libsatref_ldpc.so libldpc_port.so
.PHONY: all ref clean
