# TEST INFRASTRUCTURE ONLY. The checker of the MetOp X-band dump decoder (metop_dump_decoder), built beside the rest of the oracle
# (oracle/Makefile) with the same compiler flags:
#   oracle/_ref/libsatref_dump.so  the UNMODIFIED reference translation units of Correlator32, rotate_soft, the derandomiser and the
#                                  Reed-Solomon decoder (+ libcorrect), compiled where they lie under $(REF) (never copied), + dump_harness.cpp
#                                  (our wiring / C ABI)
#   oracle/libdump_port.so         our own C restatement of the module loop (dump_port.c) over oracle.c's rotate_soft, derandomiser and RS
# Where the reference is absent the tests read tests/golden/metop_dump_pins.json (written by tests/golden/make_metop_dump_pins.py).
REF ?= /root/reference
SRC := $(REF)/src-core
OUT := _ref
CXX := $(shell [ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
CC  := $(shell [ -x /usr/bin/gcc ] && echo /usr/bin/gcc || echo gcc)
CXXFLAGS := -std=c++17 -O2 -fPIC -DSOURCE_PATH_SIZE=0 -Ishim -I$(REF)/volk_includes -I$(SRC) -w
CFLAGS := -O2 -fPIC -I$(SRC)/libs/correct -I$(SRC) -w

REF_CXX := common/codings/correlator32.cpp common/codings/rotation.cpp common/codings/randomization.cpp common/codings/reedsolomon/reedsolomon.cpp
REF_C := libs/correct/reed-solomon/decode.c libs/correct/reed-solomon/encode.c libs/correct/reed-solomon/polynomial.c \
  libs/correct/reed-solomon/reed-solomon.c
SHIM := shim/volk/volk.h shim/volk/volk_typedefs.h shim/logger.h
OBJ := $(patsubst %.cpp,$(OUT)/obj_dump/%.o,$(REF_CXX)) $(patsubst %.c,$(OUT)/obj_dump/%.o,$(REF_C))

all: libdump_port.so ref

ref:
	@if [ -d "$(REF)/src-core" ]; then $(MAKE) --no-print-directory -f dump.mk $(OUT)/libsatref_dump.so; \
	 else echo "oracle: $(REF) absent - keeping prebuilt $(OUT)/libsatref_dump.so"; fi

$(OUT)/obj_dump/%.o: $(SRC)/%.cpp $(SHIM)
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/obj_dump/%.o: $(SRC)/%.c
	@mkdir -p $(dir $@)
	$(CC) $(CFLAGS) -c $< -o $@
$(OUT)/obj_dump/dump_harness.o: dump_harness.cpp $(SHIM)
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(OUT)/libsatref_dump.so: $(OBJ) $(OUT)/obj_dump/dump_harness.o
	$(CXX) -shared -Wl,-Bsymbolic -o $@ $^ -lstdc++ -lm

libdump_port.so: dump_port.c oracle.c oracle.h
	$(CC) -O2 -ffp-contract=off -fPIC -std=gnu11 -shared -o $@ dump_port.c oracle.c -lm

clean:
	rm -rf $(OUT)/obj_dump $(OUT)/libsatref_dump.so libdump_port.so
.PHONY: all ref clean
