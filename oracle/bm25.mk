# oracle/bm25.mk -- builds oracle/_ref/libref_bm25.so: simeon's OWN Bm25Index (third_party/simeon/src/bm25.cpp and the sources it
# links against) with the C shim ref_bm25_shim.cpp, compiled where they lie under $(REF).  Only possible where the reference tree
# exists; elsewhere the target says so and does nothing.  Nothing is copied out of $(REF); the output goes only to oracle/_ref/.
#
# bm25.cpp is compiled in a step of its own with simeon's flags for it (simd_defines + extra_cpp_args, meson.build:74-137): no
# -mfma.  With -mfma GCC contracts `out += alpha * s` into a fused multiply-add and the scores change in the last bit.
REF  ?= /root/reference
SIM  := $(REF)/third_party/simeon
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CXX  := /usr/bin/g++
FLAGS := -std=c++20 -O2 -fPIC -I$(SIM)/include -DSIMEON_HAS_AVX2=1
DEPS := $(addprefix $(SIM)/src/,hasher.cpp hash_xxh64.cpp hash_crc32c.cpp hash_tabulation.cpp tokenizer.cpp tokenizer_bpe.cpp pmi.cpp \
          arch/scalar.cpp)

.PHONY: all
all: $(HERE)_ref/libref_bm25.so
$(HERE)_ref/libref_bm25.so: $(HERE)ref_bm25_shim.cpp
	@if [ ! -f "$(SIM)/src/bm25.cpp" ]; then echo "reference tree absent at $(REF): skipping"; exit 0; fi; \
	mkdir -p $(HERE)_ref && \
	$(CXX) $(FLAGS) -c $(SIM)/src/bm25.cpp -o $(HERE)_ref/bm25.o && \
	$(CXX) $(FLAGS) -shared $(HERE)ref_bm25_shim.cpp $(HERE)_ref/bm25.o $(DEPS) -Wl,--no-undefined -o $@
