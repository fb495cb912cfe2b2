# oracle/router.mk -- builds oracle/_ref/libref_router.so: simeon's OWN QueryRouter (third_party/simeon/src/query_router.cpp) over
# its own Bm25Index (src/bm25.cpp, src/tokenizer.cpp) and the ConceptIndex blended after it (src/concept_mining.cpp, with
# src/fusion.cpp, which the router links against), with the C shim ref_router_shim.cpp, compiled where they lie under $(REF).
# Only possible where the reference tree exists; elsewhere the target says so and does nothing.  Nothing is copied out of
# $(REF); the output goes only to oracle/_ref/.
#
# Compiled with simeon's flags for them (meson.build:74-137): no -mfma, so nothing of the features, the scores or the blend is
# fused.
REF  ?= /root/reference
SIM  := $(REF)/third_party/simeon
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CXX  := /usr/bin/g++
FLAGS := -std=c++20 -O2 -fPIC -I$(SIM)/include -DSIMEON_HAS_AVX2=1
SRCS := query_router bm25 tokenizer fusion concept_mining
DEPS := $(addprefix $(SIM)/src/,hasher.cpp hash_xxh64.cpp hash_crc32c.cpp hash_tabulation.cpp tokenizer_bpe.cpp pmi.cpp arch/scalar.cpp)

.PHONY: all
all: $(HERE)_ref/libref_router.so
$(HERE)_ref/libref_router.so: $(HERE)ref_router_shim.cpp
	@if [ ! -f "$(SIM)/src/query_router.cpp" ]; then echo "reference tree absent at $(REF): skipping"; exit 0; fi; \
	mkdir -p $(HERE)_ref && \
	for s in $(SRCS); do $(CXX) $(FLAGS) -c $(SIM)/src/$$s.cpp -o $(HERE)_ref/router_$$s.o || exit 1; done && \
	$(CXX) $(FLAGS) -shared $(HERE)ref_router_shim.cpp $(addprefix $(HERE)_ref/router_,$(addsuffix .o,$(SRCS))) \
	  $(DEPS) -Wl,--no-undefined -o $@
