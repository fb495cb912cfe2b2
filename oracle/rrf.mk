# oracle/rrf.mk -- builds oracle/_ref/libref_rrf.so: simeon's OWN reciprocal-rank fusion of BM25 variants
# (third_party/simeon/src/fusion.cpp: score_bm25_variants_rrf), the Bm25Index variants it fuses (src/bm25.cpp) and the
# ConceptIndex blended onto the fused scores (src/concept_mining.cpp), with the C shim ref_rrf_shim.cpp, compiled where they lie
# under $(REF).  Only possible where the reference tree exists; elsewhere the target says so and does nothing.  Nothing is
# copied out of $(REF); the output goes only to oracle/_ref/.
#
# The three are compiled with simeon's flags for them (meson.build:74-137): no -mfma, so nothing of the scores, the ranks'
# 1 / (k + r) or the blend is fused.
REF  ?= /root/reference
SIM  := $(REF)/third_party/simeon
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CXX  := /usr/bin/g++
FLAGS := -std=c++20 -O2 -fPIC -I$(SIM)/include -DSIMEON_HAS_AVX2=1
DEPS := $(addprefix $(SIM)/src/,hasher.cpp hash_xxh64.cpp hash_crc32c.cpp hash_tabulation.cpp tokenizer.cpp tokenizer_bpe.cpp pmi.cpp \
          arch/scalar.cpp)

.PHONY: all
all: $(HERE)_ref/libref_rrf.so
$(HERE)_ref/libref_rrf.so: $(HERE)ref_rrf_shim.cpp
	@if [ ! -f "$(SIM)/src/fusion.cpp" ]; then echo "reference tree absent at $(REF): skipping"; exit 0; fi; \
	mkdir -p $(HERE)_ref && \
	$(CXX) $(FLAGS) -c $(SIM)/src/bm25.cpp -o $(HERE)_ref/rrf_bm25.o && \
	$(CXX) $(FLAGS) -c $(SIM)/src/concept_mining.cpp -o $(HERE)_ref/rrf_concept_mining.o && \
	$(CXX) $(FLAGS) -c $(SIM)/src/fusion.cpp -o $(HERE)_ref/rrf_fusion.o && \
	$(CXX) $(FLAGS) -shared $(HERE)ref_rrf_shim.cpp $(HERE)_ref/rrf_bm25.o $(HERE)_ref/rrf_concept_mining.o $(HERE)_ref/rrf_fusion.o \
	  $(DEPS) -Wl,--no-undefined -o $@
