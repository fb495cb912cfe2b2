# oracle/strategy.mk -- builds oracle/_ref/libref_strategy.so: simeon's OWN lead-text field and BM25F strategies as the lexical
# backend's strategy router builds and scores them: extract_lead_tokens (third_party/simeon/src/corpus_adapter.cpp),
# Bm25Index::add_doc(text, aux_text) and score_bm25f (src/bm25.cpp), Bm25Strategy and LeadFieldStrategy
# (src/retrieval_strategy.cpp) and the ConceptIndex blended after them (src/concept_mining.cpp, with src/fusion.cpp, which the
# strategies link against), with the C shim ref_strategy_shim.cpp, compiled where they lie under $(REF).  Only possible where
# the reference tree exists; elsewhere the target says so and does nothing.  Nothing is copied out of $(REF); the output goes
# only to oracle/_ref/.
#
# Compiled with simeon's flags for them (meson.build:74-137): no -mfma, so nothing of the scores, the BM25F weights or the
# blend is fused.
REF  ?= /root/reference
SIM  := $(REF)/third_party/simeon
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CXX  := /usr/bin/g++
FLAGS := -std=c++20 -O2 -fPIC -I$(SIM)/include -DSIMEON_HAS_AVX2=1
SRCS := bm25 corpus_adapter retrieval_strategy fusion concept_mining
DEPS := $(addprefix $(SIM)/src/,hasher.cpp hash_xxh64.cpp hash_crc32c.cpp hash_tabulation.cpp tokenizer.cpp tokenizer_bpe.cpp pmi.cpp \
          arch/scalar.cpp)

.PHONY: all
all: $(HERE)_ref/libref_strategy.so
$(HERE)_ref/libref_strategy.so: $(HERE)ref_strategy_shim.cpp
	@if [ ! -f "$(SIM)/src/retrieval_strategy.cpp" ]; then echo "reference tree absent at $(REF): skipping"; exit 0; fi; \
	mkdir -p $(HERE)_ref && \
	for s in $(SRCS); do $(CXX) $(FLAGS) -c $(SIM)/src/$$s.cpp -o $(HERE)_ref/strategy_$$s.o || exit 1; done && \
	$(CXX) $(FLAGS) -shared $(HERE)ref_strategy_shim.cpp $(addprefix $(HERE)_ref/strategy_,$(addsuffix .o,$(SRCS))) \
	  $(DEPS) -Wl,--no-undefined -o $@
