# oracle/concepts.mk -- builds oracle/_ref/libref_concepts.so: simeon's OWN ConceptIndex (third_party/simeon/src/concept_mining.cpp)
# and the Bm25Index it is mined against (src/bm25.cpp and the sources they link against) with the C shim ref_concepts_shim.cpp,
# compiled where they lie under $(REF).  Only possible where the reference tree exists; elsewhere the target says so and does
# nothing.  Nothing is copied out of $(REF); the output goes only to oracle/_ref/.
#
# bm25.cpp and concept_mining.cpp are compiled with simeon's flags for them (meson.build:74-137): no -mfma, so no multiply and
# add of the blend are fused.
REF  ?= /root/reference
SIM  := $(REF)/third_party/simeon
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CXX  := /usr/bin/g++
FLAGS := -std=c++20 -O2 -fPIC -I$(SIM)/include -DSIMEON_HAS_AVX2=1
DEPS := $(addprefix $(SIM)/src/,hasher.cpp hash_xxh64.cpp hash_crc32c.cpp hash_tabulation.cpp tokenizer.cpp tokenizer_bpe.cpp pmi.cpp \
          arch/scalar.cpp)

.PHONY: all
all: $(HERE)_ref/libref_concepts.so
$(HERE)_ref/libref_concepts.so: $(HERE)ref_concepts_shim.cpp
	@if [ ! -f "$(SIM)/src/concept_mining.cpp" ]; then echo "reference tree absent at $(REF): skipping"; exit 0; fi; \
	mkdir -p $(HERE)_ref && \
	$(CXX) $(FLAGS) -c $(SIM)/src/bm25.cpp -o $(HERE)_ref/concepts_bm25.o && \
	$(CXX) $(FLAGS) -c $(SIM)/src/concept_mining.cpp -o $(HERE)_ref/concept_mining.o && \
	$(CXX) $(FLAGS) -shared $(HERE)ref_concepts_shim.cpp $(HERE)_ref/concepts_bm25.o $(HERE)_ref/concept_mining.o $(DEPS) \
	  -Wl,--no-undefined -o $@
