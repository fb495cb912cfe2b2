# oracle/topology_kmeans.mk -- builds oracle/_ref/libref_topology_kmeans.so: the reference's OWN k-means topology engine
# (KMeansTopologyEngine, src/topology/topology_alternate_engines.cpp and the three sources it links against) with the C shim
# ref_topology_shim.cpp, compiled where they lie under $(REF).  Only possible where the reference tree exists; elsewhere the
# target says so and does nothing.  Nothing is copied out of $(REF); the output goes only to oracle/_ref/ (git-ignored).
REF  ?= /root/reference
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
CXX  := /usr/bin/g++
SRCS := $(addprefix $(REF)/src/,topology/topology_alternate_engines.cpp topology/protected_relation_cover.cpp \
          topology/topology_representatives.cpp vector/static_cosine_ann_index.cpp)

.PHONY: all
all: $(HERE)_ref/libref_topology_kmeans.so
$(HERE)_ref/libref_topology_kmeans.so: $(HERE)ref_topology_shim.cpp
	@if [ ! -f "$(REF)/src/topology/topology_alternate_engines.cpp" ]; then echo "reference tree absent at $(REF): skipping"; exit 0; fi; \
	mkdir -p $(HERE)_ref && \
	$(CXX) -std=c++20 -O2 -fPIC -shared -I$(REF)/include -I$(REF)/src -I$(REF)/third_party/sqlite-vec-cpp/include \
	  $(HERE)ref_topology_shim.cpp $(SRCS) -o $@
