# oracle/nearest.mk -- builds the TEST-ONLY CPU checker of the nearest-first iteration (beginNNTree / beginNNLeaves).
#
#   _ref/libufo_ref_nearest.so  ref_nearest.cpp (which includes ref_volumes.cpp and ref_harness.cpp)
#                               against the UNMODIFIED reference under $(REF) (only present in the build
#                               container); output in oracle/_ref/ only.
#
# Same compilers and flags as oracle/volumes.mk.  The library may not be linked or loaded by the product
# path (ufomap_b200/).

REF      ?= /root/reference
CXX      ?= g++
CXXFLAGS ?= -std=c++17 -O3 -DNDEBUG -fPIC -w
REF_CXX  ?= $(shell if [ -x /usr/bin/g++ ]; then echo /usr/bin/g++; else echo $(CXX); fi)

REF_SRCS = $(REF)/ufomap/src/map/occupancy_map.cpp \
           $(REF)/ufomap/src/map/occupancy_map_color.cpp \
           $(REF)/ufomap/src/geometry/bounding_volume.cpp \
           $(REF)/ufomap/src/geometry/collision_checks.cpp

all: ref

ref:
	@if [ -d $(REF)/ufomap/include ]; then $(MAKE) -f nearest.mk _ref/libufo_ref_nearest.so; \
	 else echo "oracle: $(REF) absent -- using prebuilt _ref/libufo_ref_nearest.so if present"; fi

_ref/libufo_ref_nearest.so: ref_nearest.cpp ref_volumes.cpp ref_harness.cpp
	mkdir -p _ref
	$(REF_CXX) $(CXXFLAGS) -shared -I$(REF)/ufomap/include -Istub -o $@ ref_nearest.cpp $(REF_SRCS) -lpthread -ldl

.PHONY: all ref
