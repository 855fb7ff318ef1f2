# oracle/color_writes.mk -- builds the TEST-ONLY CPU checkers of the colour map's writers.
#
#   libufo_oracle_color_writes.so    ufo_oracle_writes.c + ufo_oracle_color_writes.c (plain-C
#                                    restatement); built everywhere.
#   _ref/libufo_ref_color_writes.so  ref_writes.cpp + ref_color_writes.cpp against the UNMODIFIED
#                                    reference under $(REF) (only present in the build container);
#                                    output in oracle/_ref/ only.
#
# Same compilers and flags as oracle/writes.mk.  Neither library may be linked or loaded by the
# product path (ufomap_b200/).

REF      ?= /root/reference
CC       ?= gcc
CXX      ?= g++
CFLAGS   ?= -O2 -fPIC -std=c11 -Wall -Wextra -ffp-contract=off
CXXFLAGS ?= -std=c++17 -O3 -DNDEBUG -fPIC -w
REF_CXX  ?= $(shell if [ -x /usr/bin/g++ ]; then echo /usr/bin/g++; else echo $(CXX); fi)

REF_SRCS = $(REF)/ufomap/src/map/occupancy_map.cpp \
           $(REF)/ufomap/src/map/occupancy_map_color.cpp \
           $(REF)/ufomap/src/geometry/bounding_volume.cpp \
           $(REF)/ufomap/src/geometry/collision_checks.cpp

all: libufo_oracle_color_writes.so ref

libufo_oracle_color_writes.so: ufo_oracle_color_writes.c ufo_oracle_writes.c ufo_oracle.c ufo_oracle.h
	$(CC) $(CFLAGS) -shared -o $@ ufo_oracle_color_writes.c -lm

ref:
	@if [ -d $(REF)/ufomap/include ]; then $(MAKE) -f color_writes.mk _ref/libufo_ref_color_writes.so; \
	 else echo "oracle: $(REF) absent -- using prebuilt _ref/libufo_ref_color_writes.so if present"; fi

_ref/libufo_ref_color_writes.so: ref_color_writes.cpp ref_writes.cpp ref_harness.cpp
	mkdir -p _ref
	$(REF_CXX) $(CXXFLAGS) -shared -I$(REF)/ufomap/include -Istub -o $@ ref_color_writes.cpp $(REF_SRCS) -lpthread -ldl

.PHONY: all ref
