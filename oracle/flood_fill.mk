# Builds the CPU oracle of Image.floodFill (TEST INFRASTRUCTURE ONLY) as a library of its own, with the flags of the main oracle
# (Makefile): -ffp-contract=off, no fast math.  Bound in tests/flood_fill_oracle.py.
CXX      := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wextra -Wno-unused-parameter

libzo_flood_fill.so: zo_flood_fill.cpp zignal_oracle.h zo_common.h flood_fill.mk
	$(CXX) $(CXXFLAGS) -shared -o $@.tmp zo_flood_fill.cpp
	mv -f $@.tmp $@
