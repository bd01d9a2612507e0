# Builds the CPU oracle of the 8-bit histogram family and binary morphology (TEST INFRASTRUCTURE ONLY) as a library of its own,
# with the flags of the main oracle (Makefile): -ffp-contract=off, no fast math.  Bound in tests/binary_oracle.py.
CXX      := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wextra -Wno-unused-parameter

libzo_binary.so: zo_binary.cpp zignal_oracle.h zo_common.h binary.mk
	$(CXX) $(CXXFLAGS) -shared -o $@.tmp zo_binary.cpp
	mv -f $@.tmp $@
