# Builds the CPU oracle of HoughTransform (TEST INFRASTRUCTURE ONLY) as a library of its own, with the flags of the main oracle
# (Makefile): -ffp-contract=off, no fast math.  Bound in tests/hough_oracle.py.
CXX      := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wextra -Wno-unused-parameter

libzo_hough.so: zo_hough.cpp zignal_oracle.h zo_common.h hough.mk
	$(CXX) $(CXXFLAGS) -shared -o $@.tmp zo_hough.cpp
	mv -f $@.tmp $@
