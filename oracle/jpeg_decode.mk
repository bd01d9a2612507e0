# Builds the CPU oracle of the baseline JPEG decoder (TEST INFRASTRUCTURE ONLY) as a library of its own, with the flags of the main
# oracle (Makefile).  Bound in tests/jpeg_decode_oracle.py.
CXX      := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wextra -Wno-unused-parameter

libzo_jpeg_decode.so: zo_jpeg_decode.cpp jpeg_decode.mk
	$(CXX) $(CXXFLAGS) -shared -o $@.tmp zo_jpeg_decode.cpp
	mv -f $@.tmp $@
