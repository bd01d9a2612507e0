# Builds the CPU oracle of convertColor between the 33 colour formats (TEST INFRASTRUCTURE ONLY) as a library of its own, with the
# flags of the main oracle (Makefile).  Bound in tests/color_oracle.py.
CXX      := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wextra -Wno-unused-parameter

libzo_color.so: zo_color.cpp color.mk
	$(CXX) $(CXXFLAGS) -shared -o $@.tmp zo_color.cpp
	mv -f $@.tmp $@
