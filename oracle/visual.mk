# Builds the CPU oracle of Image.diff, applyColormap, the flips and invert (TEST INFRASTRUCTURE ONLY) as a library of its own, with the
# flags of the main oracle (Makefile).  Bound in tests/visual_oracle.py.
CXX      := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wextra -Wno-unused-parameter

libzo_visual.so: zo_visual.cpp zignal_oracle.h zo_common.h visual.mk
	$(CXX) $(CXXFLAGS) -shared -o $@.tmp zo_visual.cpp
	mv -f $@.tmp $@
