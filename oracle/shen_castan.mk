# Builds the CPU oracle of Image.shenCastan (TEST INFRASTRUCTURE ONLY) as a library of its own, with the flags of the main oracle
# (Makefile): -ffp-contract=off, no fast math.  It takes its summed-area tables from the main oracle's zo_integral_plane, so it links
# against libzignal_oracle.so (built first by the main Makefile) and finds it next to itself at run time.  Bound in tests/shen_castan_oracle.py.
CXX      := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wextra -Wno-unused-parameter

libzo_shen_castan.so: zo_shen_castan.cpp zignal_oracle.h zo_common.h shen_castan.mk libzignal_oracle.so
	$(CXX) $(CXXFLAGS) -shared -o $@.tmp zo_shen_castan.cpp -L. -lzignal_oracle -Wl,-rpath,'$$ORIGIN'
	mv -f $@.tmp $@
