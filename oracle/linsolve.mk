# Builds the CPU oracle of Matrix.lu, LuResult.solve, det, inv and chol (TEST INFRASTRUCTURE ONLY) as a library of its own, with the
# flags of the main oracle (Makefile).  Bound in tests/linsolve_oracle.py.
CXX      := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wextra -Wno-unused-parameter

libzo_linsolve.so: zo_linsolve.cpp linsolve.mk
	$(CXX) $(CXXFLAGS) -shared -o $@.tmp zo_linsolve.cpp
	mv -f $@.tmp $@
