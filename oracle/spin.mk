# ORACLE — test infrastructure only: the restatement of the reference's Velodyne front end into oracle/liborcspin.so (flags as Makefile).
CXX ?= g++
CXXFLAGS ?= -B/usr/lib/gcc/x86_64-linux-gnu/13/ -O3 -march=x86-64-v3 -ffp-contract=off -fno-fast-math -std=c++17 -fPIC -Wall -Wno-unused-variable
all: liborcspin.so
liborcspin.so: spin_api.cpp orc_spin.hpp orc_cloud.hpp
	$(CXX) $(CXXFLAGS) -shared -o $@.tmp spin_api.cpp && mv -f $@.tmp $@
clean:
	rm -f liborcspin.so
