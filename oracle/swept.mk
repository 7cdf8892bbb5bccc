# oracle/swept.mk — the swept-volume contour checker, beside oracle/Makefile:
#   make -C oracle -f swept.mk          _build/libsvsdf_oracle_swept.so (git-ignored)
# Flags are oracle/Makefile's (no contraction: the vertices are rounded per operation, as the contract says).
CXX := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O3 -std=c++17 -fPIC -ffp-contract=off -Wall

oracle: _build/libsvsdf_oracle_swept.so
_build/libsvsdf_oracle_swept.so: swept_capi.cpp swept_oracle.hpp
	mkdir -p _build
	$(CXX) $(CXXFLAGS) -shared -o $@ swept_capi.cpp
