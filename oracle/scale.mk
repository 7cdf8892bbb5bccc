# oracle/scale.mk — the deformable-robot (useScale) checkers, beside oracle/Makefile:
#   make -C oracle -f scale.mk          the oracle's scaled path: _build/libsvsdf_oracle_scale{,_glibc}.so
#   make -C oracle -f scale.mk ref      the reference's own code with useScale on: _ref/libref_path_scaled_{glibc,portable}.so
#                                       (only where the reference tree is present; outputs git-ignored)
# Flags are oracle/Makefile's.
CXX := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O3 -fopenmp -std=c++17 -fPIC -mfma -ffp-contract=off -Wall -Wno-unknown-pragmas
HDRS := svsdf_oracle_scale.hpp svsdf_oracle.hpp minco_oracle.hpp shapes.hpp portable_sincos.hpp ../implicit_svsdf_planner_b200/csrc/host/fwn_bvh.hpp

oracle: _build/libsvsdf_oracle_scale.so _build/libsvsdf_oracle_scale_glibc.so
_build/libsvsdf_oracle_scale.so: oracle_scale_capi.cpp $(HDRS)
	mkdir -p _build
	$(CXX) $(CXXFLAGS) -shared -o $@ oracle_scale_capi.cpp
_build/libsvsdf_oracle_scale_glibc.so: oracle_scale_capi.cpp $(HDRS)
	mkdir -p _build
	$(CXX) $(CXXFLAGS) -DORACLE_GLIBC_SINCOS -shared -o $@ oracle_scale_capi.cpp

REF_SRC ?= /root/reference
REF_INC ?= /root/reference/src/utils/include
REF_PATH_FLAGS := -O3 -DNDEBUG -std=c++17 -fPIC -fopenmp -ffp-contract=off -w -Iref_shim -I$(REF_INC) -I.
ref: _ref/libref_path_scaled_glibc.so _ref/libref_path_scaled_portable.so
_ref/scaled/.stamp: ref_extract.py ref_extract_scale.py ref_path_shim.cpp ref_shape_scaffold.inc
	python3 ref_extract_scale.py --ref $(REF_SRC)
	touch $@
SCALED_DEPS := ref_path_scaled_shim.cpp ref_scale_hook.inc ref_shim/Eigen/Eigen portable_sincos.hpp _ref/scaled/.stamp
_ref/libref_path_scaled_glibc.so: $(SCALED_DEPS)
	$(CXX) $(REF_PATH_FLAGS) -shared -o $@ ref_path_scaled_shim.cpp
_ref/libref_path_scaled_portable.so: $(SCALED_DEPS)
	$(CXX) $(REF_PATH_FLAGS) -mfma -DREF_LIBM_PORTABLE -shared -o $@ ref_path_scaled_shim.cpp
