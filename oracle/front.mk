# oracle/front.mk — the reference's own A* front end (node test and search), beside oracle/Makefile:
#   make -C oracle -f front.mk      _ref/libref_front_{glibc,portable}.so
# Only where the reference tree is present (outputs git-ignored).  The shape fragments come from oracle/ref_extract.py
# (`make -C oracle ref` first); the front-end fragments from oracle/ref_extract_front.py.  Flags are the path pin's.
CXX := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
REF_SRC ?= /root/reference
REF_INC ?= /root/reference/src/utils/include
REF_PATH_FLAGS := -O3 -DNDEBUG -std=c++17 -fPIC -fopenmp -ffp-contract=off -w -Iref_shim -I$(REF_INC) -I.
ref: _ref/libref_front_glibc.so _ref/libref_front_portable.so
_ref/front/gen/.stamp: ref_extract.py ref_extract_front.py
	mkdir -p _ref/front/gen
	python3 ref_extract_front.py --ref $(REF_SRC) --out _ref/front/gen
	touch $@
FRONT_DEPS := ref_front_shim.cpp ref_shape_scaffold.inc ref_shim/Eigen/Eigen ref_shim/ros/time_stub.hpp portable_sincos.hpp \
              _ref/front/gen/.stamp _ref/gen/.stamp
_ref/libref_front_glibc.so: $(FRONT_DEPS)
	$(CXX) $(REF_PATH_FLAGS) -shared -o $@ ref_front_shim.cpp
_ref/libref_front_portable.so: $(FRONT_DEPS)
	$(CXX) $(REF_PATH_FLAGS) -mfma -DREF_LIBM_PORTABLE -shared -o $@ ref_front_shim.cpp
