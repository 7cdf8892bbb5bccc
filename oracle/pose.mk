# oracle/pose.mk — the reference's own grad_cost_p (the pose-sampled obstacle penalty), beside oracle/Makefile:
#   make -C oracle -f pose.mk      _ref/libref_pose_{glibc,portable}.so
# Only where the reference tree is present (outputs git-ignored).  The shape fragments come from oracle/ref_extract.py, the map
# fragments from oracle/ref_extract_front.py (`make -C oracle ref` and `make -C oracle -f front.mk` first), the penalty's from
# oracle/ref_extract_pose.py.  Flags are the path pin's.
CXX := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
REF_SRC ?= /root/reference
REF_INC ?= /root/reference/src/utils/include
REF_PATH_FLAGS := -O3 -DNDEBUG -std=c++17 -fPIC -fopenmp -ffp-contract=off -w -Iref_shim -I$(REF_INC) -I.
ref: _ref/libref_pose_glibc.so _ref/libref_pose_portable.so
_ref/pose/gen/.stamp: ref_extract.py ref_extract_pose.py
	mkdir -p _ref/pose/gen
	python3 ref_extract_pose.py --ref $(REF_SRC) --out _ref/pose/gen
	touch $@
POSE_DEPS := ref_pose_shim.cpp ref_shape_scaffold.inc ref_shim/Eigen/Eigen ref_shim/ros/time_stub.hpp portable_sincos.hpp \
             _ref/pose/gen/.stamp _ref/front/gen/.stamp _ref/gen/.stamp
_ref/libref_pose_glibc.so: $(POSE_DEPS)
	$(CXX) $(REF_PATH_FLAGS) -shared -o $@ ref_pose_shim.cpp
_ref/libref_pose_portable.so: $(POSE_DEPS)
	$(CXX) $(REF_PATH_FLAGS) -mfma -DREF_LIBM_PORTABLE -shared -o $@ ref_pose_shim.cpp
