# New observations of the visual sub-map in a VIO tick (updateVisualMapPoints, src/vio.cpp:908-967) for the tests of
# esikf_vio_update_points — test infrastructure only.
#   liborc_observe.so             : the oracle's restatement (orc_observe.cpp) linked with the parity oracle's translation units
#   _ref/libfl2_ref_observe.so    : the reference's own updateVisualMapPoints (ref_observe.cpp over the driver ref_vio.cpp),
#                                   built only where the reference source exists, like the other _ref libraries (see Makefile)
# make -C oracle -f observe.mk
CXX = /usr/bin/g++
REF = /root/reference
REF_OBSERVE = $(if $(wildcard $(REF)/src/vio.cpp),_ref/libfl2_ref_observe.so,)
ORC = orc_lio.cpp orc_vio.cpp orc_capi.cpp

all: liborc_observe.so $(REF_OBSERVE)

liborc_observe.so: orc_observe.cpp $(ORC) orc_math.hpp orc_lio.hpp orc_vio.hpp
	$(CXX) -std=c++17 -fPIC -shared -fopenmp -O2 -ffp-contract=off -Wall -Wno-unused-variable -o $@ orc_observe.cpp $(ORC)

_ref/libfl2_ref_observe.so: ref_observe.cpp ref_vio.cpp $(wildcard ref_shim/*/*) $(wildcard ref_shim/*/*/*) $(REF)/src/vio.cpp $(REF)/src/frame.cpp $(REF)/src/visual_point.cpp $(REF)/src/voxel_map.cpp $(REF)/include/vio.h
	mkdir -p _ref
	$(CXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -fopenmp -DMP_EN -DMP_PROC_NUM=4 -DROOT_DIR=\"/tmp/\" -w -I ref_shim -I $(REF)/include -o $@ ref_observe.cpp
