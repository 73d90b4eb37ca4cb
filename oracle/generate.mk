# New visual map points of a VIO tick (generateVisualMapPoints, src/vio.cpp:804-906) for the tests of
# esikf_vio_generate_points — test infrastructure only.
#   liborc_generate.so             : the oracle's restatement (orc_generate.cpp) linked with the parity oracle's translation units
#   _ref/libfl2_ref_generate.so    : the reference's own generateVisualMapPoints (ref_generate.cpp over the driver ref_vio.cpp),
#                                    built only where the reference source exists, like the other _ref libraries (see Makefile)
# make -C oracle -f generate.mk
CXX = /usr/bin/g++
REF = /root/reference
REF_GENERATE = $(if $(wildcard $(REF)/src/vio.cpp),_ref/libfl2_ref_generate.so,)
ORC = orc_lio.cpp orc_vio.cpp orc_capi.cpp

all: liborc_generate.so $(REF_GENERATE)

liborc_generate.so: orc_generate.cpp $(ORC) orc_math.hpp orc_lio.hpp orc_vio.hpp
	$(CXX) -std=c++17 -fPIC -shared -fopenmp -O2 -ffp-contract=off -Wall -Wno-unused-variable -o $@ orc_generate.cpp $(ORC)

_ref/libfl2_ref_generate.so: ref_generate.cpp ref_vio.cpp $(wildcard ref_shim/*/*) $(wildcard ref_shim/*/*/*) $(REF)/src/vio.cpp $(REF)/src/frame.cpp $(REF)/src/visual_point.cpp $(REF)/src/voxel_map.cpp $(REF)/include/vio.h
	mkdir -p _ref
	$(CXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -fopenmp -DMP_EN -DMP_PROC_NUM=4 -DROOT_DIR=\"/tmp/\" -w -I ref_shim -I $(REF)/include -o $@ ref_generate.cpp
