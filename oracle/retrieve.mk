# Scan side of the visual sub-map retrieval (retrieveFromVisualSparseMap, src/vio.cpp:352-640, raycast_en off) for the tests of
# esikf_vio_retrieve_scan / esikf_vio_depth_check — test infrastructure only.
#   liborc_retrieve.so            : the oracle's restatement (orc_retrieve.cpp) linked with the parity oracle's translation units
#   _ref/libfl2_ref_retrieve.so   : the reference's own resetGrid + retrieveFromVisualSparseMap (ref_retrieve.cpp over the driver
#                                   ref_vio.cpp), built only where the reference source exists, like the other _ref libraries
# make -C oracle -f retrieve.mk
CXX = /usr/bin/g++
REF = /root/reference
REF_RETRIEVE = $(if $(wildcard $(REF)/src/vio.cpp),_ref/libfl2_ref_retrieve.so,)
ORC = orc_lio.cpp orc_vio.cpp orc_capi.cpp

all: liborc_retrieve.so $(REF_RETRIEVE)

liborc_retrieve.so: orc_retrieve.cpp $(ORC) orc_math.hpp orc_lio.hpp orc_vio.hpp
	$(CXX) -std=c++17 -fPIC -shared -fopenmp -O2 -ffp-contract=off -Wall -Wno-unused-variable -o $@ orc_retrieve.cpp $(ORC)

_ref/libfl2_ref_retrieve.so: ref_retrieve.cpp ref_vio.cpp $(wildcard ref_shim/*/*) $(wildcard ref_shim/*/*/*) $(REF)/src/vio.cpp $(REF)/src/frame.cpp $(REF)/src/visual_point.cpp $(REF)/src/voxel_map.cpp $(REF)/include/vio.h
	mkdir -p _ref
	$(CXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -fopenmp -DMP_EN -DMP_PROC_NUM=4 -DROOT_DIR=\"/tmp/\" -w -I ref_shim -I $(REF)/include -o $@ ref_retrieve.cpp
