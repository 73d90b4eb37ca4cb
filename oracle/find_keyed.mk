# The VIO front end's keyed find_correspond lookups (updateReferencePatch, the retrieval's ray casting) for the tests of
# esikf_map_device_find — test infrastructure only.
#   liborc_find_keyed.so        : the oracle's restatement (orc_find_keyed.cpp, which includes orc_find.cpp), handed OracleLIO
#                                 handles of liborc_parity.so
#   _ref/libfl2_ref_find_keyed.so : the reference's own updateReferencePatch and ray-casting retrieval on the reference's own map
#                                 (ref_find_keyed.cpp over the driver ref_vio.cpp), built only where the reference source exists,
#                                 like the other _ref libraries
# make -C oracle -f find_keyed.mk
CXX = /usr/bin/g++
REF = /root/reference
REF_FIND_KEYED = $(if $(wildcard $(REF)/src/vio.cpp),_ref/libfl2_ref_find_keyed.so,)

all: liborc_find_keyed.so $(REF_FIND_KEYED)

liborc_find_keyed.so: orc_find_keyed.cpp orc_find.cpp orc_lio.hpp orc_math.hpp
	$(CXX) -std=c++17 -fPIC -shared -O2 -ffp-contract=off -Wall -Wno-unused-variable -o $@ orc_find_keyed.cpp

_ref/libfl2_ref_find_keyed.so: ref_find_keyed.cpp ref_vio.cpp $(wildcard ref_shim/*/*) $(wildcard ref_shim/*/*/*) $(REF)/src/vio.cpp $(REF)/src/frame.cpp $(REF)/src/visual_point.cpp $(REF)/src/voxel_map.cpp $(REF)/include/vio.h
	mkdir -p _ref
	$(CXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -fopenmp -DMP_EN -DMP_PROC_NUM=4 -DROOT_DIR=\"/tmp/\" -w -I ref_shim -I $(REF)/include -o $@ ref_find_keyed.cpp
