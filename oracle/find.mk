# find_correspond (src/voxel_map.cpp:292-305) for the tests of the host mirror of the device map — test infrastructure only.
#   liborc_find.so                : the oracle's restatement (orc_find.cpp), handed OracleLIO handles of liborc_parity.so
#   _ref/libfl2_ref_find.so       : the reference's own source (ref_find.cpp over the driver ref_voxel_map.cpp), built only
#                                   where the reference source exists, like the other _ref libraries (see Makefile)
# make -C oracle -f find.mk
CXX = /usr/bin/g++
REF = /root/reference
REF_FIND = $(if $(wildcard $(REF)/src/voxel_map.cpp),_ref/libfl2_ref_find.so,)

all: liborc_find.so $(REF_FIND)

liborc_find.so: orc_find.cpp orc_lio.hpp orc_math.hpp
	$(CXX) -std=c++17 -fPIC -shared -O2 -ffp-contract=off -Wall -Wno-unused-variable -o $@ orc_find.cpp

_ref/libfl2_ref_find.so: ref_find.cpp ref_voxel_map.cpp $(wildcard ref_shim/*/*) $(REF)/src/voxel_map.cpp $(REF)/include/voxel_map.h $(REF)/include/common_lib.h
	mkdir -p _ref
	$(CXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -fopenmp -DMP_EN -DMP_PROC_NUM=4 -w -I ref_shim -I $(REF)/include -o $@ ref_find.cpp
