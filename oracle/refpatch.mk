# The patch scoring of updateReferencePatch (src/vio.cpp:1036-1097) for the tests of esikf_vio_score_ref_patches — test
# infrastructure only.
#   liborc_refpatch.so            : the oracle's restatement (orc_refpatch.cpp)
#   _ref/libfl2_ref_refpatch.so   : the reference's own updateReferencePatch with an empty plane map (ref_refpatch.cpp over the
#                                   driver ref_vio.cpp), built only where the reference source exists, like the other _ref
#                                   libraries
# make -C oracle -f refpatch.mk
CXX = /usr/bin/g++
REF = /root/reference
REF_REFPATCH = $(if $(wildcard $(REF)/src/vio.cpp),_ref/libfl2_ref_refpatch.so,)

all: liborc_refpatch.so $(REF_REFPATCH)

liborc_refpatch.so: orc_refpatch.cpp orc_math.hpp
	$(CXX) -std=c++17 -fPIC -shared -O2 -ffp-contract=off -Wall -Wno-unused-variable -o $@ orc_refpatch.cpp

_ref/libfl2_ref_refpatch.so: ref_refpatch.cpp ref_vio.cpp $(wildcard ref_shim/*/*) $(wildcard ref_shim/*/*/*) $(REF)/src/vio.cpp $(REF)/src/frame.cpp $(REF)/src/visual_point.cpp $(REF)/src/voxel_map.cpp $(REF)/include/vio.h
	mkdir -p _ref
	$(CXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -fopenmp -DMP_EN -DMP_PROC_NUM=4 -DROOT_DIR=\"/tmp/\" -w -I ref_shim -I $(REF)/include -o $@ ref_refpatch.cpp
