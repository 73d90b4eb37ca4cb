# The visual map's observation store for the tests of esikf_vmap_* — test infrastructure only.
#   liborc_vmap.so          : the oracle's restatement of the list edits of updateVisualMapPoints (src/vio.cpp:914-964) and the
#                             retrieval's reference-feature choice (:651-697) on a host copy of the store (orc_vmap.cpp)
#   _ref/libfl2_ref_vmap.so : the reference's own VisualPoint / Feature objects kept across calls and changed by its own
#                             updateVisualMapPoints, updateReferencePatch and getCloseViewObs (ref_vmap.cpp over the driver
#                             ref_vio.cpp), built only where the reference source exists, like the other _ref libraries
# make -C oracle -f vmap.mk
CXX = /usr/bin/g++
REF = /root/reference
REF_VMAP = $(if $(wildcard $(REF)/src/vio.cpp),_ref/libfl2_ref_vmap.so,)

all: liborc_vmap.so $(REF_VMAP)

liborc_vmap.so: orc_vmap.cpp
	$(CXX) -std=c++17 -fPIC -shared -O2 -ffp-contract=off -Wall -o $@ orc_vmap.cpp

_ref/libfl2_ref_vmap.so: ref_vmap.cpp ref_vio.cpp $(wildcard ref_shim/*/*) $(wildcard ref_shim/*/*/*) $(REF)/src/vio.cpp $(REF)/src/frame.cpp $(REF)/src/visual_point.cpp $(REF)/src/voxel_map.cpp $(REF)/include/vio.h
	mkdir -p _ref
	$(CXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -fopenmp -DMP_EN -DMP_PROC_NUM=4 -DROOT_DIR=\"/tmp/\" -w -I ref_shim -I $(REF)/include -o $@ ref_vmap.cpp
