# The map side of the visual sub-map retrieval (insertPointIntoVoxelMap and retrieveFromVisualSparseMap, src/vio.cpp:227-250,
# 352-782, raycast_en off) for the tests of esikf_vmap_place_points / esikf_vmap_retrieve — test infrastructure only.
#   _ref/libfl2_ref_vretrieve.so : the reference's own insertion and retrieval on one VIOManager kept across ticks
#                                  (ref_vretrieve.cpp over the driver ref_vio.cpp), built only where the reference source
#                                  exists, like the other _ref libraries. The restatement it pins is tests/vmap_retrieve_cases.py
#                                  over oracle/liborc_retrieve.so (retrieve.mk) and oracle/liborc_vmap.so (vmap.mk).
# make -C oracle -f vmap_retrieve.mk
CXX = /usr/bin/g++
REF = /root/reference
REF_VRETRIEVE = $(if $(wildcard $(REF)/src/vio.cpp),_ref/libfl2_ref_vretrieve.so,)

all: $(REF_VRETRIEVE)

_ref/libfl2_ref_vretrieve.so: ref_vretrieve.cpp ref_vio.cpp $(wildcard ref_shim/*/*) $(wildcard ref_shim/*/*/*) $(REF)/src/vio.cpp $(REF)/src/frame.cpp $(REF)/src/visual_point.cpp $(REF)/src/voxel_map.cpp $(REF)/include/vio.h
	mkdir -p _ref
	$(CXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -fopenmp -DMP_EN -DMP_PROC_NUM=4 -DROOT_DIR=\"/tmp/\" -w -I ref_shim -I $(REF)/include -o $@ ref_vretrieve.cpp
