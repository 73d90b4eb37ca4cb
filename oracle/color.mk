# The coloured scan of publish_frame_world (src/LIVMapper.cpp:435-443, 1140-1173) for the tests of esikf_rgb_set_cloud /
# esikf_rgb_colorize — test infrastructure only.
#   liborc_color.so              : the oracle's restatement (orc_color.cpp) linked with the parity oracle's translation units
#   _ref/libfl2_ref_color.so     : the reference's own updateFrameState / w2f / w2c / isInFrame / getInterpolatedPixel
#                                  (ref_color.cpp over the driver ref_vio.cpp), built only where the reference source exists,
#                                  like the other _ref libraries (see Makefile)
# make -C oracle -f color.mk
CXX = /usr/bin/g++
REF = /root/reference
REF_COLOR = $(if $(wildcard $(REF)/src/vio.cpp),_ref/libfl2_ref_color.so,)
ORC = orc_lio.cpp orc_vio.cpp orc_capi.cpp

all: liborc_color.so $(REF_COLOR)

liborc_color.so: orc_color.cpp $(ORC) orc_math.hpp orc_lio.hpp orc_vio.hpp
	$(CXX) -std=c++17 -fPIC -shared -fopenmp -O2 -ffp-contract=off -Wall -Wno-unused-variable -o $@ orc_color.cpp $(ORC)

_ref/libfl2_ref_color.so: ref_color.cpp ref_vio.cpp $(wildcard ref_shim/*/*) $(wildcard ref_shim/*/*/*) $(REF)/src/vio.cpp $(REF)/src/frame.cpp $(REF)/src/visual_point.cpp $(REF)/src/voxel_map.cpp $(REF)/include/vio.h
	mkdir -p _ref
	$(CXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -fopenmp -DMP_EN -DMP_PROC_NUM=4 -DROOT_DIR=\"/tmp/\" -w -I ref_shim -I $(REF)/include -o $@ ref_color.cpp
