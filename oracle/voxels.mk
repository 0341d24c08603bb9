# oracle/voxels.mk — the oracle libraries with the point lookup (tsdf_oracle_voxels.h).  Test infrastructure only.
#
#   make -f oracle/voxels.mk          -> oracle/libtsdf_oracle_voxels.so          (restatement + orc_containing_voxels)
#   make -f oracle/voxels.mk ref      -> oracle/_ref/libcpu_tsdf_ref_voxels.so    (the reference's own src/lib/*.cpp where they
#                                        lie + ref_capi.cpp + the entry point calling octree_->getContainingVoxel)
#
# Same compiler and flags as oracle/Makefile.
CXX      := $(shell command -v /usr/bin/g++ || echo g++)
CXXFLAGS ?= -O3 -DNDEBUG -fopenmp -ffp-contract=off -fPIC -std=c++17 -Wall -Wno-unused-variable
REF      ?= /root/reference
HERE     := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))

all: $(HERE)libtsdf_oracle_voxels.so

$(HERE)libtsdf_oracle_voxels.so: $(HERE)tsdf_oracle_voxels.cpp $(HERE)tsdf_oracle_voxels.h $(HERE)tsdf_oracle.cpp $(HERE)tsdf_oracle.h $(HERE)ref_arith.h $(HERE)mc_tables.h
	$(CXX) $(CXXFLAGS) -Wno-subobject-linkage -shared -o $@ $(HERE)tsdf_oracle_voxels.cpp

REF_SRCS := $(REF)/src/lib/octree.cpp $(REF)/src/lib/tsdf_volume_octree.cpp \
            $(REF)/src/lib/marching_cubes_tsdf_octree.cpp $(REF)/src/lib/tsdf_interface.cpp

ref: $(HERE)_ref/libcpu_tsdf_ref_voxels.so

$(HERE)_ref/libcpu_tsdf_ref_voxels.so: $(HERE)ref_voxels_capi.cpp $(HERE)tsdf_oracle_voxels.h $(HERE)ref_capi.cpp $(HERE)tsdf_oracle.h $(wildcard $(HERE)compat/*/*.h $(HERE)compat/*/*/*.h $(HERE)compat/*/*/*/*.h*) $(HERE)ref_arith.h $(HERE)mc_tables.h
	@test -d $(REF) || (echo "reference tree $(REF) not present: skipping oracle/_ref" && false)
	mkdir -p $(HERE)_ref
	$(CXX) $(CXXFLAGS) -Wno-reorder -Wno-sign-compare -Wno-unused-but-set-variable -Wno-deprecated-declarations \
	    -I$(HERE)compat -I$(REF)/include -I$(HERE) -shared -o $@ $(REF_SRCS) $(HERE)ref_voxels_capi.cpp

.PHONY: all ref
