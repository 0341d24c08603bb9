/* oracle/tsdf_oracle_leaves.h — the leaf accessors of the oracle C API (tsdf_oracle.h).  TEST INFRASTRUCTURE ONLY.
 * Implemented by the restatement (tsdf_oracle_leaves.cpp -> oracle/libtsdf_oracle_leaves.so) and by the reference's own
 * methods (ref_leaves_capi.cpp -> oracle/_ref/libcpu_tsdf_ref_leaves.so); both libraries also carry the whole tsdf_oracle.h
 * API, built by oracle/leaves.mk.  Results are owned by the library until the next call of the same function (per thread). */
#ifndef TSDF_ORACLE_LEAVES_H
#define TSDF_ORACLE_LEAVES_H
#include "tsdf_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

/* TSDFVolumeOctree::getVoxelCenters (tsdf_volume_octree.cpp:576-588): centres of Octree::getLeaves (nlevels), 3 floats each */
int64_t orc_voxel_centers (const orc_volume* v, int nlevels, const float** xyz);
/* TSDFVolumeOctree::getOccupiedVoxelIndices (cpp:590-609): 3 int32 per occupied leaf */
int64_t orc_occupied_voxel_indices (const orc_volume* v, const int32_t** ijk);

#ifdef __cplusplus
}
#endif
#endif
