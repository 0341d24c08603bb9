/* oracle/tsdf_oracle_voxels.h — the point lookup of the oracle C API (tsdf_oracle.h).  TEST INFRASTRUCTURE ONLY.
 * Implemented by the restatement (tsdf_oracle_voxels.cpp -> oracle/libtsdf_oracle_voxels.so) and by the reference's own
 * Octree::getContainingVoxel and node accessors (ref_voxels_capi.cpp -> oracle/_ref/libcpu_tsdf_ref_voxels.so); both
 * libraries also carry the whole tsdf_oracle.h API, built by oracle/voxels.mk. */
#ifndef TSDF_ORACLE_VOXELS_H
#define TSDF_ORACLE_VOXELS_H
#include "tsdf_oracle.h"
#ifdef __cplusplus
extern "C" {
#endif

/* one lookup: the layout of b200tsdf_voxel (include/b200tsdf.h); level -1 and every other field 0 for NULL */
typedef struct orc_voxel
{
  int32_t level, x, y, z;
  float cx, cy, cz, size;
  float d, w;
  uint8_t r, g, b, has_children;
} orc_voxel;

/* tsdf->octree_->getContainingVoxel (x, y, z, min_size) (octree.cpp:112-121, 628-634), then getCenter, getSize, getData,
 * getRGB and hasChildren of the node, for n points (3 floats each) */
void orc_containing_voxels (const orc_volume* v, const float* xyz, int64_t n, float min_size, orc_voxel* out);

#ifdef __cplusplus
}
#endif
#endif
