// oracle/ref_leaves_capi.cpp — the oracle C API of oracle/ref_capi.cpp plus the leaf accessors, implemented by CALLING
// THE REFERENCE'S OWN TSDFVolumeOctree::getVoxelCenters / getOccupiedVoxelIndices (tsdf_volume_octree.cpp:576-609).
// Compiled with the reference's src/lib/*.cpp where they lie into oracle/_ref/libcpu_tsdf_ref_leaves.so by oracle/leaves.mk.
// TEST INFRASTRUCTURE: pins the leaf lists (tools/make_leaf_pins.py, tests/test_leaves.py).  No reference source is copied.
#include "ref_capi.cpp"

#include "tsdf_oracle_leaves.h"

namespace {
thread_local std::vector<float> g_centers;
thread_local std::vector<int32_t> g_indices;
}

extern "C" {

int64_t orc_voxel_centers (const orc_volume* v, int nlevels, const float** xyz)
{
  pcl::PointCloud<pcl::PointXYZ>::ConstPtr c = v->tsdf->getVoxelCenters (nlevels);
  g_centers.resize (3 * c->size ());
  for (size_t i = 0; i < c->size (); ++i)
  { g_centers[3 * i] = c->points[i].x; g_centers[3 * i + 1] = c->points[i].y; g_centers[3 * i + 2] = c->points[i].z; }
  if (xyz) *xyz = g_centers.data ();
  return static_cast<int64_t> (c->size ());
}

int64_t orc_occupied_voxel_indices (const orc_volume* v, const int32_t** ijk)
{
  std::vector<Eigen::Vector3i> idx;
  v->tsdf->getOccupiedVoxelIndices (idx);
  g_indices.resize (3 * idx.size ());
  for (size_t i = 0; i < idx.size (); ++i) for (int k = 0; k < 3; ++k) g_indices[3 * i + k] = idx[i] (k);
  if (ijk) *ijk = g_indices.data ();
  return static_cast<int64_t> (idx.size ());
}

} // extern "C"
