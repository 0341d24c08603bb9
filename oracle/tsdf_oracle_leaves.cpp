// oracle/tsdf_oracle_leaves.cpp — the restatement (tsdf_oracle.cpp) plus getVoxelCenters / getOccupiedVoxelIndices over its
// pool octree: Octree::getLeaves (octree.cpp:608-617) through the restated OctreeNode::getLeaves (get_leaves, :99-109), the
// centres stored at split time (getCenter, octree.cpp:53-58) and the restated getVoxelIndex.  Built by oracle/leaves.mk into
// oracle/libtsdf_oracle_leaves.so.  TEST INFRASTRUCTURE ONLY.
#include "tsdf_oracle.cpp"

#include "tsdf_oracle_leaves.h"

namespace {
thread_local std::vector<float> g_centers;
thread_local std::vector<int32_t> g_indices;

// Octree::getLeaves (leaves, num_levels), octree.cpp:608-617
std::vector<int32_t> octree_leaves (const orc_volume* v, int num_levels)
{
  std::vector<int32_t> out;
  if (num_levels == 0) out.push_back (v->root);
  else v->get_leaves (v->root, out, num_levels - 1);
  return out;
}
}

extern "C" {

// tsdf_volume_octree.cpp:576-588
int64_t orc_voxel_centers (const orc_volume* v, int nlevels, const float** xyz)
{
  const std::vector<int32_t> lv = octree_leaves (v, nlevels);
  g_centers.resize (3 * lv.size ());
  for (size_t i = 0; i < lv.size (); ++i)
  {
    const Node& n = v->pool.at (lv[i]);
    g_centers[3 * i] = n.cx; g_centers[3 * i + 1] = n.cy; g_centers[3 * i + 2] = n.cz;
  }
  if (xyz) *xyz = g_centers.data ();
  return static_cast<int64_t> (lv.size ());
}

// tsdf_volume_octree.cpp:590-609
int64_t orc_occupied_voxel_indices (const orc_volume* v, const int32_t** ijk)
{
  const std::vector<int32_t> lv = octree_leaves (v, -1);
  g_indices.clear ();
  for (int32_t ni : lv)
  {
    const Node& n = v->pool.at (ni);
    if (n.w > 0 && std::fabs (n.d) < 1)
    {
      int x, y, z;
      v->voxel_index (n.cx, n.cy, n.cz, x, y, z);
      g_indices.push_back (x); g_indices.push_back (y); g_indices.push_back (z);
    }
  }
  if (ijk) *ijk = g_indices.data ();
  return static_cast<int64_t> (g_indices.size () / 3);
}

} // extern "C"
