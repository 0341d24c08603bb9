// oracle/tsdf_oracle_voxels.cpp — the restatement (tsdf_oracle.cpp) plus getContainingVoxel (x, y, z, min_size) over its pool
// octree: the restated Octree::getContainingVoxel bounds (octree.cpp:628-634), OctreeNode::getContainingVoxel with min_size
// (:112-121) and the node's accessors (getCenter / getSize :52-66, getData :124-130, getRGB :173-178 and the colour nodes'
// overrides, hasChildren :41-45).  Built by oracle/voxels.mk into oracle/libtsdf_oracle_voxels.so.  TEST INFRASTRUCTURE ONLY.
#include "tsdf_oracle.cpp"

#include "tsdf_oracle_voxels.h"

extern "C" {

void orc_containing_voxels (const orc_volume* v, const float* xyz, int64_t n, float min_size, orc_voxel* out)
{
  for (int64_t i = 0; i < n; ++i)
  {
    const float x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    orc_voxel o;
    std::memset (&o, 0, sizeof (o));
    o.level = -1;
    if (!(std::isnan (z) || std::fabs (x) > v->c.xsize / 2 || std::fabs (y) > v->c.ysize / 2 || std::fabs (z) > v->c.zsize / 2))
    {
      int32_t ni = v->root;
      for (;;)
      {
        const Node& nd = v->pool.at (ni);
        if (nd.child < 0 || (min_size > 0 && nd.size <= min_size)) break;
        ni = nd.child + ((x - nd.cx) > 0) * 4 + ((y - nd.cy) > 0) * 2 + ((z - nd.cz) > 0);
      }
      const Node& nd = v->pool.at (ni);
      o.level = nd.level; o.x = nd.ix; o.y = nd.iy; o.z = nd.iz;
      o.cx = nd.cx; o.cy = nd.cy; o.cz = nd.cz; o.size = nd.size;
      o.d = nd.d; o.w = nd.w;
      if (v->color) v->get_rgb (nd, o.r, o.g, o.b);
      else o.r = o.g = o.b = 127;
      o.has_children = nd.child >= 0 ? 1 : 0;
    }
    out[i] = o;
  }
}

} // extern "C"
