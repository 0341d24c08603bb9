// oracle/ref_voxels_capi.cpp — the oracle C API of oracle/ref_capi.cpp plus the point lookup, implemented by CALLING THE
// REFERENCE'S OWN tsdf->octree_->getContainingVoxel (x, y, z, min_size) (octree.cpp:628-634) and the returned node's
// getCenter, getSize, getData, getRGB and hasChildren.  Compiled with the reference's src/lib/*.cpp where they lie into
// oracle/_ref/libcpu_tsdf_ref_voxels.so by oracle/voxels.mk.  TEST INFRASTRUCTURE: pins the lookups (tools/make_voxel_pins.py,
// tests/test_voxels.py).  No reference source is copied.
#include "ref_capi.cpp"

#include "tsdf_oracle_voxels.h"

extern "C" {

void orc_containing_voxels (const orc_volume* v, const float* xyz, int64_t n, float min_size, orc_voxel* out)
{
  float root_size, sy, sz;
  v->tsdf->octree_->getRoot ()->getSize (root_size, sy, sz);
  for (int64_t i = 0; i < n; ++i)
  {
    orc_voxel o;
    std::memset (&o, 0, sizeof (o));
    o.level = -1;
    const cpu_tsdf::OctreeNode* nd = v->tsdf->octree_->getContainingVoxel (xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], min_size);
    if (nd)
    {
      nd->getCenter (o.cx, o.cy, o.cz);
      nd->getSize (o.size, sy, sz);
      nd->getData (o.d, o.w);
      nd->getRGB (o.r, o.g, o.b);
      o.has_children = nd->hasChildren () ? 1 : 0;
      // the node carries neither depth nor index: the size halves exactly per level, and the centre lies within a few ulps of
      // (index + 1/2) * size - root_size / 2
      int level = 0;
      for (float s = root_size; s > o.size; s *= 0.5f) ++level;
      o.level = level;
      const double half = 0.5 * (double) (1ll << level);
      o.x = (int32_t) std::floor ((double) o.cx / (double) o.size + half);
      o.y = (int32_t) std::floor ((double) o.cy / (double) o.size + half);
      o.z = (int32_t) std::floor ((double) o.cz / (double) o.size + half);
    }
    out[i] = o;
  }
}

} // extern "C"
