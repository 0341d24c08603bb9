// tests/cpp/leaves_example.cpp — the leaf accessors of the C++ shim: getVoxelCenters, getOccupiedVoxelIndices, isEmpty,
// getIntensityCloud, getFrustumCulledVoxels.  Built (and, on a GPU box, run) by tests/test_cpp_leaves.py, which checks the
// printed counts against the Python mirror.
#include "../../include/cpu_tsdf_b200/tsdf_volume_octree.h"
#include <cstdio>
using namespace cpu_tsdf_b200;

int main ()
{
  TSDFVolumeOctree::Ptr tsdf (new TSDFVolumeOctree (0, 14));
  if (!tsdf->ok ()) { std::printf ("no device: %d (%s)\n", tsdf->status (), tsdf->lastError ()); return tsdf->status () == B200TSDF_ENODEVICE ? 3 : 1; }
  tsdf->setGridSize (3.f, 3.f, 3.f);
  tsdf->setResolution (256, 256, 256);
  tsdf->setCameraIntrinsics (525., 525., 319.5, 239.5);
  tsdf->reset ();
  if (tsdf->status () != 0 || !tsdf->isEmpty ()) { std::printf ("reset: %s\n", tsdf->lastError ()); return 1; }
  // a fronto-parallel wall 1 m in front of the camera (as in shim_example.cpp)
  PointCloud<PointXYZ> cloud; cloud.width = 640; cloud.height = 480; cloud.points.resize (640 * 480);
  for (int v = 0; v < 480; ++v) for (int u = 0; u < 640; ++u)
  {
    PointXYZ& p = cloud.points[v * 640 + u];
    p.z = 1.0f; p.x = (u - 319.5f) / 525.f; p.y = (v - 239.5f) / 525.f;
  }
  Affine3d pose; pose.m[11] = -1.0;
  for (int i = 0; i < 3; ++i) if (!tsdf->integrateCloud (cloud, PointCloud<PointXYZ> (), pose)) { std::printf ("integrate: %s\n", tsdf->lastError ()); return 1; }
  if (tsdf->isEmpty ()) return 1;
  PointCloud<PointXYZ>::ConstPtr c4 = tsdf->getVoxelCenters ();
  PointCloud<PointXYZ>::ConstPtr all = tsdf->getVoxelCenters (-1);
  PointCloud<PointXYZ>::ConstPtr root = tsdf->getVoxelCenters (0);
  if (tsdf->status () != 0 || root->size () != 1 || root->points[0].x != 0.f) { std::printf ("getVoxelCenters: %s\n", tsdf->lastError ()); return 1; }
  std::vector<Vector3i> occ;
  tsdf->getOccupiedVoxelIndices (occ);
  if (tsdf->status () != 0 || occ.empty ()) { std::printf ("getOccupiedVoxelIndices: %s\n", tsdf->lastError ()); return 1; }
  std::vector<PointXYZ> culled;
  tsdf->getFrustumCulledVoxels (pose, culled);
  if (tsdf->status () != 0 || culled.empty ()) { std::printf ("getFrustumCulledVoxels: %s\n", tsdf->lastError ()); return 1; }
  if (tsdf->getIntensityCloud (pose)) return 1;                  // the reference's stub returns a null cloud
  // the wall is the plane z = 0: every occupied voxel sits next to it
  for (const Vector3i& v : occ) if (v.z < 120 || v.z > 135) { std::printf ("occupied voxel off the wall: %d %d %d\n", v.x, v.y, v.z); return 1; }
  std::printf ("leaves: centers4=%zu centers-1=%zu occupied=%zu culled=%zu first_culled=%.6f,%.6f,%.6f\n", c4->size (), all->size (),
               occ.size (), culled.size (), culled[0].x, culled[0].y, culled[0].z);
  tsdf->reset ();
  if (!tsdf->isEmpty () || tsdf->getVoxelCenters (-1)->size () != 512) return 1;
  return 0;
}
