// tests/cpp/shim_resize.cpp — resizePool through the C++ shim: start with a small brick pool, fuse, grow, fuse and mesh, and
// end equal to a handle that had the large pool from the start.  Built (and, on a GPU box, run) by tests/test_pool_resize_gpu.py.
#include "../../include/cpu_tsdf_b200/tsdf_volume_octree.h"
#include <cstdio>
#include <vector>
using namespace cpu_tsdf_b200;

static TSDFVolumeOctree::Ptr make (int pool_log2)
{
  TSDFVolumeOctree::Ptr t (new TSDFVolumeOctree (0, pool_log2));
  t->setGridSize (3.f, 3.f, 3.f);
  t->setResolution (256, 256, 256);
  t->setCameraIntrinsics (525., 525., 319.5, 239.5);
  t->reset ();
  return t;
}

int main ()
{
  TSDFVolumeOctree::Ptr a = make (11), b = make (14);
  if (!a->ok ()) { std::printf ("no device: %d (%s)\n", a->status (), a->lastError ()); return a->status () == B200TSDF_ENODEVICE ? 3 : 1; }
  // a tilted wall in front of the camera
  PointCloud<PointXYZ> cloud; cloud.width = 640; cloud.height = 480; cloud.points.resize (640 * 480);
  for (int v = 0; v < 480; ++v) for (int u = 0; u < 640; ++u)
  {
    const float x = (u - 319.5f) / 525.f, y = (v - 239.5f) / 525.f, z = 1.0f / (1.0f + 0.3f * x);
    PointXYZ& p = cloud.points[v * 640 + u]; p.x = x * z; p.y = y * z; p.z = z;
  }
  Affine3d pose; pose.m[11] = -1.0;
  if (!a->integrateCloud (cloud, PointCloud<PointXYZ> (), pose) || !b->integrateCloud (cloud, PointCloud<PointXYZ> (), pose)) { std::printf ("integrate: %s\n", a->lastError ()); return 1; }
  if (a->resizePool (8) || a->status () != B200TSDF_EINVAL) { std::printf ("a pool below the load limit was not refused\n"); return 1; }
  if (!a->resizePool (14)) { std::printf ("resizePool: %s\n", a->lastError ()); return 1; }
  for (int i = 0; i < 2; ++i)
    if (!a->integrateCloud (cloud, PointCloud<PointXYZ> (), pose) || !b->integrateCloud (cloud, PointCloud<PointXYZ> (), pose)) { std::printf ("integrate: %s\n", a->lastError ()); return 1; }
  TriangleSoup ma, mb;
  for (int k = 0; k < 2; ++k)
  {
    MarchingCubesTSDFOctree mc;
    mc.setInputTSDF (k ? b : a);
    mc.setMinWeight (2);
    mc.setColorByRGB (false);
    if (!mc.reconstruct (k ? mb : ma)) return 1;
  }
  std::printf ("mesh: %zu triangles after the resize, %zu on the handle created with the pool\n", ma.xyz.size () / 9, mb.xyz.size () / 9);
  if (ma.xyz.empty () || ma.xyz != mb.xyz) return 1;
  return 0;
}
