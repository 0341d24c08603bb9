// tests/cpp/voxels_example.cpp — getContainingVoxel of the C++ shim, single and batched.  Built (and, on a GPU box, run) by
// tests/test_cpp_voxels.py, which checks the printed records against the Python mirror.
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
  tsdf->setIntegrateColor (true);
  tsdf->reset ();
  // a fronto-parallel grey wall 1 m in front of the camera
  PointCloud<PointXYZRGBA> cloud; cloud.width = 640; cloud.height = 480; cloud.points.resize (640 * 480);
  for (int v = 0; v < 480; ++v) for (int u = 0; u < 640; ++u)
  {
    PointXYZRGBA& p = cloud.points[v * 640 + u];
    p.z = 1.0f; p.x = (u - 319.5f) / 525.f; p.y = (v - 239.5f) / 525.f; p.r = 200; p.g = 100; p.b = 50; p.a = 255;
  }
  Affine3d pose; pose.m[11] = -1.0;
  for (int i = 0; i < 3; ++i) if (!tsdf->integrateCloud (cloud, PointCloud<PointXYZRGBA> (), pose)) { std::printf ("integrate: %s\n", tsdf->lastError ()); return 1; }
  const float pts[4][3] = { { 0.01f, 0.02f, 0.003f }, { 0.01f, 0.02f, 0.003f }, { 2.f, 0.f, 0.f }, { 0.3f, -0.2f, 0.9f } };
  const float min_size[4] = { -1.f, 0.1f, -1.f, -1.f };
  std::vector<float> xyz;
  for (int i = 0; i < 4; ++i)
  {
    TSDFVolumeOctree::Voxel v = tsdf->getContainingVoxel (pts[i][0], pts[i][1], pts[i][2], min_size[i]);
    if (tsdf->status () != 0) { std::printf ("getContainingVoxel: %s\n", tsdf->lastError ()); return 1; }
    float d = 0, w = 0, cx = 0, cy = 0, cz = 0, s = 0, s2, s3; std::uint8_t r = 0, g = 0, b = 0;
    if (v.valid ()) { v.getData (d, w); v.getCenter (cx, cy, cz); v.getSize (s, s2, s3); v.getRGB (r, g, b); }
    std::printf ("voxel %d: valid=%d depth=%d d=%.9g w=%.9g c=%.9g,%.9g,%.9g size=%.9g rgb=%d,%d,%d children=%d\n", i, (int) v.valid (),
                 v.getDepth (), d, w, cx, cy, cz, s, r, g, b, (int) v.hasChildren ());
    if (min_size[i] < 0) xyz.insert (xyz.end (), pts[i], pts[i] + 3);
  }
  std::vector<b200tsdf_voxel> batch;
  tsdf->getContainingVoxel (xyz, batch);
  if (tsdf->status () != 0 || batch.size () != 3) return 1;
  if (batch[0].d != tsdf->getContainingVoxel (pts[0][0], pts[0][1], pts[0][2]).v.d || batch[1].level != -1) return 1;
  return 0;
}
