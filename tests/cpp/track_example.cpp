// tests/cpp/track_example.cpp — tracking through the C++ shim: trackDepthImage for a uint16 and a float map and a refused
// call.  Built (and, on a GPU box, run) by tests/test_cpp_track.py, which repeats the same calls through the Python mirror and
// compares the printed lines.
#include "../../include/cpu_tsdf_b200/tsdf_volume_octree.h"
#include <cstdio>
#include <vector>
using namespace cpu_tsdf_b200;

int main ()
{
  TSDFVolumeOctree::Ptr tsdf (new TSDFVolumeOctree (0, 14));
  if (!tsdf->ok ()) { std::printf ("no device: %d (%s)\n", tsdf->status (), tsdf->lastError ()); return tsdf->status () == B200TSDF_ENODEVICE ? 3 : 1; }
  tsdf->setGridSize (3.f, 3.f, 3.f);
  tsdf->setResolution (256, 256, 256);
  tsdf->setCameraIntrinsics (525., 525., 319.5, 239.5);
  tsdf->reset ();
  // a wall 1 m in front of the camera, tilted in x and y
  const int W = 640, H = 480;
  std::vector<std::uint16_t> d16 (W * H);
  std::vector<float> d32 (W * H);
  for (int v = 0; v < H; ++v) for (int u = 0; u < W; ++u)
  {
    d16[v * W + u] = (std::uint16_t) (1000 + u / 8 + v / 16);
    d32[v * W + u] = d16[v * W + u] * 1e-3f;
  }
  Affine3d pose; pose.m[11] = -1.0;
  for (int i = 0; i < 2; ++i)
    if (!tsdf->integrateDepthImage (d16.data (), 1e-3f, W, H, pose)) { std::printf ("integrate: %s\n", tsdf->lastError ()); return 1; }
  Affine3d a; a.m[11] = -1.0; a.m[3] = 0.01;                          // start 1 cm off along x
  b200tsdf_track_result r;
  if (!tsdf->trackDepthImage (d16.data (), 1e-3f, W, H, a, nullptr, &r)) { std::printf ("track u16: %s\n", tsdf->lastError ()); return 1; }
  std::printf ("u16: %d %d %.17g %.17g %.17g\n", r.status, r.inliers, a.m[3], a.m[7], a.m[11]);
  Affine3d b; b.m[11] = -1.02;
  if (!tsdf->trackDepthImage (d32.data (), W, H, b)) { std::printf ("track f32: %s\n", tsdf->lastError ()); return 1; }
  std::printf ("f32: %.17g %.17g %.17g\n", b.m[3], b.m[7], b.m[11]);
  b200tsdf_track_params bad;
  b200tsdf_default_track_params (&bad);
  bad.levels = 0;
  const bool refused = !tsdf->trackDepthImage (d32.data (), W, H, b, &bad);
  std::printf ("refused: %d %d\n", (int) refused, tsdf->status ());
  return 0;
}
