// tests/cpp/depth_example.cpp — depth images through the C++ shim: integrateDepthImage for uint16 and float maps, with and
// without colour, and a refused call.  Built (and, on a GPU box, run) by tests/test_cpp_depth.py, which repeats the same calls
// through the Python mirror and compares the printed lines.
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
  tsdf->setIntegrateColor (true);
  tsdf->reset ();
  // a wall 1 m in front of the camera with a hole in the middle (depth 0), tilted in x; red-green gradient
  const int W = 640, H = 480;
  std::vector<std::uint16_t> d16 (W * H);
  std::vector<float> d32 (W * H);
  std::vector<std::uint8_t> rgb (W * H * 3);
  for (int v = 0; v < H; ++v) for (int u = 0; u < W; ++u)
  {
    const int i = v * W + u;
    const bool hole = u > 300 && u < 340 && v > 220 && v < 260;
    d16[i] = hole ? 0 : (std::uint16_t) (1000 + u / 8);
    d32[i] = hole ? 0.f : 1.0f + 0.0005f * v;
    rgb[3 * i] = (std::uint8_t) (u / 3); rgb[3 * i + 1] = (std::uint8_t) (v / 2); rgb[3 * i + 2] = 77;
  }
  Affine3d pose; pose.m[11] = -1.0;
  for (int i = 0; i < 2; ++i)
    if (!tsdf->integrateDepthImage (d16.data (), 1e-3f, W, H, pose, rgb.data ())) { std::printf ("integrate u16: %s\n", tsdf->lastError ()); return 1; }
  if (!tsdf->integrateDepthImage (d32.data (), W, H, pose)) { std::printf ("integrate f32: %s\n", tsdf->lastError ()); return 1; }
  const bool refused = !tsdf->integrateDepthImage (d16.data (), 0.f, W, H, pose);
  std::printf ("refused: %d %d\n", (int) refused, tsdf->status ());
  if (!tsdf->integrateDepthImagesDevice ({}, B200TSDF_DEPTH_U16, 1e-3f, W, H, {})) { std::printf ("empty batch: %s\n", tsdf->lastError ()); return 1; }
  const float pts[4][3] = { { 0.f, 0.f, 0.f }, { 0.1f, -0.05f, 0.02f }, { -0.3f, 0.2f, -0.01f }, { 0.f, 0.f, 0.5f } };
  for (int i = 0; i < 4; ++i)
  {
    float val = 0.f;
    PointXYZ q; q.x = pts[i][0]; q.y = pts[i][1]; q.z = pts[i][2];
    const bool ok = tsdf->getFxn (q, val);
    std::printf ("fxn %d: %d %.9g\n", i, (int) ok, ok ? val : 0.f);
  }
  return 0;
}
