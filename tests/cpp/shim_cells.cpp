// tests/cpp/shim_cells.cpp — incremental meshing through the C++ shim: fuse a frame, fuse another, ask changedCells which
// coarse cells changed, mesh those cells into device memory with reconstructCellsDevice, and check every selected cell's run
// of vertices against the same cell's run in the host reconstruct ().  Built (and, on a GPU box, run) by
// tests/test_mesh_incremental_gpu.py.
#include "../../include/cpu_tsdf_b200/tsdf_volume_octree.h"
#include <cuda_runtime.h>
#include <cstdio>
#include <cstring>
#include <vector>
using namespace cpu_tsdf_b200;

// perm[k] = the layout index ((x n + y) n + z) of the k-th coarse cell in depth-first (Morton) order: the mesh's cell order
static std::vector<std::size_t> morton_cells (std::size_t ncells)
{
  int bits = 0;
  while (((std::size_t) 1 << (3 * (bits + 1))) <= ncells) ++bits;
  const std::size_t n = (std::size_t) 1 << bits;
  std::vector<std::size_t> perm (ncells);
  for (std::size_t k = 0; k < ncells; ++k)
  {
    std::size_t x = 0, y = 0, z = 0;
    for (int l = bits - 1; l >= 0; --l)
    {
      const std::size_t c = (k >> (3 * l)) & 7;
      x = (x << 1) | (c >> 2); y = (y << 1) | ((c >> 1) & 1); z = (z << 1) | (c & 1);
    }
    perm[k] = (x * n + y) * n + z;
  }
  return perm;
}

// a tilted wall in front of the camera at depth z0
static PointCloud<PointXYZ> wall (float z0)
{
  PointCloud<PointXYZ> cloud; cloud.width = 640; cloud.height = 480; cloud.points.resize (640 * 480);
  for (int v = 0; v < 480; ++v) for (int u = 0; u < 640; ++u)
  {
    const float x = (u - 319.5f) / 525.f, y = (v - 239.5f) / 525.f, z = z0 / (1.0f + 0.3f * x);
    PointXYZ& p = cloud.points[v * 640 + u]; p.x = x * z; p.y = y * z; p.z = z;
  }
  return cloud;
}

int main ()
{
  TSDFVolumeOctree::Ptr t (new TSDFVolumeOctree (0, 14));
  t->setGridSize (3.f, 3.f, 3.f);
  t->setResolution (256, 256, 256);
  t->setCameraIntrinsics (525., 525., 319.5, 239.5);
  t->reset ();
  if (!t->ok ()) { std::printf ("no device: %d (%s)\n", t->status (), t->lastError ()); return t->status () == B200TSDF_ENODEVICE ? 3 : 1; }
  Affine3d pose; pose.m[11] = -1.0;
  for (int i = 0; i < 2; ++i)
    if (!t->integrateCloud (wall (1.0f), PointCloud<PointXYZ> (), pose)) { std::printf ("integrate: %s\n", t->lastError ()); return 1; }
  std::uint64_t e1 = 0, e2 = 0;
  if (!t->changedCells (0, &e1)) { std::printf ("changedCells: %s\n", t->lastError ()); return 1; }
  // a second wall further away: only the cells near it change
  Affine3d pose2; pose2.m[11] = -1.0; pose2.m[3] = 0.4;
  for (int i = 0; i < 2; ++i)
    if (!t->integrateCloud (wall (0.7f), PointCloud<PointXYZ> (), pose2)) { std::printf ("integrate: %s\n", t->lastError ()); return 1; }
  std::vector<std::uint8_t> mask;
  if (!t->changedCells (e1, &e2, &mask) || e2 != e1 + 2) { std::printf ("changedCells: %s (epochs %llu -> %llu)\n", t->lastError (), (unsigned long long) e1, (unsigned long long) e2); return 1; }

  MarchingCubesTSDFOctree mc;
  mc.setInputTSDF (t);
  mc.setMinWeight (0);
  TriangleSoup full;
  if (!mc.reconstruct (full)) return 1;
  std::vector<std::int64_t> all_counts, counts;
  std::size_t n_all = 0, n = 0;
  if (mc.reconstructCellsDevice (nullptr, nullptr, nullptr, 0, &n_all, &all_counts) != 0) { std::printf ("count: %s\n", t->lastError ()); return 1; }
  if (n_all * 3 != full.xyz.size ()) { std::printf ("count %zu != %zu host vertices\n", n_all, full.xyz.size () / 3); return 1; }
  if (mc.reconstructCellsDevice (mask.data (), nullptr, nullptr, 0, &n, &counts) != 0) return 1;
  float* d = nullptr;
  if (cudaMalloc (&d, (n ? n : 1) * 12) != cudaSuccess) return 1;
  std::size_t n2 = 0;
  if (mc.reconstructCellsDevice (mask.data (), d, nullptr, n, &n2, &counts) != 0 || n2 != n) { std::printf ("mesh: %s\n", t->lastError ()); return 1; }
  std::vector<float> cells (3 * n);
  if (n && cudaMemcpy (cells.data (), d, n * 12, cudaMemcpyDeviceToHost) != cudaSuccess) return 1;
  cudaFree (d);

  // walk both meshes cell by cell in Morton order
  const std::vector<std::size_t> perm = morton_cells (mask.size ());
  std::size_t off_full = 0, off_cells = 0, selected = 0, nonempty = 0;
  for (std::size_t c : perm)
  {
    const std::size_t k = (std::size_t) all_counts[c];
    if (mask[c])
    {
      ++selected; nonempty += k > 0;
      if ((std::size_t) counts[c] != k) { std::printf ("cell %zu: %lld vertices, %zu in the full mesh\n", c, (long long) counts[c], k); return 1; }
      if (k && std::memcmp (&cells[3 * off_cells], &full.xyz[3 * off_full], 12 * k)) { std::printf ("cell %zu: run differs\n", c); return 1; }
      off_cells += k;
    }
    else if (counts[c]) { std::printf ("unselected cell %zu has vertices\n", c); return 1; }
    off_full += k;
  }
  std::printf ("mesh: %zu of %zu cells changed (%zu with triangles), %zu of %zu vertices re-meshed\n", selected, mask.size (), nonempty, n,
               n_all);
  return selected > 0 && selected < mask.size () && nonempty > 0 && off_cells == n ? 0 : 1;
}
