// b200_tsdf2mesh — the reference's `tsdf2mesh` utility (src/prog/tsdf2mesh.cpp:50-70) on the CUDA engine:
// load a volume written by TSDFVolumeOctree::save (the reference's or this engine's), run marching cubes,
// write a binary PLY.
#include <cpu_tsdf_b200/tsdf_volume_octree.h>

#include "ply_io.h"

#include <cstdio>
#include <string>

int main (int argc, char** argv)
{
  if (argc < 3)
  {
    std::printf ("This is a utility program meant to render a mesh from a TSDF Volume, which can be saved to disk via TSDFVolumeOctree::save(const std::string &filename).\n");
    std::printf ("Usage: %s foo.vol foo.ply [device]\n", argv[0]);
    return 1;
  }
  std::string volume_file = argv[1], mesh_file = argv[2];
  std::printf ("Converting %s -> %s\n", volume_file.c_str (), mesh_file.c_str ());
  cpu_tsdf_b200::TSDFVolumeOctree::Ptr tsdf (new cpu_tsdf_b200::TSDFVolumeOctree (argc > 3 ? std::atoi (argv[3]) : 0));
  if (!tsdf->handle ()) { std::fprintf (stderr, "no CUDA device (there is no CPU path)\n"); return 3; }
  tsdf->load (volume_file);
  if (!tsdf->ok ()) { std::fprintf (stderr, "load failed: %s\n", tsdf->lastError ()); return 1; }
  std::printf ("Loaded! Running marching cubes\n");
  cpu_tsdf_b200::MarchingCubesTSDFOctree mc;
  mc.setInputTSDF (tsdf);
  mc.setColorByConfidence (false);
  mc.setColorByRGB (false);
  cpu_tsdf_b200::TriangleSoup soup;
  if (!mc.reconstruct (soup)) { std::fprintf (stderr, "marching cubes failed: %s\n", tsdf->lastError ()); return 3; }
  b200prog::Mesh mesh; mesh.xyz = soup.xyz; mesh.tris = soup.polygons;
  std::string e = b200prog::save_ply (mesh_file, mesh, true);
  if (!e.empty ()) { std::fprintf (stderr, "%s\n", e.c_str ()); return 1; }
  return 0;
}
