// b200_integrate — the reference's `integrate` program (src/prog/integrate.cpp) on the CUDA engine.
//
//   b200_integrate --in <dir> --out <dir> [options]          (same options as the reference, see --help)
//
// Reads <dir>/*.pcd and the matching camera poses (*.txt ascii or *.transform binary: 12 floats, rows 0..2 of the
// camera->world matrix), fuses them into a TSDF octree and writes <out>/mesh.ply (+ <out>/volume.tsdf with
// --save-tsdf).  Control flow, defaults and option names follow integrate.cpp:246-722; the per-frame work that the
// reference does in host loops — unit scaling, zero->NaN, world->camera, z-buffer re-organisation (:548-635) — and
// the mesh post-processing (:103-214) run on the GPU through libb200tsdf.so.
// Not supported (exit code 2): --cloud-only (a pcl::VoxelGrid aggregate, not part of the volumetric path),
// --visualize, --num-random-splits != 1.
#include <cpu_tsdf_b200/tsdf_volume_octree.h>

#include "pcd_io.h"
#include "ply_io.h"
#include "pose_io.h"

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <filesystem>
#include <map>
#include <string>
#include <vector>

namespace fs = std::filesystem;
using namespace b200prog;

namespace {

struct Options
{
  std::map<std::string, std::string> values;
  bool has (const std::string& k) const { return values.count (k) != 0; }
  template <typename T> T get (const std::string& k, T dflt) const
  {
    auto it = values.find (k);
    if (it == values.end ()) return dflt;
    if constexpr (std::is_same<T, std::string>::value) return it->second;
    else if constexpr (std::is_integral<T>::value) return static_cast<T> (std::strtoll (it->second.c_str (), nullptr, 10));
    else return static_cast<T> (std::strtof (it->second.c_str (), nullptr));
  }
};

const char* const kValueOpts[] = { "in", "out", "volume-size", "cell-size", "max-cell-size", "num-frames", "width", "height",
  "num-random-splits", "fx", "fy", "cx", "cy", "cloud-units", "pose-units", "max-sensor-dist", "min-sensor-dist",
  "trunc-dist-pos", "trunc-dist-neg", "min-weight", "device", "pool-log2" };
const char* const kFlagOpts[] = { "help", "save-tsdf", "visualize", "verbose", "color", "flatten", "cleanup", "invert", "world",
  "organized", "zero-nans", "save-ascii", "cloud-only", "exact-vol" };

bool parse (int argc, char** argv, Options& o, std::string& err)
{
  for (int i = 1; i < argc; ++i)
  {
    std::string a = argv[i];
    if (a == "-h") a = "--help";
    if (a.rfind ("--", 0) != 0) { err = "unexpected argument " + a; return false; }
    a = a.substr (2);
    std::string val; bool has_val = false;
    auto eq = a.find ('=');
    if (eq != std::string::npos) { val = a.substr (eq + 1); a = a.substr (0, eq); has_val = true; }
    bool is_value = std::find_if (std::begin (kValueOpts), std::end (kValueOpts), [&] (const char* s) { return a == s; }) != std::end (kValueOpts);
    bool is_flag = std::find_if (std::begin (kFlagOpts), std::end (kFlagOpts), [&] (const char* s) { return a == s; }) != std::end (kFlagOpts);
    if (!is_value && !is_flag) { err = "unknown option --" + a; return false; }
    if (is_value && !has_val) { if (i + 1 >= argc) { err = "--" + a + " needs a value"; return false; } val = argv[++i]; }
    o.values[a] = val;
  }
  return true;
}

void usage (const char* argv0)
{
  std::printf ("Usage: %s --in [in_dir] --out [out_dir] [OPTS]\n", fs::path (argv0).stem ().string ().c_str ());
  std::printf ("Integrates multiple clouds and returns a mesh. Clouds are PCD files; poses are ascii (.txt) or binary float\n"
               "(.transform) files with the same prefix, giving the pose of the camera in the world frame.\n\nAllowed options:\n"
               "  --help                 produce help message\n  --in arg               Input dir\n  --out arg              Output dir\n"
               "  --save-tsdf            Save the full TSDF in the output directory\n  --volume-size arg      Volume size (default 12)\n"
               "  --cell-size arg        Size of the smallest voxel (default 0.006)\n  --max-cell-size arg    Size of the largest voxel (default 0.5)\n"
               "  --num-frames arg       Only the first N clouds are used\n  --verbose              Verbose\n"
               "  --color                Store color in addition to depth in the TSDF\n  --flatten              Flatten mesh vertices\n"
               "  --cleanup              Clean up mesh\n  --invert               Transforms are inverted (world -> camera)\n"
               "  --world                Clouds are given in the world frame\n  --organized            Clouds are already organized\n"
               "  --width arg            Image width (default 640)\n  --height arg           Image height (default 480)\n"
               "  --zero-nans            Nans are represented as (0,0,0)\n  --fx/--fy/--cx/--cy    Camera intrinsics\n"
               "  --save-ascii           Save ply file as ASCII rather than binary\n  --cloud-units arg      Units of the data, in meters\n"
               "  --pose-units arg       Units of the poses, in meters\n  --max-sensor-dist arg  Maximum distance data can be from the sensor (3.0)\n"
               "  --min-sensor-dist arg  Minimum distance data can be from the sensor (0)\n  --trunc-dist-pos arg   Positive truncation distance (0.03)\n"
               "  --trunc-dist-neg arg   Negative truncation distance (0.03)\n  --min-weight arg       Minimum weight to render (0)\n"
               "  --exact-vol            Keep the per-voxel variance accumulators so that volume.tsdf is byte-identical to the\n"
               "                         reference's (slower: selects the general update kernel)\n"
               "  --device arg           CUDA device ordinal (default 0)\n  --pool-log2 arg        log2 of the brick pool capacity (default: library default)\n");
}

// integrate.cpp:224-246 (getSharedPrefix): the common prefix of the first and last (sorted) names, cut at the first
// digit.  Deviation: the reference scans the whole path string, so a digit in a DIRECTORY name ("/data/run2/...")
// cuts the prefix there and no pose file is ever matched; here the scan starts at the file name.
std::string shared_prefix (const std::vector<std::string>& files)
{
  const std::string& first = files.front ();
  const std::string& last = files.back ();
  size_t i = fs::path (first).parent_path ().string ().length ();
  if (first.compare (0, i, last, 0, i) != 0) i = 0;
  for (; i < first.length (); i++)
  {
    bool in_name = i > fs::path (first).parent_path ().string ().length ();
    if (i >= last.length () || first[i] != last[i] || (in_name && std::isdigit ((unsigned char) first[i]))) break;
  }
  return first.substr (0, i);
}

std::string lower_ext (const fs::path& p) { std::string e = p.extension ().string (); for (auto& c : e) c = (char) std::tolower ((unsigned char) c); return e; }

} // namespace

int main (int argc, char** argv)
{
  Options opts; std::string err;
  bool ok = parse (argc, argv, opts, err);
  if (!ok || opts.has ("help") || !opts.has ("in") || !opts.has ("out"))
  {
    if (!ok) std::fprintf (stderr, "%s\n", err.c_str ());
    usage (argv[0]);
    return 1;
  }
  if (opts.has ("cloud-only") || opts.has ("visualize")) { std::fprintf (stderr, "--cloud-only / --visualize are not supported by this front end\n"); return 2; }
  const bool verbose = opts.has ("verbose"), flatten = opts.has ("flatten"), cleanup = opts.has ("cleanup"), invert = opts.has ("invert");
  const bool organized = opts.has ("organized"), world_frame = opts.has ("world"), zero_nans = opts.has ("zero-nans");
  const bool save_ascii = opts.has ("save-ascii"), save_tsdf = opts.has ("save-tsdf"), integrate_color = opts.has ("color");
  const float cloud_units = opts.get<float> ("cloud-units", 1.f), pose_units = opts.get<float> ("pose-units", 1.f);
  if (opts.get<int> ("num-random-splits", 1) != 1) { std::fprintf (stderr, "--num-random-splits != 1 is not supported\n"); return 2; }
  const float max_sensor_dist = opts.get<float> ("max-sensor-dist", 3.0f), min_sensor_dist = opts.get<float> ("min-sensor-dist", 0.f);
  const float min_weight = opts.get<float> ("min-weight", 0.f);
  const float trunc_dist_pos = opts.get<float> ("trunc-dist-pos", 0.03f), trunc_dist_neg = opts.get<float> ("trunc-dist-neg", 0.03f);
  // :345-361
  const int width = opts.get<int> ("width", 640), height = opts.get<int> ("height", 480);
  float focal_length_x = 525. * width / 640., focal_length_y = 525. * height / 480.;
  float principal_point_x = static_cast<float> (width) / 2. - 0.5, principal_point_y = static_cast<float> (height) / 2. - 0.5;
  focal_length_x = opts.get<float> ("fx", focal_length_x); focal_length_y = opts.get<float> ("fy", focal_length_y);
  principal_point_x = opts.get<float> ("cx", principal_point_x); principal_point_y = opts.get<float> ("cy", principal_point_y);

  auto t_start = std::chrono::steady_clock::now ();
  // :366-449 scrape and pair the files
  std::vector<std::string> pcd_files, pose_files, pose_files_unordered;
  bool found_pose_file = false, binary_poses = false;
  std::string pose_extension, dir = opts.get<std::string> ("in", ""), out_dir = opts.get<std::string> ("out", "");
  std::error_code ec;
  for (fs::directory_iterator itr (dir, ec), end_itr; !ec && itr != end_itr; ++itr)
  {
    std::string extension = itr->path ().extension ().string (), low = lower_ext (itr->path ()), pathname = itr->path ().string ();
    if (low == ".pcd") pcd_files.push_back (pathname);
    else if (low == ".transform" || low == ".txt")
    {
      if (found_pose_file && extension != pose_extension)
      { std::fprintf (stderr, "Files with extension %s and %s were found in this folder! Please choose a consistent extension.\n", extension.c_str (), pose_extension.c_str ()); return 1; }
      if (!found_pose_file) { found_pose_file = true; binary_poses = low == ".transform"; pose_extension = extension; }
      pose_files_unordered.push_back (pathname);
    }
  }
  if (ec) { std::fprintf (stderr, "cannot read directory %s\n", dir.c_str ()); return 1; }
  if (pcd_files.empty ()) { std::fprintf (stderr, "no PCD files in %s\n", dir.c_str ()); return 1; }
  std::sort (pcd_files.begin (), pcd_files.end ());
  std::sort (pose_files_unordered.begin (), pose_files_unordered.end ());
  std::string pcd_prefix = shared_prefix (pcd_files), pose_prefix = pose_files_unordered.empty () ? "" : shared_prefix (pose_files_unordered);
  std::printf ("Found PCD files with prefix: %s, poses with prefix: %s poses\n", pcd_prefix.c_str (), pose_prefix.c_str ());
  if (!pose_files_unordered.empty ())
    for (const std::string& pcd_path : pcd_files)
    {
      std::string suffix = fs::path (pcd_path.substr (pcd_prefix.length ())).stem ().string ();
      std::string pose_path = pose_prefix + suffix + pose_extension;
      if (fs::exists (pose_path)) pose_files.push_back (pose_path);
      else { std::fprintf (stderr, "Could not find matching transform file for %s\n", pcd_path.c_str ()); return 1; }
    }
  std::sort (pose_files.begin (), pose_files.end ());
  std::printf ("Reading in %s pose files\n", binary_poses ? "binary" : "ascii");
  std::vector<Pose> poses (pose_files.size ());
  for (size_t i = 0; i < pose_files.size (); i++)
  {
    if (!load_pose (pose_files[i], binary_poses, poses[i])) { std::fprintf (stderr, "cannot read %s\n", pose_files[i].c_str ()); return 1; }
    if (invert) poses[i] = pose_inverse (poses[i]);
    poses[i][3] *= pose_units; poses[i][7] *= pose_units; poses[i][11] *= pose_units;      // topRightCorner<3,1> *= pose_units
    if (verbose) { std::printf ("Pose[%zu]\n", i); for (int r = 0; r < 4; ++r) std::printf ("%g %g %g %g\n", poses[i][4 * r], poses[i][4 * r + 1], poses[i][4 * r + 2], poses[i][4 * r + 3]); }
  }
  // :485-510
  const float tsdf_size = opts.get<float> ("volume-size", 12.f), cell_size = opts.get<float> ("cell-size", 0.006f);
  const float max_cell_size = opts.get<float> ("max-cell-size", 0.5f);
  int desired_res = tsdf_size / cell_size, tsdf_res = 1;
  while (desired_res > tsdf_res) tsdf_res *= 2;                                              // snap to a power of two
  cpu_tsdf_b200::TSDFVolumeOctree::Ptr tsdf (new cpu_tsdf_b200::TSDFVolumeOctree (opts.get<int> ("device", 0), opts.get<int> ("pool-log2", 0)));
  if (!tsdf->handle ()) { std::fprintf (stderr, "cannot create the TSDF engine: no CUDA device (there is no CPU path)\n"); return 3; }
  tsdf->setGridSize (tsdf_size, tsdf_size, tsdf_size);
  std::printf ("Setting resolution: %d with grid size %f\n", tsdf_res, tsdf_size);
  tsdf->setResolution (tsdf_res, tsdf_res, tsdf_res);
  tsdf->setMaxVoxelSize (max_cell_size, max_cell_size, max_cell_size);
  tsdf->setImageSize (width, height);
  tsdf->setCameraIntrinsics (focal_length_x, focal_length_y, principal_point_x, principal_point_y);
  tsdf->setSensorDistanceBounds (min_sensor_dist, max_sensor_dist);
  tsdf->setIntegrateColor (integrate_color);
  tsdf->setDepthTruncationLimits (trunc_dist_pos, trunc_dist_neg);
  tsdf->setTrackVariance (opts.has ("exact-vol"));
  tsdf->reset ();
  if (!tsdf->ok ()) { std::fprintf (stderr, "reset failed: %s\n", tsdf->lastError ()); return 3; }
  // :527-676
  size_t num_frames = pcd_files.size ();
  if (opts.has ("num-frames"))
  {
    size_t n = opts.get<size_t> ("num-frames", num_frames);
    if (n <= num_frames) num_frames = n;
    else std::printf ("Warning: Manually input --num-frames=%zu, but the sequence only has %zu clouds. Ignoring user specification.\n", n, num_frames);
  }
  for (size_t i = 0; i < num_frames; i++)
  {
    std::printf ("On frame %zu / %zu\n", i + 1, num_frames);
    if (poses.size () <= i)
    {
      std::printf ("Warning: no matching pose file found for cloud %s.\nDefaulting to identity, but unless the camera never moved, this will yield a very poor mesh!\n", pcd_files[i].c_str ());
      pose_files.push_back ("not_found"); poses.push_back (pose_identity ());
    }
    else std::printf ("Cloud: %s, pose: %s\n", pcd_files[i].c_str (), pose_files[i].c_str ());
    Cloud cloud;
    std::string e = load_pcd (pcd_files[i], cloud);
    if (!e.empty ()) { std::fprintf (stderr, "%s\n", e.c_str ()); return 1; }
    const Pose pose_rel_to_first_frame = pose_mul (pose_inverse (poses[0]), poses[i]);
    cpu_tsdf_b200::Affine3d trans, w2c;
    std::copy (pose_rel_to_first_frame.begin (), pose_rel_to_first_frame.end (), trans.m);
    const Pose inv_i = pose_inverse (poses[i]);
    std::copy (inv_i.begin (), inv_i.end (), w2c.m);
    bool done;
    if (organized)
    {
      if ((int) cloud.height != height || (int) cloud.width != width)
      { std::fprintf (stderr, "Error: cloud %zu has size %u x %u, but TSDF is initialized for %d x %d pointclouds\n", i + 1, cloud.width, cloud.height, width, height); return 1; }
      // :550-571 on the host for already organized clouds (units, zero->NaN, world->camera), then integrateCloud
      for (auto& pt : cloud.points)
      {
        if (cloud_units != 1) { pt.x *= cloud_units; pt.y *= cloud_units; pt.z *= cloud_units; }
        if (zero_nans && pt.x == 0 && pt.y == 0 && pt.z == 0) pt.x = pt.y = pt.z = std::numeric_limits<float>::quiet_NaN ();
        if (world_frame)
        {
          double p0 = pt.x, p1 = pt.y, p2 = pt.z;
          pt.x = static_cast<float> (inv_i[0] * p0 + inv_i[1] * p1 + inv_i[2] * p2 + inv_i[3]);
          pt.y = static_cast<float> (inv_i[4] * p0 + inv_i[5] * p1 + inv_i[6] * p2 + inv_i[7]);
          pt.z = static_cast<float> (inv_i[8] * p0 + inv_i[9] * p1 + inv_i[10] * p2 + inv_i[11]);
        }
      }
      double m[16]; std::copy (pose_rel_to_first_frame.begin (), pose_rel_to_first_frame.end (), m);
      done = b200tsdf_integrate (tsdf->handle (), cloud.points.data (), 16, 0, 12, width, height, m) == 0;
    }
    else
      done = tsdf->integrateUnorganizedCloud (cloud.points.data (), cloud.size (), 16, 0, 12, trans, cloud_units, zero_nans, world_frame ? &w2c : nullptr);
    if (!done) { std::fprintf (stderr, "integrateCloud failed on frame %zu: %s\n", i + 1, tsdf->lastError ()); return 3; }
  }
  // :677-721
  fs::create_directory (out_dir, ec);
  cpu_tsdf_b200::MarchingCubesTSDFOctree mc;
  mc.setMinWeight (min_weight);
  mc.setInputTSDF (tsdf);
  if (integrate_color) mc.setColorByRGB (true);
  cpu_tsdf_b200::TriangleSoup soup;
  if (!mc.reconstruct (soup)) { std::fprintf (stderr, "marching cubes failed: %s\n", tsdf->lastError ()); return 3; }
  const int device = opts.get<int> ("device", 0);
  if (flatten && !cpu_tsdf_b200::flattenVertices (soup, 0.0001f, device)) { std::fprintf (stderr, "flattenVertices failed: %s\n", b200tsdf_meshpost_last_error ()); return 3; }
  if (cleanup && !cpu_tsdf_b200::cleanupMesh (soup, 0.02f, 5, device)) { std::fprintf (stderr, "cleanupMesh failed: %s\n", b200tsdf_meshpost_last_error ()); return 3; }
  std::printf ("Entire pipeline took %f ms\n", std::chrono::duration<double, std::milli> (std::chrono::steady_clock::now () - t_start).count ());
  Mesh mesh; mesh.xyz = soup.xyz; mesh.rgb = soup.rgb; mesh.tris = soup.polygons;
  std::string e = save_ply (out_dir + "/mesh.ply", mesh, !save_ascii);
  if (!e.empty ()) { std::fprintf (stderr, "%s\n", e.c_str ()); return 1; }
  std::printf ("Saved to %s/mesh.ply\n", out_dir.c_str ());
  if (save_tsdf)
  {
    tsdf->save (out_dir + "/volume.tsdf");
    std::printf ("Saved full tsdf to %s/volume.tsdf\n", out_dir.c_str ());
  }
  return 0;
}
