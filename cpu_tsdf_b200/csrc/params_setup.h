// params_setup.h — derive the engine's scalar parameters from a b200tsdf_config
// (TSDFVolumeOctree::reset, tsdf_volume_octree.cpp:201-211; Octree::init, octree.cpp:593-599).
// Shared by engine.cu and the host emulation harness in tests/emu.
#pragma once
#include "../../include/b200tsdf.h"
#include "tsdf_core.cuh"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include "host_math.h"

namespace b2 {

inline int ilog2_exact (int v) { int l = 0; while ((1 << l) < v && l < 30) ++l; return ((1 << l) == v) ? l : -1; }
// the smallest float not below t: for every float d, d < at_least (t) <=> (double) d < t (the host twin of float_at_least)
inline float at_least (double t) { float f = (float) t; if ((double) f < t) f = std::nextafterf (f, INFINITY); return f; }

// returns nullptr on success or a message describing the unsupported configuration
inline const char* derive_params (const b200tsdf_config& c, Params& p, size_t& pool, size_t& root_n)
{
  int L = ilog2_exact (c.xres);
  if (c.xres != c.yres || c.xres != c.zres || L < 0)
    return "resolution must be cubic and a power of two (SURVEY.md A.3-4: the reference octree is only exact for such grids)";
  if (!(c.xsize == c.ysize && c.xsize == c.zsize) || !(c.xsize > 0))
    return "grid size must be cubic and positive (OctreeNode keeps a single size_, octree.h:67)";
  if (!(c.max_dist_neg > 0) || !(c.max_cell_x > 0) || !(c.max_cell_y > 0) || !(c.max_cell_z > 0))
    return "max_dist_neg and max cell sizes must be positive";
  if (c.shard_count < 1 || c.shard_rank < 0 || c.shard_rank >= c.shard_count)
    return "bad shard_rank / shard_count";
  if (c.image_width <= 0 || c.image_height <= 0) return "bad image size";
  // Octree::init (float,float,float), octree.cpp:593-599
  int desired_res = std::max (c.xsize / c.max_cell_x, std::max (c.ysize / c.max_cell_y, c.zsize / c.max_cell_z));
  int C = desired_res >= 1 ? (int) std::ceil (std::log (desired_res) / std::log (2)) : 0;
  if (C < 0) C = 0;
  if (L <= C || L > 19) return "need coarse depth < log2(res) <= 19";
  int T = (L - C + 2) / 3;
  int Rtop = L - 3 * T;
  if (Rtop < 0) return "resolution too small for its coarse cell size: need log2(res) - 3*ceil((log2(res)-coarse)/3) >= 0";
  int pool_log2 = c.pool_log2 > 0 ? c.pool_log2 : 20;
  if (pool_log2 < 8 || pool_log2 > 26) return "pool_log2 out of range [8,26]";
  pool = (size_t) 1 << pool_log2;
  root_n = (size_t) 1 << (3 * Rtop);
  p.L = L; p.C = C; p.T = T; p.Rtop = Rtop; p.res = c.xres;
  p.size = c.xsize; p.half = c.xsize / 2; p.finest_size = c.xsize / c.xres;
  p.dsize = (double) c.xsize; p.dres = (double) c.xres; p.voff = (float) (c.xsize / 2.0);
  p.max_dist_pos = c.max_dist_pos; p.max_dist_neg = c.max_dist_neg; p.max_weight = c.max_weight;
  p.min_sensor = c.min_sensor_dist; p.max_sensor = c.max_sensor_dist;
  p.rc_thresh = 0.99 * c.max_dist_pos / c.max_dist_neg;
  p.fx = c.fx; p.fy = c.fy; p.cx = c.cx; p.cy = c.cy; p.width = c.image_width; p.height = c.image_height;
  p.fx_f = (float) c.fx; p.fy_f = (float) c.fy; p.cx_f = (float) c.cx; p.cy_f = (float) c.cy;
  p.fast_proj = (c.image_width < 8192 && c.image_height < 8192 && std::fabs (c.cx) < 1e4 && std::fabs (c.cy) < 1e4) ? 1 : 0;
  {
    p.rc_lo_f = at_least (-0.99); p.rc_hi_f = at_least (p.rc_thresh);
    // error of the float pixel estimate a = x*fx*rcp(z) + cx against the reference's double expression: the product
    // and the approximate reciprocal contribute < 2^-22 |x fx / z|, the final rounding 2^-24 |a| (brick_direct.cuh)
    const double M = std::max (c.image_width, c.image_height) + 2.0, cc = std::max (std::fabs (c.cx), std::fabs (c.cy));
    p.proj_guard = (float) (1.5 * ((M + cc) * std::ldexp (1.0, -22) + M * std::ldexp (1.0, -24)));
    if (!(p.proj_guard < 0.05f)) p.fast_proj = 0;
    // the operands of the brick kernels' divisions (div_with): d_new, clamped to [-max_dist_neg, max_dist_pos], over
    // max_dist_neg; the weighted sums over w + 1 <= max_weight + 1.  The sensor bounds are not among them, so the
    // integrate program's default min_sensor_dist = 0 keeps the brick kernels (div_with sends a tiny distance numerator to
    // the IEEE division).  A weight cap of 0 or >= 1e-20 keeps the colour numerators w c + c', divided by div_fast alone,
    // at 0 or >= 1e-20, far inside the region where div_fast is exact (obs_fast.cuh).
    p.exact_div_ok = (c.max_dist_neg >= 1e-6f && c.max_dist_neg <= 1e6f && std::fabs (c.max_dist_pos) <= 1e6f
                      && (c.max_weight == 0.f || c.max_weight >= 1e-20f) && c.max_weight <= 1e9f) ? 1 : 0;
  }
  p.color = c.integrate_color != 0; p.track_var = c.track_variance != 0;
  if (c.color_mode == B200TSDF_COLOR_LAB)
    return "colour mode LAB is not supported: LABNode::addObservation converts through libm pow (octree.cpp:436-470), which the device cannot reproduce bit for bit";
  if (c.color_mode != B200TSDF_COLOR_RGB && c.color_mode != B200TSDF_COLOR_RGB_NORMALIZED) return "unknown colour mode";
  p.color_norm = (p.color && c.color_mode == B200TSDF_COLOR_RGB_NORMALIZED) ? 1 : 0;
  p.shard_rank = c.shard_rank; p.shard_count = c.shard_count;
  p.pool_mask = (uint32_t) (pool - 1);
  return nullptr;
}

inline void default_config (b200tsdf_config* c)
{
  *c = b200tsdf_config{};
  c->xres = c->yres = c->zres = 512;                      // tsdf_volume_octree.cpp:54-85
  c->xsize = c->ysize = c->zsize = 3.0f;
  c->max_dist_pos = 0.03f; c->max_dist_neg = 0.03f;
  c->max_weight = 100;
  c->min_sensor_dist = 0.3f; c->max_sensor_dist = 3.0f;
  c->fx = 525.; c->fy = 525.; c->cx = 320; c->cy = 240;
  c->image_width = 640; c->image_height = 480;
  c->max_cell_x = c->max_cell_y = c->max_cell_z = 0.5f;
  c->pool_log2 = 20;
  c->shard_rank = 0; c->shard_count = 1;
  for (int i = 0; i < 4; ++i) c->global_transform[i * 5] = 1.0;
}

// the Vector4f(pt,1).dot(plane) <= 0 test of pcl::FrustumCulling with Eigen's SSE2 reduction
B2_HD bool frustum_contains (const float (*pl)[4], float cx, float cy, float cz)
{
  bool in = true;
  for (int k = 0; k < 6; ++k)
  {
    float dv = fadd (fadd (fmul (cx, pl[k][0]), fmul (cz, pl[k][2])), fadd (fmul (cy, pl[k][1]), fmul (1.0f, pl[k][3])));
    in = in && (dv <= 0.f);
  }
  return in;
}

// render / mesh parameter blocks
// renderView set-up (tsdf_volume_octree.cpp:281-289, :303-304)
inline void make_render_params (const b200tsdf_config& c, const Params& p, const double* pose, int downsample, RenderParams& r)
{
  r.width = p.width / downsample; r.height = p.height / downsample;
  r.fx = p.fx / downsample; r.fy = p.fy / downsample; r.cx = p.cx / downsample; r.cy = p.cy / downsample;
  for (int i = 0; i < 12; ++i) { r.rot[i] = (float) pose[i]; r.tfwd[i] = (float) pose[i]; }
  b2host::affine_inverse (pose, r.inv);
  r.min_step = p.max_dist_neg * 3 / 4.;
  r.half_voxel = (c.zsize / c.zres) / 2.;
}
inline void make_mc_params (const b200tsdf_config& c, const Params& p, float w_min, int color_mode, McParams& mc)
{
  mc.w_min = w_min; mc.color_mode = color_mode;
  // setInputTSDF (marching_cubes_tsdf_octree.cpp:43-83): lower_boundary_ = voxelCentre(0),
  // upper_boundary_ = voxelCentre(res); size_voxel_ = (upper - lower) * (1/res)
  float lo = voxel_center1 (p, 0), hi = voxel_center1 (p, p.res);
  for (int k = 0; k < 3; ++k) { mc.lower[k] = lo; mc.size_voxel[k] = (hi - lo) * (1.0f / (float) p.res); }
  for (int i = 0; i < 12; ++i) mc.gt[i] = c.global_transform[i];
}

} // namespace b2
