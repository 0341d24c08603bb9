// oracle/ref_capi.cpp — the oracle C API (tsdf_oracle.h) implemented by CALLING THE REFERENCE'S OWN
// CLASSES.  Linked with /root/reference/src/lib/{octree,tsdf_volume_octree,marching_cubes_tsdf_octree,
// tsdf_interface}.cpp compiled verbatim against oracle/compat/ (see oracle/Makefile `ref`) into
// oracle/_ref/libcpu_tsdf_ref.so.  TEST INFRASTRUCTURE: used to pin the restatement
// (tests/test_ref_pin.py) and as the "reference" CPU arm of bench.py.  No reference source is copied.
#include "tsdf_oracle.h"

#include <cpu_tsdf/marching_cubes_tsdf_octree.h>
#include <cpu_tsdf/tsdf_volume_octree.h>

#include <algorithm>
#include <chrono>
#include <cstring>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

struct orc_volume
{
  orc_config c;
  cpu_tsdf::TSDFVolumeOctree::Ptr tsdf;
  orc_stats stats{};
  std::vector<float> mesh_v;
  std::vector<uint8_t> mesh_c;
  int num_levels = 0, finest = 0;
};

namespace {
Eigen::Affine3d to_affine (const double* m)
{
  Eigen::Affine3d t;
  for (int i = 0; i < 16; ++i) t.matrix ().a[i] = m[i];
  return t;
}
double now_s () { return std::chrono::duration<double> (std::chrono::steady_clock::now ().time_since_epoch ()).count (); }

struct Rec { int32_t k[4]; const cpu_tsdf::OctreeNode* n; };
void collect (const cpu_tsdf::OctreeNode* n, int level, int ix, int iy, int iz, int min_level, std::vector<Rec>& out, int64_t& count)
{
  ++count;
  if (level >= min_level) out.push_back ({ { level, ix, iy, iz }, n });
  const std::vector<cpu_tsdf::OctreeNode::Ptr>& ch = n->getChildren ();
  for (size_t i = 0; i < ch.size (); ++i)                   // child i = (x>cx)*4 + (y>cy)*2 + (z>cz), octree.cpp:257-264
    collect (ch[i].get (), level + 1, 2 * ix + int ((i >> 2) & 1), 2 * iy + int ((i >> 1) & 1), 2 * iz + int (i & 1), min_level, out, count);
}
}

extern "C" {

void orc_default_config (orc_config* c)
{
  std::memset (c, 0, sizeof (*c));
  cpu_tsdf::TSDFVolumeOctree t;                              // the reference's own constructor defaults
  int xr, yr, zr; t.getResolution (xr, yr, zr);
  c->xres = xr; c->yres = yr; c->zres = zr;
  t.getGridSize (c->xsize, c->ysize, c->zsize);
  t.getDepthTruncationLimits (c->max_dist_pos, c->max_dist_neg);
  c->max_weight = t.getWeightTruncationLimit ();
  t.getSensorDistanceBounds (c->min_sensor_dist, c->max_sensor_dist);
  t.getCameraIntrinsics (c->fx, c->fy, c->cx, c->cy);
  t.getImageSize (c->image_width, c->image_height);
  c->max_cell_x = c->max_cell_y = c->max_cell_z = 0.5f;      // no getter: tsdf_volume_octree.cpp:72-74
  for (int i = 0; i < 4; ++i) c->global_transform[i * 5] = 1.0;
}

orc_volume* orc_create (const orc_config* cfg)
{
  orc_volume* v = new orc_volume;
  v->c = *cfg;
  v->tsdf.reset (new cpu_tsdf::TSDFVolumeOctree);
  return v;
}
void orc_destroy (orc_volume* v) { delete v; }

int orc_reset (orc_volume* v)
{
  const orc_config& c = v->c;
  cpu_tsdf::TSDFVolumeOctree& t = *v->tsdf;
  t.setResolution (c.xres, c.yres, c.zres);
  t.setGridSize (c.xsize, c.ysize, c.zsize);
  t.setImageSize (c.image_width, c.image_height);
  t.setDepthTruncationLimits (c.max_dist_pos, c.max_dist_neg);
  t.setWeightTruncationLimit (c.max_weight);
  t.setSensorDistanceBounds (c.min_sensor_dist, c.max_sensor_dist);
  t.setCameraIntrinsics (c.fx, c.fy, c.cx, c.cy);
  t.setMaxVoxelSize (c.max_cell_x, c.max_cell_y, c.max_cell_z);
  t.setIntegrateColor (c.integrate_color != 0);
  t.setColorMode (c.color_mode == 1 ? "RGBNormalized" : "RGB");
  t.setGlobalTransform (to_affine (c.global_transform));
#ifdef _OPENMP
  if (c.num_threads > 0) omp_set_num_threads (c.num_threads);
#endif
  t.reset ();
  // coarse depth = depth of the tree right after init
  int lv = 0; const cpu_tsdf::OctreeNode* n = t.octree_->getRoot ().get ();
  while (n->hasChildren ()) { n = n->getChildren ()[0].get (); ++lv; }
  v->num_levels = lv;
  int fl = 0; while ((1 << fl) < c.xres) ++fl;
  v->finest = fl;
  std::memset (&v->stats, 0, sizeof (v->stats));
  return 0;
}

int orc_integrate (orc_volume* v, const void* points, size_t stride, int xyz_off, int rgba_off, int width, int height, const double* pose)
{
  const uint8_t* base = static_cast<const uint8_t*> (points);
  Eigen::Affine3d trans = to_affine (pose);
  size_t n = static_cast<size_t> (width) * height;
  double t0, t1;
  // updateVoxel reads pt.r/g/b unconditionally (hpp:206), so the reference only instantiates with coloured
  // point types (src/prog/integrate.cpp uses pcl::PointXYZRGBA throughout); colour bytes are 0 when absent
  pcl::PointCloud<pcl::PointXYZRGBA> cloud (width, height);
  for (size_t i = 0; i < n; ++i)
  {
    const float* p = reinterpret_cast<const float*> (base + i * stride + xyz_off);
    pcl::PointXYZRGBA& q = cloud.points[i];
    q.x = p[0]; q.y = p[1]; q.z = p[2];
    if (rgba_off >= 0) { const uint8_t* cb = base + i * stride + rgba_off; q.b = cb[0]; q.g = cb[1]; q.r = cb[2]; q.a = cb[3]; }
  }
  t0 = now_s ();
  v->tsdf->integrateCloud (cloud, pcl::PointCloud<pcl::Normal> (), trans);
  t1 = now_s ();
  std::memset (&v->stats, 0, sizeof (v->stats));
  v->stats.t_update = t1 - t0;          // integrateCloud only (the reference has no per-phase timers)
  v->stats.n_add_observation = -1; v->stats.n_node_visits = -1; v->stats.n_presplit = -1; v->stats.n_culled_cells = -1; v->stats.n_nodes = -1;
  v->stats.n_prune_existing = -1; v->stats.n_prune_resplit = -1;
  return 0;
}

void orc_get_stats (const orc_volume* v, orc_stats* s) { *s = v->stats; }

int orc_query (const orc_volume* v, const float* xyz, int n, int what, int mode, float* val, float* grad, float* hess, uint8_t* ok)
{
  const cpu_tsdf::TSDFVolumeOctree& t = *v->tsdf;
  for (int i = 0; i < n; ++i)
  {
    pcl::PointXYZ pt (xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    float fv = 0; Eigen::Vector3f g; Eigen::Matrix3f H;
    bool good = true;
    if (mode == 0)
    {
      if (what & 1) good = good && t.getFxn (pt, fv);
      if (what & 2) good = good && t.getGradient (pt, g);
      if (what & 4) good = good && t.getHessian (pt, H);
    }
    else
    {
      if (what & 4) good = t.getFxnGradientAndHessian (pt, fv, g, H);
      else good = t.getFxnAndGradient (pt, fv, g);
    }
    ok[i] = good;
    if (!good) continue;
    if ((what & 1) && val) val[i] = fv;
    if ((what & 2) && grad) { grad[3 * i] = g (0); grad[3 * i + 1] = g (1); grad[3 * i + 2] = g (2); }
    if ((what & 4) && hess) for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) hess[9 * i + 3 * r + c] = H (r, c);
  }
  return 0;
}

// getTSDFValue / interpolateTrilinearly are protected: reach them through a derived class that republishes the names
namespace { struct TsdfAccess : cpu_tsdf::TSDFVolumeOctree { using cpu_tsdf::TSDFVolumeOctree::getTSDFValue; }; }
int orc_interpolate (const orc_volume* v, const float* xyz, int n, float* val, uint8_t* valid_in_out)
{
  const TsdfAccess& t = *static_cast<const TsdfAccess*> (v->tsdf.get ());
  for (int i = 0; i < n; ++i)
  {
    bool valid = valid_in_out[i] != 0;
    val[i] = t.getTSDFValue (xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], &valid);
    valid_in_out[i] = valid;
  }
  return 0;
}

int orc_render (const orc_volume* v, const double* pose, int downsample, void* out, size_t stride, int xyz_off, int normal_off, uint8_t* rgb_out)
{
  uint8_t* base = static_cast<uint8_t*> (out);
  Eigen::Affine3d trans = to_affine (pose);
  if (rgb_out)
  {
    pcl::PointCloud<pcl::PointXYZRGBNormal>::Ptr c = v->tsdf->renderColoredView (trans, downsample);
    for (size_t i = 0; i < c->size (); ++i)
    {
      const pcl::PointXYZRGBNormal& p = c->points[i];
      std::memcpy (base + i * stride + xyz_off, p.data, 12);
      std::memcpy (base + i * stride + normal_off, p.data_n, 12);
      rgb_out[3 * i] = p.r; rgb_out[3 * i + 1] = p.g; rgb_out[3 * i + 2] = p.b;
    }
  }
  else
  {
    pcl::PointCloud<pcl::PointNormal>::Ptr c = v->tsdf->renderView (trans, downsample);
    for (size_t i = 0; i < c->size (); ++i)
    {
      std::memcpy (base + i * stride + xyz_off, c->points[i].data, 12);
      std::memcpy (base + i * stride + normal_off, c->points[i].data_n, 12);
    }
  }
  return 0;
}

int64_t orc_mesh (orc_volume* v, float w_min, int color_mode, const float** verts, const uint8_t** rgb)
{
  cpu_tsdf::MarchingCubesTSDFOctree mc;
  mc.setInputTSDF (v->tsdf);
  mc.setMinWeight (w_min);
  mc.setColorByRGB (color_mode == 1);
  mc.setColorByConfidence (color_mode == 2);
  pcl::PolygonMesh mesh;
  mc.reconstruct (mesh);
  size_t n = mesh.cloud.width;
  v->mesh_v.resize (3 * n); v->mesh_c.clear ();
  if (color_mode) v->mesh_c.resize (3 * n);
  for (size_t i = 0; i < n; ++i)
  {
    const uint8_t* p = mesh.cloud.data.data () + i * mesh.cloud.point_step;
    std::memcpy (&v->mesh_v[3 * i], p, 12);
    if (color_mode)
    {
      const pcl::PointXYZRGB* q = reinterpret_cast<const pcl::PointXYZRGB*> (p);
      v->mesh_c[3 * i] = q->r; v->mesh_c[3 * i + 1] = q->g; v->mesh_c[3 * i + 2] = q->b;
    }
  }
  if (verts) *verts = v->mesh_v.data ();
  if (rgb) *rgb = v->mesh_c.empty () ? nullptr : v->mesh_c.data ();
  return static_cast<int64_t> (n);
}

int orc_save (const orc_volume* v, const char* path) { v->tsdf->save (path); return 0; }

int64_t orc_dump_nodes (const orc_volume* v, int32_t* keys, float* dw, uint8_t* flags, uint8_t* rgb, float* M, int32_t* ns)
{
  std::vector<Rec> recs; int64_t total = 0;
  collect (v->tsdf->octree_->getRoot ().get (), 0, 0, 0, 0, v->num_levels, recs, total);
  const_cast<orc_volume*> (v)->stats.n_nodes = total;
  if (!keys && !dw && !flags && !rgb && !M && !ns) return static_cast<int64_t> (recs.size ());
  std::sort (recs.begin (), recs.end (), [] (const Rec& a, const Rec& b) { return std::lexicographical_compare (a.k, a.k + 4, b.k, b.k + 4); });
  for (size_t i = 0; i < recs.size (); ++i)
  {
    const cpu_tsdf::OctreeNode* n = recs[i].n;
    if (keys) std::memcpy (keys + 4 * i, recs[i].k, 16);
    if (dw) { dw[2 * i] = n->d_; dw[2 * i + 1] = n->w_; }
    if (flags) flags[i] = n->hasChildren ();
    if (rgb)
    {
      uint8_t r = 0, g = 0, b = 0;
      if (!n->getRGB (r, g, b)) r = g = b = 0;               // colourless nodes: report 0 like the restatement's dump
      rgb[3 * i] = r; rgb[3 * i + 1] = g; rgb[3 * i + 2] = b;
    }
    if (M) M[i] = n->M_;
    if (ns) ns[i] = n->nsample_;
  }
  return static_cast<int64_t> (recs.size ());
}

int64_t orc_dump_color_payload (const orc_volume* v, float* out4)
{
  std::vector<Rec> recs; int64_t total = 0;
  collect (v->tsdf->octree_->getRoot ().get (), 0, 0, 0, 0, v->num_levels, recs, total);
  if (recs.empty () || !dynamic_cast<const cpu_tsdf::RGBNormalized*> (recs[0].n)) return 0;
  std::sort (recs.begin (), recs.end (), [] (const Rec& a, const Rec& b) { return std::lexicographical_compare (a.k, a.k + 4, b.k, b.k + 4); });
  for (size_t i = 0; i < recs.size (); ++i)
  {
    const cpu_tsdf::RGBNormalized* n = dynamic_cast<const cpu_tsdf::RGBNormalized*> (recs[i].n);
    out4[4 * i] = n->r_n_; out4[4 * i + 1] = n->g_n_; out4[4 * i + 2] = n->b_n_; out4[4 * i + 3] = n->i_;
  }
  return static_cast<int64_t> (recs.size ());
}

int orc_levels (const orc_volume* v, int* coarse_level, int* finest_level)
{
  if (coarse_level) *coarse_level = v->num_levels;
  if (finest_level) *finest_level = v->finest;
  return 0;
}

void orc_voxel_center (const orc_volume* v, int64_t x, int64_t y, int64_t z, float* o)
{ pcl::PointXYZ p = v->tsdf->getVoxelCenter (x, y, z); o[0] = p.x; o[1] = p.y; o[2] = p.z; }

int orc_voxel_index (const orc_volume* v, float x, float y, float z, int* o)
{ return v->tsdf->getVoxelIndex (x, y, z, o[0], o[1], o[2]); }

int orc_frustum_cull (const orc_volume* v, const double* pose, uint8_t* mask)
{
  std::vector<cpu_tsdf::OctreeNode::Ptr> voxels;
  v->tsdf->getFrustumCulledVoxels (to_affine (pose), voxels);
  int n = 1 << v->num_levels;
  std::memset (mask, 0, static_cast<size_t> (n) * n * n);
  float size = v->c.xsize / n;
  for (const auto& p : voxels)
  {
    float x, y, z; p->getCenter (x, y, z);
    int ix = static_cast<int> ((x + v->c.xsize / 2) / size), iy = static_cast<int> ((y + v->c.ysize / 2) / size), iz = static_cast<int> ((z + v->c.zsize / 2) / size);
    mask[(static_cast<size_t> (ix) * n + iy) * n + iz] = 1;
  }
  return static_cast<int> (voxels.size ());
}

} // extern "C"
