// oracle/tsdf_oracle.cpp — CPU oracle.  TEST INFRASTRUCTURE ONLY: see tsdf_oracle.h.
//
// A restatement of the reference's volumetric path (sdmiller/cpu_tsdf @ 9b973cb).  Every
// function cites the reference file:line it follows (paths relative to /root/reference).
// The tree is a pool of 8-node child groups addressed by index instead of
// boost::shared_ptr<OctreeNode>; the visit order, the float expressions and every quirk
// listed in SURVEY.md §A are kept.  Third-party (Eigen/PCL) arithmetic conventions live in
// ref_arith.h.  Build: see oracle/Makefile (-O3 -fopenmp -ffp-contract=off).
#include "tsdf_oracle.h"
#include "ref_arith.h"
#include "mc_tables.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <mutex>
#include <string>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

using namespace ref_arith;

// include/cpu_tsdf/octree.h:55-172 (OctreeNode) + :174-213 (RGBNode)
struct Node
{
  float d, w, M;
  int32_t ns;
  float cx, cy, cz, size;
  int32_t child;            // index of children_[0]; -1 = no children
  int32_t ix, iy, iz;       // integer coordinates at this node's own level (bookkeeping only)
  uint8_t level, r, g, b;
  float rn, gn, bn, in;     // RGBNormalized payload (octree.h:250-253)
};

constexpr int CHUNK_BITS = 20;
constexpr int32_t CHUNK_MASK = (1 << CHUNK_BITS) - 1;
constexpr int MAX_CHUNKS = 2048;
constexpr int MAX_THREADS = 256;

struct Pool
{
  Node* chunks[MAX_CHUNKS];
  std::atomic<int> nchunks{0};
  std::atomic<int64_t> next{0};
  std::mutex mu;
  std::vector<int32_t> freelist[MAX_THREADS];
  std::atomic<int64_t> live{0};

  Pool () { std::memset (chunks, 0, sizeof (chunks)); }
  ~Pool () { clear (); }
  void clear ()
  {
    for (int i = 0; i < nchunks.load (); ++i) std::free (chunks[i]);
    nchunks = 0; next = 0; live = 0;
    for (auto& f : freelist) f.clear ();
  }
  inline Node& at (int32_t i) { return chunks[i >> CHUNK_BITS][i & CHUNK_MASK]; }
  inline const Node& at (int32_t i) const { return chunks[i >> CHUNK_BITS][i & CHUNK_MASK]; }
  int32_t alloc (int n, int tid)
  {
    live += n;
    if (n == 8 && !freelist[tid].empty ())
    {
      int32_t i = freelist[tid].back (); freelist[tid].pop_back (); return i;
    }
    int64_t i = next.fetch_add (8);          // groups of 8 keep children contiguous inside one chunk
    while (((i + 7) >> CHUNK_BITS) >= nchunks.load ())
    {
      std::lock_guard<std::mutex> lk (mu);
      if (((i + 7) >> CHUNK_BITS) >= nchunks.load ())
      {
        if (nchunks.load () >= MAX_CHUNKS) { std::fprintf (stderr, "oracle: node pool exhausted\n"); std::abort (); }
        chunks[nchunks.load ()] = static_cast<Node*> (std::malloc (sizeof (Node) << CHUNK_BITS));
        nchunks++;
      }
    }
    return static_cast<int32_t> (i);
  }
  void free8 (int32_t first, int tid) { freelist[tid].push_back (first); live -= 8; }
};

inline int thread_id ()
{
#ifdef _OPENMP
  return omp_get_thread_num ();
#else
  return 0;
#endif
}

struct PerThread { int64_t n_add = 0, n_visit = 0, n_prune = 0, n_resplit = 0; char pad[32]; };

} // namespace

struct orc_volume
{
  orc_config c;
  Pool pool;
  int32_t root = -1;
  int num_levels = 0;          // coarse depth, octree.cpp:593-599
  int finest_level = 0;
  bool is_empty = true;
  bool color = false;          // node type "RGB" iff integrate_color_ at reset (cpp:206-209)
  bool rgbn = false;           // node type "RGBNormalized" (setColorMode, h:290)
  std::vector<int32_t> coarse; // getLeaves(max_cell...) result (depth == num_levels), DFS order
  orc_stats stats{};
  PerThread pt[MAX_THREADS];
  std::vector<float> mesh_v;
  std::vector<uint8_t> mesh_c;

  // ---- octree.h:67 ctor -------------------------------------------------------------
  void init_node (Node& n, float x, float y, float z, float size, int level, int ix, int iy, int iz) const
  {
    n.d = -1; n.w = 0; n.M = 0; n.ns = 0;
    n.cx = x; n.cy = y; n.cz = z; n.size = size;
    n.child = -1; n.ix = ix; n.iy = iy; n.iz = iz; n.level = static_cast<uint8_t> (level);
    n.r = n.g = n.b = 0;
    n.rn = n.gn = n.bn = n.in = 0;                               // octree.h:217-223
  }

  // ---- OctreeNode::split, octree.cpp:244-266 ------------------------------------------
  int32_t split (int32_t ni, int tid)
  {
    int32_t first = pool.alloc (8, tid);
    Node& n = pool.at (ni);
    float off = n.size / 4;
    float ns = n.size / 2;
    for (int i = 0; i < 8; ++i)
    {
      int bx = (i >> 2) & 1, by = (i >> 1) & 1, bz = i & 1;   // child index = (x>cx)*4+(y>cy)*2+(z>cz)
      init_node (pool.at (first + i),
                 bx ? n.cx + off : n.cx - off,
                 by ? n.cy + off : n.cy - off,
                 bz ? n.cz + off : n.cz - off,
                 ns, n.level + 1, 2 * n.ix + bx, 2 * n.iy + by, 2 * n.iz + bz);
    }
    n.child = first;
    return first;
  }

  // ---- OctreeNode::splitRecursive, octree.cpp:269-279 ---------------------------------
  void split_recursive (int32_t ni, int num_left)
  {
    if (num_left <= 0) return;
    int32_t first = split (ni, 0);
    for (int i = 0; i < 8; ++i) split_recursive (first + i, num_left - 1);
  }

  // ---- OctreeNode::getLeaves, octree.cpp:99-109 ---------------------------------------
  void get_leaves (int32_t ni, std::vector<int32_t>& out, int num_levels_left) const
  {
    const Node& n = pool.at (ni);
    for (int i = 0; i < 8 && n.child >= 0; ++i)
    {
      const Node& ch = pool.at (n.child + i);
      if (ch.child >= 0 && num_levels_left != 0) get_leaves (n.child + i, out, num_levels_left - 1);
      else out.push_back (n.child + i);
    }
  }

  // ---- OctreeNode::getContainingVoxel, octree.cpp:112-121 -----------------------------
  int32_t descend (int32_t ni, float x, float y, float z) const
  {
    for (;;)
    {
      const Node& n = pool.at (ni);
      if (n.child < 0) return ni;
      ni = n.child + ((x - n.cx) > 0) * 4 + ((y - n.cy) > 0) * 2 + ((z - n.cz) > 0);
    }
  }
  // ---- Octree::getContainingVoxel, octree.cpp:628-634 ---------------------------------
  int32_t containing (float x, float y, float z) const
  {
    if (std::isnan (z) || std::fabs (x) > c.xsize / 2 || std::fabs (y) > c.ysize / 2 || std::fabs (z) > c.zsize / 2)
      return -1;
    return descend (root, x, y, z);
  }

  // ---- getVoxelCenter, tsdf_volume_octree.cpp:553-560 ---------------------------------
  void voxel_center (size_t x, size_t y, size_t z, float* o) const
  {
    float xoff = c.xsize / 2.0, yoff = c.ysize / 2.0, zoff = c.zsize / 2.0;
    o[0] = static_cast<float> ((x + 0.5) * c.xsize / (double) c.xres - xoff);
    o[1] = static_cast<float> ((y + 0.5) * c.ysize / (double) c.yres - yoff);
    o[2] = static_cast<float> ((z + 0.5) * c.zsize / (double) c.zres - zoff);
  }
  // ---- getVoxelIndex, tsdf_volume_octree.cpp:562-574 ----------------------------------
  bool voxel_index (float x, float y, float z, int& xi, int& yi, int& zi) const
  {
    double xoff = (double) c.xsize / 2.0, yoff = (double) c.ysize / 2.0, zoff = (double) c.zsize / 2.0;
    xi = to_int (std::floor (((double) x + xoff) / (double) c.xsize * (double) c.xres));
    yi = to_int (std::floor (((double) y + yoff) / (double) c.ysize * (double) c.yres));
    zi = to_int (std::floor (((double) z + zoff) / (double) c.zsize * (double) c.zres));
    return (xi >= 0 && yi >= 0 && zi >= 0 && xi < c.xres && yi < c.yres && zi < c.zres);
  }
  // double -> int conversion as x86-64 cvttsd2si performs it (out of range / NaN -> INT_MIN)
  static int to_int (double v)
  {
    if (!(v > -2147483649.0 && v < 2147483648.0)) return INT_MIN;
    return static_cast<int> (v);
  }

  // ---- reprojectPoint, tsdf_volume_octree.cpp:611-617 ---------------------------------
  bool reproject (const float* p, int& u, int& v) const
  {
    u = to_int ((p[0] * c.fx / p[2]) + c.cx);
    v = to_int ((p[1] * c.fy / p[2]) + c.cy);
    return (p[2] > 0 && u >= 0 && u < c.image_width && v >= 0 && v < c.image_height);
  }

  // ---- OctreeNode::addObservation octree.cpp:152-163, RGBNode:: octree.cpp:328-337 -----
  void add_observation (Node& n, float d_new, float w_new, float max_weight, const uint8_t* bgr)
  {
    if (rgbn && bgr)                                              // RGBNormalized::addObservation, octree.cpp:380-393
    {
      uint8_t r = bgr[2], g = bgr[1], b = bgr[0];
      float wsum = n.w + w_new;
      float i = std::sqrt ((float) r * (float) r + (float) g * (float) g + (float) b * (float) b);
      float r_f = r / i;
      float g_f = g / i;
      float b_f = b / i;
      n.rn = (n.w * n.rn + w_new * r_f) / wsum;
      n.gn = (n.w * n.gn + w_new * g_f) / wsum;
      n.bn = (n.w * n.bn + w_new * b_f) / wsum;
      n.in = (n.w * n.in + w_new * i) / wsum;
    }
    else if (color && bgr)
    {
      uint8_t r = bgr[2], g = bgr[1], b = bgr[0];
      float wsum = n.w + w_new;
      n.r = static_cast<uint8_t> ((n.w * n.r + w_new * r) / wsum);
      n.g = static_cast<uint8_t> ((n.w * n.g + w_new * g) / wsum);
      n.b = static_cast<uint8_t> ((n.w * n.b + w_new * b) / wsum);
    }
    float d_old = n.d;
    n.d = (n.d * n.w + d_new * w_new) / (n.w + w_new);
    n.w += w_new;
    if (n.w > max_weight) n.w = max_weight;
    n.M += w_new * (d_new - n.d) * (d_new - d_old);
    ++n.ns;
  }

  // getRGB: RGBNode (octree.cpp:340-346) / RGBNormalized (octree.cpp:396-402: `r = r_n_ * i_`, a float -> uint8_t
  // conversion, which x86-64 compiles to cvttss2si + a byte truncation)
  static uint8_t f2u8 (float v)
  {
    int32_t t = (v >= -2147483648.f && v < 2147483648.f) ? static_cast<int32_t> (v) : INT32_MIN;
    return static_cast<uint8_t> (t);
  }
  void get_rgb (const Node& n, uint8_t& r, uint8_t& g, uint8_t& b) const
  {
    if (rgbn) { r = f2u8 (n.rn * n.in); g = f2u8 (n.gn * n.in); b = f2u8 (n.bn * n.in); }
    else { r = n.r; g = n.g; b = n.b; }
  }

  // ---- frame view ------------------------------------------------------------------------
  struct Frame
  {
    const uint8_t* base; size_t stride; int xyz_off, rgba_off, width, height;
    float trans_inv[16];
    inline const float* xyz (int u, int v) const   // cloud(u,v): column u, row v
    { return reinterpret_cast<const float*> (base + (static_cast<size_t> (v) * width + u) * stride + xyz_off); }
    inline const uint8_t* bgr (int u, int v) const
    { return rgba_off < 0 ? nullptr : base + (static_cast<size_t> (v) * width + u) * stride + rgba_off; }
  };

  // ---- updateVoxel, impl/tsdf_volume_octree.hpp:113-218 ------------------------------
  int update_voxel (int32_t ni, const Frame& f, int tid)
  {
    pt[tid].n_visit++;
    bool pruned = false;                                          // (event counter only: the pre-existing children were pruned)
    if (pool.at (ni).child >= 0)                                  // hpp:122-142
    {
      int32_t first = pool.at (ni).child;
      bool all_are_empty = true;
      for (int i = 0; i < 8; ++i) all_are_empty &= (update_voxel (first + i, f, tid) < 0);
      if (all_are_empty) { pool.free8 (first, tid); pool.at (ni).child = -1; }
      else return 1;
      pt[tid].n_prune++;
      pruned = true;
    }
    Node& n = pool.at (ni);
    float ctr[3] = { n.cx, n.cy, n.cz }, v_g[3];
    pcl_transform_point_f (f.trans_inv, ctr, v_g);                // hpp:143-145
    if (v_g[2] < c.min_sensor_dist || v_g[2] > c.max_sensor_dist) return 0;   // hpp:146
    int u, v;
    if (!reproject (v_g, u, v)) return 0;                         // hpp:148-150
    const float* p = f.xyz (u, v);
    if (std::isnan (p[2])) return 0;                              // hpp:151-153
    float d_new = (p[2] - v_g[2]);                                // hpp:159
    float max_size = static_cast<float> (std::sqrt (3.0) * n.size);   // getMaxSize, octree.cpp:68-72
    if (std::fabs (d_new) < 3 * max_size / 4.)                    // hpp:161
    {
      if (n.size > c.xsize / c.xres && n.size > c.ysize / c.yres && n.size > c.zsize / c.zres)   // hpp:165
      {
        if (pruned) pt[tid].n_resplit++;
        int32_t first = split (ni, tid);
        bool all_are_empty = true;
        for (int i = 0; i < 8; ++i) all_are_empty &= (update_voxel (first + i, f, tid) < 0);
        if (all_are_empty) { pool.free8 (first, tid); pool.at (ni).child = -1; }
        else return 1;
      }
    }
    if (d_new > c.max_dist_pos) d_new = c.max_dist_pos;           // hpp:189-196
    else if (d_new < -c.max_dist_neg) return 0;
    d_new /= c.max_dist_neg;                                      // hpp:198
    float w_new = 1;                                              // hpp:200 (weight_by_* unreachable)
    add_observation (n, d_new, w_new, c.max_weight, f.bgr (u, v));   // hpp:205-208
    pt[tid].n_add++;
    if (n.d < -0.99) return 0;                                    // hpp:209-214
    else if (n.d < 0.99 * c.max_dist_pos / c.max_dist_neg) return 1;
    else return -1;
  }

  // ---- getFrustumCulledVoxels, tsdf_volume_octree.cpp:619-652 -------------------------
  Frustum frustum (const double* pose) const
  {
    float cam[16];
    // trans.matrix().cast<float>() * cam2robot: columns (z_cam, -y_cam, x_cam, t), exact (cpp:633-638)
    for (int r = 0; r < 3; ++r)
    {
      cam[r * 4 + 0] = static_cast<float> (pose[r * 4 + 2]);
      cam[r * 4 + 1] = -static_cast<float> (pose[r * 4 + 1]);
      cam[r * 4 + 2] = static_cast<float> (pose[r * 4 + 0]);
      cam[r * 4 + 3] = static_cast<float> (pose[r * 4 + 3]);
    }
    cam[12] = cam[13] = cam[14] = 0; cam[15] = 1;
    float hfov = static_cast<float> (1.1 * 2 * std::fabs (std::atan (0.5 * c.image_width / c.fx) * 180 / M_PI));
    float vfov = static_cast<float> (1.1 * 2 * std::fabs (std::atan (0.5 * c.image_height / c.fy) * 180 / M_PI));
    return pcl_frustum_planes (cam, hfov, vfov, c.min_sensor_dist, c.max_sensor_dist);
  }

  // ---- trilinear, tsdf_volume_octree.cpp:486-541 ----------------------------------------
  float interpolate_trilinearly (float x, float y, float z, bool* valid) const
  {
    int xi, yi, zi;
    bool exists = voxel_index (x, y, z, xi, yi, zi);
    if (!exists || xi <= 0 || xi >= c.xres - 1 || yi <= 0 || yi >= c.yres - 1 || zi <= 0 || zi >= c.zres - 1)
    {
      if (valid) *valid = false;
      return std::numeric_limits<float>::quiet_NaN ();
    }
    float v[3];
    voxel_center (xi, yi, zi, v);
    if (x < v[0]) xi -= 1;
    if (y < v[1]) yi -= 1;
    if (z < v[2]) zi -= 1;
    voxel_center (xi, yi, zi, v);
    float a = (x - v[0]) * c.xres / c.xsize;
    float b = (y - v[1]) * c.yres / c.ysize;
    float cc = (z - v[2]) * c.zres / c.zsize;
    const Node* n[8];   // order: o, x, y, z, xy, xz, yz, xyz
    static const int off[8][3] = { {0,0,0}, {1,0,0}, {0,1,0}, {0,0,1}, {1,1,0}, {1,0,1}, {0,1,1}, {1,1,1} };
    for (int k = 0; k < 8; ++k)
    {
      float p[3];
      voxel_center (xi + off[k][0], yi + off[k][1], zi + off[k][2], p);
      n[k] = &pool.at (containing (p[0], p[1], p[2]));
    }
    if (valid) for (int k = 0; k < 8; ++k) *valid &= (n[k]->w > 0);
    const Node *vo = n[0], *vox = n[1], *voy = n[2], *voz = n[3], *voxy = n[4], *voxz = n[5], *voyz = n[6], *voxyz = n[7];
    return (vo->d    * (1 - a) * (1 - b) * (1 - cc) +
            voz->d   * (1 - a) * (1 - b) * (cc)     +
            voy->d   * (1 - a) * (b)     * (1 - cc) +
            voyz->d  * (1 - a) * (b)     * (cc)     +
            vox->d   * (a)     * (1 - b) * (1 - cc) +
            voxz->d  * (a)     * (1 - b) * (cc)     +
            voxy->d  * (a)     * (b)     * (1 - cc) +
            voxyz->d * (a)     * (b)     * (cc));
  }

  // ---- getNeighbors, tsdf_volume_octree.cpp:796-828 ------------------------------------
  bool get_neighbors (const float* p, const Node** nb, float (*centers)[3]) const
  {
    int xi, yi, zi;
    if (!voxel_index (p[0], p[1], p[2], xi, yi, zi)) return false;
    float v[3];
    voxel_center (xi, yi, zi, v);
    if (p[0] < v[0]) xi -= 1;
    if (p[1] < v[1]) yi -= 1;
    if (p[2] < v[2]) zi -= 1;
    if (xi < 0 || xi >= c.xres - 1 || yi < 0 || yi >= c.yres - 1 || zi < 0 || zi >= c.zres - 1) return false;
    int k = 0;
    for (int dx = 0; dx <= 1; dx++)
      for (int dy = 0; dy <= 1; dy++)
        for (int dz = 0; dz <= 1; dz++)
        {
          voxel_center (xi + dx, yi + dy, zi + dz, centers[k]);
          int32_t ni = containing (centers[k][0], centers[k][1], centers[k][2]);
          if (ni < 0) return false;
          nb[k++] = &pool.at (ni);
        }
    return true;
  }
};

namespace {
inline int sgn (float x) { return (x > 0 ? 1 : -1); }   // tsdf_volume_octree.cpp:674-678
inline double now_s ()
{
  return std::chrono::duration<double> (std::chrono::steady_clock::now ().time_since_epoch ()).count ();
}
}

extern "C" {

// ---- TSDFVolumeOctree ctor defaults, tsdf_volume_octree.cpp:54-85 -------------------------
void orc_default_config (orc_config* c)
{
  std::memset (c, 0, sizeof (*c));
  c->xres = c->yres = c->zres = 512;
  c->xsize = c->ysize = c->zsize = 3.0f;
  c->max_dist_pos = 0.03f; c->max_dist_neg = 0.03f;
  c->max_weight = 100;
  c->min_sensor_dist = 0.3f; c->max_sensor_dist = 3.0f;
  c->fx = 525.; c->fy = 525.; c->cx = 320; c->cy = 240;
  c->image_width = 640; c->image_height = 480;
  c->max_cell_x = c->max_cell_y = c->max_cell_z = 0.5f;
  c->integrate_color = 0;
  c->color_mode = 0; c->reserved_ = 0;
  c->num_threads = 0;
  for (int i = 0; i < 4; ++i) c->global_transform[i * 5] = 1.0;
}

orc_volume* orc_create (const orc_config* cfg)
{
  orc_volume* v = new orc_volume;
  v->c = *cfg;
  return v;
}

void orc_destroy (orc_volume* v) { delete v; }

// ---- reset, tsdf_volume_octree.cpp:201-219; Octree::init octree.cpp:584-599 ---------------
int orc_reset (orc_volume* v)
{
  const orc_config& c = v->c;
  v->pool.clear ();
  v->is_empty = true;
  v->color = c.integrate_color != 0;
  v->rgbn = v->color && c.color_mode == 1;
  v->root = v->pool.alloc (1, 0);
  v->init_node (v->pool.at (v->root), 0, 0, 0, c.xsize, 0, 0, 0, 0);   // size_ = size_x (octree.h:67)
  int desired_res = std::max (c.xsize / c.max_cell_x, std::max (c.ysize / c.max_cell_y, c.zsize / c.max_cell_z));
  v->num_levels = std::ceil (std::log (desired_res) / std::log (2));
  v->split_recursive (v->root, v->num_levels);
  int fl = 0;
  while ((1 << fl) < c.xres) ++fl;
  v->finest_level = fl;
  v->coarse.clear ();
  if (v->num_levels == 0) v->coarse.push_back (v->root);                // octree.cpp:613-616
  else v->get_leaves (v->root, v->coarse, v->num_levels - 1);
  // leaves already carry (d=-1, w=0) from the node ctor; setData(-1,0) at cpp:214-218 is a no-op
  std::memset (&v->stats, 0, sizeof (v->stats));
  return 0;
}

// ---- integrateCloud, impl/tsdf_volume_octree.hpp:48-103 -----------------------------------
int orc_integrate (orc_volume* v, const void* points, size_t stride, int xyz_off, int rgba_off,
                   int width, int height, const double* pose)
{
  const orc_config& c = v->c;
  if (v->root < 0) return -1;
  orc_volume::Frame f;
  f.base = static_cast<const uint8_t*> (points); f.stride = stride; f.xyz_off = xyz_off;
  f.rgba_off = v->color ? rgba_off : -1; f.width = width; f.height = height;
  double inv[16];
  affine_inverse (pose, inv);                                     // hpp:54
  float trans_f[16];
  for (int i = 0; i < 16; ++i) { f.trans_inv[i] = static_cast<float> (inv[i]); trans_f[i] = static_cast<float> (pose[i]); }
  for (auto& p : v->pt) { p.n_add = 0; p.n_visit = 0; p.n_prune = 0; p.n_resplit = 0; }

  double t0 = now_s ();
  int64_t nsplit = 0;
  for (int u = 0; u < width; ++u)                                 // hpp:59-90 (num_random_splits_ == 1)
    for (int vv = 0; vv < height; ++vv)
    {
      const float* p = f.xyz (u, vv);
      if (std::isnan (p[2])) continue;
      float pw[3];
      affine_mul<float> (trans_f, p, pw);                         // hpp:76 (noise == 0 for perm 0)
      int32_t ni = v->containing (pw[0], pw[1], pw[2]);
      if (ni < 0) continue;
      while (v->pool.at (ni).size > c.xsize / c.xres)            // hpp:80 getMinSize() > xsize_/xres_
      {
        nsplit++;
        v->split (ni, 0);
        ni = v->descend (ni, pw[0], pw[1], pw[2]);
      }
    }
  double t1 = now_s ();

  Frustum F = v->frustum (pose);                                  // hpp:93-94
  std::vector<int32_t> culled;
  for (int32_t ni : v->coarse)
  {
    const Node& n = v->pool.at (ni);
    if (pcl_frustum_contains (F, n.cx, n.cy, n.cz)) culled.push_back (ni);
  }
  double t2 = now_s ();

  int nthreads = c.num_threads;
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads ();
  if (nthreads > MAX_THREADS) nthreads = MAX_THREADS;
#pragma omp parallel for num_threads(nthreads) schedule(static)
#endif
  for (int64_t i = 0; i < static_cast<int64_t> (culled.size ()); ++i)   // hpp:95-99
    v->update_voxel (culled[i], f, thread_id ());
  double t3 = now_s ();

  v->is_empty = false;                                            // hpp:101
  orc_stats& s = v->stats;
  s.n_add_observation = 0; s.n_node_visits = 0; s.n_prune_existing = 0; s.n_prune_resplit = 0;
  for (auto& p : v->pt)
  {
    s.n_add_observation += p.n_add; s.n_node_visits += p.n_visit;
    s.n_prune_existing += p.n_prune; s.n_prune_resplit += p.n_resplit;
  }
  s.n_presplit = nsplit; s.n_culled_cells = static_cast<int64_t> (culled.size ());
  s.n_nodes = v->pool.live.load ();
  s.t_presplit = t1 - t0; s.t_cull = t2 - t1; s.t_update = t3 - t2;
  (void) nthreads;
  return 0;
}

void orc_get_stats (const orc_volume* v, orc_stats* s) { *s = v->stats; }

// ---- getFxn / getGradient / getHessian / combined, tsdf_volume_octree.cpp:655-794 ---------
int orc_query (const orc_volume* v, const float* xyz, int n, int what, int mode,
               float* val, float* grad, float* hess, uint8_t* ok)
{
  const orc_config& cfg = v->c;
  for (int i = 0; i < n; ++i)
  {
    const float* p = xyz + 3 * i;
    const Node* nb[8]; float ctrs[8][3];
    bool good = v->get_neighbors (p, nb, ctrs);
    ok[i] = good;
    if (!good) continue;
    float c = cfg.xsize / cfg.xres;
    float fv = 0, g[3] = { 0, 0, 0 }, h01 = 0, h02 = 0, h12 = 0;
    for (int k = 0; k < 8; ++k)
    {
      const Node* vox = nb[k];
      // getFxn/getGradient measure to the leaf's own centre (cpp:667, 693); getHessian and the
      // combined variants use the finest-voxel centres (cpp:715, 744, 777).
      // The reference calls unqualified fabs() on floats: with <cmath> alone that is the C
      // double fabs(double), so each (c - fabs(..)) factor and the whole product are DOUBLE and
      // only the `+=` rounds back to float (verified against the verbatim build, oracle/_ref).
      float lx = vox->cx, ly = vox->cy, lz = vox->cz;
      float fx_ = ctrs[k][0], fy_ = ctrs[k][1], fz_ = ctrs[k][2];
      float vx = mode ? fx_ : lx, vy = mode ? fy_ : ly, vz = mode ? fz_ : lz;
      double ax = c - fabs ((double) (p[0] - vx)), ay = c - fabs ((double) (p[1] - vy)), az = c - fabs ((double) (p[2] - vz));
      double bx = c - fabs ((double) (p[0] - fx_)), by = c - fabs ((double) (p[1] - fy_)), bz = c - fabs ((double) (p[2] - fz_));
      fv   += ax * ay * az * vox->d;
      g[0] += -sgn (p[0] - vx) * ay * az * vox->d;
      g[1] += ax * -sgn (p[1] - vy) * az * vox->d;
      g[2] += ax * ay * -sgn (p[2] - vz) * vox->d;
      h01 += sgn (p[0] - fx_) * sgn (p[1] - fy_) * bz * vox->d;
      h02 += sgn (p[0] - fx_) * by * sgn (p[2] - fz_) * vox->d;
      h12 += bx * sgn (p[1] - fy_) * sgn (p[2] - fz_) * vox->d;
    }
    float c3 = (c * c * c);
    if ((what & 1) && val) val[i] = fv / c3;
    if ((what & 2) && grad) { grad[3 * i] = g[0] / c3; grad[3 * i + 1] = g[1] / c3; grad[3 * i + 2] = g[2] / c3; }
    if ((what & 4) && hess)
    {
      float* H = hess + 9 * i;
      for (int k = 0; k < 9; ++k) H[k] = 0;
      H[1] = h01 / c3; H[2] = h02 / c3; H[5] = h12 / c3;
      H[3] = H[1]; H[6] = H[2]; H[7] = H[5];
    }
  }
  return 0;
}

// ---- interpolateTrilinearly through getTSDFValue (use_trilinear_interpolation_ is true and has no setter, cpp:80, :454-541) ----
int orc_interpolate (const orc_volume* v, const float* xyz, int n, float* val, uint8_t* valid_in_out)
{
  for (int i = 0; i < n; ++i)
  {
    bool valid = valid_in_out[i] != 0;
    val[i] = v->interpolate_trilinearly (xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], &valid);
    valid_in_out[i] = valid;
  }
  return 0;
}

// ---- renderView, tsdf_volume_octree.cpp:278-424 (+ renderColoredView :427-450) -------------
int orc_render (const orc_volume* v, const double* pose, int downsampleBy, void* out, size_t stride,
                int xyz_off, int normal_off, uint8_t* rgb_out)
{
  const orc_config& c = v->c;
  const float qnan = std::numeric_limits<float>::quiet_NaN ();
  int new_width = c.image_width / downsampleBy;
  int new_height = c.image_height / downsampleBy;
  double new_fx = c.fx / downsampleBy, new_fy = c.fy / downsampleBy;
  double new_cx = c.cx / downsampleBy, new_cy = c.cy / downsampleBy;
  float min_step = c.max_dist_neg * 3 / 4.;
  float rot[16], org[3], trans_f[16];
  for (int i = 0; i < 16; ++i) { rot[i] = static_cast<float> (pose[i]); trans_f[i] = rot[i]; }   // rotation() of a rigid pose
  org[0] = static_cast<float> (pose[3]); org[1] = static_cast<float> (pose[7]); org[2] = static_cast<float> (pose[11]);
  double inv[16];
  affine_inverse (pose, inv);
  int64_t npix = static_cast<int64_t> (new_width) * new_height;
  uint8_t* base = static_cast<uint8_t*> (out);
  int nthreads = c.num_threads;
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads ();
#pragma omp parallel for num_threads(nthreads) schedule(dynamic, 256)
#endif
  for (int64_t i = 0; i < npix; ++i)
  {
    size_t x = i % new_width;
    size_t y = i / new_width;
    float* P = reinterpret_cast<float*> (base + i * stride + xyz_off);
    float* N = reinterpret_cast<float*> (base + i * stride + normal_off);
    P[0] = P[1] = P[2] = 0; N[0] = N[1] = N[2] = 0;              // PointNormal default ctor
    if (rgb_out) rgb_out[3 * i] = rgb_out[3 * i + 1] = rgb_out[3 * i + 2] = 0;
    bool found_crossing = false;
    float du[3] = { static_cast<float> ((x - new_cx) / new_fx), static_cast<float> ((y - new_cy) / new_fy), 1 };
    normalize3 (du);
    { float t[3]; linear_mul<float> (rot, du, t); du[0] = t[0]; du[1] = t[1]; du[2] = t[2]; }
    float p[3] = { org[0], org[1], org[2] };
    float d = 0, w = 0, last_w = 0, last_d = 0;
    float t = c.min_sensor_dist;
    for (int k = 0; k < 3; ++k) p[k] += t * du[k];
    float step = min_step;
    bool hit_voxel = false;
    while (t < c.max_sensor_dist)
    {
      int32_t ni = v->containing (p[0], p[1], p[2]);
      if (ni >= 0)
      {
        const Node* voxel = &v->pool.at (ni);
        hit_voxel = true;
        d = voxel->d; w = voxel->w;
        if (((d < 0 && last_d > 0) || (d > 0 && last_d < 0)) && last_w && w)
        {
          found_crossing = true;
          float old_t = t - step;
          step = (c.zsize / c.zres) / 2.;
          float new_d, new_w;
          float last_new_d = d, last_new_w = w;
          while (t >= old_t)
          {
            t -= step;
            for (int k = 0; k < 3; ++k) p[k] -= step * du[k];
            ni = v->containing (p[0], p[1], p[2]);
            if (ni < 0) break;
            new_d = v->pool.at (ni).d; new_w = v->pool.at (ni).w;
            if ((last_d > 0 && new_d > 0) || (last_d < 0 && new_d < 0))
            {
              last_d = new_d; last_w = new_w;
              d = last_new_d; w = last_new_w;
              t += step;
              for (int k = 0; k < 3; ++k) p[k] += step * du[k];
              break;
            }
            last_new_d = d; last_new_w = w;
          }
          break;
        }
        last_d = d; last_w = w;
        step = std::max ((float) voxel->size / 4.f, (float) (std::fabs (d) * c.max_dist_neg));
      }
      else if (hit_voxel) break;
      t += step;
      for (int k = 0; k < 3; ++k) p[k] += step * du[k];
    }
    if (!found_crossing) { P[0] = P[1] = P[2] = qnan; continue; }
    bool has_data = true;
    float tcurr = t, tprev = t - step;
    last_d = v->interpolate_trilinearly (org[0] + tprev * du[0], org[1] + tprev * du[1], org[2] + tprev * du[2], &has_data);
    d = v->interpolate_trilinearly (org[0] + tcurr * du[0], org[1] + tcurr * du[1], org[2] + tcurr * du[2], &has_data);
    // cpp:385-388 sets NaN but cpp:389-390 overwrites it (no `continue`)
    // fabs() is the C double version here too: the whole right-hand side is evaluated in double
    float t_star = t + step * (-1 + fabs ((double) (last_d / (last_d - d))));
    float pt[3] = { org[0] + t_star * du[0], org[1] + t_star * du[1], org[2] + t_star * du[2] };
    P[0] = pt[0]; P[1] = pt[1]; P[2] = pt[2];
    int32_t ni = v->containing (pt[0], pt[1], pt[2]);
    if (ni < 0) { N[0] = N[1] = N[2] = qnan; continue; }
    float size = v->pool.at (ni).size;
    bool valid = true;
    float d_xm = v->interpolate_trilinearly (pt[0] - size, pt[1], pt[2], &valid);
    float d_xp = v->interpolate_trilinearly (pt[0] + size, pt[1], pt[2], &valid);
    float d_ym = v->interpolate_trilinearly (pt[0], pt[1] - size, pt[2], &valid);
    float d_yp = v->interpolate_trilinearly (pt[0], pt[1] + size, pt[2], &valid);
    float d_zm = v->interpolate_trilinearly (pt[0], pt[1], pt[2] - size, &valid);
    float d_zp = v->interpolate_trilinearly (pt[0], pt[1], pt[2] + size, &valid);
    if (!valid) { N[0] = N[1] = N[2] = qnan; continue; }
    float dF[3];
    dF[0] = (d_xp - d_xm) * c.max_dist_neg / (2 * size);
    dF[1] = (d_yp - d_ym) * c.max_dist_neg / (2 * size);
    dF[2] = (d_zp - d_zm) * c.max_dist_neg / (2 * size);
    normalize3 (dF);
    N[0] = dF[0]; N[1] = dF[1]; N[2] = dF[2];
  }
  // pcl::transformPointCloudWithNormals (*cloud, *cloud, trans.inverse ()), cpp:422 (is_dense == false)
  for (int64_t i = 0; i < npix; ++i)
  {
    float* P = reinterpret_cast<float*> (base + i * stride + xyz_off);
    float* N = reinterpret_cast<float*> (base + i * stride + normal_off);
    if (!std::isfinite (P[0]) || !std::isfinite (P[1]) || !std::isfinite (P[2])) continue;
    float q[3], m[3];
    pcl_transform_se3_d (inv, P, q);
    pcl_transform_so3_d (inv, N, m);
    if (rgb_out)                                                   // renderColoredView, cpp:436-448
    {
      float vt[3];
      affine_mul<float> (trans_f, q, vt);
      int32_t ni = v->containing (vt[0], vt[1], vt[2]);
      if (ni >= 0)
      {
        const Node& n = v->pool.at (ni);
        if (v->color) v->get_rgb (n, rgb_out[3 * i], rgb_out[3 * i + 1], rgb_out[3 * i + 2]);
        else rgb_out[3 * i] = rgb_out[3 * i + 1] = rgb_out[3 * i + 2] = 127;   // OctreeNode::getRGB, octree.cpp:173-178
      }
    }
    P[0] = q[0]; P[1] = q[1]; P[2] = q[2];
    N[0] = m[0]; N[1] = m[1]; N[2] = m[2];
  }
  return 0;
}

// ---- MarchingCubesTSDFOctree, src/lib/marching_cubes_tsdf_octree.cpp -----------------------
namespace {
struct MC
{
  orc_volume* v; float w_min; int color_mode;
  float lower[3], size_voxel[3];
  const float qnan = std::numeric_limits<float>::quiet_NaN ();

  // getGridValue, marching_cubes_tsdf_octree.cpp:91-106
  float grid_value (int x, int y, int z) const
  {
    float ctr[3];
    v->voxel_center (x, y, z, ctr);
    const Node& n = v->pool.at (v->containing (ctr[0], ctr[1], ctr[2]));
    if (n.w < w_min || std::fabs (n.d) >= 1) return qnan;
    return n.d * v->c.max_dist_neg;
  }
  // getValidNeighborList1D, marching_cubes_tsdf_octree.cpp:145-177
  bool neighbors (float* leaf, const int* idx) const
  {
    static const int o[8][3] = { {0,0,0}, {1,0,0}, {1,0,1}, {0,0,1}, {0,1,0}, {1,1,0}, {1,1,1}, {0,1,1} };
    for (int k = 0; k < 8; ++k)
    {
      leaf[k] = grid_value (idx[0] + o[k][0], idx[1] + o[k][1], idx[2] + o[k][2]);
      if (std::isnan (leaf[k])) return false;
    }
    return true;
  }
  // pcl::MarchingCubes::interpolateEdge (pcl/surface/impl/marching_cubes.hpp), iso_level_ = 0
  static void interpolate_edge (const float* p1, const float* p2, float v1, float v2, float* o)
  {
    const float mu = (0.0f - v1) / (v2 - v1);
    for (int k = 0; k < 3; ++k) o[k] = p1[k] + mu * (p2[k] - p1[k]);
  }
  // pcl::MarchingCubes::createSurface (pcl/surface/impl/marching_cubes.hpp)
  void create_surface (const float* leaf, const int* idx, std::vector<float>& out) const
  {
    int cubeindex = 0;
    for (int k = 0; k < 8; ++k) if (leaf[k] < 0.0f) cubeindex |= (1 << k);
    if (mc_tables::edge_table[cubeindex] == 0) return;
    float center[3], p[8][3];
    for (int k = 0; k < 3; ++k) center[k] = lower[k] + size_voxel[k] * static_cast<float> (idx[k]);
    for (int i = 0; i < 8; ++i)
    {
      p[i][0] = center[0]; p[i][1] = center[1]; p[i][2] = center[2];
      if (i & 0x4) p[i][1] = center[1] + size_voxel[1];
      if (i & 0x2) p[i][2] = center[2] + size_voxel[2];
      if ((i & 0x1) ^ ((i >> 1) & 0x1)) p[i][0] = center[0] + size_voxel[0];
    }
    float vl[12][3];
    for (int e = 0; e < 12; ++e)
      if (mc_tables::edge_table[cubeindex] & (1 << e))
      {
        int a = mc_tables::edge_corners[e][0], b = mc_tables::edge_corners[e][1];
        interpolate_edge (p[a], p[b], leaf[a], leaf[b], vl[e]);
      }
    for (int i = 0; mc_tables::tri_table[cubeindex][i] != -1; i += 3)
      for (int j = 0; j < 3; ++j)
      {
        const float* q = vl[mc_tables::tri_table[cubeindex][i + j]];
        out.push_back (q[0]); out.push_back (q[1]); out.push_back (q[2]);
      }
  }
  // reconstructVoxel, marching_cubes_tsdf_octree.cpp:179-236
  void reconstruct (int32_t ni, std::vector<float>& out, std::vector<uint8_t>& col)
  {
    const Node& n = v->pool.at (ni);
    if (n.child >= 0) { for (int i = 0; i < 8; ++i) reconstruct (n.child + i, out, col); return; }
    if (!(n.w >= w_min && std::fabs (n.d) < 1)) return;
    int idx[3];
    v->voxel_index (n.cx, n.cy, n.cz, idx[0], idx[1], idx[2]);
    if (idx[0] <= 0 || idx[0] >= v->c.xres - 1 || idx[1] <= 0 || idx[1] >= v->c.yres - 1 || idx[2] <= 0 || idx[2] >= v->c.zres - 1) return;
    float leaf[8];
    if (!neighbors (leaf, idx)) return;
    size_t before = out.size () / 3;
    create_surface (leaf, idx, out);
    if (color_mode)
      for (size_t i = before; i < out.size () / 3; ++i)
      {
        uint8_t r = 0, g = 0, b = 0;
        if (color_mode == 2)
        {
          float std_dev = (100. - n.w) / 100.;
          r = std::max (0., std::min ((1 - std_dev) * 255., 255.));
          g = 0;
          b = std::max (0., std::min ((std_dev) * 255., 255.));
        }
        else if (color_mode == 1 && v->color) v->get_rgb (n, r, g, b);
        col.push_back (r); col.push_back (g); col.push_back (b);
      }
  }
};
}

int64_t orc_mesh (orc_volume* v, float w_min, int color_mode, const float** verts, const uint8_t** rgb)
{
  MC mc; mc.v = v; mc.w_min = w_min; mc.color_mode = color_mode;
  // setInputTSDF (cpp:43-83): bounding box of the 8 "corner" points = voxelCentre(0|res); the
  // +/- half-voxel terms at :64-66 cancel exactly.  size_voxel_ = (upper-lower) * (1/res).
  float lo[3], hi[3];
  v->voxel_center (0, 0, 0, lo);
  v->voxel_center (v->c.xres, v->c.yres, v->c.zres, hi);
  int res[3] = { v->c.xres, v->c.yres, v->c.zres };
  for (int k = 0; k < 3; ++k) { mc.lower[k] = lo[k]; mc.size_voxel[k] = (hi[k] - lo[k]) * (1.0f / static_cast<float> (res[k])); }
  v->mesh_v.clear (); v->mesh_c.clear ();
  mc.reconstruct (v->root, v->mesh_v, v->mesh_c);
  // pcl::transformPointCloud (cloud, cloud, getGlobalTransform ()), cpp:122/128 (dense cloud, double math)
  for (size_t i = 0; i < v->mesh_v.size (); i += 3)
  {
    float q[3];
    pcl_transform_se3_d (v->c.global_transform, &v->mesh_v[i], q);
    v->mesh_v[i] = q[0]; v->mesh_v[i + 1] = q[1]; v->mesh_v[i + 2] = q[2];
  }
  if (verts) *verts = v->mesh_v.data ();
  if (rgb) *rgb = v->mesh_c.empty () ? nullptr : v->mesh_c.data ();
  return static_cast<int64_t> (v->mesh_v.size () / 3);
}

// ---- save, tsdf_volume_octree.cpp:222-245; Octree::serialize octree.cpp:645-657;
//      OctreeNode::serialize :289-304; RGBNode::serialize :360-367;
//      eigen_extensions::serializeASCII eigen_extensions.h:249-257 ----------------------------
namespace {
std::string fmt16 (double x) { char b[64]; std::snprintf (b, sizeof (b), "%.16g", x); return b; }
void write_node (const orc_volume* v, std::FILE* f, int32_t ni)
{
  const Node& n = v->pool.at (ni);
  // RGBNormalized::serialize (octree.cpp:417-424) writes sizeof (uint8_t) = the FIRST BYTE of each of its four floats
  if (v->rgbn) { std::fwrite (&n.rn, 1, 1, f); std::fwrite (&n.gn, 1, 1, f); std::fwrite (&n.bn, 1, 1, f); std::fwrite (&n.in, 1, 1, f); }
  else if (v->color) { std::fwrite (&n.r, 1, 1, f); std::fwrite (&n.g, 1, 1, f); std::fwrite (&n.b, 1, 1, f); }
  std::fwrite (&n.d, 4, 1, f); std::fwrite (&n.w, 4, 1, f);
  std::fwrite (&n.cx, 4, 1, f); std::fwrite (&n.cy, 4, 1, f); std::fwrite (&n.cz, 4, 1, f);
  std::fwrite (&n.size, 4, 1, f); std::fwrite (&n.M, 4, 1, f); std::fwrite (&n.ns, 4, 1, f);
  size_t nchild = n.child >= 0 ? 8 : 0;
  std::fwrite (&nchild, sizeof (size_t), 1, f);
  for (size_t i = 0; i < nchild; ++i) write_node (v, f, n.child + static_cast<int32_t> (i));
}
}

int orc_save (const orc_volume* v, const char* path)
{
  const orc_config& c = v->c;
  std::FILE* f = std::fopen (path, "wb");
  if (!f) return -1;
  std::string h = "# TSDFVolumeOctree Meta Information\n";
  h += std::to_string (c.xres) + " " + std::to_string (c.yres) + " " + std::to_string (c.zres) + "\n";
  h += fmt16 (c.xsize) + " " + fmt16 (c.ysize) + " " + fmt16 (c.zsize) + "\n";
  h += fmt16 (c.max_dist_pos) + "\n" + fmt16 (c.max_dist_neg) + "\n" + fmt16 (c.max_weight) + "\n";
  h += fmt16 (c.min_sensor_dist) + "\n" + fmt16 (c.max_sensor_dist) + "\n";
  h += fmt16 (c.max_cell_x) + " " + fmt16 (c.max_cell_y) + " " + fmt16 (c.max_cell_z) + "\n";
  h += fmt16 (c.fx) + " " + fmt16 (c.fy) + " " + fmt16 (c.cx) + " " + fmt16 (c.cy) + "\n";
  h += std::to_string (c.image_width) + " " + std::to_string (c.image_height) + "\n";
  h += std::string (v->is_empty ? "1" : "0") + "\n0\n0\n";       // is_empty_, weight_by_depth_, weight_by_variance_
  h += "% 4 4\n";
  // Eigen operator<< default IOFormat: columns aligned to the widest coefficient
  std::string cell[16]; size_t width = 0;
  for (int i = 0; i < 16; ++i) { cell[i] = fmt16 (c.global_transform[i]); width = std::max (width, cell[i].size ()); }
  for (int r = 0; r < 4; ++r)
  {
    for (int k = 0; k < 4; ++k)
    {
      if (k) h += " ";
      h += std::string (width - cell[r * 4 + k].size (), ' ') + cell[r * 4 + k];
    }
    h += "\n";
  }
  h += std::string (v->rgbn ? "RGBNormalized" : (v->color ? "RGB" : "NOCOLOR")) + "\n#OCTREEBINARY\n";
  std::fwrite (h.data (), 1, h.size (), f);
  size_t res[3] = { (size_t) c.xres, (size_t) c.yres, (size_t) c.zres };
  std::fwrite (res, sizeof (size_t), 3, f);
  std::fwrite (&c.xsize, 4, 1, f); std::fwrite (&c.ysize, 4, 1, f); std::fwrite (&c.zsize, 4, 1, f);
  write_node (v, f, v->root);
  std::fclose (f);
  return 0;
}

// ---- test helpers ---------------------------------------------------------------------------
namespace {
struct Rec { int32_t k[4]; int32_t ni; };
void collect (const orc_volume* v, int32_t ni, std::vector<Rec>& out)
{
  const Node& n = v->pool.at (ni);
  if (n.level >= v->num_levels) out.push_back ({ { n.level, n.ix, n.iy, n.iz }, ni });
  if (n.child >= 0) for (int i = 0; i < 8; ++i) collect (v, n.child + i, out);
}
}

int64_t orc_dump_nodes (const orc_volume* v, int32_t* keys, float* dw, uint8_t* flags,
                        uint8_t* rgb, float* M, int32_t* ns)
{
  std::vector<Rec> recs;
  collect (v, v->root, recs);
  if (!keys && !dw && !flags && !rgb && !M && !ns) return static_cast<int64_t> (recs.size ());
  std::sort (recs.begin (), recs.end (), [] (const Rec& a, const Rec& b) {
    return std::lexicographical_compare (a.k, a.k + 4, b.k, b.k + 4); });
  for (size_t i = 0; i < recs.size (); ++i)
  {
    const Node& n = v->pool.at (recs[i].ni);
    if (keys) std::memcpy (keys + 4 * i, recs[i].k, 16);
    if (dw) { dw[2 * i] = n.d; dw[2 * i + 1] = n.w; }
    if (flags) flags[i] = n.child >= 0;
    if (rgb) v->get_rgb (n, rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]);
    if (M) M[i] = n.M;
    if (ns) ns[i] = n.ns;
  }
  return static_cast<int64_t> (recs.size ());
}

int64_t orc_dump_color_payload (const orc_volume* v, float* out4)
{
  if (!v->rgbn) return 0;
  std::vector<Rec> recs;
  collect (v, v->root, recs);
  std::sort (recs.begin (), recs.end (), [] (const Rec& a, const Rec& b) {
    return std::lexicographical_compare (a.k, a.k + 4, b.k, b.k + 4); });
  for (size_t i = 0; i < recs.size (); ++i)
  {
    const Node& n = v->pool.at (recs[i].ni);
    out4[4 * i] = n.rn; out4[4 * i + 1] = n.gn; out4[4 * i + 2] = n.bn; out4[4 * i + 3] = n.in;
  }
  return static_cast<int64_t> (recs.size ());
}

int orc_levels (const orc_volume* v, int* coarse_level, int* finest_level)
{
  if (coarse_level) *coarse_level = v->num_levels;
  if (finest_level) *finest_level = v->finest_level;
  return 0;
}

void orc_voxel_center (const orc_volume* v, int64_t x, int64_t y, int64_t z, float* o) { v->voxel_center (x, y, z, o); }

int orc_voxel_index (const orc_volume* v, float x, float y, float z, int* o)
{ return v->voxel_index (x, y, z, o[0], o[1], o[2]); }

int orc_frustum_cull (const orc_volume* v, const double* pose, uint8_t* mask)
{
  Frustum F = v->frustum (pose);
  int n = 1 << v->num_levels, kept = 0;
  std::memset (mask, 0, static_cast<size_t> (n) * n * n);
  for (int32_t ni : v->coarse)
  {
    const Node& nd = v->pool.at (ni);
    if (pcl_frustum_contains (F, nd.cx, nd.cy, nd.cz)) { mask[(static_cast<size_t> (nd.ix) * n + nd.iy) * n + nd.iz] = 1; ++kept; }
  }
  return kept;
}

} // extern "C"
