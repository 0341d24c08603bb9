// tests/emu/emu.cpp — HOST EMULATION of the engine's device code.  TEST HARNESS ONLY.
//
// There is no GPU in the development container, so this file compiles the engine's
// __host__ __device__ core (cpu_tsdf_b200/csrc/tsdf_core.cuh — the very code the CUDA kernels
// call) for the host and drives it serially: one "thread" per pixel / cell / point in a plain
// loop.  The not-gpu tests compare it with the oracle to validate the flat layout, the hash
// directory and the per-node arithmetic before any GPU time is spent.  It is NOT part of the
// product: libb200tsdf.so has no CPU path and nothing in cpu_tsdf_b200/ loads this library.
#define B2_EMU_BFS 1
#include "../../cpu_tsdf_b200/csrc/tsdf_core.cuh"
#include "../../cpu_tsdf_b200/csrc/organize.cuh"
#include "../../cpu_tsdf_b200/csrc/meshpost_core.cuh"
#include "../../cpu_tsdf_b200/csrc/host_math.h"
#include "../../cpu_tsdf_b200/csrc/params_setup.h"
#include "../../oracle/mc_tables.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

using namespace b2;

// record capacity of the breadth-first fresh-subtree visit in the emulated frames (B2_EMU_BFS_CAP: 0 = recursion only,
// 8..1024 = every split goes through fresh_children_bfs with that many records; small values exercise the overflow path)
namespace b2 { int b2_emu_bfs_cap = 128; }

struct Emu
{
  b200tsdf_config cfg;
  Params p{};
  std::vector<uint64_t> keys; std::vector<float2> nodes; std::vector<uint32_t> split;
  std::vector<uchar4> rgb; std::vector<float> M; std::vector<int> ns;
  std::vector<float2> root_dw; std::vector<uint32_t> root_split; std::vector<uchar4> root_rgb;
  std::vector<float> root_M; std::vector<int> root_ns;
  int err = 0;
  long long n_updates = 0, n_visits = 0, n_culled = 0;
  std::vector<float> mesh_v; std::vector<unsigned char> mesh_c;
};

struct Rec { int32_t k[4]; float d, w; uint8_t split, r, g, b; float M; int32_t ns; };

static void collect (const Params& p, const NodePos& n, std::vector<Rec>& out)
{
  Rec r; r.k[0] = n.level; r.k[1] = n.x; r.k[2] = n.y; r.k[3] = n.z;
  float2 dw = *node_dw (p, n);
  r.d = dw.x; r.w = dw.y; r.r = r.g = r.b = 0; r.M = 0; r.ns = 0;
  if (n.slot < 0)
  {
    if (p.root_rgb) { uchar4 c = p.root_rgb[n.idx]; r.r = c.x; r.g = c.y; r.b = c.z; }
    if (p.root_M) { r.M = p.root_M[n.idx]; r.ns = p.root_ns[n.idx]; }
  }
  else
  {
    size_t i = (size_t) n.slot * BRICK_NODES + n.idx;
    if (p.rgb) { uchar4 c = p.rgb[i]; r.r = c.x; r.g = c.y; r.b = c.z; }
    if (p.M) { r.M = p.M[i]; r.ns = p.ns[i]; }
  }
  bool sp = is_split (p, n);
  r.split = sp;
  out.push_back (r);
  if (!sp) return;
  int cs = children_slot (p, n, false);
  if (cs < 0) return;
  for (int c = 0; c < 8; ++c) collect (p, make_child (p, n, c, cs), out);
}

// The kernels' walk of the flat layout (k_mesh_bricks / k_leaves_bricks, then k_mesh_roots / k_leaves_roots) in plain loops:
// every node of every claimed brick whose root has children, then every root-array entry.  visit (b, dw, slot, i) gets the
// node as brick_node describes it, its {sdf, weight} and its storage (slot -1: root array, i = root index).
template <typename Visit>
static void walk_nodes (const Params& p, const Visit& visit)
{
  for (size_t slot = 0; slot <= p.pool_mask; ++slot)
  {
    if (p.keys[slot] == KEY_EMPTY) continue;
    int t, bx, by, bz;
    brick_key_decode (p.keys[slot], t, bx, by, bz);
    if (!brick_root_is_split (p, t, bx, by, bz)) continue;
    const uint32_t* sw = p.split + slot * BRICK_SPLIT_WORDS;
    for (int i = 0; i < BRICK_NODES; ++i)
      visit (brick_node (p, sw, tier_root_level (p, t), bx, by, bz, true, i), p.nodes[slot * BRICK_NODES + i], (int) slot, i);
  }
  const int n = 1 << p.Rtop;
  for (int i = 0; i < n * n * n; ++i)
  {
    const NodePos nd = make_root (p, i / (n * n), (i / n) % n, i % n);
    BrickNode b; b.level = p.Rtop; b.x = nd.x; b.y = nd.y; b.z = nd.z; b.exists = true; b.split = is_split (p, nd);
    visit (b, p.root_dw[nd.idx], -1, nd.idx);
  }
}

extern "C" {

Emu* emu_create (const b200tsdf_config* cfg) { Emu* e = new Emu; e->cfg = *cfg; return e; }
void emu_destroy (Emu* e) { delete e; }

int emu_reset (Emu* e)
{
  if (const char* c = std::getenv ("B2_EMU_BFS_CAP")) b2_emu_bfs_cap = std::min (1024, std::atoi (c) / 8 * 8);
  size_t pool, root_n;
  if (derive_params (e->cfg, e->p, pool, root_n)) return -1;
  Params& p = e->p;
  e->keys.assign (pool, KEY_EMPTY);
  e->nodes.assign (pool * BRICK_NODES, make_float2 (-1.f, 0.f));
  e->split.assign (pool * BRICK_SPLIT_WORDS, 0u);
  e->root_dw.assign (root_n, make_float2 (-1.f, 0.f));
  e->root_split.assign ((root_n + 31) / 32, 0u);
  p.keys = e->keys.data (); p.nodes = e->nodes.data (); p.split = e->split.data ();
  p.root_dw = e->root_dw.data (); p.root_split = e->root_split.data ();
  p.rgb = nullptr; p.M = nullptr; p.ns = nullptr; p.root_rgb = nullptr; p.root_M = nullptr; p.root_ns = nullptr;
  if (p.color)
  {
    e->rgb.assign (pool * BRICK_NODES, make_uchar4 (0, 0, 0, 0)); e->root_rgb.assign (root_n, make_uchar4 (0, 0, 0, 0));
    p.rgb = e->rgb.data (); p.root_rgb = e->root_rgb.data ();
  }
  if (p.track_var)
  {
    e->M.assign (pool * BRICK_NODES, 0.f); e->ns.assign (pool * BRICK_NODES, 0);
    e->root_M.assign (root_n, 0.f); e->root_ns.assign (root_n, 0);
    p.M = e->M.data (); p.ns = e->ns.data (); p.root_M = e->root_M.data (); p.root_ns = e->root_ns.data ();
  }
  e->err = 0; p.err = &e->err;
  if (p.Rtop < p.C)
  {
    int n = 1 << p.Rtop;
    for (int x = 0; x < n; ++x) for (int y = 0; y < n; ++y) for (int z = 0; z < n; ++z) find_or_insert_brick (p, p.T - 1, x, y, z);
  }
  return 0;
}

int emu_integrate (Emu* e, const void* points, size_t stride, int xyz_off, int rgba_off, int W, int H, const double* pose)
{
  const Params& p = e->p;
  Frame f;
  f.pts = (const unsigned char*) points; f.stride = (int) stride; f.xyz_off = xyz_off; f.rgba_off = p.color ? rgba_off : -1;
  f.width = W; f.height = H;
  double inv[12];
  b2host::affine_inverse (pose, inv);
  for (int i = 0; i < 12; ++i) { f.tinv[i] = (float) inv[i]; f.tfwd[i] = (float) pose[i]; }
  // k_presplit
  for (int i = 0; i < W * H; ++i)
  {
    int u = i % W, v = i / W;
    const float* pt = frame_xyz (f, u, v);
    if (is_nan (pt[2])) continue;
    float pw[3];
    affine_mul_f (f.tfwd, pt[0], pt[1], pt[2], pw);
    int fx_, fy_, fz_;
    if (!world_to_finest (p, pw[0], pw[1], pw[2], fx_, fy_, fz_)) continue;
    int sh = p.L - p.C;
    if (!owns_cell (p, fx_ >> sh, fy_ >> sh, fz_ >> sh)) continue;
    presplit_point (p, fx_, fy_, fz_);
  }
  // k_cull + k_update_dfs
  float pl[6][4];
  b2host::frustum_planes (pose, p.width, p.height, p.fx, p.fy, p.min_sensor, p.max_sensor, pl);
  int n = 1 << p.C;
  Counters cnt; cnt.n_updates = 0; cnt.n_visits = 0;
  e->n_culled = 0;
  for (int x = 0; x < n; ++x) for (int y = 0; y < n; ++y) for (int z = 0; z < n; ++z)
  {
    if (!frustum_contains (pl, center1d (p, p.C, x), center1d (p, p.C, y), center1d (p, p.C, z))) continue;
    if (!owns_cell (p, x, y, z)) continue;
    e->n_culled++;
    NodePos nd;
    if (!locate_node (p, p.C, x, y, z, nd)) return -2;
    update_voxel_dfs (p, f, nd, cnt);
  }
  e->n_updates = cnt.n_updates; e->n_visits = cnt.n_visits;
  return e->err;
}

void emu_stats (const Emu* e, long long* out3) { out3[0] = e->n_updates; out3[1] = e->n_visits; out3[2] = e->n_culled; }

long long emu_dump_nodes (const Emu* e, int32_t* keys, float* dw, uint8_t* flags, uint8_t* rgb, float* M, int32_t* ns)
{
  const Params& p = e->p;
  std::vector<Rec> recs;
  int n = 1 << p.C;
  for (int x = 0; x < n; ++x) for (int y = 0; y < n; ++y) for (int z = 0; z < n; ++z)
  {
    NodePos nd;
    if (!locate_node (p, p.C, x, y, z, nd)) return -1;
    collect (p, nd, recs);
  }
  if (!keys && !dw && !flags && !rgb && !M && !ns) return (long long) recs.size ();
  std::sort (recs.begin (), recs.end (), [] (const Rec& a, const Rec& b) { return std::lexicographical_compare (a.k, a.k + 4, b.k, b.k + 4); });
  for (size_t i = 0; i < recs.size (); ++i)
  {
    const Rec& r = recs[i];
    if (keys) std::memcpy (keys + 4 * i, r.k, 16);
    if (dw) { dw[2 * i] = r.d; dw[2 * i + 1] = r.w; }
    if (flags) flags[i] = r.split;
    if (rgb) { rgb[3 * i] = r.r; rgb[3 * i + 1] = r.g; rgb[3 * i + 2] = r.b; }
    if (M) M[i] = r.M;
    if (ns) ns[i] = r.ns;
  }
  return (long long) recs.size ();
}

int emu_query (const Emu* e, const float* xyz, int n, int what, int mode, float* val, float* grad, float* hess, uint8_t* ok)
{
  for (int i = 0; i < n; ++i)
  {
    float v, g[3], hs[9];
    bool good = query_point (e->p, xyz + 3 * i, mode, &v, g, hs);
    ok[i] = good;
    if (!good) continue;
    if (what & 1) val[i] = v;
    if (what & 2) { grad[3 * i] = g[0]; grad[3 * i + 1] = g[1]; grad[3 * i + 2] = g[2]; }
    if (what & 4) for (int k = 0; k < 9; ++k) hess[9 * i + k] = hs[k];
  }
  return 0;
}

// k_interpolate: valid_in_out holds the caller's flags on entry and is only ever cleared
int emu_interpolate (const Emu* e, const float* xyz, int n, float* val, uint8_t* valid_in_out)
{
  for (int i = 0; i < n; ++i)
  {
    bool v = valid_in_out[i] != 0;
    val[i] = interpolate_trilinearly (e->p, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], &v);
    valid_in_out[i] = v ? 1 : 0;
  }
  return 0;
}

int emu_render (const Emu* e, const double* pose, int downsample, void* out, size_t stride, int xyz_off, int normal_off, uint8_t* rgb_out)
{
  RenderParams r;
  make_render_params (e->cfg, e->p, pose, downsample, r);
  unsigned char* base = (unsigned char*) out;
  for (int y = 0; y < r.height; ++y) for (int x = 0; x < r.width; ++x)
  {
    size_t i = (size_t) y * r.width + x;
    float P[3], N[3];
    render_pixel (e->p, r, x, y, P, N, rgb_out ? rgb_out + 3 * i : nullptr);
    std::memcpy (base + i * stride + xyz_off, P, 12);
    std::memcpy (base + i * stride + normal_off, N, 12);
  }
  return 0;
}

long long emu_mesh (Emu* e, float w_min, int color_mode, const float** verts, const uint8_t** cols)
{
  const Params& p = e->p;
  McParams mc;
  make_mc_params (e->cfg, p, w_min, color_mode, mc);
  e->mesh_v.clear (); e->mesh_c.clear ();
  // k_mesh_bricks / k_mesh_roots: one cube per existing leaf at or below the coarse depth, then sorted by the order key
  std::vector<std::pair<unsigned long long, size_t> > order;
  walk_nodes (p, [&] (const BrickNode& b, float2 dw, int slot, int i)
  {
    if (!b.exists || b.split || b.level < p.C) return;
    const NodePos q = brick_node_pos (p, b, slot, i);
    float v[45]; unsigned char cc[45];
    int nt = mc_leaf (p, mc, q, dw.x, dw.y, mc_tables::edge_table, mc_tables::tri_table, v, color_mode ? cc : nullptr);
    for (int k = 0; k < 9 * nt; ++k) { e->mesh_v.push_back (v[k]); if (color_mode) e->mesh_c.push_back (cc[k]); }
    for (int t = 0; t < nt; ++t) order.push_back ({ (mc_order_key (p, q) << 3) | (unsigned long long) t, order.size () });
  });
  // the engine sorts its (unordered) emission by mc_order_key: the result must be the reference's own order
  std::sort (order.begin (), order.end ());
  {
    std::vector<float> sv (e->mesh_v.size ()); std::vector<unsigned char> sc (e->mesh_c.size ());
    for (size_t t = 0; t < order.size (); ++t)
    {
      size_t src = order[t].second;
      std::copy (e->mesh_v.begin () + 9 * src, e->mesh_v.begin () + 9 * src + 9, sv.begin () + 9 * t);
      if (color_mode) std::copy (e->mesh_c.begin () + 9 * src, e->mesh_c.begin () + 9 * src + 9, sc.begin () + 9 * t);
    }
    e->mesh_v.swap (sv); e->mesh_c.swap (sc);
  }
  *verts = e->mesh_v.data ();
  if (cols) *cols = color_mode ? e->mesh_c.data () : nullptr;
  return (long long) (e->mesh_v.size () / 3);
}

int emu_levels (const Emu* e, int* out4) { out4[0] = e->p.C; out4[1] = e->p.L; out4[2] = e->p.T; out4[3] = e->p.Rtop; return 0; }

int emu_frustum_cull (const Emu* e, const double* pose, uint8_t* mask)
{
  const Params& p = e->p;
  float pl[6][4];
  b2host::frustum_planes (pose, p.width, p.height, p.fx, p.fy, p.min_sensor, p.max_sensor, pl);
  int n = 1 << p.C, kept = 0;
  for (int x = 0; x < n; ++x) for (int y = 0; y < n; ++y) for (int z = 0; z < n; ++z)
  {
    bool in = frustum_contains (pl, center1d (p, p.C, x), center1d (p, p.C, y), center1d (p, p.C, z));
    mask[((size_t) x * n + y) * n + z] = in; kept += in;
  }
  return kept;
}

} // extern "C"

// organize.cuh driven serially in REVERSE point order (the device order is arbitrary): the result must
// not depend on it
extern "C" long long emu_organize (const void* points, size_t n, size_t stride, int xyz_off, int rgba_off, const float* intr,
                                   int width, int height, float cloud_units, int zero_nans, const double* tf,
                                   void* out, size_t out_stride, int out_rgba_off)
{
  OrgParams o{};
  o.fx = intr[0]; o.fy = intr[1]; o.cx = intr[2]; o.cy = intr[3]; o.width = width; o.height = height;
  o.cloud_units = cloud_units; o.zero_nans = zero_nans; o.has_tf = tf != nullptr;
  if (tf) for (int i = 0; i < 12; ++i) o.tf[i] = tf[i];
  const unsigned char* pts = (const unsigned char*) points;
  size_t npix = (size_t) width * height;
  std::vector<unsigned long long> zkey (npix, ~0ull);
  for (size_t j = n; j-- > 0;)
  {
    float x, y, z;
    org_load (pts, stride, xyz_off, j, x, y, z);
    org_prepare (o, x, y, z);
    int pix = org_pixel (o, x, y, z);
    if (pix < 0) continue;
    zkey[pix] = std::min (zkey[pix], org_key (z, (unsigned int) j));
  }
  long long filled = 0;
  for (size_t i = 0; i < npix; ++i)
  {
    filled += zkey[i] != ~0ull;
    org_emit (o, pts, stride, xyz_off, rgba_off, zkey[i], (unsigned char*) out + i * out_stride, out_stride, out_rgba_off);
  }
  return filled;
}


// ---- meshpost_core.cuh driven serially, every per-element loop in REVERSE order -------------------------
namespace {
struct HostGrid
{
  std::vector<uint64_t> keys; std::vector<int> head, next; PointGrid g{};
  HostGrid (const float* pts, int n, double cell)
  {
    size_t slots = 1024; while (slots < 2 * (size_t) n) slots <<= 1;
    keys.assign (slots, GRID_EMPTY); head.assign (slots, -1); next.assign (std::max (n, 1), -1);
    g.keys = keys.data (); g.head = head.data (); g.next = next.data (); g.mask = (uint32_t) (slots - 1); g.inv_cell = 1.0 / cell; g.pts = pts;
    for (int i = n; i-- > 0;) grid_insert (g, i);
  }
};
}

extern "C" void emu_mesh_flatten (const float* verts, size_t nverts, const int32_t* tris, size_t ntris, float min_dist,
                                  float* out_verts, size_t* out_nverts, int32_t* out_tris, size_t* out_ntris, int* rounds_out)
{
  int nv = (int) nverts;
  const float r2 = min_dist > 0.f ? (float) ((double) min_dist * (double) min_dist) : 0.f;
  HostGrid G (verts, nv, std::max ((double) min_dist * 1.001, 1e-7));
  std::vector<unsigned char> state (std::max (nv, 1), FV_UNDECIDED);
  int rounds = 0;
  for (bool again = true; again; ++rounds)
  {
    again = false;
    for (int i = nv; i-- > 0;) again |= fv_round (G.g, r2, state.data (), i);
  }
  if (rounds_out) *rounds_out = rounds;
  std::vector<int> rep (nv), rank (nv);
  size_t k = 0;
  for (int i = 0; i < nv; ++i) { rank[i] = (int) k; if (state[i] == FV_KEPT) { for (int c = 0; c < 3; ++c) out_verts[3 * k + c] = verts[3 * (size_t) i + c]; ++k; } }
  for (int i = nv; i-- > 0;) rep[i] = fv_target (G.g, r2, state.data (), i);
  size_t f = 0;
  for (size_t t = 0; t < ntris; ++t)
  {
    int a = rank[rep[tris[3 * t]]], b = rank[rep[tris[3 * t + 1]]], c = rank[rep[tris[3 * t + 2]]];
    if (a == b || b == c || c == a) continue;
    out_tris[3 * f] = a; out_tris[3 * f + 1] = b; out_tris[3 * f + 2] = c; ++f;
  }
  *out_nverts = k; *out_ntris = f;
}

extern "C" void emu_mesh_cleanup (const float* verts, size_t nverts, const int32_t* tris, size_t ntris, float face_dist, int K,
                                  float* out_verts, size_t* out_nverts, int32_t* out_tris, size_t* out_ntris)
{
  int nt = (int) ntris;
  const float r2 = face_dist > 0.f ? (float) ((double) face_dist * (double) face_dist) : 0.f;
  std::vector<float> cent (3 * std::max<size_t> (ntris, 1));
  for (int t = nt; t-- > 0;) face_centroid (verts, tris + 3 * (size_t) t, cent.data () + 3 * (size_t) t);
  HostGrid G (cent.data (), nt, std::max ((double) face_dist * 1.001, 1e-7));
  std::vector<int> cnt (nt), nb ((size_t) std::max (nt, 1) * (CM_MAX_K - 1)), parent (nt), touches (nt, 0), size (nt, 0), has_big (nt, 0), keep (nt);
  for (int t = nt; t-- > 0;) { cnt[t] = cm_count (G.g, r2, K, t, nb.data ()); parent[t] = t; }
  for (int t = nt; t-- > 0;)
  {
    if (cnt[t] >= K) continue;
    for (int k = 0; k < cnt[t]; ++k) { int j = nb[(size_t) t * (CM_MAX_K - 1) + k]; if (cnt[j] >= K) touches[t] = 1; else uf_union (parent.data (), t, j); }
  }
  for (int t = nt; t-- > 0;) if (cnt[t] < K) { int r = uf_find (parent.data (), t); size[r]++; if (touches[t]) has_big[r] = 1; }
  for (int t = 0; t < nt; ++t)
  {
    bool remove = false;
    if (cnt[t] < K) { int r = uf_find (parent.data (), t); remove = !has_big[r] && size[r] <= K; }
    keep[t] = !remove;
  }
  std::vector<int> used (nverts, 0), vrank (nverts, 0);
  for (int t = 0; t < nt; ++t) if (keep[t]) for (int c = 0; c < 3; ++c) used[tris[3 * (size_t) t + c]] = 1;
  size_t k = 0;
  for (size_t i = 0; i < nverts; ++i) { vrank[i] = (int) k; if (used[i]) { for (int c = 0; c < 3; ++c) out_verts[3 * k + c] = verts[3 * i + c]; ++k; } }
  size_t f = 0;
  for (int t = 0; t < nt; ++t) if (keep[t]) { for (int c = 0; c < 3; ++c) out_tris[3 * f + c] = vrank[tris[3 * (size_t) t + c]]; ++f; }
  *out_nverts = k; *out_ntris = f;
}
