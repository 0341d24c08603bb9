// vol_io.cuh — the per-record routines of the device .vol writer and parser (DESIGN.md §3e), shared by the kernels of
// engine.cu, the host loader there and the host emulation of the tests.
//
// A .vol body is the reference's pre-order walk of the octree (OctreeNode::serialize, octree.cpp:289-304; RGBNode :360-367;
// RGBNormalized :416-424), one fixed-size record per node: the colour bytes (3 for RGB, the first byte of each of the four
// RGBNormalized floats, none for NOCOLOR), d, w, the centre, the size, M, nsample, then nchild as a size_t (0 or 8).
// Every record carries its own centre and size, so each one can be written, and read back, on its own.
#pragma once
#include "tsdf_core.cuh"

namespace b2 {

constexpr int VOL_SLOT_GEOM = -2;            // a record of a level above the root arrays: geometry only, always 8 children
constexpr int VOL_KEY_LEVEL_BITS = 5;

B2_HD int vol_record_bytes (bool color, bool color_norm) { return color_norm ? 44 : (color ? 43 : 40); }
B2_HD int vol_color_bytes (bool color, bool color_norm) { return color_norm ? 4 : (color ? 3 : 0); }

// Position of a node in the pre-order walk: the bit-interleaved finest coordinates of its first voxel, then its level.  A
// node sorts before its whole subtree (same first voxel, smaller level), and the subtree before the next sibling.
// 3 L + 5 bits (at most 62).
B2_HD unsigned long long vol_key (const Params& p, int level, int x, int y, int z)
{
  NodePos n; n.level = level; n.x = x; n.y = y; n.z = z;
  return (mc_order_key (p, n) << VOL_KEY_LEVEL_BITS) | (unsigned long long) level;
}
B2_HD void vol_key_decode (const Params& p, unsigned long long k, int& level, int& x, int& y, int& z)
{
  level = (int) (k & ((1u << VOL_KEY_LEVEL_BITS) - 1));
  morton_decode (p.L, k >> VOL_KEY_LEVEL_BITS, x, y, z);
  x >>= p.L - level; y >>= p.L - level; z >>= p.L - level;
}

// One node of the walk, as the sort carries it: its key, its storage (slot: brick, -1 root arrays, VOL_SLOT_GEOM none) and
// whether the file gives it children.  Four 32-bit words.
struct VolNode { uint32_t key_lo, key_hi; int32_t slot; uint32_t idx_nchild; };
B2_HD VolNode vol_node (unsigned long long key, int slot, int idx, bool children)
{
  VolNode v; v.key_lo = (uint32_t) key; v.key_hi = (uint32_t) (key >> 32); v.slot = slot;
  v.idx_nchild = (uint32_t) idx | (children ? 0x80000000u : 0u);
  return v;
}

// Whether the writer gives a stored node children: it has them (is_split) and the brick that holds them exists.
B2_HD bool vol_has_children (const Params& p, const NodePos& n)
{
  return is_split (p, n) && children_slot (p, n, false) >= 0;
}

B2_HD void vol_put (unsigned char* o, const void* v, int bytes)
{
  const unsigned char* s = (const unsigned char*) v;
  for (int i = 0; i < bytes; ++i) o[i] = s[i];
}

// The record of one node, written at o (vol_record_bytes bytes); the state is read where write_vol_node read it.
B2_HD void vol_format (const Params& p, const VolNode& v, unsigned char* o)
{
  int level, x, y, z;
  vol_key_decode (p, ((unsigned long long) v.key_hi << 32) | v.key_lo, level, x, y, z);
  NodePos n;
  n.level = level; n.x = x; n.y = y; n.z = z;
  n.cx = center1d (p, level, x); n.cy = center1d (p, level, y); n.cz = center1d (p, level, z);
  n.size = level_size (p, level);
  n.slot = v.slot; n.idx = (int) (v.idx_nchild & 0x7FFFFFFFu);
  float d = -1.f, w = 0.f, M = 0.f; int ns = 0;
  unsigned char col[4] = { 0, 0, 0, 0 };
  if (v.slot != VOL_SLOT_GEOM)
  {
    const float2 dw = *node_dw (p, n); d = dw.x; w = dw.y;
    if (p.color_norm)
    {
      const float4 q = *node_rgbn (p, n);
      const float qs[4] = { q.x, q.y, q.z, q.w };
      for (int k = 0; k < 4; ++k) col[k] = (unsigned char) (float_bits (qs[k]) & 0xFFu);   // little-endian first byte
    }
    if (n.slot < 0)
    {
      if (p.root_rgb && !p.color_norm) { const uchar4 c = p.root_rgb[n.idx]; col[0] = c.x; col[1] = c.y; col[2] = c.z; }
      if (p.root_M) { M = p.root_M[n.idx]; ns = p.root_ns[n.idx]; }
    }
    else
    {
      const size_t i = (size_t) n.slot * BRICK_NODES + n.idx;
      if (p.rgb && !p.color_norm) { const uchar4 c = p.rgb[i]; col[0] = c.x; col[1] = c.y; col[2] = c.z; }
      if (p.M) { M = p.M[i]; ns = p.ns[i]; }
    }
  }
  const int cb = vol_color_bytes (p.color != 0, p.color_norm != 0);
  vol_put (o, col, cb); o += cb;
  vol_put (o, &d, 4); vol_put (o + 4, &w, 4);
  vol_put (o + 8, &n.cx, 4); vol_put (o + 12, &n.cy, 4); vol_put (o + 16, &n.cz, 4); vol_put (o + 20, &n.size, 4);
  vol_put (o + 24, &M, 4); vol_put (o + 28, &ns, 4);
  const unsigned long long nchild = (v.idx_nchild & 0x80000000u) ? 8ull : 0ull;
  vol_put (o + 32, &nchild, 8);
}

// ---- parsing ----------------------------------------------------------------------------------------------------------
// One record as read: its fields, and the node its size and centre name.  `placed` is false when nchild is neither 0 nor 8,
// no level of the grid has that size bit for bit, or no node of that level has that centre bit for bit.
struct VolRec
{
  unsigned char c[3];
  float d, w, M; int ns;
  unsigned long long nchild;
  bool placed;
  int level, x, y, z;
};

B2_HD void vol_get (const unsigned char* s, void* v, int bytes)
{
  unsigned char* o = (unsigned char*) v;
  for (int i = 0; i < bytes; ++i) o[i] = s[i];
}

// the index i in [0, 2^level) with center1d (level, i) == c bit for bit, or -1.  center1d is monotonic in i, so a binary
// search over the bisection the writer's accumulation performs finds the only candidate.
B2_HD int vol_index_of_center (const Params& p, int level, float c)
{
  const uint32_t cb = float_bits (c);
  int lo = 0, hi = (1 << level) - 1;
  while (lo < hi)
  {
    const int mid = lo + ((hi - lo) >> 1);
    if (center1d (p, level, mid) < c) lo = mid + 1; else hi = mid;
  }
  return float_bits (center1d (p, level, lo)) == cb ? lo : -1;
}

B2_HD VolRec vol_parse (const Params& p, const unsigned char* r, bool rgb)
{
  VolRec v;
  v.c[0] = v.c[1] = v.c[2] = 0;
  if (rgb) { v.c[0] = r[0]; v.c[1] = r[1]; v.c[2] = r[2]; r += 3; }
  float cx, cy, cz, size;
  vol_get (r, &v.d, 4); vol_get (r + 4, &v.w, 4);
  vol_get (r + 8, &cx, 4); vol_get (r + 12, &cy, 4); vol_get (r + 16, &cz, 4); vol_get (r + 20, &size, 4);
  vol_get (r + 24, &v.M, 4); vol_get (r + 28, &v.ns, 4);
  vol_get (r + 32, &v.nchild, 8);
  v.placed = false; v.level = -1; v.x = v.y = v.z = -1;
  if (v.nchild != 0 && v.nchild != 8) return v;
  const uint32_t sb = float_bits (size);
  for (int l = 0; l <= p.L; ++l)
    if (float_bits (level_size (p, l)) == sb) { v.level = l; break; }
  if (v.level < 0) return v;
  v.x = vol_index_of_center (p, v.level, cx); v.y = vol_index_of_center (p, v.level, cy); v.z = vol_index_of_center (p, v.level, cz);
  v.placed = v.x >= 0 && v.y >= 0 && v.z >= 0;
  return v;
}

// the node the walk visits after a leaf at (level, x, y, z): the next sibling of the nearest ancestor-or-self that is not a
// last child.  False for the last node of the tree.
B2_HD bool vol_successor (int& level, int& x, int& y, int& z)
{
  while (level > 0 && (x & 1) && (y & 1) && (z & 1)) { x >>= 1; y >>= 1; z >>= 1; --level; }
  if (level == 0) return false;
  const int c = (((x & 1) << 2) | ((y & 1) << 1) | (z & 1)) + 1;
  x = (x & ~1) | (c >> 2); y = (y & ~1) | ((c >> 1) & 1); z = (z & ~1) | (c & 1);
  return true;
}

// The checks of one record against the tree: the host loader's depth rules (a level above the coarse depth must have
// children, the finest level must not) and, given the previous record, that this is the node the walk visits next.  i == 0:
// the root.
B2_HD bool vol_record_fits (const Params& p, const VolRec& v, bool first, const VolRec& prev)
{
  if (!v.placed) return false;
  if (v.level < p.C && v.nchild != 8) return false;
  if (v.level == p.L && v.nchild) return false;
  if (first) return v.level == 0;
  if (!prev.placed) return false;
  int l = prev.level, x = prev.x, y = prev.y, z = prev.z;
  if (prev.nchild) { ++l; x *= 2; y *= 2; z *= 2; }
  else if (!vol_successor (l, x, y, z)) return false;
  return v.level == l && v.x == x && v.y == y && v.z == z;
}

// Every check of record i of a tree of n records (k_vol_check, one record per thread): false when it fails.  ood: the record
// is stored (level >= Rtop) with a {d, w} outside the fast route's domain (edit_in_fast_domain).
B2_HD bool vol_check_record (const Params& p, const unsigned char* body, size_t i, size_t n, int rbytes, bool rgb, bool& ood)
{
  ood = false;
  const VolRec v = vol_parse (p, body + i * rbytes, rgb);
  const VolRec prev = i ? vol_parse (p, body + (i - 1) * rbytes, rgb) : v;
  if (!vol_record_fits (p, v, i == 0, prev)) return false;
  if (i == n - 1)
  {
    int l = v.level, x = v.x, y = v.y, z = v.z;
    if (v.nchild || vol_successor (l, x, y, z)) return false;          // the last record closes the tree
  }
  ood = v.level >= p.Rtop && !edit_in_fast_domain (v.d, v.w);
  return true;
}

// Where a loaded record goes (VolLoader::node): above the root arrays nowhere; at Rtop the root-array entry `root`; below,
// node idx of brick (t, bx, by, bz).  A record with children sets split bit `mask` of word `word` (of the root bitset, or of
// the brick's split words) only at or below the coarse depth and above the finest level.
struct VolPlace { bool stored, root, set_split; int root_idx, t, bx, by, bz, idx; uint32_t word, mask; };
B2_HD VolPlace vol_place (const Params& p, int level, int x, int y, int z, bool children)
{
  VolPlace o = {};
  o.stored = level >= p.Rtop;
  if (!o.stored) return o;
  if (level == p.Rtop)
  {
    o.root = true;
    o.root_idx = root_index (p, x, y, z);
    o.set_split = children && level >= p.C;
    o.word = (uint32_t) (o.root_idx >> 5); o.mask = 1u << (o.root_idx & 31);
    return o;
  }
  o.t = tier_of_level (p, level);
  const int k = level - tier_root_level (p, o.t);
  o.bx = x >> k; o.by = y >> k; o.bz = z >> k;
  const int j = path_index (k, x, y, z);
  o.idx = node_offset (k) + j;
  o.set_split = children && level >= p.C && level < p.L;
  o.word = (uint32_t) (split_word_base (k) + (j >> 5)); o.mask = 1u << (j & 31);
  return o;
}

// One checked record stored into a volume that reset() left fresh, where vol_place puts it: the device parser's store
// (k_vol_place) and the host emulation's.  Bricks are claimed with find_or_insert_brick (pool exhaustion raises
// ERR_POOL_FULL, as k_load_bricks does) and split bits set with an atomic or, so records may be stored in any order.
B2_HD void vol_store (const Params& p, const VolRec& v)
{
  const VolPlace o = vol_place (p, v.level, v.x, v.y, v.z, v.nchild != 0);
  if (!o.stored) return;
  const uchar4 c = make_uchar4 (v.c[0], v.c[1], v.c[2], 0);
  if (o.root)
  {
    p.root_dw[o.root_idx] = make_float2 (v.d, v.w);
    if (p.root_rgb) p.root_rgb[o.root_idx] = c;
    if (p.root_M) { p.root_M[o.root_idx] = v.M; p.root_ns[o.root_idx] = v.ns; }
    if (o.set_split) atomic_or32 (&p.root_split[o.word], o.mask);
    return;
  }
  const int slot = find_or_insert_brick (p, o.t, o.bx, o.by, o.bz);
  if (slot < 0) return;
  const size_t k = (size_t) slot * BRICK_NODES + o.idx;
  p.nodes[k] = make_float2 (v.d, v.w);
  if (p.rgb) p.rgb[k] = c;
  if (p.M) { p.M[k] = v.M; p.ns[k] = v.ns; }
  if (o.set_split) atomic_or32 (&p.split[(size_t) slot * BRICK_SPLIT_WORDS + o.word], o.mask);
}

} // namespace b2
