// tests/emu/leaves_emu.cpp — HOST EMULATION of the engine's leaf enumeration (k_leaves_bricks / k_leaves_roots /
// k_leaves_level in engine.cu).  TEST HARNESS ONLY.
//
// Compiles the emulation of emu.cpp and adds emu_leaves: the same traversal of the flat layout, one "warp" per claimed
// brick and one "thread" per root-array entry in plain loops, through the same __host__ __device__ predicate and record
// (leaf_selected, brick_node, leaf_record in tsdf_core.cuh), then a sort by order key in place of the radix sort.
#include "emu.cpp"

namespace {
struct LeafRec { unsigned long long key; uint32_t v[3]; };
}

extern "C" {

// getLeaves (nlevels) [occupied: getOccupiedVoxelIndices] -> number of records; out (3 x 32 bits per record) may be null
long long emu_leaves (Emu* e, int nlevels, int occupied, uint32_t* out)
{
  const Params& p = e->p;
  std::vector<LeafRec> recs;
  if (!occupied && nlevels >= 0 && (nlevels < p.C || nlevels == 0))
  {
    const unsigned long long count = 1ull << (3 * nlevels);
    if (out)
      for (unsigned long long i = 0; i < count; ++i)
      {
        int x, y, z;
        morton_decode (nlevels, i, x, y, z);
        leaf_record (p, nlevels, x, y, z, false, out + 3 * i);
      }
    return (long long) count;
  }
  for (size_t slot = 0; slot <= p.pool_mask; ++slot)
  {
    const uint64_t key = p.keys[slot];
    if (key == KEY_EMPTY) continue;
    const int t = (int) (key >> 60) - 1;
    const int bx = (int) ((key >> 40) & 0xFFFFF), by = (int) ((key >> 20) & 0xFFFFF), bz = (int) (key & 0xFFFFF);
    const int R = tier_root_level (p, t);
    if (nlevels >= 0 && R + 1 > nlevels) continue;
    bool root_split = true;
    if (R >= p.C)
    {
      NodePos r;
      root_split = locate_node (p, R, bx, by, bz, r) && is_split (p, r);
    }
    if (!root_split) continue;
    const uint32_t* sw = p.split + slot * BRICK_SPLIT_WORDS;
    for (int i = 0; i < BRICK_NODES; ++i)
    {
      const BrickNode b = brick_node (p, sw, R, bx, by, bz, true, i);
      const float2 dw = p.nodes[slot * BRICK_NODES + i];
      if (!leaf_selected (b.level, b.exists, b.split, nlevels, occupied != 0, dw.x, dw.y)) continue;
      LeafRec r; NodePos n; n.level = b.level; n.x = b.x; n.y = b.y; n.z = b.z;
      r.key = mc_order_key (p, n);
      leaf_record (p, b.level, b.x, b.y, b.z, occupied != 0, r.v);
      recs.push_back (r);
    }
  }
  const int nr = 1 << p.Rtop;
  for (int i = 0; i < nr * nr * nr; ++i)
  {
    const int z = i % nr, y = (i / nr) % nr, x = i / (nr * nr);
    const NodePos nd = make_root (p, x, y, z);
    const float2 dw = p.root_dw[nd.idx];
    if (!leaf_selected (p.Rtop, true, is_split (p, nd), nlevels, occupied != 0, dw.x, dw.y)) continue;
    LeafRec r;
    r.key = mc_order_key (p, nd);
    leaf_record (p, p.Rtop, x, y, z, occupied != 0, r.v);
    recs.push_back (r);
  }
  std::sort (recs.begin (), recs.end (), [] (const LeafRec& a, const LeafRec& b) { return a.key < b.key; });
  if (out)
    for (size_t i = 0; i < recs.size (); ++i) std::memcpy (out + 3 * i, recs[i].v, 12);
  return (long long) recs.size ();
}

} // extern "C"
