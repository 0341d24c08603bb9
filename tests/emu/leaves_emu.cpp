// tests/emu/leaves_emu.cpp — HOST EMULATION of the engine's leaf enumeration (k_leaves_bricks / k_leaves_roots /
// k_leaves_level in engine.cu).  TEST HARNESS ONLY.
//
// Compiles the emulation of emu.cpp and adds emu_leaves: the kernels' walk of the flat layout (walk_nodes, shared with
// emu_mesh) through the same __host__ __device__ predicate and record (leaf_selected, leaf_record in tsdf_core.cuh), then
// a sort by order key in place of the radix sort.
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
  walk_nodes (p, [&] (const BrickNode& b, float2 dw, int, int)
  {
    if (!leaf_selected (b.level, b.exists, b.split, nlevels, occupied != 0, dw.x, dw.y)) return;
    LeafRec r; NodePos n; n.level = b.level; n.x = b.x; n.y = b.y; n.z = b.z;
    r.key = mc_order_key (p, n);
    leaf_record (p, b.level, b.x, b.y, b.z, occupied != 0, r.v);
    recs.push_back (r);
  });
  std::sort (recs.begin (), recs.end (), [] (const LeafRec& a, const LeafRec& b) { return a.key < b.key; });
  if (out)
    for (size_t i = 0; i < recs.size (); ++i) std::memcpy (out + 3 * i, recs[i].v, 12);
  return (long long) recs.size ();
}

} // extern "C"
