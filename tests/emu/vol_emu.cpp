// tests/emu/vol_emu.cpp — HOST EMULATION of the engine's .vol writer and parser (k_vol_roots / k_vol_bricks / k_vol_format
// and k_vol_slots / k_vol_check / k_vol_place in engine.cu).  TEST HARNESS ONLY.
//
// Compiles the emulation of emu.cpp and adds emu_vol_body, the writer's emission through the same __host__ __device__ routines
// (vol_key, vol_node, vol_has_children, vol_format in vol_io.cuh) with a sort by key in place of the radix sort, and
// emu_vol_parse, the parser's checks and placement (vol_check_record, vol_store) one record at a time.
#include "emu.cpp"
#include "../../cpu_tsdf_b200/csrc/vol_io.cuh"

namespace {
struct Keyed { unsigned long long key; VolNode v; };
}

extern "C" {

// the body bytes of the volume's .vol (vol_record_bytes per node) -> number of nodes; out may be null
long long emu_vol_body (Emu* e, unsigned char* out)
{
  const Params& p = e->p;
  std::vector<Keyed> recs;
  walk_nodes (p, [&] (const BrickNode& b, float2, int slot, int i)
  {
    if (!b.exists) return;
    NodePos n; n.level = b.level; n.x = b.x; n.y = b.y; n.z = b.z; n.slot = slot; n.idx = i;
    const bool children = slot < 0 ? vol_has_children (p, make_root (p, b.x, b.y, b.z)) : (b.split && children_slot (p, n, false) >= 0);
    const unsigned long long k = vol_key (p, b.level, b.x, b.y, b.z);
    recs.push_back ({ k, vol_node (k, slot, slot < 0 ? root_index (p, b.x, b.y, b.z) : i, children) });
    if (slot >= 0) return;
    for (int c = 1; c <= p.Rtop; ++c)                          // the geometry-only ancestors whose child-0 chain this is
    {
      const int m = (1 << c) - 1;
      if ((b.x & m) || (b.y & m) || (b.z & m)) break;
      const unsigned long long ka = vol_key (p, p.Rtop - c, b.x >> c, b.y >> c, b.z >> c);
      recs.push_back ({ ka, vol_node (ka, VOL_SLOT_GEOM, 0, true) });
    }
  });
  std::sort (recs.begin (), recs.end (), [] (const Keyed& a, const Keyed& b) { return a.key < b.key; });
  const int rb = vol_record_bytes (p.color != 0, p.color_norm != 0);
  if (out)
    for (size_t i = 0; i < recs.size (); ++i) vol_format (p, recs[i].v, out + i * rb);
  return (long long) recs.size ();
}

// The parser on a body of len bytes (rgb: 43-byte records, else 40) for the emulation's current grid: 1 and the records placed
// into the (freshly reset) volume when every check holds, 0 when one fails (nothing placed), with *n_out the records of the
// tree (or -1 when it does not close) and *ood_out the stored {d, w} outside the fast route's domain.
int emu_vol_parse (Emu* e, const unsigned char* body, size_t len, int rgb, long long* n_out, long long* ood_out)
{
  const Params& p = e->p;
  const int rb = vol_record_bytes (rgb != 0, false);
  const size_t nrec = len / rb;
  long long open = 1, n = -1;
  for (size_t i = 0; i < nrec && n < 0; ++i)
  {
    unsigned long long nchild;
    vol_get (body + i * rb + rb - 8, &nchild, 8);
    open += nchild == 8 ? 7 : -1;
    if (open == 0) n = (long long) i + 1;
  }
  *n_out = n; *ood_out = 0;
  if (n < 0) return 0;
  long long ood = 0;
  for (long long i = 0; i < n; ++i)
  {
    bool out;
    if (!vol_check_record (p, body, (size_t) i, (size_t) n, rb, rgb != 0, out)) return 0;
    ood += out;
  }
  *ood_out = ood;
  for (long long i = 0; i < n; ++i) vol_store (p, vol_parse (p, body + i * rb, rgb != 0));
  if (e->err & ERR_POOL_FULL) return -1;
  return 1;
}

} // extern "C"
