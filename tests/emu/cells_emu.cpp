// tests/emu/cells_emu.cpp — HOST EMULATION of the engine's change epochs and cell-restricted marching cubes (DESIGN.md §3g).
// TEST HARNESS ONLY.
//
// Compiles the emulation of emu.cpp and adds, over an epoch state of its own (EmuEpochs, the handle's epoch, all_epoch and
// Params::cell_epoch in engine.cu):
//   cells_reset / cells_integrate / cells_edits: emu_reset, emu_integrate and the node writes with the engine's stamps: the
//     frame's cull loop stamps every cell it queues (k_front), the shared presplit_point stamps the cells where it sets a
//     new split bit, and the edit store stamps the cell of every node it writes (k_edit_store);
//   cells_changed: b200tsdf_changed_cells over the shared cell_changed;
//   cells_mesh: the k_mesh_bricks / k_mesh_roots walk restricted to McParams::cell_mask, with per-cell vertex counts.
#include "emu.cpp"

#include <vector>

struct EmuEpochs
{
  std::vector<unsigned long long> cell_epoch;
  unsigned long long epoch = 0, all_epoch = 0;
};

extern "C" {

EmuEpochs* cells_create () { return new EmuEpochs; }
void cells_destroy (EmuEpochs* s) { delete s; }

int cells_reset (Emu* e, EmuEpochs* s)
{
  if (int rc = emu_reset (e)) return rc;
  s->cell_epoch.assign ((size_t) 1 << (3 * e->p.C), 0ull);
  e->p.cell_epoch = s->cell_epoch.data ();
  s->all_epoch = ++s->epoch;                                       // reset changes the whole volume
  return 0;
}

// emu_integrate with the stamps of k_front
int cells_integrate (Emu* e, EmuEpochs* s, const void* points, size_t stride, int xyz_off, int rgba_off, int W, int H, const double* pose)
{
  const Params& p = e->p;
  Frame f;
  f.pts = (const unsigned char*) points; f.stride = (int) stride; f.xyz_off = xyz_off; f.rgba_off = p.color ? rgba_off : -1;
  f.width = W; f.height = H;
  double inv[12];
  b2host::affine_inverse (pose, inv);
  for (int i = 0; i < 12; ++i) { f.tinv[i] = (float) inv[i]; f.tfwd[i] = (float) pose[i]; }
  const unsigned long long epoch = ++s->epoch;
  for (int i = 0; i < W * H; ++i)                                  // k_front's pixel threads
  {
    const float* pt = frame_xyz (f, i % W, i / W);
    if (is_nan (pt[2])) continue;
    float pw[3];
    affine_mul_f (f.tfwd, pt[0], pt[1], pt[2], pw);
    int fx_, fy_, fz_;
    if (!world_to_finest (p, pw[0], pw[1], pw[2], fx_, fy_, fz_)) continue;
    const int sh = p.L - p.C;
    if (!owns_cell (p, fx_ >> sh, fy_ >> sh, fz_ >> sh)) continue;
    presplit_point (p, fx_, fy_, fz_, epoch);
  }
  float pl[6][4];
  b2host::frustum_planes (pose, p.width, p.height, p.fx, p.fy, p.min_sensor, p.max_sensor, pl);
  const int n = 1 << p.C;
  Counters cnt; cnt.n_updates = 0; cnt.n_visits = 0;
  e->n_culled = 0;
  for (int x = 0; x < n; ++x) for (int y = 0; y < n; ++y) for (int z = 0; z < n; ++z)   // k_front's cull threads, then the update
  {
    if (!frustum_contains (pl, center1d (p, p.C, x), center1d (p, p.C, y), center1d (p, p.C, z))) continue;
    if (!owns_cell (p, x, y, z)) continue;
    e->n_culled++;
    stamp_cell (p, (x * n + y) * n + z, epoch);
    NodePos nd;
    if (!locate_node (p, p.C, x, y, z, nd)) return -2;
    update_voxel_dfs (p, f, nd, cnt);
  }
  e->n_updates = cnt.n_updates; e->n_visits = cnt.n_visits;
  return e->err;
}

// the node writes of tests/emu/edits_emu.cpp with the stamps of k_edit_store: a batch that writes a node takes the next epoch
long long cells_edits (Emu* e, EmuEpochs* s, const float* xyz, long long n, float min_size, const float* d, const float* w, uint8_t* status)
{
  const Params& p = e->p;
  size_t slots = 1024;
  while (slots < 2 * (size_t) n) slots <<= 1;
  const uint32_t mask = (uint32_t) (slots - 1);
  std::vector<uint64_t> keys (slots, EDIT_EMPTY), addr (n);
  std::vector<int> last (slots, -1);
  std::vector<uint8_t> st (n);
  long long ood = 0;
  for (long long i = 0; i < n; ++i)
  {
    uint64_t a = 0;
    st[i] = (uint8_t) edit_resolve (p, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], min_size, d[i], w[i], a);
    if (st[i] != EDIT_WRITTEN) continue;
    addr[i] = a;
    edit_claim (keys.data (), last.data (), mask, a, (int) i);
    ood += !edit_in_fast_domain (d[i], w[i]);
  }
  bool wrote = false;
  for (long long i = 0; i < n; ++i)
    if (st[i] == EDIT_WRITTEN && edit_wins (keys.data (), last.data (), mask, addr[i], (int) i))
    {
      edit_store (p, addr[i], d[i], w[i]);
      stamp_cell (p, edit_cell (p, addr[i]), s->epoch + 1);
      wrote = true;
    }
  if (wrote) ++s->epoch;
  if (status) for (long long i = 0; i < n; ++i) status[i] = st[i];
  return ood;
}

// b200tsdf_changed_cells
unsigned long long cells_changed (const Emu* e, const EmuEpochs* s, unsigned long long since, uint8_t* mask)
{
  const int C = e->p.C;
  for (int i = 0; i < 1 << (3 * C); ++i)
    mask[i] = since == 0 || s->all_epoch > since || cell_changed (C, s->cell_epoch.data (), since, i);
  return s->epoch;
}

// emu_mesh restricted to the leaves of the cells with mask[c] != 0 (mask null: every cell); cell_nverts (8^C) receives the
// vertex count of each cell
long long cells_mesh (Emu* e, float w_min, int color_mode, const uint8_t* mask, const float** verts, const uint8_t** cols,
                      int64_t* cell_nverts)
{
  const Params& p = e->p;
  McParams mc;
  make_mc_params (e->cfg, p, w_min, color_mode, mc);
  mc.cell_mask = mask;
  std::fill (cell_nverts, cell_nverts + ((size_t) 1 << (3 * p.C)), (int64_t) 0);
  e->mesh_v.clear (); e->mesh_c.clear ();
  std::vector<std::pair<unsigned long long, size_t> > order;
  walk_nodes (p, [&] (const BrickNode& b, float2 dw, int slot, int i)
  {
    if (!b.exists || b.split || b.level < p.C || !mc_cell_selected (p, mc, b.level, b.x, b.y, b.z)) return;
    const NodePos q = brick_node_pos (p, b, slot, i);
    float v[45]; unsigned char cc[45];
    const int nt = mc_leaf (p, mc, q, dw.x, dw.y, mc_tables::edge_table, mc_tables::tri_table, v, color_mode ? cc : nullptr);
    cell_nverts[coarse_cell (p, b.level, b.x, b.y, b.z)] += 3 * nt;
    for (int k = 0; k < 9 * nt; ++k) { e->mesh_v.push_back (v[k]); if (color_mode) e->mesh_c.push_back (cc[k]); }
    for (int t = 0; t < nt; ++t) order.push_back ({ (mc_order_key (p, q) << 3) | (unsigned long long) t, order.size () });
  });
  std::sort (order.begin (), order.end ());
  std::vector<float> sv (e->mesh_v.size ()); std::vector<unsigned char> sc (e->mesh_c.size ());
  for (size_t t = 0; t < order.size (); ++t)
  {
    const size_t src = order[t].second;
    std::copy (e->mesh_v.begin () + 9 * src, e->mesh_v.begin () + 9 * src + 9, sv.begin () + 9 * t);
    if (color_mode) std::copy (e->mesh_c.begin () + 9 * src, e->mesh_c.begin () + 9 * src + 9, sc.begin () + 9 * t);
  }
  e->mesh_v.swap (sv); e->mesh_c.swap (sc);
  *verts = e->mesh_v.data ();
  *cols = color_mode ? e->mesh_c.data () : nullptr;
  return (long long) (e->mesh_v.size () / 3);
}

} // extern "C"
