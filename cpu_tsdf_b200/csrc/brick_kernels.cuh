// brick_kernels.cuh — the fast integrate path: level-synchronous work queues above the finest
// tier and one warp per 8^3 voxel block at the finest tier.
//
// updateVoxel (impl/tsdf_volume_octree.hpp:113-218) is a depth-first recursion whose per-node
// decisions depend only on (a) the node's own stored state, (b) the frame, and (c) the return
// codes of its children.  That makes it separable into
//   1. a top-down sweep over levels C .. B-1 (B = L-3, the block-root level): one thread per
//      visited node decides "already split / split now by proximity / update as a leaf" and
//      appends its children to the next level's queue (k_upper_down);
//   2. one warp per visited block root sweeps the 1+8+64+512-node subtree top-down and bottom-up with warp
//      ballots, updating the brick in place (k_bricks, brick_direct.cuh);
//   3. a bottom-up sweep over levels B-1 .. C that folds the children's return codes, prunes
//      all-empty children and applies the fall-through leaf update (k_upper_up).
// Speculative splits are safe because storage of non-existent nodes is always fresh (see
// tsdf_core.cuh).  The one case that is not separable — a node whose pre-existing children are
// all pruned AND which then re-splits in the same call (SURVEY.md §A.14) — is an ordinary leaf visit of the
// flat layout once the prune has been written (leaf_visit_warp8 / update_voxel_dfs for that subtree only).
#pragma once
#include "tsdf_core.cuh"
#include "obs_fast.cuh"

namespace b2 {

struct QNode
{
  int x, y, z;        // integer coordinates at the queue's level
  int slot, idx;      // storage of the node's own state (slot < 0: root arrays)
  int kind;           // 0 = finished (rc valid), 1 = interior with pre-existing children, 2 = interior split this frame
  int child_base;     // index of the first of its 8 children in the next level's queue
  int rc;             // updateVoxel return code
};

// one frame's parameters as the hot kernels read them (device memory: a captured launch can be replayed on another frame)
struct FrameRec
{
  Frame f;
  float pl[6][4];          // frustum planes (host_math.h)
  int cset;                // which of the two per-frame counter sets this frame uses
  int timing;              // 1: the brick kernel stamps kt[] with %globaltimer (profiling; works inside a replayed graph)
  int pad_[2];
  unsigned long long kt[2];// [0] start of the brick kernel (ns), [1] end of its last block; zeroed by the record upload
};
// programmatic dependent launch: the hot kernels of a frame are launched with programmatic stream serialization, so the next
// kernel's blocks become resident while this one drains and only wait (pdl_wait) before they touch what it wrote
__device__ __forceinline__ void pdl_launch_dependents () { asm volatile ("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait () { asm volatile ("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ unsigned long long global_ns () { unsigned long long t; asm volatile ("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }

constexpr int MAX_QLEVELS = 8;
// Block roots are queued in BL_CLASSES lists by expected work (the number of interior level-2 nodes the brick had in the
// previous frame: its finest rounds), heaviest class first, so that the short bricks fill the tail of the brick kernel.
// Counter slots of a frame's set: class 0 = 9, classes 1.. = 12, 13, 14.
constexpr int BL_CLASSES = 4;
__host__ __device__ __forceinline__ int bl_count_slot (int c) { return c == 0 ? 9 : 11 + c; }
__device__ __forceinline__ int bl_class (int work) { return (work < 28) + (work < 16) + (work < 6); }
struct Queues
{
  QNode* q[MAX_QLEVELS];    // q[i] holds level C+i
  int cap[MAX_QLEVELS];
  int* n;                   // n[i] = entries in q[i]   (device memory)
};

enum { KIND_DONE = 0, KIND_OLD = 1, KIND_NEW = 2 };

__device__ __forceinline__ NodePos qnode_pos (const Params& p, int level, const QNode& e)
{
  NodePos n;
  n.level = level; n.x = e.x; n.y = e.y; n.z = e.z;
  n.cx = center1d (p, level, e.x); n.cy = center1d (p, level, e.y); n.cz = center1d (p, level, e.z);
  n.size = level_size (p, level);
  n.slot = e.slot; n.idx = e.idx;
  return n;
}

// Appends the 8 children of `n` to the next level's queue.  Called by every lane of the warp with
// `want` saying whether this lane pushes: one atomicAdd per warp reserves the whole range.
__device__ __forceinline__ bool push_children (const Params& p, const Queues& Q, int* qn, int li, bool want, const NodePos& n, int cs, QNode& e)
{
  const unsigned lane = threadIdx.x & 31;
  const unsigned mask = __ballot_sync (0xffffffffu, want);
  if (!mask) return false;
  int base = 0;
  const int leader = __ffs (mask) - 1;
  if ((int) lane == leader) base = atomicAdd (&qn[li + 1], 8 * __popc (mask));
  base = __shfl_sync (0xffffffffu, base, leader);
  if (!want) return false;
  base += 8 * __popc (mask & ((1u << lane) - 1));
  if (base + 8 > Q.cap[li + 1]) { raise_err (p, ERR_QUEUE_FULL); e.kind = KIND_DONE; e.rc = 0; return false; }
  e.child_base = base;
  for (int c = 0; c < 8; ++c)
  {
    NodePos ch = make_child (p, n, c, cs);
    QNode q; q.x = ch.x; q.y = ch.y; q.z = ch.z; q.slot = ch.slot; q.idx = ch.idx; q.kind = KIND_DONE; q.child_base = -1; q.rc = 0;
    Q.q[li + 1][base + c] = q;
  }
  return true;
}

__device__ __forceinline__ void warp_add_stats (unsigned long long* stats, unsigned long long upd, unsigned long long vis)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
  {
    upd += __shfl_down_sync (0xffffffffu, upd, o);
    vis += __shfl_down_sync (0xffffffffu, vis, o);
  }
  if ((threadIdx.x & 31) == 0)
  {
    if (upd) atomicAdd (&stats[0], upd);
    if (vis) atomicAdd (&stats[1], vis);
  }
}

// ---- 1. top-down over the upper levels: one thread per queued node ---------------------------------
// `block_level`: the queue holds block roots (level L-3); interior ones go to the block list with their
// brick slot instead of having their children queued.
// The frame comes from its record in device memory and the counters from the record's counter set (Q.n = the base of all
// sets), so that the launch can be captured into a graph and replayed like the other kernels of a frame.
#define B2_UPPER_FRAME(fr)                                                                   \
  __shared__ Frame s_uf_;                                                                    \
  {                                                                                          \
    const int* src_ = reinterpret_cast<const int*> (&(fr)->f);                               \
    int* dst_ = reinterpret_cast<int*> (&s_uf_);                                             \
    for (int w_ = threadIdx.x; w_ < (int) (sizeof (Frame) / sizeof (int)); w_ += blockDim.x) dst_[w_] = src_[w_]; \
  }                                                                                          \
  __syncthreads ();                                                                          \
  const Frame& f = s_uf_;                                                                    \
  int* const qn = Q.n + 16 * (fr)->cset;

__global__ void k_upper_down (Params p, const FrameRec* __restrict__ fr, Queues Q, int li, int block_level, int* __restrict__ blist,
                              unsigned long long* __restrict__ stats)
{
  B2_UPPER_FRAME (fr)
  int* const bcount = qn + 9;
  int level = p.C + li;
  int count = qn[li];
  if (count > Q.cap[li]) count = Q.cap[li];
  unsigned long long upd = 0, vis = 0;
  const int stride = gridDim.x * blockDim.x;
  const int rounds = (count + stride - 1) / stride;                 // warp-uniform trip count (the pushes use warp collectives)
  for (int r = 0; r < rounds; ++r)
  {
    const int i = r * stride + blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = i < count;
    QNode e; NodePos n; int cs = -1;
    bool push = false, to_blocks = false;
    e.kind = KIND_DONE; e.rc = 0; e.child_base = -1;
    if (active)
    {
      e = Q.q[li][i];
      n = qnode_pos (p, level, e);
      vis++;
      uint32_t m; uint32_t* sw = split_word (p, n, m);
      if (*sw & m)                                                    // hpp:122
      {
        cs = children_slot (p, n, false);
        if (cs < 0) { raise_err (p, ERR_MISSING_BRICK); e.kind = KIND_DONE; e.rc = 0; }
        else { e.kind = KIND_OLD; push = !block_level; to_blocks = block_level; }
      }
      else
      {
        Obs o = observe (p, f, n.cx, n.cy, n.cz, n.size);
        if (!o.valid) { e.kind = KIND_DONE; e.rc = 0; }
        else if (o.near_ && n.size > p.finest_size)                    // hpp:161-166
        {
          cs = children_slot (p, n, true);
          if (cs < 0) { e.kind = KIND_DONE; e.rc = 0; }
          else
          {
            e.kind = KIND_NEW; push = !block_level; to_blocks = block_level;
            atomicOr (sw, m);                                          // split (): children are fresh by invariant
          }
        }
        else
        {
          bool updated;
          e.rc = leaf_update (p, f, n, o, updated);
          e.kind = KIND_DONE;
          upd += updated;
        }
      }
    }
    if (!block_level) push_children (p, Q, qn, li, push, n, cs, e);
    else
    {
      // interior block roots go to the block list (one atomic per warp)
      const unsigned lane = threadIdx.x & 31;
      const unsigned mask = __ballot_sync (0xffffffffu, to_blocks);
      if (mask)
      {
        int base = 0;
        const int leader = __ffs (mask) - 1;
        if ((int) lane == leader) base = atomicAdd (bcount, __popc (mask));
        base = __shfl_sync (0xffffffffu, base, leader);
        if (to_blocks) { e.child_base = cs; blist[base + __popc (mask & ((1u << lane) - 1))] = i; }
      }
    }
    if (active) Q.q[li][i] = e;
  }
  warp_add_stats (stats, upd, vis);
}

// ---- 3. bottom-up over the upper levels -------------------------------------------------------------
__global__ void k_upper_up (Params p, const FrameRec* __restrict__ fr, Queues Q, int li, unsigned long long* __restrict__ stats)
{
  B2_UPPER_FRAME (fr)
  int level = p.C + li;
  int count = qn[li];
  if (count > Q.cap[li]) count = Q.cap[li];
  unsigned long long upd = 0, vis = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x)
  {
    QNode e = Q.q[li][i];
    if (e.kind == KIND_DONE) continue;
    const QNode* ch = Q.q[li + 1] + e.child_base;
    bool all_empty = true;
    for (int c = 0; c < 8; ++c) all_empty &= (ch[c].rc < 0);
    if (!all_empty) { e.rc = 1; }                                   // hpp:140 / :185
    else
    {
      NodePos n = qnode_pos (p, level, e);
      uint32_t m; uint32_t* sw = split_word (p, n, m);
      atomicAnd (sw, ~m);                                           // children.clear ()
      int cs = children_slot (p, n, false);
      if (cs >= 0) for (int c = 0; c < 8; ++c) reset_node (p, make_child (p, n, c, cs));
      if (e.kind == KIND_NEW)
      {
        Obs o = observe (p, f, n.cx, n.cy, n.cz, n.size);           // same observation as in the down sweep
        bool updated;
        e.rc = leaf_update (p, f, n, o, updated);                   // hpp:189-214 (falls through after :181)
        upd += updated;
      }
      else
      {
        // pre-existing children pruned: the node is visited as a leaf and may re-split (hpp:136 -> :161)
        Counters cnt; cnt.n_updates = 0; cnt.n_visits = 0;
        e.rc = update_voxel_dfs (p, f, n, cnt);
        upd += cnt.n_updates; vis += cnt.n_visits - 1;
      }
    }
    e.kind = KIND_DONE;
    Q.q[li][i].rc = e.rc;
  }
  __syncwarp ();
  warp_add_stats (stats, upd, vis);
}

// ---- helpers of the bottom-up sweeps ---------------------------------------------------------------------------
// fold the children's return codes into an interior node (hpp:131-142 / :176-188 + fall-through)
__device__ __noinline__ int upper_fold_slow (const Params& p, const Frame& f, const NodePos& n, unsigned long long& upd, unsigned long long& vis)
{
  Counters cnt; cnt.n_updates = 0; cnt.n_visits = 0;
  int rc = update_voxel_dfs (p, f, n, cnt);
  upd += cnt.n_updates; vis += cnt.n_visits - 1;
  if (p.diag) { atomicAdd (&p.diag[0], 1ull); atomicAdd (&p.diag[1], (unsigned long long) cnt.n_visits); }
  return rc;
}
// leaf visit (hpp:143-218) of a node whose pre-existing children were just pruned, by one WARP: if the node
// re-splits, its eight fresh children are visited by lanes 0..7 in parallel (their subtrees are disjoint).
// All 32 lanes must call it with the same node.  Returns the node's return code in every lane.
__device__ __noinline__ int leaf_visit_warp8 (const Params& p, const Frame& f, const NodePos& n, unsigned long long& upd, unsigned long long& vis)
{
  const int lane = threadIdx.x & 31;
  Obs o = observe (p, f, n.cx, n.cy, n.cz, n.size);
  if (!o.valid) return 0;
  Counters cnt; cnt.n_updates = 0; cnt.n_visits = 0;
  if (o.near_ && n.size > p.finest_size)
  {
    uint32_t m; uint32_t* sw = split_word (p, n, m);
    int cs = -1;
    if (lane == 0) cs = children_slot (p, n, true);
    cs = __shfl_sync (0xffffffffu, cs, 0);
    if (cs >= 0)
    {
      if (lane == 0) atomicOr (sw, m);
      __syncwarp ();
      int rc = -1;
      NodePos ch;
      if (lane < 8)
      {
        ch = make_child (p, n, lane, cs);
        Obs oc = observe (p, f, ch.cx, ch.cy, ch.cz, ch.size);
        rc = visit_fresh_leaf (p, f, ch, oc, cnt);
      }
      const unsigned nonneg = __ballot_sync (0xffffffffu, lane < 8 && rc >= 0);
      upd += cnt.n_updates; vis += cnt.n_visits;
      if (nonneg) return 1;
      if (lane == 0) atomicAnd (sw, ~m);
      if (lane < 8) reset_node (p, ch);
      __syncwarp ();
    }
  }
  int rc = 0;
  if (lane == 0) { bool updated; rc = leaf_update (p, f, n, o, updated); upd += updated; }
  return __shfl_sync (0xffffffffu, rc, 0);
}

// The leaf visit of a COARSE node by the whole warp with the breadth-first routine (tsdf_core.cuh, fresh_children_bfs):
// a re-split coarse cell drags a subtree of a few dozen fresh nodes over three or four levels behind it, which the
// eight-lane version above walks depth first, one lane per child (~40 us, the straggler of k_celltop_up).  rec/counter:
// this warp's FRESH_RECS records and one int in shared memory.
constexpr int FRESH_RECS = 128;
struct CoopWarp
{
  __device__ __forceinline__ int lane () const { return threadIdx.x & 31; }
  __device__ __forceinline__ int nlanes () const { return 32; }
  __device__ __forceinline__ void sync () const { __syncwarp (); }
};
__device__ __noinline__ int leaf_visit_warp_bfs (const Params& p, const Frame& f, const NodePos& n, FreshRec* rec, int* counter,
                                                 unsigned long long& upd, unsigned long long& vis)
{
  const int lane = threadIdx.x & 31;
  Obs o = observe (p, f, n.cx, n.cy, n.cz, n.size);
  if (!o.valid) return 0;
  if (o.near_ && n.size > p.finest_size)
  {
    uint32_t m; uint32_t* sw = split_word (p, n, m);
    int cs = -1;
    if (lane == 0) cs = children_slot (p, n, true);
    cs = __shfl_sync (0xffffffffu, cs, 0);
    if (cs >= 0)
    {
      if (lane == 0) atomicOr (sw, m);
      __syncwarp ();
      Counters cnt; cnt.n_updates = 0; cnt.n_visits = 0;
      const bool stays = fresh_children_bfs (p, f, n, cs, rec, FRESH_RECS, counter, CoopWarp (), cnt);
      upd += cnt.n_updates; vis += cnt.n_visits;
      if (stays) return 1;
      if (lane == 0) atomicAnd (sw, ~m);
      if (lane < 8) reset_node (p, rec[lane].n);
      __syncwarp ();
    }
  }
  int rc = 0;
  if (lane == 0) { bool updated; rc = leaf_update (p, f, n, o, updated); upd += updated; }
  return __shfl_sync (0xffffffffu, rc, 0);
}

// The same leaf visit for up to FOUR nodes at once: the warp is split into four groups of eight lanes, group g
// (lanes 8g..8g+7) visits node `n` (identical in the eight lanes of a group) when `active`; lane 8g+c handles child c
// of a re-split.  All 32 lanes must call it.  Returns the group's node's return code in each of its lanes.
// (A pruned-then-resplit node costs five or six dependent memory round trips; a cell that has many of them in one
// frame used to serialise them and made its warp the straggler of k_celltop_up.)
__device__ __noinline__ int leaf_visit_groups (const Params& p, const Frame& f, const NodePos& n, bool active,
                                               unsigned long long& upd, unsigned long long& vis)
{
  const int lane = threadIdx.x & 31, sub = lane & 7, g = lane >> 3;
  const unsigned gmask = 0xFFu << (8 * g);
  Obs o; o.valid = false; o.near_ = false; o.u = o.v = 0; o.d_new = 0.f;
  if (active) o = observe (p, f, n.cx, n.cy, n.cz, n.size);
  const bool live = active && o.valid;                                  // !valid: return 0 without touching the node
  const bool want_split = live && o.near_ && n.size > p.finest_size;
  uint32_t m = 0; uint32_t* sw = nullptr;
  int cs = -1;
  if (want_split) { sw = split_word (p, n, m); if (sub == 0) cs = children_slot (p, n, true); }
  cs = __shfl_sync (0xffffffffu, cs, 8 * g);
  const bool split = want_split && cs >= 0;
  if (split && sub == 0) atomicOr (sw, m);
  __syncwarp ();
  Counters cnt; cnt.n_updates = 0; cnt.n_visits = 0;
  int crc = -1;
  NodePos ch = n;
  if (split)
  {
    ch = make_child (p, n, sub, cs);
    Obs oc = observe (p, f, ch.cx, ch.cy, ch.cz, ch.size);
    crc = visit_fresh_leaf (p, f, ch, oc, cnt);
  }
  const unsigned nonneg = __ballot_sync (0xffffffffu, split && crc >= 0) & gmask;
  upd += cnt.n_updates; vis += cnt.n_visits;
  if (split && !nonneg)                                                 // children.clear () again
  {
    if (sub == 0) atomicAnd (sw, ~m);
    reset_node (p, ch);
  }
  __syncwarp ();
  int rc = 0;
  if (split && nonneg) rc = 1;
  else if (live && sub == 0) { bool updated; rc = leaf_update (p, f, n, o, updated); upd += updated; }
  return __shfl_sync (0xffffffffu, rc, 8 * g);
}
// drives leaf_visit_groups over the lanes flagged in `slow` (each holding its node in `n`), four per round; a flagged
// lane gets its node's return code in `rc`
__device__ __forceinline__ void leaf_visit_slow_lanes (const Params& p, const Frame& f, bool slow, const NodePos& n, int t1, int& rc,
                                                       unsigned long long& upd, unsigned long long& vis)
{
  const int lane = threadIdx.x & 31, g = lane >> 3;
  uint32_t sm = __ballot_sync (0xffffffffu, slow);
  while (sm)
  {
    int srcs[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { srcs[k] = sm ? __ffs (sm) - 1 : -1; if (sm) sm &= sm - 1; }
    int src = srcs[0]; if (g == 1) src = srcs[1]; if (g == 2) src = srcs[2]; if (g == 3) src = srcs[3];
    const int from = src >= 0 ? src : 0;
    NodePos q;
    q.level = __shfl_sync (0xffffffffu, n.level, from); q.x = __shfl_sync (0xffffffffu, n.x, from); q.y = __shfl_sync (0xffffffffu, n.y, from); q.z = __shfl_sync (0xffffffffu, n.z, from);
    q.cx = __shfl_sync (0xffffffffu, n.cx, from); q.cy = __shfl_sync (0xffffffffu, n.cy, from); q.cz = __shfl_sync (0xffffffffu, n.cz, from);
    q.size = __shfl_sync (0xffffffffu, n.size, from); q.slot = t1; q.idx = __shfl_sync (0xffffffffu, n.idx, from);
    __threadfence_block ();
    const int r = leaf_visit_groups (p, f, q, src >= 0, upd, vis);
#pragma unroll
    for (int k = 0; k < 4; ++k) { const int rk = __shfl_sync (0xffffffffu, r, 8 * k); if (lane == srcs[k]) rc = rk; }
  }
}

// ---- 2. one warp per interior block root: k_bricks, brick_direct.cuh ------------------------------------------------------
__device__ __forceinline__ void path_center (const float* c0, float off, int k, int j, float* c)
{
  // centre of the level-k node with hierarchical index j below a root centred at c0 (octree.cpp:251-264)
  float x = c0[0], y = c0[1], z = c0[2];
  for (int l = k - 1; l >= 0; --l)
  {
    int cc = (j >> (3 * l)) & 7;
    x = (cc & 4) ? fadd (x, off) : fsub (x, off);
    y = (cc & 2) ? fadd (y, off) : fsub (y, off);
    z = (cc & 1) ? fadd (z, off) : fsub (z, off);
    off *= 0.5f;
  }
  c[0] = x; c[1] = y; c[2] = z;
}

// ---- 1c/3c. upper sweeps for the common shape: coarse cell == root of a tier-1 brick, block roots 3 levels below ----
// k_celltop_down: one CTA per culled coarse cell.  All 585 nodes of the cell's upper pyramid (cell + 8 + 64 + 512
// block roots) are OBSERVED SPECULATIVELY in parallel (observation is a pure function of geometry and frame) while
// the tier-1 brick is staged into shared memory, so the level-by-level decisions run from shared memory instead
// of a chain of dependent DRAM loads.  Interior block roots are queued for k_bricks.
// k_celltop_up: one WARP per cell folds the return codes with ballots (the bottom-up half of the block sweep, operating on
// the brick in global memory: only pruned nodes are touched).
constexpr int TOP_THREADS = 256;
constexpr int TOP_NODES = 585;                       // flat index f: 0 = cell, 1..8, 9..72, 73..584
struct CellTop                                       // per-cell scratch between the two sweeps
{
  int t1slot, nblk;
  unsigned char kind[592];
  signed char rc[592];
  float dnew[73];
  int uv[73];
};
struct TopSmem
{
  float2 dw[BRICK_NODES];
  uchar4 rgb[BRICK_NODES];
  float o_dnew[TOP_NODES];
  int o_uv[TOP_NODES];
  uint32_t o_bgra[TOP_NODES];
  unsigned char o_flags[592];                        // bit0 valid, bit1 near
  unsigned char kind[592];
  signed char rc[592];
  unsigned char dirty[592];
  uint32_t split[BRICK_SPLIT_WORDS];
  uint32_t split_old[BRICK_SPLIT_WORDS];
  QNode cell;
  int t1slot, root_interior;
  float c0[3];
};

__device__ __forceinline__ void top_kj (int f, int& k, int& j)
{ if (f == 0) { k = 0; j = 0; } else if (f < 9) { k = 1; j = f - 1; } else if (f < 73) { k = 2; j = f - 9; } else { k = 3; j = f - 73; } }

// The "cell" of these two kernels is a SUPERCELL: the root of a tier-1 brick, at level SL = L - 6 (its block roots are the 512
// level-3 nodes of that brick).  Three grid shapes:
//   C == SL (2048^3 / 10 m, 512^3 / 3 m): the supercells are the culled coarse cells (qslot 0);
//   C <  SL (4096^3 / 10 m, 1024^3 / 3 m): the coarse levels C .. SL-1 are swept by k_upper_down / k_upper_up and the supercells
//           are the interior nodes they queued at level SL (qslot SL - C);
//   C >  SL (256^3 / 3 m, 128^3 / 3 m, ...): the coarse cells lie INSIDE the brick, at relative level C - SL.  Every tier-1 root
//           is a supercell (static list, qslot < 0); the levels above C are virtual — they exist by Octree::init
//           (octree.cpp:584-599), carry no state, are never observed, updated or pruned — and a node of level C is visited
//           only when it passes the frustum cull and belongs to this shard (cpp:619-652), exactly like a queued coarse cell.
template <bool COLOR>
__global__ void __launch_bounds__ (TOP_THREADS) k_celltop_down (Params p, const FrameRec* __restrict__ fr, QNode* __restrict__ cells, int* __restrict__ d_count,
                                                               QNode* __restrict__ gq, CellTop* __restrict__ tops, int cell_cap,
                                                               int* __restrict__ blist, int bl_stride, unsigned long long* __restrict__ stats,
                                                               int SL, int qslot, int static_count)
{
  __shared__ __align__ (16) TopSmem S;
  __shared__ Frame s_f_;
  __shared__ float s_pl_[6][4];
  const int tid = threadIdx.x, lane = tid & 31;
  pdl_launch_dependents ();
  {
    const int* src_ = reinterpret_cast<const int*> (&fr->f); int* dst_ = reinterpret_cast<int*> (&s_f_);
    for (int w_ = tid; w_ < (int) (sizeof (Frame) / sizeof (int)); w_ += TOP_THREADS) dst_[w_] = src_[w_];
    if (tid < 24) s_pl_[tid >> 2][tid & 3] = fr->pl[tid >> 2][tid & 3];
  }
  int* const cnt_ = d_count + 16 * fr->cset;
  __syncthreads ();
  pdl_wait ();                                          // everything below reads what the previous kernel wrote
  const Frame& f = s_f_;
  unsigned long long upd = 0, vis = 0;
  int count = qslot >= 0 ? cnt_[qslot] : static_count;
  if (count > cell_cap) { if (tid == 0 && blockIdx.x == 0) raise_err (p, ERR_QUEUE_FULL); count = cell_cap; }
  const int cell_lvl = p.C - SL;                        // relative level of the coarse cells (<= 0: the supercell is at or below the coarse depth)
  const float sizeC = level_size (p, SL);
  const float off1 = sizeC * 0.25f;
  const double thr[4] = { near_threshold (sizeC), near_threshold (sizeC * 0.5f), near_threshold (sizeC * 0.25f), near_threshold (sizeC * 0.125f) };
  const float thrf[4] = { float_at_least (thr[0]), float_at_least (thr[1]), float_at_least (thr[2]), float_at_least (thr[3]) };
  const bool have_bgra = COLOR && p.color && f.rgba_off >= 0;
  FrameHot F; F.pix = p.pix;
  for (int ci = blockIdx.x; ci < count; ci += gridDim.x)
  {
    __syncthreads ();
    if (tid == 0)
    {
      S.cell = cells[ci];
      S.c0[0] = center1d (p, SL, S.cell.x); S.c0[1] = center1d (p, SL, S.cell.y); S.c0[2] = center1d (p, SL, S.cell.z);
    }
    __syncthreads ();
    const QNode cell = S.cell;
    const float c0[3] = { S.c0[0], S.c0[1], S.c0[2] };
    // ---- speculative observation of every node (independent loads, issued before anything else is waited on) ----
    for (int n = tid; n < TOP_NODES; n += TOP_THREADS)
    {
      int k, j; top_kj (n, k, j);
      float c[3];
      if (k == 0) { c[0] = c0[0]; c[1] = c0[1]; c[2] = c0[2]; } else path_center (c0, off1, k, j, c);
      float vg[3];
      pcl_transform_point_f (f.tinv, c[0], c[1], c[2], vg);                           // hpp:145
      const ObsF o = observe_fast<COLOR> (p, F, vg[0], vg[1], vg[2]);
      S.o_dnew[n] = o.d_new; S.o_uv[n] = o.uv;
      S.o_bgra[n] = (have_bgra && o.valid) ? o.bgra : 0u;
      S.o_flags[n] = (unsigned char) ((o.valid ? 1 : 0) | ((o.valid && fabsf (o.d_new) < thrf[k]) ? 2 : 0));
      S.kind[n] = KIND_DONE; S.rc[n] = 0; S.dirty[n] = 0;
    }
    // ---- the supercell itself (its state lives in the root arrays or in the tier above; none when it is virtual) ----
    if (tid == 0)
    {
      int kind = KIND_DONE, rc = 0, slot = -1;
      if (cell_lvl > 0)
      {
        kind = KIND_OLD;                                               // above the coarse depth: always split, no state
        slot = find_brick (p, 1, cell.x, cell.y, cell.z);
        if (slot < 0) { raise_err (p, ERR_MISSING_BRICK); kind = KIND_DONE; }
      }
      else
      {
        NodePos nc; nc.level = SL; nc.x = cell.x; nc.y = cell.y; nc.z = cell.z; nc.cx = c0[0]; nc.cy = c0[1]; nc.cz = c0[2]; nc.size = sizeC; nc.slot = cell.slot; nc.idx = cell.idx;
        uint32_t m; uint32_t* sw = split_word (p, nc, m);
        vis++;
        if (*sw & m) { kind = KIND_OLD; slot = find_brick (p, 1, cell.x, cell.y, cell.z); if (slot < 0) { raise_err (p, ERR_MISSING_BRICK); kind = KIND_DONE; } }
        else
        {
          Obs o = observe_thr (p, f, c0[0], c0[1], c0[2], thr[0]);
          if (o.valid)
          {
            if (o.near_) { slot = find_or_insert_brick (p, 1, cell.x, cell.y, cell.z); if (slot >= 0) { kind = KIND_NEW; atomicOr (sw, m); } }
            else { bool u_; rc = leaf_update (p, f, nc, o, u_); upd += u_; }
          }
        }
        if (kind == KIND_DONE) cells[ci].rc = rc;                      // (read by k_upper_up when coarse levels lie above the supercell)
      }
      S.root_interior = kind; S.t1slot = slot;
      S.kind[0] = (unsigned char) kind; S.rc[0] = (signed char) rc;     // (written after the init loop of this thread: n = 0 is tid 0's)
    }
    __syncthreads ();
    const int t1 = S.t1slot;
    CellTop* top = tops + ci;
    if (S.root_interior == KIND_DONE)
    {
      if (tid == 0) { top->t1slot = -1; top->nblk = 0; top->kind[0] = KIND_DONE; top->rc[0] = S.rc[0]; }
      continue;
    }
    // ---- stage the tier-1 brick ----
    float2* gdw = p.nodes + (size_t) t1 * BRICK_NODES;
    uchar4* grgb = COLOR ? p.rgb + (size_t) t1 * BRICK_NODES : nullptr;
    uint32_t* gsw = p.split + (size_t) t1 * BRICK_SPLIT_WORDS;
    {
      const float4* g4 = reinterpret_cast<const float4*> (gdw);
      float4* s4 = reinterpret_cast<float4*> (S.dw);
      for (int i = tid; i < BRICK_NODES / 2; i += TOP_THREADS) s4[i] = g4[i];
      if (COLOR)
      {
        const uint4* gc = reinterpret_cast<const uint4*> (grgb);
        uint4* sc = reinterpret_cast<uint4*> (S.rgb);
        for (int i = tid; i < BRICK_NODES / 4; i += TOP_THREADS) sc[i] = gc[i];
      }
      if (tid < BRICK_SPLIT_WORDS) { uint32_t w = gsw[tid]; S.split[tid] = w; S.split_old[tid] = w; }
    }
    __syncthreads ();
    // ---- level by level from shared memory ----
    for (int k = 1; k <= 3; ++k)
    {
      const int nlev = 1 << (3 * k), base = (k == 1) ? 1 : (k == 2 ? 9 : 73), pbase = (k == 1) ? 0 : (k == 2 ? 1 : 9);
      for (int j = tid; j < nlev; j += TOP_THREADS)
      {
        const int n = base + j;
        if (S.kind[pbase + (j >> 3)] == KIND_DONE) continue;          // parent is not interior: node not visited
        if (k < cell_lvl) { S.kind[n] = KIND_OLD; continue; }          // above the coarse depth: virtual
        if (k == cell_lvl)
        {
          // a coarse cell: visited only when its centre passes the frustum cull and this shard owns it (cpp:619-652)
          float c[3]; path_center (c0, off1, k, j, c);
          int lx = 0, ly = 0, lz = 0;
          for (int q = k - 1; q >= 0; --q) { const int cc = (j >> (3 * q)) & 7; lx = (lx << 1) | (cc >> 2); ly = (ly << 1) | ((cc >> 1) & 1); lz = (lz << 1) | (cc & 1); }
          if (!frustum_contains (s_pl_, c[0], c[1], c[2]) || !owns_cell (p, (cell.x << k) | lx, (cell.y << k) | ly, (cell.z << k) | lz)) continue;
        }
        vis++;
        const bool sold = (S.split_old[split_word_base (k) + (j >> 5)] >> (j & 31)) & 1;
        int kind = KIND_DONE, rc = 0;
        if (sold) kind = KIND_OLD;
        else if (S.o_flags[n] & 1)
        {
          if (S.o_flags[n] & 2) { kind = KIND_NEW; atomicOr (&S.split[split_word_base (k) + (j >> 5)], 1u << (j & 31)); }
          else
          {
            const int si = n - 1;                                  // in-brick node index
            float M = 0.f; int ns = 0; bool u_;
            const bool have = COLOR && f.rgba_off >= 0;
            rc = leaf_update_core (p, S.o_dnew[n], have, S.o_bgra[n], S.dw[si], S.rgb[si], M, ns, u_);
            if (u_) { S.dirty[n] = 1; upd++; }
          }
        }
        S.kind[n] = (unsigned char) kind; S.rc[n] = (signed char) rc;
      }
      __syncthreads ();
    }
    // ---- interior block roots -> block list (+ their QNode for k_bricks) ----
    constexpr int STRIDE = 585;
    for (int base = 0; base < 512; base += TOP_THREADS)
    {
      const int j3 = base + tid, n = 73 + j3;
      const int kind = S.kind[n];
      const bool interior = kind != KIND_DONE;
      int bslot = -1;
      if (interior)
      {
        int lx = 0, ly = 0, lz = 0;
        for (int q = 2; q >= 0; --q) { int c = (j3 >> (3 * q)) & 7; lx = (lx << 1) | (c >> 2); ly = (ly << 1) | ((c >> 1) & 1); lz = (lz << 1) | (c & 1); }
        const int X = (cell.x << 3) | lx, Y = (cell.y << 3) | ly, Z = (cell.z << 3) | lz;
        bslot = (kind == KIND_OLD) ? find_brick (p, 0, X, Y, Z) : find_or_insert_brick (p, 0, X, Y, Z);
        if (bslot < 0) { if (kind == KIND_OLD) raise_err (p, ERR_MISSING_BRICK); }
        QNode e; e.x = X; e.y = Y; e.z = Z; e.slot = t1; e.idx = 72 + j3; e.kind = kind; e.child_base = bslot; e.rc = 0;
        gq[(size_t) ci * STRIDE + 73 + j3] = e;
      }
      const bool push = interior && bslot >= 0;
      const int cls = push ? bl_class (p.work[bslot]) : -1;
#pragma unroll
      for (int c = 0; c < BL_CLASSES; ++c)
      {
        const unsigned mask = __ballot_sync (0xffffffffu, cls == c);
        if (mask)
        {
          int b = 0;
          const int leader = __ffs (mask) - 1;
          if (lane == leader) b = atomicAdd (cnt_ + bl_count_slot (c), __popc (mask));
          b = __shfl_sync (0xffffffffu, b, leader);
          if (cls == c) blist[(size_t) c * bl_stride + b + __popc (mask & ((1u << lane) - 1))] = ci * STRIDE + 73 + j3;
        }
      }
    }
    // ---- write back what changed, and the scratch for the bottom-up sweep ----
    for (int n = 1 + tid; n < TOP_NODES; n += TOP_THREADS)
      if (S.dirty[n]) { gdw[n - 1] = S.dw[n - 1]; if (COLOR) grgb[n - 1] = S.rgb[n - 1]; }
    if (tid < BRICK_SPLIT_WORDS && S.split[tid] != S.split_old[tid]) gsw[tid] = S.split[tid];
    for (int n = tid; n < 592; n += TOP_THREADS) { top->kind[n] = n < TOP_NODES ? S.kind[n] : 0; top->rc[n] = n < TOP_NODES ? S.rc[n] : 0; }
    for (int n = tid; n < 73; n += TOP_THREADS) { top->dnew[n] = S.o_dnew[n]; top->uv[n] = S.o_uv[n]; }
    if (tid == 0) { top->t1slot = t1; top->nblk = 0; }
  }
  __syncwarp ();
  warp_add_stats (stats, upd, vis);
}

// fall-through update (hpp:189-214) of an upper node whose children were all pruned; state in GLOBAL memory
__device__ __forceinline__ int top_fallthrough_new (const Params& p, const Frame& f, const NodePos& n, float dnew, int uv, unsigned long long& upd)
{
  Obs o; o.valid = true; o.near_ = true; o.d_new = dnew; o.u = uv & 0xFFFF; o.v = uv >> 16;
  bool u_; int rc = leaf_update (p, f, n, o, u_); upd += u_;
  return rc;
}

template <bool COLOR>
__global__ void __launch_bounds__ (128) k_celltop_up (Params gp, const FrameRec* __restrict__ fr, QNode* __restrict__ cells, const int* __restrict__ d_count,
                                                      const QNode* __restrict__ gq, const CellTop* __restrict__ tops, int cell_cap,
                                                      unsigned long long* __restrict__ stats, int SL, int qslot, int static_count)
{
  // Params / Frame live in shared memory here: the out-of-line slow path takes them by reference, which
  // would otherwise make every thread copy the kernel parameters to its stack in the prologue
  __shared__ Params sp_;
  __shared__ Frame sf_;
  __shared__ FreshRec s_rec[4][FRESH_RECS];          // per-warp records of the breadth-first re-split visit
  __shared__ int s_cnt[4];
  pdl_launch_dependents ();
  {
    const int* s1 = reinterpret_cast<const int*> (&gp); int* d1 = reinterpret_cast<int*> (&sp_);
    for (int w = threadIdx.x; w < (int) (sizeof (Params) / sizeof (int)); w += blockDim.x) d1[w] = s1[w];
    const int* s2 = reinterpret_cast<const int*> (&fr->f); int* d2 = reinterpret_cast<int*> (&sf_);
    for (int w = threadIdx.x; w < (int) (sizeof (Frame) / sizeof (int)); w += blockDim.x) d2[w] = s2[w];
  }
  __syncthreads ();
  pdl_wait ();
  const Params& p = sp_;
  const Frame& f = sf_;
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  unsigned long long upd = 0, vis = 0;
  int count = qslot >= 0 ? d_count[16 * fr->cset + qslot] : static_count;
  if (count > cell_cap) count = cell_cap;
  if (fr->timing && blockIdx.x == 0 && threadIdx.x == 0 && fr->kt[1] > fr->kt[0])
  { atomicAdd (&stats[5], fr->kt[1] - fr->kt[0]); atomicAdd (&stats[6], 1ull); }          // device-timed brick kernel of this frame
  const float sizeC = level_size (p, SL);
  const float off1 = sizeC * 0.25f;
  const int cell_lvl = p.C - SL;                        // see k_celltop_down
  constexpr int STRIDE = 585;
  const long long c_entry = clock64 ();
  for (int ci = warp; ci < count; ci += nwarps)
  {
    const long long tc0 = clock64 ();
    int dbg_slow2 = 0, dbg_slow1 = 0, dbg_ft = 0;
    const CellTop* top = tops + ci;
    const int t1 = top->t1slot;
    if (t1 < 0) continue;                                            // the cell was a leaf: nothing to fold
    const QNode cell = cells[ci];
    const float c0[3] = { center1d (p, SL, cell.x), center1d (p, SL, cell.y), center1d (p, SL, cell.z) };
    float2* gdw = p.nodes + (size_t) t1 * BRICK_NODES;
    uchar4* grgb = COLOR ? p.rgb + (size_t) t1 * BRICK_NODES : nullptr;
    uint32_t* gsw = p.split + (size_t) t1 * BRICK_SPLIT_WORDS;
    // ---- level 3 (block roots): "rc >= 0" ballots, j3 = lane + 32 i ----
    const int kind1 = lane < 8 ? top->kind[1 + lane] : KIND_DONE;
    int kind2[2]; kind2[0] = top->kind[9 + lane]; kind2[1] = top->kind[9 + 32 + lane];
    const uint32_t int1 = __ballot_sync (0xffffffffu, kind1 != KIND_DONE);
    uint32_t int2[2]; int2[0] = __ballot_sync (0xffffffffu, kind2[0] != KIND_DONE); int2[1] = __ballot_sync (0xffffffffu, kind2[1] != KIND_DONE);
    uint32_t nonneg_mine = 0;
    {
      // all loads first (16 independent kind/rc bytes per lane, then the interior block roots' return codes)
      int k3[16], r3[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) { k3[i] = top->kind[73 + lane + 32 * i]; r3[i] = top->rc[73 + lane + 32 * i]; }
#pragma unroll
      for (int i = 0; i < 16; ++i) if (k3[i] != KIND_DONE) r3[i] = gq[(size_t) ci * STRIDE + 73 + lane + 32 * i].rc;
#pragma unroll
      for (int i = 0; i < 16; ++i)
      {
        const int j2 = (lane + 32 * i) >> 3;
        const bool visited = ((j2 < 32 ? int2[0] : int2[1]) >> (j2 & 31)) & 1;
        const uint32_t nn = __ballot_sync (0xffffffffu, visited && r3[i] >= 0);
        if (lane == i) nonneg_mine = nn;
      }
    }
    const long long cA = clock64 ();
    // ---- level 2 ----
    uint32_t nonneg2[2];
#pragma unroll
    for (int i2 = 0; i2 < 2; ++i2)
    {
      const int j2 = lane + 32 * i2;
      const uint32_t nn = __shfl_sync (0xffffffffu, nonneg_mine, (lane >> 2) + 8 * i2);
      int rc = top->rc[9 + j2];
      bool slow = false;
      NodePos n;
      if (kind2[i2] != KIND_DONE)
      {
        if (((nn >> (8 * (lane & 3))) & 0xFFu) != 0 || 2 < cell_lvl) rc = 1;      // (a virtual level is never pruned)
        else
        {
          // prune: children.clear () -> split bit off, eight block-root nodes back to the fresh state
          atomicAnd (&gsw[1 + (j2 >> 5)], ~(1u << (j2 & 31)));
          for (int c = 0; c < 8; ++c) { gdw[72 + 8 * j2 + c] = make_float2 (-1.f, 0.f); if (COLOR) grgb[72 + 8 * j2 + c] = make_uchar4 (0, 0, 0, 0); }
          float c[3]; path_center (c0, off1, 2, j2, c);
          n.level = SL + 2; n.cx = c[0]; n.cy = c[1]; n.cz = c[2]; n.size = sizeC * 0.25f; n.slot = t1; n.idx = 8 + j2;
          { int lx = 0, ly = 0, lz = 0; for (int q = 1; q >= 0; --q) { int cc = (j2 >> (3 * q)) & 7; lx = (lx << 1) | (cc >> 2); ly = (ly << 1) | ((cc >> 1) & 1); lz = (lz << 1) | (cc & 1); }
            n.x = (cell.x << 2) | lx; n.y = (cell.y << 2) | ly; n.z = (cell.z << 2) | lz; }
          if (kind2[i2] == KIND_NEW) { rc = top_fallthrough_new (p, f, n, top->dnew[9 + j2], top->uv[9 + j2], upd); dbg_ft++; }
          else slow = true;
        }
      }
      // pre-existing children pruned: leaf visits, four nodes per round (eight lanes each)
      dbg_slow2 += __popc (__ballot_sync (0xffffffffu, slow));
      leaf_visit_slow_lanes (p, f, slow, n, t1, rc, upd, vis);
      const bool visited2 = (int1 >> (j2 >> 3)) & 1;
      nonneg2[i2] = __ballot_sync (0xffffffffu, visited2 && rc >= 0);
    }
    const long long cB = clock64 ();
    // ---- level 1 ----
    int rc1 = lane < 8 ? (int) top->rc[1 + lane] : 0;
    {
      bool slow = false;
      NodePos n;
      if (lane < 8 && kind1 != KIND_DONE)
      {
        const uint32_t nn = nonneg2[lane >> 2];
        if (((nn >> (8 * (lane & 3))) & 0xFFu) != 0 || 1 < cell_lvl) rc1 = 1;
        else
        {
          atomicAnd (&gsw[0], ~(1u << lane));
          for (int c = 0; c < 8; ++c) { gdw[8 + 8 * lane + c] = make_float2 (-1.f, 0.f); if (COLOR) grgb[8 + 8 * lane + c] = make_uchar4 (0, 0, 0, 0); }
          float c[3]; path_center (c0, off1, 1, lane, c);
          n.level = SL + 1; n.cx = c[0]; n.cy = c[1]; n.cz = c[2]; n.size = sizeC * 0.5f; n.slot = t1; n.idx = lane;
          n.x = (cell.x << 1) | ((lane >> 2) & 1); n.y = (cell.y << 1) | ((lane >> 1) & 1); n.z = (cell.z << 1) | (lane & 1);
          if (kind1 == KIND_NEW) rc1 = top_fallthrough_new (p, f, n, top->dnew[1 + lane], top->uv[1 + lane], upd);
          else slow = true;
        }
      }
      dbg_slow1 += __popc (__ballot_sync (0xffffffffu, slow));
      leaf_visit_slow_lanes (p, f, slow, n, t1, rc1, upd, vis);
    }
    const uint32_t nonneg1 = __ballot_sync (0xffffffffu, lane < 8 && rc1 >= 0);
    const long long cC = clock64 ();
    int dbg_cell = 0;
    // ---- the cell ----
    int rc_cell = 1;
    if ((nonneg1 & 0xFFu) == 0 && cell_lvl <= 0)
    {
      dbg_cell = top->kind[0] == KIND_NEW ? 1 : 2;
      NodePos nc; nc.level = SL; nc.x = cell.x; nc.y = cell.y; nc.z = cell.z; nc.cx = c0[0]; nc.cy = c0[1]; nc.cz = c0[2]; nc.size = sizeC; nc.slot = cell.slot; nc.idx = cell.idx;
      if (lane == 0) { uint32_t m; uint32_t* sw = split_word (p, nc, m); atomicAnd (sw, ~m); }
      if (lane < 8) { gdw[lane] = make_float2 (-1.f, 0.f); if (COLOR) grgb[lane] = make_uchar4 (0, 0, 0, 0); }
      __syncwarp ();
      if (top->kind[0] == KIND_NEW) { if (lane == 0) rc_cell = top_fallthrough_new (p, f, nc, top->dnew[0], top->uv[0], upd); rc_cell = __shfl_sync (0xffffffffu, rc_cell, 0); }
      else { __threadfence_block (); rc_cell = leaf_visit_warp_bfs (p, f, nc, s_rec[threadIdx.x >> 5], &s_cnt[threadIdx.x >> 5], upd, vis); }
    }
    if (lane == 0 && cell_lvl <= 0) cells[ci].rc = rc_cell;              // (read by k_upper_up when coarse levels lie above the supercell)
    if (p.dbg && lane == 0)
    {
      const long long cD = clock64 ();
      const unsigned long long tag = ((unsigned long long) (dbg_slow2 & 0xFF) << 24) | ((unsigned long long) (dbg_slow1 & 0xF) << 20) | ((unsigned long long) (dbg_cell & 3) << 18) | (unsigned long long) (ci & 0x3FFFF);
      atomicMax (&p.dbg[0], ((unsigned long long) (cD - tc0) << 32) | tag);
      atomicMax (&p.dbg[1], ((unsigned long long) (cA - tc0) << 32) | tag);
      atomicMax (&p.dbg[2], ((unsigned long long) (cB - cA) << 32) | tag);
      atomicMax (&p.dbg[3], ((unsigned long long) (cC - cB) << 32) | tag);
      atomicMax (&p.dbg[4], ((unsigned long long) (cD - cC) << 32) | tag);
      atomicMax (&p.dbg[5], ((unsigned long long) (tc0 - c_entry) << 32) | tag);
      atomicAdd (&p.dbg[6], (unsigned long long) dbg_slow2); atomicAdd (&p.dbg[7], (unsigned long long) dbg_slow1);
      atomicAdd (&p.dbg[8], (unsigned long long) (dbg_cell == 2)); atomicAdd (&p.dbg[9], (unsigned long long) (dbg_cell == 1));
      atomicAdd (&p.dbg[10], 1ull);
    }
  }
  __syncwarp ();
  warp_add_stats (stats, upd, vis);
}

} // namespace b2
