// engine.cu — libb200tsdf.so: handle, device memory, kernels and the C ABI (include/b200tsdf.h).
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -fmad=false (see
// __graft_entry__.build).  There is no CPU path: b200tsdf_create fails without a CUDA device.
#include "../../include/b200tsdf.h"
#include "tsdf_core.cuh"
#include "mc_tables.cuh"
#include "host_math.h"
#include "params_setup.h"
#include "brick_kernels.cuh"
#include "brick_direct.cuh"
#include "organize.cuh"
#include "depth.cuh"
#include "track.cuh"
#include "mesh_sort.h"
#include "host_pack.h"
#include "vol_io.cuh"
#include "pool_rehash.cuh"

#include <cuda_runtime.h>
#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <vector>

using namespace b2;

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (call);                                                                       \
    if (e_ != cudaSuccess) return h->fail (B200TSDF_ECUDA, std::string (#call) + ": " + cudaGetErrorString (e_)); \
  } while (0)

namespace {

struct Planes { float pl[6][4]; };

// A device buffer, freed when it goes out of scope, so error returns free it too.  One owned by a host call names its
// stream: work queued there may still read the buffer, so the stream is drained before the memory is released.  One of the
// handle has no stream: it is released by grow, or after b200tsdf_destroy has synchronised the handle's streams.
template <typename T>
struct DevBuf
{
  T* p = nullptr;
  size_t cap = 0;                               // elements allocated
  cudaStream_t s = nullptr;
  DevBuf () = default;
  explicit DevBuf (cudaStream_t stream) : s (stream) {}
  DevBuf (DevBuf&& o) noexcept : p (o.p), cap (o.cap), s (o.s) { o.p = nullptr; o.cap = 0; }
  DevBuf& operator= (DevBuf&& o) noexcept { std::swap (p, o.p); std::swap (cap, o.cap); std::swap (s, o.s); return *this; }
  DevBuf (const DevBuf&) = delete;
  DevBuf& operator= (const DevBuf&) = delete;
  ~DevBuf () { release (); }
  void release ()
  {
    if (!p) return;
    if (s) cudaStreamSynchronize (s);
    cudaFree (p);
    p = nullptr; cap = 0;
  }
  cudaError_t alloc (size_t n)                  // exactly n elements; n == 0 leaves the buffer null
  {
    release ();
    return grow (n);
  }
  cudaError_t grow (size_t n)                   // at least n elements: kept when they fit, else freed before the new allocation
  {
    if (n <= cap) return cudaSuccess;
    release ();
    const cudaError_t e = cudaMalloc (&p, n * sizeof (T));
    if (e != cudaSuccess) { p = nullptr; return e; }
    cap = n;
    return e;
  }
  cudaError_t upload (const std::vector<T>& v)  // a device copy of v
  {
    cudaError_t e = alloc (v.size ());
    if (e == cudaSuccess && !v.empty ()) e = cudaMemcpy (p, v.data (), v.size () * sizeof (T), cudaMemcpyHostToDevice);
    return e;
  }
  operator T* () const { return p; }
};

// Pinned host memory of the handle, freed with it
template <typename T>
struct Pinned
{
  T* p = nullptr;
  Pinned () = default;
  Pinned (const Pinned&) = delete;
  Pinned& operator= (const Pinned&) = delete;
  ~Pinned () { if (p) cudaFreeHost (p); }
  cudaError_t alloc (size_t n) { return cudaHostAlloc ((void**) &p, n * sizeof (T), cudaHostAllocDefault); }
  operator T* () const { return p; }
};

// A stream or event of the handle, destroyed with it
template <typename X, cudaError_t (*destroy) (X)>
struct Owned
{
  X x = nullptr;
  Owned () = default;
  Owned (const Owned&) = delete;
  Owned& operator= (const Owned&) = delete;
  ~Owned () { if (x) destroy (x); }
  operator X () const { return x; }
};
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
using Event = Owned<cudaEvent_t, cudaEventDestroy>;

// d_stats[0..ST_N) are cumulative since reset(); [ST_N..2*ST_N) is the snapshot taken at the start of
// the current frame (so last-frame = cum - prev without a host round trip); the last slot is scratch
enum StatSlot { ST_UPDATES = 0, ST_VISITS = 1, ST_BLOCKS = 2, ST_N = 8, ST_TOTAL = 2 * ST_N + 1, ST_SCRATCH = 2 * ST_N };
constexpr int KRING = 64;     // ring of event pairs around the dominant kernel
constexpr int FRAME_RING = 64;  // per-frame records in flight (device ring + its pinned host image)
constexpr int BATCH_SEGS = 16;  // host staging segments of the batch path
constexpr int RENDER_CHUNK = 32;  // poses per render launch (blockIdx.z)
constexpr int RENDER_SEGS = 8;    // pinned staging segments of RENDER_CHUNK render records
// A batch of m unorganised clouds has an organise block right behind its m frame records (OrgBatch, then m OrgRecs), so both
// go to the device in one copy; BRING_SPAN = FrameRec slots per record half (device) and per staging segment (host).
static_assert (FRAME_RING / 2 == ORG_MAX_FRAMES, "an organise batch is one record half");
constexpr size_t ORG_HDR = (sizeof (OrgBatch) + 15) & ~(size_t) 15;
constexpr int BRING_SPAN = FRAME_RING / 2 + (int) ((ORG_HDR + ORG_MAX_FRAMES * sizeof (OrgRec) + sizeof (FrameRec) - 1) / sizeof (FrameRec));
OrgBatch* org_block (FrameRec* recs, int m) { return reinterpret_cast<OrgBatch*> (recs + m); }
OrgRec* org_recs (FrameRec* recs, int m) { return reinterpret_cast<OrgRec*> (reinterpret_cast<unsigned char*> (recs + m) + ORG_HDR); }
// a batch of depth frames has its depth block (DepthBatch) in the same place
static_assert (sizeof (DepthBatch) <= ORG_HDR + ORG_MAX_FRAMES * sizeof (OrgRec), "a depth block fits where the organise block goes");
DepthBatch* depth_block (FrameRec* recs, int m) { return reinterpret_cast<DepthBatch*> (recs + m); }
// what comes in front of the frames of a batch: nothing (organised clouds), the organise launches, or the depth unprojection
enum FrontEnd { FRONT_NONE, FRONT_ORGANIZE, FRONT_DEPTH };
constexpr int DEPTH_SLOTS = 3;  // pinned staging slots (and device raw buffers) of b200tsdf_integrate_depth

// ---------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------
__global__ void k_fill_fresh (float2* __restrict__ nodes, size_t n)
{
  size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
  size_t stride = (size_t) gridDim.x * blockDim.x;
  for (; i < n; i += stride) nodes[i] = make_float2 (-1.f, 0.f);
}

// top-tier bricks that contain the coarse cells themselves (Rtop < C) are permanent
__global__ void k_insert_top_bricks (Params p)
{
  int n = 1 << p.Rtop;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * n * n) return;
  int z = i % n, y = (i / n) % n, x = i / (n * n);
  find_or_insert_brick (p, p.T - 1, x, y, z);
}

// the static supercell list of grids whose coarse cells lie inside the tier-1 bricks: every root-array node (level Rtop = L - 6)
__global__ void k_build_superq (Params p, QNode* __restrict__ q, int n)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int nn = 1 << p.Rtop;
  QNode e; e.x = i / (nn * nn); e.y = (i / nn) % nn; e.z = i % nn; e.slot = -1; e.idx = i; e.kind = KIND_DONE; e.child_base = -1; e.rc = 0;
  q[i] = e;
}

// frustum cull of the coarse cells (tsdf_volume_octree.cpp:619-652); planes come from the host
__global__ void k_cull (Params p, Planes P, unsigned char* __restrict__ mask)
{
  int n = 1 << p.C;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * n * n) return;
  int z = i % n, y = (i / n) % n, x = i / (n * n);
  float cx = center1d (p, p.C, x), cy = center1d (p, p.C, y), cz = center1d (p, p.C, z);
  mask[i] = frustum_contains (P.pl, cx, cy, cz) ? 1 : 0;
}

// b200tsdf_changed_cells: the mask of cell_changed over the 8^C cells
__global__ void k_changed_cells (int C, const unsigned long long* __restrict__ cell_epoch, unsigned long long since,
                                 unsigned char* __restrict__ mask)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 1 << (3 * C)) return;
  mask[i] = cell_changed (C, cell_epoch, since, i) ? 1 : 0;
}

// frame front end in ONE launch: blocks [0, cull_blocks) run the frustum cull of the coarse cells, the
// rest the per-pixel pre-split.  The two are independent (the cull reads only geometry).  The work-list
// counters and the statistics snapshot are reset by the frame-begin bookkeeping of the previous k_front launch.
// The frame's parameters come from a record in device memory (FrameRec), so a captured launch can be replayed.
#define B2_STAGE_FRAME(fr)                                                      \
  __shared__ FrameRec s_fr_;                                                    \
  {                                                                             \
    const int* src_ = reinterpret_cast<const int*> (fr);                        \
    int* dst_ = reinterpret_cast<int*> (&s_fr_);                                \
    for (int w_ = threadIdx.x; w_ < (int) (sizeof (FrameRec) / sizeof (int)); w_ += blockDim.x) dst_[w_] = src_[w_]; \
  }                                                                             \
  __syncthreads ();                                                             \
  const Frame& f = s_fr_.f;

// q0 / q1: the cell queue of a frame with counter set 0 / 1 (null: no queue); fold: the fold marks (FoldState) when the route
// publishes them, else null.
//
// A gated frame (FrameRec::gated, set by the host only when the previous frame's route published the marks) does not wait for
// the previous frame's k_celltop_up as a whole.  Every block waits for `opened == seq - 1`: the previous frame's k_front is then
// complete, so its visited marks are final and, through its block 0's griddepcontrol.wait, every frame before it is complete.
// That is what makes the two counter sets, planes and cell queues enough: what this frame writes was last used by frame
// seq - 2.  A pixel thread then waits only until the previous frame has folded its own supercell, if that frame visits it: a
// pre-split reads and writes only its supercell's state (the root split bit, the tier-1 brick, the tier-0 bricks below it) and
// the brick hash, whose slot order nothing observes.  Only block 0 executes griddepcontrol.wait, last, followed by the
// frame-begin bookkeeping, so the kernel still completes after the previous frame's last kernel and k_celltop_down's own wait
// orders all of that frame before this frame's updates; every other block exits as soon as its own work is done.
// No deadlock: this kernel starts only after every CTA of the previous frame's k_celltop_up has executed
// griddepcontrol.launch_dependents (its first statement), and so after every CTA of that frame's other kernels has started; all
// of them are resident, and the frames before it are complete.  A waiting thread therefore waits only on resident work.
__global__ void k_front (Params p, const FrameRec* __restrict__ fr, int cull_blocks, int* __restrict__ list, int* __restrict__ d_count,
                         QNode* __restrict__ q0, QNode* __restrict__ q1, uint32_t* __restrict__ fold, unsigned long long* __restrict__ stats)
{
  pdl_launch_dependents ();
  B2_STAGE_FRAME (fr)
  // what depends only on the frame and the caller's cloud is done before waiting for the previous frame: the frustum test
  // of a coarse cell, and a pixel's point load, world transform and descent to its finest voxel.  The blocks that are
  // resident while the previous frame's bottom-up sweep drains so hide the cloud's DRAM latency behind it.
  const bool cull = (int) blockIdx.x < cull_blocks;
  const int n = 1 << p.C;
  int i, x = 0, y = 0, z = 0;
  bool act;                                             // cull: the cell is culled in and owned; pixel: inside the image
  bool split_it = false;                                // pixel: its finest voxel is in the volume and in an owned cell
  int fx_ = 0, fy_ = 0, fz_ = 0;
  uint32_t zb = 0u, bgra = 0u;
  if (cull)
  {
    i = blockIdx.x * blockDim.x + threadIdx.x;
    act = i < n * n * n;
    if (act)
    {
      z = i % n; y = (i / n) % n; x = i / (n * n);
      const float cx = center1d (p, p.C, x), cy = center1d (p, p.C, y), cz = center1d (p, p.C, z);
      act = frustum_contains (s_fr_.pl, cx, cy, cz) && owns_cell (p, x, y, z);
    }
  }
  else
  {
    i = (blockIdx.x - cull_blocks) * blockDim.x + threadIdx.x;
    act = i < f.width * f.height;
    if (act)
    {
      const int u = i % f.width, v = i / f.width;
      const float* pt = frame_xyz (f, u, v);
      zb = reinterpret_cast<const uint32_t*> (pt)[2];
      if (p.color && f.rgba_off >= 0) bgra = *reinterpret_cast<const uint32_t*> (frame_bgr (f, u, v));
      const float zf = __uint_as_float (zb);
      if (!is_nan (zf))                                                 // hpp:64
      {
        float pw[3];
        affine_mul_f (f.tfwd, pt[0], pt[1], zf, pw);                    // hpp:76
        split_it = world_to_finest (p, pw[0], pw[1], pw[2], fx_, fy_, fz_);
        if (split_it && p.shard_count > 1)
        {
          const int sh = p.L - p.C;
          split_it = owns_cell (p, fx_ >> sh, fy_ >> sh, fz_ >> sh);
        }
      }
    }
  }
  const int cset = s_fr_.cset;
  const bool gated = s_fr_.gated != 0;
  const FoldState fs = fold_state (fold, p.C);
  if (gated)
  {
    if (threadIdx.x == 0) wait_mark (p, fs.opened, s_fr_.seq - 1u);
    __syncthreads ();
  }
  else pdl_wait ();                                     // the previous frame's bottom-up sweep has finished
  int* count = d_count + 16 * cset;
  int* next_counts = d_count + 16 * (cset ^ 1);
  // frame-begin bookkeeping (was a launch of its own): snapshot the cumulative counters, and clear the counter
  // set the NEXT frame will use (the sets alternate, so nothing in this frame touches it)
  auto frame_begin = [&] () {
    if (blockIdx.x == 0 && threadIdx.x < 16)
    {
      if (p.dbg && threadIdx.x == 0) atomicAdd (&p.dbg[gated ? 11 : 12], 1ull);   // which k_front ran (b200tsdf_debug_timing)
      if (threadIdx.x < ST_N) stats[ST_N + threadIdx.x] = stats[threadIdx.x];
      next_counts[threadIdx.x] = 0;
    }
  };
  if (!gated) frame_begin ();
  if (cull)
  {
    if (act)
    {
      int k = atomicAdd (count, 1);
      list[k] = i;
      if (q0)
      {
        NodePos nd;
        if (!locate_node (p, p.C, x, y, z, nd)) { raise_err (p, ERR_MISSING_BRICK); nd.slot = -1; nd.idx = 0; }
        QNode e; e.x = x; e.y = y; e.z = z; e.slot = nd.slot; e.idx = nd.idx; e.kind = KIND_DONE; e.child_base = -1; e.rc = 0;
        (cset ? q1 : q0)[k] = e;
      }
      if (fold) fs.visited[(size_t) cset * (n * n * n) + i] = s_fr_.seq;
      stamp_cell (p, i, s_fr_.epoch);                   // the frame's updates, splits and prunes of this cell
    }
  }
  else
  {
    // the pixel plane the observations of this frame read (frame_plane): a bit copy of every pixel, NaN depths, points
    // outside the volume and points in another shard's cells included, because an observation may project onto any pixel.
    // The previous readers of this plane are frame seq - 2's kernels, which are complete.
    if (act)
    {
      uint32_t* pix = frame_plane (p, cset);
      if (p.color) reinterpret_cast<uint2*> (pix)[i] = make_uint2 (zb, bgra);
      else pix[i] = zb;
    }
    if (gated)
    {
      // wait for the previous frame's fold of this pixel's supercell, one poll per distinct cell of the warp
      const int sh = p.L - p.C;
      const int cell = split_it ? (((fx_ >> sh) * n + (fy_ >> sh)) * n + (fz_ >> sh)) : -1;
      const uint32_t prev = s_fr_.seq - 1u;
      const uint32_t* prev_visited = fs.visited + (size_t) (cset ^ 1) * (n * n * n);
      const int lane = threadIdx.x & 31;
      unsigned todo = __ballot_sync (0xffffffffu, cell >= 0);
      while (todo)
      {
        const int leader = __ffs (todo) - 1;
        const int c = __shfl_sync (0xffffffffu, cell, leader);
        todo &= ~__ballot_sync (0xffffffffu, cell == c);
        if (lane == leader && ld_relaxed (prev_visited + c) == prev) wait_mark (p, fs.folded + c, prev);
      }
      __syncwarp ();
    }
    if (split_it) presplit_point (p, fx_, fy_, fz_, s_fr_.epoch);
  }
  if (gated && blockIdx.x == 0 && threadIdx.x < 16)
  {
    pdl_wait ();                                        // the previous frame's bottom-up sweep has finished
    frame_begin ();
  }
}

// general path: one thread per culled coarse cell runs updateVoxel depth-first.  The frame and its counter set come from
// the record, like the other kernels of a frame, so the launch can be captured and replayed.
__global__ void k_update_dfs (Params p, const FrameRec* __restrict__ fr, const int* __restrict__ list, const int* __restrict__ d_count,
                              unsigned long long* __restrict__ stats)
{
  const int* count = d_count + 16 * fr->cset;
  if ((int) (blockIdx.x * blockDim.x) >= *count) return;  // (whole block: the grid covers every coarse cell)
  B2_SHARED_FRAME (fr)
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= *count) return;
  int n = 1 << p.C;
  int id = list[i];
  int z = id % n, y = (id / n) % n, x = id / (n * n);
  NodePos node;
  if (!locate_node (p, p.C, x, y, z, node)) { raise_err (p, ERR_MISSING_BRICK); return; }
  Counters cnt; cnt.n_updates = 0; cnt.n_visits = 0;
  update_voxel_dfs (p, f, node, cnt);
  atomicAdd (&stats[ST_UPDATES], (unsigned long long) cnt.n_updates);
  atomicAdd (&stats[ST_VISITS], (unsigned long long) cnt.n_visits);
}

// read-side kernels keep Params in shared memory (see find_leaf in tsdf_core.cuh)
#define B2_STAGE_PARAMS(gp)                                                     \
  __shared__ Params sp_;                                                        \
  {                                                                             \
    const int* src_ = reinterpret_cast<const int*> (&gp);                       \
    int* dst_ = reinterpret_cast<int*> (&sp_);                                  \
    for (int w_ = threadIdx.x; w_ < (int) (sizeof (Params) / sizeof (int)); w_ += blockDim.x) dst_[w_] = src_[w_]; \
  }                                                                             \
  __syncthreads ();                                                             \
  const Params& p = sp_;

__global__ void k_query (Params gp, const float* __restrict__ xyz, int n, int what, int mode,
                         float* val, float* grad, float* hess, unsigned char* ok)
{
  B2_STAGE_PARAMS (gp)
  const size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t) n) return;
  float v, g[3], hs[9];
  bool good = query_point (p, xyz + 3 * i, mode, &v, g, hs);
  ok[i] = good ? 1 : 0;
  if (!good) return;
  if (what & 1) val[i] = v;
  if (what & 2) { grad[3 * i] = g[0]; grad[3 * i + 1] = g[1]; grad[3 * i + 2] = g[2]; }
  if (what & 4) for (int k = 0; k < 9; ++k) hess[9 * i + k] = hs[k];
}

// getTSDFValue = interpolateTrilinearly (tsdf_volume_octree.cpp:454-541), one thread per point
__global__ void k_interpolate (Params gp, const float* __restrict__ xyz, int n, float* __restrict__ val, unsigned char* __restrict__ valid)
{
  B2_STAGE_PARAMS (gp)
  const size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t) n) return;
  bool v = valid[i] != 0;
  val[i] = interpolate_trilinearly (p, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], &v);
  valid[i] = v ? 1 : 0;
}

// Octree::getContainingVoxel (x, y, z, min_size) and the node's accessors, one thread per point
__global__ void k_voxels (Params gp, const float* __restrict__ xyz, size_t n, float min_size, VoxelRec* __restrict__ out)
{
  B2_STAGE_PARAMS (gp)
  const size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[i] = find_voxel (p, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], min_size);
}

// OctreeNode::setData for a batch of points (tsdf_core.cuh, edit_resolve): per point its status and node address, the bid
// for the node in the table, and the count of accepted writes outside the fast route's domain in *ood
__global__ void k_edit_resolve (Params gp, const float* __restrict__ xyz, int n, float min_size, const float* __restrict__ d,
                                const float* __restrict__ w, unsigned char* __restrict__ status, uint64_t* __restrict__ addr,
                                uint64_t* __restrict__ keys, int* __restrict__ last, uint32_t mask, unsigned long long* __restrict__ ood)
{
  B2_STAGE_PARAMS (gp)
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool out = false;
  if (i < n)
  {
    const float di = d[i], wi = w[i];
    uint64_t a = 0;
    const int st = edit_resolve (p, xyz[3 * (size_t) i], xyz[3 * (size_t) i + 1], xyz[3 * (size_t) i + 2], min_size, di, wi, a);
    status[i] = (unsigned char) st;
    if (st == EDIT_WRITTEN)
    {
      addr[i] = a;
      edit_claim (keys, last, mask, a, i);
      out = !edit_in_fast_domain (di, wi);
    }
  }
  // one add per warp: a batch written wholly outside the domain does not queue n atomics on one word
  const unsigned m = __ballot_sync (0xffffffffu, out);
  if (m && (threadIdx.x & 31) == 0) atomicAdd (ood, (unsigned long long) __popc (m));
}

// the last point of the batch that reached each node stores its {d, w}, stamps the node's cell with `epoch` and sets *wrote
__global__ void k_edit_store (Params p, int n, const float* __restrict__ d, const float* __restrict__ w,
                              const unsigned char* __restrict__ status, const uint64_t* __restrict__ addr,
                              uint64_t* __restrict__ keys, const int* __restrict__ last, uint32_t mask,
                              unsigned long long epoch, int* __restrict__ wrote)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || status[i] != EDIT_WRITTEN) return;
  const uint64_t a = addr[i];
  if (!edit_wins (keys, last, mask, a, i)) return;
  edit_store (p, a, d[i], w[i]);
  stamp_cell (p, edit_cell (p, a), epoch);
  *wrote = 1;
}

// Dense crop of the box [i0, i1) x [j0, j1) x [k0, k1): one CTA per 8x8x8 tile (the finest voxels of one level L-3 node),
// clipped to the box.  Thread 0 walks the tile's path once (dense_tile_walk); every voxel then resolves its leaf from the
// tier-0 brick's split words, staged with the path in shared memory.  Outputs are [i][j][k], k fastest: eight consecutive
// threads write one run along k.
struct DenseBox { int i0, j0, k0, i1, j1, k1; int ti0, tj0, tk0, ntj, ntk; };
constexpr int DENSE_THREADS = 256;

__global__ void __launch_bounds__ (DENSE_THREADS) k_dense (Params gp, DenseBox b, float* __restrict__ d_d, float* __restrict__ d_w,
                                                           unsigned char* __restrict__ d_rgb, signed char* __restrict__ d_level)
{
  __shared__ DenseTile st;
  B2_STAGE_PARAMS (gp)
  const unsigned tile = blockIdx.x;
  const int tz = b.tk0 + (int) (tile % (unsigned) b.ntk);
  const int ty = b.tj0 + (int) ((tile / (unsigned) b.ntk) % (unsigned) b.ntj);
  const int tx = b.ti0 + (int) (tile / ((unsigned) b.ntk * (unsigned) b.ntj));
  if (threadIdx.x == 0) dense_tile_walk (p, tx, ty, tz, st);
  __syncthreads ();
  const size_t nj = (size_t) (b.j1 - b.j0), nk = (size_t) (b.k1 - b.k0);
  for (int v = threadIdx.x; v < 512; v += DENSE_THREADS)
  {
    const int X = 8 * tx + (v >> 6), Y = 8 * ty + ((v >> 3) & 7), Z = 8 * tz + (v & 7);
    if (X < b.i0 || X >= b.i1 || Y < b.j0 || Y >= b.j1 || Z < b.k0 || Z >= b.k1) continue;
    float2 dw; uchar4 c; int level;
    dense_voxel (p, st, X, Y, Z, dw, c, level);
    const size_t o = ((size_t) (X - b.i0) * nj + (size_t) (Y - b.j0)) * nk + (size_t) (Z - b.k0);
    if (d_d) d_d[o] = dw.x;
    if (d_w) d_w[o] = dw.y;
    if (d_rgb) { d_rgb[3 * o] = c.x; d_rgb[3 * o + 1] = c.y; d_rgb[3 * o + 2] = c.z; }
    if (d_level) d_level[o] = (signed char) level;
  }
}

// renderView for a batch of poses: blockIdx.z is the pose within the launch, and each block stages that pose's record.  Pixels
// are row-major, one image after the other; each gets 12 bytes of xyz at xyz_off and 12 of normal at normal_off (4-byte
// aligned), and no other byte of the caller's buffer is written.  rgb: 3 bytes per pixel, or null.
__global__ void k_render (Params gp, const RenderParams* __restrict__ recs, unsigned char* __restrict__ out, size_t stride,
                          int xyz_off, int normal_off, unsigned char* __restrict__ rgb)
{
  __shared__ RenderParams sr_;
  for (int w = threadIdx.x; w < (int) (sizeof (RenderParams) / sizeof (int)); w += blockDim.x)
    reinterpret_cast<int*> (&sr_)[w] = reinterpret_cast<const int*> (recs + blockIdx.z)[w];
  B2_STAGE_PARAMS (gp)                                  // (its barrier also covers the record)
  const RenderParams& r = sr_;
  // 8x8 pixel tiles keep neighbouring rays in one warp-pair
  int tx = threadIdx.x % 8, ty = threadIdx.x / 8;
  int x = blockIdx.x * 8 + tx, y = blockIdx.y * 8 + ty;
  if (x >= r.width || y >= r.height) return;
  const size_t i = ((size_t) blockIdx.z * r.height + y) * r.width + x;
  float P[3], N[3];
  render_pixel (p, r, x, y, P, N, rgb ? rgb + 3 * i : nullptr);
  float* o = reinterpret_cast<float*> (out + i * stride + xyz_off);
  o[0] = P[0]; o[1] = P[1]; o[2] = P[2];
  o = reinterpret_cast<float*> (out + i * stride + normal_off);
  o[0] = N[0]; o[1] = N[1]; o[2] = N[2];
}

__global__ void k_list_bricks (Params p, int* __restrict__ list, int* __restrict__ count)
{
  size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i > p.pool_mask) return;
  if (p.keys[i] != KEY_EMPTY) list[atomicAdd (count, 1)] = (int) i;
}

// number of claimed directory slots (statistics): one atomic per warp
__global__ void k_count_bricks (Params p, int* __restrict__ count)
{
  size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
  const bool used = i <= p.pool_mask && p.keys[i] != KEY_EMPTY;
  const unsigned m = __ballot_sync (0xffffffffu, used);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd (count, __popc (m));
}

__global__ void k_gather_bricks (Params p, const int* __restrict__ list, int n,
                                 float2* nodes, uint32_t* split, uchar4* rgb, float* M, int* ns)
{
  int b = blockIdx.x;
  if (b >= n) return;
  size_t s = (size_t) list[b];
  for (int i = threadIdx.x; i < BRICK_NODES; i += blockDim.x)
  {
    nodes[(size_t) b * BRICK_NODES + i] = p.nodes[s * BRICK_NODES + i];
    if (rgb) rgb[(size_t) b * BRICK_NODES + i] = p.rgb[s * BRICK_NODES + i];
    if (M) { M[(size_t) b * BRICK_NODES + i] = p.M[s * BRICK_NODES + i]; ns[(size_t) b * BRICK_NODES + i] = p.ns[s * BRICK_NODES + i]; }
  }
  for (int i = threadIdx.x; i < BRICK_SPLIT_WORDS; i += blockDim.x)
    split[(size_t) b * BRICK_SPLIT_WORDS + i] = p.split[s * BRICK_SPLIT_WORDS + i];
}

__global__ void k_gather_rgbn (Params p, const int* __restrict__ list, int n, float4* __restrict__ out)
{
  int b = blockIdx.x;
  if (b >= n) return;
  size_t s = (size_t) list[b];
  for (int i = threadIdx.x; i < BRICK_NODES; i += blockDim.x) out[(size_t) b * BRICK_NODES + i] = p.rgbn[s * BRICK_NODES + i];
}

// .vol import: claim each brick's slot and copy its payload in
__global__ void k_load_bricks (Params p, const uint64_t* __restrict__ keys, int n, const float2* __restrict__ nodes, const uint32_t* __restrict__ split,
                               const uchar4* __restrict__ rgb, const float* __restrict__ M, const int* __restrict__ ns)
{
  __shared__ int slot_s;
  int b = blockIdx.x;
  if (b >= n) return;
  if (threadIdx.x == 0)
  {
    int t, bx, by, bz;
    brick_key_decode (keys[b], t, bx, by, bz);
    slot_s = find_or_insert_brick (p, t, bx, by, bz);
  }
  __syncthreads ();
  if (slot_s < 0) return;
  size_t s = (size_t) slot_s;
  for (int i = threadIdx.x; i < BRICK_NODES; i += blockDim.x)
  {
    p.nodes[s * BRICK_NODES + i] = nodes[(size_t) b * BRICK_NODES + i];
    if (p.rgb && rgb) p.rgb[s * BRICK_NODES + i] = rgb[(size_t) b * BRICK_NODES + i];
    if (p.M && M) { p.M[s * BRICK_NODES + i] = M[(size_t) b * BRICK_NODES + i]; p.ns[s * BRICK_NODES + i] = ns[(size_t) b * BRICK_NODES + i]; }
  }
  for (int i = threadIdx.x; i < BRICK_SPLIT_WORDS; i += blockDim.x) p.split[s * BRICK_SPLIT_WORDS + i] = split[(size_t) b * BRICK_SPLIT_WORDS + i];
}

// b200tsdf_resize_pool: the claimed old slots in list[0, n) into the fresh pool of `to`, one warp per brick (REHASH_THREADS / 32
// bricks per CTA).  A brick that finds no slot within MAX_PROBE raises ERR_POOL_FULL on to.err and is dropped.
constexpr int REHASH_THREADS = 256;
__global__ void __launch_bounds__ (REHASH_THREADS) k_pool_rehash (Params from, Params to, const int* __restrict__ list, int n)
{
  const int b = (int) ((blockIdx.x * (unsigned) REHASH_THREADS + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (b >= n) return;
  const uint32_t s = (uint32_t) list[b];
  int d = 0;
  if (lane == 0) d = rehash_claim (from, to, s);
  d = __shfl_sync (0xffffffffu, d, 0);
  if (d >= 0) rehash_brick (from, to, s, (uint32_t) d, lane, 32);
}

// shard import: scatter coarse-cell (root array) entries
__global__ void k_import_roots (Params p, int n, const int* __restrict__ idx, const float2* __restrict__ dw, const unsigned char* __restrict__ split,
                                const uchar4* __restrict__ rgb, const float* __restrict__ M, const int* __restrict__ ns)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int r = idx[i];
  p.root_dw[r] = dw[i];
  if (split[i]) atomicOr (&p.root_split[r >> 5], 1u << (r & 31)); else atomicAnd (&p.root_split[r >> 5], ~(1u << (r & 31)));
  if (p.root_rgb) p.root_rgb[r] = rgb[i];
  if (p.root_M) { p.root_M[r] = M[i]; p.root_ns[r] = ns[i]; }
}

// ---- the read-side walk of the flat layout (marching cubes, getLeaves): one warp per claimed brick whose root has children,
// every node through brick_node, and one thread per root-array entry.  The emission order depends on the hash layout and on
// atomics; the host sorts the records by order key afterwards. ----

// exclusive prefix of the lanes' counts n and one atomicAdd on *total per warp: `first` = this lane's first output slot.
// False when the whole warp has nothing to write.  Every lane of the warp must call it.
__device__ __forceinline__ bool warp_reserve (unsigned long long* total, int n, unsigned long long& first)
{
  const int lane = threadIdx.x & 31;
  int incl = n;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync (0xffffffffu, incl, o); if (lane >= o) incl += v; }
  const int wtotal = __shfl_sync (0xffffffffu, incl, 31);
  if (wtotal == 0) return false;
  unsigned long long wbase = 0;
  if (lane == 0) wbase = atomicAdd (total, (unsigned long long) wtotal);
  first = __shfl_sync (0xffffffffu, wbase, 0) + (unsigned long long) (incl - n);
  return true;
}

// one cube's triangles from slot tri0 on, with their order keys (mc_order_key << 3 | triangle)
__device__ __forceinline__ void mc_emit (const Params& p, const McParams& mc, const NodePos& n, float2 dw, int ntri, unsigned long long tri0,
                                         float* verts, unsigned char* cols, unsigned long long* okeys)
{
  mc_leaf (p, mc, n, dw.x, dw.y, b200tsdf_mc::edge_table, b200tsdf_mc::tri_table, verts + tri0 * 9, cols ? cols + tri0 * 9 : nullptr);
  const unsigned long long k = mc_order_key (p, n) << 3;
  for (int t = 0; t < ntri; ++t) okeys[tri0 + t] = k | (unsigned long long) t;
}

// whether a brick rooted at level R, coordinates (bx, by, bz), holds a leaf of a selected cell (McParams::cell_mask): the
// brick's one cell when R >= C, else any of its 8^(C - R) cells.  Every lane of the warp must call it.
__device__ __forceinline__ bool mc_brick_selected (const Params& p, const McParams& mc, int R, int bx, int by, int bz)
{
  if (!mc.cell_mask) return true;
  const int d = p.C - R;
  if (d <= 0) return mc.cell_mask[coarse_cell (p, R, bx, by, bz)] != 0;
  if (d > 3) return false;                                      // every node of the brick lies above the coarse depth
  bool any = false;
  for (int c = threadIdx.x & 31; c < 1 << (3 * d); c += 32)
  {
    int x = bx, y = by, z = bz;
    for (int q = d - 1; q >= 0; --q) { const int o = (c >> (3 * q)) & 7; x = (x << 1) | (o >> 2); y = (y << 1) | ((o >> 1) & 1); z = (z << 1) | (o & 1); }
    any |= mc.cell_mask[coarse_cell (p, p.C, x, y, z)] != 0;
  }
  return __any_sync (0xffffffffu, any);
}

// the count pass adds a cube's triangles to its cell (McParams::cell_tris)
__device__ __forceinline__ void mc_count_cell (const Params& p, const McParams& mc, const NodePos& n, int ntri)
{
  if (mc.cell_tris && ntri) atomicAdd (&mc.cell_tris[coarse_cell (p, n.level, n.x, n.y, n.z)], (unsigned long long) ntri);
}

// marching cubes: one cube per existing leaf at or below the coarse depth, in the selected cells (McParams::cell_mask).
// CELLS = false: McParams::cell_mask and cell_tris are null, and their tests are compiled out (the full mesh).
template <bool EMIT, bool CELLS>
__global__ void k_mesh_bricks (Params gp, McParams mc, const int* __restrict__ list, int nbricks,
                               unsigned long long* __restrict__ total, float* __restrict__ verts, unsigned char* __restrict__ cols,
                               unsigned long long* __restrict__ okeys)
{
  B2_STAGE_PARAMS (gp)
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= nbricks) return;
  const int slot = list[warp];
  int t, bx, by, bz;
  brick_key_decode (p.keys[slot], t, bx, by, bz);
  const int R = tier_root_level (p, t);
  if (CELLS && !mc_brick_selected (p, mc, R, bx, by, bz)) return;
  if (!brick_root_is_split (p, t, bx, by, bz)) return;         // nothing below an unsplit root exists
  const uint32_t* sw = p.split + (size_t) slot * BRICK_SPLIT_WORDS;
  for (int base = 0; base < BRICK_NODES; base += 32)
  {
    const int i = base + lane;
    int ntri = 0;
    NodePos n; float2 dw;
    if (i < BRICK_NODES)
    {
      const BrickNode b = brick_node (p, sw, R, bx, by, bz, true, i);
      if (b.exists && !b.split && b.level >= p.C && (!CELLS || mc_cell_selected (p, mc, b.level, b.x, b.y, b.z)))
      {
        n = brick_node_pos (p, b, slot, i);
        dw = p.nodes[(size_t) slot * BRICK_NODES + i];
        ntri = mc_leaf (p, mc, n, dw.x, dw.y, b200tsdf_mc::edge_table, b200tsdf_mc::tri_table, nullptr, nullptr);
        if (CELLS && !EMIT) mc_count_cell (p, mc, n, ntri);
      }
    }
    unsigned long long tri0;
    if (!warp_reserve (total, ntri, tri0)) continue;
    if (EMIT && ntri > 0) mc_emit (p, mc, n, dw, ntri, tri0, verts, cols, okeys);
  }
}

// leaves held in the root arrays (unsplit coarse cells when Rtop == C)
template <bool EMIT, bool CELLS>
__global__ void k_mesh_roots (Params gp, McParams mc, unsigned long long* __restrict__ total, float* __restrict__ verts, unsigned char* __restrict__ cols,
                              unsigned long long* __restrict__ okeys)
{
  B2_STAGE_PARAMS (gp)
  const int n = 1 << p.Rtop;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int ntri = 0;
  NodePos nd; float2 dw;
  if (i < n * n * n)                                           // (the block size is a multiple of 32: every lane reaches warp_reserve)
  {
    nd = make_root (p, i / (n * n), (i / n) % n, i % n);
    if (!is_split (p, nd) && (!CELLS || mc_cell_selected (p, mc, nd.level, nd.x, nd.y, nd.z)))
    {
      dw = p.root_dw[nd.idx];
      ntri = mc_leaf (p, mc, nd, dw.x, dw.y, b200tsdf_mc::edge_table, b200tsdf_mc::tri_table, nullptr, nullptr);
      if (CELLS && !EMIT) mc_count_cell (p, mc, nd, ntri);
    }
  }
  unsigned long long tri0;
  if (!warp_reserve (total, ntri, tri0)) return;
  if (EMIT && ntri > 0) mc_emit (p, mc, nd, dw, ntri, tri0, verts, cols, okeys);
}

// getLeaves (getVoxelCenters / getOccupiedVoxelIndices): leaf_selected as predicate and one 12-byte record (centre or voxel
// index) plus its order key per selected node
__device__ __forceinline__ void leaf_emit (const Params& p, int level, int x, int y, int z, bool index, unsigned long long o,
                                           unsigned long long* okeys, uint32_t* rec)
{
  NodePos n; n.level = level; n.x = x; n.y = y; n.z = z;
  okeys[o] = mc_order_key (p, n);
  leaf_record (p, level, x, y, z, index, rec + 3 * o);
}

template <bool EMIT>
__global__ void k_leaves_bricks (Params gp, const int* __restrict__ list, int nbricks, int nlevels, int occupied,
                                 unsigned long long* __restrict__ total, unsigned long long* __restrict__ okeys, uint32_t* __restrict__ rec)
{
  B2_STAGE_PARAMS (gp)
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= nbricks) return;
  const int slot = list[warp];
  int t, bx, by, bz;
  brick_key_decode (p.keys[slot], t, bx, by, bz);
  const int R = tier_root_level (p, t);
  if (nlevels >= 0 && R + 1 > nlevels) return;                 // the whole brick lies below the depth limit
  if (!brick_root_is_split (p, t, bx, by, bz)) return;         // nothing below an unsplit root exists
  const uint32_t* sw = p.split + (size_t) slot * BRICK_SPLIT_WORDS;
  for (int base = 0; base < BRICK_NODES; base += 32)
  {
    const int i = base + lane;
    BrickNode b{};
    bool sel = false;
    if (i < BRICK_NODES)
    {
      b = brick_node (p, sw, R, bx, by, bz, true, i);
      float2 dw = make_float2 (-1.f, 0.f);
      if (occupied) dw = p.nodes[(size_t) slot * BRICK_NODES + i];
      sel = leaf_selected (b.level, b.exists, b.split, nlevels, occupied != 0, dw.x, dw.y);
    }
    unsigned long long o;
    if (!warp_reserve (total, sel ? 1 : 0, o)) continue;
    if (EMIT && sel) leaf_emit (p, b.level, b.x, b.y, b.z, occupied != 0, o, okeys, rec);
  }
}

// root-array entries (coarse cells when Rtop == C; above the coarse depth they always have children)
template <bool EMIT>
__global__ void k_leaves_roots (Params gp, int nlevels, int occupied, unsigned long long* __restrict__ total,
                                unsigned long long* __restrict__ okeys, uint32_t* __restrict__ rec)
{
  B2_STAGE_PARAMS (gp)
  const int n = 1 << p.Rtop;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int z = i % n, y = (i / n) % n, x = i / (n * n);
  bool sel = false;
  if (i < n * n * n)                                           // (the block size is a multiple of 32: every lane reaches warp_reserve)
  {
    const NodePos nd = make_root (p, x, y, z);
    const float2 dw = p.root_dw[nd.idx];
    sel = leaf_selected (p.Rtop, true, is_split (p, nd), nlevels, occupied != 0, dw.x, dw.y);
  }
  unsigned long long o;
  if (!warp_reserve (total, sel ? 1 : 0, o)) return;
  if (EMIT && sel) leaf_emit (p, p.Rtop, x, y, z, occupied != 0, o, okeys, rec);
}

// getLeaves (nlevels) for 0 <= nlevels < C (or nlevels == 0): every node of that depth, written straight into place
__global__ void k_leaves_level (Params gp, int level, unsigned long long count, uint32_t* __restrict__ rec)
{
  B2_STAGE_PARAMS (gp)
  unsigned long long i = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  int x, y, z;
  morton_decode (level, i, x, y, z);
  leaf_record (p, level, x, y, z, false, rec + 3 * i);
}

// ---- .vol save on the device (DESIGN.md §3e): every node of the walk as a VolNode with its pre-order key, sorted, then
// formatted into byte-packed records ----

// the root-array entries, and the geometry-only levels above them: the ancestor at level l < Rtop is emitted by the entry
// whose coordinates are its child-0 chain
template <bool EMIT>
__global__ void k_vol_roots (Params gp, unsigned long long* __restrict__ total, unsigned long long* __restrict__ okeys, VolNode* __restrict__ out)
{
  B2_STAGE_PARAMS (gp)
  const int n = 1 << p.Rtop;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int z = i % n, y = (i / n) % n, x = i / (n * n);
  int cnt = 0;
  if (i < n * n * n)                                           // (the block size is a multiple of 32: every lane reaches warp_reserve)
  {
    cnt = 1;
    for (int l = p.Rtop - 1; l >= 0; --l)
    {
      const int m = (1 << (p.Rtop - l)) - 1;
      if ((x & m) || (y & m) || (z & m)) break;
      ++cnt;
    }
  }
  unsigned long long o;
  if (!warp_reserve (total, cnt, o)) return;
  if (!EMIT || !cnt) return;
  const NodePos nd = make_root (p, x, y, z);
  okeys[o] = vol_key (p, p.Rtop, x, y, z);
  out[o] = vol_node (okeys[o], -1, nd.idx, vol_has_children (p, nd));
  for (int c = 1; c < cnt; ++c)
  {
    const int l = p.Rtop - c;
    okeys[o + c] = vol_key (p, l, x >> c, y >> c, z >> c);
    out[o + c] = vol_node (okeys[o + c], VOL_SLOT_GEOM, 0, true);
  }
}

// every node of every claimed brick whose root has children: one warp per brick, through brick_node as the mesh and the leaf
// lists walk it
template <bool EMIT>
__global__ void k_vol_bricks (Params gp, const int* __restrict__ list, int nbricks, unsigned long long* __restrict__ total,
                              unsigned long long* __restrict__ okeys, VolNode* __restrict__ out)
{
  B2_STAGE_PARAMS (gp)
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= nbricks) return;
  const int slot = list[warp];
  int t, bx, by, bz;
  brick_key_decode (p.keys[slot], t, bx, by, bz);
  if (!brick_root_is_split (p, t, bx, by, bz)) return;
  const int R = tier_root_level (p, t);
  const uint32_t* sw = p.split + (size_t) slot * BRICK_SPLIT_WORDS;
  for (int base = 0; base < BRICK_NODES; base += 32)
  {
    const int i = base + lane;
    BrickNode b{};
    bool sel = false;
    if (i < BRICK_NODES)
    {
      b = brick_node (p, sw, R, bx, by, bz, true, i);
      sel = b.exists;
    }
    unsigned long long o;
    if (!warp_reserve (total, sel ? 1 : 0, o)) continue;
    if (EMIT && sel)
    {
      NodePos n; n.level = b.level; n.x = b.x; n.y = b.y; n.z = b.z; n.slot = slot; n.idx = i;
      const bool children = b.split && children_slot (p, n, false) >= 0;
      okeys[o] = vol_key (p, b.level, b.x, b.y, b.z);
      out[o] = vol_node (okeys[o], slot, i, children);
    }
  }
}

// the sorted nodes [first, first + n) as byte-packed records at out: each thread formats one record into shared memory, then
// the block copies its records out in one coalesced run
constexpr int VOL_FORMAT_THREADS = 256;
__global__ void __launch_bounds__ (VOL_FORMAT_THREADS) k_vol_format (Params gp, const VolNode* __restrict__ nodes, size_t first, size_t n,
                                                                      int rbytes, unsigned char* __restrict__ out)
{
  B2_STAGE_PARAMS (gp)
  __shared__ unsigned char buf[VOL_FORMAT_THREADS * 44];
  const size_t b0 = (size_t) blockIdx.x * VOL_FORMAT_THREADS;
  const size_t i = b0 + threadIdx.x;
  if (i < n) vol_format (p, nodes[first + i], buf + threadIdx.x * rbytes);
  __syncthreads ();
  const size_t m = min ((size_t) VOL_FORMAT_THREADS, n - b0) * (size_t) rbytes;
  unsigned char* o = out + b0 * rbytes;
  for (size_t k = threadIdx.x; k < m; k += VOL_FORMAT_THREADS) o[k] = buf[k];
}

// ---- .vol load on the device: one record per thread ----

// nchild - 1 of each record: the open-slot count after record i is 1 + the inclusive sum up to i
__global__ void k_vol_slots (const unsigned char* __restrict__ body, size_t nrec, int rbytes, long long* __restrict__ delta)
{
  const size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nrec) return;
  unsigned long long nchild;
  vol_get (body + i * rbytes + rbytes - 8, &nchild, 8);
  delta[i] = nchild == 8 ? 7 : -1;
}

// res[0] = the first record after which no slot is open (min over the records that close the tree)
__global__ void k_vol_end (const long long* __restrict__ incl, size_t nrec, unsigned long long* __restrict__ res)
{
  const size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nrec && incl[i] == -1) atomicMin (res, (unsigned long long) i);
}

// every check of records [0, n): res[1] = records that fail, res[2] = stored {d, w} outside the fast route's domain
__global__ void k_vol_check (Params gp, const unsigned char* __restrict__ body, size_t n, int rbytes, int rgb, unsigned long long* __restrict__ res)
{
  B2_STAGE_PARAMS (gp)
  const size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
  bool bad = false, out = false;
  if (i < n) bad = !vol_check_record (p, body, i, n, rbytes, rgb != 0, out);
  const unsigned mb = __ballot_sync (0xffffffffu, bad), mo = __ballot_sync (0xffffffffu, out);
  if ((threadIdx.x & 31) == 0)
  {
    if (mb) atomicAdd (res + 1, (unsigned long long) __popc (mb));
    if (mo) atomicAdd (res + 2, (unsigned long long) __popc (mo));
  }
}

// records [0, n), all checked, into the freshly reset volume: vol_place as the host loader places them
__global__ void k_vol_place (Params gp, const unsigned char* __restrict__ body, size_t n, int rbytes, int rgb)
{
  B2_STAGE_PARAMS (gp)
  const size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  vol_store (p, vol_parse (p, body + i * rbytes, rgb != 0));
}

} // namespace

// ---------------------------------------------------------------------------------------------
// handle
// ---------------------------------------------------------------------------------------------
// ---- pinned staging for the host-packed uploads ---------------------------------------------------------------
// The packing threads read the caller's points and write the staging while the copy engine reads the staging: when all of it
// sits behind ONE socket's memory controllers that socket can become the bottleneck (tools/microbench/pack_numa.cu compares
// the placements).  The staging is therefore interleaved over the NUMA nodes (mbind; best effort — a refusal leaves default
// placement) and then pinned with cudaHostRegister.
struct Staging
{
  unsigned char* p = nullptr; size_t bytes = 0;
  Staging () = default;
  Staging (const Staging&) = delete;
  Staging& operator= (const Staging&) = delete;
  ~Staging () { release (); }
  int alloc (size_t n)
  {
    release ();
    const size_t pg = 1ul << 21;                                     // (rounded to 2 MB: friendlier to transparent huge pages)
    n = (n + pg - 1) / pg * pg;
    void* m = mmap (nullptr, n, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (m == MAP_FAILED) return -1;
    unsigned long mask = 0;
    if (FILE* f = std::fopen ("/sys/devices/system/node/has_memory", "r"))
    {
      char line[256] = {};
      if (std::fgets (line, sizeof (line), f))
        for (const char* c = line; *c;)
        {
          char* e = nullptr; const long lo = std::strtol (c, &e, 10); if (e == c) break;
          long hi = lo; if (*e == '-') { const char* b = e + 1; hi = std::strtol (b, &e, 10); if (e == b) break; }
          for (long k = lo; k <= hi && k < 64; ++k) if (k >= 0) mask |= 1ul << k;
          c = e; if (*c == ',') ++c; else break;
        }
      std::fclose (f);
    }
    if (mask & (mask - 1)) (void) syscall (SYS_mbind, m, n, 3 /* MPOL_INTERLEAVE */, &mask, (unsigned long) (8 * sizeof (mask)), 0u);
    std::memset (m, 0, n);                                           // fault the pages in under that policy, before pinning
    if (cudaHostRegister (m, n, cudaHostRegisterDefault) != cudaSuccess) { cudaGetLastError (); munmap (m, n); return -1; }
    p = static_cast<unsigned char*> (m); bytes = n;
    return 0;
  }
  void release ()
  {
    if (!p) return;
    cudaHostUnregister (p); munmap (p, bytes);
    p = nullptr; bytes = 0;
  }
};

// The volume's device storage (the storage pointers of Params, see b200tsdf::storage_into) for one pool size, root-array size
// and payload; assigning a fresh Volume frees it
struct Volume
{
  size_t pool = 0, root_n = 0;
  bool color = false, var = false, norm = false;
  DevBuf<uint64_t> keys; DevBuf<float2> nodes; DevBuf<uint32_t> split; DevBuf<unsigned char> work;
  DevBuf<uchar4> rgb; DevBuf<float> M; DevBuf<int> ns; DevBuf<float4> rgbn;
  DevBuf<float2> root_dw; DevBuf<uint32_t> root_split; DevBuf<uchar4> root_rgb; DevBuf<float4> root_rgbn;
  DevBuf<float> root_M; DevBuf<int> root_ns;
};

constexpr int CELL_CAP = 16384;  // supercells of one frame on the supercell path (d_celltop; d_cellq holds 585 entries each)

struct b200tsdf
{
  // declared first, so that they are destroyed last: b200tsdf_destroy synchronises them and then frees everything below
  Stream stream, copy_stream, gather_stream;   // compute | H2D uploads | pack + NVLink all-gather
  b200tsdf_config cfg_pending{}, cfg{};
  bool has_volume = false;
  Params p{};
  int device = 0, sm_count = 0;            // cudaDevAttrMultiProcessorCount, read in b200tsdf_create
  Volume vol;
  DevBuf<int> d_err;
  DevBuf<unsigned char> d_frame[2];
  Event ev_copied[2], ev_consumed[2];
  Event ev_t0, ev_t1;
  uint64_t frame_no = 0;
  int count_set = 0;             // which of the two per-frame counter sets the last frame used
  DevBuf<int> d_culled; DevBuf<int> d_count; DevBuf<unsigned long long> d_stats;
  DevBuf<uint32_t> d_pix;        // Params::pix (grow-only)
  // change epochs (DESIGN.md §3g): every mutation advances `epoch`; the device stamps the cells it may touch in d_cell_epoch
  // (Params::cell_epoch, 8^C), and a change of the whole volume sets all_epoch instead.  d_cell_mask / d_cell_tris: the cell
  // selection and per-cell triangle counts of b200tsdf_mesh_cells_device.  All three are sized by reset() (grow-only).
  uint64_t epoch = 0, all_epoch = 0;
  DevBuf<unsigned long long> d_cell_epoch; DevBuf<unsigned char> d_cell_mask; DevBuf<unsigned long long> d_cell_tris;
  bool timed = false;
  bool time_frames = false;      // set between profile_begin / profile_end: per-frame event records (ev_t0/ev_t1 and the ring around the dominant kernel)
  bool is_empty = true;          // TSDFVolumeOctree::is_empty_ (cpp:205, hpp:101)
  bool loaded_on_device = false; // the last load placed its body with the device parser (b200tsdf_load_path)
  // fast-path work queues (levels C .. L-3), and the lists of block roots, BL_CLASSES lists of blist_cap () entries
  Queues Q{}; int q_levels = 0; DevBuf<QNode> q_mem;
  DevBuf<int> d_blist;
  int blist_cap () const { return (int) (d_blist.cap / BL_CLASSES); }
  // fused per-cell upper sweeps (coarse cells are the top-tier roots and the block roots are <= 3 levels below)
  // supercell path: sl = level of the tier-1 roots, nup = coarse levels above them (swept by k_upper_*), super_static = number of
  // supercells when every tier-1 root is one (coarse cells inside the brick)
  DevBuf<QNode> d_cellq; DevBuf<CellTop> d_celltop; DevBuf<QNode> d_superq;
  // the per-supercell gate of k_front (FoldState, brick_kernels.cuh): on the route whose supercells are the culled coarse cells
  // the fold marks, and the cell queue of frames with counter set 1 (Q.q[0] serves set 0)
  DevBuf<uint32_t> d_fold; DevBuf<QNode> d_q1;
  uint32_t frame_seq = 0;        // FrameRec::seq of the last frame
  bool fold_prev = false;        // the last frame's route published fold marks (the next one on that route may be gated)
  bool half_launched = false;    // a launch of a direct frame failed (part of it may be queued): calls refused until reset ()
  bool top_path = false; int sl = 0, nup = 0, super_static = 0;
  bool fast_path = false;
  // device copy of Params (the rare out-of-line paths read it through a pointer) and the ring of per-frame records
  DevBuf<Params> d_params;
  DevBuf<unsigned long long> d_dbg;        // phase-timing counters of k_celltop_up once b200tsdf_debug_timing armed them
  Pinned<int> h_err;                       // pinned image of the device error bits, refreshed behind every frame (see note_device_err)
  DevBuf<FrameRec> d_ring; Pinned<FrameRec> h_ring; uint64_t ring_seq = 0;
  Event ev_ring[2];
  // batches (b200tsdf_integrate_batch_device): their own record ring, used half by half, and one captured graph per
  // (half, batch size); a graph is valid until the next reset()
  // device slots: two halves of FRAME_RING / 2 records, reused in stream order; host staging: BATCH_SEGS segments written round
  // robin — the host only waits when it is BATCH_SEGS batches ahead of the device
  // (each half and each segment is BRING_SPAN slots: the frame records, then the organise block of an unorganised batch)
  DevBuf<FrameRec> d_bring; Pinned<FrameRec> h_bring; int bring_half = 0; int bring_seg = 0; bool bring_used[BATCH_SEGS] = {};
  Event ev_bring[BATCH_SEGS];
  Event ev_half_done[2]; bool half_used[2] = { false, false };
  cudaGraphExec_t batch_exec[2][FRAME_RING / 2 + 1] = {};
  cudaGraphExec_t unorg_exec[2][FRAME_RING / 2 + 1] = {};   // the same with the three organise launches in front
  cudaGraphExec_t depth_exec[2][FRAME_RING / 2 + 1] = {};   // the same with the depth unprojection in front
  // unorganised batches: the keys, filled counters and 16-byte organised images of one record half (organise and fuse of both
  // halves run on `stream`, so one set serves both); allocated at the first unorganised integrate, freed by reset()
  DevBuf<unsigned char> d_org;
  // depth frames from host memory (b200tsdf_integrate_depth): the caller's depth and colour are copied into one of
  // DEPTH_SLOTS pinned slots, uploaded on copy_stream into that slot's device buffer and unprojected from there.  A slot is
  // rewritten once its upload has run (ev_dcopied), its device buffer once the unprojection that read it has (ev_dconsumed).
  Staging h_depth[DEPTH_SLOTS]; DevBuf<unsigned char> d_depth_raw[DEPTH_SLOTS];
  Event ev_dcopied[DEPTH_SLOTS], ev_dconsumed[DEPTH_SLOTS];
  uint64_t depth_no = 0;
  // tracking (track.cuh): one block of inputs and state per call (pinned image and device copy), the per-tile sums of the
  // finest possible level, and one captured graph per (schedule shape, input kind), dropped with the batch graphs
  Pinned<TrackBlock> h_track; DevBuf<TrackBlock> d_track; DevBuf<double> d_track_part;
  struct TrackGraph { int key[10]; cudaGraphExec_t exec; };
  std::vector<TrackGraph> track_exec;
  // multi-GPU (multigpu.cuh): NCCL communicator (opaque here), row-sliced uploads
  void* comm = nullptr; int comm_rank = 0, comm_size = 1;
  DevBuf<unsigned char> d_rows_raw[2], d_rows_full[2];
  int rows_set = 0; bool rows_used[2] = { false, false }; int rows_last_up[2] = { 0, 0 };
  int rows_chunk = 0;            // frames per upload/fuse pipeline stage of b200tsdf_integrate_batch_rows (B200TSDF_ROWS_CHUNK=1..32; 0: 1 or 2 with host packing, else 8)
  Event ev_rows_up[2][32], ev_rows_ready[2][32], ev_rows_done[2];
  // host packing of the uploaded rows (host_pack.h): pinned staging per buffer set, the pool is created on first use
  int host_pack = -1;            // B200TSDF_HOST_PACK: 1 pack on the host, 0 upload the caller's points as they are (packed on the device when gathered); -1 by rank count
  int pack_threads = 0;          // B200TSDF_PACK_THREADS (0 = min (16, hardware threads / (2 ranks)))
  b2host::PackPool* pack_pool = nullptr;
  Staging h_pack[2];
  Staging h_fpack[2];            // the same for the frame-at-a-time upload (d_frame[]), as many bytes as each of d_frame[] holds
  long long nvlink_bytes = 0, prof_nvlink0 = 0;
  int launches_per_frame = 0; long long graph_launches = 0, prof_graph0 = 0;
  // measurement
  Event ev_p0, ev_p1;
  Event kring[KRING][2];
  int kring_head = 0, kring_pending = 0;
  double prof_ms_kernel = 0; long long prof_kernel_launches = 0, prof_frames = 0;
  long long launches = 0, prof_launch0 = 0, h2d_bytes = 0, d2h_bytes = 0, prof_h2d0 = 0, prof_d2h0 = 0;
  unsigned long long prof_stats0[ST_N] = {};
  void drain_kring (int keep)
  {
    while (kring_pending > keep)
    {
      int i = (kring_head - kring_pending + 4 * KRING) % KRING;
      float ms = 0.f;
      cudaEventSynchronize (kring[i][1]);
      if (cudaEventElapsedTime (&ms, kring[i][0], kring[i][1]) == cudaSuccess) { prof_ms_kernel += ms; prof_kernel_launches++; }
      kring_pending--;
    }
  }
  std::string err;
  void* mesh_v = nullptr; void* mesh_c = nullptr;           // b200tsdf_mesh results (malloc'ed)
  void* leaf_xyz = nullptr; void* leaf_ijk = nullptr;       // b200tsdf_voxel_centers / _occupied_voxel_indices results
  // grow-only device scratch for the read-side calls (queries, render): no allocation per call
  DevBuf<unsigned char> d_scratch;
  // render records (b200tsdf_render_batch_device): one device chunk, reused in stream order, and RENDER_SEGS pinned staging
  // segments written round robin, each free again once the copy that read it has run
  DevBuf<RenderParams> d_rrec; Pinned<RenderParams> h_rrec; int rrec_seg = 0; bool rrec_used[RENDER_SEGS] = {};
  Event ev_rrec[RENDER_SEGS];
  int scratch (size_t bytes)
  {
    if (bytes <= d_scratch.cap) return 0;
    if (d_scratch.grow (bytes + bytes / 2 + 4096)) return fail (B200TSDF_ENOMEM, "device scratch allocation failed");
    return 0;
  }
  // the device pointers of Params: the volume storage and the handle's buffers the kernels write
  void storage_into (Params& q) const
  {
    q.keys = vol.keys; q.nodes = vol.nodes; q.split = vol.split; q.work = vol.work;
    q.rgb = vol.rgb; q.M = vol.M; q.ns = vol.ns; q.rgbn = vol.rgbn;
    q.root_dw = vol.root_dw; q.root_split = vol.root_split; q.root_rgb = vol.root_rgb; q.root_rgbn = vol.root_rgbn;
    q.root_M = vol.root_M; q.root_ns = vol.root_ns;
    q.err = d_err; q.pix = d_pix; q.dbg = d_dbg; q.cell_epoch = d_cell_epoch;
  }
  void mark_all () { all_epoch = ++epoch; }   // a change of the whole volume: every cell counts as changed
  ~b200tsdf ();

  int fail (int code, const std::string& m) { err = m; return code; }
};

namespace {

// launch with programmatic stream serialization (see pdl_wait in brick_kernels.cuh); also valid inside a stream capture
template <typename... KArgs, typename... Args>
cudaError_t launch_pdl (void (*kernel) (KArgs...), dim3 grid, dim3 block, cudaStream_t s, const Args&... args)
{
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = 0; cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx (&cfg, kernel, KArgs (args)...);
}

void comm_release (b200tsdf* h);          // multigpu.cuh

void drop_track_graphs (b200tsdf* h)
{
  for (auto& g : h->track_exec) cudaGraphExecDestroy (g.exec);
  h->track_exec.clear ();
}

void drop_batch_graphs (b200tsdf* h)
{
  for (int a = 0; a < 2; ++a)
    for (int n = 0; n <= FRAME_RING / 2; ++n)
    {
      if (h->batch_exec[a][n]) { cudaGraphExecDestroy (h->batch_exec[a][n]); h->batch_exec[a][n] = nullptr; }
      if (h->unorg_exec[a][n]) { cudaGraphExecDestroy (h->unorg_exec[a][n]); h->unorg_exec[a][n] = nullptr; }
      if (h->depth_exec[a][n]) { cudaGraphExecDestroy (h->depth_exec[a][n]); h->depth_exec[a][n] = nullptr; }
    }
  drop_track_graphs (h);
}

int check_device_err (b200tsdf* h)
{
  int e = 0;
  if (cudaMemcpyAsync (&e, h->d_err, sizeof (int), cudaMemcpyDeviceToHost, h->stream) != cudaSuccess) return h->fail (B200TSDF_ECUDA, "error flag readback failed");
  if (cudaStreamSynchronize (h->stream) != cudaSuccess) return h->fail (B200TSDF_ECUDA, std::string ("stream: ") + cudaGetErrorString (cudaGetLastError ()));
  if (e & ERR_POOL_FULL) return h->fail (B200TSDF_ENOMEM, "brick pool exhausted (raise pool_log2)");
  if (e & ERR_MISSING_BRICK) return h->fail (B200TSDF_ESTATE, "internal: split node without brick");
  if (e & ERR_QUEUE_FULL) return h->fail (B200TSDF_ENOMEM, "internal: work queue overflow");
  if (e & ERR_FOLD_WAIT) return h->fail (B200TSDF_ESTATE, "internal: k_front waited too long for the previous frame's fold");
  return 0;
}

// Deferred error reporting for the calls that do not wait for their kernels: a 4-byte copy of the (sticky) device error bits
// into pinned memory is queued behind the work, and every entry point looks at the pinned word first.  An overflow
// (pool, queue) or an inconsistency is therefore reported by the call that follows the frame which hit it, at the latest
// by b200tsdf_sync / get_stats / mesh / save, instead of being served silently (ADVICE r1).
int pending_device_err (b200tsdf* h)
{
  if (h->half_launched) return h->fail (B200TSDF_ESTATE, "an earlier frame was left half launched by a CUDA error; reset() the handle");
  const int e = *(volatile int*) h->h_err;
  if (!e) return 0;
  if (e & ERR_POOL_FULL) return h->fail (B200TSDF_ENOMEM, "brick pool exhausted in an earlier frame (raise pool_log2); the volume is incomplete");
  if (e & ERR_MISSING_BRICK) return h->fail (B200TSDF_ESTATE, "internal: split node without brick (earlier frame)");
  if (e & ERR_FOLD_WAIT) return h->fail (B200TSDF_ESTATE, "internal: k_front waited too long for the previous frame's fold (earlier frame)");
  return h->fail (B200TSDF_ENOMEM, "internal: work queue overflow in an earlier frame; the volume is incomplete");
}
void note_device_err (b200tsdf* h, cudaStream_t s) { cudaMemcpyAsync (h->h_err, h->d_err, sizeof (int), cudaMemcpyDeviceToHost, s); }

void fill_frame (const b200tsdf* h, Frame& f, const unsigned char* d_pts, size_t stride, int xyz_off, int rgba_off, int W, int H, const double* pose)
{
  f.pts = d_pts; f.stride = (int) stride; f.xyz_off = xyz_off; f.rgba_off = h->p.color ? rgba_off : -1; f.width = W; f.height = H;
  double inv[12];
  b2host::affine_inverse (pose, inv);                                 // hpp:54: trans.inverse ().cast<float> ()
  for (int i = 0; i < 12; ++i) { f.tinv[i] = (float) inv[i]; f.tfwd[i] = (float) pose[i]; }
}

// The claimed brick slots, listed into the handle's grow-only scratch.  Returns their number, or a B200TSDF_ error (< 0).
// The list lives until the next use of the scratch.
int list_bricks (b200tsdf* h, int*& list)
{
  if (int rc = h->scratch (h->vol.pool * sizeof (int))) return rc;
  list = (int*) h->d_scratch.p;
  int* d_n = h->d_count + 40;
  cudaStream_t s = h->stream;
  CK (cudaMemsetAsync (d_n, 0, sizeof (int), s));
  k_list_bricks<<<(unsigned) ((h->vol.pool + 255) / 256), 256, 0, s>>> (h->p, list, d_n);
  int nb = 0;
  CK (cudaMemcpyAsync (&nb, d_n, sizeof (int), cudaMemcpyDeviceToHost, s));
  CK (cudaStreamSynchronize (s));
  return nb;
}

// A failed device allocation is reported as B200TSDF_ENOMEM; the runtime's last error is cleared so that no later call
// reports it.
int alloc_failed (b200tsdf* h, const std::string& what)
{
  cudaGetLastError ();
  return h->fail (B200TSDF_ENOMEM, "device allocation failed (" + what + ")");
}

// Every brick slot of the pool q points at (pool slots) fresh, by the invariant of tsdf_core.cuh (OctreeNode ctor: d=-1, w=0;
// octree.h:71-74): no key, no split bit, zero colour / variance payload and work byte.  Enqueued on the handle's stream.
int fresh_pool (b200tsdf* h, const Params& q, size_t pool)
{
  cudaStream_t s = h->stream;
  const size_t nn = pool * BRICK_NODES;
  CK (cudaMemsetAsync (q.keys, 0, pool * sizeof (uint64_t), s));
  CK (cudaMemsetAsync (q.split, 0, pool * BRICK_SPLIT_WORDS * sizeof (uint32_t), s));
  CK (cudaMemsetAsync (q.work, 0, pool, s));
  k_fill_fresh<<<h->sm_count * 8, 256, 0, s>>> (q.nodes, nn);
  if (q.rgb) CK (cudaMemsetAsync (q.rgb, 0, nn * sizeof (uchar4), s));
  if (q.M) { CK (cudaMemsetAsync (q.M, 0, nn * sizeof (float), s)); CK (cudaMemsetAsync (q.ns, 0, nn * sizeof (int), s)); }
  if (q.rgbn) CK (cudaMemsetAsync (q.rgbn, 0, nn * sizeof (float4), s));
  return B200TSDF_OK;
}

// `bytes` of device memory into `host` (reallocated with malloc, at least one byte), after the work queued before them
int download (b200tsdf* h, const void* d, size_t bytes, void*& host)
{
  std::free (host);
  host = std::malloc (std::max<size_t> (bytes, 1));
  if (!host) return h->fail (B200TSDF_ENOMEM, "host allocation failed");
  if (bytes) CK (cudaMemcpyAsync (host, d, bytes, cudaMemcpyDeviceToHost, h->stream));
  CK (cudaStreamSynchronize (h->stream));
  CK (cudaGetLastError ());
  return B200TSDF_OK;
}

// The enumeration behind marching cubes and getLeaves, in the reference's depth-first order.  launch (emit, total, keys, v, c)
// enqueues the caller's kernels: with emit = std::false_type they add their record count to *total, with std::true_type they
// also write their records at the slots they reserve, with the order key of each in keys.  A record is `words` 32-bit words
// in v, plus `words` bytes in c.  The records are counted; then dest (count, v_out, c_out) names the device buffers that
// receive them (v_out: count * words words; c_out: count * words bytes, or null for no colour bytes), or leaves v_out null
// to stop after the count, or returns an error.  Otherwise the records are emitted into device buffers of exactly that size
// and sorted by the low key_bits of their keys straight into v_out / c_out.  A failed allocation returns B200TSDF_ENOMEM.
template <typename Launch, typename Dest>
int sorted_records (b200tsdf* h, const char* what, int words, int key_bits, const Launch& launch, const Dest& dest,
                    unsigned long long& count)
{
  cudaStream_t s = h->stream;
  unsigned long long* d_total = h->d_stats + ST_SCRATCH;
  count = 0;
  CK (cudaMemsetAsync (d_total, 0, sizeof (count), s));
  launch (std::false_type (), d_total, nullptr, nullptr, nullptr);
  CK (cudaMemcpyAsync (&count, d_total, sizeof (count), cudaMemcpyDeviceToHost, s));
  CK (cudaStreamSynchronize (s));
  void* v_out = nullptr; unsigned char* c_out = nullptr;
  if (int rc = dest (count, v_out, c_out)) return rc;
  if (!count || !v_out) return B200TSDF_OK;
  const size_t nw = (size_t) count * words, nc = c_out ? nw : 0;
  DevBuf<uint32_t> v (s); DevBuf<unsigned char> c (s); DevBuf<unsigned long long> k (s);
  if (v.alloc (nw) || c.alloc (nc) || k.alloc (count)) return alloc_failed (h, what);
  CK (cudaMemsetAsync (d_total, 0, sizeof (count), s));
  launch (std::true_type (), d_total, k, v, c);
  const int e = b2_sort_records (s, (size_t) count, key_bits, k, words, v, c, v_out, c_out);
  if (e == (int) cudaErrorMemoryAllocation) return alloc_failed (h, std::string (what) + " sort");
  if (e) return h->fail (B200TSDF_ECUDA, std::string (what) + " sort: " + cudaGetErrorString ((cudaError_t) e));
  return B200TSDF_OK;
}

// sorted_records into library-owned host memory: the records are sorted into device buffers of their exact size and copied
// into host_v / *host_c (see download; host_c == null: no colour bytes)
template <typename Launch>
int sorted_records_host (b200tsdf* h, const char* what, int words, int key_bits, const Launch& launch,
                         void*& host_v, void** host_c, unsigned long long& count)
{
  DevBuf<uint32_t> v2 (h->stream); DevBuf<unsigned char> c2 (h->stream);
  auto dest = [&] (unsigned long long n, void*& v_out, unsigned char*& c_out)
  {
    if (!n) return (int) B200TSDF_OK;
    if (v2.alloc ((size_t) n * words) || (host_c && c2.alloc ((size_t) n * words))) return alloc_failed (h, what);
    v_out = v2; c_out = c2;
    return (int) B200TSDF_OK;
  };
  if (int rc = sorted_records (h, what, words, key_bits, launch, dest, count)) return rc;
  const size_t nw = (size_t) count * words;
  if (int rc = download (h, v2, nw * 4, host_v)) return rc;
  return host_c ? download (h, c2, nw, *host_c) : B200TSDF_OK;
}

bool create_events (Event* e, int n, unsigned flags)
{
  for (int i = 0; i < n; ++i)
    if (cudaEventCreateWithFlags (&e[i].x, flags) != cudaSuccess) return false;
  return true;
}

} // namespace

b200tsdf::~b200tsdf ()
{
  drop_batch_graphs (this);
  delete pack_pool;
  std::free (mesh_v); std::free (mesh_c); std::free (leaf_xyz); std::free (leaf_ijk);
}

extern "C" {

void b200tsdf_default_config (b200tsdf_config* c) { if (c) default_config (c); }

int b200tsdf_create (const b200tsdf_config* cfg, b200tsdf_t** out)
{
  if (!out) return B200TSDF_EINVAL;
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount (&ndev) != cudaSuccess || ndev == 0) return B200TSDF_ENODEVICE;
  b200tsdf* h = new b200tsdf;
  if (cfg) h->cfg_pending = *cfg; else b200tsdf_default_config (&h->cfg_pending);
  h->device = h->cfg_pending.device;
  if (const char* e = std::getenv ("B200TSDF_ROWS_CHUNK")) { const int v = std::atoi (e); if (v >= 1 && v <= 32) h->rows_chunk = v; }
  if (const char* e = std::getenv ("B200TSDF_HOST_PACK")) h->host_pack = std::atoi (e) != 0 ? 1 : 0;
  if (const char* e = std::getenv ("B200TSDF_PACK_THREADS")) { const int v = std::atoi (e); if (v >= 1 && v <= 256) h->pack_threads = v; }
  if (h->device < 0 || h->device >= ndev) { delete h; return B200TSDF_EINVAL; }
  const unsigned nt = cudaEventDisableTiming;
  bool ok = cudaSetDevice (h->device) == cudaSuccess
         && cudaDeviceGetAttribute (&h->sm_count, cudaDevAttrMultiProcessorCount, h->device) == cudaSuccess
         && cudaStreamCreateWithFlags (&h->stream.x, cudaStreamNonBlocking) == cudaSuccess
         && cudaStreamCreateWithFlags (&h->copy_stream.x, cudaStreamNonBlocking) == cudaSuccess
         && cudaStreamCreateWithFlags (&h->gather_stream.x, cudaStreamNonBlocking) == cudaSuccess
         && !h->d_err.grow (1) && !h->d_count.grow (64) && !h->d_stats.grow (ST_TOTAL) && !h->d_params.grow (1)
         && !h->d_ring.grow (FRAME_RING) && !h->d_bring.grow (2 * BRING_SPAN) && !h->d_rrec.grow (RENDER_CHUNK)
         && !h->h_err.alloc (1) && !h->h_ring.alloc (FRAME_RING) && !h->h_bring.alloc ((size_t) BATCH_SEGS * BRING_SPAN)
         && !h->h_rrec.alloc ((size_t) RENDER_SEGS * RENDER_CHUNK)
         && create_events (h->ev_ring, 2, nt) && create_events (h->ev_rows_done, 2, nt) && create_events (h->ev_bring, BATCH_SEGS, nt)
         && create_events (h->ev_half_done, 2, nt) && create_events (h->ev_copied, 2, nt) && create_events (h->ev_consumed, 2, nt)
         && create_events (h->ev_dcopied, DEPTH_SLOTS, nt) && create_events (h->ev_dconsumed, DEPTH_SLOTS, nt)
         && create_events (h->ev_rrec, RENDER_SEGS, nt) && create_events (&h->ev_rows_ready[0][0], 64, nt) && create_events (&h->ev_rows_up[0][0], 64, nt)
         && create_events (&h->ev_t0, 1, cudaEventDefault) && create_events (&h->ev_t1, 1, cudaEventDefault)
         && create_events (&h->ev_p0, 1, cudaEventDefault) && create_events (&h->ev_p1, 1, cudaEventDefault)
         && create_events (&h->kring[0][0], 2 * KRING, cudaEventDefault);
  if (!ok) { delete h; return B200TSDF_ECUDA; }
  *h->h_err = 0;
  cudaMemset (h->d_err, 0, sizeof (int)); cudaMemset (h->d_stats, 0, ST_TOTAL * sizeof (unsigned long long));
  // the depth-first general path recurses up to (L - C + 1) levels
  cudaDeviceSetLimit (cudaLimitStackSize, 16384);
  *out = h;
  return B200TSDF_OK;
}

void b200tsdf_destroy (b200tsdf_t* h)
{
  if (!h) return;
  cudaSetDevice (h->device);
  if (h->stream) cudaStreamSynchronize (h->stream);
  if (h->copy_stream) cudaStreamSynchronize (h->copy_stream);
  if (h->gather_stream) cudaStreamSynchronize (h->gather_stream);
  comm_release (h);
  delete h;
}

const char* b200tsdf_last_error (const b200tsdf_t* h) { return h ? h->err.c_str () : "null handle"; }

int b200tsdf_set_config (b200tsdf_t* h, const b200tsdf_config* cfg)
{
  if (!h || !cfg) return B200TSDF_EINVAL;
  int dev = h->cfg_pending.device;
  const b200tsdf_config before = h->cfg_pending;
  h->cfg_pending = *cfg;
  h->cfg_pending.device = dev;               // a handle is bound to its device at creation
  if (std::memcmp (&before, &h->cfg_pending, sizeof (before))) h->mark_all ();
  // setGlobalTransform is the one setter that does not wait for reset () in the reference: global_transform_ is only read by
  // save () and the mesher (tsdf_volume_octree.h:131-133, cpp:242, marching_cubes_tsdf_octree.cpp:122-128)
  std::memcpy (h->cfg.global_transform, cfg->global_transform, sizeof (h->cfg.global_transform));
  return B200TSDF_OK;
}

int b200tsdf_get_config (const b200tsdf_t* h, b200tsdf_config* cfg)
{
  if (!h || !cfg) return B200TSDF_EINVAL;
  *cfg = h->cfg_pending;
  return B200TSDF_OK;
}

// ---- reset (tsdf_volume_octree.cpp:201-219, Octree::init octree.cpp:584-599) --------------------
// The integrate route of configuration np: which kernels fuse a frame, and the capacities of their work queues (Q.cap; reset
// installs the queues once their memory is allocated)
static void choose_route (b200tsdf* h, const Params& np, int debug_flags)
{
  // work queues for levels C .. B = L-3 (fast path needs the block-root level at or below the coarse depth)
  // the brick kernels divide with div_recip / div_with, which equal __fdiv_rn only inside Params::exact_div_ok; other
  // truncation limits and weight caps are fused by the general depth-first kernel, which uses the IEEE division
  const int Bl = np.L - 3;
  h->fast_path = (Bl >= np.C) && !np.track_var && !np.color_norm && !(debug_flags & 1) && np.exact_div_ok && (Bl - np.C + 1 <= MAX_QLEVELS);
  h->q_levels = h->fast_path ? (Bl - np.C + 1) : 0;
  h->Q = Queues {};
  for (int i = 0; i < h->q_levels; ++i) h->Q.cap[i] = np.C + i >= 7 ? 1 << 21 : 1 << (3 * (np.C + i));
  // supercell path (k_celltop_down / k_bricks / k_celltop_up, brick_kernels.cuh): needs tier-1 bricks (T >= 2), whose roots sit
  // at level SL = L - 6.  Coarse levels above SL are swept by k_upper_*; coarse cells below SL are handled inside the brick.
  h->sl = np.L - 6;
  h->nup = std::max (0, h->sl - np.C);
  h->super_static = 0;
  h->top_path = h->fast_path && np.T >= 2 && h->sl >= 0 && !(debug_flags & 2);
  if (h->top_path && np.C > h->sl)
  {
    // every tier-1 root is a supercell; they must be the root-array nodes (T == 2) and fit the per-cell scratch
    if (np.Rtop != h->sl || h->sl > 4) h->top_path = false;
    else h->super_static = 1 << (3 * h->sl);
  }
}

int b200tsdf_reset (b200tsdf_t* h)
{
  if (!h) return B200TSDF_EINVAL;
  cudaSetDevice (h->device);
  const b200tsdf_config& c = h->cfg_pending;
  Params np = h->p;
  size_t pool = 0, root_n = 0;
  if (const char* msg = derive_params (c, np, pool, root_n)) return h->fail (B200TSDF_EINVAL, msg);
  const bool color = np.color != 0, var = np.track_var != 0, norm = np.color_norm != 0;

  // from here on a failure leaves the handle without a volume until a reset succeeds
  h->has_volume = false;
  CK (cudaStreamSynchronize (h->stream));
  CK (cudaStreamSynchronize (h->copy_stream));
  drop_batch_graphs (h);                                   // captured launches carry the old configuration
  h->d_org.release ();                                     // (sized by the old image size; the graphs that used it are gone)
  for (int i = 0; i < BATCH_SEGS; ++i) h->bring_used[i] = false;
  h->half_used[0] = h->half_used[1] = false;
  choose_route (h, np, c.debug_flags);
  const bool fold = h->top_path && h->sl == np.C;          // publishes_folds of the new route

  Volume& v = h->vol;
  if (pool != v.pool || root_n != v.root_n || color != v.color || var != v.var || norm != v.norm)
  {
    v = {};                                                // (the old storage is freed before the new one is allocated)
    const size_t nn = pool * BRICK_NODES;
    if (v.keys.grow (pool) || v.nodes.grow (nn) || v.split.grow (pool * BRICK_SPLIT_WORDS) || v.work.grow (pool)
        || (color && v.rgb.grow (nn)) || (var && (v.M.grow (nn) || v.ns.grow (nn)))
        || v.root_dw.grow (root_n) || v.root_split.grow ((root_n + 31) / 32) || (color && v.root_rgb.grow (root_n))
        || (norm && (v.rgbn.grow (nn) || v.root_rgbn.grow (root_n))) || (var && (v.root_M.grow (root_n) || v.root_ns.grow (root_n))))
      return alloc_failed (h, "volume storage");
    v.pool = pool; v.root_n = root_n; v.color = color; v.var = var; v.norm = norm;
  }
  size_t q_total = 0;
  for (int i = 0; i < h->q_levels; ++i) q_total += (size_t) h->Q.cap[i];
  size_t bl = h->q_levels ? (size_t) h->Q.cap[h->q_levels - 1] : 0;
  if (h->top_path) bl = std::max (bl, (size_t) CELL_CAP * 512);
  if (h->d_culled.grow ((size_t) 1 << (3 * np.C))
      || h->d_pix.grow (2 * (size_t) np.width * np.height * (color ? 2 : 1))    // two planes alternate by counter set (frame_plane)
      || h->q_mem.grow (q_total)
      || h->d_blist.grow (bl * BL_CLASSES)                                      // one list per work class
      || (h->top_path && (h->d_cellq.grow ((size_t) CELL_CAP * 585) || h->d_celltop.grow (CELL_CAP)))
      || (h->super_static && h->d_superq.grow (4096))
      || (fold && (h->d_fold.grow (fold_words (np.C)) || h->d_q1.grow ((size_t) h->Q.cap[0]))))
    return alloc_failed (h, "work queues");
  const size_t ncells = (size_t) 1 << (3 * np.C);
  if (h->d_cell_epoch.grow (ncells) || h->d_cell_mask.grow (ncells) || h->d_cell_tris.grow (ncells))
    return alloc_failed (h, "cell epochs");

  // install the configuration
  Params& p = h->p;
  p = np;
  h->storage_into (p);
  h->Q.n = h->d_count;
  for (size_t i = 0, off = 0; i < (size_t) h->q_levels; off += (size_t) h->Q.cap[i++]) h->Q.q[i] = h->q_mem + off;
  CK (cudaMemcpyAsync (h->d_params, &p, sizeof (Params), cudaMemcpyHostToDevice, h->stream));
  CK (cudaStreamSynchronize (h->stream));                            // (&p is host memory that may change after reset)
  // fresh state everywhere (OctreeNode ctor: d=-1, w=0; octree.h:71-74)
  cudaStream_t s = h->stream;
  if (int rc = fresh_pool (h, p, pool)) return rc;
  k_fill_fresh<<<64, 256, 0, s>>> (p.root_dw, root_n);
  CK (cudaMemsetAsync (p.root_split, 0, ((root_n + 31) / 32) * sizeof (uint32_t), s));
  if (color) CK (cudaMemsetAsync (p.root_rgb, 0, root_n * sizeof (uchar4), s));
  if (norm) CK (cudaMemsetAsync (p.root_rgbn, 0, root_n * sizeof (float4), s));
  if (var) { CK (cudaMemsetAsync (p.root_M, 0, root_n * sizeof (float), s)); CK (cudaMemsetAsync (p.root_ns, 0, root_n * sizeof (int), s)); }
  CK (cudaMemsetAsync (h->d_err, 0, sizeof (int), s));
  *h->h_err = 0;
  CK (cudaMemsetAsync (h->d_count, 0, 64 * sizeof (int), s));
  h->count_set = 0;
  if (h->d_fold) CK (cudaMemsetAsync (h->d_fold, 0, h->d_fold.cap * sizeof (uint32_t), s));
  h->fold_prev = false;
  h->half_launched = false;
  CK (cudaMemsetAsync (h->d_stats, 0, ST_TOTAL * sizeof (unsigned long long), s));
  CK (cudaMemsetAsync (h->d_cell_epoch, 0, ncells * sizeof (unsigned long long), s));
  h->mark_all ();
  h->kring_pending = 0; h->kring_head = 0;
  if (np.Rtop < np.C) k_insert_top_bricks<<<(unsigned) ((root_n + 127) / 128), 128, 0, s>>> (p);
  if (h->top_path && h->super_static) k_build_superq<<<(h->super_static + 127) / 128, 128, 0, s>>> (p, h->d_superq, h->super_static);
  CK (cudaGetLastError ());
  h->cfg = c;
  h->frame_no = 0;
  h->timed = false;
  h->is_empty = true;
  h->loaded_on_device = false;
  h->has_volume = true;
  return check_device_err (h);
}

// ---- resizing the brick pool of a live volume (DESIGN.md §3f) ----------------------------------------
// Every claimed brick is rehashed into a fresh pool of the new size, next to the old one, which is freed only once the new one
// holds every brick.  Like reset (), the handle takes the new storage in one step at the end: a refusal or a failed allocation
// leaves it as it was.
int b200tsdf_resize_pool (b200tsdf_t* h, int pool_log2)
{
  if (!h) return B200TSDF_EINVAL;
  cudaSetDevice (h->device);
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "resize_pool before reset()");
  CK (cudaStreamSynchronize (h->copy_stream));
  CK (cudaStreamSynchronize (h->gather_stream));
  int e = 0;
  CK (cudaMemcpyAsync (&e, h->d_err, sizeof (int), cudaMemcpyDeviceToHost, h->stream));
  CK (cudaStreamSynchronize (h->stream));
  if (e || h->half_launched)
    return h->fail (B200TSDF_ESTATE, "resize_pool on a volume with an error latched by an earlier call; reset() the handle");
  const size_t pool = pool_capacity_of (pool_log2);
  if (!pool) return h->fail (B200TSDF_EINVAL, "pool_log2 out of range [8,26]");
  int* list = nullptr;
  const int nb = list_bricks (h, list);
  if (nb < 0) return nb;
  if (!rehash_fits (nb, (long long) pool))
    return h->fail (B200TSDF_EINVAL, "resize_pool: " + std::to_string (nb) + " bricks do not fit a pool of " + std::to_string (pool)
                                     + " at the load limit of 7/8");

  // the new pool, fresh, beside the old one
  const Volume& v = h->vol;
  Volume nv;
  const size_t nn = pool * BRICK_NODES;
  if (nv.keys.grow (pool) || nv.nodes.grow (nn) || nv.split.grow (pool * BRICK_SPLIT_WORDS) || nv.work.grow (pool)
      || (v.color && nv.rgb.grow (nn)) || (v.var && (nv.M.grow (nn) || nv.ns.grow (nn))) || (v.norm && nv.rgbn.grow (nn)))
    return alloc_failed (h, "resized brick pool");
  DevBuf<int> d_rerr (h->stream);                      // the rehash's own error bits: the handle's d_err stays as it is
  if (d_rerr.grow (1)) return alloc_failed (h, "resize_pool error flag");
  Params to = h->p;
  to.keys = nv.keys; to.nodes = nv.nodes; to.split = nv.split; to.work = nv.work;
  to.rgb = nv.rgb; to.M = nv.M; to.ns = nv.ns; to.rgbn = nv.rgbn;
  to.pool_mask = (uint32_t) (pool - 1);
  to.err = d_rerr;
  cudaStream_t s = h->stream;
  if (int rc = fresh_pool (h, to, pool)) return rc;
  CK (cudaMemsetAsync (d_rerr, 0, sizeof (int), s));
  if (nb) k_pool_rehash<<<(unsigned) ((nb + REHASH_THREADS / 32 - 1) / (REHASH_THREADS / 32)), REHASH_THREADS, 0, s>>> (h->p, to, list, nb);
  CK (cudaGetLastError ());
  int re = 0;
  CK (cudaMemcpyAsync (&re, d_rerr, sizeof (int), cudaMemcpyDeviceToHost, s));
  CK (cudaStreamSynchronize (s));
  if (re & ERR_POOL_FULL)
    return h->fail (B200TSDF_EINVAL, "resize_pool: a brick found no slot within the probe limit of the new pool; the volume is unchanged");

  // install: the new pool with the old root arrays; the old pool is freed with nv
  nv.root_dw = std::move (h->vol.root_dw); nv.root_split = std::move (h->vol.root_split); nv.root_rgb = std::move (h->vol.root_rgb);
  nv.root_rgbn = std::move (h->vol.root_rgbn); nv.root_M = std::move (h->vol.root_M); nv.root_ns = std::move (h->vol.root_ns);
  nv.pool = pool; nv.root_n = v.root_n; nv.color = v.color; nv.var = v.var; nv.norm = v.norm;
  std::swap (h->vol, nv);
  drop_batch_graphs (h);                                   // captured launches carry the old storage in their Params
  h->storage_into (h->p);
  h->p.pool_mask = to.pool_mask;
  h->cfg.pool_log2 = h->cfg_pending.pool_log2 = pool_log2 > 0 ? pool_log2 : 20;
  if (cudaMemcpyAsync (h->d_params, &h->p, sizeof (Params), cudaMemcpyHostToDevice, s) != cudaSuccess || cudaStreamSynchronize (s) != cudaSuccess)
  {
    h->has_volume = false;
    return h->fail (B200TSDF_ECUDA, std::string ("resize_pool: installing the new pool failed: ") + cudaGetErrorString (cudaGetLastError ()));
  }
  return B200TSDF_OK;
}

// ---- integrateCloud (hpp:48-103) ------------------------------------------------------------------
// The route whose kernels publish the fold marks of FoldState (brick_kernels.cuh), and whose k_front may therefore wait per
// supercell: the supercells are the culled coarse cells (C == SL, no k_upper_* levels) and the frame's last kernel is
// k_celltop_up.  Other routes wait for the previous frame's last kernel before any octree work.  It follows the handle's
// current route, including the switch to the general kernel after out-of-domain writes.
static bool publishes_folds (const b200tsdf* h) { return h->fast_path && h->top_path && h->sl == h->p.C; }

// The frame's parameters (pose, planes, cloud pointer, counter set) are written into a FrameRec; the hot kernels
// read it from the device ring, so the very same launches can be captured once into a CUDA graph and replayed.
static void fill_rec (b200tsdf* h, FrameRec& r, const unsigned char* d_pts, size_t stride, int xyz_off, int rgba_off, int W, int H, const double* pose)
{
  const Params& p = h->p;
  fill_frame (h, r.f, d_pts, stride, xyz_off, rgba_off, W, H, pose);
  b2host::frustum_planes (pose, p.width, p.height, p.fx, p.fy, p.min_sensor, p.max_sensor, r.pl);
  h->count_set ^= 1;                                                  // counter sets alternate between frames
  r.cset = h->count_set;
  r.timing = h->time_frames ? 1 : 0;
  r.seq = ++h->frame_seq;
  r.epoch = ++h->epoch;
  const bool pub = publishes_folds (h);
  r.gated = pub && h->fold_prev;                                      // (the previous frame's kernels publish the marks it waits on)
  h->fold_prev = pub;
  r.kt[0] = r.kt[1] = 0;
}

// The numbering fill_rec gives frames (seq, counter set, gate) becomes the handle's only once they are enqueued: a call that
// fails before that puts it back on return, so that the next frame is numbered and gated as if the failed ones had never been
// filled.  (A gated k_front waits for `opened == seq - 1`, which a frame that was numbered but never launched would not publish.)
// Every argument is checked before the first fill_rec, so only a CUDA error can still fail here.  A launch that fails inside
// launch_frame outside a graph may leave part of that frame on the stream: integrate_on_device then latches half_launched, so
// that every later call that would queue work on the handle returns B200TSDF_ESTATE until reset (), which starts the numbering
// afresh (counter set 0, no gate, fold marks cleared).
struct FrameNumbering
{
  b200tsdf* h; uint32_t seq; int cset; bool fold_prev; uint64_t epoch; bool enqueued = false;
  explicit FrameNumbering (b200tsdf* h_) : h (h_), seq (h_->frame_seq), cset (h_->count_set), fold_prev (h_->fold_prev), epoch (h_->epoch) {}
  ~FrameNumbering () { if (!enqueued) { h->frame_seq = seq; h->count_set = cset; h->fold_prev = fold_prev; h->epoch = epoch; } }
};

// the launches of one frame; every kernel reads the frame from *d_rec, so the launches can be captured and replayed.
// with_events: bracket the dominant kernel with an event pair of the ring (never inside a capture)
// front_pdl: k_front reads the frame's cloud before its griddepcontrol.wait, so it may only overlap the kernel before it when
// that kernel did not write the cloud.  After the organise launches of an unorganised batch it is a plain launch (a full
// dependency on the gather that wrote the images).
static int launch_frame (b200tsdf* h, cudaStream_t s, const FrameRec* d_rec, bool with_events, bool front_pdl = true)
{
  const Params& p = h->p;
  const int npix = h->cfg.image_width * h->cfg.image_height;   // (every frame has this size: check_cloud_layout)
  const int ncells = 1 << (3 * p.C);
  // on the route that publishes fold marks, frames alternate between two cell queues (k_front fills the next frame's while
  // this frame's k_celltop_up still reads its own); other routes use Q.q[0] for both counter sets
  const bool pub = publishes_folds (h);
  uint32_t* const fold = pub ? h->d_fold.p : nullptr;
  QNode* const q1 = pub ? h->d_q1 : h->Q.q[0];
  {
    const int cull_blocks = (ncells + 255) / 256;
    const dim3 grid (cull_blocks + (npix + 255) / 256);
    if (front_pdl) CK (launch_pdl (k_front, grid, dim3 (256), s, p, d_rec, cull_blocks, h->d_culled, h->d_count, h->Q.q[0], q1, fold, h->d_stats));
    else k_front<<<grid, 256, 0, s>>> (p, d_rec, cull_blocks, h->d_culled, h->d_count, h->Q.q[0], q1, fold, h->d_stats);
  }
  h->launches += 1;
  int kr = -1;
  if (with_events)
  {
    if (h->kring_pending >= KRING) h->drain_kring (KRING / 2);
    kr = h->kring_head;
  }
  if (h->fast_path)
  {
    const int nl = h->q_levels;
    QNode* bq = nullptr;                                   // the queue the block-root entries of k_bricks live in
    if (h->top_path)
    {
      // coarse levels above the supercells, top-down (none for 2048^3 / 10 m and 512^3 / 3 m)
      for (int li = 0; li < h->nup; ++li) { k_upper_down<<<h->sm_count * 2, 128, 0, s>>> (p, d_rec, h->Q, li, 0, h->d_blist, h->d_stats); h->launches++; }
      QNode* cells = h->super_static ? h->d_superq : h->Q.q[h->nup];
      const int qslot = h->super_static ? -1 : h->nup;
      auto kd = p.color ? k_celltop_down<true> : k_celltop_down<false>;
      CK (launch_pdl (kd, dim3 (h->sm_count * 4), dim3 (TOP_THREADS), s, p, d_rec, cells, pub ? q1 : cells, h->d_count, h->d_cellq, h->d_celltop, CELL_CAP, h->d_blist, h->blist_cap (), h->d_stats, h->sl, qslot, h->super_static, fold));
      h->launches++;
      bq = h->d_cellq;
    }
    else
    {
      for (int li = 0; li < nl; ++li) { k_upper_down<<<h->sm_count * 2, 128, 0, s>>> (p, d_rec, h->Q, li, li == nl - 1, h->d_blist, h->d_stats); h->launches++; }
      bq = h->Q.q[nl - 1];
    }
    if (kr >= 0) CK (cudaEventRecord (h->kring[kr][0], s));
    // the dominant kernel: one warp per interior block root, the brick updated in place
    {
      auto kb = p.color ? k_bricks<true> : k_bricks<false>;
      const dim3 g (h->sm_count * BD_CTAS), b (BD_WARPS * 32);
      if (h->top_path) CK (launch_pdl (kb, g, b, s, p, (const Params*) h->d_params, d_rec, bq, (const int*) h->d_blist, h->blist_cap (), h->d_count, h->d_stats, p.L - 3));
      else kb<<<g, b, 0, s>>> (p, h->d_params, d_rec, bq, h->d_blist, h->blist_cap (), h->d_count, h->d_stats, p.L - 3);
    }
    if (kr >= 0) CK (cudaEventRecord (h->kring[kr][1], s));
    h->launches++;
    if (h->top_path)
    {
      QNode* cells = h->super_static ? h->d_superq : h->Q.q[h->nup];
      const int qslot = h->super_static ? -1 : h->nup;
      auto ku = p.color ? k_celltop_up<true> : k_celltop_up<false>;
      CK (launch_pdl (ku, dim3 (h->sm_count), dim3 (128), s, p, d_rec, cells, pub ? q1 : cells, (const int*) h->d_count, (const QNode*) h->d_cellq, (const CellTop*) h->d_celltop, CELL_CAP, h->d_stats, h->sl, qslot, h->super_static, fold));
      h->launches++;
      for (int li = h->nup - 1; li >= 0; --li) { k_upper_up<<<h->sm_count * 2, 128, 0, s>>> (p, d_rec, h->Q, li, h->d_stats); h->launches++; }
    }
    else
      for (int li = nl - 2; li >= 0; --li) { k_upper_up<<<h->sm_count * 2, 128, 0, s>>> (p, d_rec, h->Q, li, h->d_stats); h->launches++; }
  }
  else
  {
    if (kr >= 0) CK (cudaEventRecord (h->kring[kr][0], s));
    // general path: every culled cell depth-first (grid covers the worst case; threads past *count exit)
    k_update_dfs<<<(ncells + 31) / 32, 32, 0, s>>> (p, d_rec, h->d_culled, h->d_count, h->d_stats);
    if (kr >= 0) CK (cudaEventRecord (h->kring[kr][1], s));
    h->launches++;
  }
  if (kr >= 0) { h->kring_head = (kr + 1) % KRING; h->kring_pending++; }
  h->prof_frames++;
  return B200TSDF_OK;
}

// a slot of the record ring for the next frame: the host image is only rewritten once the copy that read it FRAME_RING
// frames ago has certainly executed
static int ring_slot (b200tsdf* h, int& slot)
{
  slot = (int) (h->ring_seq % FRAME_RING);
  const int half = FRAME_RING / 2;
  if (h->ring_seq >= (uint64_t) FRAME_RING && slot % half == 0) CK (cudaEventSynchronize (h->ev_ring[slot / half]));
  return B200TSDF_OK;
}
static int ring_advance (b200tsdf* h, int slot, cudaStream_t s)
{
  const int half = FRAME_RING / 2;
  if (slot % half == half - 1) CK (cudaEventRecord (h->ev_ring[slot / half], s));   // covers the copies of this half
  h->ring_seq++;
  return B200TSDF_OK;
}

static int integrate_on_device (b200tsdf* h, const unsigned char* d_pts, size_t stride, int xyz_off, int rgba_off, int W, int H, const double* pose)
{
  cudaStream_t s = h->stream;
  if (int rc = pending_device_err (h)) return rc;
  int slot = 0;
  { int rc = ring_slot (h, slot); if (rc) return rc; }
  FrameRec& rec = h->h_ring[slot];
  FrameNumbering num (h);
  fill_rec (h, rec, d_pts, stride, xyz_off, rgba_off, W, H, pose);
  if (h->time_frames) CK (cudaEventRecord (h->ev_t0, s));
  CK (cudaMemcpyAsync (h->d_ring + slot, &rec, sizeof (FrameRec), cudaMemcpyHostToDevice, s));
  { int rc = launch_frame (h, s, h->d_ring + slot, h->time_frames); if (rc) { h->half_launched = true; return rc; } }
  num.enqueued = true;
  if (h->time_frames) CK (cudaEventRecord (h->ev_t1, s));
  note_device_err (h, s);
  { int rc = ring_advance (h, slot, s); if (rc) return rc; }
  CK (cudaGetLastError ());
  h->timed = h->time_frames;
  h->is_empty = false;                                             // hpp:101
  return B200TSDF_OK;
}

// layout of an organized cloud as the integrate entry points accept it (ADVICE r1: the same checks everywhere)
static int check_cloud_layout (b200tsdf* h, size_t stride, int xyz_off, int rgba_off, int width, int height)
{
  if (width <= 0 || height <= 0) return h->fail (B200TSDF_EINVAL, "bad cloud shape");
  if (stride < 12 || (stride & 3) || xyz_off < 0 || (xyz_off & 3) || (size_t) xyz_off + 12 > stride
      || (rgba_off >= 0 && ((size_t) rgba_off + 4 > stride || (rgba_off & 3))))
    return h->fail (B200TSDF_EINVAL, "bad point layout (need 4-byte aligned xyz_off + 12 <= stride and rgba_off + 4 <= stride)");
  if ((double) width * (double) height * (double) stride >= 2147483648.0) return h->fail (B200TSDF_EINVAL, "organized cloud of 2 GiB or more");
  if (width != h->cfg.image_width || height != h->cfg.image_height)
    return h->fail (B200TSDF_EINVAL, "organized cloud size differs from setImageSize() (the reference indexes cloud(u,v) with the image size, cpp:611-617)");
  return B200TSDF_OK;
}

int b200tsdf_integrate_device (b200tsdf_t* h, const void* d_points, size_t stride, int xyz_off, int rgba_off,
                               int width, int height, const double* pose)
{
  if (!h || !d_points || !pose) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "integrateCloud before reset()");
  if (int rc = check_cloud_layout (h, stride, xyz_off, rgba_off, width, height)) return rc;
  cudaSetDevice (h->device);
  return integrate_on_device (h, (const unsigned char*) d_points, stride, xyz_off, rgba_off, width, height, pose);
}

// a batch of frames resident in device memory: one upload of the frame records, one graph launch
// The two halves of a batch: (1) the frame records are written into a host staging segment and uploaded on `rec_stream`
// into one half of the device slots; (2) the captured launches of that half are replayed on the compute stream.  The row
// path (multigpu.cuh) uploads the records on its copy stream AHEAD of the frames themselves — a record upload issued on
// the compute stream would queue behind every frame copy already submitted to the one host-to-device copy engine.
// ob / orecs: the organise block of an unorganised batch, db: the depth block of a depth batch; either travels in the same
// copy behind the frame records
// The caller has checked every argument (d_points[i] are not null) and holds a FrameNumbering until batch_launch has returned.
static int batch_records (b200tsdf* h, int m, const void* const* d_points, size_t stride, int xyz_off, int rgba_off, int width, int height,
                          const double* poses_c2w, cudaStream_t rec_stream, const OrgBatch* ob = nullptr, const OrgRec* orecs = nullptr,
                          const DepthBatch* db = nullptr)
{
  const int a = h->bring_half, sg = h->bring_seg;
  if (h->bring_used[sg]) CK (cudaEventSynchronize (h->ev_bring[sg]));    // the copy that last read this staging segment has run
  FrameRec* recs = h->h_bring + (size_t) sg * BRING_SPAN;
  for (int i = 0; i < m; ++i)
    fill_rec (h, recs[i], (const unsigned char*) d_points[i], stride, xyz_off, rgba_off, width, height, poses_c2w + 16 * (size_t) i);
  size_t bytes = (size_t) m * sizeof (FrameRec);
  if (ob)
  {
    *org_block (recs, m) = *ob;
    std::memcpy (org_recs (recs, m), orecs, (size_t) m * sizeof (OrgRec));
    bytes += ORG_HDR + (size_t) m * sizeof (OrgRec);
  }
  else if (db)
  {
    *depth_block (recs, m) = *db;
    bytes += sizeof (DepthBatch);
  }
  // the device half is rewritten only after the launches that last read it (other stream: wait for their event)
  if (rec_stream != h->stream && h->half_used[a]) CK (cudaStreamWaitEvent (rec_stream, h->ev_half_done[a], 0));
  CK (cudaMemcpyAsync (h->d_bring + a * BRING_SPAN, recs, bytes, cudaMemcpyHostToDevice, rec_stream));
  CK (cudaEventRecord (h->ev_bring[sg], rec_stream));      // the staging segment is free again once this copy has run
  h->bring_used[sg] = true; h->bring_seg = (sg + 1) % BATCH_SEGS;
  return B200TSDF_OK;
}
// the organised images of the unorganised batch path (layout: keys HALF*npix*8 | filled counters HALF*8 | images HALF*npix*16)
static size_t org_npix (const b200tsdf* h) { return (size_t) h->cfg.image_width * h->cfg.image_height; }
static unsigned long long* org_keys (const b200tsdf* h) { return reinterpret_cast<unsigned long long*> (h->d_org.p); }
static unsigned long long* org_filled (const b200tsdf* h) { return org_keys (h) + ORG_MAX_FRAMES * org_npix (h); }
static unsigned char* org_images (const b200tsdf* h) { return h->d_org + ORG_MAX_FRAMES * org_npix (h) * 8 + 256; }
static int org_buffers (b200tsdf* h)
{
  if (h->d_org.grow (ORG_MAX_FRAMES * org_npix (h) * (8 + 16) + 256)) return alloc_failed (h, "organised images of an unorganised batch");
  return B200TSDF_OK;
}

// the three organise launches of m frames (organize.cuh): keys cleared, every point z-buffered, m images gathered
static int launch_organize (b200tsdf* h, cudaStream_t s, const OrgBatch* d_ob, const OrgRec* d_recs, int m,
                            unsigned long long* zkey, unsigned long long* filled, unsigned char* out)
{
  const int npix = (int) org_npix (h);
  const dim3 pix_grid ((npix + 255) / 256, m);
  k_org_clear<<<pix_grid, 256, 0, s>>> (zkey, npix, filled);
  k_org_zmin<<<h->sm_count * 8, 256, 0, s>>> (d_ob, d_recs, m, npix, zkey);
  k_org_gather<<<pix_grid, 256, 0, s>>> (d_ob, d_recs, npix, zkey, out, filled);
  h->launches += 3;
  CK (cudaGetLastError ());
  return B200TSDF_OK;
}

// the unprojection of m depth frames (depth.cuh) into m images of 16-byte pixels
static int launch_depth (b200tsdf* h, cudaStream_t s, const DepthBatch* d_db, int m, unsigned char* out)
{
  const int npix = (int) org_npix (h);
  k_depth_unproject<<<dim3 ((npix + 255) / 256, m), 256, 0, s>>> (d_db, npix, out);
  h->launches += 1;
  CK (cudaGetLastError ());
  return B200TSDF_OK;
}

// front: FRONT_ORGANIZE, the records carry the organise block of an unorganised batch (batch_records), whose three launches
// come first; FRONT_DEPTH, they carry the depth block of a depth batch, whose unprojection comes first
static int batch_launch (b200tsdf* h, int m, FrontEnd front = FRONT_NONE)
{
  cudaStream_t s = h->stream;
  const int a = h->bring_half;
  FrameRec* const d_recs = h->d_bring + a * BRING_SPAN;
  // (nothing of a frame is baked into the launches: they read the record)
  cudaGraphExec_t& exec = (front == FRONT_ORGANIZE ? h->unorg_exec : front == FRONT_DEPTH ? h->depth_exec : h->batch_exec)[a][m];
  const int front_launches = front == FRONT_ORGANIZE ? 3 : front == FRONT_DEPTH ? 1 : 0;
  if (!exec)
  {
    const long long l0 = h->launches, f0 = h->prof_frames;
    cudaGraph_t g = nullptr;
    CK (cudaStreamBeginCapture (s, cudaStreamCaptureModeThreadLocal));
    int rc = B200TSDF_OK;
    if (front == FRONT_ORGANIZE) rc = launch_organize (h, s, org_block (d_recs, m), org_recs (d_recs, m), m, org_keys (h), org_filled (h), org_images (h));
    if (front == FRONT_DEPTH) rc = launch_depth (h, s, depth_block (d_recs, m), m, org_images (h));
    // (the first k_front of an unorganised or depth batch reads what the front end wrote: no programmatic overlap with it, see
    // launch_frame)
    for (int i = 0; i < m && rc == B200TSDF_OK; ++i) rc = launch_frame (h, s, d_recs + i, false, !(front != FRONT_NONE && i == 0));
    cudaError_t ce = cudaStreamEndCapture (s, &g);
    h->launches_per_frame = (int) ((h->launches - l0 - front_launches) / std::max (1, m));
    h->launches = l0; h->prof_frames = f0;
    if (rc) { if (g) cudaGraphDestroy (g); return rc; }
    if (ce != cudaSuccess) return h->fail (B200TSDF_ECUDA, std::string ("graph capture: ") + cudaGetErrorString (ce));
    ce = cudaGraphInstantiate (&exec, g, 0);
    cudaGraphDestroy (g);
    if (ce != cudaSuccess) { exec = nullptr; return h->fail (B200TSDF_ECUDA, std::string ("graph instantiate: ") + cudaGetErrorString (ce)); }
  }
  CK (cudaGraphLaunch (exec, s));
  CK (cudaEventRecord (h->ev_half_done[a], s));
  h->half_used[a] = true;
  note_device_err (h, s);
  h->bring_half ^= 1;
  h->launches += front_launches + (long long) m * h->launches_per_frame; h->graph_launches++;
  h->prof_frames += m;
  h->timed = false;
  h->is_empty = false;
  return B200TSDF_OK;
}

int b200tsdf_integrate_batch_device (b200tsdf_t* h, int n, const void* const* d_points, size_t stride, int xyz_off, int rgba_off,
                                     int width, int height, const double* poses_c2w)
{
  if (!h || n < 0 || (n && (!d_points || !poses_c2w))) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "integrateCloud before reset()");
  if (int rc = check_cloud_layout (h, stride, xyz_off, rgba_off, width, height)) return rc;
  // every pointer of every record half, before any of them is numbered or fused: a refused batch enqueues nothing
  for (int i = 0; i < n; ++i) if (!d_points[i]) return h->fail (B200TSDF_EINVAL, "null cloud in batch");
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  constexpr int HALF = FRAME_RING / 2;
  for (int done = 0; done < n;)
  {
    const int m = std::min (HALF, n - done);
    FrameNumbering num (h);
    if (int rc = batch_records (h, m, d_points + done, stride, xyz_off, rgba_off, width, height, poses_c2w + 16 * (size_t) done, h->stream)) return rc;
    if (int rc = batch_launch (h, m)) return rc;
    num.enqueued = true;
    done += m;
  }
  CK (cudaGetLastError ());
  return B200TSDF_OK;
}

// the host threads that pack uploaded points to 16-byte pixels (host_pack.h), created on first use
static void ensure_pack_pool (b200tsdf* h, int nr)
{
  if (h->pack_pool) return;
  int t = h->pack_threads;
  if (t <= 0) { const int hw = (int) std::thread::hardware_concurrency (); t = std::max (1, std::min (16, hw / (2 * nr))); }
  // B200TSDF_PACK_CPUS: "local" = the cores next to this GPU's PCIe root (sysfs local_cpulist), or an explicit cpulist
  std::string cpus;
  if (const char* e = std::getenv ("B200TSDF_PACK_CPUS"))
  {
    cpus = e;
    if (cpus == "local")
    {
      cpus.clear ();
      char bus[32] = {};
      if (cudaDeviceGetPCIBusId (bus, sizeof (bus), h->device) == cudaSuccess)
      {
        for (char* c = bus; *c; ++c) *c = (char) std::tolower ((unsigned char) *c);
        if (FILE* f = std::fopen ((std::string ("/sys/bus/pci/devices/") + bus + "/local_cpulist").c_str (), "r"))
        {
          char line[512] = {};
          if (std::fgets (line, sizeof (line), f)) { cpus = line; while (!cpus.empty () && (cpus.back () == '\n' || cpus.back () == ' ')) cpus.pop_back (); }
          std::fclose (f);
        }
      }
    }
  }
  // (no exception may cross the C ABI: if the threads cannot be created the caller's thread packs alone)
  try { h->pack_pool = new b2host::PackPool (t, cpus); }
  catch (...) { h->pack_pool = new b2host::PackPool (1); }
}

// is the upload of `stride`-byte points packed on the host?  (-1: by rank count, see b200tsdf_integrate_batch_rows)
static bool host_pack_wanted (const b200tsdf* h, size_t stride, int nr) { return (h->host_pack < 0 ? nr <= 1 : h->host_pack != 0) && stride > 16; }

static int integrate_host (b200tsdf* h, const void* points, size_t stride, int xyz_off, int rgba_off,
                           int width, int height, const double* pose, bool wait_copy)
{
  if (!h || !points || !pose) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "integrateCloud before reset()");
  if (int rc = check_cloud_layout (h, stride, xyz_off, rgba_off, width, height)) return rc;
  cudaSetDevice (h->device);
  // points wider than 16 bytes are packed to {x, y, z, bgra} by the host threads into pinned staging (also the way out of a
  // pageable pcl cloud at full PCIe speed); the caller's buffer is free again when this call returns
  const bool hpack = host_pack_wanted (h, stride, h->comm ? h->comm_size : 1);
  const size_t npts = (size_t) width * height;
  const size_t bytes = hpack ? npts * 16 : npts * stride;
  const size_t frame_cap = std::min (h->d_frame[0].cap, h->d_frame[1].cap);
  if (bytes > frame_cap || (hpack && !h->h_fpack[0].p))
  {
    CK (cudaStreamSynchronize (h->stream)); CK (cudaStreamSynchronize (h->copy_stream));
    const size_t cap = std::max (bytes, frame_cap);
    for (int i = 0; i < 2; ++i)
    {
      CK (h->d_frame[i].grow (cap));
      h->h_fpack[i].release ();
      if (hpack && h->h_fpack[i].alloc (cap))
      {
        // no pinned staging to be had on this system: upload the points as they are from now on
        h->host_pack = 0;
        for (int k = 0; k < 2; ++k) { h->h_fpack[k].release (); h->d_frame[k].release (); }   // (re-sized by the unpacked path)
        return integrate_host (h, points, stride, xyz_off, rgba_off, width, height, pose, wait_copy);
      }
    }
    h->frame_no = 0;
  }
  // double-buffered upload on the copy stream: frame i+1 crosses PCIe while frame i is fused
  int b = (int) (h->frame_no & 1);
  if (h->frame_no >= 2)
  {
    CK (cudaEventSynchronize (h->ev_copied[b]));           // the upload of frame i-2 has left the caller's buffer / the staging (the documented contract)
    CK (cudaStreamWaitEvent (h->copy_stream, h->ev_consumed[b], 0));
  }
  const void* src = points;
  size_t f_stride = stride; int f_xyz = xyz_off, f_rgba = rgba_off;
  if (hpack)
  {
    ensure_pack_pool (h, h->comm ? h->comm_size : 1);
    const int nb = (int) std::max<size_t> (1, std::min<size_t> (4 * (size_t) h->pack_pool->threads (), npts / 4096));
    const int pack_rgba = h->p.color ? rgba_off : -1;
    unsigned char* stage = h->h_fpack[b].p;
    std::function<void (int)> job = [&] (int j)
    {
      const size_t p0 = npts * (size_t) j / nb, p1 = npts * (size_t) (j + 1) / nb;
      b2host::pack_points16 (static_cast<const unsigned char*> (points) + p0 * stride, stride, xyz_off, pack_rgba, p1 - p0, stage + p0 * 16);
    };
    h->pack_pool->run (nb, job);
    src = stage; f_stride = 16; f_xyz = 0; f_rgba = (h->p.color && rgba_off >= 0) ? 12 : -1;
  }
  CK (cudaMemcpyAsync (h->d_frame[b], src, bytes, cudaMemcpyHostToDevice, h->copy_stream));
  h->h2d_bytes += (long long) bytes;
  CK (cudaEventRecord (h->ev_copied[b], h->copy_stream));
  CK (cudaStreamWaitEvent (h->stream, h->ev_copied[b], 0));
  int rc = integrate_on_device (h, h->d_frame[b], f_stride, f_xyz, f_rgba, width, height, pose);
  if (rc) return rc;
  CK (cudaEventRecord (h->ev_consumed[b], h->stream));
  h->frame_no++;
  if (wait_copy && !hpack) CK (cudaEventSynchronize (h->ev_copied[b]));       // the caller may reuse its buffer now
  return B200TSDF_OK;
}

int b200tsdf_integrate (b200tsdf_t* h, const void* points, size_t stride, int xyz_off, int rgba_off,
                        int width, int height, const double* pose)
{ return integrate_host (h, points, stride, xyz_off, rgba_off, width, height, pose, true); }

int b200tsdf_integrate_async (b200tsdf_t* h, const void* points, size_t stride, int xyz_off, int rgba_off,
                              int width, int height, const double* pose)
{ return integrate_host (h, points, stride, xyz_off, rgba_off, width, height, pose, false); }

// ---- unorganised clouds (integrate.cpp:548-635) ------------------------------------------------
// Every organise goes through the batched kernels of organize.cuh: b200tsdf_organize is a batch of one frame written in the
// caller's layout, b200tsdf_integrate_unorganized an upload plus a batch of one, and the batch entry point m frames per record
// half, each half one graph launch.
namespace {

// the checks every organise entry point applies to its input points (org_load reads them as floats: 4-byte aligned)
int org_args (b200tsdf* h, size_t stride, int xyz_off, int rgba_off, const b200tsdf_organize_opts* opts)
{
  if (!opts) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "organize before reset() (the image size and intrinsics are read at reset)");
  if (stride < 12 || (stride & 3) || xyz_off < 0 || (xyz_off & 3) || (size_t) xyz_off + 12 > stride
      || (rgba_off >= 0 && ((size_t) rgba_off + 4 > stride || (rgba_off & 3))))
    return h->fail (B200TSDF_EINVAL, "bad point layout (need 4-byte aligned stride, xyz_off and rgba_off, xyz_off + 12 <= stride and rgba_off + 4 <= stride)");
  return B200TSDF_OK;
}

int org_count (b200tsdf* h, const void* points, size_t n)
{
  if (!points && n) return h->fail (B200TSDF_EINVAL, "null cloud with points");
  if (n >= (1ull << 32)) return h->fail (B200TSDF_EINVAL, "more than 2^32-1 points in one cloud");
  return B200TSDF_OK;
}

OrgBatch org_batch (const b200tsdf* h, const b200tsdf_organize_opts* opts, size_t stride, int xyz_off, int rgba_off,
                    size_t out_stride, int out_rgba_off)
{
  OrgBatch b{};
  // the program keeps its intrinsics as float globals (integrate.cpp:63-68, 349-361)
  b.o.fx = (float) h->cfg.fx; b.o.fy = (float) h->cfg.fy; b.o.cx = (float) h->cfg.cx; b.o.cy = (float) h->cfg.cy;
  b.o.width = h->cfg.image_width; b.o.height = h->cfg.image_height;
  b.o.cloud_units = opts->cloud_units; b.o.zero_nans = opts->zero_nans;
  b.stride = stride; b.xyz_off = xyz_off; b.rgba_off = rgba_off;
  b.out_stride = out_stride; b.out_rgba_off = out_rgba_off;
  return b;
}

// w2c: a row-major 4x4 world -> camera matrix or null
OrgRec org_rec (const void* d_pts, size_t n, unsigned long long first, const double* w2c)
{
  OrgRec r{};
  r.pts = static_cast<const unsigned char*> (d_pts); r.count = n; r.first = first;
  r.has_tf = w2c != nullptr;
  if (w2c) for (int i = 0; i < 12; ++i) r.tf[i] = w2c[i];
  return r;
}

// n frames, HALF per record half: the organised images are 16-byte pixels {x, y, z, bgra} in d_org, fused like an organised
// batch (stride 16, xyz at 0, colour at 12).  The arguments have been checked.
int unorganized_batches (b200tsdf* h, int n, const void* const* d_points, const size_t* counts, size_t stride, int xyz_off, int rgba_off,
                         const b200tsdf_organize_opts* opts, const double* poses_c2w)
{
  constexpr int HALF = FRAME_RING / 2;
  if (int rc = org_buffers (h)) return rc;
  const OrgBatch ob = org_batch (h, opts, stride, xyz_off, rgba_off, 16, 12);
  const size_t npix = org_npix (h);
  for (int done = 0; done < n;)
  {
    const int m = std::min (HALF, n - done);
    const void* imgs[HALF]; OrgRec recs[HALF];
    unsigned long long first = 0;
    for (int i = 0; i < m; ++i)
    {
      const int k = done + i;
      imgs[i] = org_images (h) + (size_t) i * npix * 16;
      recs[i] = org_rec (d_points[k], counts[k], first, opts->world_to_camera ? opts->world_to_camera + 16 * (size_t) k : nullptr);
      first += counts[k];
    }
    FrameNumbering num (h);
    if (int rc = batch_records (h, m, imgs, 16, 0, 12, h->cfg.image_width, h->cfg.image_height, poses_c2w + 16 * (size_t) done, h->stream, &ob, recs)) return rc;
    if (int rc = batch_launch (h, m, FRONT_ORGANIZE)) return rc;
    num.enqueued = true;
    done += m;
  }
  CK (cudaGetLastError ());
  return B200TSDF_OK;
}

} // namespace

int b200tsdf_organize (b200tsdf_t* h, const void* points, size_t n, size_t stride, int xyz_off, int rgba_off,
                       const b200tsdf_organize_opts* opts, void* out, size_t out_stride, int out_rgba_off, int64_t* n_filled)
{
  if (!h || !out) return B200TSDF_EINVAL;
  if (int rc = org_args (h, stride, xyz_off, rgba_off, opts)) return rc;
  if (int rc = org_count (h, points, n)) return rc;
  if (out_stride < 16 || (out_stride & 3) || (out_rgba_off >= 0 && ((size_t) out_rgba_off + 4 > out_stride || out_rgba_off < 12)))
    return h->fail (B200TSDF_EINVAL, "bad organized layout");
  cudaSetDevice (h->device);
  const size_t npix = org_npix (h);
  // scratch: [organise block | points n*stride | zkey npix*8 | filled counter 8 | organized npix*out_stride]
  const size_t off_pts = (ORG_HDR + sizeof (OrgRec) + 255) & ~(size_t) 255, off_key = (off_pts + n * stride + 255) & ~(size_t) 255, off_cnt = off_key + npix * 8, off_out = off_cnt + 256;
  { int rc = h->scratch (off_out + npix * out_stride + 64); if (rc) return rc; }
  unsigned char* d = h->d_scratch;
  unsigned char hdr[ORG_HDR + sizeof (OrgRec)];
  const OrgBatch ob = org_batch (h, opts, stride, xyz_off, rgba_off, out_stride, out_rgba_off);
  const OrgRec rec = org_rec (d + off_pts, n, 0, opts->world_to_camera);
  std::memcpy (hdr, &ob, sizeof (ob)); std::memcpy (hdr + ORG_HDR, &rec, sizeof (rec));
  cudaStream_t s = h->stream;
  CK (cudaMemcpyAsync (d, hdr, sizeof (hdr), cudaMemcpyHostToDevice, s));          // (pageable: staged before the call returns)
  if (n) { CK (cudaMemcpyAsync (d + off_pts, points, n * stride, cudaMemcpyHostToDevice, s)); h->h2d_bytes += (long long) (n * stride); }
  unsigned long long* d_filled = (unsigned long long*) (d + off_cnt);
  if (int rc = launch_organize (h, s, (const OrgBatch*) d, (const OrgRec*) (d + ORG_HDR), 1, (unsigned long long*) (d + off_key), d_filled, d + off_out))
    return rc;
  const size_t bytes = npix * out_stride;
  unsigned long long filled = 0;
  // bytes of a pixel that the layout does not name (padding) are zero in the result
  CK (cudaMemcpyAsync (out, d + off_out, bytes, cudaMemcpyDeviceToHost, s));
  CK (cudaMemcpyAsync (&filled, d_filled, 8, cudaMemcpyDeviceToHost, s));
  CK (cudaStreamSynchronize (s));
  h->d2h_bytes += (long long) bytes + 8;
  if (n_filled) *n_filled = (int64_t) filled;
  return B200TSDF_OK;
}

int b200tsdf_integrate_unorganized (b200tsdf_t* h, const void* points, size_t n, size_t stride, int xyz_off, int rgba_off,
                                    const b200tsdf_organize_opts* opts, const double* pose)
{
  if (!h || !pose) return B200TSDF_EINVAL;
  if (int rc = org_args (h, stride, xyz_off, rgba_off, opts)) return rc;
  if (int rc = org_count (h, points, n)) return rc;
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  // the points go to the scratch on the handle's stream (after the launches that last read it), then a batch of one
  { int rc = h->scratch (n * stride + 64); if (rc) return rc; }
  if (n) { CK (cudaMemcpyAsync (h->d_scratch, points, n * stride, cudaMemcpyHostToDevice, h->stream)); h->h2d_bytes += (long long) (n * stride); }
  const void* d_pts = h->d_scratch;
  return unorganized_batches (h, 1, &d_pts, &n, stride, xyz_off, rgba_off, opts, pose);
}

int b200tsdf_integrate_unorganized_batch_device (b200tsdf_t* h, int n, const void* const* d_points, const size_t* counts,
                                                 size_t stride, int xyz_off, int rgba_off,
                                                 const b200tsdf_organize_opts* opts, const double* poses_c2w)
{
  if (!h || n < 0 || (n && (!d_points || !counts || !poses_c2w))) return B200TSDF_EINVAL;
  if (int rc = org_args (h, stride, xyz_off, rgba_off, opts)) return rc;
  for (int i = 0; i < n; ++i) if (int rc = org_count (h, d_points[i], counts[i])) return rc;   // (nothing is enqueued for a refused batch)
  if (!n) return B200TSDF_OK;
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  return unorganized_batches (h, n, d_points, counts, stride, xyz_off, rgba_off, opts, poses_c2w);
}

// ---- depth images (depth.cuh, DESIGN.md §3h) ----------------------------------------------------
// A depth frame is one integrateCloud of the organised cloud depth_pixel makes from it: the batch's depth block travels behind
// its frame records, k_depth_unproject writes the images of the unorganised batch path (org_images), and the frames fuse from
// there, m frames per record half, each half one graph launch.
namespace {

// the checks every depth entry point applies before anything is enqueued
int depth_args (b200tsdf* h, int format, float scale, int width, int height)
{
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "depth image before reset() (the image size and intrinsics are read at reset)");
  if (h->p.shard_count > 1 || h->comm) return h->fail (B200TSDF_ESTATE, "depth images on a shard: integrate them on an unsharded handle");
  if (format != B200TSDF_DEPTH_U16 && format != B200TSDF_DEPTH_F32) return h->fail (B200TSDF_EINVAL, "bad depth format");
  if (!(scale > 0.f && scale <= 3.402823466e38f)) return h->fail (B200TSDF_EINVAL, "depth scale must be finite and > 0");
  if (width != h->cfg.image_width || height != h->cfg.image_height)
    return h->fail (B200TSDF_EINVAL, "depth image size differs from setImageSize() (the intrinsics belong to that size)");
  return B200TSDF_OK;
}

size_t depth_elem (int format) { return format == B200TSDF_DEPTH_U16 ? 2 : 4; }

int depth_ptr (b200tsdf* h, const void* depth, int format)
{
  if (!depth) return h->fail (B200TSDF_EINVAL, "null depth image");
  if (reinterpret_cast<uintptr_t> (depth) % depth_elem (format)) return h->fail (B200TSDF_EINVAL, "depth image not aligned to its element size");
  return B200TSDF_OK;
}

DepthBatch depth_batch (const b200tsdf* h, int format, float scale)
{
  DepthBatch b{};
  b.fx = (float) h->cfg.fx; b.fy = (float) h->cfg.fy; b.cx = (float) h->cfg.cx; b.cy = (float) h->cfg.cy;
  b.scale = scale; b.width = h->cfg.image_width; b.height = h->cfg.image_height; b.format = format;
  return b;
}

// n depth frames resident in device memory, HALF per record half.  The arguments have been checked and org_buffers sized.
// A colour image on a volume without colour is not read (the frame fuses with rgba_off = -1, as a cloud's colour would be
// ignored there).
int depth_batches (b200tsdf* h, int n, const void* const* d_depth, int format, float scale, const void* const* d_rgb, const double* poses_c2w)
{
  constexpr int HALF = FRAME_RING / 2;
  const bool color = h->p.color && d_rgb;
  DepthBatch db = depth_batch (h, format, scale);
  const size_t npix = org_npix (h);
  for (int done = 0; done < n;)
  {
    const int m = std::min (HALF, n - done);
    const void* imgs[HALF];
    for (int i = 0; i < m; ++i)
    {
      imgs[i] = org_images (h) + (size_t) i * npix * 16;
      db.depth[i] = d_depth[done + i];
      db.rgb[i] = color ? static_cast<const unsigned char*> (d_rgb[done + i]) : nullptr;
    }
    FrameNumbering num (h);
    if (int rc = batch_records (h, m, imgs, 16, 0, color ? 12 : -1, h->cfg.image_width, h->cfg.image_height, poses_c2w + 16 * (size_t) done,
                                h->stream, nullptr, nullptr, &db)) return rc;
    if (int rc = batch_launch (h, m, FRONT_DEPTH)) return rc;
    num.enqueued = true;
    done += m;
  }
  CK (cudaGetLastError ());
  return B200TSDF_OK;
}

// The caller's depth (dbytes) and colour (cbytes, 0: none) copied into pinned slot b and uploaded on copy_stream into that
// slot's device buffer d_raw; the handle's stream waits for the upload.  The caller records ev_dconsumed[b] on the stream
// behind the last launch that reads d_raw, and advances depth_no.
int stage_depth (b200tsdf* h, const void* depth, size_t dbytes, const uint8_t* rgb, size_t cbytes, int& b, unsigned char*& d_raw)
{
  const size_t slot_bytes = org_npix (h) * 7;                         // the widest frame: float32 depth and colour
  if (!h->h_depth[0].p || h->h_depth[0].bytes < slot_bytes || h->d_depth_raw[0].cap < slot_bytes)
  {
    CK (cudaStreamSynchronize (h->stream)); CK (cudaStreamSynchronize (h->copy_stream));
    for (int i = 0; i < DEPTH_SLOTS; ++i)
    {
      if (h->h_depth[i].alloc (slot_bytes)) { for (int k = 0; k < DEPTH_SLOTS; ++k) h->h_depth[k].release (); return alloc_failed (h, "pinned staging of depth images"); }
      if (h->d_depth_raw[i].grow (slot_bytes)) return alloc_failed (h, "device buffers of depth images");
    }
    h->depth_no = 0;
  }
  // the slot's last upload has run (so its staging is free), and that upload's unprojection has read the device buffer
  // before the next upload rewrites it; fusion of earlier frames is never waited for here
  b = (int) (h->depth_no % DEPTH_SLOTS);
  if (h->depth_no >= (uint64_t) DEPTH_SLOTS)
  {
    CK (cudaEventSynchronize (h->ev_dcopied[b]));
    CK (cudaStreamWaitEvent (h->copy_stream, h->ev_dconsumed[b], 0));
  }
  unsigned char* stage = h->h_depth[b].p;
  std::memcpy (stage, depth, dbytes);                                 // the caller's buffers are free when this call returns
  if (cbytes) std::memcpy (stage + dbytes, rgb, cbytes);
  d_raw = h->d_depth_raw[b];
  CK (cudaMemcpyAsync (d_raw, stage, dbytes + cbytes, cudaMemcpyHostToDevice, h->copy_stream));
  h->h2d_bytes += (long long) (dbytes + cbytes);
  CK (cudaEventRecord (h->ev_dcopied[b], h->copy_stream));
  CK (cudaStreamWaitEvent (h->stream, h->ev_dcopied[b], 0));
  return B200TSDF_OK;
}

} // namespace

int b200tsdf_integrate_depth (b200tsdf_t* h, const void* depth, int depth_format, float depth_scale, const uint8_t* rgb,
                              int width, int height, const double* pose_c2w)
{
  if (!h || !pose_c2w) return B200TSDF_EINVAL;
  if (int rc = depth_args (h, depth_format, depth_scale, width, height)) return rc;
  if (int rc = depth_ptr (h, depth, depth_format)) return rc;
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  if (int rc = org_buffers (h)) return rc;
  const size_t npix = org_npix (h), dbytes = npix * depth_elem (depth_format), cbytes = rgb && h->p.color ? npix * 3 : 0;
  int b = 0;
  unsigned char* d_raw = nullptr;
  if (int rc = stage_depth (h, depth, dbytes, rgb, cbytes, b, d_raw)) return rc;
  const void* d_depth = d_raw;
  const void* d_rgb = d_raw + dbytes;
  if (int rc = depth_batches (h, 1, &d_depth, depth_format, depth_scale, cbytes ? &d_rgb : nullptr, pose_c2w)) return rc;
  CK (cudaEventRecord (h->ev_dconsumed[b], h->stream));
  h->depth_no++;
  return B200TSDF_OK;
}

int b200tsdf_integrate_depth_batch_device (b200tsdf_t* h, int n, const void* const* d_depth, int depth_format, float depth_scale,
                                           const void* const* d_rgb, int width, int height, const double* poses_c2w)
{
  if (!h || n < 0 || (n && (!d_depth || !poses_c2w))) return B200TSDF_EINVAL;
  if (int rc = depth_args (h, depth_format, depth_scale, width, height)) return rc;
  // every pointer of every record half, before any frame is numbered: a refused batch enqueues nothing
  for (int i = 0; i < n; ++i)
  {
    if (int rc = depth_ptr (h, d_depth[i], depth_format)) return rc;
    if (d_rgb && !d_rgb[i]) return h->fail (B200TSDF_EINVAL, "null colour image in batch");
  }
  if (!n) return B200TSDF_OK;
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  if (int rc = org_buffers (h)) return rc;
  return depth_batches (h, n, d_depth, depth_format, depth_scale, d_rgb, poses_c2w);
}

int b200tsdf_depth_to_cloud_device (b200tsdf_t* h, const void* d_depth, int depth_format, float depth_scale, const uint8_t* d_rgb,
                                    int width, int height, void* d_out)
{
  if (!h) return B200TSDF_EINVAL;
  if (int rc = depth_args (h, depth_format, depth_scale, width, height)) return rc;
  if (int rc = depth_ptr (h, d_depth, depth_format)) return rc;
  if (!d_out || reinterpret_cast<uintptr_t> (d_out) % 16) return h->fail (B200TSDF_EINVAL, "output image null or not 16-byte aligned");
  cudaSetDevice (h->device);
  if (int rc = h->scratch (sizeof (DepthBatch))) return rc;
  DepthBatch db = depth_batch (h, depth_format, depth_scale);
  db.depth[0] = d_depth; db.rgb[0] = d_rgb;
  cudaStream_t s = h->stream;
  CK (cudaMemcpyAsync (h->d_scratch, &db, sizeof (db), cudaMemcpyHostToDevice, s));          // (pageable: staged before the call returns)
  if (int rc = launch_depth (h, s, reinterpret_cast<const DepthBatch*> (h->d_scratch.p), 1, static_cast<unsigned char*> (d_out))) return rc;
  CK (cudaStreamSynchronize (s));
  return B200TSDF_OK;
}

// ---- tracking (track.cuh, DESIGN.md §3i) -------------------------------------------------------------------------------
// One call: the inputs and the initial state go up in one copy, the captured graph of the schedule runs (the depth
// unprojection first for a depth map, then k_track_terms and k_track_solve per iteration; once a level has converged or the
// call has stopped, the remaining launches return at once), and the state comes back in one copy behind it.
namespace {

constexpr int TRACK_GRAPHS = 8;   // captured schedules kept per handle (the oldest goes first)

int track_args (b200tsdf* h, const double* pose0, const b200tsdf_track_params* prm, const b200tsdf_track_result* res)
{
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "tracking before reset()");
  if (h->p.shard_count > 1 || h->comm) return h->fail (B200TSDF_ESTATE, "tracking on a shard: track against an unsharded handle");
  if (!pose0 || !prm || !res) return h->fail (B200TSDF_EINVAL, "null pose, tracking parameters or result");
  for (int i = 0; i < 16; ++i)
    if (!std::isfinite (pose0[i])) return h->fail (B200TSDF_EINVAL, "initial pose not finite");
  if (prm->levels < 1 || prm->levels > TRACK_LEVELS) return h->fail (B200TSDF_EINVAL, "tracking levels outside 1..4");
  for (int l = 0; l < prm->levels; ++l)
  {
    if (prm->stride[l] < 1) return h->fail (B200TSDF_EINVAL, "tracking stride < 1");
    if (prm->iters[l] < 0 || prm->iters[l] > TRACK_MAX_ITERS) return h->fail (B200TSDF_EINVAL, "tracking iterations outside 0..64");
  }
  if (!(prm->huber_delta > 0.f && std::isfinite (prm->huber_delta)) || !(prm->d_max > 0.f) || !std::isfinite (prm->w_min))
    return h->fail (B200TSDF_EINVAL, "huber_delta and d_max must be > 0 (huber_delta finite), w_min finite");
  if (!(prm->damping >= 0.0 && std::isfinite (prm->damping)) || !(prm->eps_rot >= 0.0 && std::isfinite (prm->eps_rot))
      || !(prm->eps_trans >= 0.0 && std::isfinite (prm->eps_trans)) || prm->min_inliers < 0)
    return h->fail (B200TSDF_EINVAL, "damping, eps_rot and eps_trans must be finite and >= 0, min_inliers >= 0");
  return B200TSDF_OK;
}

TrackInput track_input (const b200tsdf* h, const b200tsdf_track_params* prm, const void* pts, size_t stride, int xyz_off)
{
  TrackInput in{};
  in.pts = static_cast<const unsigned char*> (pts); in.stride = (int) stride; in.xyz_off = xyz_off;
  in.width = h->cfg.image_width; in.height = h->cfg.image_height;
  in.levels = prm->levels; in.min_inliers = prm->min_inliers;
  in.huber = prm->huber_delta; in.d_max = prm->d_max; in.w_min = prm->w_min;
  in.damping = prm->damping; in.eps_rot = prm->eps_rot; in.eps_trans = prm->eps_trans;
  return in;
}

// the launches of one schedule on stream s (being captured)
void track_enqueue (b200tsdf* h, cudaStream_t s, bool depth, const b200tsdf_track_params* prm, int cap)
{
  TrackBlock* blk = h->d_track;
  const int W = h->cfg.image_width, H = h->cfg.image_height;
  if (depth) k_depth_unproject<<<dim3 ((unsigned) ((org_npix (h) + 255) / 256), 1), 256, 0, s>>> (&blk->db, (int) org_npix (h), org_images (h));
  for (int l = 0; l < prm->levels; ++l)
  {
    const int tiles = (track_samples (W, H, prm->stride[l]) + TRACK_TILE - 1) / TRACK_TILE;
    for (int k = 0; k < prm->iters[l]; ++k)
    {
      k_track_terms<<<tiles, TRACK_BLOCK, 0, s>>> (h->p, blk, l, prm->stride[l], h->d_track_part, cap);
      k_track_solve<<<1, 32, 0, s>>> (blk, l, tiles, h->d_track_part, cap);
    }
  }
}

// The arguments have been checked; in.pts is the cloud (for a depth map, the organised image db unprojects into).  dslot >= 0:
// a host depth map staged in that slot, released behind the unprojection.
int track_run (b200tsdf* h, const TrackInput& in, const DepthBatch* db, int dslot, const double* pose0, const b200tsdf_track_params* prm,
               b200tsdf_track_result* res, b200tsdf_track_iter* log)
{
  cudaStream_t s = h->stream;
  const int cap = (track_samples (h->cfg.image_width, h->cfg.image_height, 1) + TRACK_TILE - 1) / TRACK_TILE;
  if (!h->h_track.p && h->h_track.alloc (1)) { h->h_track.p = nullptr; return alloc_failed (h, "pinned tracking block"); }
  if (h->d_track.grow (1)) return alloc_failed (h, "tracking block");
  if (h->d_track_part.cap < (size_t) cap * TRACK_NS)
  {
    drop_track_graphs (h);                                   // (the captured schedules name the old buffer)
    if (h->d_track_part.grow ((size_t) cap * TRACK_NS)) return alloc_failed (h, "tracking tile sums");
  }
  TrackBlock& B = *h->h_track.p;
  B.in = in;
  if (db) B.db = *db;
  std::memset (&B.st, 0, sizeof (TrackState));
  track_set_pose (B.st, pose0);
  CK (cudaMemcpyAsync (h->d_track.p, &B, offsetof (TrackBlock, st) + offsetof (TrackState, log), cudaMemcpyHostToDevice, s));
  int total = 0;
  for (int l = 0; l < prm->levels; ++l) total += prm->iters[l];
  if (total)
  {
    int key[10] = { db ? 1 : 0, prm->levels };
    for (int l = 0; l < prm->levels; ++l) { key[2 + l] = prm->stride[l]; key[6 + l] = prm->iters[l]; }
    cudaGraphExec_t exec = nullptr;
    for (const auto& g : h->track_exec)
      if (std::memcmp (g.key, key, sizeof (key)) == 0) exec = g.exec;
    if (!exec)
    {
      cudaGraph_t g = nullptr;
      CK (cudaStreamBeginCapture (s, cudaStreamCaptureModeThreadLocal));
      track_enqueue (h, s, db != nullptr, prm, cap);
      const cudaError_t le = cudaGetLastError ();
      const cudaError_t ce = cudaStreamEndCapture (s, &g);
      if (le != cudaSuccess || ce != cudaSuccess)
      {
        if (g) cudaGraphDestroy (g);
        return h->fail (B200TSDF_ECUDA, std::string ("tracking graph capture: ") + cudaGetErrorString (le != cudaSuccess ? le : ce));
      }
      const cudaError_t ie = cudaGraphInstantiate (&exec, g, 0);
      cudaGraphDestroy (g);
      if (ie != cudaSuccess) return h->fail (B200TSDF_ECUDA, std::string ("tracking graph instantiate: ") + cudaGetErrorString (ie));
      if ((int) h->track_exec.size () >= TRACK_GRAPHS)
      {
        cudaGraphExecDestroy (h->track_exec.front ().exec);
        h->track_exec.erase (h->track_exec.begin ());
      }
      b200tsdf::TrackGraph tg;
      std::memcpy (tg.key, key, sizeof (key)); tg.exec = exec;
      h->track_exec.push_back (tg);
    }
    CK (cudaGraphLaunch (exec, s));
  }
  if (dslot >= 0)
  {
    CK (cudaEventRecord (h->ev_dconsumed[dslot], s));
    h->depth_no++;
  }
  CK (cudaMemcpyAsync (&B.st, &h->d_track.p->st, sizeof (TrackState), cudaMemcpyDeviceToHost, s));
  note_device_err (h, s);
  CK (cudaStreamSynchronize (s));
  if (int rc = pending_device_err (h)) return rc;
  const TrackState& st = B.st;
  static_assert (sizeof (TrackIter) == sizeof (b200tsdf_track_iter), "the log's layout");
  std::memcpy (res->pose_c2w, st.T, sizeof (st.T));
  res->status = track_final_status (st, prm->levels);
  for (int l = 0; l < TRACK_LEVELS; ++l) res->iters[l] = st.iters[l];
  res->inliers = st.inliers; res->n_log = st.nlog; res->reserved = 0; res->rms = st.rms;
  std::memcpy (res->A, st.A, sizeof (st.A)); std::memcpy (res->b, st.b, sizeof (st.b));
  if (log && st.nlog) std::memcpy (log, st.log, (size_t) st.nlog * sizeof (TrackIter));
  return B200TSDF_OK;
}

} // namespace

void b200tsdf_default_track_params (b200tsdf_track_params* prm)
{
  if (!prm) return;
  *prm = b200tsdf_track_params{};
  prm->levels = 3;
  prm->stride[0] = 4; prm->stride[1] = 2; prm->stride[2] = 1; prm->stride[3] = 1;
  prm->iters[0] = 10; prm->iters[1] = 6; prm->iters[2] = 4; prm->iters[3] = 0;
  prm->huber_delta = 0.3f; prm->d_max = 0.95f; prm->w_min = 0.f; prm->min_inliers = 100;
  prm->damping = 1e-4; prm->eps_rot = 1e-5; prm->eps_trans = 1e-5;
}

int b200tsdf_track_cloud_device (b200tsdf_t* h, const void* d_points, size_t stride, int xyz_off, int width, int height,
                                 const double* pose0_c2w, const b200tsdf_track_params* prm, b200tsdf_track_result* res,
                                 b200tsdf_track_iter* log)
{
  if (!h) return B200TSDF_EINVAL;
  if (int rc = track_args (h, pose0_c2w, prm, res)) return rc;
  if (!d_points || reinterpret_cast<uintptr_t> (d_points) % 4) return h->fail (B200TSDF_EINVAL, "cloud null or not 4-byte aligned");
  if (int rc = check_cloud_layout (h, stride, xyz_off, -1, width, height)) return rc;
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  return track_run (h, track_input (h, prm, d_points, stride, xyz_off), nullptr, -1, pose0_c2w, prm, res, log);
}

int b200tsdf_track_depth_device (b200tsdf_t* h, const void* d_depth, int depth_format, float depth_scale, int width, int height,
                                 const double* pose0_c2w, const b200tsdf_track_params* prm, b200tsdf_track_result* res,
                                 b200tsdf_track_iter* log)
{
  if (!h) return B200TSDF_EINVAL;
  if (int rc = depth_args (h, depth_format, depth_scale, width, height)) return rc;
  if (int rc = track_args (h, pose0_c2w, prm, res)) return rc;
  if (int rc = depth_ptr (h, d_depth, depth_format)) return rc;
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  if (int rc = org_buffers (h)) return rc;
  DepthBatch db = depth_batch (h, depth_format, depth_scale);
  db.depth[0] = d_depth; db.rgb[0] = nullptr;
  return track_run (h, track_input (h, prm, org_images (h), 16, 0), &db, -1, pose0_c2w, prm, res, log);
}

int b200tsdf_track_depth (b200tsdf_t* h, const void* depth, int depth_format, float depth_scale, int width, int height,
                          const double* pose0_c2w, const b200tsdf_track_params* prm, b200tsdf_track_result* res,
                          b200tsdf_track_iter* log)
{
  if (!h) return B200TSDF_EINVAL;
  if (int rc = depth_args (h, depth_format, depth_scale, width, height)) return rc;
  if (int rc = track_args (h, pose0_c2w, prm, res)) return rc;
  if (int rc = depth_ptr (h, depth, depth_format)) return rc;
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  if (int rc = org_buffers (h)) return rc;
  int b = 0;
  unsigned char* d_raw = nullptr;
  if (int rc = stage_depth (h, depth, org_npix (h) * depth_elem (depth_format), nullptr, 0, b, d_raw)) return rc;
  DepthBatch db = depth_batch (h, depth_format, depth_scale);
  db.depth[0] = d_raw; db.rgb[0] = nullptr;
  return track_run (h, track_input (h, prm, org_images (h), 16, 0), &db, b, pose0_c2w, prm, res, log);
}

int b200tsdf_sync (b200tsdf_t* h)
{
  if (!h) return B200TSDF_EINVAL;
  cudaSetDevice (h->device);
  CK (cudaStreamSynchronize (h->copy_stream));
  CK (cudaStreamSynchronize (h->gather_stream));
  return check_device_err (h);
}

int b200tsdf_get_stats (b200tsdf_t* h, b200tsdf_stats* s)
{
  if (!h || !s) return B200TSDF_EINVAL;
  std::memset (s, 0, sizeof (*s));
  if (!h->has_volume) return B200TSDF_OK;
  cudaSetDevice (h->device);
  int rc = b200tsdf_sync (h);
  if (rc) return rc;
  unsigned long long st[2 * ST_N]; int cnt[16];
  CK (cudaMemcpy (st, h->d_stats, sizeof (st), cudaMemcpyDeviceToHost));
  CK (cudaMemcpy (cnt, h->d_count + 16 * h->count_set, sizeof (cnt), cudaMemcpyDeviceToHost));
  h->d2h_bytes += (long long) (sizeof (st) + sizeof (cnt));
  s->n_updates = (int64_t) (st[ST_UPDATES] - st[ST_N + ST_UPDATES]);
  s->n_node_visits = (int64_t) (st[ST_VISITS] - st[ST_N + ST_VISITS]);
  s->n_block_visits = (int64_t) (st[ST_BLOCKS] - st[ST_N + ST_BLOCKS]);
  s->reserved = 0; s->n_bail = 0; s->n_slow_visits = 0;   // (kept for the layout; always 0)
  s->n_culled_cells = cnt[0];
  s->pool_capacity = (int64_t) h->vol.pool;
  s->coarse_level = h->p.C; s->finest_level = h->p.L; s->tiers = h->p.T;
  // allocated bricks (no allocation, no list: this call sits in measured loops)
  int* d_n = h->d_count + 40;
  CK (cudaMemsetAsync (d_n, 0, sizeof (int), h->stream));
  k_count_bricks<<<(unsigned) ((h->vol.pool + 255) / 256), 256, 0, h->stream>>> (h->p, d_n);
  int nb = 0;
  CK (cudaMemcpyAsync (&nb, d_n, sizeof (int), cudaMemcpyDeviceToHost, h->stream));
  CK (cudaStreamSynchronize (h->stream));
  s->n_bricks = nb;
  if (h->timed)
  {
    float ms = 0.f;
    if (cudaEventElapsedTime (&ms, h->ev_t0, h->ev_t1) == cudaSuccess) s->ms_last_integrate = ms;
    int last = (h->kring_head + KRING - 1) % KRING;
    if (h->kring_pending > 0 && cudaEventElapsedTime (&ms, h->kring[last][0], h->kring[last][1]) == cudaSuccess) s->ms_last_kernel = ms;
  }
  return B200TSDF_OK;
}

// ---- point queries (tsdf_volume_octree.cpp:655-794) -------------------------------------------------
static int query_args (b200tsdf* h, const float* xyz, int n, int what, const float* val, const float* grad, const float* hess, const uint8_t* ok)
{
  if (!h || !xyz || !ok || n < 0) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "query before reset()");
  if (((what & 1) && !val) || ((what & 2) && !grad) || ((what & 4) && !hess)) return h->fail (B200TSDF_EINVAL, "missing output buffer");
  return B200TSDF_OK;
}

int b200tsdf_query_device (b200tsdf_t* h, const float* d_xyz, int n, int what, int mode,
                           float* d_val, float* d_grad, float* d_hess, uint8_t* d_ok)
{
  if (int rc = query_args (h, d_xyz, n, what, d_val, d_grad, d_hess, d_ok)) return rc;
  if (n == 0) return B200TSDF_OK;
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  k_query<<<(n + 127) / 128, 128, 0, h->stream>>> (h->p, d_xyz, n, what, mode, d_val, d_grad, d_hess, d_ok);
  CK (cudaGetLastError ());
  note_device_err (h, h->stream);
  return B200TSDF_OK;
}

int b200tsdf_query (b200tsdf_t* h, const float* xyz, int n, int what, int mode,
                    float* val, float* grad, float* hess, uint8_t* ok)
{
  if (int rc = query_args (h, xyz, n, what, val, grad, hess, ok)) return rc;
  if (n == 0) return B200TSDF_OK;
  cudaSetDevice (h->device);
  // one scratch block: xyz (12n) | val (4n) | grad (12n) | hess (36n) | ok (n)
  { int rc = h->scratch ((size_t) n * 65 + 64); if (rc) return rc; }
  float* d_xyz = (float*) h->d_scratch.p;
  float* d_val = d_xyz + (size_t) 3 * n;
  float* d_grad = d_val + n;
  float* d_hess = d_grad + (size_t) 3 * n;
  unsigned char* d_ok = (unsigned char*) (d_hess + (size_t) 9 * n);
  cudaStream_t s = h->stream;
  CK (cudaMemcpyAsync (d_xyz, xyz, (size_t) n * 12, cudaMemcpyHostToDevice, s));
  // the kernel writes the ok points only: the caller's values go in first, so that the rest come back as they were
  if (what & 1) CK (cudaMemcpyAsync (d_val, val, (size_t) n * 4, cudaMemcpyHostToDevice, s));
  if (what & 2) CK (cudaMemcpyAsync (d_grad, grad, (size_t) n * 12, cudaMemcpyHostToDevice, s));
  if (what & 4) CK (cudaMemcpyAsync (d_hess, hess, (size_t) n * 36, cudaMemcpyHostToDevice, s));
  if (int rc = b200tsdf_query_device (h, d_xyz, n, what, mode, d_val, d_grad, d_hess, d_ok)) return rc;
  CK (cudaMemcpyAsync (ok, d_ok, (size_t) n, cudaMemcpyDeviceToHost, s));
  if (what & 1) CK (cudaMemcpyAsync (val, d_val, (size_t) n * 4, cudaMemcpyDeviceToHost, s));
  if (what & 2) CK (cudaMemcpyAsync (grad, d_grad, (size_t) n * 12, cudaMemcpyDeviceToHost, s));
  if (what & 4) CK (cudaMemcpyAsync (hess, d_hess, (size_t) n * 36, cudaMemcpyDeviceToHost, s));
  note_device_err (h, s);
  CK (cudaStreamSynchronize (s));
  return pending_device_err (h);
}

// ---- getTSDFValue / interpolateTrilinearly (tsdf_volume_octree.cpp:454-541) ---------------------------------
int b200tsdf_interpolate_device (b200tsdf_t* h, const float* d_xyz, int n, float* d_val, uint8_t* d_valid_in_out)
{
  if (!h || !d_xyz || !d_val || !d_valid_in_out || n < 0) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "getTSDFValue before reset()");
  if (n == 0) return B200TSDF_OK;
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  k_interpolate<<<(n + 127) / 128, 128, 0, h->stream>>> (h->p, d_xyz, n, d_val, d_valid_in_out);
  CK (cudaGetLastError ());
  note_device_err (h, h->stream);
  return B200TSDF_OK;
}

int b200tsdf_interpolate (b200tsdf_t* h, const float* xyz, int n, float* val, uint8_t* valid_in_out)
{
  if (!h || !xyz || !val || !valid_in_out || n < 0) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "getTSDFValue before reset()");
  if (n == 0) return B200TSDF_OK;
  cudaSetDevice (h->device);
  { int rc = h->scratch ((size_t) n * 17 + 64); if (rc) return rc; }
  float* d_xyz = (float*) h->d_scratch.p;
  float* d_val = d_xyz + (size_t) 3 * n;
  unsigned char* d_ok = (unsigned char*) (d_val + n);
  cudaStream_t s = h->stream;
  CK (cudaMemcpyAsync (d_xyz, xyz, (size_t) n * 12, cudaMemcpyHostToDevice, s));
  CK (cudaMemcpyAsync (d_ok, valid_in_out, (size_t) n, cudaMemcpyHostToDevice, s));
  if (int rc = b200tsdf_interpolate_device (h, d_xyz, n, d_val, d_ok)) return rc;
  CK (cudaMemcpyAsync (val, d_val, (size_t) n * 4, cudaMemcpyDeviceToHost, s));
  CK (cudaMemcpyAsync (valid_in_out, d_ok, (size_t) n, cudaMemcpyDeviceToHost, s));
  note_device_err (h, s);
  CK (cudaStreamSynchronize (s));
  return pending_device_err (h);
}

// ---- octree_->getContainingVoxel and dense crops (octree.cpp:112-121, 628-643; tsdf_volume_octree.cpp:553-560) -------------
static_assert (sizeof (VoxelRec) == sizeof (b200tsdf_voxel) && sizeof (b200tsdf_voxel) == 44, "b200tsdf_voxel layout");

static int voxel_read_state (b200tsdf* h, const char* what)
{
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, std::string (what) + " before reset()");
  if (h->p.shard_count > 1)
    return h->fail (B200TSDF_ESTATE, std::string (what) + " on a shard: a shard keeps the coarse cells it does not own as unsplit leaves; "
                    "read the replica built by b200tsdf_gather_volume");
  return B200TSDF_OK;
}

static bool aligned4 (const void* a) { return ((uintptr_t) a & 3u) == 0; }

int b200tsdf_containing_voxels_device (b200tsdf_t* h, const float* d_xyz, size_t n, float min_size, b200tsdf_voxel* d_out)
{
  if (!h) return B200TSDF_EINVAL;
  if (int rc = voxel_read_state (h, "getContainingVoxel")) return rc;
  if (n == 0) return B200TSDF_OK;
  if (!d_xyz || !d_out) return h->fail (B200TSDF_EINVAL, "missing point or output buffer");
  if (!aligned4 (d_xyz) || !aligned4 (d_out)) return h->fail (B200TSDF_EINVAL, "point and output buffers must be 4-byte aligned");
  if (n > ((size_t) INT_MAX) * 128) return h->fail (B200TSDF_EINVAL, "too many points for one call");
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  k_voxels<<<(unsigned) ((n + 127) / 128), 128, 0, h->stream>>> (h->p, d_xyz, n, min_size, reinterpret_cast<VoxelRec*> (d_out));
  CK (cudaGetLastError ());
  note_device_err (h, h->stream);
  return B200TSDF_OK;
}

int b200tsdf_containing_voxels (b200tsdf_t* h, const float* xyz, size_t n, float min_size, b200tsdf_voxel* out)
{
  if (!h) return B200TSDF_EINVAL;
  if (int rc = voxel_read_state (h, "getContainingVoxel")) return rc;
  if (n == 0) return B200TSDF_OK;
  if (!xyz || !out) return h->fail (B200TSDF_EINVAL, "missing point or output buffer");
  cudaSetDevice (h->device);
  // one scratch block: xyz (12 n) | records (44 n)
  { int rc = h->scratch (n * (12 + sizeof (b200tsdf_voxel)) + 64); if (rc) return rc; }
  float* d_xyz = (float*) h->d_scratch.p;
  b200tsdf_voxel* d_out = (b200tsdf_voxel*) (d_xyz + 3 * n);
  cudaStream_t s = h->stream;
  CK (cudaMemcpyAsync (d_xyz, xyz, n * 12, cudaMemcpyHostToDevice, s));
  if (int rc = b200tsdf_containing_voxels_device (h, d_xyz, n, min_size, d_out)) return rc;
  CK (cudaMemcpyAsync (out, d_out, n * sizeof (b200tsdf_voxel), cudaMemcpyDeviceToHost, s));
  note_device_err (h, s);
  CK (cudaStreamSynchronize (s));
  return pending_device_err (h);
}

// ---- octree_->getContainingVoxel (x, y, z, min_size)->setData (d, w) (octree.cpp:112-121, 144-150, 628-634) -------------
// Work space of a batch of n writes: the table (keys and last index, a power of two of at least 2 n slots), the node address
// of every point, and its status when the caller takes none.
struct EditWork { uint64_t* keys; int* last; uint64_t* addr; unsigned char* status; uint32_t mask; };
static size_t edit_table_slots (size_t n) { size_t s = 1024; while (s < 2 * n) s <<= 1; return s; }
static size_t edit_work_bytes (size_t n) { return edit_table_slots (n) * 12 + n * 9 + 64; }
static EditWork edit_work (unsigned char* base, size_t n)
{
  EditWork e;
  const size_t slots = edit_table_slots (n);
  e.keys = (uint64_t*) base; e.addr = e.keys + slots; e.last = (int*) (e.addr + n); e.status = (unsigned char*) (e.last + slots);
  e.mask = (uint32_t) (slots - 1);
  return e;
}

// the writes, queued behind every integrate on the handle's stream; returns once they are done.  An accepted write outside the
// fast route's domain moves the handle to the general kernel until the next reset() or load() (DESIGN.md §3d).
static int edit_batch (b200tsdf* h, const float* d_xyz, size_t n, float min_size, const float* d_d, const float* d_w,
                       uint8_t* d_status, unsigned char* work)
{
  cudaStream_t s = h->stream;
  EditWork e = edit_work (work, n);
  unsigned char* status = d_status ? d_status : e.status;
  unsigned long long* d_ood = h->d_stats + ST_SCRATCH;
  int* d_wrote = h->d_count + 41;
  CK (cudaMemsetAsync (d_wrote, 0, sizeof (int), s));
  CK (cudaMemsetAsync (e.keys, 0xFF, (size_t) (e.mask + 1ull) * sizeof (uint64_t), s));
  CK (cudaMemsetAsync (e.last, 0xFF, (size_t) (e.mask + 1ull) * sizeof (int), s));
  CK (cudaMemsetAsync (d_ood, 0, sizeof (unsigned long long), s));
  const unsigned blocks = (unsigned) ((n + 127) / 128);
  k_edit_resolve<<<blocks, 128, 0, s>>> (h->p, d_xyz, (int) n, min_size, d_d, d_w, status, e.addr, e.keys, e.last, e.mask, d_ood);
  k_edit_store<<<blocks, 128, 0, s>>> (h->p, (int) n, d_d, d_w, status, e.addr, e.keys, e.last, e.mask, h->epoch + 1, d_wrote);
  CK (cudaGetLastError ());
  unsigned long long ood = 0;
  int wrote = 0;
  CK (cudaMemcpyAsync (&ood, d_ood, sizeof (ood), cudaMemcpyDeviceToHost, s));
  CK (cudaMemcpyAsync (&wrote, d_wrote, sizeof (wrote), cudaMemcpyDeviceToHost, s));
  note_device_err (h, s);
  CK (cudaStreamSynchronize (s));
  if (wrote) ++h->epoch;                                     // the epoch the written cells were stamped with
  if (ood && h->fast_path)
  {
    h->fast_path = false; h->top_path = false;
    drop_batch_graphs (h);                                   // the captured launches take the fast route
  }
  return pending_device_err (h);
}

static int edit_args (b200tsdf* h, size_t n, const void* xyz, const float* d, const float* w)
{
  if (int rc = voxel_read_state (h, "setData")) return rc;
  if (n == 0) return B200TSDF_OK;
  if (!xyz || !d || !w) return h->fail (B200TSDF_EINVAL, "missing point, d or w buffer");
  if (n > (size_t) INT_MAX) return h->fail (B200TSDF_EINVAL, "too many points for one call (more than 2^31 - 1)");
  return B200TSDF_OK;
}

int b200tsdf_set_containing_voxels_device (b200tsdf_t* h, const float* d_xyz, size_t n, float min_size, const float* d_d,
                                           const float* d_w, uint8_t* d_status)
{
  if (!h) return B200TSDF_EINVAL;
  if (int rc = edit_args (h, n, d_xyz, d_d, d_w)) return rc;
  if (n == 0) return B200TSDF_OK;
  if (!aligned4 (d_xyz) || !aligned4 (d_d) || !aligned4 (d_w)) return h->fail (B200TSDF_EINVAL, "point, d and w buffers must be 4-byte aligned");
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  { int rc = h->scratch (edit_work_bytes (n)); if (rc) return rc; }
  return edit_batch (h, d_xyz, n, min_size, d_d, d_w, d_status, h->d_scratch);
}

int b200tsdf_set_containing_voxels (b200tsdf_t* h, const float* xyz, size_t n, float min_size, const float* d, const float* w,
                                    uint8_t* status)
{
  if (!h) return B200TSDF_EINVAL;
  if (int rc = edit_args (h, n, xyz, d, w)) return rc;
  if (n == 0) return B200TSDF_OK;
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  // one scratch block: xyz (12 n) | d (4 n) | w (4 n) | status (n) | the work space of edit_batch (16-byte aligned)
  const size_t in_bytes = (n * 21 + 15) & ~(size_t) 15;
  { int rc = h->scratch (in_bytes + edit_work_bytes (n)); if (rc) return rc; }
  float* d_xyz = (float*) h->d_scratch.p;
  float* d_d = d_xyz + 3 * n;
  float* d_w = d_d + n;
  uint8_t* d_status = (uint8_t*) (d_w + n);
  cudaStream_t s = h->stream;
  CK (cudaMemcpyAsync (d_xyz, xyz, n * 12, cudaMemcpyHostToDevice, s));
  CK (cudaMemcpyAsync (d_d, d, n * 4, cudaMemcpyHostToDevice, s));
  CK (cudaMemcpyAsync (d_w, w, n * 4, cudaMemcpyHostToDevice, s));
  if (int rc = edit_batch (h, d_xyz, n, min_size, d_d, d_w, d_status, h->d_scratch + in_bytes)) return rc;
  if (status)
  {
    CK (cudaMemcpyAsync (status, d_status, n, cudaMemcpyDeviceToHost, s));
    CK (cudaStreamSynchronize (s));
  }
  return B200TSDF_OK;
}

int b200tsdf_dense_device (b200tsdf_t* h, const int32_t box[6], float* d_d, float* d_w, uint8_t* d_rgb, int8_t* d_level)
{
  if (!h) return B200TSDF_EINVAL;
  if (int rc = voxel_read_state (h, "dense crop")) return rc;
  if (!box) return h->fail (B200TSDF_EINVAL, "missing box");
  if (!d_d && !d_w && !d_rgb && !d_level) return h->fail (B200TSDF_EINVAL, "no output buffer");
  for (int a = 0; a < 3; ++a)
    if (!(0 <= box[a] && box[a] < box[a + 3] && box[a + 3] <= h->p.res))
      return h->fail (B200TSDF_EINVAL, "box must satisfy 0 <= lo < hi <= resolution on every axis");
  if (!aligned4 (d_d) || !aligned4 (d_w)) return h->fail (B200TSDF_EINVAL, "d_d and d_w must be 4-byte aligned");
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  DenseBox b;
  b.i0 = box[0]; b.j0 = box[1]; b.k0 = box[2]; b.i1 = box[3]; b.j1 = box[4]; b.k1 = box[5];
  b.ti0 = b.i0 >> 3; b.tj0 = b.j0 >> 3; b.tk0 = b.k0 >> 3;
  const int nti = ((b.i1 - 1) >> 3) - b.ti0 + 1;
  b.ntj = ((b.j1 - 1) >> 3) - b.tj0 + 1; b.ntk = ((b.k1 - 1) >> 3) - b.tk0 + 1;
  const unsigned long long tiles = (unsigned long long) nti * b.ntj * b.ntk;      // one CTA per tile: 2^27 for a whole 4096^3 grid
  if (tiles > (unsigned long long) INT_MAX) return h->fail (B200TSDF_EINVAL, "box too large for one call (more than 2^31 - 1 tiles of 8^3)");
  k_dense<<<(unsigned) tiles, DENSE_THREADS, 0, h->stream>>> (h->p, b, d_d, d_w, d_rgb, (signed char*) d_level);
  CK (cudaGetLastError ());
  note_device_err (h, h->stream);
  return B200TSDF_OK;
}

// ---- renderView / renderColoredView (tsdf_volume_octree.cpp:278-450) ----------------------------------
static int render_args (b200tsdf* h, int downsample, size_t stride, int xyz_off, int normal_off)
{
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "renderView before reset()");
  if (stride < 12 || xyz_off < 0 || normal_off < 0 || (size_t) xyz_off + 12 > stride || (size_t) normal_off + 12 > stride)
    return h->fail (B200TSDF_EINVAL, "bad output point layout (need xyz_off + 12 <= stride and normal_off + 12 <= stride)");
  if (h->p.width / downsample <= 0 || h->p.height / downsample <= 0) return h->fail (B200TSDF_EINVAL, "downsample too large");
  return B200TSDF_OK;
}

// n poses, RENDER_CHUNK per launch: the chunk's records are built on the host (make_render_params), staged in pinned memory and
// copied to the device in one copy ahead of the launch on the handle's stream
static int render_enqueue (b200tsdf* h, int n, const double* poses, int downsample, unsigned char* d_out, size_t stride,
                           int xyz_off, int normal_off, unsigned char* d_rgb)
{
  cudaStream_t s = h->stream;
  const Params& p = h->p;
  const int W = p.width / downsample, H = p.height / downsample;
  const size_t npix = (size_t) W * H;
  for (int i0 = 0; i0 < n; i0 += RENDER_CHUNK)
  {
    const int m = std::min (RENDER_CHUNK, n - i0), sg = h->rrec_seg;
    if (h->rrec_used[sg]) CK (cudaEventSynchronize (h->ev_rrec[sg]));
    RenderParams* recs = h->h_rrec + (size_t) sg * RENDER_CHUNK;
    for (int k = 0; k < m; ++k) make_render_params (h->cfg, p, poses + 16 * (size_t) (i0 + k), downsample, recs[k]);
    CK (cudaMemcpyAsync (h->d_rrec, recs, (size_t) m * sizeof (RenderParams), cudaMemcpyHostToDevice, s));
    CK (cudaEventRecord (h->ev_rrec[sg], s));
    h->rrec_used[sg] = true; h->rrec_seg = (sg + 1) % RENDER_SEGS;
    const dim3 grid ((W + 7) / 8, (H + 7) / 8, m);
    k_render<<<grid, 64, 0, s>>> (p, h->d_rrec, d_out + (size_t) i0 * npix * stride, stride, xyz_off, normal_off,
                                  d_rgb ? d_rgb + (size_t) i0 * npix * 3 : nullptr);
    CK (cudaGetLastError ());
  }
  return B200TSDF_OK;
}

int b200tsdf_render_batch_device (b200tsdf_t* h, int n, const double* poses_c2w, int downsample, void* d_out, size_t stride,
                                  int xyz_off, int normal_off, uint8_t* d_rgb)
{
  if (!h || n < 1 || !poses_c2w || !d_out || downsample < 1) return B200TSDF_EINVAL;
  if (int rc = render_args (h, downsample, stride, xyz_off, normal_off)) return rc;
  if ((stride & 3) || (xyz_off & 3) || (normal_off & 3) || ((uintptr_t) d_out & 3))
    return h->fail (B200TSDF_EINVAL, "bad output point layout (device images need 4-byte aligned d_out, stride, xyz_off and normal_off)");
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  if (int rc = render_enqueue (h, n, poses_c2w, downsample, (unsigned char*) d_out, stride, xyz_off, normal_off, d_rgb)) return rc;
  note_device_err (h, h->stream);
  return B200TSDF_OK;
}

int b200tsdf_render (b200tsdf_t* h, const double* pose, int downsample, void* out, size_t stride,
                     int xyz_off, int normal_off, uint8_t* rgb_out)
{
  if (!h || !pose || !out || downsample < 1) return B200TSDF_EINVAL;
  if (int rc = render_args (h, downsample, stride, xyz_off, normal_off)) return rc;
  cudaSetDevice (h->device);
  const size_t npix = (size_t) (h->p.width / downsample) * (h->p.height / downsample);
  // a batch of one into scratch ({xyz, normal} per pixel), then only xyz and normal go into the caller's points: the other
  // bytes keep what the caller put there
  { int rc = h->scratch (npix * 6 * sizeof (float) + npix * 3 + 64); if (rc) return rc; }
  unsigned char* d_rgb = rgb_out ? h->d_scratch + npix * 6 * sizeof (float) : nullptr;
  cudaStream_t s = h->stream;
  if (int rc = render_enqueue (h, 1, pose, downsample, h->d_scratch, 6 * sizeof (float), 0, 3 * sizeof (float), d_rgb)) return rc;
  std::vector<float> tmp (npix * 6);
  CK (cudaMemcpyAsync (tmp.data (), h->d_scratch, npix * 6 * sizeof (float), cudaMemcpyDeviceToHost, s));
  if (rgb_out) CK (cudaMemcpyAsync (rgb_out, d_rgb, npix * 3, cudaMemcpyDeviceToHost, s));
  note_device_err (h, s);
  CK (cudaStreamSynchronize (s));
  if (int rc = pending_device_err (h)) return rc;
  unsigned char* base = (unsigned char*) out;
  for (size_t i = 0; i < npix; ++i)
  {
    std::memcpy (base + i * stride + xyz_off, &tmp[6 * i], 12);
    std::memcpy (base + i * stride + normal_off, &tmp[6 * i + 3], 12);
  }
  return B200TSDF_OK;
}

} // extern "C"

// ---- marching cubes (marching_cubes_tsdf_octree.cpp:108-236) --------------------------------------------
// The one mesh path of b200tsdf_mesh, b200tsdf_mesh_device and b200tsdf_mesh_cells_device: the brick walk as count and emit
// launches, handed to sort (launch), which runs them through sorted_records with the caller's destination.  A triangle is one
// record of 9 words (its three vertices) and 9 colour bytes, which is already the layout of the result.  mask (host, 8^C
// bytes, or null for every cell) restricts the walk to the leaves of the selected coarse cells; cell_tris (host, 8^C, or null)
// receives each cell's triangle count from the count pass.
template <typename Sort>
static int marching_cubes (b200tsdf* h, float w_min, int color_mode, const Sort& sort, const uint8_t* mask = nullptr,
                           unsigned long long* cell_tris = nullptr)
{
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "reconstruct before reset()");
  cudaSetDevice (h->device);
  const Params& p = h->p;
  McParams mc;
  make_mc_params (h->cfg, p, w_min, color_mode, mc);
  cudaStream_t s = h->stream;
  const size_t ncells = (size_t) 1 << (3 * p.C);
  if (mask)
  {
    CK (cudaMemcpyAsync (h->d_cell_mask, mask, ncells, cudaMemcpyHostToDevice, s));
    mc.cell_mask = h->d_cell_mask;
  }
  if (cell_tris)
  {
    CK (cudaMemsetAsync (h->d_cell_tris, 0, ncells * sizeof (unsigned long long), s));
    mc.cell_tris = h->d_cell_tris;
  }
  int* list = nullptr;
  const int nb = list_bricks (h, list);
  if (nb < 0) return nb;
  const unsigned bgrid = (unsigned) (((size_t) nb * 32 + 127) / 128), rgrid = (unsigned) ((h->vol.root_n + 127) / 128);
  auto launch = [&] (auto emit, unsigned long long* total, unsigned long long* keys, void* v, unsigned char* c)
  {
    constexpr bool E = decltype (emit)::value;
    if (mask || cell_tris)
    {
      if (nb) k_mesh_bricks<E, true><<<bgrid, 128, 0, s>>> (p, mc, list, nb, total, (float*) v, c, keys);
      k_mesh_roots<E, true><<<rgrid, 128, 0, s>>> (p, mc, total, (float*) v, c, keys);
    }
    else
    {
      if (nb) k_mesh_bricks<E, false><<<bgrid, 128, 0, s>>> (p, mc, list, nb, total, (float*) v, c, keys);
      k_mesh_roots<E, false><<<rgrid, 128, 0, s>>> (p, mc, total, (float*) v, c, keys);
    }
  };
  if (int rc = sort (launch)) return rc;
  if (cell_tris) CK (cudaMemcpyAsync (cell_tris, h->d_cell_tris, ncells * sizeof (unsigned long long), cudaMemcpyDeviceToHost, s));
  return check_device_err (h);
}

extern "C" {

int b200tsdf_mesh (b200tsdf_t* h, float w_min, int color_mode, float** verts, uint8_t** rgb, size_t* nverts)
{
  if (!h || !verts || !nverts) return B200TSDF_EINVAL;
  std::free (h->mesh_c); h->mesh_c = nullptr;
  unsigned long long ntri = 0;
  const int key_bits = 3 * h->p.L + 3;
  auto sort = [&] (const auto& launch)
  { return sorted_records_host (h, "triangles", 9, key_bits, launch, h->mesh_v, color_mode ? &h->mesh_c : nullptr, ntri); };
  if (int rc = marching_cubes (h, w_min, color_mode, sort)) return rc;
  *nverts = (size_t) ntri * 3;
  *verts = ntri ? (float*) h->mesh_v : nullptr;
  if (rgb) *rgb = ntri ? (uint8_t*) h->mesh_c : nullptr;
  return B200TSDF_OK;
}

int b200tsdf_mesh_device (b200tsdf_t* h, float w_min, int color_mode, float* d_verts, uint8_t* d_rgb, size_t capacity,
                          size_t* nverts)
{
  return b200tsdf_mesh_cells_device (h, w_min, color_mode, nullptr, d_verts, d_rgb, capacity, nverts, nullptr);
}

int b200tsdf_mesh_cells_device (b200tsdf_t* h, float w_min, int color_mode, const uint8_t* mask, float* d_verts, uint8_t* d_rgb,
                                size_t capacity, size_t* nverts, int64_t* cell_nverts)
{
  if (!h || !nverts) return B200TSDF_EINVAL;
  *nverts = 0;
  if ((uintptr_t) d_verts & 3) return h->fail (B200TSDF_EINVAL, "d_verts must be 4-byte aligned");
  if ((mask || cell_nverts) && h->has_volume && h->p.shard_count > 1)
    return h->fail (B200TSDF_ESTATE, "mesh of selected cells on a shard: mesh the replica built by b200tsdf_gather_volume");
  unsigned long long ntri = 0;
  auto dest = [&] (unsigned long long n, void*& v_out, unsigned char*& c_out)
  {
    *nverts = (size_t) n * 3;
    if (!d_verts) return (int) B200TSDF_OK;                                        // count only
    if (capacity < *nverts)
      return h->fail (B200TSDF_EINVAL, "capacity " + std::to_string (capacity) + " < " + std::to_string (*nverts) + " vertices");
    v_out = d_verts; c_out = color_mode ? d_rgb : nullptr;
    return (int) B200TSDF_OK;
  };
  auto sort = [&] (const auto& launch) { return sorted_records (h, "triangles", 9, 3 * h->p.L + 3, launch, dest, ntri); };
  // the per-cell triangle counts land in cell_nverts itself, then become vertex counts
  static_assert (sizeof (int64_t) == sizeof (unsigned long long), "cell_nverts holds the device's 64-bit counts");
  if (int rc = marching_cubes (h, w_min, color_mode, sort, mask, reinterpret_cast<unsigned long long*> (cell_nverts))) return rc;
  if (cell_nverts)
    for (size_t c = 0, n = (size_t) 1 << (3 * h->p.C); c < n; ++c) cell_nverts[c] *= 3;
  return B200TSDF_OK;
}

int b200tsdf_changed_cells (b200tsdf_t* h, uint64_t since, uint64_t* now, uint8_t* mask)
{
  if (!h || !now) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "changed_cells before reset()");
  if (h->p.shard_count > 1)
    return h->fail (B200TSDF_ESTATE, "changed_cells on a shard: shards keep no change epochs; mesh the replica built by b200tsdf_gather_volume");
  cudaSetDevice (h->device);
  cudaStream_t s = h->stream;
  const int n = 1 << h->p.C;
  const size_t ncells = (size_t) n * n * n;
  if (mask && !(since == 0 || h->all_epoch > since))
  {
    k_changed_cells<<<(unsigned) ((ncells + 255) / 256), 256, 0, s>>> (h->p.C, h->d_cell_epoch, (unsigned long long) since, h->d_cell_mask);
    CK (cudaGetLastError ());
    CK (cudaMemcpyAsync (mask, h->d_cell_mask, ncells, cudaMemcpyDeviceToHost, s));
  }
  if (int rc = check_device_err (h)) return rc;              // (waits for the handle's stream)
  if (int rc = pending_device_err (h)) return rc;
  if (mask && (since == 0 || h->all_epoch > since)) std::memset (mask, 1, ncells);
  *now = h->epoch;
  return B200TSDF_OK;
}

} // extern "C"

// ---- flattenVertices / cleanupMesh on device arrays (b2_mesh_flatten / b2_mesh_cleanup, meshpost.cu) ----------------------
static bool overlaps (const void* a, size_t na, const void* b, size_t nb)
{
  const uintptr_t x = (uintptr_t) a, y = (uintptr_t) b;
  return na && nb && x < y + nb && y < x + na;
}

// the checks that need no data; the routine checks the indices on the device
static int meshpost_device_args (b200tsdf* h, const float* d_verts, size_t nverts, const int32_t* d_tris, size_t ntris,
                                 const float* d_out_verts, const int32_t* d_out_tris, size_t* out_nverts, size_t* out_ntris)
{
  if (!out_nverts || !out_ntris) return h->fail (B200TSDF_EINVAL, "null argument");
  *out_nverts = 0; *out_ntris = 0;
  if ((!d_verts || !d_out_verts) && nverts) return h->fail (B200TSDF_EINVAL, "null vertex array");
  if (!d_out_tris && ntris) return h->fail (B200TSDF_EINVAL, "null triangle array");
  if (nverts >= (size_t) 1 << 31 || ntris >= ((size_t) 1 << 31) / 3) return h->fail (B200TSDF_EINVAL, "mesh too large for 32-bit indices");
  if (!d_tris && nverts != 3 * ntris) return h->fail (B200TSDF_EINVAL, "a triangle soup (d_tris == NULL) needs nverts == 3 * ntris");
  if (((uintptr_t) d_verts | (uintptr_t) d_tris | (uintptr_t) d_out_verts | (uintptr_t) d_out_tris) & 3)
    return h->fail (B200TSDF_EINVAL, "device arrays must be 4-byte aligned");
  const size_t bv = 12 * nverts, bt = 12 * ntris, bt_in = d_tris ? bt : 0;          // a soup has no triangle input
  if (overlaps (d_out_verts, bv, d_verts, bv) || overlaps (d_out_verts, bv, d_tris, bt_in) || overlaps (d_out_verts, bv, d_out_tris, bt)
      || overlaps (d_out_tris, bt, d_verts, bv) || overlaps (d_out_tris, bt, d_tris, bt_in))
    return h->fail (B200TSDF_EINVAL, "outputs overlap the inputs or each other");
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "mesh post-processing before reset()");
  cudaSetDevice (h->device);
  return pending_device_err (h);
}

extern "C" {

int b200tsdf_mesh_flatten_device (b200tsdf_t* h, const float* d_verts, size_t nverts, const int32_t* d_tris, size_t ntris,
                                  float min_dist, float* d_out_verts, int32_t* d_out_tris, size_t* out_nverts, size_t* out_ntris)
{
  if (!h) return B200TSDF_EINVAL;
  if (int rc = meshpost_device_args (h, d_verts, nverts, d_tris, ntris, d_out_verts, d_out_tris, out_nverts, out_ntris)) return rc;
  B2MeshScratch scratch;
  std::string err;
  if (int rc = b2_mesh_flatten (h->stream, scratch, d_verts, nverts, d_tris, ntris, min_dist, d_out_verts, d_out_tris,
                                out_nverts, out_ntris, err))
    return h->fail (rc, "flattenVertices: " + err);
  return B200TSDF_OK;
}

int b200tsdf_mesh_cleanup_device (b200tsdf_t* h, const float* d_verts, size_t nverts, const int32_t* d_tris, size_t ntris,
                                  float face_dist, int min_neighbors,
                                  float* d_out_verts, int32_t* d_out_tris, size_t* out_nverts, size_t* out_ntris)
{
  if (!h) return B200TSDF_EINVAL;
  if (min_neighbors < 1 || min_neighbors > 16) return h->fail (B200TSDF_EINVAL, "min_neighbors must be in 1..16");
  if (int rc = meshpost_device_args (h, d_verts, nverts, d_tris, ntris, d_out_verts, d_out_tris, out_nverts, out_ntris)) return rc;
  B2MeshScratch scratch;
  std::string err;
  if (int rc = b2_mesh_cleanup (h->stream, scratch, d_verts, nverts, d_tris, ntris, face_dist, min_neighbors, d_out_verts, d_out_tris,
                                out_nverts, out_ntris, err))
    return h->fail (rc, "cleanupMesh: " + err);
  return B200TSDF_OK;
}

void b200tsdf_free (void* p) { (void) p; /* mesh buffers are owned by the handle */ }

int b200tsdf_voxel_center (const b200tsdf_t* h, int64_t x, int64_t y, int64_t z, float* o)
{
  if (!h || !o || !h->has_volume) return B200TSDF_EINVAL;
  o[0] = voxel_center1 (h->p, x); o[1] = voxel_center1 (h->p, y); o[2] = voxel_center1 (h->p, z);
  return B200TSDF_OK;
}

int b200tsdf_voxel_index (const b200tsdf_t* h, float x, float y, float z, int32_t* o, int32_t* inside)
{
  if (!h || !o || !h->has_volume) return B200TSDF_EINVAL;
  int xi, yi, zi;
  bool in = voxel_index (h->p, x, y, z, xi, yi, zi);
  o[0] = xi; o[1] = yi; o[2] = zi;
  if (inside) *inside = in;
  return B200TSDF_OK;
}

int b200tsdf_frustum_cull (b200tsdf_t* h, const double* pose, uint8_t* mask, int32_t* kept)
{
  if (!h || !pose || !mask) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "cull before reset()");
  cudaSetDevice (h->device);
  const Params& p = h->p;
  Planes P;
  b2host::frustum_planes (pose, p.width, p.height, p.fx, p.fy, p.min_sensor, p.max_sensor, P.pl);
  int ncells = 1 << (3 * p.C);
  DevBuf<unsigned char> d_mask (h->stream);
  CK (d_mask.alloc (ncells));
  k_cull<<<(ncells + 127) / 128, 128, 0, h->stream>>> (p, P, d_mask);
  CK (cudaMemcpyAsync (mask, d_mask, ncells, cudaMemcpyDeviceToHost, h->stream));
  CK (cudaStreamSynchronize (h->stream));
  if (kept) { int k = 0; for (int i = 0; i < ncells; ++i) k += mask[i]; *kept = k; }
  return B200TSDF_OK;
}

} // extern "C"

namespace {

// Octree::getLeaves (nlevels) on the device, one record per selected node (leaf_selected), in the reference's depth-first
// order.  The records land in `out` (3 x 32 bits each, malloc'ed, owned by the handle).  The brick list lives in the handle's
// grow-only scratch (pool-sized, like the query buffers); the record and sort buffers are sized by the result (hundreds of MB
// for a large volume) and are released before returning rather than kept on the handle.
int enumerate_leaves (b200tsdf* h, int nlevels, bool occupied, const char* what, void*& out, size_t* n)
{
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, std::string (what) + " before reset()");
  if (h->p.shard_count > 1)
    return h->fail (B200TSDF_ESTATE, std::string (what) + " on a shard: a shard keeps the coarse cells it does not own as unsplit leaves; "
                    "enumerate on the replica built by b200tsdf_gather_volume");
  cudaSetDevice (h->device);
  if (int rc = pending_device_err (h)) return rc;
  const Params& p = h->p;
  cudaStream_t s = h->stream;
  unsigned long long count = 0;
  if (!occupied && nlevels >= 0 && (nlevels < p.C || nlevels == 0))
  {
    // every node of that depth exists (Octree::init) and none is ever pruned: 8^nlevels records, already in order
    count = 1ull << (3 * nlevels);
    DevBuf<uint32_t> rec (s);
    if (rec.alloc (count * 3)) return alloc_failed (h, "voxel centres");
    k_leaves_level<<<(unsigned) ((count + 127) / 128), 128, 0, s>>> (p, nlevels, count, rec);
    if (int rc = download (h, rec, count * 12, out)) return rc;
  }
  else
  {
    int* list = nullptr;
    const int nb = list_bricks (h, list);
    if (nb < 0) return nb;
    const int occ = occupied ? 1 : 0;
    const unsigned bgrid = (unsigned) (((size_t) nb * 32 + 127) / 128), rgrid = (unsigned) ((h->vol.root_n + 127) / 128);
    auto launch = [&] (auto emit, unsigned long long* total, unsigned long long* keys, void* rec, unsigned char*)
    {
      constexpr bool E = decltype (emit)::value;
      if (nb) k_leaves_bricks<E><<<bgrid, 128, 0, s>>> (p, list, nb, nlevels, occ, total, keys, (uint32_t*) rec);
      k_leaves_roots<E><<<rgrid, 128, 0, s>>> (p, nlevels, occ, total, keys, (uint32_t*) rec);
    };
    if (int rc = sorted_records_host (h, "leaf records", 3, 3 * p.L, launch, out, nullptr, count)) return rc;
  }
  h->d2h_bytes += (long long) (count * 12);
  *n = (size_t) count;
  return check_device_err (h);
}

} // namespace

extern "C" {

int b200tsdf_voxel_centers (b200tsdf_t* h, int nlevels, float** xyz, size_t* n)
{
  if (!h || !xyz || !n) return B200TSDF_EINVAL;
  *xyz = nullptr; *n = 0;
  int rc = enumerate_leaves (h, nlevels, false, "getVoxelCenters", h->leaf_xyz, n);
  if (rc) { *n = 0; return rc; }
  *xyz = (float*) h->leaf_xyz;
  return B200TSDF_OK;
}

int b200tsdf_occupied_voxel_indices (b200tsdf_t* h, int32_t** ijk, size_t* n)
{
  if (!h || !ijk || !n) return B200TSDF_EINVAL;
  *ijk = nullptr; *n = 0;
  int rc = enumerate_leaves (h, -1, true, "getOccupiedVoxelIndices", h->leaf_ijk, n);
  if (rc) { *n = 0; return rc; }
  *ijk = (int32_t*) h->leaf_ijk;
  return B200TSDF_OK;
}

int b200tsdf_is_empty (b200tsdf_t* h, int32_t* out)
{
  if (!h || !out) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "isEmpty before reset()");
  *out = h->is_empty ? 1 : 0;
  return B200TSDF_OK;
}

} // extern "C"

extern "C" {

// Diagnostics (not part of include/b200tsdf.h): phase timing of k_celltop_up.  First call arms it; every call returns and
// clears the 16 counters ([0..5] max SM cycles << 32 | tag of total / level-3 / level-2 / level-1 / cell / wait-before-first-cell,
// [6..10] slow level-2 nodes, slow level-1 nodes, cell leaf visits, cell fall-throughs, cells folded; [11] frames whose k_front
// waited per supercell, [12] frames whose k_front waited for the previous frame's last kernel).
int b200tsdf_debug_timing (b200tsdf_t* h, unsigned long long* out16)
{
  if (!h || !out16) return B200TSDF_EINVAL;
  cudaSetDevice (h->device);
  CK (cudaStreamSynchronize (h->stream));
  if (!h->d_dbg)
  {
    CK (h->d_dbg.grow (16)); CK (cudaMemset (h->d_dbg, 0, 16 * 8));
    h->p.dbg = h->d_dbg;                                   // armed from the next frame on (this handle only)
    drop_batch_graphs (h);
  }
  CK (cudaMemcpy (out16, h->d_dbg, 16 * 8, cudaMemcpyDeviceToHost));
  CK (cudaMemset (h->d_dbg, 0, 16 * 8));
  return B200TSDF_OK;
}

int b200tsdf_profile_begin (b200tsdf_t* h)
{
  if (!h) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "profile before reset()");
  cudaSetDevice (h->device);
  CK (cudaStreamSynchronize (h->copy_stream));
  CK (cudaStreamSynchronize (h->stream));
  h->drain_kring (0);
  h->prof_ms_kernel = 0; h->prof_kernel_launches = 0; h->prof_frames = 0;
  h->time_frames = true; h->prof_graph0 = h->graph_launches; h->prof_nvlink0 = h->nvlink_bytes;
  h->prof_launch0 = h->launches; h->prof_h2d0 = h->h2d_bytes; h->prof_d2h0 = h->d2h_bytes;
  CK (cudaMemcpy (h->prof_stats0, h->d_stats, sizeof (h->prof_stats0), cudaMemcpyDeviceToHost));
  CK (cudaEventRecord (h->ev_p0, h->stream));
  return B200TSDF_OK;
}

int b200tsdf_profile_end (b200tsdf_t* h, b200tsdf_profile* out)
{
  if (!h || !out) return B200TSDF_EINVAL;
  cudaSetDevice (h->device);
  CK (cudaEventRecord (h->ev_p1, h->stream));
  CK (cudaStreamSynchronize (h->copy_stream));
  CK (cudaEventSynchronize (h->ev_p1));
  h->drain_kring (0);
  std::memset (out, 0, sizeof (*out));
  float ms = 0.f;
  CK (cudaEventElapsedTime (&ms, h->ev_p0, h->ev_p1));
  unsigned long long st[ST_N];
  CK (cudaMemcpy (st, h->d_stats, sizeof (st), cudaMemcpyDeviceToHost));
  out->ms_elapsed = ms;
  out->ms_kernel = h->prof_ms_kernel; out->kernel_launches = h->prof_kernel_launches;
  out->total_launches = h->launches - h->prof_launch0;
  out->n_frames = h->prof_frames;
  out->n_updates = (int64_t) (st[ST_UPDATES] - h->prof_stats0[ST_UPDATES]);
  out->n_node_visits = (int64_t) (st[ST_VISITS] - h->prof_stats0[ST_VISITS]);
  out->ms_kernel_device = 1e-6 * (double) (st[5] - h->prof_stats0[5]);
  out->kernel_launches_device = (int64_t) (st[6] - h->prof_stats0[6]);
  out->graph_launches = h->graph_launches - h->prof_graph0;
  out->nvlink_bytes = h->nvlink_bytes - h->prof_nvlink0;
  h->time_frames = false;
  out->h2d_bytes = h->h2d_bytes - h->prof_h2d0; out->d2h_bytes = h->d2h_bytes - h->prof_d2h0;
  return check_device_err (h);
}

} // extern "C"

// ---------------------------------------------------------------------------------------------
// host snapshot: a compact host copy of the volume with its own (re-hashed) directory, walked with
// the same tsdf_core.cuh routines.  Used for the node dump (tests) and the recursive .vol writer
// (I/O); it is not a compute path.
// ---------------------------------------------------------------------------------------------
namespace {

struct Snapshot
{
  Params p{};
  std::vector<uint64_t> keys; std::vector<float2> nodes; std::vector<uint32_t> split;
  std::vector<uchar4> rgb; std::vector<float> M; std::vector<int> ns;
  std::vector<float2> root_dw; std::vector<uint32_t> root_split; std::vector<uchar4> root_rgb;
  std::vector<float> root_M; std::vector<int> root_ns;
  std::vector<float4> rgbn, root_rgbn;
  int err = 0;
};

int take_snapshot (b200tsdf* h, Snapshot& S)
{
  cudaSetDevice (h->device);
  int rc = b200tsdf_sync (h);
  if (rc) return rc;
  const Params& dp = h->p;
  cudaStream_t s = h->stream;
  int* d_list = nullptr;
  const int nb = list_bricks (h, d_list);
  if (nb < 0) return nb;
  std::vector<int> list (nb);
  std::vector<uint64_t> dkeys (h->vol.pool);
  CK (cudaMemcpy (dkeys.data (), dp.keys, h->vol.pool * sizeof (uint64_t), cudaMemcpyDeviceToHost));
  if (nb) CK (cudaMemcpy (list.data (), d_list, (size_t) nb * sizeof (int), cudaMemcpyDeviceToHost));
  const size_t nn = (size_t) nb * BRICK_NODES;
  DevBuf<float2> g_nodes (s); DevBuf<uint32_t> g_split (s); DevBuf<uchar4> g_rgb (s); DevBuf<float> g_M (s); DevBuf<int> g_ns (s); DevBuf<float4> g_q (s);
  CK (g_nodes.alloc (nn)); CK (g_split.alloc ((size_t) nb * BRICK_SPLIT_WORDS));
  if (dp.rgb) CK (g_rgb.alloc (nn));
  if (dp.M) { CK (g_M.alloc (nn)); CK (g_ns.alloc (nn)); }
  if (dp.rgbn) CK (g_q.alloc (nn));
  if (nb)
  {
    k_gather_bricks<<<nb, 128, 0, s>>> (dp, d_list, nb, g_nodes, g_split, g_rgb, g_M, g_ns);
    if (dp.rgbn) k_gather_rgbn<<<nb, 128, 0, s>>> (dp, d_list, nb, g_q);
  }
  CK (cudaStreamSynchronize (s));
  std::vector<float2> c_nodes (nn); std::vector<uint32_t> c_split ((size_t) nb * BRICK_SPLIT_WORDS);
  std::vector<uchar4> c_rgb; std::vector<float> c_M; std::vector<int> c_ns; std::vector<float4> c_rgbn;
  if (nb)
  {
    CK (cudaMemcpy (c_nodes.data (), g_nodes, c_nodes.size () * sizeof (float2), cudaMemcpyDeviceToHost));
    CK (cudaMemcpy (c_split.data (), g_split, c_split.size () * sizeof (uint32_t), cudaMemcpyDeviceToHost));
    if (dp.rgb) { c_rgb.resize (nn); CK (cudaMemcpy (c_rgb.data (), g_rgb, nn * sizeof (uchar4), cudaMemcpyDeviceToHost)); }
    if (dp.M)
    {
      c_M.resize (nn); c_ns.resize (nn);
      CK (cudaMemcpy (c_M.data (), g_M, nn * sizeof (float), cudaMemcpyDeviceToHost));
      CK (cudaMemcpy (c_ns.data (), g_ns, nn * sizeof (int), cudaMemcpyDeviceToHost));
    }
    if (dp.rgbn) { c_rgbn.resize (nn); CK (cudaMemcpy (c_rgbn.data (), g_q, nn * sizeof (float4), cudaMemcpyDeviceToHost)); }
  }
  // compact directory
  size_t hp = 16;
  while (hp < (size_t) nb * 2) hp <<= 1;
  S.p = dp;
  S.keys.assign (hp, KEY_EMPTY);
  S.nodes.assign (hp * BRICK_NODES, make_float2 (-1.f, 0.f));
  S.split.assign (hp * BRICK_SPLIT_WORDS, 0u);
  if (dp.rgb) S.rgb.assign (hp * BRICK_NODES, make_uchar4 (0, 0, 0, 0));
  if (dp.M) { S.M.assign (hp * BRICK_NODES, 0.f); S.ns.assign (hp * BRICK_NODES, 0); }
  if (dp.rgbn) S.rgbn.assign (hp * BRICK_NODES, make_float4 (0.f, 0.f, 0.f, 0.f));
  S.p.rgbn = dp.rgbn ? S.rgbn.data () : nullptr;
  S.p.keys = S.keys.data (); S.p.pool_mask = (uint32_t) (hp - 1);
  S.p.nodes = S.nodes.data (); S.p.split = S.split.data ();
  S.p.rgb = dp.rgb ? S.rgb.data () : nullptr; S.p.M = dp.M ? S.M.data () : nullptr; S.p.ns = dp.M ? S.ns.data () : nullptr;
  S.p.err = &S.err;
  for (int i = 0; i < nb; ++i)
  {
    int t, bx, by, bz;
    brick_key_decode (dkeys[list[i]], t, bx, by, bz);
    int slot = find_or_insert_brick (S.p, t, bx, by, bz);
    std::memcpy (&S.nodes[(size_t) slot * BRICK_NODES], &c_nodes[(size_t) i * BRICK_NODES], BRICK_NODES * sizeof (float2));
    std::memcpy (&S.split[(size_t) slot * BRICK_SPLIT_WORDS], &c_split[(size_t) i * BRICK_SPLIT_WORDS], BRICK_SPLIT_WORDS * sizeof (uint32_t));
    if (dp.rgb) std::memcpy (&S.rgb[(size_t) slot * BRICK_NODES], &c_rgb[(size_t) i * BRICK_NODES], BRICK_NODES * sizeof (uchar4));
    if (dp.rgbn) std::memcpy (&S.rgbn[(size_t) slot * BRICK_NODES], &c_rgbn[(size_t) i * BRICK_NODES], BRICK_NODES * sizeof (float4));
    if (dp.M)
    {
      std::memcpy (&S.M[(size_t) slot * BRICK_NODES], &c_M[(size_t) i * BRICK_NODES], BRICK_NODES * sizeof (float));
      std::memcpy (&S.ns[(size_t) slot * BRICK_NODES], &c_ns[(size_t) i * BRICK_NODES], BRICK_NODES * sizeof (int));
    }
  }
  size_t rn = h->vol.root_n;
  S.root_dw.resize (rn); S.root_split.resize ((rn + 31) / 32);
  CK (cudaMemcpy (S.root_dw.data (), dp.root_dw, rn * sizeof (float2), cudaMemcpyDeviceToHost));
  CK (cudaMemcpy (S.root_split.data (), dp.root_split, S.root_split.size () * sizeof (uint32_t), cudaMemcpyDeviceToHost));
  S.p.root_dw = S.root_dw.data (); S.p.root_split = S.root_split.data ();
  S.p.root_rgb = nullptr; S.p.root_M = nullptr; S.p.root_ns = nullptr; S.p.root_rgbn = nullptr;
  if (dp.root_rgbn) { S.root_rgbn.resize (rn); CK (cudaMemcpy (S.root_rgbn.data (), dp.root_rgbn, rn * sizeof (float4), cudaMemcpyDeviceToHost)); S.p.root_rgbn = S.root_rgbn.data (); }
  if (dp.root_rgb) { S.root_rgb.resize (rn); CK (cudaMemcpy (S.root_rgb.data (), dp.root_rgb, rn * sizeof (uchar4), cudaMemcpyDeviceToHost)); S.p.root_rgb = S.root_rgb.data (); }
  if (dp.root_M)
  {
    S.root_M.resize (rn); S.root_ns.resize (rn);
    CK (cudaMemcpy (S.root_M.data (), dp.root_M, rn * sizeof (float), cudaMemcpyDeviceToHost));
    CK (cudaMemcpy (S.root_ns.data (), dp.root_ns, rn * sizeof (int), cudaMemcpyDeviceToHost));
    S.p.root_M = S.root_M.data (); S.p.root_ns = S.root_ns.data ();
  }
  return B200TSDF_OK;
}

struct NodeRec { int32_t k[4]; float d, w; uint8_t split, r, g, b; float M; int32_t ns; float q[4]; };

void node_payload (const Params& p, const NodePos& n, NodeRec& r)
{
  float2 dw = *node_dw (p, n);
  r.d = dw.x; r.w = dw.y; r.r = r.g = r.b = 0; r.M = 0.f; r.ns = 0; r.q[0] = r.q[1] = r.q[2] = r.q[3] = 0.f;
  if (p.color_norm)
  {
    const float4 q = *node_rgbn (p, n); r.q[0] = q.x; r.q[1] = q.y; r.q[2] = q.z; r.q[3] = q.w;
    const uchar4 c = node_get_rgb (p, n); r.r = c.x; r.g = c.y; r.b = c.z;                 // getRGB, octree.cpp:396-402
  }
  if (n.slot < 0)
  {
    if (p.root_rgb && !p.color_norm) { uchar4 c = p.root_rgb[n.idx]; r.r = c.x; r.g = c.y; r.b = c.z; }
    if (p.root_M) { r.M = p.root_M[n.idx]; r.ns = p.root_ns[n.idx]; }
  }
  else
  {
    size_t i = (size_t) n.slot * BRICK_NODES + n.idx;
    if (p.rgb && !p.color_norm) { uchar4 c = p.rgb[i]; r.r = c.x; r.g = c.y; r.b = c.z; }
    if (p.M) { r.M = p.M[i]; r.ns = p.ns[i]; }
  }
}

void collect_nodes (const Params& p, const NodePos& n, std::vector<NodeRec>& out)
{
  NodeRec r; r.k[0] = n.level; r.k[1] = n.x; r.k[2] = n.y; r.k[3] = n.z;
  node_payload (p, n, r);
  bool sp = is_split (p, n);
  r.split = sp;
  out.push_back (r);
  if (!sp) return;
  int cs = children_slot (p, n, false);
  if (cs < 0) return;
  for (int c = 0; c < 8; ++c) collect_nodes (p, make_child (p, n, c, cs), out);
}

// OctreeNode::serialize (octree.cpp:289-304) / RGBNode::serialize (:360-367), recursive
void write_vol_node (const Params& p, std::FILE* f, const NodePos& n, bool have_state)
{
  NodeRec r; r.d = -1.f; r.w = 0.f; r.r = r.g = r.b = 0; r.M = 0.f; r.ns = 0; r.q[0] = r.q[1] = r.q[2] = r.q[3] = 0.f;
  if (have_state) node_payload (p, n, r);
  // RGBNormalized::serialize writes sizeof (uint8_t) of each of its four FLOATS, i.e. their first bytes (octree.cpp:417-424)
  if (p.color_norm) for (int k = 0; k < 4; ++k) std::fwrite (&r.q[k], 1, 1, f);
  else if (p.color) { std::fwrite (&r.r, 1, 1, f); std::fwrite (&r.g, 1, 1, f); std::fwrite (&r.b, 1, 1, f); }
  std::fwrite (&r.d, 4, 1, f); std::fwrite (&r.w, 4, 1, f);
  std::fwrite (&n.cx, 4, 1, f); std::fwrite (&n.cy, 4, 1, f); std::fwrite (&n.cz, 4, 1, f);
  std::fwrite (&n.size, 4, 1, f); std::fwrite (&r.M, 4, 1, f); std::fwrite (&r.ns, 4, 1, f);
  bool sp = have_state ? is_split (p, n) : true;
  int cs = -1;
  if (sp && have_state) { cs = children_slot (p, n, false); if (cs < 0) sp = false; }
  size_t nchild = sp ? 8 : 0;
  std::fwrite (&nchild, sizeof (size_t), 1, f);
  if (!sp) return;
  for (int c = 0; c < 8; ++c)
  {
    if (have_state) write_vol_node (p, f, make_child (p, n, c, cs), true);
    else
    {
      // levels above the root arrays carry no state: geometry only
      NodePos ch = n;
      int bx = (c >> 2) & 1, by = (c >> 1) & 1, bz = c & 1;
      float off = n.size * 0.25f;
      ch.level = n.level + 1; ch.x = 2 * n.x + bx; ch.y = 2 * n.y + by; ch.z = 2 * n.z + bz;
      ch.cx = bx ? n.cx + off : n.cx - off; ch.cy = by ? n.cy + off : n.cy - off; ch.cz = bz ? n.cz + off : n.cz - off;
      ch.size = n.size * 0.5f;
      if (ch.level == p.Rtop) { ch.slot = -1; ch.idx = root_index (p, ch.x, ch.y, ch.z); write_vol_node (p, f, ch, true); }
      else write_vol_node (p, f, ch, false);
    }
  }
}

std::string fmt16 (double x) { char b[64]; std::snprintf (b, sizeof (b), "%.16g", x); return b; }

} // namespace

extern "C" {

int64_t b200tsdf_download_nodes (b200tsdf_t* h, int32_t* keys, float* dw, uint8_t* flags,
                                 uint8_t* rgb, float* M, int32_t* ns)
{
  if (!h || !h->has_volume) return B200TSDF_EINVAL;
  Snapshot S;
  int rc = take_snapshot (h, S);
  if (rc) return rc;
  const Params& p = S.p;
  std::vector<NodeRec> recs;
  int n = 1 << p.C;
  for (int x = 0; x < n; ++x) for (int y = 0; y < n; ++y) for (int z = 0; z < n; ++z)
  {
    NodePos nd;
    if (!locate_node (p, p.C, x, y, z, nd)) return h->fail (B200TSDF_ESTATE, "coarse cell without storage");
    collect_nodes (p, nd, recs);
  }
  if (!keys && !dw && !flags && !rgb && !M && !ns) return (int64_t) recs.size ();
  std::sort (recs.begin (), recs.end (), [] (const NodeRec& a, const NodeRec& b) {
    return std::lexicographical_compare (a.k, a.k + 4, b.k, b.k + 4); });
  for (size_t i = 0; i < recs.size (); ++i)
  {
    const NodeRec& r = recs[i];
    if (keys) std::memcpy (keys + 4 * i, r.k, 16);
    if (dw) { dw[2 * i] = r.d; dw[2 * i + 1] = r.w; }
    if (flags) flags[i] = r.split;
    if (rgb) { rgb[3 * i] = r.r; rgb[3 * i + 1] = r.g; rgb[3 * i + 2] = r.b; }
    if (M) M[i] = r.M;
    if (ns) ns[i] = r.ns;
  }
  return (int64_t) recs.size ();
}

int64_t b200tsdf_download_color_payload (b200tsdf_t* h, float* out4)
{
  if (!h || !h->has_volume || !out4) return B200TSDF_EINVAL;
  if (!h->p.color_norm) return 0;
  Snapshot S;
  int rc = take_snapshot (h, S);
  if (rc) return rc;
  const Params& p = S.p;
  std::vector<NodeRec> recs;
  int n = 1 << p.C;
  for (int x = 0; x < n; ++x) for (int y = 0; y < n; ++y) for (int z = 0; z < n; ++z)
  {
    NodePos nd;
    if (!locate_node (p, p.C, x, y, z, nd)) return h->fail (B200TSDF_ESTATE, "coarse cell without storage");
    collect_nodes (p, nd, recs);
  }
  std::sort (recs.begin (), recs.end (), [] (const NodeRec& a, const NodeRec& b) {
    return std::lexicographical_compare (a.k, a.k + 4, b.k, b.k + 4); });
  for (size_t i = 0; i < recs.size (); ++i) std::memcpy (out4 + 4 * i, recs[i].q, 16);
  return (int64_t) recs.size ();
}

} // extern "C"

// ---- .vol save and load (DESIGN.md §3e) ------------------------------------------------------------------------------------
namespace {

constexpr int VOL_HOST_IO = 4;                      // debug_flags bit 2 (of the configuration set last): .vol through the host
                                                    // writer and the host loader
constexpr size_t VOL_CHUNK = (size_t) 1 << 19;      // records per pinned staging buffer of the file writer
constexpr size_t VOL_LOAD_CHUNK = (size_t) 1 << 25; // bytes per pinned staging buffer of the file loader
constexpr size_t VOL_HEAD_PROBE = (size_t) 1 << 16; // bytes of a device image copied to the host for its header

struct File
{
  std::FILE* f = nullptr;
  File (const File&) = delete;
  File& operator= (const File&) = delete;
  explicit File (std::FILE* x) : f (x) {}
  ~File () { if (f) std::fclose (f); }
  operator std::FILE* () const { return f; }
};

// the text header (tsdf_volume_octree.cpp:222-245; serializeASCII eigen_extensions.h:249-257) and the octree header
// (Octree::serialize octree.cpp:645-657: the resolution as three size_t, the size as three float) in front of the body
std::string vol_header (const b200tsdf* h)
{
  const b200tsdf_config& c = h->cfg;
  std::string hd = "# TSDFVolumeOctree Meta Information\n";
  hd += std::to_string (c.xres) + " " + std::to_string (c.yres) + " " + std::to_string (c.zres) + "\n";
  hd += fmt16 (c.xsize) + " " + fmt16 (c.ysize) + " " + fmt16 (c.zsize) + "\n";
  hd += fmt16 (c.max_dist_pos) + "\n" + fmt16 (c.max_dist_neg) + "\n" + fmt16 (c.max_weight) + "\n";
  hd += fmt16 (c.min_sensor_dist) + "\n" + fmt16 (c.max_sensor_dist) + "\n";
  hd += fmt16 (c.max_cell_x) + " " + fmt16 (c.max_cell_y) + " " + fmt16 (c.max_cell_z) + "\n";
  hd += fmt16 (c.fx) + " " + fmt16 (c.fy) + " " + fmt16 (c.cx) + " " + fmt16 (c.cy) + "\n";
  hd += std::to_string (c.image_width) + " " + std::to_string (c.image_height) + "\n";
  hd += std::string (h->is_empty ? "1" : "0") + "\n0\n0\n";     // is_empty_, weight_by_depth_, weight_by_variance_
  hd += "% 4 4\n";
  std::string cell[16]; size_t width = 0;
  for (int i = 0; i < 16; ++i) { cell[i] = fmt16 (c.global_transform[i]); width = std::max (width, cell[i].size ()); }
  for (int r = 0; r < 4; ++r)
  {
    for (int k = 0; k < 4; ++k) { if (k) hd += " "; hd += std::string (width - cell[r * 4 + k].size (), ' ') + cell[r * 4 + k]; }
    hd += "\n";
  }
  hd += std::string (h->p.color_norm ? "RGBNormalized" : (h->p.color ? "RGB" : "NOCOLOR")) + "\n#OCTREEBINARY\n";
  const size_t res[3] = { (size_t) c.xres, (size_t) c.yres, (size_t) c.zres };
  hd.append ((const char*) res, sizeof (res));
  hd.append ((const char*) &c.xsize, 4); hd.append ((const char*) &c.ysize, 4); hd.append ((const char*) &c.zsize, 4);
  return hd;
}

// the host writer: a host snapshot walked recursively (write_vol_node)
int save_host (b200tsdf* h, const char* path)
{
  Snapshot S;
  int rc = take_snapshot (h, S);
  if (rc) return rc;
  std::FILE* f = std::fopen (path, "wb");
  if (!f) return h->fail (B200TSDF_EIO, std::string ("cannot open ") + path);
  const std::string hd = vol_header (h);
  std::fwrite (hd.data (), 1, hd.size (), f);
  NodePos root;
  root.level = 0; root.x = root.y = root.z = 0; root.cx = root.cy = root.cz = 0.f; root.size = S.p.size; root.slot = -1; root.idx = 0;
  write_vol_node (S.p, f, root, S.p.Rtop == 0);
  bool bad = std::ferror (f);
  std::fclose (f);
  return bad ? h->fail (B200TSDF_EIO, "write failed") : B200TSDF_OK;
}

// Every node of the volume as a VolNode, sorted into the file's order in `nodes` (`count` of them), after the work queued
// on the handle.  admit (count, go) sees the count first: it may refuse (its error is returned) or leave go false to stop
// there.
template <typename Admit>
int vol_walk (b200tsdf* h, DevBuf<VolNode>& nodes, unsigned long long& count, const Admit& admit)
{
  int* d_list = nullptr;
  const int nb = list_bricks (h, d_list);
  if (nb < 0) return nb;
  const Params& p = h->p;
  cudaStream_t s = h->stream;
  const unsigned nroot = 1u << (3 * p.Rtop);
  auto launch = [&] (auto emit, unsigned long long* total, unsigned long long* k, uint32_t* v, unsigned char*)
  {
    constexpr bool E = decltype (emit)::value;
    k_vol_roots<E><<<(nroot + 127) / 128, 128, 0, s>>> (p, total, k, (VolNode*) v);
    if (nb) k_vol_bricks<E><<<(unsigned) ((nb + 3) / 4), 128, 0, s>>> (p, d_list, nb, total, k, (VolNode*) v);
  };
  auto dest = [&] (unsigned long long n, void*& v_out, unsigned char*&)
  {
    bool go = false;
    if (int rc = admit (n, go)) return rc;
    if (!go || !n) return (int) B200TSDF_OK;
    if (nodes.alloc ((size_t) n)) return alloc_failed (h, "vol records");
    v_out = nodes.p;
    return (int) B200TSDF_OK;
  };
  static_assert (sizeof (VolNode) == 16, "a VolNode is four sort words");
  return sorted_records (h, "vol records", 4, 3 * p.L + VOL_KEY_LEVEL_BITS, launch, dest, count);
}

void vol_format_launch (b200tsdf* h, const VolNode* nodes, size_t first, size_t n, unsigned char* out)
{
  const int rb = vol_record_bytes (h->p.color != 0, h->p.color_norm != 0);
  if (n) k_vol_format<<<(unsigned) ((n + VOL_FORMAT_THREADS - 1) / VOL_FORMAT_THREADS), VOL_FORMAT_THREADS, 0, h->stream>>> (h->p, nodes, first, n, rb, out);
}

// the device writer into a file: the sorted nodes are formatted a chunk at a time, and the D2H copy of each chunk into one
// of two pinned buffers overlaps the fwrite of the one before
int save_device_file (b200tsdf* h, const char* path)
{
  if (int rc = b200tsdf_sync (h)) return rc;
  cudaStream_t s = h->stream;
  DevBuf<VolNode> nodes (s);
  unsigned long long count = 0;
  if (int rc = vol_walk (h, nodes, count, [] (unsigned long long, bool& go) { go = true; return (int) B200TSDF_OK; })) return rc;
  const size_t rb = (size_t) vol_record_bytes (h->p.color != 0, h->p.color_norm != 0);
  const size_t chunk = std::max<size_t> (1, std::min<size_t> (VOL_CHUNK, (size_t) count));
  DevBuf<unsigned char> d_chunk (s);
  Pinned<unsigned char> pin[2];
  Event ev[2];
  if (d_chunk.alloc (chunk * rb)) return alloc_failed (h, "vol staging");
  for (int k = 0; k < 2; ++k)
  {
    if (pin[k].alloc (chunk * rb) != cudaSuccess) { cudaGetLastError (); return h->fail (B200TSDF_ENOMEM, "pinned host allocation failed"); }
    CK (cudaEventCreateWithFlags (&ev[k].x, cudaEventDisableTiming));
  }
  File f (std::fopen (path, "wb"));
  if (!f) return h->fail (B200TSDF_EIO, std::string ("cannot open ") + path);
  const std::string hd = vol_header (h);
  std::fwrite (hd.data (), 1, hd.size (), f);
  int last = -1; size_t pending = 0;
  for (size_t first = 0, k = 0; first < count; first += chunk, ++k)
  {
    const size_t n = std::min<size_t> (chunk, (size_t) count - first);
    const int b = (int) (k & 1);
    vol_format_launch (h, nodes, first, n, d_chunk);
    CK (cudaMemcpyAsync (pin[b], d_chunk, n * rb, cudaMemcpyDeviceToHost, s));
    CK (cudaEventRecord (ev[b], s));
    if (last >= 0) { CK (cudaEventSynchronize (ev[last])); std::fwrite (pin[last], 1, pending, f); }
    last = b; pending = n * rb;
  }
  if (last >= 0) { CK (cudaEventSynchronize (ev[last])); std::fwrite (pin[last], 1, pending, f); }
  CK (cudaGetLastError ());
  const bool bad = std::ferror (f) != 0;
  const bool closed = std::fclose (f.f) == 0;
  f.f = nullptr;
  return (bad || !closed) ? h->fail (B200TSDF_EIO, "write failed") : B200TSDF_OK;
}

// ---- load (tsdf_volume_octree.cpp:248-275; Octree::deserialize octree.cpp:659-678; OctreeNode::deserialize :306-325) ----

// the text and octree headers from f into c (the handle's pending configuration with the file's values), rgb and is_empty;
// `name` prefixes the messages.  f is left at the first body byte.
int vol_read_header (b200tsdf* h, std::FILE* f, const std::string& name, b200tsdf_config& c, bool& rgb, int& is_empty)
{
  c = h->cfg_pending;
  char line[1024];
  auto fail = [&] (const std::string& m) { return h->fail (B200TSDF_EIO, name + ": " + m); };
  if (!std::fgets (line, sizeof (line), f)) return fail ("empty file");
  int wd = 0, wv = 0;
  is_empty = 0;
  double gt[16];
  int nread = std::fscanf (f, "%d %d %d %f %f %f %f %f %f %f %f %f %f %f %lf %lf %lf %lf %d %d %d %d %d",
                           &c.xres, &c.yres, &c.zres, &c.xsize, &c.ysize, &c.zsize, &c.max_dist_pos, &c.max_dist_neg, &c.max_weight,
                           &c.min_sensor_dist, &c.max_sensor_dist, &c.max_cell_x, &c.max_cell_y, &c.max_cell_z,
                           &c.fx, &c.fy, &c.cx, &c.cy, &c.image_width, &c.image_height, &is_empty, &wd, &wv);
  if (nread != 23) return fail ("bad header");
  // the reference has no setter for these two: only a .vol written with them set turns the alternative weightings on (hpp:200-204)
  if (wd || wv) return fail ("weight_by_depth_ / weight_by_variance_ volumes are not supported (the fusion here uses w_new = 1)");
  char pct[8]; int rr = 0, cc = 0;
  if (std::fscanf (f, " %1s %d %d", pct, &rr, &cc) != 3 || pct[0] != '%' || rr != 4 || cc != 4) return fail ("bad transform header");
  for (int i = 0; i < 16; ++i) if (std::fscanf (f, "%lf", &gt[i]) != 1) return fail ("bad transform");
  char type[64];
  if (std::fscanf (f, "%63s", type) != 1) return fail ("missing node type");
  rgb = std::string (type) == "RGB";
  if (!rgb && std::string (type) != "NOCOLOR") return fail (std::string ("unsupported node type ") + type);
  do { if (!std::fgets (line, sizeof (line), f)) return fail ("missing #OCTREEBINARY"); } while (!(line[0] == '#' && line[1] == 'O'));
  size_t res3[3]; float size3[3];
  if (std::fread (res3, sizeof (size_t), 3, f) != 3 || std::fread (size3, 4, 3, f) != 3) return fail ("truncated octree header");
  c.integrate_color = rgb ? 1 : 0;
  for (int i = 0; i < 16; ++i) c.global_transform[i] = gt[i];
  return B200TSDF_OK;
}

// the host loader: one record at a time, recursively, into a host image of the volume
struct VolLoader
{
  std::FILE* f; bool rgb; const Params* p; bool bad = false; std::string why;
  unsigned long long ood = 0;                  // stored {d, w} outside the fast route's domain (edit_in_fast_domain)
  std::vector<float2> root_dw; std::vector<uint32_t> root_split; std::vector<uchar4> root_rgb; std::vector<float> root_M; std::vector<int> root_ns;
  std::vector<uint64_t> keys; std::vector<float2> nodes; std::vector<uint32_t> split; std::vector<uchar4> rgbv; std::vector<float> Mv; std::vector<int> nsv;
  std::unordered_map<uint64_t, int> index;
  int brick_of (int t, int x, int y, int z)
  {
    uint64_t key = brick_key (t, x, y, z);
    auto it = index.find (key);
    if (it != index.end ()) return it->second;
    index[key] = (int) keys.size ();
    keys.push_back (key);
    nodes.resize (keys.size () * BRICK_NODES, make_float2 (-1.f, 0.f));
    split.resize (keys.size () * BRICK_SPLIT_WORDS, 0u);
    rgbv.resize (keys.size () * BRICK_NODES, make_uchar4 (0, 0, 0, 0));
    Mv.resize (keys.size () * BRICK_NODES, 0.f); nsv.resize (keys.size () * BRICK_NODES, 0);
    return (int) keys.size () - 1;
  }
  void node (int level, int x, int y, int z)
  {
    if (bad) return;
    unsigned char c3[3] = { 0, 0, 0 };
    float v[7]; int nsamp; size_t nchild;
    bool ok = true;
    if (rgb) ok = ok && std::fread (c3, 1, 3, f) == 3;
    ok = ok && std::fread (v, 4, 7, f) == 7 && std::fread (&nsamp, 4, 1, f) == 1 && std::fread (&nchild, sizeof (size_t), 1, f) == 1;
    if (!ok || (nchild != 0 && nchild != 8)) { bad = true; why = "truncated or malformed node record"; return; }
    const Params& P = *p;
    if (level < P.C && nchild != 8) { bad = true; why = "tree is shallower than the coarse depth implied by max_cell_size"; return; }
    if (level > P.L || (level == P.L && nchild)) { bad = true; why = "tree is deeper than the resolution"; return; }
    const VolPlace o = vol_place (P, level, x, y, z, nchild != 0);
    if (o.stored)
    {
      if (!edit_in_fast_domain (v[0], v[1])) ++ood;
      if (o.root)
      {
        const int ri = o.root_idx;
        root_dw[ri] = make_float2 (v[0], v[1]); root_rgb[ri] = make_uchar4 (c3[0], c3[1], c3[2], 0); root_M[ri] = v[6]; root_ns[ri] = nsamp;
        if (o.set_split) root_split[o.word] |= o.mask;
      }
      else
      {
        const int b = brick_of (o.t, o.bx, o.by, o.bz);
        const size_t k = (size_t) b * BRICK_NODES + o.idx;
        nodes[k] = make_float2 (v[0], v[1]); rgbv[k] = make_uchar4 (c3[0], c3[1], c3[2], 0); Mv[k] = v[6]; nsv[k] = nsamp;
        if (o.set_split) split[(size_t) b * BRICK_SPLIT_WORDS + o.word] |= o.mask;
      }
    }
    for (size_t c = 0; c < nchild; ++c) node (level + 1, 2 * x + (int) ((c >> 2) & 1), 2 * y + (int) ((c >> 1) & 1), 2 * z + (int) (c & 1));
  }
};

// the body at f through the host loader into the freshly reset volume; `name` prefixes the message of a malformed body
int load_host_body (b200tsdf* h, std::FILE* f, bool rgb, const std::string& name, unsigned long long& ood)
{
  const Params& p = h->p;
  VolLoader L; L.f = f; L.rgb = rgb; L.p = &p;
  size_t rn = h->vol.root_n;
  L.root_dw.assign (rn, make_float2 (-1.f, 0.f)); L.root_split.assign ((rn + 31) / 32, 0u);
  L.root_rgb.assign (rn, make_uchar4 (0, 0, 0, 0)); L.root_M.assign (rn, 0.f); L.root_ns.assign (rn, 0);
  L.node (0, 0, 0, 0);
  if (L.bad) return h->fail (B200TSDF_EIO, name + ": " + L.why);
  ood = L.ood;
  cudaSetDevice (h->device);
  CK (cudaMemcpy (p.root_dw, L.root_dw.data (), rn * sizeof (float2), cudaMemcpyHostToDevice));
  CK (cudaMemcpy (p.root_split, L.root_split.data (), L.root_split.size () * sizeof (uint32_t), cudaMemcpyHostToDevice));
  if (p.root_rgb) CK (cudaMemcpy (p.root_rgb, L.root_rgb.data (), rn * sizeof (uchar4), cudaMemcpyHostToDevice));
  if (p.root_M) { CK (cudaMemcpy (p.root_M, L.root_M.data (), rn * sizeof (float), cudaMemcpyHostToDevice)); CK (cudaMemcpy (p.root_ns, L.root_ns.data (), rn * sizeof (int), cudaMemcpyHostToDevice)); }
  int nb = (int) L.keys.size ();
  if (nb)
  {
    cudaStream_t s = h->stream;
    DevBuf<uint64_t> dk (s); DevBuf<float2> dn (s); DevBuf<uint32_t> ds (s); DevBuf<uchar4> dc (s); DevBuf<float> dM (s); DevBuf<int> dns (s);
    CK (dk.upload (L.keys)); CK (dn.upload (L.nodes)); CK (ds.upload (L.split));
    if (p.rgb) CK (dc.upload (L.rgbv));
    if (p.M) { CK (dM.upload (L.Mv)); CK (dns.upload (L.nsv)); }
    k_load_bricks<<<nb, 128, 0, s>>> (p, dk, nb, dn, ds, dc, dM, dns);
    CK (cudaStreamSynchronize (s));
  }
  return B200TSDF_OK;
}

// The parallel parser: the body (len bytes of device memory) into the freshly reset volume.  1 when every check held and the
// records are placed; 0 when one failed or its work space cannot be allocated, with the volume untouched (the caller runs the
// host loader on the same bytes); < 0 on a CUDA error.
int load_device_body (b200tsdf* h, const unsigned char* d_body, size_t len, bool rgb, unsigned long long& ood)
{
  const int rb = vol_record_bytes (rgb, false);
  const size_t nrec = len / rb;
  if (!nrec || nrec >= ((size_t) 1 << 31)) return 0;
  cudaStream_t s = h->stream;
  DevBuf<long long> delta (s), incl (s);
  DevBuf<unsigned long long> res (s);
  if (delta.alloc (nrec) || incl.alloc (nrec) || res.alloc (3)) { cudaGetLastError (); return 0; }
  const unsigned long long init[3] = { ~0ull, 0ull, 0ull };
  CK (cudaMemcpyAsync (res, init, sizeof (init), cudaMemcpyHostToDevice, s));
  const unsigned blocks = (unsigned) ((nrec + 255) / 256);
  k_vol_slots<<<blocks, 256, 0, s>>> (d_body, nrec, rb, delta);
  CK (cudaGetLastError ());
  const int e = b2_inclusive_sum (s, delta, incl, nrec);
  if (e == (int) cudaErrorMemoryAllocation) { cudaGetLastError (); return 0; }
  if (e) return h->fail (B200TSDF_ECUDA, std::string ("vol parse scan: ") + cudaGetErrorString ((cudaError_t) e));
  k_vol_end<<<blocks, 256, 0, s>>> (incl, nrec, res);
  unsigned long long out[3];
  CK (cudaMemcpyAsync (out, res, sizeof (out), cudaMemcpyDeviceToHost, s));
  CK (cudaStreamSynchronize (s));
  if (out[0] == ~0ull) return 0;                             // the tree does not close inside the body
  const size_t n = (size_t) out[0] + 1;
  const unsigned nblocks = (unsigned) ((n + 255) / 256);
  k_vol_check<<<nblocks, 256, 0, s>>> (h->p, d_body, n, rb, rgb ? 1 : 0, res);
  CK (cudaMemcpyAsync (out, res, sizeof (out), cudaMemcpyDeviceToHost, s));
  CK (cudaStreamSynchronize (s));
  if (out[1]) return 0;
  ood = out[2];
  k_vol_place<<<nblocks, 256, 0, s>>> (h->p, d_body, n, rb, rgb ? 1 : 0);
  CK (cudaGetLastError ());
  return 1;
}

// after a body is in: isEmpty from the header, the fast route only for values fusion produces, and the device error bits
int load_finish (b200tsdf* h, int is_empty, unsigned long long ood, bool on_device)
{
  h->mark_all ();
  h->is_empty = is_empty != 0;
  h->loaded_on_device = on_device;
  if (ood && h->fast_path)
  {
    h->fast_path = false; h->top_path = false;
    drop_batch_graphs (h);                                   // the captured launches take the fast route
  }
  return check_device_err (h);
}

} // namespace

extern "C" {

// save (tsdf_volume_octree.cpp:222-245; Octree::serialize octree.cpp:645-657; serializeASCII
// eigen_extensions.h:249-257)
int b200tsdf_save (b200tsdf_t* h, const char* path)
{
  if (!h || !path) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "save before reset()");
  cudaSetDevice (h->device);
  return (h->cfg_pending.debug_flags & VOL_HOST_IO) ? save_host (h, path) : save_device_file (h, path);
}

int b200tsdf_save_device (b200tsdf_t* h, void* d_buf, size_t capacity, size_t* nbytes)
{
  if (!h || !nbytes) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "save before reset()");
  cudaSetDevice (h->device);
  if (int rc = b200tsdf_sync (h)) return rc;
  const std::string hd = vol_header (h);
  const size_t rb = (size_t) vol_record_bytes (h->p.color != 0, h->p.color_norm != 0);
  cudaStream_t s = h->stream;
  DevBuf<VolNode> nodes (s);
  unsigned long long count = 0;
  auto admit = [&] (unsigned long long n, bool& go)
  {
    const size_t need = hd.size () + (size_t) n * rb;
    *nbytes = need;
    if (!d_buf) return (int) B200TSDF_OK;
    if (capacity < need) return h->fail (B200TSDF_EINVAL, "save buffer too small");
    go = true;
    return (int) B200TSDF_OK;
  };
  if (int rc = vol_walk (h, nodes, count, admit)) return rc;
  if (!d_buf) return B200TSDF_OK;
  unsigned char* o = (unsigned char*) d_buf;
  CK (cudaMemcpyAsync (o, hd.data (), hd.size (), cudaMemcpyHostToDevice, s));
  vol_format_launch (h, nodes, 0, (size_t) count, o + hd.size ());
  CK (cudaGetLastError ());
  CK (cudaStreamSynchronize (s));
  return B200TSDF_OK;
}

int b200tsdf_load (b200tsdf_t* h, const char* path)
{
  if (!h || !path) return B200TSDF_EINVAL;
  File f (std::fopen (path, "rb"));
  if (!f) return h->fail (B200TSDF_EIO, std::string ("cannot open ") + path);
  b200tsdf_config c; bool rgb = false; int is_empty = 0;
  if (int rc = vol_read_header (h, f, path, c, rgb, is_empty)) return rc;
  h->cfg_pending = c;
  if (int rc = b200tsdf_reset (h)) return rc;
  cudaSetDevice (h->device);
  unsigned long long ood = 0;
  if (!(h->cfg.debug_flags & VOL_HOST_IO))
  {
    // the body to the device in one buffer: the fread of each chunk overlaps the H2D copy of the one before.  When the
    // buffers cannot be had, the host loader reads the file as it did before there was a device parser.
    const long body = std::ftell (f);
    std::fseek (f, 0, SEEK_END);
    const long end = std::ftell (f);
    std::fseek (f, body, SEEK_SET);
    const size_t len = (body >= 0 && end > body) ? (size_t) (end - body) : 0;
    const size_t chunk = std::max<size_t> (1, std::min (VOL_LOAD_CHUNK, len));
    cudaStream_t s = h->stream;
    DevBuf<unsigned char> d_body (s);
    Pinned<unsigned char> pin[2];
    Event ev[2];
    bool staged = d_body.alloc (len) == cudaSuccess;
    for (int k = 0; k < 2 && len && staged; ++k)
    {
      staged = pin[k].alloc (chunk) == cudaSuccess;
      if (staged) CK (cudaEventCreateWithFlags (&ev[k].x, cudaEventDisableTiming));
    }
    if (!staged) cudaGetLastError ();
    size_t got = 0;
    for (size_t k = 0; staged && got < len; ++k)
    {
      const int b = (int) (k & 1);
      if (k >= 2) CK (cudaEventSynchronize (ev[b]));
      const size_t want = std::min (chunk, len - got);
      const size_t r = std::fread (pin[b], 1, want, f);
      if (r) { CK (cudaMemcpyAsync (d_body.p + got, pin[b], r, cudaMemcpyHostToDevice, s)); CK (cudaEventRecord (ev[b], s)); }
      got += r;
      if (r < want) break;
    }
    const int r = staged ? load_device_body (h, d_body, got, rgb, ood) : 0;
    if (r < 0) return r;
    if (r == 1) return load_finish (h, is_empty, ood, true);
    std::fseek (f, body, SEEK_SET);
  }
  if (int rc = load_host_body (h, f, rgb, path, ood)) return rc;
  return load_finish (h, is_empty, ood, false);
}

int b200tsdf_load_path (b200tsdf_t* h, int32_t* on_device)
{
  if (!h || !on_device) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "load path before reset()");
  *on_device = h->loaded_on_device ? 1 : 0;
  return B200TSDF_OK;
}

int b200tsdf_load_device (b200tsdf_t* h, const void* d_buf, size_t nbytes)
{
  if (!h || (!d_buf && nbytes)) return B200TSDF_EINVAL;
  const std::string name = "device image";
  if (!nbytes) return h->fail (B200TSDF_EIO, name + ": empty file");
  cudaSetDevice (h->device);
  const unsigned char* d = (const unsigned char*) d_buf;
  // the header through the same stdio code as a file: fmemopen over a host copy of the image's first bytes, or of the whole
  // image when the header does not end well inside them
  std::vector<unsigned char> head (std::min (nbytes, VOL_HEAD_PROBE));
  b200tsdf_config c; bool rgb = false; int is_empty = 0;
  long body = 0;
  for (;;)
  {
    CK (cudaMemcpy (head.data (), d, head.size (), cudaMemcpyDeviceToHost));
    File f (fmemopen (head.data (), head.size (), "rb"));
    if (!f) return h->fail (B200TSDF_EIO, name + ": cannot open the header copy");
    const int rc = vol_read_header (h, f, name, c, rgb, is_empty);
    body = rc ? 0 : std::ftell (f);
    const bool whole = head.size () == nbytes;
    if (whole || (!rc && body >= 0 && (size_t) body + 1 < head.size ()))
    {
      if (rc) return rc;
      break;
    }
    head.resize (nbytes);
  }
  h->cfg_pending = c;
  if (int rc = b200tsdf_reset (h)) return rc;
  cudaSetDevice (h->device);
  unsigned long long ood = 0;
  if (!(h->cfg.debug_flags & VOL_HOST_IO))
  {
    const int r = load_device_body (h, d + body, nbytes - (size_t) body, rgb, ood);
    if (r < 0) return r;
    if (r == 1) return load_finish (h, is_empty, ood, true);
  }
  const size_t blen = nbytes - (size_t) body;
  std::vector<unsigned char> host (std::max<size_t> (blen, 1));
  if (blen) CK (cudaMemcpy (host.data (), d + body, blen, cudaMemcpyDeviceToHost));
  File f (fmemopen (host.data (), host.size (), "rb"));
  if (!f) return h->fail (B200TSDF_EIO, name + ": cannot open the body copy");
  if (!blen) std::fseek (f, 0, SEEK_END);                    // (fmemopen takes no empty buffer)
  if (int rc = load_host_body (h, f, rgb, name, ood)) return rc;
  return load_finish (h, is_empty, ood, false);
}

// ---- shard export / import ------------------------------------------------------------------------------------
namespace {
struct ShardHeader { uint32_t magic, version; int32_t L, C, T, Rtop, color, var; uint32_t n_roots, n_bricks; float size; uint32_t pad; };
constexpr uint32_t SHARD_MAGIC = 0x42325348;   // "B2SH"
}

int b200tsdf_export_shard (b200tsdf_t* h, void* buf, size_t capacity, size_t* nbytes)
{
  if (!h || !nbytes) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "export before reset()");
  if (h->p.Rtop != h->p.C) return h->fail (B200TSDF_EINVAL, "shard export needs a grid whose coarse cells are the top-tier roots");
  if (h->p.color_norm) return h->fail (B200TSDF_EINVAL, "shard export does not carry the RGBNormalized payload");
  Snapshot S;
  int rc = take_snapshot (h, S);
  if (rc) return rc;
  const Params& p = S.p;
  const bool color = p.rgb != nullptr, var = p.M != nullptr;
  // owned coarse cells and the bricks below them
  std::vector<int> roots;
  int n = 1 << p.C;
  for (int x = 0; x < n; ++x) for (int y = 0; y < n; ++y) for (int z = 0; z < n; ++z) if (owns_cell (p, x, y, z)) roots.push_back (root_index (p, x, y, z));
  std::vector<uint32_t> bricks;
  for (uint32_t s = 0; s <= p.pool_mask; ++s)
  {
    uint64_t key = p.keys[s];
    if (key == KEY_EMPTY) continue;
    int t, bx, by, bz;
    brick_key_decode (key, t, bx, by, bz);
    int sh = tier_root_level (p, t) - p.C;
    if (owns_cell (p, bx >> sh, by >> sh, bz >> sh)) bricks.push_back (s);
  }
  const size_t root_rec = 4 + 8 + 1 + 4 + 4 + 4, brick_rec = 8 + BRICK_NODES * 8 + BRICK_SPLIT_WORDS * 4 + (color ? BRICK_NODES * 4 : 0) + (var ? BRICK_NODES * 8 : 0);
  size_t need = sizeof (ShardHeader) + roots.size () * root_rec + bricks.size () * brick_rec;
  *nbytes = need;
  if (!buf) return B200TSDF_OK;
  if (capacity < need) return h->fail (B200TSDF_EINVAL, "export buffer too small");
  unsigned char* o = (unsigned char*) buf;
  ShardHeader hd{}; hd.magic = SHARD_MAGIC; hd.version = 1; hd.L = p.L; hd.C = p.C; hd.T = p.T; hd.Rtop = p.Rtop; hd.color = color; hd.var = var;
  hd.n_roots = (uint32_t) roots.size (); hd.n_bricks = (uint32_t) bricks.size (); hd.size = p.size;
  std::memcpy (o, &hd, sizeof (hd)); o += sizeof (hd);
  for (int r : roots)
  {
    std::memcpy (o, &r, 4); o += 4;
    std::memcpy (o, &p.root_dw[r], 8); o += 8;
    *o++ = (unsigned char) ((p.root_split[r >> 5] >> (r & 31)) & 1);
    uchar4 c = p.root_rgb ? p.root_rgb[r] : make_uchar4 (0, 0, 0, 0); std::memcpy (o, &c, 4); o += 4;
    float M = p.root_M ? p.root_M[r] : 0.f; int nsv = p.root_ns ? p.root_ns[r] : 0;
    std::memcpy (o, &M, 4); o += 4; std::memcpy (o, &nsv, 4); o += 4;
  }
  for (uint32_t s : bricks)
  {
    std::memcpy (o, &p.keys[s], 8); o += 8;
    std::memcpy (o, &p.nodes[(size_t) s * BRICK_NODES], BRICK_NODES * 8); o += BRICK_NODES * 8;
    std::memcpy (o, &p.split[(size_t) s * BRICK_SPLIT_WORDS], BRICK_SPLIT_WORDS * 4); o += BRICK_SPLIT_WORDS * 4;
    if (color) { std::memcpy (o, &p.rgb[(size_t) s * BRICK_NODES], BRICK_NODES * 4); o += BRICK_NODES * 4; }
    if (var) { std::memcpy (o, &p.M[(size_t) s * BRICK_NODES], BRICK_NODES * 4); o += BRICK_NODES * 4; std::memcpy (o, &p.ns[(size_t) s * BRICK_NODES], BRICK_NODES * 4); o += BRICK_NODES * 4; }
  }
  return B200TSDF_OK;
}

int b200tsdf_import_shard (b200tsdf_t* h, const void* buf, size_t nbytes)
{
  if (!h || !buf || nbytes < sizeof (ShardHeader)) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "import before reset()");
  const Params& p = h->p;
  ShardHeader hd; std::memcpy (&hd, buf, sizeof (hd));
  const bool color = p.rgb != nullptr, var = p.M != nullptr;
  if (hd.magic != SHARD_MAGIC || hd.version != 1) return h->fail (B200TSDF_EINVAL, "not a shard buffer");
  if (hd.L != p.L || hd.C != p.C || hd.T != p.T || hd.Rtop != p.Rtop || hd.size != p.size || (hd.color != 0) != color || (hd.var != 0) != var)
    return h->fail (B200TSDF_EINVAL, "shard was exported from a different grid configuration");
  const size_t root_rec = 4 + 8 + 1 + 4 + 4 + 4, brick_rec = 8 + BRICK_NODES * 8 + BRICK_SPLIT_WORDS * 4 + (color ? BRICK_NODES * 4 : 0) + (var ? BRICK_NODES * 8 : 0);
  if (nbytes != sizeof (ShardHeader) + (size_t) hd.n_roots * root_rec + (size_t) hd.n_bricks * brick_rec) return h->fail (B200TSDF_EINVAL, "truncated shard buffer");
  cudaSetDevice (h->device);
  int rc = b200tsdf_sync (h);
  if (rc) return rc;
  h->mark_all ();                                          // (before the first write: a failure below may leave part of it)
  const unsigned char* o = (const unsigned char*) buf + sizeof (ShardHeader);
  size_t nr = hd.n_roots, nb = hd.n_bricks;
  std::vector<int> ridx (nr); std::vector<float2> rdw (nr); std::vector<unsigned char> rsp (nr); std::vector<uchar4> rrgb (nr); std::vector<float> rM (nr); std::vector<int> rns (nr);
  for (size_t i = 0; i < nr; ++i)
  {
    std::memcpy (&ridx[i], o, 4); o += 4; std::memcpy (&rdw[i], o, 8); o += 8; rsp[i] = *o++;
    std::memcpy (&rrgb[i], o, 4); o += 4; std::memcpy (&rM[i], o, 4); o += 4; std::memcpy (&rns[i], o, 4); o += 4;
    if (ridx[i] < 0 || (size_t) ridx[i] >= h->vol.root_n) return h->fail (B200TSDF_EINVAL, "corrupt shard buffer");
  }
  std::vector<uint64_t> keys (nb); std::vector<float2> nodes (nb * BRICK_NODES); std::vector<uint32_t> split (nb * BRICK_SPLIT_WORDS);
  std::vector<uchar4> rgb (color ? nb * BRICK_NODES : 0); std::vector<float> Mv (var ? nb * BRICK_NODES : 0); std::vector<int> nsv (var ? nb * BRICK_NODES : 0);
  for (size_t i = 0; i < nb; ++i)
  {
    std::memcpy (&keys[i], o, 8); o += 8;
    std::memcpy (&nodes[i * BRICK_NODES], o, BRICK_NODES * 8); o += BRICK_NODES * 8;
    std::memcpy (&split[i * BRICK_SPLIT_WORDS], o, BRICK_SPLIT_WORDS * 4); o += BRICK_SPLIT_WORDS * 4;
    if (color) { std::memcpy (&rgb[i * BRICK_NODES], o, BRICK_NODES * 4); o += BRICK_NODES * 4; }
    if (var) { std::memcpy (&Mv[i * BRICK_NODES], o, BRICK_NODES * 4); o += BRICK_NODES * 4; std::memcpy (&nsv[i * BRICK_NODES], o, BRICK_NODES * 4); o += BRICK_NODES * 4; }
  }
  cudaStream_t s = h->stream;
  if (nr)
  {
    DevBuf<int> d_idx (s); DevBuf<float2> d_dw (s); DevBuf<unsigned char> d_sp (s); DevBuf<uchar4> d_rgb (s); DevBuf<float> d_M (s); DevBuf<int> d_ns (s);
    CK (d_idx.upload (ridx)); CK (d_dw.upload (rdw)); CK (d_sp.upload (rsp)); CK (d_rgb.upload (rrgb)); CK (d_M.upload (rM)); CK (d_ns.upload (rns));
    k_import_roots<<<(unsigned) ((nr + 127) / 128), 128, 0, s>>> (p, (int) nr, d_idx, d_dw, d_sp, d_rgb, d_M, d_ns);
    CK (cudaStreamSynchronize (s));
  }
  if (nb)
  {
    DevBuf<uint64_t> dk (s); DevBuf<float2> dn (s); DevBuf<uint32_t> ds (s); DevBuf<uchar4> dc (s); DevBuf<float> dM (s); DevBuf<int> dns (s);
    CK (dk.upload (keys)); CK (dn.upload (nodes)); CK (ds.upload (split));
    CK (dc.upload (rgb)); CK (dM.upload (Mv)); CK (dns.upload (nsv));      // (empty without colour / variance: null)
    k_load_bricks<<<(unsigned) nb, 128, 0, s>>> (p, dk, (int) nb, dn, ds, dc, dM, dns);
    CK (cudaStreamSynchronize (s));
  }
  h->is_empty = false;
  return check_device_err (h);
}

} // extern "C"


#include "multigpu.cuh"
