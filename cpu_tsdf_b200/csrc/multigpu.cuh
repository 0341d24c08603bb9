// multigpu.cuh — the two places where the sharded engine moves data between GPUs, both over NVLink through NCCL
// (included at the end of engine.cu: it needs the handle).
//
//  1. b200tsdf_integrate_batch_rows: every rank integrates every frame (the volume is sharded by coarse cell, SURVEY.md
//     §8e), but a rank receives only its 1/N slice of each frame's rows from its host: the slice crosses PCIe once, is packed
//     to 16-byte pixels {x, y, z, b g r a} and all-gathered over NVLink into the full frame on every GPU (one grouped NCCL
//     launch per batch), then the batch is fused by one graph launch.  The end-to-end rate of a node is then bound by
//     N PCIe links instead of one.
//  2. b200tsdf_gather_volume: renderView / queries / marching cubes read across shards, so they run on a full replica
//     (DESIGN.md §5).  The replica is built device to device: every rank packs what it owns into device buffers and
//     ncclSend's them to the root, which scatters them into a full-size handle — no host staging.
//
// NCCL is loaded at run time (dlopen "libnccl.so.2": the process' own copy when torch is loaded) so that the library has no link-time
// dependency on it; without it the two entry points return B200TSDF_ESTATE and everything else works.
#pragma once
#include <dlfcn.h>
#include <chrono>
#include <nccl.h>

namespace {

struct NcclApi
{
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId) (ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank) (ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy) (ncclComm_t) = nullptr;
  ncclResult_t (*AllGather) (const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send) (const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv) (void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart) () = nullptr;
  ncclResult_t (*GroupEnd) () = nullptr;
  const char* (*GetErrorString) (ncclResult_t) = nullptr;
  bool ok = false;
};

NcclApi& nccl_api ()
{
  static NcclApi a;
  static bool tried = false;
  if (tried) return a;
  tried = true;
  for (const char* name : { "libnccl.so.2", "libnccl.so" })
  {
    a.lib = dlopen (name, RTLD_NOW | RTLD_GLOBAL);
    if (a.lib) break;
  }
  if (!a.lib) return a;
  auto sym = [&] (const char* n) { return dlsym (a.lib, n); };
  a.GetUniqueId = (decltype (a.GetUniqueId)) sym ("ncclGetUniqueId");
  a.CommInitRank = (decltype (a.CommInitRank)) sym ("ncclCommInitRank");
  a.CommDestroy = (decltype (a.CommDestroy)) sym ("ncclCommDestroy");
  a.AllGather = (decltype (a.AllGather)) sym ("ncclAllGather");
  a.Send = (decltype (a.Send)) sym ("ncclSend");
  a.Recv = (decltype (a.Recv)) sym ("ncclRecv");
  a.GroupStart = (decltype (a.GroupStart)) sym ("ncclGroupStart");
  a.GroupEnd = (decltype (a.GroupEnd)) sym ("ncclGroupEnd");
  a.GetErrorString = (decltype (a.GetErrorString)) sym ("ncclGetErrorString");
  a.ok = a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.AllGather && a.Send && a.Recv && a.GroupStart && a.GroupEnd && a.GetErrorString;
  return a;
}

#define NK(call)                                                                                   \
  do {                                                                                             \
    ncclResult_t r_ = (call);                                                                      \
    if (r_ != ncclSuccess) return h->fail (B200TSDF_ECUDA, std::string (#call) + ": " + nccl_api ().GetErrorString (r_)); \
  } while (0)

// this rank's rows of one frame: `stride`-byte points in, 16-byte pixels {x, y, z, bgra} out
__global__ void k_pack_rows (const unsigned char* __restrict__ in, size_t stride, int xyz_off, int rgba_off, int npts, uint4* __restrict__ out)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npts) return;
  const unsigned char* p = in + (size_t) i * stride;
  const uint32_t* f = reinterpret_cast<const uint32_t*> (p + xyz_off);
  uint4 o; o.x = f[0]; o.y = f[1]; o.z = f[2];
  o.w = rgba_off >= 0 ? *reinterpret_cast<const uint32_t*> (p + rgba_off) : 0u;
  out[i] = o;
}

// ---- shard gather: owned root-array entries of a shard, merged on the root by ownership --------------------------
__global__ void k_merge_roots (Params p, int n, int src_rank, int nranks, const float2* __restrict__ dw, const uint32_t* __restrict__ split, const uchar4* __restrict__ rgb)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int nn = 1 << p.Rtop;
  const int z = i % nn, y = (i / nn) % nn, x = i / (nn * nn);
  Params q = p; q.shard_rank = src_rank; q.shard_count = nranks;
  if (!owns_cell (q, x, y, z)) return;
  p.root_dw[i] = dw[i];
  const uint32_t m = 1u << (i & 31);
  if (split[i >> 5] & m) atomicOr (&p.root_split[i >> 5], m); else atomicAnd (&p.root_split[i >> 5], ~m);
  if (p.root_rgb && rgb) p.root_rgb[i] = rgb[i];
}
__global__ void k_gather_keys (Params p, const int* __restrict__ list, int n, uint64_t* __restrict__ keys)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keys[i] = p.keys[list[i]];
}

void comm_release (b200tsdf* h)
{
  if (h->comm && nccl_api ().ok) nccl_api ().CommDestroy ((ncclComm_t) h->comm);
  h->comm = nullptr; h->comm_rank = 0; h->comm_size = 1;
}

} // namespace

extern "C" {

int b200tsdf_comm_unique_id (void* id128)
{
  if (!id128) return B200TSDF_EINVAL;
  NcclApi& a = nccl_api ();
  if (!a.ok) return B200TSDF_ESTATE;
  ncclUniqueId id;
  if (a.GetUniqueId (&id) != ncclSuccess) return B200TSDF_ECUDA;
  static_assert (sizeof (ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  std::memcpy (id128, &id, 128);
  return B200TSDF_OK;
}

int b200tsdf_comm_init (b200tsdf_t* h, const void* id128, int rank, int nranks)
{
  if (!h || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return B200TSDF_EINVAL;
  NcclApi& a = nccl_api ();
  if (!a.ok) return h->fail (B200TSDF_ESTATE, "NCCL (libnccl.so.2) could not be loaded");
  cudaSetDevice (h->device);
  if (h->comm) { a.CommDestroy ((ncclComm_t) h->comm); h->comm = nullptr; }
  ncclUniqueId id; std::memcpy (&id, id128, 128);
  ncclComm_t c = nullptr;
  NK (a.CommInitRank (&c, nranks, id, rank));
  h->comm = c; h->comm_rank = rank; h->comm_size = nranks;
  return B200TSDF_OK;
}

int b200tsdf_row_slice (const b200tsdf_t* h, int height, int* row0, int* row1)
{
  if (!h || !row0 || !row1 || height <= 0) return B200TSDF_EINVAL;
  const int n = h->comm ? h->comm_size : 1, r = h->comm ? h->comm_rank : 0;
  const int per = (height + n - 1) / n;
  *row0 = std::min (height, r * per); *row1 = std::min (height, (r + 1) * per);
  return B200TSDF_OK;
}

// rows[i]: HOST pointer to this rank's rows [row0, row1) of frame i (b200tsdf_row_slice), `stride`-byte points
int b200tsdf_integrate_batch_rows (b200tsdf_t* h, int n, const void* const* rows, size_t stride, int xyz_off, int rgba_off,
                                   int width, int height, const double* poses_c2w)
{
  if (!h || n < 0 || (n && (!rows || !poses_c2w))) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "integrateCloud before reset()");
  if (int rc = check_cloud_layout (h, stride, xyz_off, rgba_off, width, height)) return rc;
  constexpr int HALF = FRAME_RING / 2;
  if (n > HALF) return h->fail (B200TSDF_EINVAL, "at most 32 frames per batch");
  if (n == 0) return B200TSDF_OK;
  cudaSetDevice (h->device);
  NcclApi& a = nccl_api ();
  const int nr = h->comm ? h->comm_size : 1, rk = h->comm ? h->comm_rank : 0;
  const int per = (height + nr - 1) / nr;                       // rows per rank (the last rank's slice may be short)
  const int row0 = std::min (height, rk * per), row1 = std::min (height, (rk + 1) * per);
  const size_t slice_raw = (size_t) (row1 - row0) * width * stride;
  const size_t slice16 = (size_t) per * width * 16, frame16 = slice16 * nr;
  // host packing (host_pack.h): the caller's rows are packed to 16-byte pixels by host threads into pinned staging and only
  // those cross PCIe; without it the points are uploaded as they are (and packed on the device when there is a gather)
  // The host's packing rate is shared by all ranks of the machine (tools/microbench/pack_bench.cu measures it), while every
  // rank has a PCIe link of its own: packing on the host halves the bytes one link carries and wins for one rank, but the
  // shared packing rate falls behind the sum of the links as ranks are added; with more than one rank the raw slices are
  // therefore packed on the device.  B200TSDF_HOST_PACK=0 / 1 forces the choice.
  const bool hpack = host_pack_wanted (h, stride, nr);
  // frames per pipeline stage: with host packing short stages keep the copy engine right behind the packing threads; a stage
  // costs one NCCL launch when there is a gather, and device-side packing amortises its launches over 8
  const int ROWS_CHUNK = h->rows_chunk > 0 ? h->rows_chunk : (hpack ? (nr == 1 ? 1 : 2) : 8);
  // two buffer sets, used alternately: set s is rewritten only after the batch that read it two calls ago has been fused
  const int s = h->rows_set;
  const size_t need_raw = hpack ? 0 : (size_t) HALF * per * width * stride, need_full = (size_t) HALF * frame16, need_pack = hpack ? (size_t) HALF * slice16 : 0;
  if (need_raw > h->rows_raw_cap || need_full > h->rows_full_cap || need_pack > h->pack_cap)
  {
    CK (cudaStreamSynchronize (h->stream)); CK (cudaStreamSynchronize (h->copy_stream)); CK (cudaStreamSynchronize (h->gather_stream));
    for (int k = 0; k < 2; ++k)
    {
      cudaFree (h->d_rows_raw[k]); cudaFree (h->d_rows_full[k]); h->d_rows_raw[k] = h->d_rows_full[k] = nullptr;
      h->h_pack[k].release ();
      h->rows_raw_cap = h->rows_full_cap = h->pack_cap = 0;
      if (need_raw) CK (cudaMalloc (&h->d_rows_raw[k], need_raw));
      CK (cudaMalloc (&h->d_rows_full[k], need_full));
      if (need_pack && h->h_pack[k].alloc (need_pack))
      {
        // no pinned staging to be had on this system: upload the points as they are from now on (the caps are 0: everything is re-sized)
        h->host_pack = 0;
        for (int j = 0; j < 2; ++j) h->h_pack[j].release ();
        return b200tsdf_integrate_batch_rows (h, n, rows, stride, xyz_off, rgba_off, width, height, poses_c2w);
      }
      h->rows_used[k] = false;
    }
    h->rows_raw_cap = need_raw; h->rows_full_cap = need_full; h->pack_cap = need_pack;
  }
  if (hpack) ensure_pack_pool (h, nr);
  // three-stage pipeline over chunks of frames: the copy stream only uploads (the copy engine never waits for a kernel), the
  // gather stream packs and all-gathers, the compute stream fuses.  Chunks are ROWS_CHUNK frames, the last one is halved down
  // to 2 so that little is left to upload and fuse once the last pixel has been packed.
  cudaStream_t cs = h->copy_stream, gs = h->gather_stream;
  if (int rc = pending_device_err (h)) return rc;
  if (h->rows_used[s]) { CK (cudaStreamWaitEvent (cs, h->ev_rows_done[s], 0)); CK (cudaStreamWaitEvent (gs, h->ev_rows_done[s], 0)); }
  const int npts = (row1 - row0) * width;
  const int out_rgba = (h->p.color && rgba_off >= 0) ? 12 : -1;
  for (int i = 0; i < n; ++i) if (!rows[i] && slice_raw) return h->fail (B200TSDF_EINVAL, "null row slice in batch");
  int cbeg[HALF + 1];
  const int nchunks = b2host::stage_schedule (n, ROWS_CHUNK, cbeg);
  static const bool trace = std::getenv ("B200TSDF_TRACE_ROWS") != nullptr;
  double t_wait = 0, t_pack = 0, t_enq = 0;
  auto now = [] { return std::chrono::duration<double, std::milli> (std::chrono::steady_clock::now ().time_since_epoch ()).count (); };

  // host packing: every job packs one block of rows of one frame, jobs in frame order; the pool works through the whole batch
  // while this thread hands each chunk to the GPU as soon as its last block is packed (and packs along while it waits)
  std::atomic<int> chunk_left[HALF];
  int nb = 1;
  unsigned char* const stage = hpack ? h->h_pack[s].p : nullptr;
  const int pack_rgba = h->p.color ? rgba_off : -1;
  std::function<void (int)> job = [&] (int j)
  {
    const int i = j / nb, b = j % nb;
    const size_t p0 = (size_t) npts * b / nb, p1 = (size_t) npts * (b + 1) / nb;
    b2host::pack_points16 (static_cast<const unsigned char*> (rows[i]) + p0 * stride, stride, xyz_off, pack_rgba, p1 - p0, stage + (size_t) i * slice16 + p0 * 16);
    int c = 0; while (cbeg[c + 1] <= i) ++c;
    chunk_left[c].fetch_sub (1, std::memory_order_release);
  };
  struct PoolGuard { b2host::PackPool* p; ~PoolGuard () { if (p) p->end (); } } guard { nullptr };     // `job` must outlive the workers on every return path
  {
    // the uploads of the call before last (same buffer set) have left the host: the packed staging may be rewritten, and the
    // caller's rows of that call are free (the contract of the unpacked path: valid "until two further calls")
    double t0 = trace ? now () : 0;
    if (h->rows_used[s]) CK (cudaEventSynchronize (h->ev_rows_up[s][h->rows_last_up[s]]));
    if (trace) t_wait += now () - t0;
  }
  if (hpack && npts)
  {
    nb = std::max (1, std::min ((4 * h->pack_pool->threads () + ROWS_CHUNK - 1) / ROWS_CHUNK, npts / 4096));
    for (int c = 0; c < nchunks; ++c) chunk_left[c].store ((cbeg[c + 1] - cbeg[c]) * nb, std::memory_order_relaxed);
    guard.p = h->pack_pool;
    h->pack_pool->begin (n * nb, job);
  }
  for (int c = 0; c < nchunks; ++c)
  {
    const int c0 = cbeg[c], m = cbeg[c + 1] - c0;
    const bool raw_in_place = nr == 1 && !hpack;           // one rank, no host packing: fused where the points landed
    const void* ptrs[HALF];
    for (int i = 0; i < m; ++i)
      ptrs[i] = raw_in_place ? (const void*) (h->d_rows_raw[s] + (size_t) (c0 + i) * per * width * stride)
                             : (const void*) (h->d_rows_full[s] + (size_t) (c0 + i) * frame16);
    const size_t f_stride = raw_in_place ? stride : 16; const int f_xyz = raw_in_place ? xyz_off : 0, f_rgba = raw_in_place ? rgba_off : out_rgba;
    double t0 = trace ? now () : 0;
    if (hpack && npts)
      while (chunk_left[c].load (std::memory_order_acquire) > 0)
        if (!h->pack_pool->help ()) std::this_thread::yield ();
    if (trace) { const double t = now (); t_pack += t - t0; t0 = t; }
    // the chunk's frame records travel on the copy stream ahead of its frames
    if (int rc = batch_records (h, m, ptrs, f_stride, f_xyz, f_rgba, width, height, poses_c2w + 16 * (size_t) c0, cs)) return rc;
    if (hpack)
    {
      if (npts)
      {
        if (nr == 1) CK (cudaMemcpyAsync (h->d_rows_full[s] + (size_t) c0 * frame16, stage + (size_t) c0 * slice16, (size_t) m * slice16, cudaMemcpyHostToDevice, cs));
        else
          for (int i = c0; i < c0 + m; ++i)
            CK (cudaMemcpyAsync (h->d_rows_full[s] + (size_t) i * frame16 + (size_t) rk * slice16, stage + (size_t) i * slice16, (size_t) npts * 16, cudaMemcpyHostToDevice, cs));
        h->h2d_bytes += (long long) m * npts * 16;
      }
    }
    else
      for (int i = c0; i < c0 + m; ++i)
      {
        if (slice_raw) CK (cudaMemcpyAsync (h->d_rows_raw[s] + (size_t) i * per * width * stride, rows[i], slice_raw, cudaMemcpyHostToDevice, cs));
        h->h2d_bytes += (long long) slice_raw;
      }
    cudaEvent_t up = h->ev_rows_up[s][c], ready = up;
    CK (cudaEventRecord (up, cs));
    h->rows_last_up[s] = c;
    if (nr > 1)
    {
      CK (cudaStreamWaitEvent (gs, up, 0));
      for (int i = c0; i < c0 + m && npts && !hpack; ++i)
      {
        uint4* dst = reinterpret_cast<uint4*> (h->d_rows_full[s] + (size_t) i * frame16 + (size_t) rk * slice16);
        k_pack_rows<<<(npts + 255) / 256, 256, 0, gs>>> (h->d_rows_raw[s] + (size_t) i * per * width * stride, stride, xyz_off, h->p.color ? rgba_off : -1, npts, dst);
      }
      if (!hpack) h->launches += m;
      // one grouped launch: m in-place all-gathers, frame i's slices land row-major in its full 16-byte image
      NK (a.GroupStart ());
      for (int i = c0; i < c0 + m; ++i)
      {
        unsigned char* full = h->d_rows_full[s] + (size_t) i * frame16;
        NK (a.AllGather (full + (size_t) rk * slice16, full, slice16, ncclChar, (ncclComm_t) h->comm, gs));
      }
      NK (a.GroupEnd ());
      h->nvlink_bytes += (long long) m * (long long) slice16 * (nr - 1);
      ready = h->ev_rows_ready[s][c];
      CK (cudaEventRecord (ready, gs));
    }
    CK (cudaStreamWaitEvent (h->stream, ready, 0));
    if (int rc = batch_launch (h, m)) return rc;
    if (trace) t_enq += now () - t0;
  }
  CK (cudaEventRecord (h->ev_rows_done[s], h->stream));
  if (trace) std::fprintf (stderr, "[b200tsdf rows] %d frames in %d chunks: staging wait %.2f ms, pack (this thread waiting / helping) %.2f ms, enqueue %.2f ms\n", n, nchunks, t_wait, t_pack, t_enq);
  h->rows_used[s] = true; h->rows_set ^= 1;
  return B200TSDF_OK;
}

// Collective over the handle's communicator: every rank's shard is sent device to device to `root`, where it is merged into
// `full` (a handle with shard_count 1 and the same grid configuration, already reset; NULL on the other ranks).
int b200tsdf_gather_volume (b200tsdf_t* h, b200tsdf_t* full, int root)
{
  if (!h) return B200TSDF_EINVAL;
  if (!h->has_volume) return h->fail (B200TSDF_ESTATE, "gather before reset()");
  if (!h->comm) return h->fail (B200TSDF_ESTATE, "gather needs b200tsdf_comm_init");
  NcclApi& a = nccl_api ();
  const int nr = h->comm_size, rk = h->comm_rank;
  if (root < 0 || root >= nr) return B200TSDF_EINVAL;
  if (h->p.Rtop != h->p.C) return h->fail (B200TSDF_EINVAL, "shard gather needs a grid whose coarse cells are the top-tier roots");
  if (h->p.track_var) return h->fail (B200TSDF_EINVAL, "shard gather does not carry the variance accumulators");
  if (h->p.color_norm) return h->fail (B200TSDF_EINVAL, "shard gather does not carry the RGBNormalized payload");
  if (rk == root)
  {
    if (!full || !full->has_volume) return h->fail (B200TSDF_EINVAL, "the root needs a reset full-size handle to gather into");
    if (full->device != h->device) return h->fail (B200TSDF_EINVAL, "the full handle must live on the root's device");
    if (full->p.L != h->p.L || full->p.C != h->p.C || full->p.size != h->p.size || full->p.color != h->p.color || full->p.track_var)
      return h->fail (B200TSDF_EINVAL, "the full handle has a different grid configuration");
  }
  cudaSetDevice (h->device);
  { int rc = b200tsdf_sync (h); if (rc) return rc; }
  if (rk == root) { int rc = b200tsdf_sync (full); if (rc) return h->fail (rc, b200tsdf_last_error (full)); }
  cudaStream_t s = h->stream;
  const Params& p = h->p;
  const bool color = p.rgb != nullptr;
  const size_t rn = h->root_n, rsw = (rn + 31) / 32;
  // what this rank owns, packed on the device
  int* d_list = nullptr;
  const int nb = list_bricks (h, d_list);
  if (nb < 0) return nb;
  DevBuf<long long> d_counts (s);
  CK (d_counts.alloc ((size_t) nr + 1));
  long long mine = nb;
  CK (cudaMemcpyAsync (d_counts + nr, &mine, sizeof (long long), cudaMemcpyHostToDevice, s));
  NK (a.AllGather (d_counts + nr, d_counts, 1, ncclInt64, (ncclComm_t) h->comm, s));
  std::vector<long long> counts (nr);
  CK (cudaMemcpyAsync (counts.data (), d_counts, (size_t) nr * sizeof (long long), cudaMemcpyDeviceToHost, s));
  CK (cudaStreamSynchronize (s));
  DevBuf<uint64_t> g_keys (s); DevBuf<float2> g_nodes (s); DevBuf<uint32_t> g_split (s); DevBuf<uchar4> g_rgb (s);
  CK (g_keys.alloc (nb)); CK (g_nodes.alloc ((size_t) nb * BRICK_NODES)); CK (g_split.alloc ((size_t) nb * BRICK_SPLIT_WORDS));
  if (color) CK (g_rgb.alloc ((size_t) nb * BRICK_NODES));
  if (nb)
  {
    k_gather_keys<<<(nb + 255) / 256, 256, 0, s>>> (p, d_list, nb, g_keys);
    k_gather_bricks<<<nb, 128, 0, s>>> (p, d_list, nb, g_nodes, g_split, g_rgb, nullptr, nullptr);
  }
  int rc_out = B200TSDF_OK;
  if (rk != root)
  {
    NK (a.GroupStart ());
    NK (a.Send (p.root_dw, rn * 8, ncclChar, root, (ncclComm_t) h->comm, s));
    NK (a.Send (p.root_split, rsw * 4, ncclChar, root, (ncclComm_t) h->comm, s));
    if (color) NK (a.Send (p.root_rgb, rn * 4, ncclChar, root, (ncclComm_t) h->comm, s));
    if (nb)
    {
      NK (a.Send (g_keys, (size_t) nb * 8, ncclChar, root, (ncclComm_t) h->comm, s));
      NK (a.Send (g_nodes, (size_t) nb * BRICK_NODES * 8, ncclChar, root, (ncclComm_t) h->comm, s));
      NK (a.Send (g_split, (size_t) nb * BRICK_SPLIT_WORDS * 4, ncclChar, root, (ncclComm_t) h->comm, s));
      if (color) NK (a.Send (g_rgb, (size_t) nb * BRICK_NODES * 4, ncclChar, root, (ncclComm_t) h->comm, s));
    }
    NK (a.GroupEnd ());
    h->nvlink_bytes += (long long) (rn * 8 + rsw * 4 + (color ? rn * 4 : 0)) + (long long) nb * (8 + BRICK_NODES * 8 + BRICK_SPLIT_WORDS * 4 + (color ? BRICK_NODES * 4 : 0));
    CK (cudaStreamSynchronize (s));
  }
  else
  {
    const Params& fp = full->p;
    // own shard: same device, straight from this handle's arrays
    k_merge_roots<<<(unsigned) ((rn + 127) / 128), 128, 0, s>>> (fp, (int) rn, rk, nr, p.root_dw, p.root_split, p.root_rgb);
    if (nb) k_load_bricks<<<nb, 128, 0, s>>> (fp, g_keys, nb, g_nodes, g_split, g_rgb, nullptr, nullptr);
    long long maxb = 1;
    for (int r = 0; r < nr; ++r) if (r != root) maxb = std::max (maxb, counts[r]);
    DevBuf<float2> r_dw (s); DevBuf<uint32_t> r_split (s); DevBuf<uchar4> r_rgb (s);
    DevBuf<uint64_t> b_keys (s); DevBuf<float2> b_nodes (s); DevBuf<uint32_t> b_split (s); DevBuf<uchar4> b_rgb (s);
    CK (r_dw.alloc (rn)); CK (r_split.alloc (rsw)); if (color) CK (r_rgb.alloc (rn));
    CK (b_keys.alloc ((size_t) maxb)); CK (b_nodes.alloc ((size_t) maxb * BRICK_NODES)); CK (b_split.alloc ((size_t) maxb * BRICK_SPLIT_WORDS));
    if (color) CK (b_rgb.alloc ((size_t) maxb * BRICK_NODES));
    for (int r = 0; r < nr && rc_out == B200TSDF_OK; ++r)
    {
      if (r == root) continue;
      const long long cb = counts[r];
      NK (a.GroupStart ());
      NK (a.Recv (r_dw, rn * 8, ncclChar, r, (ncclComm_t) h->comm, s));
      NK (a.Recv (r_split, rsw * 4, ncclChar, r, (ncclComm_t) h->comm, s));
      if (color) NK (a.Recv (r_rgb, rn * 4, ncclChar, r, (ncclComm_t) h->comm, s));
      if (cb)
      {
        NK (a.Recv (b_keys, (size_t) cb * 8, ncclChar, r, (ncclComm_t) h->comm, s));
        NK (a.Recv (b_nodes, (size_t) cb * BRICK_NODES * 8, ncclChar, r, (ncclComm_t) h->comm, s));
        NK (a.Recv (b_split, (size_t) cb * BRICK_SPLIT_WORDS * 4, ncclChar, r, (ncclComm_t) h->comm, s));
        if (color) NK (a.Recv (b_rgb, (size_t) cb * BRICK_NODES * 4, ncclChar, r, (ncclComm_t) h->comm, s));
      }
      NK (a.GroupEnd ());
      k_merge_roots<<<(unsigned) ((rn + 127) / 128), 128, 0, s>>> (fp, (int) rn, r, nr, r_dw, r_split, r_rgb);
      if (cb) k_load_bricks<<<(unsigned) cb, 128, 0, s>>> (fp, b_keys, (int) cb, b_nodes, b_split, b_rgb, nullptr, nullptr);
      CK (cudaStreamSynchronize (s));                       // the receive buffers are reused for the next rank
    }
    full->is_empty = false;
    // errors raised by the scatter (pool of the full handle too small) are on the FULL handle's flag
    int e = 0;
    cudaMemcpy (&e, full->d_err, sizeof (int), cudaMemcpyDeviceToHost);
    if (e & ERR_POOL_FULL) rc_out = h->fail (B200TSDF_ENOMEM, "brick pool of the full handle exhausted (raise its pool_log2)");
  }
  return rc_out;
}

} // extern "C"
