// meshpost.cu — flattenVertices / cleanupMesh of the reference's `integrate` program on the GPU
// (src/prog/integrate.cpp:103-214; SURVEY.md §8(f) row 3).  Part of libb200tsdf.so; see
// meshpost_core.cuh for the formulation.  Ordered compaction uses cub::DeviceScan (CUDA toolkit).
// b2_mesh_flatten / b2_mesh_cleanup (mesh_sort.h) are the one implementation: the host entry points below upload, run them on
// a stream of their own and download; the device entry points of engine.cu run them on the handle's stream.
#include "../../include/b200tsdf.h"
#include "meshpost_core.cuh"

#include "mesh_sort.h"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cuda_runtime.h>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

using namespace b2;

namespace {

thread_local std::string g_meshpost_err;

// one post-processing call: its stream, its scratch and where its error message goes
struct Ctx
{
  cudaStream_t s;
  B2MeshScratch& B;
  std::string& err;
};

int fail (Ctx& X, int code, const std::string& m) { X.err = m; return code; }

#define MCK(call)                                                                                   \
  do {                                                                                              \
    cudaError_t e_ = (call);                                                                        \
    if (e_ != cudaSuccess) return fail (X, B200TSDF_ECUDA, std::string (#call) + ": " + cudaGetErrorString (e_)); \
  } while (0)
#define MNN(ptr) do { if (!(ptr)) return fail (X, B200TSDF_ENOMEM, "device allocation failed (mesh post-processing)"); } while (0)

constexpr int TPB = 256;
inline unsigned nblk (size_t n) { return (unsigned) ((n + TPB - 1) / TPB); }

// corner k of triangle t: from the index array, or 3t + k in a triangle soup (tris == null)
__device__ __forceinline__ int corner (const int* __restrict__ tris, size_t t, int k)
{
  return tris ? tris[3 * t + k] : (int) (3 * t + k);
}

// ---- shared kernels --------------------------------------------------------------------------------
__global__ void k_grid_clear (uint64_t* keys, int* head, size_t slots)
{
  size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i < slots) { keys[i] = GRID_EMPTY; head[i] = -1; }
}
__global__ void k_grid_insert (PointGrid g, int n)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) grid_insert (g, i);
}
__global__ void k_iota (int* a, int n)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = i;
}
// every index in 0..nverts-1, else *bad = 1
__global__ void k_check_indices (const int* __restrict__ tris, size_t n, int nverts, int* bad)
{
  size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && (unsigned) tris[i] >= (unsigned) nverts) *bad = 1;
}

int build_grid (Ctx& X, PointGrid& g, const float* d_pts, int n, double cell)
{
  size_t slots = 1024;
  while (slots < 2 * (size_t) n) slots <<= 1;
  g.keys = X.B.get<uint64_t> (slots); g.head = X.B.get<int> (slots); g.next = X.B.get<int> (n);
  MNN (g.keys); MNN (g.head); MNN (g.next);
  g.mask = (uint32_t) (slots - 1); g.inv_cell = 1.0 / cell; g.pts = d_pts;
  k_grid_clear<<<nblk (slots), TPB, 0, X.s>>> (g.keys, g.head, slots);
  if (n) k_grid_insert<<<nblk (n), TPB, 0, X.s>>> (g, n);
  MCK (cudaGetLastError ());
  return 0;
}

int exclusive_scan (Ctx& X, const int* in, int* out, size_t n)
{
  size_t bytes = 0;
  MCK (cub::DeviceScan::ExclusiveSum (nullptr, bytes, in, out, (int) n, X.s));
  void* tmp = X.B.get<unsigned char> (bytes);
  MNN (tmp);
  MCK (cub::DeviceScan::ExclusiveSum (tmp, bytes, in, out, (int) n, X.s));
  return 0;
}

int last_plus (Ctx& X, const int* flag, const int* scan, size_t n, size_t* total)
{
  *total = 0;
  if (!n) return 0;
  int a = 0, b = 0;
  MCK (cudaMemcpyAsync (&a, flag + n - 1, 4, cudaMemcpyDeviceToHost, X.s));
  MCK (cudaMemcpyAsync (&b, scan + n - 1, 4, cudaMemcpyDeviceToHost, X.s));
  MCK (cudaStreamSynchronize (X.s));
  *total = (size_t) a + (size_t) b;
  return 0;
}

// the index check of both routines: one flag word, read back before anything is written
int check_indices (Ctx& X, const int* d_tris, size_t ntris, size_t nverts)
{
  if (!d_tris || !ntris) return 0;
  int* bad = X.B.get<int> (1);
  MNN (bad);
  MCK (cudaMemsetAsync (bad, 0, 4, X.s));
  k_check_indices<<<nblk (3 * ntris), TPB, 0, X.s>>> (d_tris, 3 * ntris, (int) nverts, bad);
  MCK (cudaGetLastError ());
  int h = 0;
  MCK (cudaMemcpyAsync (&h, bad, 4, cudaMemcpyDeviceToHost, X.s));
  MCK (cudaStreamSynchronize (X.s));
  return h ? fail (X, B200TSDF_EINVAL, "triangle index out of range") : 0;
}

// ---- flattenVertices -------------------------------------------------------------------------------
__global__ void k_fv_round (PointGrid g, float r2, unsigned char* state, int n, int* remaining)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool und = i < n && fv_round (g, r2, state, i);
  unsigned m = __ballot_sync (0xffffffffu, und);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd (remaining, __popc (m));
}
// fall-back for pathological chains (each round only resolves the head of a chain): index order, one thread
__global__ void k_fv_serial (PointGrid g, float r2, unsigned char* state, int n)
{
  for (int i = 0; i < n; ++i) fv_round (g, r2, state, i);
}
__global__ void k_fv_target (PointGrid g, float r2, const unsigned char* state, int n, int* rep, int* kept)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  rep[i] = fv_target (g, r2, state, i);
  kept[i] = state[i] == FV_KEPT;
}
__global__ void k_fv_vertices (const float* verts, const int* kept, const int* rank, int n, float* out)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !kept[i]) return;
  size_t o = 3 * (size_t) rank[i];
  out[o] = verts[3 * (size_t) i]; out[o + 1] = verts[3 * (size_t) i + 1]; out[o + 2] = verts[3 * (size_t) i + 2];
}
// integrate.cpp:129-146: remap the corners (into rtris: the caller's triangles are only read), flag the faces that stay
__global__ void k_fv_faces (const int* tris, const int* rep, const int* rank, int nt, int* rtris, int* keep)
{
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  int a = rank[rep[corner (tris, t, 0)]], b = rank[rep[corner (tris, t, 1)]], c = rank[rep[corner (tris, t, 2)]];
  rtris[3 * (size_t) t] = a; rtris[3 * (size_t) t + 1] = b; rtris[3 * (size_t) t + 2] = c;
  keep[t] = !(a == b || b == c || c == a);
}
__global__ void k_compact_tris (const int* tris, const int* keep, const int* pos, int nt, int* out)
{
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt || !keep[t]) return;
  size_t o = 3 * (size_t) pos[t];
  out[o] = tris[3 * (size_t) t]; out[o + 1] = tris[3 * (size_t) t + 1]; out[o + 2] = tris[3 * (size_t) t + 2];
}

// ---- cleanupMesh -----------------------------------------------------------------------------------
__global__ void k_cm_centroids (const float* verts, const int* tris, int nt, float* cent)
{
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  const int c[3] = { corner (tris, t, 0), corner (tris, t, 1), corner (tris, t, 2) };
  face_centroid (verts, c, cent + 3 * (size_t) t);
}
__global__ void k_cm_count (PointGrid g, float r2, int K, int nt, int* cnt, int* nb)
{
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < nt) cnt[t] = cm_count (g, r2, K, t, nb);
}
__global__ void k_cm_union (int K, int nt, const int* cnt, const int* nb, int* parent, int* touches_big)
{
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt || cnt[t] >= K) return;
  int big = 0;
  for (int k = 0; k < cnt[t]; ++k)
  {
    int j = nb[(size_t) t * (CM_MAX_K - 1) + k];
    if (cnt[j] >= K) big = 1; else uf_union (parent, t, j);
  }
  touches_big[t] = big;
}
__global__ void k_cm_sizes (int K, int nt, const int* cnt, int* parent, const int* touches_big, int* size, int* has_big)
{
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt || cnt[t] >= K) return;
  int r = uf_find (parent, t);
  atomicAdd (&size[r], 1);
  if (touches_big[t]) has_big[r] = 1;
}
// EuclideanClusterExtraction returns the clusters with 1..K points; their faces are erased (integrate.cpp:168-183)
__global__ void k_cm_keep (int K, int nt, const int* cnt, int* parent, const int* size, const int* has_big, int* keep)
{
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  bool remove = false;
  if (cnt[t] < K) { int r = uf_find (parent, t); remove = !has_big[r] && size[r] <= K; }
  keep[t] = !remove;
}
__global__ void k_cm_mark_vertices (const int* tris, const int* keep, int nt, int* used)
{
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt || !keep[t]) return;
  used[corner (tris, t, 0)] = 1; used[corner (tris, t, 1)] = 1; used[corner (tris, t, 2)] = 1;
}
__global__ void k_cm_faces (const int* tris, const int* keep, const int* pos, const int* vrank, int nt, int* out)
{
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt || !keep[t]) return;
  size_t o = 3 * (size_t) pos[t];
  out[o] = vrank[corner (tris, t, 0)]; out[o + 1] = vrank[corner (tris, t, 1)]; out[o + 2] = vrank[corner (tris, t, 2)];
}

// ---- the host entry points: argument checks, a stream of their own, upload and download ------------------------------
int check_mesh_args (Ctx& X, const float* verts, size_t nverts, const int32_t* tris, size_t ntris,
                     float** out_verts, size_t* out_nverts, int32_t** out_tris, size_t* out_ntris)
{
  if ((!verts && nverts) || (!tris && ntris) || !out_verts || !out_nverts || !out_tris || !out_ntris)
    return fail (X, B200TSDF_EINVAL, "null argument");
  if (nverts >= (size_t) 1 << 31 || ntris >= ((size_t) 1 << 31) / 3) return fail (X, B200TSDF_EINVAL, "mesh too large for 32-bit indices");
  *out_verts = nullptr; *out_tris = nullptr; *out_nverts = 0; *out_ntris = 0;
  return 0;
}

struct HostCall
{
  cudaStream_t s = nullptr;
  B2MeshScratch B;
  ~HostCall () { if (s) cudaStreamDestroy (s); }
};

int open_device (Ctx& X, HostCall& H, int device)
{
  int ndev = 0;
  if (cudaGetDeviceCount (&ndev) != cudaSuccess || device < 0 || device >= ndev)
    return fail (X, B200TSDF_ENODEVICE, "no such CUDA device (mesh post-processing has no CPU path)");
  MCK (cudaSetDevice (device));
  MCK (cudaStreamCreateWithFlags (&H.s, cudaStreamNonBlocking));
  X.s = H.s;
  return 0;
}

// the host mesh in device copies, and device outputs sized like it
int upload_mesh (Ctx& X, const float* verts, size_t nverts, const int32_t* tris, size_t ntris,
                 float*& d_verts, int*& d_tris, float*& d_out_verts, int*& d_out_tris)
{
  d_verts = X.B.get<float> (3 * nverts); d_tris = X.B.get<int> (3 * ntris);
  d_out_verts = X.B.get<float> (3 * nverts); d_out_tris = X.B.get<int> (3 * ntris);
  MNN (d_verts); MNN (d_tris); MNN (d_out_verts); MNN (d_out_tris);
  if (nverts) MCK (cudaMemcpyAsync (d_verts, verts, nverts * 12, cudaMemcpyHostToDevice, X.s));
  if (ntris) MCK (cudaMemcpyAsync (d_tris, tris, ntris * 12, cudaMemcpyHostToDevice, X.s));
  return 0;
}

// copies the compacted mesh back into malloc'ed host arrays (released with b200tsdf_free)
int download_mesh (Ctx& X, const float* d_verts, size_t nv, const int* d_tris, size_t nt,
                   float** out_verts, size_t* out_nverts, int32_t** out_tris, size_t* out_ntris)
{
  float* hv = (float*) std::malloc (std::max<size_t> (nv, 1) * 12);
  int32_t* ht = (int32_t*) std::malloc (std::max<size_t> (nt, 1) * 12);
  if (!hv || !ht) { std::free (hv); std::free (ht); return fail (X, B200TSDF_ENOMEM, "host allocation failed"); }
  cudaError_t e = cudaSuccess;
  if (nv) e = cudaMemcpyAsync (hv, d_verts, nv * 12, cudaMemcpyDeviceToHost, X.s);
  if (e == cudaSuccess && nt) e = cudaMemcpyAsync (ht, d_tris, nt * 12, cudaMemcpyDeviceToHost, X.s);
  if (e == cudaSuccess) e = cudaStreamSynchronize (X.s);
  if (e != cudaSuccess) { std::free (hv); std::free (ht); return fail (X, B200TSDF_ECUDA, cudaGetErrorString (e)); }
  *out_verts = hv; *out_nverts = nv; *out_tris = ht; *out_ntris = nt;
  return 0;
}

} // namespace

int b2_mesh_flatten (cudaStream_t s, B2MeshScratch& B, const float* d_verts, size_t nverts, const int32_t* d_tris, size_t ntris,
                     float min_dist, float* d_out_verts, int32_t* d_out_tris, size_t* out_nverts, size_t* out_ntris, std::string& err)
{
  Ctx X{ s, B, err };
  *out_nverts = 0; *out_ntris = 0;
  if (int rc = check_indices (X, d_tris, ntris, nverts)) return rc;
  const int nv = (int) nverts, nt = (int) ntris;
  unsigned char* state = B.get<unsigned char> (nverts);
  int *rep = B.get<int> (nverts), *kept = B.get<int> (nverts), *rank = B.get<int> (nverts), *remaining = B.get<int> (1);
  int *keep = B.get<int> (ntris), *pos = B.get<int> (ntris), *rtris = B.get<int> (3 * ntris);
  MNN (state); MNN (rep); MNN (kept); MNN (rank); MNN (remaining); MNN (keep); MNN (pos); MNN (rtris);
  MCK (cudaMemsetAsync (state, FV_UNDECIDED, std::max<size_t> (nverts, 1), s));
  // pcl::search::KdTree::radiusSearch (i, min_dist): FLANN compares squared float distances with float (radius*radius)
  const float r2 = min_dist > 0.f ? (float) ((double) min_dist * (double) min_dist) : 0.f;      // radius <= 0 (or NaN): nothing is in range
  PointGrid g{};
  if (int rc = build_grid (X, g, d_verts, nv, std::max ((double) min_dist * 1.001, 1e-7))) return rc;
  int left = nv;
  for (int round = 0; left > 0 && round < 48; ++round)
  {
    MCK (cudaMemsetAsync (remaining, 0, 4, s));
    k_fv_round<<<nblk (nv), TPB, 0, s>>> (g, r2, state, nv, remaining);
    MCK (cudaMemcpyAsync (&left, remaining, 4, cudaMemcpyDeviceToHost, s));
    MCK (cudaStreamSynchronize (s));
  }
  if (left > 0) k_fv_serial<<<1, 1, 0, s>>> (g, r2, state, nv);
  size_t nv_new = 0, nt_new = 0;
  if (nv)
  {
    k_fv_target<<<nblk (nv), TPB, 0, s>>> (g, r2, state, nv, rep, kept);
    if (int rc = exclusive_scan (X, kept, rank, nverts)) return rc;
    k_fv_vertices<<<nblk (nv), TPB, 0, s>>> (d_verts, kept, rank, nv, d_out_verts);
    if (int rc = last_plus (X, kept, rank, nverts, &nv_new)) return rc;
  }
  if (nt)
  {
    k_fv_faces<<<nblk (nt), TPB, 0, s>>> (d_tris, rep, rank, nt, rtris, keep);
    if (int rc = exclusive_scan (X, keep, pos, ntris)) return rc;
    k_compact_tris<<<nblk (nt), TPB, 0, s>>> (rtris, keep, pos, nt, d_out_tris);
    if (int rc = last_plus (X, keep, pos, ntris, &nt_new)) return rc;
  }
  MCK (cudaGetLastError ());
  MCK (cudaStreamSynchronize (s));
  *out_nverts = nv_new; *out_ntris = nt_new;
  return 0;
}

int b2_mesh_cleanup (cudaStream_t s, B2MeshScratch& B, const float* d_verts, size_t nverts, const int32_t* d_tris, size_t ntris,
                     float face_dist, int min_neighbors, float* d_out_verts, int32_t* d_out_tris, size_t* out_nverts, size_t* out_ntris,
                     std::string& err)
{
  Ctx X{ s, B, err };
  *out_nverts = 0; *out_ntris = 0;
  if (int rc = check_indices (X, d_tris, ntris, nverts)) return rc;
  const int nv = (int) nverts, nt = (int) ntris, K = min_neighbors;
  float* cent = B.get<float> (3 * ntris);
  int *cnt = B.get<int> (ntris), *nb = B.get<int> (ntris * (CM_MAX_K - 1)), *parent = B.get<int> (ntris), *touches = B.get<int> (ntris);
  int *size = B.get<int> (ntris), *has_big = B.get<int> (ntris), *keep = B.get<int> (ntris), *pos = B.get<int> (ntris);
  int *used = B.get<int> (nverts), *vrank = B.get<int> (nverts);
  MNN (cent); MNN (cnt); MNN (nb); MNN (parent); MNN (touches); MNN (size); MNN (has_big); MNN (keep); MNN (pos); MNN (used); MNN (vrank);
  size_t nv_new = 0, nt_new = 0;
  if (nt)
  {
    // EuclideanClusterExtraction::setClusterTolerance (face_dist): radiusSearch with float (tolerance * tolerance)
    const float r2 = face_dist > 0.f ? (float) ((double) face_dist * (double) face_dist) : 0.f;
    k_cm_centroids<<<nblk (nt), TPB, 0, s>>> (d_verts, d_tris, nt, cent);
    PointGrid g{};
    if (int rc = build_grid (X, g, cent, nt, std::max ((double) face_dist * 1.001, 1e-7))) return rc;
    k_cm_count<<<nblk (nt), TPB, 0, s>>> (g, r2, K, nt, cnt, nb);
    k_iota<<<nblk (nt), TPB, 0, s>>> (parent, nt);
    MCK (cudaMemsetAsync (size, 0, ntris * 4, s)); MCK (cudaMemsetAsync (has_big, 0, ntris * 4, s));
    MCK (cudaMemsetAsync (touches, 0, ntris * 4, s));
    k_cm_union<<<nblk (nt), TPB, 0, s>>> (K, nt, cnt, nb, parent, touches);
    k_cm_sizes<<<nblk (nt), TPB, 0, s>>> (K, nt, cnt, parent, touches, size, has_big);
    k_cm_keep<<<nblk (nt), TPB, 0, s>>> (K, nt, cnt, parent, size, has_big, keep);
    if (int rc = exclusive_scan (X, keep, pos, ntris)) return rc;
    if (int rc = last_plus (X, keep, pos, ntris, &nt_new)) return rc;
  }
  // integrate.cpp:184-213: drop the vertices no remaining face uses, keep the order of the rest
  if (nv)
  {
    MCK (cudaMemsetAsync (used, 0, nverts * 4, s));
    if (nt) k_cm_mark_vertices<<<nblk (nt), TPB, 0, s>>> (d_tris, keep, nt, used);
    if (int rc = exclusive_scan (X, used, vrank, nverts)) return rc;
    k_fv_vertices<<<nblk (nv), TPB, 0, s>>> (d_verts, used, vrank, nv, d_out_verts);
    if (int rc = last_plus (X, used, vrank, nverts, &nv_new)) return rc;
    if (nt) k_cm_faces<<<nblk (nt), TPB, 0, s>>> (d_tris, keep, pos, vrank, nt, d_out_tris);
  }
  MCK (cudaGetLastError ());
  MCK (cudaStreamSynchronize (s));
  *out_nverts = nv_new; *out_ntris = nt_new;
  return 0;
}

extern "C" const char* b200tsdf_meshpost_last_error (void) { return g_meshpost_err.c_str (); }
extern "C" void b200tsdf_mesh_free (void* p) { std::free (p); }

extern "C" int b200tsdf_mesh_flatten (int device, const float* verts, size_t nverts, const int32_t* tris, size_t ntris, float min_dist,
                                      float** out_verts, size_t* out_nverts, int32_t** out_tris, size_t* out_ntris)
{
  HostCall H;
  Ctx X{ nullptr, H.B, g_meshpost_err };
  if (int rc = check_mesh_args (X, verts, nverts, tris, ntris, out_verts, out_nverts, out_tris, out_ntris)) return rc;
  if (int rc = open_device (X, H, device)) return rc;
  float *d_verts, *d_out_verts; int *d_tris, *d_out_tris;
  if (int rc = upload_mesh (X, verts, nverts, tris, ntris, d_verts, d_tris, d_out_verts, d_out_tris)) return rc;
  size_t nv = 0, nt = 0;
  if (int rc = b2_mesh_flatten (H.s, H.B, d_verts, nverts, d_tris, ntris, min_dist, d_out_verts, d_out_tris, &nv, &nt, g_meshpost_err))
    return rc;
  return download_mesh (X, d_out_verts, nv, d_out_tris, nt, out_verts, out_nverts, out_tris, out_ntris);
}

extern "C" int b200tsdf_mesh_cleanup (int device, const float* verts, size_t nverts, const int32_t* tris, size_t ntris,
                                      float face_dist, int min_neighbors,
                                      float** out_verts, size_t* out_nverts, int32_t** out_tris, size_t* out_ntris)
{
  HostCall H;
  Ctx X{ nullptr, H.B, g_meshpost_err };
  if (int rc = check_mesh_args (X, verts, nverts, tris, ntris, out_verts, out_nverts, out_tris, out_ntris)) return rc;
  if (min_neighbors < 1 || min_neighbors > CM_MAX_K) return fail (X, B200TSDF_EINVAL, "min_neighbors must be in 1..16");
  if (int rc = open_device (X, H, device)) return rc;
  float *d_verts, *d_out_verts; int *d_tris, *d_out_tris;
  if (int rc = upload_mesh (X, verts, nverts, tris, ntris, d_verts, d_tris, d_out_verts, d_out_tris)) return rc;
  size_t nv = 0, nt = 0;
  if (int rc = b2_mesh_cleanup (H.s, H.B, d_verts, nverts, d_tris, ntris, face_dist, min_neighbors, d_out_verts, d_out_tris, &nv, &nt,
                                g_meshpost_err))
    return rc;
  return download_mesh (X, d_out_verts, nv, d_out_tris, nt, out_verts, out_nverts, out_tris, out_ntris);
}

// ---- record ordering for b200tsdf_mesh (triangles) and the leaf enumeration (engine.cu) ----------------------------------
namespace {
__global__ void k_gather_records (const unsigned int* __restrict__ order, size_t ntri, int words, const uint32_t* __restrict__ v,
                                  const unsigned char* __restrict__ c, uint32_t* __restrict__ vo, unsigned char* __restrict__ co)
{
  // `words` threads per record: thread q copies 32-bit word q (and colour byte q) of the record
  size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ntri * words) return;
  size_t t = i / words, q = i - t * words, src = (size_t) order[t] * words + q;
  vo[i] = v[src];
  if (c) co[i] = c[src];
}
}

int b2_inclusive_sum (cudaStream_t s, const long long* d_in, long long* d_out, size_t n)
{
  if (!n) return 0;
  if (n >= ((size_t) 1 << 31)) return (int) cudaErrorInvalidValue;
  void* tmp = nullptr;
  size_t bytes = 0;
  cudaError_t e = cub::DeviceScan::InclusiveSum (nullptr, bytes, d_in, d_out, (int) n, s);
  if (e == cudaSuccess) e = cudaMalloc (&tmp, bytes);
  if (e == cudaSuccess) e = cub::DeviceScan::InclusiveSum (tmp, bytes, d_in, d_out, (int) n, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize (s);
  cudaFree (tmp);
  return (int) e;
}

int b2_sort_records (cudaStream_t s, size_t ntri, int key_bits, unsigned long long* d_keys, int words, const void* d_v, const unsigned char* d_c,
                     void* d_v_out, unsigned char* d_c_out)
{
  if (!ntri) return 0;
  if (ntri >= ((size_t) 1 << 31) || words < 1) return (int) cudaErrorInvalidValue;
  unsigned long long* keys2 = nullptr; unsigned int *idx = nullptr, *idx2 = nullptr; void* tmp = nullptr;
  size_t bytes = 0;
  cudaError_t e = cudaMalloc (&keys2, ntri * 8);
  if (e == cudaSuccess) e = cudaMalloc (&idx, ntri * 4);
  if (e == cudaSuccess) e = cudaMalloc (&idx2, ntri * 4);
  if (e == cudaSuccess) { k_iota<<<nblk (ntri), TPB, 0, s>>> ((int*) idx, (int) ntri); e = cudaGetLastError (); }
  if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs (nullptr, bytes, d_keys, keys2, idx, idx2, (int) ntri, 0, key_bits, s);
  if (e == cudaSuccess) e = cudaMalloc (&tmp, bytes);
  if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs (tmp, bytes, d_keys, keys2, idx, idx2, (int) ntri, 0, key_bits, s);
  if (e == cudaSuccess)
  {
    k_gather_records<<<nblk (ntri * words), TPB, 0, s>>> (idx2, ntri, words, (const uint32_t*) d_v, d_c, (uint32_t*) d_v_out, d_c_out);
    e = cudaGetLastError ();
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize (s);
  cudaFree (keys2); cudaFree (idx); cudaFree (idx2); cudaFree (tmp);
  return (int) e;
}
