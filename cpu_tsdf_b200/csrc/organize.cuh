// organize.cuh — z-buffer re-organisation of unorganised clouds (the front end of the
// reference's `integrate` program, src/prog/integrate.cpp:548-635).
//
// The reference walks the points in order and keeps, per pixel, the point with the smallest z
// (`isnan(old.z) || old.z > pt.z`, :603-606): the winner is the minimum of (z, input index) in
// lexicographic order.  z is positive for every accepted point (reprojectPoint requires z > 0,
// :216-222), so its IEEE bit pattern orders like the value and one 64-bit atomicMin per point
// on the key (z bits << 32 | index) reproduces the sequential result exactly and in any order.
//
// A batch of m clouds is organised by three launches, whatever m is.  Nothing of a frame is a launch argument: the
// shared block (OrgBatch) and one record per frame (OrgRec) sit in device memory, so the launches can be captured once
// into a CUDA graph and replayed on other clouds, other counts and other options.
//   k_org_clear   zkey[frame][pixel] = ~0, filled[frame] = 0
//   k_org_zmin    a grid-stride loop over the batch's concatenated points: the frame from the prefix offsets, then
//                 units, zero->NaN, world->camera, project, atomicMin on the key of (z, index within the frame)
//   k_org_gather  one thread per pixel of each frame: recompute the winner's point and write it (or the default point
//                 with z = NaN)
#pragma once
#include "tsdf_core.cuh"
#include <cstring>

namespace b2 {

struct OrgParams
{
  float fx, fy, cx, cy;          // float, as the program's globals (integrate.cpp:63-68)
  int width, height;
  float cloud_units;
  int zero_nans, has_tf;
  double tf[12];                 // poses[i].inverse() rows 0..2 (:570-571)
};

// float -> int the way cvttss2si does it: NaN / out of range -> INT_MIN
B2_HD int to_int_x86_f (float v)
{
  if (!(v >= -2147483648.f && v < 2147483648.f)) return INT_MIN;
  return (int) v;
}

// :550-571 — the per-point preprocessing, in the program's order
B2_HD void org_prepare (const OrgParams& o, float& x, float& y, float& z)
{
  if (o.cloud_units != 1.f) { x = fmul (x, o.cloud_units); y = fmul (y, o.cloud_units); z = fmul (z, o.cloud_units); }
  if (o.zero_nans && x == 0.f && y == 0.f && z == 0.f) x = y = z = nanf ("");
  if (o.has_tf)
  {
    // pcl::transformPointCloud<PointT, double>: float (m0*x + m1*y + m2*z + m3), left to right in double
    const double* m = o.tf;
    double p0 = x, p1 = y, p2 = z;
    x = (float) dadd (dadd (dadd (dmul (m[0], p0), dmul (m[1], p1)), dmul (m[2],  p2)), m[3]);
    y = (float) dadd (dadd (dadd (dmul (m[4], p0), dmul (m[5], p1)), dmul (m[6],  p2)), m[7]);
    z = (float) dadd (dadd (dadd (dmul (m[8], p0), dmul (m[9], p1)), dmul (m[10], p2)), m[11]);
  }
}

// reprojectPoint (integrate.cpp:216-222): float arithmetic, truncating conversion; -1 = rejected
B2_HD int org_pixel (const OrgParams& o, float x, float y, float z)
{
  int u = to_int_x86_f (fadd (fdiv (fmul (x, o.fx), z), o.cx));
  int v = to_int_x86_f (fadd (fdiv (fmul (y, o.fy), z), o.cy));
  if (is_nan (z) || !(z > 0.f) || u < 0 || u >= o.width || v < 0 || v >= o.height) return -1;
  return v * o.width + u;
}

B2_HD unsigned long long org_key (float z, unsigned int j)
{
#ifdef __CUDA_ARCH__
  return ((unsigned long long) __float_as_uint (z) << 32) | j;
#else
  unsigned int b; memcpy (&b, &z, 4);
  return ((unsigned long long) b << 32) | j;
#endif
}

B2_HD void org_load (const unsigned char* pts, size_t stride, int xyz_off, size_t j, float& x, float& y, float& z)
{
  const float* q = (const float*) (pts + j * stride + xyz_off);
  x = q[0]; y = q[1]; z = q[2];
}

// one pixel of the organized cloud (integrate.cpp:596-607 result)
B2_HD void org_emit (const OrgParams& o, const unsigned char* pts, size_t stride, int xyz_off, int rgba_off,
                     unsigned long long key, unsigned char* out, size_t out_stride, int out_rgba_off)
{
  float x = 0.f, y = 0.f, z = nanf ("");
  unsigned char c[4] = { 0, 0, 0, 255 };                  // default PointXYZRGBA: b,g,r = 0, a = 255
  if (key != ~0ull)
  {
    size_t j = (size_t) (key & 0xffffffffull);
    org_load (pts, stride, xyz_off, j, x, y, z);
    org_prepare (o, x, y, z);
    if (rgba_off >= 0) { const unsigned char* s = pts + j * stride + rgba_off; c[0] = s[0]; c[1] = s[1]; c[2] = s[2]; c[3] = s[3]; }
  }
  for (size_t b = 0; b < out_stride / 4; ++b) ((unsigned int*) out)[b] = 0u;   // padding bytes are zero
  float* q = (float*) out;
  q[0] = x; q[1] = y; q[2] = z;
  if (out_stride >= 32) q[3] = 1.f;
  if (out_rgba_off >= 0) { unsigned char* d = out + out_rgba_off; d[0] = c[0]; d[1] = c[1]; d[2] = c[2]; d[3] = c[3]; }
}

// ---- batches ---------------------------------------------------------------------------------------
constexpr int ORG_MAX_FRAMES = 32;       // frames per organise batch (one record half of the batch path)

// what every frame of a batch shares (device memory, one block per batch)
struct OrgBatch
{
  OrgParams o;                   // intrinsics, image size, units, zero_nans; has_tf / tf are per frame (OrgRec)
  unsigned long long stride;     // input points: `stride` bytes each, xyz at xyz_off, colour bytes at rgba_off or -1
  int xyz_off, rgba_off;
  unsigned long long out_stride; // organised pixels: xyz at 0, colour bytes at out_rgba_off or -1 (see org_emit)
  int out_rgba_off, pad_;
};

// one frame of a batch (device memory)
struct OrgRec
{
  const unsigned char* pts;      // the frame's points (may be null when count == 0)
  unsigned long long count;      // number of points (< 2^32: the key keeps the index within the frame in 32 bits)
  unsigned long long first;      // flat index of the frame's first point in the batch's concatenation (prefix sum of count)
  int has_tf, pad_;
  double tf[12];                 // world -> camera rows 0..2 when has_tf
};

// the parameters org_prepare / org_pixel / org_emit take for frame r of batch b
B2_HD OrgParams org_frame_params (const OrgBatch& b, const OrgRec& r)
{
  OrgParams o = b.o;
  o.has_tf = r.has_tf;
  for (int i = 0; i < 12; ++i) o.tf[i] = r.tf[i];
  return o;
}

// the frame of flat point index k (k < first[m-1] + count[m-1]): the last frame whose first point is at or before k.  A frame
// without points has the same offset as the frame after it and is never chosen.
B2_HD int org_frame_of (const unsigned long long* first, int m, unsigned long long k)
{
  int lo = 0, hi = m - 1;
  while (lo < hi)
  {
    const int mid = (lo + hi + 1) >> 1;
    if (first[mid] <= k) lo = mid; else hi = mid - 1;
  }
  return lo;
}

#ifdef __CUDACC__
// grid (pixel blocks, m)
__global__ void k_org_clear (unsigned long long* __restrict__ zkey, int npix, unsigned long long* __restrict__ n_filled)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < npix) zkey[(size_t) blockIdx.y * npix + i] = ~0ull;
  if (i == 0) n_filled[blockIdx.y] = 0ull;
}

// persistent grid (its size depends only on the device): every point of the batch, frame found from the prefix offsets
__global__ void k_org_zmin (const OrgBatch* __restrict__ gb, const OrgRec* __restrict__ recs, int m, int npix,
                            unsigned long long* __restrict__ zkey)
{
  __shared__ OrgParams s_o[ORG_MAX_FRAMES];
  __shared__ const unsigned char* s_pts[ORG_MAX_FRAMES];
  __shared__ unsigned long long s_first[ORG_MAX_FRAMES];
  __shared__ unsigned long long s_total;
  __shared__ unsigned long long s_stride;
  __shared__ int s_xyz_off;
  for (int f = threadIdx.x; f < m; f += blockDim.x)
  {
    s_o[f] = org_frame_params (*gb, recs[f]);
    s_pts[f] = recs[f].pts; s_first[f] = recs[f].first;
  }
  if (threadIdx.x == 0) { s_total = recs[m - 1].first + recs[m - 1].count; s_stride = gb->stride; s_xyz_off = gb->xyz_off; }
  __syncthreads ();
  const unsigned long long total = s_total;
  for (unsigned long long k = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (unsigned long long) gridDim.x * blockDim.x)
  {
    const int f = org_frame_of (s_first, m, k);
    const unsigned long long j = k - s_first[f];           // the index within its frame: ties go to its earliest point
    const OrgParams& o = s_o[f];
    float x, y, z;
    org_load (s_pts[f], s_stride, s_xyz_off, j, x, y, z);
    org_prepare (o, x, y, z);
    const int pix = org_pixel (o, x, y, z);
    if (pix < 0) continue;
    const unsigned long long key = org_key (z, (unsigned int) j);
    unsigned long long* zk = zkey + (size_t) f * npix + pix;
    if (key < *zk) atomicMin (zk, key);                    // the plain read filters most losers
  }
}

// grid (pixel blocks, m): frame blockIdx.y's image starts at out + frame * npix * out_stride
__global__ void k_org_gather (const OrgBatch* __restrict__ gb, const OrgRec* __restrict__ recs, int npix,
                              const unsigned long long* __restrict__ zkey, unsigned char* __restrict__ out,
                              unsigned long long* __restrict__ n_filled)
{
  __shared__ OrgParams s_o;
  __shared__ const unsigned char* s_pts;
  const int f = blockIdx.y;
  if (threadIdx.x == 0) { s_o = org_frame_params (*gb, recs[f]); s_pts = recs[f].pts; }
  __syncthreads ();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool filled = false;
  if (i < npix)
  {
    const size_t q = (size_t) f * npix + i;
    const unsigned long long key = zkey[q];
    filled = key != ~0ull;
    const size_t os = gb->out_stride;
    org_emit (s_o, s_pts, gb->stride, gb->xyz_off, gb->rgba_off, key, out + q * os, os, gb->out_rgba_off);
  }
  const unsigned bal = __ballot_sync (0xffffffffu, filled);
  if ((threadIdx.x & 31) == 0 && bal) atomicAdd (&n_filled[f], (unsigned long long) __popc (bal));
}
#endif

} // namespace b2
