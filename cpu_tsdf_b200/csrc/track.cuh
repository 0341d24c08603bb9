// track.cuh — point-to-SDF camera tracking against the volume (DESIGN.md §3i).
//
// One call refines a camera->world pose T so that the live frame's points land on the zero level set of the volume: each
// sample's residual is getFxnAndGradient's value at the transformed point (query_point, mode 1) and its Jacobian comes from
// that gradient.  Gauss-Newton with a Huber weight, damped, over up to TRACK_LEVELS levels of strided samples.
//
// For every iteration at level l with stride s and estimate T:
//   samples   pixels (u, v) with u % s == 0, v % s == 0 and a finite xyz; sample j = (v / s) * ceil (W / s) + u / s
//   q         (float) rows 0..2 of T applied with affine_mul_f (the pre-split's mapping, hpp:76)
//   r, g      query_point mode 1 at q; inlier iff it returns true, every neighbour leaf has w > w_min and |r| < d_max
//   J         [q x g ; g] in double (left perturbation T <- Exp (xi) T, xi = (omega, v))
//   rho       1 if |r| <= delta, else delta / |r|
//   sums      A = sum rho J J^T (upper triangle, 21), b = sum rho J r (6), sum rho r^2, sum r^2, inlier count (TRACK_NS)
//   solve     (A + lambda diag (A)) xi = -b by LDL^T; T <- Exp (xi) T (Rodrigues), rotation re-orthonormalised
//
// Reduction order (fixed by sample index, no floating-point atomics): a tile is TRACK_TILE consecutive samples; thread t of
// the tile's CTA adds samples t, t + 256, t + 512, t + 768 in that order; the 32 lanes of a warp are added by the tree
// v[i] += v[i + h], h = 16, 8, 4, 2, 1; the 8 warp sums by the same tree with h = 4, 2, 1.  The solve warp's lane j adds
// tiles j, j + 32, j + 64, ... in order, and the 32 lanes go through the warp tree.  The host emulation runs the same loops
// with track_tree for the shuffles.
//
// Everything above the kernels is __host__ __device__: tests/emu runs the same code serially.
#pragma once
#include "tsdf_core.cuh"
#include "depth.cuh"

namespace b2 {

constexpr int TRACK_LEVELS = 4, TRACK_MAX_ITERS = 64, TRACK_LOG = TRACK_LEVELS * TRACK_MAX_ITERS;
constexpr int TRACK_BLOCK = 256, TRACK_PER_THREAD = 4, TRACK_TILE = TRACK_BLOCK * TRACK_PER_THREAD;
enum TrackSum { TS_A = 0, TS_B = 21, TS_RHO_R2 = 27, TS_R2 = 28, TS_N = 29, TRACK_NS = 30 };
enum TrackStatus { TRACK_CONVERGED = 0, TRACK_MAX_ITERS_ST = 1, TRACK_TOO_FEW_INLIERS = 2, TRACK_SINGULAR = 3 };

// the per-call inputs, in device memory (nothing of them is baked into a captured graph)
struct TrackInput
{
  const unsigned char* pts;                 // organised cloud: pixel (u, v) at pts + (v * width + u) * stride, xyz at xyz_off
  int stride, xyz_off, width, height;
  int levels, min_inliers;
  float huber, d_max, w_min;
  double damping, eps_rot, eps_trans;
};

// one iteration of the log (layout of b200tsdf_track_iter)
struct TrackIter { int level, inliers; double cost; double step[6]; };

// written by k_track_solve; the host reads it back once per call
struct TrackState
{
  double T[16];                             // the current estimate, row-major camera->world
  float tfwd[12];                           // (float) of its rows 0..2, what k_track_terms applies
  int stop, status;                         // stop: the call ended early with status
  int conv[TRACK_LEVELS];                   // level l ended by the convergence test
  int iters[TRACK_LEVELS];
  int inliers, nlog;
  double rms;                               // sqrt (sum r^2 / inliers) of the last iteration
  double A[36], b[6];                       // normal equations of the last iteration (undamped)
  TrackIter log[TRACK_LOG];
};

// one upload per call: inputs, the depth block of a depth frame, and the state before the first iteration
struct TrackBlock
{
  TrackInput in;
  DepthBatch db;
  TrackState st;
};

B2_HD double dsub (double a, double b) { return dadd (a, -b); }
B2_HD double dsqrt (double a)
{
#ifdef __CUDA_ARCH__
  return __dsqrt_rn (a);
#else
  return sqrt (a);
#endif
}
B2_HD bool dfinite (double a) { return a - a == 0.0; }
B2_HD float f32_of (double a) { return (float) a; }

B2_HD void track_set_pose (TrackState& st, const double* T)
{
  for (int i = 0; i < 16; ++i) st.T[i] = T[i];
  for (int i = 0; i < 12; ++i) st.tfwd[i] = f32_of (T[i]);            // as Frame::tfwd is made (fill_frame)
}

// number of samples of a W x H frame at stride s, and the pixel of sample j
B2_HD int track_cols (int w, int s) { return (w + s - 1) / s; }
B2_HD int track_samples (int w, int h, int s) { return track_cols (w, s) * track_cols (h, s); }

// sample j's contribution, added into acc[TRACK_NS] (nothing for a pixel without a finite xyz or a point that is no inlier)
B2_HD void track_term (const Params& p, const TrackInput& in, const float* tfwd, int s, int j, double* acc)
{
  const int cw = track_cols (in.width, s);
  const int u = (j % cw) * s, v = (j / cw) * s;
  const float* x = reinterpret_cast<const float*> (in.pts + ((size_t) v * in.width + u) * in.stride + in.xyz_off);
  const float px = x[0], py = x[1], pz = x[2];
  if (!(px - px == 0.f && py - py == 0.f && pz - pz == 0.f)) return;
  float q[3], r, g[3], wl;
  affine_mul_f (tfwd, px, py, pz, q);
  if (!query_point_w (p, q, 1, &r, g, nullptr, &wl)) return;
  if (!(wl > in.w_min) || !(fabsf (r) < in.d_max)) return;
  const double qx = q[0], qy = q[1], qz = q[2], gx = g[0], gy = g[1], gz = g[2], rd = r;
  const double J[6] = { dsub (dmul (qy, gz), dmul (qz, gy)), dsub (dmul (qz, gx), dmul (qx, gz)), dsub (dmul (qx, gy), dmul (qy, gx)), gx, gy, gz };
  const double ar = fabs (rd), delta = in.huber;
  const double rho = ar <= delta ? 1.0 : ddiv (delta, ar);
  int k = TS_A;
  for (int a = 0; a < 6; ++a)
  {
    const double rj = dmul (rho, J[a]);
    for (int c = a; c < 6; ++c, ++k) acc[k] = dadd (acc[k], dmul (rj, J[c]));
    acc[TS_B + a] = dadd (acc[TS_B + a], dmul (rj, rd));
  }
  acc[TS_RHO_R2] = dadd (acc[TS_RHO_R2], dmul (dmul (rho, rd), rd));
  acc[TS_R2] = dadd (acc[TS_R2], dmul (rd, rd));
  acc[TS_N] = dadd (acc[TS_N], 1.0);
}

// ---- the reduction order, stated for the host (the kernels do the same with shuffles) ----------------------------------
// v[n][TRACK_NS], n a power of two: v[0] <- the tree v[i] += v[i + h], h = n/2 .. 1
B2_HD void track_tree (double (*v)[TRACK_NS], int n)
{
  for (int h = n / 2; h >= 1; h /= 2)
    for (int i = 0; i < h; ++i)
      for (int k = 0; k < TRACK_NS; ++k) v[i][k] = dadd (v[i][k], v[i + h][k]);
}

// ---- solve6: (A + lambda diag (A)) x = -b by LDL^T; false on a pivot that is not > 0 ------------------------------------
B2_HD bool solve6 (const double* A, double lambda, const double* b, double* x)
{
  double L[6][6], D[6], y[6];
  for (int j = 0; j < 6; ++j)
  {
    double d = dadd (A[7 * j], dmul (lambda, A[7 * j]));
    for (int k = 0; k < j; ++k) d = dsub (d, dmul (dmul (L[j][k], L[j][k]), D[k]));
    if (!(d > 0.0)) return false;
    D[j] = d;
    for (int i = j + 1; i < 6; ++i)
    {
      double m = A[6 * i + j];
      for (int k = 0; k < j; ++k) m = dsub (m, dmul (dmul (L[i][k], L[j][k]), D[k]));
      L[i][j] = ddiv (m, d);
    }
  }
  for (int i = 0; i < 6; ++i)
  {
    double t = -b[i];
    for (int k = 0; k < i; ++k) t = dsub (t, dmul (L[i][k], y[k]));
    y[i] = t;
  }
  for (int i = 5; i >= 0; --i)
  {
    double t = ddiv (y[i], D[i]);
    for (int k = i + 1; k < 6; ++k) t = dsub (t, dmul (L[k][i], x[k]));
    x[i] = t;
  }
  return true;
}

// ---- se3_exp_left: Tout = Exp (xi) T, xi = (omega, v); rotation rows re-orthonormalised --------------------------------
// sin t / t, (1 - cos t) / t^2 and (t - sin t) / t^3 by their Taylor series in x = t^2 (Horner, 16 terms: below 1e-20 for
// t <= pi), so that host and device round alike (the libm sin / cos differ between them)
B2_HD double track_series (double x, int first)
{
  // sum_k (-x)^k / (2k + first)!  =  1/first! (1 - x / ((first+1)(first+2)) (1 - x / ((first+3)(first+4)) (...)))
  double s = 1.0;
  for (int k = 15; k >= 1; --k)
  {
    const double n = (double) (2 * k + first);
    s = dsub (1.0, dmul (ddiv (x, dmul (n - 1.0, n)), s));
  }
  double f = 1.0;
  for (int i = 2; i <= first; ++i) f = dmul (f, (double) i);
  return ddiv (s, f);
}

B2_HD void se3_exp_left (const double* xi, const double* T, double* out)
{
  const double w0 = xi[0], w1 = xi[1], w2 = xi[2];
  const double th2 = dadd (dadd (dmul (w0, w0), dmul (w1, w1)), dmul (w2, w2));
  const double a = track_series (th2, 1), b = track_series (th2, 2), c = track_series (th2, 3);
  const double W[9] = { 0.0, -w2, w1, w2, 0.0, -w0, -w1, w0, 0.0 };
  double W2[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j)
      W2[3 * i + j] = dadd (dadd (dmul (W[3 * i], W[j]), dmul (W[3 * i + 1], W[3 + j])), dmul (W[3 * i + 2], W[6 + j]));
  double R[9], V[9];
  for (int i = 0; i < 9; ++i)
  {
    const double id = (i % 4 == 0) ? 1.0 : 0.0;
    R[i] = dadd (dadd (id, dmul (a, W[i])), dmul (b, W2[i]));
    V[i] = dadd (dadd (id, dmul (b, W[i])), dmul (c, W2[i]));
  }
  double t[3];
  for (int i = 0; i < 3; ++i) t[i] = dadd (dadd (dmul (V[3 * i], xi[3]), dmul (V[3 * i + 1], xi[4])), dmul (V[3 * i + 2], xi[5]));
  double M[9], tn[3];
  for (int i = 0; i < 3; ++i)
  {
    for (int j = 0; j < 3; ++j)
      M[3 * i + j] = dadd (dadd (dmul (R[3 * i], T[j]), dmul (R[3 * i + 1], T[4 + j])), dmul (R[3 * i + 2], T[8 + j]));
    tn[i] = dadd (dadd (dadd (dmul (R[3 * i], T[3]), dmul (R[3 * i + 1], T[7])), dmul (R[3 * i + 2], T[11])), t[i]);
  }
  // Gram-Schmidt on the rows: r0 / |r0|, r1 - (r0.r1) r0 normalised, r2 = r0 x r1
  double* r0 = M; double* r1 = M + 3; double* r2 = M + 6;
  double n0 = dsqrt (dadd (dadd (dmul (r0[0], r0[0]), dmul (r0[1], r0[1])), dmul (r0[2], r0[2])));
  for (int k = 0; k < 3; ++k) r0[k] = ddiv (r0[k], n0);
  const double d01 = dadd (dadd (dmul (r0[0], r1[0]), dmul (r0[1], r1[1])), dmul (r0[2], r1[2]));
  for (int k = 0; k < 3; ++k) r1[k] = dsub (r1[k], dmul (d01, r0[k]));
  double n1 = dsqrt (dadd (dadd (dmul (r1[0], r1[0]), dmul (r1[1], r1[1])), dmul (r1[2], r1[2])));
  for (int k = 0; k < 3; ++k) r1[k] = ddiv (r1[k], n1);
  r2[0] = dsub (dmul (r0[1], r1[2]), dmul (r0[2], r1[1]));
  r2[1] = dsub (dmul (r0[2], r1[0]), dmul (r0[0], r1[2]));
  r2[2] = dsub (dmul (r0[0], r1[1]), dmul (r0[1], r1[0]));
  for (int i = 0; i < 3; ++i)
  {
    for (int j = 0; j < 3; ++j) out[4 * i + j] = M[3 * i + j];
    out[4 * i + 3] = tn[i];
  }
  out[12] = 0.0; out[13] = 0.0; out[14] = 0.0; out[15] = 1.0;
}

// ---- one Gauss-Newton update from the summed terms of iteration `level` ------------------------------------------------
B2_HD void track_update (TrackState& st, const TrackInput& in, int level, const double* sums)
{
  int k = TS_A;
  for (int a = 0; a < 6; ++a)
  {
    for (int c = a; c < 6; ++c, ++k) { st.A[6 * a + c] = sums[k]; st.A[6 * c + a] = sums[k]; }
    st.b[a] = sums[TS_B + a];
  }
  const int n = (int) sums[TS_N];
  st.inliers = n;
  st.rms = n ? dsqrt (ddiv (sums[TS_R2], (double) n)) : 0.0;
  st.iters[level]++;
  TrackIter& e = st.log[st.nlog++];
  e.level = level; e.inliers = n; e.cost = sums[TS_RHO_R2];
  for (int i = 0; i < 6; ++i) e.step[i] = 0.0;
  if (n < in.min_inliers) { st.stop = 1; st.status = TRACK_TOO_FEW_INLIERS; return; }
  double xi[6];
  bool ok = solve6 (st.A, in.damping, st.b, xi);
  for (int i = 0; i < 6 && ok; ++i) ok = dfinite (xi[i]);
  if (!ok) { st.stop = 1; st.status = TRACK_SINGULAR; return; }
  double Tn[16];
  se3_exp_left (xi, st.T, Tn);
  for (int i = 0; i < 12 && ok; ++i) ok = dfinite (Tn[i]);
  if (!ok) { st.stop = 1; st.status = TRACK_SINGULAR; return; }
  track_set_pose (st, Tn);
  for (int i = 0; i < 6; ++i) e.step[i] = xi[i];
  const double nw = dsqrt (dadd (dadd (dmul (xi[0], xi[0]), dmul (xi[1], xi[1])), dmul (xi[2], xi[2])));
  const double nv = dsqrt (dadd (dadd (dmul (xi[3], xi[3]), dmul (xi[4], xi[4])), dmul (xi[5], xi[5])));
  if (nw < in.eps_rot && nv < in.eps_trans) st.conv[level] = 1;
}

// the status of a call that did not stop early: converged iff its last level ended by the convergence test
B2_HD int track_final_status (const TrackState& st, int levels)
{
  if (st.stop) return st.status;
  return st.conv[levels - 1] ? TRACK_CONVERGED : TRACK_MAX_ITERS_ST;
}

#ifdef __CUDACC__
// one CTA of TRACK_BLOCK threads per tile of TRACK_TILE samples at stride s; tile sums go to part[k * cap + tile]
__global__ void __launch_bounds__ (TRACK_BLOCK) k_track_terms (Params gp, const TrackBlock* __restrict__ blk, int level, int s,
                                                               double* __restrict__ part, int cap)
{
  const TrackState& st = blk->st;
  if (st.stop || st.conv[level]) return;
  __shared__ Params sp;
  __shared__ float s_tf[12];
  __shared__ double s_w[TRACK_BLOCK / 32][TRACK_NS];
  {
    const int* src = reinterpret_cast<const int*> (&gp);
    int* dst = reinterpret_cast<int*> (&sp);
    for (int w = threadIdx.x; w < (int) (sizeof (Params) / sizeof (int)); w += blockDim.x) dst[w] = src[w];
    if (threadIdx.x < 12) s_tf[threadIdx.x] = st.tfwd[threadIdx.x];
  }
  __syncthreads ();
  const TrackInput& in = blk->in;
  const int n = track_samples (in.width, in.height, s);
  double acc[TRACK_NS];
  for (int k = 0; k < TRACK_NS; ++k) acc[k] = 0.0;
  const int base = blockIdx.x * TRACK_TILE + threadIdx.x;
  for (int i = 0; i < TRACK_PER_THREAD; ++i)
  {
    const int j = base + i * TRACK_BLOCK;
    if (j < n) track_term (sp, in, s_tf, s, j, acc);
  }
  for (int h = 16; h >= 1; h /= 2)
    for (int k = 0; k < TRACK_NS; ++k) acc[k] = dadd (acc[k], __shfl_down_sync (0xffffffffu, acc[k], h));
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0)
    for (int k = 0; k < TRACK_NS; ++k) s_w[wid][k] = acc[k];
  __syncthreads ();
  if (threadIdx.x < TRACK_NS)
  {
    const int k = threadIdx.x;
    double v[8];
    for (int w = 0; w < 8; ++w) v[w] = s_w[w][k];
    for (int h = 4; h >= 1; h /= 2)
      for (int w = 0; w < h; ++w) v[w] = dadd (v[w], v[w + h]);
    part[(size_t) k * cap + blockIdx.x] = v[0];
  }
}

// one warp: the tiles' sums in the fixed order, then lane 0 solves and updates the state
__global__ void __launch_bounds__ (32) k_track_solve (TrackBlock* __restrict__ blk, int level, int tiles, const double* __restrict__ part, int cap)
{
  TrackState& st = blk->st;
  if (st.stop || st.conv[level]) return;
  const int lane = threadIdx.x;
  double acc[TRACK_NS];
  for (int k = 0; k < TRACK_NS; ++k) acc[k] = 0.0;
  for (int t = lane; t < tiles; t += 32)
    for (int k = 0; k < TRACK_NS; ++k) acc[k] = dadd (acc[k], part[(size_t) k * cap + t]);
  for (int h = 16; h >= 1; h /= 2)
    for (int k = 0; k < TRACK_NS; ++k) acc[k] = dadd (acc[k], __shfl_down_sync (0xffffffffu, acc[k], h));
  if (lane == 0) track_update (st, blk->in, level, acc);
}
#endif

} // namespace b2
