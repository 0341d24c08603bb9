// tests/emu/track_emu.cpp — HOST EMULATION of the tracking kernels (track.cuh, DESIGN.md §3i).  TEST HARNESS ONLY.
//
// Compiles the emulation of emu.cpp and adds, on the emulated volume:
//   track_run: one b200tsdf_track_cloud_device call, the launches of its graph in order — k_track_terms' tiles (track_term per
//     sample, each thread's samples in order, the warp and CTA trees) and k_track_solve's fold of the tiles (lane sums, warp
//     tree) and track_update — with the same result and log;
//   track_samples_dump: every sample's point q, query result, r, g, smallest neighbour weight and inlier flag at one pose;
//   track_sums_once: the sums of one iteration at one pose, in the kernels' order;
//   track_solve6 / track_exp: solve6 and se3_exp_left.
// A depth map is tracked as the cloud of 16-byte pixels k_depth_unproject makes of it (depth_emu.cpp).
#include "emu.cpp"
#include "../../cpu_tsdf_b200/csrc/track.cuh"

#include <vector>

namespace {

TrackInput make_input (const b200tsdf_track_params* prm, const void* pts, int stride, int xyz_off, int W, int H)
{
  TrackInput in{};
  in.pts = static_cast<const unsigned char*> (pts); in.stride = stride; in.xyz_off = xyz_off; in.width = W; in.height = H;
  in.levels = prm->levels; in.min_inliers = prm->min_inliers;
  in.huber = prm->huber_delta; in.d_max = prm->d_max; in.w_min = prm->w_min;
  in.damping = prm->damping; in.eps_rot = prm->eps_rot; in.eps_trans = prm->eps_trans;
  return in;
}

// k_track_terms for every tile: part[k * tiles + tile]
void terms (const Params& p, const TrackInput& in, const float* tfwd, int s, std::vector<double>& part, int& tiles)
{
  const int n = track_samples (in.width, in.height, s);
  tiles = (n + TRACK_TILE - 1) / TRACK_TILE;
  part.assign ((size_t) tiles * TRACK_NS, 0.0);
  std::vector<double> v ((size_t) TRACK_BLOCK * TRACK_NS);
  double (*t)[TRACK_NS] = reinterpret_cast<double (*)[TRACK_NS]> (v.data ());
  for (int b = 0; b < tiles; ++b)
  {
    std::fill (v.begin (), v.end (), 0.0);
    for (int th = 0; th < TRACK_BLOCK; ++th)
      for (int i = 0; i < TRACK_PER_THREAD; ++i)
      {
        const int j = b * TRACK_TILE + th + i * TRACK_BLOCK;
        if (j < n) track_term (p, in, tfwd, s, j, t[th]);
      }
    double w[TRACK_BLOCK / 32][TRACK_NS];
    for (int k = 0; k < TRACK_BLOCK / 32; ++k)
    {
      track_tree (t + 32 * k, 32);
      for (int c = 0; c < TRACK_NS; ++c) w[k][c] = t[32 * k][c];
    }
    track_tree (w, TRACK_BLOCK / 32);
    for (int c = 0; c < TRACK_NS; ++c) part[(size_t) c * tiles + b] = w[0][c];
  }
}

// k_track_solve's fold of the tiles into sums[TRACK_NS]
void fold (const std::vector<double>& part, int tiles, double* sums)
{
  double lanes[32][TRACK_NS] = {};
  for (int l = 0; l < 32; ++l)
    for (int b = l; b < tiles; b += 32)
      for (int c = 0; c < TRACK_NS; ++c) lanes[l][c] = dadd (lanes[l][c], part[(size_t) c * tiles + b]);
  track_tree (lanes, 32);
  for (int c = 0; c < TRACK_NS; ++c) sums[c] = lanes[0][c];
}

} // namespace

extern "C" {

int track_run (const Emu* e, const void* pts, int stride, int xyz_off, int W, int H, const double* pose0,
               const b200tsdf_track_params* prm, b200tsdf_track_result* res, b200tsdf_track_iter* log)
{
  const TrackInput in = make_input (prm, pts, stride, xyz_off, W, H);
  TrackState* st = new TrackState ();
  track_set_pose (*st, pose0);
  std::vector<double> part;
  for (int l = 0; l < prm->levels; ++l)
    for (int k = 0; k < prm->iters[l]; ++k)
    {
      if (st->stop || st->conv[l]) continue;
      int tiles = 0;
      terms (e->p, in, st->tfwd, prm->stride[l], part, tiles);
      double sums[TRACK_NS];
      fold (part, tiles, sums);
      track_update (*st, in, l, sums);
    }
  std::memcpy (res->pose_c2w, st->T, sizeof (st->T));
  res->status = track_final_status (*st, prm->levels);
  for (int l = 0; l < TRACK_LEVELS; ++l) res->iters[l] = st->iters[l];
  res->inliers = st->inliers; res->n_log = st->nlog; res->reserved = 0; res->rms = st->rms;
  std::memcpy (res->A, st->A, sizeof (st->A)); std::memcpy (res->b, st->b, sizeof (st->b));
  if (log && st->nlog) std::memcpy (log, st->log, (size_t) st->nlog * sizeof (TrackIter));
  delete st;
  return 0;
}

// per sample j < track_samples (W, H, s): q[3], r, g[3], wlo, flags (bit0 finite xyz, bit1 query ok, bit2 inlier)
int track_samples_dump (const Emu* e, const void* pts, int stride, int xyz_off, int W, int H, const double* pose, int s,
                        const b200tsdf_track_params* prm, float* q, float* r, float* g, float* wlo, uint8_t* flags)
{
  const TrackInput in = make_input (prm, pts, stride, xyz_off, W, H);
  TrackState st{};
  track_set_pose (st, pose);
  const int n = track_samples (W, H, s), cw = track_cols (W, s);
  for (int j = 0; j < n; ++j)
  {
    const int u = (j % cw) * s, v = (j / cw) * s;
    const float* x = reinterpret_cast<const float*> (in.pts + ((size_t) v * W + u) * stride + xyz_off);
    flags[j] = 0;
    if (!(std::isfinite (x[0]) && std::isfinite (x[1]) && std::isfinite (x[2]))) continue;
    flags[j] = 1;
    affine_mul_f (st.tfwd, x[0], x[1], x[2], q + 3 * j);
    if (!query_point_w (e->p, q + 3 * j, 1, r + j, g + 3 * j, nullptr, wlo + j)) continue;
    flags[j] |= 2;
    double acc[TRACK_NS] = {};
    track_term (e->p, in, st.tfwd, s, j, acc);
    if (acc[TS_N] == 1.0) flags[j] |= 4;
  }
  return n;
}

void track_sums_once (const Emu* e, const void* pts, int stride, int xyz_off, int W, int H, const double* pose, int s,
                      const b200tsdf_track_params* prm, double* sums)
{
  const TrackInput in = make_input (prm, pts, stride, xyz_off, W, H);
  TrackState st{};
  track_set_pose (st, pose);
  std::vector<double> part;
  int tiles = 0;
  terms (e->p, in, st.tfwd, s, part, tiles);
  fold (part, tiles, sums);
}

int track_solve6 (const double* A, double lambda, const double* b, double* x) { return solve6 (A, lambda, b, x) ? 1 : 0; }
void track_exp (const double* xi, const double* T, double* out) { se3_exp_left (xi, T, out); }

} // extern "C"
