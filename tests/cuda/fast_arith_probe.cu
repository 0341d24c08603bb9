// fast_arith_probe.cu — test-only entry points (ctypes) that run the brick kernels' arithmetic shortcuts on the device:
// div_recip / div_with against __fdiv_rn, the guarded projection of observe_issue, tsdf_core.cuh::project1 and
// float_at_least.  Every entry point calls the engine's own header functions; Params comes from derive_params, so
// fast_proj, proj_guard and exact_div_ok are the values the engine would use.  Built by tests/cuda/build_probe.py into
// a library of its own that libb200tsdf.so does not link.  Entry points return 0, or a CUDA error code, or -1 when
// derive_params refuses the configuration.
#include "../../cpu_tsdf_b200/csrc/params_setup.h"
#include "../../cpu_tsdf_b200/csrc/obs_fast.cuh"
#include <cuda_runtime.h>
#include <vector>

using namespace b2;

namespace {

// exponent bucket of the division map: 0 for +-0, ilogb (|x|) + 150 otherwise (1 = 2^-149 ... 277 = 2^127)
constexpr int NE = 278;
__device__ __forceinline__ int ebucket (float x)
{
  const uint32_t m = __float_as_uint (x) & 0x7FFFFFFFu;
  if (m == 0u) return 0;
  const int e = (int) (m >> 23);
  return e ? e + 23 : 32 - __clz (m);            // normal: (e - 127) + 150; subnormal: bit length of the mantissa
}

__device__ __forceinline__ uint64_t splitmix (uint64_t& s)
{
  uint64_t z = (s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

struct Miss { unsigned long long* n; float* first; int max_first; };

// div_fast (RAW, the unguarded sequence) or div_with against __fdiv_rn
template <bool RAW>
__device__ __forceinline__ void check_div (float a, float b, float r, unsigned long long* hist, const Miss& m)
{
  const float w = RAW ? div_fast (a, b, r) : div_with (a, b, r), e = __fdiv_rn (a, b);
  if (__float_as_uint (w) != __float_as_uint (e))
  {
    if (hist) atomicAdd (hist + ebucket (a) * NE + ebucket (b), 1ull);
    const unsigned long long k = atomicAdd (m.n, 1ull);
    if (k < (unsigned long long) m.max_first)
    { m.first[4 * k] = a; m.first[4 * k + 1] = b; m.first[4 * k + 2] = w; m.first[4 * k + 3] = e; }
  }
}

__global__ void k_div (int n, const float* a, const float* b, float* ow, float* oe)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  ow[i] = div_with (a[i], b[i], div_recip (b[i]));
  oe[i] = __fdiv_rn (a[i], b[i]);
}

// div_fast, one thread per divisor: every mantissa (step `mstep`) of binade `bexp[blockIdx.y]`, against every numerator
__global__ void k_div_map (const int* bexp, int mstep, const float* num, int n_num, unsigned long long* hist, Miss m)
{
  const uint32_t mant = (blockIdx.x * blockDim.x + threadIdx.x) * (uint32_t) mstep;
  if (mant >= (1u << 23)) return;
  const float b = __uint_as_float (((uint32_t) (bexp[blockIdx.y] + 127) << 23) | mant);
  const float r = div_recip (b);
  for (int j = 0; j < n_num; ++j) check_div<true> (num[j], b, r, hist, m);
}

// div_with (or div_fast when `raw`) on random pairs: b with its bits uniform over [bits (b_lo), bits (b_hi)] (b_lo > 0); a = +-0 with probability 1/64, otherwise
// |a| with its bits uniform over [bits (a_min), bits (a_max)] and a random sign when `signed_a`; with `neg_le_b` a negative
// numerator is drawn again from [a_min, b] (the clamped observation d_new >= -max_dist_neg)
__global__ void k_div_random (uint64_t seed, int per_thread, float b_lo, float b_hi, float a_min, float a_max, int signed_a,
                              int neg_le_b, int raw, Miss m)
{
  uint64_t s = seed ^ ((uint64_t) (blockIdx.x * blockDim.x + threadIdx.x) * 0xD1B54A32D192ED03ull);
  const uint32_t bl = __float_as_uint (b_lo), bh = __float_as_uint (b_hi), al = __float_as_uint (a_min), ah = __float_as_uint (a_max);
  for (int it = 0; it < per_thread; ++it)
  {
    const uint64_t x = splitmix (s), y = splitmix (s);
    const float b = __uint_as_float (bl + (uint32_t) ((x & 0xFFFFFFFFull) % (uint64_t) (bh - bl + 1)));
    const bool neg = signed_a && ((x >> 32) & 1);
    uint32_t ab;
    if (((x >> 33) & 63) == 0) ab = 0u;
    else
    {
      const uint32_t hi = (neg && neg_le_b && __float_as_uint (b) < ah) ? __float_as_uint (b) : ah;
      ab = al + (uint32_t) ((y & 0xFFFFFFFFull) % (uint64_t) (hi - al + 1));
    }
    const float a = __uint_as_float (ab | (neg ? 0x80000000u : 0u));
    if (raw) check_div<true> (a, b, div_recip (b), nullptr, m);
    else check_div<false> (a, b, div_recip (b), nullptr, m);
  }
}

__global__ void k_observe (Params p, int n, const float* vx, const float* vy, const float* vz, int* ou, int* ov, int* oin,
                           float* oau, float* oav)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  FrameHot F; F.pix = p.pix;
  const ObsP o = observe_issue<false> (p, F, vx[i], vy[i], vz[i]);
  oin[i] = o.inimg;
  ou[i] = o.uv & 0xFFFF; ov[i] = o.uv >> 16;
  const float r = rcp_approx (vz[i]);
  oau[i] = proj_estimate (vx[i], p.fx_f, r, p.cx_f); oav[i] = proj_estimate (vy[i], p.fy_f, r, p.cy_f);
}

__global__ void k_project1 (Params p, int n, int axis, const float* x, const float* z, int* out, float* oa)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double fd = axis ? p.fy : p.fx, cd = axis ? p.cy : p.cx;
  const float ff = axis ? p.fy_f : p.fx_f, cf = axis ? p.cy_f : p.cx_f;
  out[i] = project1 (p, x[i], z[i], fd, cd, ff, cf);
  oa[i] = project1_estimate (x[i], z[i], ff, cf);
}

__global__ void k_at_least (int n, const double* t, float* out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = float_at_least (t[i]);
}

__global__ void k_near_threshold (int n, const float* size, double* out)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = near_threshold (size[i]);
}

template <class T> struct Dev
{
  T* p = nullptr;
  explicit Dev (size_t n) { cudaMalloc (&p, (n ? n : 1) * sizeof (T)); }
  Dev (const T* h, size_t n) : Dev (n) { cudaMemcpy (p, h, n * sizeof (T), cudaMemcpyHostToDevice); }
  void get (T* h, size_t n) const { cudaMemcpy (h, p, n * sizeof (T), cudaMemcpyDeviceToHost); }
  ~Dev () { cudaFree (p); }
  Dev (const Dev&) = delete;
};

int status () { cudaError_t e = cudaDeviceSynchronize (); if (e == cudaSuccess) e = cudaGetLastError (); return (int) e; }
int blocks (long long n, int t = 256) { return (int) ((n + t - 1) / t); }

struct MissDev
{
  Dev<unsigned long long> n; Dev<float> first; int max_first;
  explicit MissDev (int mf) : n (1), first (4 * (size_t) mf), max_first (mf) { cudaMemset (n.p, 0, sizeof (unsigned long long)); }
  Miss view () const { return Miss { n.p, first.p, max_first }; }
  void get (unsigned long long* n_out, float* first_out) const
  {
    n.get (n_out, 1);
    first.get (first_out, 4 * (size_t) (*n_out < (unsigned long long) max_first ? *n_out : max_first));
  }
};

} // namespace

extern "C" {

struct ProbeParams
{
  int fast_proj, exact_div_ok, width, height, L;
  float proj_guard, rc_lo_f, rc_hi_f;
  double rc_thresh;
};

int probe_params (const b200tsdf_config* c, ProbeParams* out)
{
  Params p{}; size_t pool, root_n;
  if (derive_params (*c, p, pool, root_n)) return -1;
  out->fast_proj = p.fast_proj; out->exact_div_ok = p.exact_div_ok; out->width = p.width; out->height = p.height; out->L = p.L;
  out->proj_guard = p.proj_guard; out->rc_lo_f = p.rc_lo_f; out->rc_hi_f = p.rc_hi_f; out->rc_thresh = p.rc_thresh;
  return 0;
}

int probe_div (int n, const float* a, const float* b, float* out_with, float* out_ieee)
{
  Dev<float> da (a, n), db (b, n), dw (n), de (n);
  k_div<<<blocks (n), 256>>> (n, da.p, db.p, dw.p, de.p);
  int e = status ();
  dw.get (out_with, n); de.get (out_ieee, n);
  return e;
}

// hist: [278 x 278] counts of mismatching pairs by (exponent bucket of a, of b); first: up to max_first (a, b, with, ieee)
int probe_div_map (int n_bexp, const int* bexp, int mstep, int n_num, const float* num, unsigned long long* hist,
                   unsigned long long* n_miss, float* first, int max_first)
{
  Dev<int> db (bexp, n_bexp); Dev<float> dn (num, n_num); Dev<unsigned long long> dh ((size_t) NE * NE);
  cudaMemset (dh.p, 0, sizeof (unsigned long long) * NE * NE);
  MissDev m (max_first);
  const dim3 grid (blocks (((1 << 23) + mstep - 1) / mstep), n_bexp);
  k_div_map<<<grid, 256>>> (db.p, mstep, dn.p, n_num, dh.p, m.view ());
  int e = status ();
  dh.get (hist, (size_t) NE * NE); m.get (n_miss, first);
  return e;
}

int probe_div_random (unsigned long long seed, long long n, float b_lo, float b_hi, float a_min, float a_max, int signed_a,
                      int neg_le_b, int raw, unsigned long long* n_miss, float* first, int max_first)
{
  MissDev m (max_first);
  const int threads = 132 * 2048, per = (int) ((n + threads - 1) / threads);
  k_div_random<<<threads / 256, 256>>> (seed, per, b_lo, b_hi, a_min, a_max, signed_a, neg_le_b, raw, m.view ());
  int e = status ();
  m.get (n_miss, first);
  return e;
}

// observe_issue<false> on a zero pixel plane of width x height entries: u, v (valid when inimg), inimg, and the float
// estimates au, av of the fast projection (computed whether or not fast_proj is on)
int probe_observe (const b200tsdf_config* c, int n, const float* vx, const float* vy, const float* vz, int* out_u, int* out_v,
                   int* out_inimg, float* out_au, float* out_av)
{
  Params p{}; size_t pool, root_n;
  if (derive_params (*c, p, pool, root_n)) return -1;
  Dev<uint32_t> pix ((size_t) p.width * p.height);
  cudaMemset (pix.p, 0, sizeof (uint32_t) * (size_t) p.width * p.height);
  p.pix = pix.p;
  Dev<float> dx (vx, n), dy (vy, n), dz (vz, n), dau (n), dav (n);
  Dev<int> du (n), dv (n), di (n);
  k_observe<<<blocks (n), 256>>> (p, n, dx.p, dy.p, dz.p, du.p, dv.p, di.p, dau.p, dav.p);
  int e = status ();
  du.get (out_u, n); dv.get (out_v, n); di.get (out_inimg, n); dau.get (out_au, n); dav.get (out_av, n);
  return e;
}

// project1 along axis 0 (fx, cx) or 1 (fy, cy), and its float estimate
int probe_project1 (const b200tsdf_config* c, int axis, int n, const float* x, const float* z, int* out, float* out_a)
{
  Params p{}; size_t pool, root_n;
  if (derive_params (*c, p, pool, root_n)) return -1;
  Dev<float> dx (x, n), dz (z, n), da (n);
  Dev<int> dout (n);
  k_project1<<<blocks (n), 256>>> (p, n, axis, dx.p, dz.p, dout.p, da.p);
  int e = status ();
  dout.get (out, n); da.get (out_a, n);
  return e;
}

// float_at_least (t) on the device and params_setup.h's at_least (t) on the host, for each t
int probe_at_least (int n, const double* t, float* out_dev, float* out_host)
{
  Dev<double> dt (t, n); Dev<float> d (n);
  k_at_least<<<blocks (n), 256>>> (n, dt.p, d.p);
  int e = status ();
  d.get (out_dev, n);
  for (int i = 0; i < n; ++i) out_host[i] = at_least (t[i]);
  return e;
}

// near_threshold (size) on the device and on the host
int probe_near_threshold (int n, const float* size, double* out_dev, double* out_host)
{
  Dev<float> ds (size, n); Dev<double> d (n);
  k_near_threshold<<<blocks (n), 256>>> (n, ds.p, d.p);
  int e = status ();
  d.get (out_dev, n);
  for (int i = 0; i < n; ++i) out_host[i] = near_threshold (size[i]);
  return e;
}

} // extern "C"
