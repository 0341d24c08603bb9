// tests/emu/org_batch_emu.cpp — HOST EMULATION of the batched organise kernels.  TEST HARNESS ONLY.
//
// Drives k_org_zmin / k_org_gather's per-point and per-pixel code of organize.cuh serially on the host: the batch's points are
// concatenated, each flat index is mapped to its frame and its index within the frame (org_frame_of) and z-buffered with that
// frame's parameters (org_frame_params), in REVERSE flat order (the device order is arbitrary: the result must not depend on it).
#include "../../cpu_tsdf_b200/csrc/tsdf_core.cuh"
#include "../../cpu_tsdf_b200/csrc/organize.cuh"

#include <algorithm>
#include <vector>

using namespace b2;

// m clouds pts[i] of counts[i] points; w2c: null or m row-major 4x4 matrices.  out: m images of width*height pixels of out_stride
// bytes; zkey: m*width*height keys; filled: m counts; map (may be null): per flat point index {frame, index within the frame}.
extern "C" int emu_organize_batch (int m, const void* const* pts, const unsigned long long* counts, size_t stride, int xyz_off, int rgba_off,
                                   const float* intr, int width, int height, float cloud_units, int zero_nans, const double* w2c,
                                   void* out, size_t out_stride, int out_rgba_off, unsigned long long* zkey, long long* filled,
                                   unsigned long long* map)
{
  if (m < 1 || m > ORG_MAX_FRAMES) return -1;
  OrgBatch b{};
  b.o.fx = intr[0]; b.o.fy = intr[1]; b.o.cx = intr[2]; b.o.cy = intr[3]; b.o.width = width; b.o.height = height;
  b.o.cloud_units = cloud_units; b.o.zero_nans = zero_nans;
  b.stride = stride; b.xyz_off = xyz_off; b.rgba_off = rgba_off; b.out_stride = out_stride; b.out_rgba_off = out_rgba_off;
  std::vector<OrgRec> recs (m);
  unsigned long long first[ORG_MAX_FRAMES], total = 0;
  for (int f = 0; f < m; ++f)
  {
    recs[f] = OrgRec{};
    recs[f].pts = (const unsigned char*) pts[f]; recs[f].count = counts[f]; recs[f].first = total;
    recs[f].has_tf = w2c != nullptr;
    if (w2c) for (int i = 0; i < 12; ++i) recs[f].tf[i] = w2c[16 * f + i];
    first[f] = total; total += counts[f];
  }
  const size_t npix = (size_t) width * height;
  std::fill (zkey, zkey + (size_t) m * npix, ~0ull);
  for (unsigned long long k = total; k-- > 0;)
  {
    const int f = org_frame_of (first, m, k);
    const unsigned long long j = k - first[f];
    if (map) { map[2 * k] = (unsigned long long) f; map[2 * k + 1] = j; }
    const OrgParams o = org_frame_params (b, recs[f]);
    float x, y, z;
    org_load (recs[f].pts, b.stride, b.xyz_off, j, x, y, z);
    org_prepare (o, x, y, z);
    const int pix = org_pixel (o, x, y, z);
    if (pix < 0) continue;
    unsigned long long& zk = zkey[(size_t) f * npix + pix];
    zk = std::min (zk, org_key (z, (unsigned int) j));
  }
  for (int f = 0; f < m; ++f)
  {
    const OrgParams o = org_frame_params (b, recs[f]);
    filled[f] = 0;
    for (size_t i = 0; i < npix; ++i)
    {
      const size_t q = (size_t) f * npix + i;
      filled[f] += zkey[q] != ~0ull;
      org_emit (o, recs[f].pts, b.stride, b.xyz_off, b.rgba_off, zkey[q], (unsigned char*) out + q * out_stride, out_stride, out_rgba_off);
    }
  }
  return 0;
}
