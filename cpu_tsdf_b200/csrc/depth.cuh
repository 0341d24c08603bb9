// depth.cuh — depth images to organised pixels (DESIGN.md §3h).
//
// A depth frame is exactly one integrateCloud of the organised cloud that depth_pixel makes from it: the W x H depth map
// (uint16 sensor units or float32) and an optional registered R,G,B image become the 16-byte pixels {x, y, z, bgra} that the
// unorganised batch path already fuses (stride 16, xyz at 0, colour at 12).  Nothing of the fusion changes.
//
// For pixel (u, v), with the handle's intrinsics rounded to float, every operation float32, rounded to nearest, no contraction:
//   z = (float) D[v*W + u] * scale
//   invalid (D == 0, or z not finite): x = y = z = NaN (0x7fc00000)
//   x = ((float) u - cx) * z / fx,  y = ((float) v - cy) * z / fy      (negative z passes through, as in a cloud)
//   colour word: bytes b, g, r, 255 from the image, or 0, 0, 0, 255 (the default pcl::PointXYZRGBA) without one
//
// k_depth_unproject: one thread per pixel, grid (pixel blocks, m frames); the frames' parameters (DepthBatch) sit in device
// memory behind the batch's frame records, so the launch is captured once and replayed like the organise launches.
#pragma once
#include "tsdf_core.cuh"
#include "organize.cuh"
#include <cstring>

namespace b2 {

constexpr int DEPTH_U16 = 1, DEPTH_F32 = 2;   // B200TSDF_DEPTH_U16, B200TSDF_DEPTH_F32

// one batch of at most ORG_MAX_FRAMES depth frames (device memory)
struct DepthBatch
{
  float fx, fy, cx, cy;                          // (float) of the handle's intrinsics
  float scale;                                   // metres per depth unit: finite and > 0
  int width, height, format;                     // format: DEPTH_U16 or DEPTH_F32
  const void* depth[ORG_MAX_FRAMES];             // W*H values, aligned to their size
  const unsigned char* rgb[ORG_MAX_FRAMES];      // W*H*3 bytes R, G, B, or null
};

B2_HD float depth_qnan ()
{
#ifdef __CUDA_ARCH__
  return __int_as_float (0x7fc00000);
#else
  const unsigned int b = 0x7fc00000u; float f; memcpy (&f, &b, 4); return f;
#endif
}

// the raw value of pixel i as float (exact for uint16)
B2_HD float depth_raw (const void* depth, int format, size_t i)
{
  return format == DEPTH_U16 ? (float) static_cast<const unsigned short*> (depth)[i] : static_cast<const float*> (depth)[i];
}

// the pixel (u, v) of raw depth d and colour bytes rgb (R, G, B; null: none) as {x, y, z} and the colour word
B2_HD void depth_pixel (const DepthBatch& b, float d, const unsigned char* rgb, int u, int v, float* xyz, unsigned int& bgra)
{
  float z = fmul (d, b.scale);
  if (d == 0.f || !(z >= -3.402823466e38f && z <= 3.402823466e38f))
    xyz[0] = xyz[1] = xyz[2] = depth_qnan ();
  else
  {
    xyz[0] = fdiv (fmul (fsub ((float) u, b.cx), z), b.fx);
    xyz[1] = fdiv (fmul (fsub ((float) v, b.cy), z), b.fy);
    xyz[2] = z;
  }
  bgra = rgb ? (unsigned int) rgb[2] | (unsigned int) rgb[1] << 8 | (unsigned int) rgb[0] << 16 | 0xff000000u : 0xff000000u;
}

#ifdef __CUDACC__
// grid (pixel blocks, m): frame blockIdx.y's image starts at out + frame * npix * 16 (16-byte aligned)
__global__ void k_depth_unproject (const DepthBatch* __restrict__ gb, int npix, unsigned char* __restrict__ out)
{
  const int f = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix) return;
  const DepthBatch& b = *gb;
  const int w = b.width;
  const unsigned char* rgb = b.rgb[f];
  float xyz[3]; unsigned int bgra;
  depth_pixel (b, depth_raw (b.depth[f], b.format, (size_t) i), rgb ? rgb + (size_t) i * 3 : nullptr, i % w, i / w, xyz, bgra);
  reinterpret_cast<uint4*> (out)[(size_t) f * npix + i] = make_uint4 (__float_as_uint (xyz[0]), __float_as_uint (xyz[1]), __float_as_uint (xyz[2]), bgra);
}
#endif

} // namespace b2
