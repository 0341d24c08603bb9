// tests/emu/depth_emu.cpp — HOST EMULATION of k_depth_unproject (depth.cuh).  TEST HARNESS ONLY.
//
// Runs the kernel's per-pixel routine (depth_raw, depth_pixel) serially on the host and writes the same 16-byte pixels
// {x, y, z, bgra}.
#include "../../cpu_tsdf_b200/csrc/tsdf_core.cuh"
#include "../../cpu_tsdf_b200/csrc/depth.cuh"

#include <cstring>

using namespace b2;

// intr: fx, fy, cx, cy as float; rgb: width*height*3 bytes or null; out: width*height*16 bytes
extern "C" void emu_depth_to_cloud (const void* depth, int format, float scale, const unsigned char* rgb, int width, int height,
                                    const float* intr, unsigned char* out)
{
  DepthBatch b{};
  b.fx = intr[0]; b.fy = intr[1]; b.cx = intr[2]; b.cy = intr[3];
  b.scale = scale; b.width = width; b.height = height; b.format = format;
  const size_t npix = (size_t) width * height;
  for (size_t i = 0; i < npix; ++i)
  {
    float xyz[3]; unsigned int bgra;
    depth_pixel (b, depth_raw (depth, format, i), rgb ? rgb + i * 3 : nullptr, (int) (i % width), (int) (i / width), xyz, bgra);
    std::memcpy (out + i * 16, xyz, 12);
    std::memcpy (out + i * 16 + 12, &bgra, 4);
  }
}
