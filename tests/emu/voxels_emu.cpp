// tests/emu/voxels_emu.cpp — HOST EMULATION of the engine's point lookup and dense crop (k_voxels / k_dense in engine.cu).
// TEST HARNESS ONLY.
//
// Compiles the emulation of emu.cpp and adds emu_voxels (find_voxel, the routine of k_voxels) and emu_dense: k_dense's tiles
// in order, each walked once by dense_tile_walk and its voxels resolved by dense_voxel, clipped to the box and written at the
// kernel's offsets.  Both routines are the kernels' own __host__ __device__ code in tsdf_core.cuh.
#include "emu.cpp"

extern "C" {

void emu_voxels (Emu* e, const float* xyz, long long n, float min_size, VoxelRec* out)
{
  for (long long i = 0; i < n; ++i) out[i] = find_voxel (e->p, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], min_size);
}

// box = {i0, j0, k0, i1, j1, k1}; any output may be null
void emu_dense (Emu* e, const int32_t* box, float* d, float* w, uint8_t* rgb, int8_t* level)
{
  const Params& p = e->p;
  const size_t nj = (size_t) (box[4] - box[1]), nk = (size_t) (box[5] - box[2]);
  DenseTile t;
  for (int tx = box[0] >> 3; tx <= (box[3] - 1) >> 3; ++tx)
    for (int ty = box[1] >> 3; ty <= (box[4] - 1) >> 3; ++ty)
      for (int tz = box[2] >> 3; tz <= (box[5] - 1) >> 3; ++tz)
      {
        dense_tile_walk (p, tx, ty, tz, t);
        for (int v = 0; v < 512; ++v)
        {
          const int X = 8 * tx + (v >> 6), Y = 8 * ty + ((v >> 3) & 7), Z = 8 * tz + (v & 7);
          if (X < box[0] || X >= box[3] || Y < box[1] || Y >= box[4] || Z < box[2] || Z >= box[5]) continue;
          float2 dw; uchar4 c; int lv;
          dense_voxel (p, t, X, Y, Z, dw, c, lv);
          const size_t o = ((size_t) (X - box[0]) * nj + (size_t) (Y - box[1])) * nk + (size_t) (Z - box[2]);
          if (d) d[o] = dw.x;
          if (w) w[o] = dw.y;
          if (rgb) { rgb[3 * o] = c.x; rgb[3 * o + 1] = c.y; rgb[3 * o + 2] = c.z; }
          if (level) level[o] = (int8_t) lv;
        }
      }
}

} // extern "C"
