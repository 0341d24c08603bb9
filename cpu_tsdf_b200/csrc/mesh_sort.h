// mesh_sort.h — internal: sort fixed-size records by 64-bit order keys (meshpost.cu, cub::DeviceRadixSort).
#pragma once
#include <cuda_runtime.h>
#include <cstddef>

// d_keys (n, destroyed), d_v (`words` 32-bit words per record, moved as raw bits), d_c (`words` bytes per record or null)
// -> d_v_out / d_c_out in ascending key order.  key_bits = number of significant low bits of the keys.  Used with 9 words
// (a triangle's three vertices, with its nine colour bytes) by b200tsdf_mesh and with 3 words (a leaf's centre or voxel
// index) by the leaf enumeration.  Returns 0 or a cudaError_t.
int b2_sort_records (cudaStream_t s, size_t n, int key_bits, unsigned long long* d_keys, int words, const void* d_v, const unsigned char* d_c,
                     void* d_v_out, unsigned char* d_c_out);
