// mesh_sort.h — internal: the mesh back end of meshpost.cu, shared by the host entry points there and the device entry points
// of engine.cu: record sorting (cub::DeviceRadixSort) and the flattenVertices / cleanupMesh routines.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>
#include <string>
#include <vector>

// d_keys (n, destroyed), d_v (`words` 32-bit words per record, moved as raw bits), d_c (`words` bytes per record or null)
// -> d_v_out / d_c_out in ascending key order.  key_bits = number of significant low bits of the keys.  Used with 9 words
// (a triangle's three vertices, with its nine colour bytes) by b200tsdf_mesh and with 3 words (a leaf's centre or voxel
// index) by the leaf enumeration.  Returns 0 or a cudaError_t.
int b2_sort_records (cudaStream_t s, size_t n, int key_bits, unsigned long long* d_keys, int words, const void* d_v, const unsigned char* d_c,
                     void* d_v_out, unsigned char* d_c_out);

// d_out[i] = d_in[0] + ... + d_in[i] (n < 2^31), used by the .vol parser (engine.cu).  Returns 0 or a cudaError_t with the
// stream synchronised.
int b2_inclusive_sum (cudaStream_t s, const long long* d_in, long long* d_out, size_t n);

// Device scratch of one post-processing call: every allocation is released with the object.  The routines below end with
// their stream synchronised, so nothing still reads it then.
struct B2MeshScratch
{
  std::vector<void*> all;
  B2MeshScratch () = default;
  B2MeshScratch (const B2MeshScratch&) = delete;
  B2MeshScratch& operator= (const B2MeshScratch&) = delete;
  ~B2MeshScratch () { for (void* p : all) cudaFree (p); }
  template <typename T> T* get (size_t n)          // null when the allocation fails
  {
    void* p = nullptr;
    if (cudaMalloc (&p, (n ? n : 1) * sizeof (T)) != cudaSuccess) { cudaGetLastError (); return nullptr; }
    all.push_back (p);
    return (T*) p;
  }
};

// flattenVertices / cleanupMesh (src/prog/integrate.cpp:103-214) on device arrays, on stream s.  d_tris == null: a triangle
// soup, triangle t = {3t, 3t+1, 3t+2} (nverts == 3 * ntris).  The caller checks the sizes (nverts < 2^31, 3 * ntris < 2^31,
// min_neighbors in 1..16) and that outputs and inputs do not overlap; the routines check the indices on the device first and
// return B200TSDF_EINVAL, with no output byte written, when one is out of range.  Outputs: d_out_verts (3 * nverts floats)
// and d_out_tris (3 * ntris int32) receive *out_nverts / *out_ntris entries, no byte past them is written, and the inputs are
// only read.  Returns 0 with the outputs written and the stream synchronised, or a B200TSDF_E* code with a message in err.
int b2_mesh_flatten (cudaStream_t s, B2MeshScratch& scratch, const float* d_verts, size_t nverts, const int32_t* d_tris, size_t ntris,
                     float min_dist, float* d_out_verts, int32_t* d_out_tris, size_t* out_nverts, size_t* out_ntris, std::string& err);
int b2_mesh_cleanup (cudaStream_t s, B2MeshScratch& scratch, const float* d_verts, size_t nverts, const int32_t* d_tris, size_t ntris,
                     float face_dist, int min_neighbors, float* d_out_verts, int32_t* d_out_tris, size_t* out_nverts, size_t* out_ntris,
                     std::string& err);
