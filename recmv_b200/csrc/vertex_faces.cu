// Vertex-face incidence of a triangle mesh (DESIGN section 1o): the flattened (face, vertex) pair lists that the remesh
// step builds from openmesh's `vertex_face_indices()` (OptimGarmentNetwork.py:715-735), without the host copy.
//
// faces [F,3] int64 -> fid [3F], vid [3F] int64: one pair per face corner, grouped by vertex in ascending order and,
// within a vertex, in ascending face index (ascending corner for a face that names the vertex twice).  The lengths
// are 3F whatever the mesh, so the caller allocates them without reading anything back.
//   1. corner_keys_kernel  one thread per corner e = 3 f + k: key = its vertex (V for a face with an index outside
//                          [0, V)), value e; such a face sets the flag (segments.cuh);
//   2. CUB radix sort      stable, so each vertex's corners stay in increasing e order;
//   3. vf_write_kernel     one thread per sorted position: (e / 3, key), or (-1, -1) for the corners keyed V, which
//                          sort last.
// The sort is the one the vertex normals use; the order depends on the keys alone, not on the launch shape, so two
// runs are bit-identical.
#include "common.cuh"
#include "segments.cuh"

namespace recmv {
namespace {

struct VertexFacesWs {
  unsigned *keys_in, *keys_out, *vals_in, *vals_out;
  void* temp;   // CUB's temporary storage, last: the size query adds sort_temp_bytes to the bytes taken
};

VertexFacesWs vertex_faces_layout(Carve& c, long long M) {
  VertexFacesWs w;
  w.keys_in = c.take<unsigned>(M);
  w.keys_out = c.take<unsigned>(M);
  w.vals_in = c.take<unsigned>(M);
  w.vals_out = c.take<unsigned>(M);
  w.temp = c.take<char>(0, 1);
  return w;
}

__global__ void __launch_bounds__(kSegThreads) vf_write_kernel(const unsigned* __restrict__ keys,
                                                                const unsigned* __restrict__ vals, long long M,
                                                                unsigned V, long long* __restrict__ fid,
                                                                long long* __restrict__ vid) {
  const long long i = blockIdx.x * (long long)kSegThreads + threadIdx.x;
  if (i >= M) return;
  const unsigned k = keys[i];
  const bool ok = k < V;
  fid[i] = ok ? (long long)(vals[i] / 3u) : -1;
  vid[i] = ok ? (long long)k : -1;
}

int vertex_faces_shape(int64_t F, int V) {
  if (V < 0 || F < 0) return RECMV_E_SHAPE;
  if (3 * F > 0x7fffffffLL || V == 0x7fffffff) return RECMV_E_RANGE;   // int sort positions; V is the sentinel key
  return RECMV_OK;
}

}  // namespace
}  // namespace recmv

using namespace recmv;

extern "C" int recmv_vertex_faces_workspace_bytes(int64_t F, int V, size_t* bytes) {
  if (!bytes) return RECMV_E_NULL;
  int s = vertex_faces_shape(F, V);
  if (s) return s;
  const long long M = 3 * (long long)F;
  size_t temp = 0;
  s = sort_temp_bytes(M, (unsigned)V, &temp);
  if (s) return s;
  *bytes = layout_bytes(vertex_faces_layout, M) + temp;
  return RECMV_OK;
}

extern "C" int recmv_vertex_faces(const int64_t* faces, int64_t F, int V, void* workspace, int64_t* fid, int64_t* vid,
                                  int32_t* flags, recmv_stream_t stream) {
  int s = vertex_faces_shape(F, V);
  if (s) return s;
  if (!flags) return RECMV_E_NULL;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e = cudaMemsetAsync(flags, 0, sizeof(int32_t), st);   // the flag describes this call's faces
  if (e != cudaSuccess) return (int)e;
  if (F == 0) return RECMV_OK;
  if (!faces || !workspace || !fid || !vid) return RECMV_E_NULL;
  const long long M = 3 * (long long)F;
  const VertexFacesWs w = carve(workspace, vertex_faces_layout, M);
  const unsigned nb = (unsigned)((M + kSegThreads - 1) / kSegThreads);
  corner_keys_kernel<<<nb, kSegThreads, 0, st>>>((const long long*)faces, M, V, w.keys_in, w.vals_in, flags);
  s = launch_status();
  if (s) return s;
  s = sort_pairs(w.temp, w.keys_in, w.keys_out, w.vals_in, w.vals_out, M, (unsigned)V, st);
  if (s) return s;
  vf_write_kernel<<<nb, kSegThreads, 0, st>>>(w.keys_out, w.vals_out, M, (unsigned)V, (long long*)fid,
                                              (long long*)vid);
  return launch_status();
}
