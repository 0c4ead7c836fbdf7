// Marching-cubes surface meshes of one row of a label mask (lm_mesh_counts_dev, lm_mesh_emit_dev; see mesh.cu, DESIGN §4.14).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace lm {

constexpr int kMeshConfigs = 256;
constexpr int kMeshMaxTriangles = 16;   // per configuration (the generated table has at most 5)

// The triangle table as the caller passes it (host memory): configuration c owns triangles [off[c], off[c + 1]), each
// three codes (corner a << 2) | axis m naming the cube edge from corner a to corner a + e_m.
struct MeshTable {
  const int32_t* off;     // [257]
  const uint8_t* codes;   // [off[256]][3]
};

// Placement of the doubled coordinates u: x = u2 / 2, y = u1 / 2, z = u0 / 2 and
// p_c = ((o_c + D[c][0] (s_x x)) + D[c][1] (s_y y)) + D[c][2] (s_z z), every product and sum rounded on its own; `ras`
// negates p_0 and p_1; `reverse` swaps the last two vertices of every triangle.
struct MeshPlacement {
  double o[3], d[9], s[3];
  int ras, reverse;
};

// Device work buffers of the mesh calls, grown on demand and reused across calls.
struct MeshWork {
  void* d = nullptr;   // the table, the per-line vertex and triangle counts (scanned in place) and the block totals
  size_t bytes = 0;
  int reserve(size_t need);
  void release();
};

// V and T of `row` (1..255: mask == row, 256: mask != 0) of the (n0,n1,n2) uint8 mask padded with one voxel of outside.
// Synchronises `st`.
int mesh_counts(MeshWork& w, const uint8_t* d_mask, int n0, int n1, int n2, int row, const MeshTable& tab, int64_t* n_vertices,
                int64_t* n_triangles, int num_sms, cudaStream_t st, int64_t* launches);

// Recounts the row and writes its V vertices (d_index2 (V,3) int32, d_vertices (V,3) float64) and T triangles
// (d_triangles (T,3) int32).  Returns -2 when the recount differs from n_vertices / n_triangles.  Synchronises `st`.
int mesh_emit(MeshWork& w, const uint8_t* d_mask, int n0, int n1, int n2, int row, const MeshTable& tab,
              const MeshPlacement& place, int64_t n_vertices, int64_t n_triangles, int32_t* d_index2, double* d_vertices,
              int32_t* d_triangles, int num_sms, cudaStream_t st, int64_t* launches);

}  // namespace lm
