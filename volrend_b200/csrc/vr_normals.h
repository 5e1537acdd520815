// vr_normals.h -- internal interface between the C-ABI (vr_api.cu: vr_mesh_estimate_normals) and the
// vertex-normal kernels (vr_normals.cu).  See DESIGN.md section 11.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vrb {

// estimate_normals (reference src/mesh.cpp:63-97) on a device vertex buffer: overwrites floats 6..8 of each of the
// n_verts 9-float vertices.  faces == nullptr: n_verts / 3 consecutive triangles; otherwise n_faces triangles of
// `faces` (faces with an index >= n_verts contribute nothing).  Stream-ordered; scratch comes from the rasterizer's
// pool.  Requires n_verts <= INT_MAX and 3 * n_faces <= INT_MAX.  *launches counts the kernels it ran.
cudaError_t normals_estimate(float* vert, long long n_verts, const uint32_t* faces, long long n_faces,
                             cudaStream_t stream, int* launches);

}  // namespace vrb
