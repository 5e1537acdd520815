// vr_raster.h -- internal interface between the C-ABI (vr_api.cu: vr_draw_meshes) and the mesh
// rasterizer kernels (vr_raster.cu).  See DESIGN.md section 8.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vrb {

// One mesh as the kernels see it: the model-view matrix is folded on the host (in double).
struct RasterMesh {
    const float* vert;      // n_verts * 9 floats: position, colour, normal (mesh.cpp:26)
    const uint32_t* faces;  // n_prims * face_size indices, or nullptr = consecutive vertices
    int n_verts, face_size, unlit, pad_;
    float mv[12];           // camera-from-model, 3x4 column-major (w2c * model)
    float m3[9];            // model 3x3, column-major (normal transform: mat3x3(M), mesh.cpp:118)
    long long base;         // global index of this mesh's first primitive (draw order)
    long long n_prims;
};

struct RasterFrame {
    int W, H;
    float fx, fy, cx, cy;
    float cam_pos[3];       // world camera position (the shader's camPos, mesh.cpp:376)
};

// Largest frame side the rasterizer accepts (bounding boxes are packed as 16-bit coordinates).
constexpr int kRasterMaxSide = 32768;
// Largest number of primitives per call: draw sequence numbers are 1 + 8 * primitive + sub-triangle in 32 bits.
constexpr long long kRasterMaxPrims = 1LL << 29;

// Draws `n` meshes (host array, base/n_prims filled, n_prims > 0) over rgba8/depth; returns the first
// CUDA error.  `large_cap` = upper bound of the clipped sub-primitives (6 per triangle, 1 per line/point).
cudaError_t raster_draw(const RasterFrame& f, const RasterMesh* meshes, int n, long long total_prims,
                        long long large_cap, uint8_t* rgba8, float* depth, cudaStream_t stream);
constexpr int kRasterLaunches = 4;

// The rasterizer's stream-ordered scratch pool of the current device (it keeps what it has reserved); the normal
// estimation (vr_normals.cu) allocates from it too.
cudaError_t scratch_pool(cudaMemPool_t* out);

}  // namespace vrb
