// vr_raster.h -- internal interface between the C-ABI (vr_api.cu: vr_draw_meshes, vr_draw_meshes_batch) and the
// mesh rasterizer kernels (vr_raster.cu).  See DESIGN.md sections 8 and 15.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vrb {

// One mesh as the kernels see it: the model-view matrix is folded on the host (in double).
struct RasterMesh {
    const float* vert;      // n_verts * 9 floats: position, colour, normal (mesh.cpp:26)
    const uint32_t* faces;  // n_prims * face_size indices, or nullptr = consecutive vertices
    int n_verts, face_size, unlit;
    int view;               // index of the mesh's view in the launch's frame array
    float mv[12];           // camera-from-model of that view, 3x4 column-major (w2c * model)
    float m3[9];            // model 3x3, column-major (normal transform: mat3x3(M), mesh.cpp:118)
    long long base;         // launch-wide index of this mesh's first primitive (view-major, draw order)
    long long n_prims;
};

// One view of a launch.  Every view of a launch has the same W and H.
struct RasterFrame {
    int W, H;
    float fx, fy, cx, cy;
    float cam_pos[3];       // the shader's camPos = -transpose(mat3(w2c)) * w2c[3] (mesh.cpp:376)
    long long large_off;    // this view's region of the large-primitive list (entries)
    uint8_t* rgba8;         // W * H * 4 bytes
    float* depth;           // W * H floats
};

// Largest frame side the rasterizer accepts (bounding boxes are packed as 16-bit coordinates).
constexpr int kRasterMaxSide = 32768;
// Largest number of primitives per launch: draw sequence numbers are 1 + 8 * primitive + sub-triangle in 32 bits.
constexpr long long kRasterMaxPrims = 1LL << 29;
// Largest number of views per launch (the views are a grid dimension of z_init, raster_big and resolve).
constexpr int kRasterMaxViews = 65535;
// Scratch of one launch (z-buffers, 8 B per pixel, and large-primitive lists, 16 B per entry) stays at or under this
// bound; a batch is split into launches to keep it so.  Only a single view that needs more by itself exceeds it.
constexpr size_t kRasterScratchBytes = 256u << 20;

// Scratch bytes of one view: its z-buffer and its region of the large-primitive list.
inline size_t raster_view_bytes(long long npx, long long large_cap) { return (size_t)(npx * 8 + large_cap * 16); }

// Draws the `n` meshes (host array, view-major, base/n_prims/view filled, n_prims > 0) of `n_views` views (host
// array of frames with large_off filled) in one launch of each kernel; returns the first CUDA error.  A view's
// large_cap = upper bound of its clipped sub-primitives (6 per triangle, 1 per line/point); `large_total` is their
// sum.
cudaError_t raster_draw(const RasterFrame* frames, int n_views, const RasterMesh* meshes, int n, long long total_prims,
                        long long large_total, cudaStream_t stream);
constexpr int kRasterLaunches = 4;

// The rasterizer's stream-ordered scratch pool of the current device (it keeps what it has reserved); the normal
// estimation (vr_normals.cu) allocates from it too.
cudaError_t scratch_pool(cudaMemPool_t* out);

}  // namespace vrb
