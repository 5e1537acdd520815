// vr_iso.h -- internal interface between the C-ABI (vr_api.cu: vr_tree_isosurface) and the marching-cubes kernels
// that extract a surface mesh from a device tree (vr_iso.cu).  See DESIGN.md section 23.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "vr_types.h"

namespace vrb {

constexpr int kIsoMaxDepth = 11;   // lattice levels 1 .. 11: (2^11 + 2)^3 points, 24-bit positions

struct IsoArgs {
    TreeDev tree;
    int depth;            // lattice level L: R = 2^L cells per axis
    float level;          // inside: sigma > level
    float* vert;          // fill: [n_verts][9] (position, colour, normal)
    uint32_t* faces;      // fill: [n_faces][3]
    bool color;           // fill: the colour slots receive the inside endpoint's lattice index (iso_color reads it)
    int slab_planes;      // x-planes per slab (>= 2), or 0: as many as fit the scratch budget
};

// Counts (fill == false) or writes (fill == true) the mesh slab by slab on `stream`.  Counting synchronises the stream
// once, to read the totals into *n_verts / *n_faces; filling is stream-ordered and writes vertex positions, colours
// (white, or the inside endpoints for iso_color) and zero normals, and the faces.  Scratch comes from the device's
// default stream-ordered pool.  *launches counts the kernels and CUB calls.
cudaError_t iso_run(const IsoArgs& a, bool fill, cudaStream_t stream, long long* n_verts, long long* n_faces,
                    int* launches);

// The colour pass, after the normals: each vertex's colour becomes the colour of its inside endpoint's leaf seen
// along -normal, with basis_minmax [bmin, bmax] (vr_tree_eval's).  Stream-ordered.
cudaError_t iso_color(const TreeDev& tree, int depth, float* vert, long long n_verts, int32_t bmin, int32_t bmax,
                      cudaStream_t stream, int* launches);

}  // namespace vrb
