// vr_wire.h -- internal interface between the C-ABI (vr_api.cu: vr_tree_wireframe) and the grid-wireframe
// kernels (vr_wire.cu).  See DESIGN.md section 9.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vrb {

// Cell levels are 1 (the root's 8 cells) .. 24 (the finest the 24-bit position grid holds).
constexpr int kWireLevels = 26;

// The octree as the wireframe kernels read it: the wide tables of the march kernels.
struct WireTree {
    const uint32_t* wide;
    long long n_tables;
    int wide_p;        // TreeDev::wide_p
    int max_level;     // deepest leaf level (TreeDev::max_depth)
    float offset[3], scale[3];
};

// Cells of the whole octree by level: leaf[l] leaves and inner[l] internal cells (= nodes of depth l) at level l.
struct WireLevels {
    long long leaf[kWireLevels], inner[kWireLevels];
};

// Fills `out` by walking every table once.  Synchronises `stream`; *launches counts the kernels it ran.
cudaError_t wire_levels(const WireTree& t, WireLevels& out, cudaStream_t stream, int* launches);

// Number of cells N3Tree::gen_wireframe(max_depth) emits: the leaves down to level max(max_depth, 0) + 1 and
// every internal cell of that level.
long long wire_cells(const WireTree& t, const WireLevels& lv, int max_depth);

// Writes the wireframe of the cut at max_depth (wire_cells(...) * 24 vertices of 9 floats) to `out`, stream-ordered;
// scratch memory comes from the stream-ordered allocator.  *launches counts the kernels it ran.
cudaError_t wire_fill(const WireTree& t, const WireLevels& lv, int max_depth, float* out, cudaStream_t stream,
                      int* launches);

}  // namespace vrb
