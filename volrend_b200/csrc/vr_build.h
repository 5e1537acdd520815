// vr_build.h -- internal interface between the C-ABI (vr_api.cu: vr_tree_build) and the kernels that build an N3Tree
// from voxel cells (vr_build.cu).  See DESIGN.md section 21.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vrb {

constexpr int kBuildMaxLevel = 23;   // kMaxTreeDepth: the deepest leaf vr_tree_create accepts

struct BuildArgs {
    const int32_t* cells;     // [n][4]: level, i, j, k
    const uint16_t* rows;     // fp16 [n][data_dim]
    long long n;              // <= INT32_MAX
    int data_dim;
    bool merge;
    int32_t* child;           // [max_nodes * 8] or nullptr: count only
    uint16_t* data;           // [max_nodes * 8 * data_dim] or nullptr
    long long max_nodes;
    long long node_limit;     // larger results are refused (kBuildTooLarge)
};

// Inputs tree_build refuses after looking at them (*reject); nothing is written then.
enum { kBuildOk = 0, kBuildBadCell = 1, kBuildOverlap = 2, kBuildTooLarge = 3, kBuildCapacity = 4 };

// Builds the canonical tree of the cells.  Synchronises `stream` once, when the node count is known (it sizes the
// node scratch and decides the capacity refusal); everything else is stream-ordered, with scratch from the device's
// default stream-ordered pool.  *n_nodes is the node count whenever the cells are valid; the outputs are written only
// when they are non-null, *reject is kBuildOk and the count fits max_nodes.  *launches counts the kernels and CUB calls.
cudaError_t tree_build(const BuildArgs& a, cudaStream_t stream, long long* n_nodes, int* reject, int* launches);

}  // namespace vrb
