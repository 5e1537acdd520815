// vr_tv.h -- internal interface between the C-ABI (vr_api.cu: vr_tree_leaf_neighbors, vr_tree_leaf_tv) and the
// total-variation kernels (vr_tv.cu).  See DESIGN.md section 20.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "vr_types.h"
#include "vr_wire.h"

namespace vrb {

// The columns of a data row the TV prior acts on: the ones vr_tree_leaf_grads writes.  Colour: channel c's
// coefficient k < n_coef at column c * coef_stride + k (RGBA: n_coef 1, stride 1); sigma: the last column.
struct TvColumns {
    int32_t data_dim, n_coef, coef_stride;
};

// Writes the forward neighbour of every reachable leaf slot along x, y and z (nbr[slot * 3 + axis]) and -1 everywhere
// else, for n_slots slots.  w / lv: the tree's wide tables and cell counts (wire_levels); wslot: its slot map.
// Stream-ordered; *launches counts the kernels it ran.
cudaError_t tv_neighbors(const WireTree& w, const WireLevels& lv, const TreeDev& tree, const uint32_t* wslot,
                         long long n_slots, int32_t* nbr, cudaStream_t stream, int* launches);

// Adds the gradient of the TV energy of `data` (n_slots rows of cols.data_dim floats) to `grad` and, when `energy` is
// not null, the energy to *energy.  scale_sigma / scale_color: lambda / N_leaf of each group (0: the group is skipped).
// Stream-ordered; the sums are atomic, so their last bits depend on the order the atomics land in.
cudaError_t tv_pass(const float* data, const int32_t* nbr, long long n_slots, TvColumns cols, double scale_sigma,
                    double scale_color, float* grad, double* energy, cudaStream_t stream, int* launches);

}  // namespace vrb
