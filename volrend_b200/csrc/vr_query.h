// vr_query.h -- point queries of a device tree: vr_tree_query, vr_tree_eval and vr_probe_lumisphere (vr_query.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "vr_types.h"

namespace vrb {

struct QueryLaunch {
    TreeDev tree;
    const float* xyz;    // device [n][3] world points, or nullptr: the single point `point`
    float point[3];
    const float* dir;    // eval: device [n][3] directions
    long long n;
    // query outputs (any may be null)
    uint16_t* data;      // [n][3 * max(kbd, 1) + 1] fp16 rows: colour coefficients, sigma last
    float* cube;         // [n]
    float* local;        // [n][3]
    float* coef;         // [n][n_coef]: the first n_coef colour coefficients as floats (vr_probe_lumisphere)
    int32_t n_coef;
    // eval outputs (any may be null)
    float* rgb;          // [n][3]
    float* sigma;        // [n]
    int32_t bmin, bmax;  // basis_minmax clamped to the tree's basis
};

// One launch of the query kernel (eval = false) or the eval kernel for kernel basis `kbd` on `stream`.
cudaError_t query_launch(const QueryLaunch& Q, int kbd, bool eval, int num_sms, cudaStream_t stream);

}  // namespace vrb
