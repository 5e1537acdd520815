// vr_quant.h -- internal interface between the C-ABI (vr_api.cu: vr_tree_compress) and the median-cut colour
// quantisation kernels (vr_quant.cu).  See DESIGN.md section 12.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vrb {

struct QuantArgs {
    const uint16_t* data;        // fp16 [n_child][data_dim], channel-major coefficients, sigma last
    long long n_child;
    int data_dim, n_retain, bits;
    float thresh;                // fp16_rn(sigma_thresh), as a float: a slot is kept iff sigma > thresh
    uint16_t* colors;            // fp16 [n_quant][65536][3]
    uint16_t* qmap;              // u16  [n_quant][n_child]
    uint16_t* sigma;             // fp16 [n_child]
    uint16_t* retained;          // fp16 [n_retain][n_child][3] or nullptr when n_retain == 0
};

// Inputs quant_compress refuses after looking at the data (*reject)
enum { kQuantOk = 0, kQuantNonFinite = 1, kQuantTooManyPoints = 2 };

// Median-cut compression of one tree.  Synchronises `stream` once, after the kept count is known (it sizes the
// scratch); everything after that is stream-ordered.  Nothing is written, and *reject says why, when a quantised
// coefficient of a kept slot is Inf or NaN (kQuantNonFinite) or n_quant * kept > INT32_MAX (kQuantTooManyPoints).
// Requires n_child <= INT32_MAX.  *launches counts the kernels (and CUB calls) it ran.
cudaError_t quant_compress(const QuantArgs& a, cudaStream_t stream, long long* n_kept, int* reject, int* launches);

}  // namespace vrb
