// vr_kernels.h -- host-side launch interface of the march kernels (one TU per basis size).
#pragma once
#include <cuda_runtime.h>

#include "vr_types.h"

namespace vrb {

// Kernel variants (vr_set_variant); 0 = the default for the launch and the tree's basis size.
//   kVariantQueue:  persistent warps + warp-shared shading queue (vr_march_q.cuh), >= 4 basis functions
//   kVariantInline: persistent warps, inline shading (vr_march.cuh); its id, 3 + 16 * 193, stays what callers set
constexpr int kVariantQueue = 7, kVariantInline = 3 + 16 * 193;

struct LaunchCfg {
    int variant;
    int max_ctas;    // > 0: cap the persistent grid (leaves SMs to a concurrent copy/collective kernel)
    bool count;      // instrumented build: accumulate vr_counters
    bool surface;    // write a cudaSurfaceObject instead of linear memory
    int num_sms;
    unsigned int* queue;  // persistent kernels: {work head, done CTAs}
    cudaStream_t stream;
};

template <int KBD>
cudaError_t launch_march(LaunchDev& P, const LaunchCfg& cfg);

template <int KBD>
bool variant_supported(int variant);

// The weights pass of vr_tree_leaf_weights: the inline-shading kernel's kOutWeights instantiation (vr_march.cuh).  It
// reads no colour record, so one kernel serves every basis size; it is built in the VR_KBD=1 object.
cudaError_t launch_weights(LaunchDev& P, const LaunchCfg& cfg);

extern template cudaError_t launch_march<-1>(LaunchDev&, const LaunchCfg&);
extern template cudaError_t launch_march<1>(LaunchDev&, const LaunchCfg&);
extern template cudaError_t launch_march<4>(LaunchDev&, const LaunchCfg&);
extern template cudaError_t launch_march<9>(LaunchDev&, const LaunchCfg&);
extern template cudaError_t launch_march<16>(LaunchDev&, const LaunchCfg&);
extern template cudaError_t launch_march<25>(LaunchDev&, const LaunchCfg&);
extern template bool variant_supported<-1>(int);
extern template bool variant_supported<1>(int);
extern template bool variant_supported<4>(int);
extern template bool variant_supported<9>(int);
extern template bool variant_supported<16>(int);
extern template bool variant_supported<25>(int);

}  // namespace vrb
