// vr_kernels.h -- host-side launch interface of the march kernels (one TU per basis size).
#pragma once
#include <cuda_runtime.h>

#include "vr_types.h"

namespace vrb {

// Kernel variants (vr_set_variant); 0 = the default for the launch and the tree's basis size.
//   kVariantQueue:  persistent warps + warp-shared shading queue (vr_march_q.cuh), >= 4 basis functions
//   kVariantInline: persistent warps, inline shading (vr_march.cuh); its id, 3 + 16 * 193, stays what callers set
constexpr int kVariantQueue = 7, kVariantInline = 3 + 16 * 193;

// The kernel bases the march kernels are built for (vr_kernels_inst.cu, one object per entry of the Makefile's KBDS).
constexpr bool kbd_built(int kbd) { return kbd == -1 || kbd == 1 || kbd == 4 || kbd == 9 || kbd == 16 || kbd == 25; }

enum class MarchKernel { kNotBuilt, kInline, kQueue };

// The kernel that a launch of n_views views on a tree of kernel basis kbd runs under vr_set_variant(variant).
// Default (DESIGN.md 4): the queue pays ~30 instructions per march iteration (ballots, ring bookkeeping) for a 3x
// denser colour block: a loss in batches, where other warps hide the inline block's latency, a win on single frames,
// where the long-ray tail of the frame is what is waited for.  With 25 basis functions its per-ray basis values
// (112 B) push the CTA's shared memory over the 8-CTA budget.  Both kernels produce identical bits.
inline MarchKernel march_kernel(int kbd, int variant, int n_views) {
    if (!kbd_built(kbd)) return MarchKernel::kNotBuilt;
    if (variant == 0) return n_views == 1 && kbd >= 4 && kbd <= 16 ? MarchKernel::kQueue : MarchKernel::kInline;
    if (variant == kVariantInline) return MarchKernel::kInline;
    if (variant == kVariantQueue && kbd >= 4) return MarchKernel::kQueue;
    return MarchKernel::kNotBuilt;
}

struct LaunchCfg {
    bool queue;      // the shading-queue kernel, else the inline-shading one (march_kernel)
    bool count;      // instrumented build: accumulate vr_counters
    bool surface;    // write a cudaSurfaceObject instead of linear memory
    int num_sms;
    unsigned int* work_counter;  // persistent kernels: {work head, done CTAs}
    cudaStream_t stream;
};

template <int KBD>
cudaError_t launch_march(LaunchDev& P, const LaunchCfg& cfg);

// The weights pass of vr_tree_leaf_weights: the inline-shading kernel's kOutWeights instantiation (vr_march.cuh).  It
// reads no colour record, so one kernel serves every basis size; it is built in the VR_KBD=1 object.
cudaError_t launch_weights(LaunchDev& P, const LaunchCfg& cfg);

extern template cudaError_t launch_march<-1>(LaunchDev&, const LaunchCfg&);
extern template cudaError_t launch_march<1>(LaunchDev&, const LaunchCfg&);
extern template cudaError_t launch_march<4>(LaunchDev&, const LaunchCfg&);
extern template cudaError_t launch_march<9>(LaunchDev&, const LaunchCfg&);
extern template cudaError_t launch_march<16>(LaunchDev&, const LaunchCfg&);
extern template cudaError_t launch_march<25>(LaunchDev&, const LaunchCfg&);

}  // namespace vrb
