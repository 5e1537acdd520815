// vr_probe.h -- lumisphere probe: the leaf lookup shared by vr_probe_lumisphere and the overlay of vr_draw_probe.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "vr_types.h"

namespace vrb {

// retrieve_cursor_lumisphere_kernel (volrend.cu:175-191): table entry of the leaf that holds world point (x, y, z),
// clamped into the box as in n3tree_query.hpp:17-19.  The leaf's colour record is tree.wrecs + entry * rec_bytes.
__device__ __forceinline__ uint32_t probe_leaf_entry(const TreeDev& tree, float x, float y, float z) {
    float p[3] = {tree.offset[0] + tree.scale[0] * x, tree.offset[1] + tree.scale[1] * y,
                  tree.offset[2] + tree.scale[2] * z};
    uint32_t u[3];
    for (int i = 0; i < 3; ++i) {
        p[i] = fmaxf(fminf(p[i], 1.f - 1e-6f), 0.f);
        u[i] = __float2uint_rz(p[i] * tree.pos_scale);
    }
    uint32_t T = 0, eidx = 0;
    constexpr uint32_t M = (1u << kWideLv) - 1u;
    for (int j = 0; j < 16; ++j) {
        const int sh = (24 - kWideLv) - kWideLv * j;
        eidx = T * (uint32_t)kWideEntries + ((((u[0] >> sh) & M) << (2 * kWideLv)) | (((u[1] >> sh) & M) << kWideLv) | ((u[2] >> sh) & M));
        const uint32_t w = tree.wide[eidx];
        if (w & kLeafBit) break;
        T = w;
    }
    return eidx;
}

// One overlay launch: the probe disc of every view, over the pixels [cx0, cx0+cw) x [cy0, cy0+ch) of the frame (the
// candidate corner of volrend.cu:100-101 clipped to the frame and to the tile [x0, x0+w) x [y0, y0+h)).
struct ProbeLaunch {
    TreeDev tree;
    float probe[3];          // world coordinates
    int32_t disp;            // probe_disp_size (> 0)
    int32_t bmin, bmax;      // basis_minmax clamped to the tree's basis
    CamDev cam;              // used when cams == nullptr
    const CamDev* cams;      // device array of n_views cameras
    int32_t n_views;
    int32_t x0, y0, w, h;    // tile of the output buffers
    int32_t cx0, cy0, cw, ch;
    uint8_t* rgba8;          // tile-sized RGBA8 per view, or nullptr
    float4* rgbaf;           // tile-sized float4 per view, or nullptr
    cudaSurfaceObject_t surf;  // full-frame RGBA8 surface (one view, no tile), or 0
};

// Launches the overlay kernel for kernel basis `kbd` on `stream` (a normal launch: no programmatic dependent launch).
cudaError_t probe_draw(const ProbeLaunch& P, int kbd, cudaStream_t stream);

}  // namespace vrb
