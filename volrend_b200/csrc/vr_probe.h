// vr_probe.h -- lumisphere probe: the leaf lookup shared by vr_probe_lumisphere and the overlay of vr_draw_probe.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "vr_types.h"

namespace vrb {

// Tree-space position p of world point (x, y, z) (offset + scale * xyz, volrend.cu:180-182), clamped into the box as
// in n3tree_query.hpp:17-19 (a NaN coordinate clamps to 1 - 1e-6), and its cell coordinates u on the tables' grid.
__device__ __forceinline__ void probe_position(const TreeDev& tree, float x, float y, float z, float (&p)[3],
                                               uint32_t (&u)[3]) {
    p[0] = tree.offset[0] + tree.scale[0] * x;
    p[1] = tree.offset[1] + tree.scale[1] * y;
    p[2] = tree.offset[2] + tree.scale[2] * z;
    for (int i = 0; i < 3; ++i) {
        p[i] = fmaxf(fminf(p[i], 1.f - 1e-6f), 0.f);
        u[i] = __float2uint_rz(p[i] * tree.pos_scale);
    }
}

// query_single_from_root (n3tree_query.hpp:13-48) on the wide tables: descends from table T at step j (j = 0, T = 0:
// the root) to the entry of the leaf holding u and returns it; w receives the leaf word and j the leaf's step.
// The table visited at step k is stored at tab[k * tab_stride] when tab is not null (the restart point of a later
// descent).  The leaf's colour record is tree.wrecs + entry * rec_bytes.
__device__ __forceinline__ uint32_t descend_wide(const TreeDev& tree, const uint32_t (&u)[3], int& j, uint32_t T,
                                                 uint32_t& w, uint32_t* tab, int tab_stride) {
    uint32_t eidx = 0;
    constexpr uint32_t M = (1u << kWideLv) - 1u;
    for (; j < 16; ++j) {
        if (tab) tab[j * tab_stride] = T;
        const int sh = (24 - kWideLv) - kWideLv * j;
        eidx = T * (uint32_t)kWideEntries + ((((u[0] >> sh) & M) << (2 * kWideLv)) | (((u[1] >> sh) & M) << kWideLv) | ((u[2] >> sh) & M));
        w = tree.wide[eidx];
        if (w & kLeafBit) break;
        T = w;
    }
    return eidx;
}

// retrieve_cursor_lumisphere_kernel (volrend.cu:175-191): table entry of the leaf that holds world point (x, y, z).
__device__ __forceinline__ uint32_t probe_leaf_entry(const TreeDev& tree, float x, float y, float z) {
    float p[3];
    uint32_t u[3], w;
    probe_position(tree, x, y, z, p, u);
    int j = 0;
    return descend_wide(tree, u, j, 0u, w, nullptr, 0);
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
