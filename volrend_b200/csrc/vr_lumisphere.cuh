// vr_lumisphere.cuh -- the colour of one leaf seen along one direction, as the probe disc of render_kernel computes
// it (volrend.cu:111-128).  Shared by the disc overlay (vr_probe.cu) and vr_tree_eval (vr_query.cu).
#pragma once
#include "vr_march.cuh"

namespace vrb {

// maybe_precalc_basis (lumisphere.hpp:9-87) as render_kernel's disc instance computes it.  It is the march's basis
// (sh_basis / sg_basis) except for one contraction: this instance fuses -y*y into 4zz - xx - yy (B[11], B[13]).
template <int KBD>
__device__ __forceinline__ void disc_basis(const TreeDev& tree, float x, float y, float z,
                                           float (&B)[BasisCount<KBD>::n]) {
    if (tree.format == VR_FMT_SH) {
        sh_basis<KBD>(x, y, z, B);
        if constexpr (KBD >= 16) {
            const float z4 = __fmaf_rn(-y, y, __fmaf_rn(__fmul_rn(z, z), 4.f, -__fmul_rn(x, x)));
            B[11] = (float)__dmul_rn(__dmul_rn((double)y, -0.4570457994644658), (double)z4);
            B[13] = (float)__dmul_rn((double)z4, __dmul_rn((double)x, -0.4570457994644658));
        }
    } else {
#pragma unroll
        for (int i = 0; i < BasisCount<KBD>::n; ++i) B[i] = 0.f;
        sg_basis<KBD>(tree, x, y, z, B);
    }
}

// volrend.cu:111-128: per channel t, tmp = fma(coef(t*KBD + j), basis[j], tmp) for j = bmin .. bmax, then
// 1 / fma(2^n, ex2(r), 1) (the sigmoid); RGBA trees (KBD < 0) give coefficients 0..2 unchanged.
template <int KBD, class Coef>
__device__ __forceinline__ void lumisphere_rgb(const TreeDev& tree, float dx, float dy, float dz, int bmin, int bmax,
                                               Coef coef, float (&out)[3]) {
    if constexpr (KBD < 0) {
        out[0] = coef(0); out[1] = coef(1); out[2] = coef(2);
    } else {
        float B[BasisCount<KBD>::n];
        disc_basis<KBD>(tree, dx, dy, dz, B);
#pragma unroll
        for (int t = 0; t < 3; ++t) {
            float tmp = 0.f;
#pragma unroll
            for (int j = 0; j < BasisCount<KBD>::n; ++j)
                if (j >= bmin && j <= bmax) tmp = __fmaf_rn(coef(t * KBD + j), B[j], tmp);
            float e, sc;
            expf_parts(-tmp, e, sc);
            out[t] = __frcp_rn(__fmaf_rn(sc, e, 1.f));
        }
    }
}

}  // namespace vrb
