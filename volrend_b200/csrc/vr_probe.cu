// vr_probe.cu -- the lumisphere probe disc (volrend.cu:100-134) drawn over finished frames.
//
// The reference draws the disc inside render_kernel: a pixel of the top-right corner whose centre falls inside the
// disc is not marched but coloured with the probed leaf's view-dependent colour, seen along the direction the disc
// point faces.  Its output is therefore "march every pixel, then overwrite the disc pixels", which is what this
// kernel does after the march kernels have written the frame; they stay unchanged.
//
// Every floating-point operation is the instruction the reference's sm_90 SASS of render_kernel issues, so that the
// disc rim, the direction and the colour come out bit for bit:
//   h = float(S) * 0.5;  a = xx / h - 1 (= -cen[0]);  b = yy / h - 1 (= cen[1]);  c = fma(a, a, b * b)
//   c <= 1:  s = sqrt(1 - c) (= -cen[2]);  dir[i] = fma(-m[6+i], s, fma(b, m[3+i], -(a * m[i])))
//   colour:  tmp = fma(coeff[i], basis[i], tmp) for i = basis_minmax[0] .. basis_minmax[1];  1 / fma(2^n, ex2(r), 1)
// The integer candidate test wraps like the 32-bit adds of the SASS.
#include <cuda_runtime.h>

#include "vr_lumisphere.cuh"
#include "vr_probe.h"

namespace vrb {
namespace {

template <int KBD>
__global__ void __launch_bounds__(256) probe_disc_kernel(const ProbeLaunch P) {
    constexpr int kCoef = KBD < 0 ? 3 : 3 * KBD;
    __shared__ float s_coef[kCoef];
    __shared__ uint32_t s_entry;
    if (threadIdx.x == 0) s_entry = probe_leaf_entry(P.tree, P.probe[0], P.probe[1], P.probe[2]);
    __syncthreads();
    const unsigned short* rec = reinterpret_cast<const unsigned short*>(P.tree.wrecs + (size_t)s_entry * P.tree.rec_bytes);
    for (int i = threadIdx.x; i < kCoef; i += blockDim.x) s_coef[i] = __half2float(__ushort_as_half(rec[i]));
    __syncthreads();

    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)P.cw * P.ch) return;
    const int view = blockIdx.y;
    const int x = P.cx0 + (int)(i % P.cw), y = P.cy0 + (int)(i / P.cw);
    const CamDev& cam = P.cams ? P.cams[view] : P.cam;
    const int S = P.disp;
    const int xx = (int)((uint32_t)x + 5u - (uint32_t)cam.width + (uint32_t)S), yy = y - 5;
    const float h = __fmul_rn((float)S, 0.5f);
    const float a = __fadd_rn(__fdiv_rn((float)xx, h), -1.f);
    const float b = __fadd_rn(__fdiv_rn((float)yy, h), -1.f);
    const float c = __fmaf_rn(a, a, __fmul_rn(b, b));
    if (!(c <= 1.f)) return;  // marched normally: the frame already holds it

    float d[3] = {0.f, 0.f, 0.f};
    if constexpr (KBD >= 0) {
        const float s = __fsqrt_rn(__fsub_rn(1.f, c));
        const float* m = cam.c2w;
#pragma unroll
        for (int k = 0; k < 3; ++k) d[k] = __fmaf_rn(-m[6 + k], s, __fmaf_rn(b, m[3 + k], -__fmul_rn(a, m[k])));
    }
    float out[3];
    lumisphere_rgb<KBD>(P.tree, d[0], d[1], d[2], P.bmin, P.bmax, [&](int k) { return s_coef[k]; }, out);
    // volrend.cu:153-163 with alpha 1: the background or existing colour enters with weight 0
    float o[4] = {__fadd_rn(out[0], 0.f), __fadd_rn(out[1], 0.f), __fadd_rn(out[2], 0.f), 1.f};
    const uint32_t q = quantise(o);
    if (P.surf) {
        surf2Dwrite(q, P.surf, x * 4, y, cudaBoundaryModeZero);
        return;
    }
    const size_t off = ((size_t)view * P.h + (y - P.y0)) * P.w + (x - P.x0);
    if (P.rgba8) reinterpret_cast<uint32_t*>(P.rgba8)[off] = q;
    if (P.rgbaf) P.rgbaf[off] = make_float4(o[0], o[1], o[2], o[3]);
}

template <int KBD>
cudaError_t launch(const ProbeLaunch& P, cudaStream_t stream) {
    const long long n = (long long)P.cw * P.ch;
    const dim3 grid((unsigned)((n + 255) / 256), (unsigned)P.n_views);
    probe_disc_kernel<KBD><<<grid, 256, 0, stream>>>(P);
    return cudaGetLastError();
}

}  // namespace

cudaError_t probe_draw(const ProbeLaunch& P, int kbd, cudaStream_t stream) {
    switch (kbd) {
        case -1: return launch<-1>(P, stream);
        case 1: return launch<1>(P, stream);
        case 4: return launch<4>(P, stream);
        case 9: return launch<9>(P, stream);
        case 16: return launch<16>(P, stream);
        case 25: return launch<25>(P, stream);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace vrb
