// vr_ssim.cu -- per-view SSIM of two image batches and its gradient.  See DESIGN.md section 22.
//
// Definition (JaxNeRF's compute_ssim): an 11-tap Gaussian (sigma 1.5) applied separably with valid filtering to x, y,
// x^2, y^2 and xy of each RGB plane; clipped variances and covariance; the SSIM map averaged over the 3 channels and
// the (H-10) x (W-10) valid pixels.
//
// Forward: one CTA per 32x32 output tile of one view.  It loads the tile's 42x42 inputs of x and y (all three
// channels, float4 loads for RGBA rows) into shared memory, shifted by a per-tile, per-channel constant (the midpoint
// of x and y at the tile centre): the moments are formed from the shifted values, so E[x^2] - mu^2 does not lose the
// variance of a bright flat region to cancellation in float32.  Variances and covariance do not change under the
// shift; the means get it added back.  A horizontal pass writes the five moments of 42 rows x 32 columns, a
// vertical pass gives the tile's SSIM values; each CTA writes its sum (double) to its own slot, and one block per
// view adds the slots in a fixed order, so the result is bit-reproducible.
//
// Backward (a gather: every dx element is written by exactly one thread): one CTA per 32x32 input tile recomputes
// a = ds/dmu_x, b = ds/dE[x^2], c = ds/dE[xy] on the 42x42 output pixels whose windows touch the tile (from 52x52
// inputs, one channel at a time), then applies the transposed filter.  With the tile's shift k,
//   sum_q f (a_q + 2 x_p b_q + y_p c_q) = sum_q f a'_q + 2 (x_p - k) sum_q f b_q + (y_p - k) sum_q f c_q,
//   a'_q = a_q + (2 b_q + c_q) k,
// so the large, nearly cancelling terms of a bright flat region are never formed.  Recomputing beats storing a, b, c
// (and the means) from the forward pass: that would move 9 to 15 floats per pixel through HBM, against 7 read here.
//
// Flat windows: where all 121 inputs of a window of x (or y) are equal, its variance and the covariance are set to
// exactly 0, as they are in exact arithmetic.  Rounding would otherwise leave them a few ulps either side of 0 and
// pick the covariance clip's branch at random, and that branch switches the gradient term through E[xy] on and off.
// The horizontal pass writes each row's value where the row is flat (NaN elsewhere); the vertical pass compares them.
#include <cmath>
#include <cstdint>

#include "vr_ssim.h"

namespace vrb {
namespace {

constexpr int kTB = 256;
constexpr int kTaps = 11;
constexpr int kFT = 32, kFI = kFT + kTaps - 1;                    // forward: output tile, its input span
constexpr int kBT = 32, kBO = kBT + kTaps - 1, kBI = kBO + kTaps - 1;  // backward: input tile, outputs, inputs
constexpr float kC1 = 1e-4f, kC2 = 9e-4f;                        // (0.01 * max_val)^2, (0.03 * max_val)^2
constexpr int kMaxGridZ = 65535;
constexpr int kHm = 7;   // horizontal pass outputs: the five moments and the flat-row values of x and y
constexpr size_t kFwdSmem = sizeof(float) * (6 * kFI * kFI + kHm * kFI * kFT);
constexpr size_t kBwdSmem = sizeof(float) * (2 * kBI * kBI + kHm * kBI * kBO + 3 * kBO * kBO);

struct Filter {
    float f[kTaps];
};

// One view of an image batch: rows of `ch` floats; vec4 when ch == 4 and the base is 16-byte aligned.
struct Img {
    const float* p;
    int ch;
    bool vec4;
};

__device__ __forceinline__ void load_rgb(const Img& im, size_t pix, float v[3]) {
    if (im.vec4) {
        const float4 q = __ldg(reinterpret_cast<const float4*>(im.p) + pix);
        v[0] = q.x; v[1] = q.y; v[2] = q.z;
    } else {
        const float* s = im.p + pix * im.ch;
        v[0] = __ldg(s); v[1] = __ldg(s + 1); v[2] = __ldg(s + 2);
    }
}

// The filtered moments of one output pixel, of inputs shifted by k: mx = mu_x - k, xx = E[(x-k)^2], ...; flat_x /
// flat_y: the window of x / y holds one value, so its variance and the covariance are exactly 0.
struct Moments {
    float mx, my, xx, yy, xy;
    bool flat_x, flat_y;
};

// Adds tap weight f of the shifted inputs xv, yv.  x and y go through the same operations, so identical images give
// bitwise-identical moments (and SSIM exactly 1, gradient exactly 0).
__device__ __forceinline__ void add_tap(Moments& m, float f, float xv, float yv) {
    const float fx = f * xv, fy = f * yv;
    m.mx = fmaf(f, xv, m.mx);
    m.my = fmaf(f, yv, m.my);
    m.xx = fmaf(fx, xv, m.xx);
    m.yy = fmaf(fy, yv, m.yy);
    m.xy = fmaf(fx, yv, m.xy);
}

// SSIM of one output pixel from shifted moments (k: the shift); with kGrad also a' = ds/dmu_x + (2b + c) k, b and c.
// Products that must cancel exactly for identical images are rounded separately (__fmul_rn keeps them out of FMAs).
template <bool kGrad>
__device__ __forceinline__ float ssim_value(const Moments& m, float k, float* ga, float* gb, float* gc) {
    const float mx = m.mx + k, my = m.my + k;
    const float vx = m.flat_x ? 0.f : m.xx - __fmul_rn(m.mx, m.mx);
    const float vy = m.flat_y ? 0.f : m.yy - __fmul_rn(m.my, m.my);
    const float sxx = fmaxf(vx, 0.f), syy = fmaxf(vy, 0.f);
    const float sxy0 = m.flat_x || m.flat_y ? 0.f : m.xy - __fmul_rn(m.mx, m.my);
    const float pr = sxx * syy, rt = sqrtf(pr);
    const bool clip = fabsf(sxy0) > rt;
    const float sxy = clip ? copysignf(rt, sxy0) : sxy0;
    const float A = __fadd_rn(2.f * __fmul_rn(mx, my), kC1);
    const float C = __fadd_rn(__fadd_rn(__fmul_rn(mx, mx), __fmul_rn(my, my)), kC1);
    const float B = __fadd_rn(2.f * sxy, kC2), D = __fadd_rn(sxx + syy, kC2);
    const float s = __fmul_rn(A, B) / __fmul_rn(C, D);
    if (kGrad) {
        const float ag = A / __fmul_rn(C, D);    // ds/dsxy = 2 ag, ds/dsxx = -s / D = -ag B / D
        const float r = B / D;
        float dsxx = -(ag * r), c = 2.f * ag;
        if (clip) {
            if (pr > 0.f) dsxx += (sxy0 > 0.f ? c : -c) * syy / (2.f * rt);
            c = 0.f;
        }
        const float b = vx >= 0.f ? dsxx : 0.f;
        const float direct = 2.f / C * (__fmul_rn(r, my) - __fmul_rn(s, mx));
        *ga = direct - (__fmul_rn(2.f * m.mx, b) + __fmul_rn(m.my, c));
        *gb = b;
        *gc = c;
    }
    return s;
}

// The shift of a tile: the midpoint of x's and y's channel values at (cx, cy), clamped into the image.  One shift for
// both keeps the rounding of near-identical images correlated (their SSIM is close to 1 and the errors cancel); the
// midpoint keeps it small where x and y differ by a constant (a render against a target of another background).
__device__ __forceinline__ void tile_shift(const Img& x, const Img& y, int cx, int cy, int H, int W, float k[3]) {
    const size_t pix = (size_t)min(cy, H - 1) * W + min(cx, W - 1);
    float kx[3], ky[3];
    load_rgb(x, pix, kx);
    load_rgb(y, pix, ky);
#pragma unroll
    for (int c = 0; c < 3; ++c) k[c] = 0.5f * (kx[c] + ky[c]);
}

__device__ __forceinline__ double block_sum(double v, double* part) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
    __syncthreads();
    double b = 0.0;
    if (threadIdx.x == 0)
        for (int i = 0; i < kTB / 32; ++i) b += part[i];
    return b;
}

__global__ void __launch_bounds__(kTB) ssim_fwd_kernel(Img x, Img y, int H, int W, Filter f, double* __restrict__ partial) {
    extern __shared__ float sm[];
    float* xs = sm;                        // [3][kFI][kFI], shifted
    float* ys = xs + 3 * kFI * kFI;
    float* hm = ys + 3 * kFI * kFI;        // [kHm][kFI rows][kFT cols]
    __shared__ double part[kTB / 32];
    const int tid = threadIdx.x;
    const int x0 = blockIdx.x * kFT, y0 = blockIdx.y * kFT, Ho = H - (kTaps - 1), Wo = W - (kTaps - 1);
    const size_t plane = (size_t)H * W;
    x.p += blockIdx.z * plane * x.ch;
    y.p += blockIdx.z * plane * y.ch;
    float k[3];
    tile_shift(x, y, x0 + kFT / 2, y0 + kFT / 2, H, W, k);
    for (int i = tid; i < kFI * kFI; i += kTB) {
        const int gx = x0 + i % kFI, gy = y0 + i / kFI;
        float xv[3] = {0.f, 0.f, 0.f}, yv[3] = {0.f, 0.f, 0.f};
        if (gx < W && gy < H) {
            load_rgb(x, (size_t)gy * W + gx, xv);
            load_rgb(y, (size_t)gy * W + gx, yv);
#pragma unroll
            for (int c = 0; c < 3; ++c) { xv[c] -= k[c]; yv[c] -= k[c]; }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) { xs[c * kFI * kFI + i] = xv[c]; ys[c * kFI * kFI + i] = yv[c]; }
    }
    double acc = 0.0;
    const int tx = tid & 31, ty = tid >> 5;
    for (int c = 0; c < 3; ++c) {
        __syncthreads();
        const float* xc = xs + c * kFI * kFI;
        const float* yc = ys + c * kFI * kFI;
        for (int i = tid; i < kFI * kFT; i += kTB) {
            const int r = i / kFT, j = i % kFT;
            Moments m{};
            const float x0v = xc[r * kFI + j], y0v = yc[r * kFI + j];
            bool fx = true, fy = true;
#pragma unroll
            for (int t = 0; t < kTaps; ++t) {
                const float xv = xc[r * kFI + j + t], yv = yc[r * kFI + j + t];
                add_tap(m, f.f[t], xv, yv);
                fx &= xv == x0v;
                fy &= yv == y0v;
            }
            hm[i] = m.mx; hm[kFI * kFT + i] = m.my; hm[2 * kFI * kFT + i] = m.xx;
            hm[3 * kFI * kFT + i] = m.yy; hm[4 * kFI * kFT + i] = m.xy;
            hm[5 * kFI * kFT + i] = fx ? x0v : NAN; hm[6 * kFI * kFT + i] = fy ? y0v : NAN;
        }
        __syncthreads();
        for (int r = ty; r < kFT; r += kTB / 32) {
            if (x0 + tx >= Wo || y0 + r >= Ho) continue;
            Moments m{};
            const float hx = hm[5 * kFI * kFT + r * kFT + tx], hy = hm[6 * kFI * kFT + r * kFT + tx];
            m.flat_x = hx == hx;    // NaN: a row that is not flat
            m.flat_y = hy == hy;
#pragma unroll
            for (int t = 0; t < kTaps; ++t) {
                const int o = (r + t) * kFT + tx;
                m.flat_x &= hm[5 * kFI * kFT + o] == hx;
                m.flat_y &= hm[6 * kFI * kFT + o] == hy;
                const float ft = f.f[t];
                m.mx = fmaf(ft, hm[o], m.mx);
                m.my = fmaf(ft, hm[kFI * kFT + o], m.my);
                m.xx = fmaf(ft, hm[2 * kFI * kFT + o], m.xx);
                m.yy = fmaf(ft, hm[3 * kFI * kFT + o], m.yy);
                m.xy = fmaf(ft, hm[4 * kFI * kFT + o], m.xy);
            }
            acc += (double)ssim_value<false>(m, k[c], nullptr, nullptr, nullptr);
        }
    }
    const double b = block_sum(acc, part);
    if (tid == 0) partial[((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = b;
}

// One block per view: the view's n_tiles partial sums in a fixed order, times inv_count.
__global__ void __launch_bounds__(kTB) ssim_sum_kernel(const double* __restrict__ partial, int n_tiles, double inv_count,
                                                       double* __restrict__ ssim) {
    __shared__ double part[kTB / 32];
    const double* p = partial + (size_t)blockIdx.x * n_tiles;
    double acc = 0.0;
    for (int i = threadIdx.x; i < n_tiles; i += kTB) acc += p[i];
    const double b = block_sum(acc, part);
    if (threadIdx.x == 0) ssim[blockIdx.x] = b * inv_count;
}

__global__ void __launch_bounds__(kTB) ssim_bwd_kernel(Img x, Img y, int H, int W, Filter f, float* __restrict__ dx,
                                                       float scale) {
    extern __shared__ float sm[];
    float* xs = sm;                        // [kBI][kBI], shifted, one channel
    float* ys = xs + kBI * kBI;
    float* hm = ys + kBI * kBI;            // [kHm][kBI rows][kBO cols]; later [3][kBO rows][kBT cols]
    float* g = hm + kHm * kBI * kBO;       // a', b, c: [3][kBO][kBO]
    const int tid = threadIdx.x;
    const int x0 = blockIdx.x * kBT, y0 = blockIdx.y * kBT, Ho = H - (kTaps - 1), Wo = W - (kTaps - 1);
    const int qx0 = x0 - (kTaps - 1), qy0 = y0 - (kTaps - 1);   // first output (and input) pixel of the halo
    const size_t plane = (size_t)H * W;
    const int dch = x.ch;
    x.p += blockIdx.z * plane * x.ch;
    y.p += blockIdx.z * plane * y.ch;
    dx += blockIdx.z * plane * dch;
    float k[3];
    tile_shift(x, y, x0 + kBT / 2, y0 + kBT / 2, H, W, k);
    for (int c = 0; c < 3; ++c) {
        if (c > 0) __syncthreads();
        for (int i = tid; i < kBI * kBI; i += kTB) {
            const int gx = qx0 + i % kBI, gy = qy0 + i / kBI;
            float xv = 0.f, yv = 0.f;
            if (gx >= 0 && gx < W && gy >= 0 && gy < H) {
                const size_t pix = (size_t)gy * W + gx;
                xv = __ldg(x.p + pix * x.ch + c) - k[c];
                yv = __ldg(y.p + pix * y.ch + c) - k[c];
            }
            xs[i] = xv;
            ys[i] = yv;
        }
        __syncthreads();
        for (int i = tid; i < kBI * kBO; i += kTB) {
            const int r = i / kBO, j = i % kBO;
            Moments m{};
            const float x0v = xs[r * kBI + j], y0v = ys[r * kBI + j];
            bool fx = true, fy = true;
#pragma unroll
            for (int t = 0; t < kTaps; ++t) {
                const float xv = xs[r * kBI + j + t], yv = ys[r * kBI + j + t];
                add_tap(m, f.f[t], xv, yv);
                fx &= xv == x0v;
                fy &= yv == y0v;
            }
            hm[i] = m.mx; hm[kBI * kBO + i] = m.my; hm[2 * kBI * kBO + i] = m.xx;
            hm[3 * kBI * kBO + i] = m.yy; hm[4 * kBI * kBO + i] = m.xy;
            hm[5 * kBI * kBO + i] = fx ? x0v : NAN; hm[6 * kBI * kBO + i] = fy ? y0v : NAN;
        }
        __syncthreads();
        for (int i = tid; i < kBO * kBO; i += kTB) {
            const int r = i / kBO, j = i % kBO;
            const int qx = qx0 + j, qy = qy0 + r;
            float a = 0.f, b = 0.f, cc = 0.f;
            if (qx >= 0 && qx < Wo && qy >= 0 && qy < Ho) {
                Moments m{};
                const float hx = hm[5 * kBI * kBO + r * kBO + j], hy = hm[6 * kBI * kBO + r * kBO + j];
                m.flat_x = hx == hx;
                m.flat_y = hy == hy;
#pragma unroll
                for (int t = 0; t < kTaps; ++t) {
                    const int o = (r + t) * kBO + j;
                    m.flat_x &= hm[5 * kBI * kBO + o] == hx;
                    m.flat_y &= hm[6 * kBI * kBO + o] == hy;
                    const float ft = f.f[t];
                    m.mx = fmaf(ft, hm[o], m.mx);
                    m.my = fmaf(ft, hm[kBI * kBO + o], m.my);
                    m.xx = fmaf(ft, hm[2 * kBI * kBO + o], m.xx);
                    m.yy = fmaf(ft, hm[3 * kBI * kBO + o], m.yy);
                    m.xy = fmaf(ft, hm[4 * kBI * kBO + o], m.xy);
                }
                ssim_value<true>(m, k[c], &a, &b, &cc);
            }
            g[i] = a; g[kBO * kBO + i] = b; g[2 * kBO * kBO + i] = cc;
        }
        __syncthreads();
        // transposed filter along x: input column j of the tile takes outputs j + 10 - t of the halo
        for (int i = tid; i < kBO * kBT; i += kTB) {
            const int r = i / kBT, j = i % kBT;
            float sa = 0.f, sb = 0.f, sc = 0.f;
#pragma unroll
            for (int t = 0; t < kTaps; ++t) {
                const int o = r * kBO + j + (kTaps - 1) - t;
                const float ft = f.f[t];
                sa = fmaf(ft, g[o], sa);
                sb = fmaf(ft, g[kBO * kBO + o], sb);
                sc = fmaf(ft, g[2 * kBO * kBO + o], sc);
            }
            hm[i] = sa; hm[kBO * kBT + i] = sb; hm[2 * kBO * kBT + i] = sc;
        }
        __syncthreads();
        for (int i = tid; i < kBT * kBT; i += kTB) {
            const int r = i / kBT, j = i % kBT;
            const int px = x0 + j, py = y0 + r;
            if (px >= W || py >= H) continue;
            float sa = 0.f, sb = 0.f, sc = 0.f;
#pragma unroll
            for (int t = 0; t < kTaps; ++t) {
                const int o = (r + (kTaps - 1) - t) * kBT + j;
                const float ft = f.f[t];
                sa = fmaf(ft, hm[o], sa);
                sb = fmaf(ft, hm[kBO * kBT + o], sb);
                sc = fmaf(ft, hm[2 * kBO * kBT + o], sc);
            }
            const int li = (r + kTaps - 1) * kBI + j + kTaps - 1;
            const float v = sa + (__fmul_rn(2.f * xs[li], sb) + __fmul_rn(ys[li], sc));
            float* d = dx + ((size_t)py * W + px) * dch + c;
            *d = fmaf(scale, v, *d);
        }
    }
}

Img image(const float* p, int ch) {
    return Img{p, ch, ch == 4 && (reinterpret_cast<uintptr_t>(p) & 15u) == 0};
}

}  // namespace

cudaError_t ssim_pass(const float* x, int x_channels, const float* y, int y_channels, int n_views, int height, int width,
                      double* ssim, float* dx, float dx_scale, cudaStream_t stream, int* launches) {
    if (n_views == 0) return cudaSuccess;
    // per device, so set on every call (it is cheap)
    cudaError_t e = cudaFuncSetAttribute(ssim_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFwdSmem);
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(ssim_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBwdSmem);
    if (e != cudaSuccess) return e;
    Filter f;
    {
        double w[kTaps], sum = 0.0;
        for (int i = 0; i < kTaps; ++i) sum += (w[i] = exp(-0.5 * ((i - 5) / 1.5) * ((i - 5) / 1.5)));
        for (int i = 0; i < kTaps; ++i) f.f[i] = (float)(w[i] / sum);
    }
    const int Ho = height - (kTaps - 1), Wo = width - (kTaps - 1);
    const dim3 ftiles((Wo + kFT - 1) / kFT, (Ho + kFT - 1) / kFT);
    const int n_tiles = (int)(ftiles.x * ftiles.y);
    double* partial = nullptr;
    e = cudaMallocAsync((void**)&partial, sizeof(double) * n_tiles * n_views, stream);
    if (e != cudaSuccess) return e;
    const size_t plane = (size_t)height * width;
    const double inv_count = 1.0 / (3.0 * Ho * Wo);
    const float scale = (float)((double)dx_scale * inv_count);
    const dim3 btiles((width + kBT - 1) / kBT, (height + kBT - 1) / kBT);
    for (int v0 = 0; v0 < n_views && e == cudaSuccess; v0 += kMaxGridZ) {
        const int nv = n_views - v0 < kMaxGridZ ? n_views - v0 : kMaxGridZ;
        const Img xi = image(x + v0 * plane * x_channels, x_channels), yi = image(y + v0 * plane * y_channels, y_channels);
        ssim_fwd_kernel<<<dim3(ftiles.x, ftiles.y, nv), kTB, kFwdSmem, stream>>>(xi, yi, height, width, f,
                                                                               partial + (size_t)v0 * n_tiles);
        ++*launches;
        if (dx) {
            ssim_bwd_kernel<<<dim3(btiles.x, btiles.y, nv), kTB, kBwdSmem, stream>>>(
                xi, yi, height, width, f, dx + v0 * plane * x_channels, scale);
            ++*launches;
        }
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        ssim_sum_kernel<<<n_views, kTB, 0, stream>>>(partial, n_tiles, inv_count, ssim);
        ++*launches;
        e = cudaGetLastError();
    }
    const cudaError_t ef = cudaFreeAsync(partial, stream);
    return e != cudaSuccess ? e : ef;
}

}  // namespace vrb
