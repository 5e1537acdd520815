// vr_tv.cu -- total variation between neighbouring leaves: the leaf-neighbour table and the TV gradient pass.
// See DESIGN.md section 20.
//
// Neighbours: the wireframe's walk (vr_wire_walk.cuh) yields every leaf once with its table entry, level L and integer
// corner i on the 2^L grid; the forward neighbour along axis a is the leaf that holds the point (i + e_a) 2^-L, found
// by the descent of vr_tree_query (descend_wide) from the root and mapped to its slot through the slot map.
//
// TV: one thread per (slot, column) of the slots that have a neighbour; the differences, the root and the energy in
// double, one float atomicAdd per term into the gradient.
#include <cmath>

#include "vr_probe.h"
#include "vr_tv.h"
#include "vr_wire_walk.cuh"

namespace vrb {
namespace {

constexpr int kTvTB = 256;
constexpr double kTvEps = 1e-8;

// The sink of the neighbour walk: every leaf writes its own three entries of nbr.  Under table parity 1 the root table
// repeats leaf entries, but the walk emits each cell once, from the first entry that covers it.
struct NbrSink {
    static constexpr bool kCount = false;
    TreeDev tree;
    const uint32_t* wslot;
    int32_t* nbr;
    __device__ __forceinline__ void operator()(uint32_t table, uint32_t e, int L, uint32_t x, uint32_t y,
                                               uint32_t z) const {
        const uint32_t slot = __ldg(wslot + (size_t)table * kWideEntries + e);
        // the corner on the tables' 2^(24 - wide_p) position grid: exact, as leaf level + wide_p <= 24
        const int sh = 24 - tree.wide_p - L;
        const uint32_t c[3] = {x, y, z};
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            int32_t n = -1;
            if (c[a] + 1u < (1u << L)) {
                uint32_t u[3] = {x << sh, y << sh, z << sh};
                u[a] = (c[a] + 1u) << sh;
                int j = 0;
                uint32_t w;
                n = (int32_t)__ldg(wslot + descend_wide(tree, u, j, 0u, w, nullptr, 0));
            }
            nbr[(size_t)slot * 3 + a] = n;
        }
    }
};

// n_color colour columns (0 when the colour weight is 0), then sigma when sigma_on.  Every leaf but the one at the
// tree's (+x, +y, +z) corner has a forward neighbour; that leaf's terms are sqrt(eps) each and `corner` adds them.
__global__ void __launch_bounds__(kTvTB) tv_kernel(const float* __restrict__ v, const int32_t* __restrict__ nbr,
                                                   long long n_slots, TvColumns cols, int n_color, int n_cols,
                                                   double sc_sigma, double sc_color, double corner,
                                                   float* __restrict__ grad, double* __restrict__ energy) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    double e_loc = 0.0;
    if (g < n_slots * n_cols) {
        const long long s = g / n_cols;
        const int j = (int)(g - s * n_cols);
        const int32_t n[3] = {__ldg(nbr + 3 * s), __ldg(nbr + 3 * s + 1), __ldg(nbr + 3 * s + 2)};
        if (n[0] >= 0 || n[1] >= 0 || n[2] >= 0) {
            const bool colour = j < n_color;
            const int col = colour ? (j / cols.n_coef) * cols.coef_stride + j % cols.n_coef : cols.data_dim - 1;
            const double lam = colour ? sc_color : sc_sigma;
            const size_t dd = (size_t)cols.data_dim;
            const double vs = (double)__ldg(v + (size_t)s * dd + col);
            double d[3], ss = kTvEps;
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                d[a] = n[a] >= 0 ? (double)__ldg(v + (size_t)n[a] * dd + col) - vs : 0.0;
                ss += d[a] * d[a];
            }
            const double r = sqrt(ss);
            e_loc = lam * r;
            const double k = lam / r;
            atomicAdd(grad + (size_t)s * dd + col, (float)(-((d[0] + d[1]) + d[2]) * k));
#pragma unroll
            for (int a = 0; a < 3; ++a)
                if (n[a] >= 0) atomicAdd(grad + (size_t)n[a] * dd + col, (float)(d[a] * k));
        }
    }
    if (!energy) return;
    if (g == 0) e_loc += corner;
    __shared__ double part[kTvTB / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) e_loc += __shfl_down_sync(0xffffffffu, e_loc, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = e_loc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double b = 0.0;
        for (int i = 0; i < kTvTB / 32; ++i) b += part[i];
        atomicAdd(energy, b);
    }
}

}  // namespace

cudaError_t tv_neighbors(const WireTree& w, const WireLevels& lv, const TreeDev& tree, const uint32_t* wslot,
                         long long n_slots, int32_t* nbr, cudaStream_t stream, int* launches) {
    cudaError_t e = cudaMemsetAsync(nbr, 0xff, (size_t)n_slots * 3 * sizeof(int32_t), stream);
    if (e != cudaSuccess) return e;
    // the deepest cut: every cell the walk ends at is a leaf
    return wire_walk(w, lv, kWireLevels - 2, NbrSink{tree, wslot, nbr}, stream, launches);
}

cudaError_t tv_pass(const float* data, const int32_t* nbr, long long n_slots, TvColumns cols, double scale_sigma,
                    double scale_color, float* grad, double* energy, cudaStream_t stream, int* launches) {
    const int n_color = scale_color > 0.0 ? 3 * cols.n_coef : 0;
    const int n_cols = n_color + (scale_sigma > 0.0 ? 1 : 0);
    if (n_cols == 0 || n_slots == 0) return cudaSuccess;
    const double corner = sqrt(kTvEps) * (n_color * scale_color + (n_cols > n_color ? scale_sigma : 0.0));
    const long long threads = n_slots * n_cols;
    tv_kernel<<<(unsigned int)((threads + kTvTB - 1) / kTvTB), kTvTB, 0, stream>>>(
        data, nbr, n_slots, cols, n_color, n_cols, scale_sigma, scale_color, corner, grad, energy);
    ++*launches;
    return cudaGetLastError();
}

}  // namespace vrb
