// vr_cull.cu -- tile culling of batch launches (DESIGN.md 3): the coarse max-sigma grid of a tree and the per-launch
// tile-coverage pass that tells the batch march which 4x8-pixel tiles cannot shade a sample.
//
// A ray that shades no sample leaves the march with T = 1 and r = g = b = +0, which is exactly the output of the miss
// path of render_pixel (vr_march.cuh).  A sample shades only when the sigma of its leaf is above sigma_thresh, and that
// leaf overlaps a grid cell whose maximum sigma is then above sigma_thresh too.  So a tile whose pixel rays pass near
// no such cell can take the miss path without marching, and the frames stay the same bit for bit.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cmath>

#include "vr_march.cuh"
#include "vr_tree.h"

using namespace vrb;

namespace {

constexpr int kTB = 256;
// A marked cell whose tile box exceeds this many tiles (a 128x256-pixel box) marks the whole view instead of its tiles:
// a close-up batch then costs one store per mask word per block instead of an atomic per word and tile row of every
// large cell.  Cells of the bench views cover about 5x3 tiles.
constexpr int kCellTilesMax = 1024;

// Position of entry g of a table whose origin is o on the march's position grid (TreeDev::pos_scale; the tree's unit
// cube is [0, lim)^3, lim = 2^(24 - wide_p)); false when the entry lies outside the cube (the virtual octants of the
// root table with wide_p = 1, never looked up).  Table level j resolves the position bits 23 - 2j and 22 - 2j.
__device__ __forceinline__ bool entry_origin(uint4 o, long long g, uint32_t lim, uint32_t& x, uint32_t& y, uint32_t& z,
                                             int& sh) {
    const uint32_t e = (uint32_t)(g & (kWideEntries - 1));
    sh = 24 - kWideLv - kWideLv * (int)o.w;
    constexpr uint32_t M = (1u << kWideLv) - 1;
    x = o.x | (((e >> (2 * kWideLv)) & M) << sh);
    y = o.y | (((e >> kWideLv) & M) << sh);
    z = o.z | ((e & M) << sh);
    return x < lim && y < lim && z < lim;
}

// org[child] of every child table of a table of level j (level-synchronous, from the root down).
__global__ void table_origin_kernel(const uint32_t* __restrict__ wide, uint4* __restrict__ org, long long n_entries,
                                    uint32_t j, uint32_t lim) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_entries) return;
    const uint4 o = org[g / kWideEntries];
    if (o.w != j) return;
    uint32_t x, y, z;
    int sh;
    if (!entry_origin(o, g, lim, x, y, z, sh)) return;
    const uint32_t w = wide[g];
    if (!(w & kLeafBit)) org[w] = make_uint4(x, y, z, j + 1);
}

// Every leaf entry of a reachable table raises the cells its cube overlaps to its sigma (NaN sigma never shades and is
// left out), and lowers grid[kSigmaGridCells], the smallest sigma.  An entry of a leaf above the table's levels is one
// of the copies that tile the leaf's cube, so the copies together cover exactly the leaf.
__global__ void sigma_grid_kernel(const uint32_t* __restrict__ wide, const uint4* __restrict__ org, long long n_entries,
                                  uint32_t lim, int cell_shift, uint32_t* __restrict__ grid) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_entries) return;
    const uint4 o = org[g / kWideEntries];
    if (o.w == ~0u) return;
    uint32_t x, y, z;
    int sh;
    if (!entry_origin(o, g, lim, x, y, z, sh)) return;
    const uint32_t w = wide[g];
    if (!(w & kLeafBit)) return;
    const float s = __half2float(__ushort_as_half((unsigned short)(w & 0xffffu)));
    if (s != s) return;
    const uint32_t key = sigma_key(__float_as_uint(s));
    atomicMin(grid + kSigmaGridCells, key);
    const uint32_t span = (1u << sh) - 1u;
    for (uint32_t cx = x >> cell_shift; cx <= (x + span) >> cell_shift; ++cx)
        for (uint32_t cy = y >> cell_shift; cy <= (y + span) >> cell_shift; ++cy)
            for (uint32_t cz = z >> cell_shift; cz <= (z + span) >> cell_shift; ++cz)
                atomicMax(grid + ((cx * kSigmaGridN + cy) * kSigmaGridN + cz), key);
}

// ---------------------------------------------------------------------------------------- tile coverage
// Bits b0..b1 (inclusive) of a view's mask.
__device__ void set_bits(uint32_t* m, uint32_t b0, uint32_t b1) {
    for (uint32_t wi = b0 >> 5; wi <= (b1 >> 5); ++wi) {
        const uint32_t lo = wi == (b0 >> 5) ? (b0 & 31u) : 0u, hi = wi == (b1 >> 5) ? (b1 & 31u) : 31u;
        const uint32_t bits = (hi == 31u ? 0xffffffffu : ((2u << hi) - 1u)) & ~((1u << lo) - 1u);
        atomicOr(m + wi, bits);
    }
}

// Frame row of the last output row of tile row ty (frame_row is increasing in the output row).
__device__ __forceinline__ int tile_last_row(const LaunchDev& P, int ty) {
    return P.y0 + frame_row(P, min(ty * kTH + kTH - 1, P.h - 1));
}

// blockIdx.y = view, one thread per grid cell.  A cell whose maximum sigma is above the view's sigma_thresh marks every
// tile with a pixel whose ray can come near it: the cell, grown by eps in tree space, is projected with the pinhole
// model of ray_geometry (pixel px looks along (px - W/2) / fx, no half-pixel offset), and the bounding box of its
// corners, grown by dpx pixels, is rounded outwards to pixels and then to tiles.  The bounds (DESIGN.md 3):
//   eps = 1e-5 (4 + |c|_1), c the camera centre in tree space: a sample position is fma(t, d, c) on the 2^(24 - p)
//     grid, a few fp32 roundings (2^-24 relative each) of numbers no larger than |c|_1 + sqrt(3) away from the exact
//     point of the pixel's ray, then clamped into the box, which brings it no further from an exact point inside it;
//   dpx = 1 + 1e-5 (|fx| + |fy|) (1 + |vx| + |vy|)^2 pixels: the fp32 direction of a pixel's ray differs from the
//     exact (vx, vy, -1) by a few ulps, a far smaller angle than this, and 1 pixel covers the rounding of the box.
// The whole view is marked when the tree is NDC, when render_bbox leaves the unit cube (samples outside the cube are
// clamped onto its faces), when sigma_thresh is below the sigma of every leaf, when the camera frame is singular or
// not finite, when a marked cell reaches the camera plane (it may contain the camera), and when a marked cell covers
// more than kCellTilesMax tiles.
__global__ void __launch_bounds__(kTB) tile_mask_kernel(const __grid_constant__ LaunchDev P) {
    __shared__ double s_m[9], s_c[3], s_eps, s_dpx;
    __shared__ float s_thr;
    __shared__ int s_all, s_hit;
    pdl_launch_dependents();   // the march may become resident; it reads the mask only after its wait
    const int v = blockIdx.y;
    const CamDev& cam = P.cams[v];
    const OptDev& opt = P.opts ? P.opts[v] : P.opt;
    const TreeDev& T = P.tree;
    if (threadIdx.x == 0) {
        bool all = T.ndc_width > 0.f;
        for (int i = 0; i < 3; ++i)
            all = all || !(opt.render_bbox[i] >= 0.f && opt.render_bbox[i + 3] <= 1.f) || !(T.scale[i] != 0.f) ||
                  !isfinite(T.scale[i]) || !isfinite(T.offset[i]);
        const float thr = opt.sigma_thresh;
        all = all || thr < __uint_as_float(sigma_key_bits(T.sigma_grid[kSigmaGridCells]));
        // ray of pixel (px, py): C + s M (vx, vy, 1), s >= 0, M = [c2w column 0, column 1, -column 2]
        const double M[9] = {cam.c2w[0], cam.c2w[3], -(double)cam.c2w[6],
                             cam.c2w[1], cam.c2w[4], -(double)cam.c2w[7],
                             cam.c2w[2], cam.c2w[5], -(double)cam.c2w[8]};
        const double a0 = M[4] * M[8] - M[5] * M[7], a1 = M[5] * M[6] - M[3] * M[8], a2 = M[3] * M[7] - M[4] * M[6];
        const double det = M[0] * a0 + M[1] * a1 + M[2] * a2;
        all = all || !(fabs(det) > 0.0) || !isfinite(det) || !isfinite(cam.fx) || !isfinite(cam.fy);
        if (!all) {
            const double id = 1.0 / det;
            s_m[0] = a0 * id; s_m[1] = (M[2] * M[7] - M[1] * M[8]) * id; s_m[2] = (M[1] * M[5] - M[2] * M[4]) * id;
            s_m[3] = a1 * id; s_m[4] = (M[0] * M[8] - M[2] * M[6]) * id; s_m[5] = (M[2] * M[3] - M[0] * M[5]) * id;
            s_m[6] = a2 * id; s_m[7] = (M[1] * M[6] - M[0] * M[7]) * id; s_m[8] = (M[0] * M[4] - M[1] * M[3]) * id;
            double l1 = 0.0;
            for (int i = 0; i < 3; ++i) {
                s_c[i] = cam.c2w[9 + i];
                l1 += fabs((double)T.scale[i] * cam.c2w[9 + i] + T.offset[i]);
            }
            s_eps = 1e-5 * (4.0 + l1);
            all = !isfinite(s_eps);
        }
        s_dpx = 1e-5 * (fabs((double)cam.fx) + fabs((double)cam.fy));
        s_thr = thr;
        s_all = all;
        s_hit = 0;
    }
    __syncthreads();
    uint32_t* mask = const_cast<uint32_t*>(P.tile_mask) + (size_t)v * P.mask_words;
    const int cell = blockIdx.x * blockDim.x + threadIdx.x;
    if (!s_all && cell < kSigmaGridCells &&
        __uint_as_float(sigma_key_bits(T.sigma_grid[cell])) > s_thr) {
        const int ci[3] = {cell >> (2 * kSigmaGridLevel), (cell >> kSigmaGridLevel) & (kSigmaGridN - 1),
                           cell & (kSigmaGridN - 1)};
        double lo[3], hi[3];   // the grown cell in world space, minus the camera centre
        for (int i = 0; i < 3; ++i) {
            const double a = ((double)ci[i] / kSigmaGridN - s_eps - T.offset[i]) / T.scale[i];
            const double b = ((double)(ci[i] + 1) / kSigmaGridN + s_eps - T.offset[i]) / T.scale[i];
            lo[i] = fmin(a, b) - s_c[i];
            hi[i] = fmax(a, b) - s_c[i];
        }
        double wmin = INFINITY, wmax = -INFINITY, xmin = INFINITY, xmax = -INFINITY, ymin = INFINITY,
               ymax = -INFINITY;
        double vmax = 0.0;
        for (int k = 0; k < 8; ++k) {
            const double q0 = (k & 4) ? hi[0] : lo[0], q1 = (k & 2) ? hi[1] : lo[1], q2 = (k & 1) ? hi[2] : lo[2];
            const double u = s_m[0] * q0 + s_m[1] * q1 + s_m[2] * q2;
            const double vv = s_m[3] * q0 + s_m[4] * q1 + s_m[5] * q2;
            const double w = s_m[6] * q0 + s_m[7] * q1 + s_m[8] * q2;
            wmin = fmin(wmin, w); wmax = fmax(wmax, w);
            const double vx = u / w, vy = vv / w;
            vmax = fmax(vmax, fabs(vx) + fabs(vy));
            const double px = vx * cam.fx + 0.5 * cam.width, py = 0.5 * cam.height - vy * cam.fy;
            xmin = fmin(xmin, px); xmax = fmax(xmax, px);
            ymin = fmin(ymin, py); ymax = fmax(ymax, py);
        }
        if (wmax < 0.0) {
            // behind the camera: no sample of a ray (t >= 0) lies in it
        } else if (!(wmin > 0.0)) {
            s_hit = 1;
        } else {
            const double d = 1.0 + s_dpx * (1.0 + vmax) * (1.0 + vmax);
            const double fx0 = ceil(xmin - d), fx1 = floor(xmax + d), fy0 = ceil(ymin - d), fy1 = floor(ymax + d);
            if (!(isfinite(fx0) && isfinite(fx1) && isfinite(fy0) && isfinite(fy1))) {
                s_hit = 1;
            } else if (fx1 >= P.x0 && fx0 <= P.x0 + P.w - 1 && fy1 >= P.y0) {
                const int px0 = (int)fmax(fx0, (double)P.x0), px1 = (int)fmin(fx1, (double)(P.x0 + P.w - 1));
                const int tx0 = (px0 - P.x0) / kTW, tx1 = (px1 - P.x0) / kTW;
                // tile rows [ty0, ty1]: the first whose last frame row is >= fy0, the last whose first is <= fy1
                const double top = fy0, bot = fy1;
                int a = 0, b = P.tiles_y;
                while (a < b) { const int m = (a + b) >> 1; if (tile_last_row(P, m) >= top) b = m; else a = m + 1; }
                const int ty0 = a;
                a = 0; b = P.tiles_y;
                while (a < b) { const int m = (a + b) >> 1; if (P.y0 + frame_row(P, m * kTH) > bot) b = m; else a = m + 1; }
                const int ty1 = a - 1;
                if ((long long)(ty1 - ty0 + 1) * (tx1 - tx0 + 1) > kCellTilesMax)
                    s_hit = 1;   // a cell this close to the camera: the whole view, in bounded work
                else
                    for (int ty = ty0; ty <= ty1; ++ty)
                        set_bits(mask, (uint32_t)(ty * P.tiles_x + tx0), (uint32_t)(ty * P.tiles_x + tx1));
            }
        }
    }
    __syncthreads();
    if ((s_all && blockIdx.x == 0) || s_hit)
        for (int i = threadIdx.x; i < P.mask_words; i += blockDim.x) mask[i] = 0xffffffffu;
}

}  // namespace

int vrb::build_sigma_grid(vr_tree* t, cudaStream_t stream, bool with_org) {
    const TreeDev& D = t->dev;
    const long long n_entries = D.wide_entries;
    const unsigned blocks = (unsigned)((n_entries + kTB - 1) / kTB);
    const uint32_t lim = 1u << (24 - D.wide_p);
    int launches = 0;
    if (with_org) {
        // org[table] = {x, y, z, table level} of the table's origin on the march's position grid; ~0u: not reachable
        static const uint4 root = make_uint4(0u, 0u, 0u, 0u);
        if (cudaMemsetAsync(t->tab_org, 0xff, (size_t)t->n_tables * sizeof(uint4), stream) != cudaSuccess ||
            cudaMemcpyAsync(t->tab_org, &root, sizeof(uint4), cudaMemcpyHostToDevice, stream) != cudaSuccess)
            return -1;
        // table levels on a root-to-leaf path of leaves up to max_depth + wide_p levels below the (virtual) root
        const int levels = wide_table_levels(D.max_depth + D.wide_p);
        for (int j = 0; j + 1 < levels; ++j) {
            table_origin_kernel<<<blocks, kTB, 0, stream>>>(D.wide, t->tab_org, n_entries, (uint32_t)j, lim);
            ++launches;
        }
    }
    if (cudaMemsetAsync(t->sigma_grid, 0, (size_t)kSigmaGridCells * 4, stream) != cudaSuccess ||
        cudaMemsetAsync(t->sigma_grid + kSigmaGridCells, 0xff, 4, stream) != cudaSuccess)
        return -1;
    sigma_grid_kernel<<<blocks, kTB, 0, stream>>>(D.wide, t->tab_org, n_entries, lim, 24 - D.wide_p - kSigmaGridLevel,
                                                   t->sigma_grid);
    ++launches;
    if (cudaGetLastError() != cudaSuccess) return -1;
    return launches;
}

int vrb::launch_tile_mask(vr_tree* t, LaunchDev& P, cudaStream_t stream) {
    P.tiles_x = (P.w + kTW - 1) / kTW;   // (as the launch's set_work computes them)
    P.tiles_y = (P.h + kTH - 1) / kTH;
    const int words = (P.tiles_x * P.tiles_y + 31) / 32;
    const size_t need = (size_t)words * P.n_views;
    {
        // Under the lock, as the camera ring: the buffer belongs to (tree, stream).  Growing it frees the old one;
        // cudaFree waits for the launches that still read it.  A stream's batches rarely change size, so this
        // happens on its first batch and when a larger one comes.
        std::lock_guard<std::mutex> lk(t->res_mu);
        StreamRes& sr = t->res.at(stream);
        if (need > sr.mask_cap) {
            VR_CUDA(cudaFree(sr.tile_mask));
            sr.tile_mask = nullptr; sr.mask_cap = 0;
            VR_CUDA(cudaMalloc(&sr.tile_mask, need * 4));
            sr.mask_cap = need;
        }
        P.tile_mask = sr.tile_mask;
    }
    P.mask_words = words;
    VR_CUDA(cudaMemsetAsync(const_cast<uint32_t*>(P.tile_mask), 0, need * 4, stream));
    tile_mask_kernel<<<dim3(kSigmaGridCells / kTB, P.n_views), kTB, 0, stream>>>(P);
    VR_CUDA(cudaGetLastError());
    return VR_OK;
}
