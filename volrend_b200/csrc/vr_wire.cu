// vr_wire.cu -- the octree grid as a line mesh: N3Tree::gen_wireframe (reference src/n3tree.cpp:365-434)
// generated on the device from the wide tables, bit for bit.  See DESIGN.md section 9.
//
// The reference walks the host tree depth first and pushes 24 vertices per emitted cell.  Here the cells are
// generated level by level (one thread per table entry), keyed by their Morton code, sorted (which restores the
// depth-first pre-order), and expanded to vertices.
#include <cooperative_groups.h>
#include <cub/device/device_radix_sort.cuh>
#include <cuda/std/tuple>

#include <algorithm>
#include <climits>
#include <cstring>
#include <type_traits>

#include "vr_types.h"
#include "vr_wire.h"

namespace cg = cooperative_groups;

namespace vrb {
namespace {

constexpr int kTB = 256;
constexpr int kWriteCells = 32;        // cells per CTA of the vertex writer
constexpr int kCellFloats = 24 * 9;    // 12 segments = 24 vertices of position, colour, normal
constexpr int kKey64Levels = 21;       // 3 bits per level

// A node the expansion visits: its table id and its integer corner on the grid of its own depth.
struct WireNode {
    uint32_t table, x, y, z;
};

// Cell order.  The reference visits octants x-major, then y, then z, and descends before moving on, so its output
// order is the order of the cells' Morton codes (x the most significant bit of each level) once every corner is
// left-aligned to the deepest emitted level Lc.  Emitted cells are disjoint, so the codes are distinct.
// Lc <= 21 fits 64 bits; deeper cuts keep levels 1..21 in `hi` and the rest in `lo`.
struct Key128 {
    unsigned long long hi, lo;
};
struct Key128Bits {
    __host__ __device__ ::cuda::std::tuple<unsigned long long&, unsigned long long&> operator()(Key128& k) const {
        return {k.hi, k.lo};
    }
};

__device__ __forceinline__ unsigned long long spread3(uint32_t v) {   // bit i -> bit 3i (21 bits)
    unsigned long long x = v & 0x1fffffu;
    x = (x | x << 32) & 0x1f00000000ffffull;
    x = (x | x << 16) & 0x1f0000ff0000ffull;
    x = (x | x << 8) & 0x100f00f00f00f00full;
    x = (x | x << 4) & 0x10c30c30c30c30c3ull;
    x = (x | x << 2) & 0x1249249249249249ull;
    return x;
}
__device__ __forceinline__ uint32_t compact3(unsigned long long x) {  // bit 3i -> bit i
    x &= 0x1249249249249249ull;
    x = (x ^ (x >> 2)) & 0x10c30c30c30c30c3ull;
    x = (x ^ (x >> 4)) & 0x100f00f00f00f00full;
    x = (x ^ (x >> 8)) & 0x1f0000ff0000ffull;
    x = (x ^ (x >> 16)) & 0x1f00000000ffffull;
    x = (x ^ (x >> 32)) & 0x1fffffull;
    return (uint32_t)x;
}
__device__ __forceinline__ unsigned long long interleave(uint32_t x, uint32_t y, uint32_t z) {
    return spread3(x) << 2 | spread3(y) << 1 | spread3(z);
}

// c[]: corner left-aligned to Lc bits
__device__ __forceinline__ void make_key(unsigned long long& k, const uint32_t c[3], int) {
    k = interleave(c[0], c[1], c[2]);
}
__device__ __forceinline__ void make_key(Key128& k, const uint32_t c[3], int Lc) {
    const int lo = Lc - kKey64Levels;
    const uint32_t m = (1u << lo) - 1u;
    k.hi = interleave(c[0] >> lo, c[1] >> lo, c[2] >> lo);
    k.lo = interleave(c[0] & m, c[1] & m, c[2] & m);
}
__device__ __forceinline__ void key_corner(const unsigned long long& k, int, uint32_t c[3]) {
    c[0] = compact3(k >> 2); c[1] = compact3(k >> 1); c[2] = compact3(k);
}
__device__ __forceinline__ void key_corner(const Key128& k, int Lc, uint32_t c[3]) {
    const int lo = Lc - kKey64Levels;
    c[0] = compact3(k.hi >> 2) << lo | compact3(k.lo >> 2);
    c[1] = compact3(k.hi >> 1) << lo | compact3(k.lo >> 1);
    c[2] = compact3(k.hi) << lo | compact3(k.lo);
}

// One slot per calling thread from a global counter, one atomic per group of converged threads.
template <class T>
__device__ __forceinline__ T claim(T* ctr) {
    cg::coalesced_group grp = cg::coalesced_threads();
    T base = 0;
    if (grp.thread_rank() == 0) base = atomicAdd(ctr, (T)grp.size());
    return grp.shfl(base, 0) + (T)grp.thread_rank();
}

// One thread per entry of every table in `in` (nodes of depth d).  An entry resolves kWideLv levels below its node:
// at sub-level k it lies in the cell of level d + k + 1 whose node has depth d + k.  That cell ends the walk when it
// is a leaf or when d + k >= max_depth; it is then emitted (count mode: tallied in hist) by the first of the
// 8^(kWideLv-1-k) entries it covers.  An entry that never ends is the table id of a node of depth d + kWideLv, which
// joins the next frontier.  The root table of wide_p = v sits at depth -v; its first v levels are the virtual
// root's octant 0, so only entries with zero virtual bits are real.
template <class K, bool kCount>
__global__ void __launch_bounds__(kTB) wire_expand_kernel(const uint32_t* __restrict__ wide, const WireNode* __restrict__ in,
                                                          long long n_in, int d, int v, int max_depth, int Lc,
                                                          WireNode* __restrict__ next, unsigned int* __restrict__ n_next,
                                                          K* __restrict__ keys, uint8_t* __restrict__ lvls,
                                                          unsigned long long* __restrict__ n_cells,
                                                          unsigned long long* __restrict__ hist) {
    constexpr int LV = kWideLv;
    constexpr uint32_t M = (1u << LV) - 1u;
    __shared__ unsigned int tally[2 * kWireLevels];   // count mode: leaves, then internal cells, by level
    if (kCount) {
        for (int i = threadIdx.x; i < 2 * kWireLevels; i += blockDim.x) tally[i] = 0;
        __syncthreads();
    }
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long f = g >> (3 * LV);
    const uint32_t e = (uint32_t)(g & (kWideEntries - 1));
    const int k0 = d < 0 ? -d : 0;
    const uint32_t ex = (e >> (2 * LV)) & M, ey = (e >> LV) & M, ez = e & M;
    if (f < n_in && ((ex | ey | ez) >> (LV - k0)) == 0) {
        const WireNode F = in[f];
        const uint32_t w = wide[(size_t)F.table * kWideEntries + e];
        // leaf word: bits 23..30 hold 103 + leaf level + v (build_wide_kernel)
        const int leaf_lvl = (w & kLeafBit) ? (int)((w >> 23) & 0xffu) - 103 - v : -1;
        bool inner = true;
        for (int k = k0; k < LV; ++k) {
            const int dn = d + k, sh = LV - 1 - k;
            const bool first = ((ex | ey | ez) & ((1u << sh) - 1u)) == 0u;
            if (leaf_lvl == dn + 1 || dn >= max_depth) {
                if (first) {
                    if (kCount) {
                        atomicAdd(&tally[dn + 1], 1u);
                    } else {
                        const int L = dn + 1, up = Lc - L;
                        const uint32_t c[3] = {((F.x << (k + 1)) | (ex >> sh)) << up, ((F.y << (k + 1)) | (ey >> sh)) << up,
                                               ((F.z << (k + 1)) | (ez >> sh)) << up};
                        const unsigned long long s = claim(n_cells);
                        make_key(keys[s], c, Lc);
                        lvls[s] = (uint8_t)L;
                    }
                }
                inner = false;
                break;
            }
            if (kCount && first) atomicAdd(&tally[kWireLevels + dn + 1], 1u);
        }
        if (inner) {
            const unsigned int s = claim(n_next);
            next[s] = WireNode{w, (F.x << LV) | ex, (F.y << LV) | ey, (F.z << LV) | ez};
        }
    }
    if (kCount) {
        __syncthreads();
        for (int i = threadIdx.x; i < 2 * kWireLevels; i += blockDim.x)
            if (tally[i]) atomicAdd(hist + i, (unsigned long long)tally[i]);
    }
}

// Vertex order inside a cell: for each (a, b) in (0,0), (0,1), (1,0), (1,1), the x-, y- and z-parallel edges whose two
// other corner selectors, in axis order, are (a, b); each edge from its low to its high end.  Bit v of
// sel_mask(axis): vertex v sits on the cell's high bound along `axis`.
constexpr uint32_t sel_mask(int axis) {
    uint32_t m = 0;
    for (int ab = 0; ab < 4; ++ab)
        for (int edge = 0; edge < 3; ++edge)
            for (int end = 0; end < 2; ++end) {
                const int first_other = edge == 0 ? 1 : 0;
                const int s = axis == edge ? end : axis == first_other ? (ab >> 1) : (ab & 1);
                m |= (uint32_t)s << (6 * ab + 2 * edge + end);
            }
    return m;
}
constexpr uint32_t kSelX = sel_mask(0), kSelY = sel_mask(1), kSelZ = sel_mask(2);

struct WireXf {
    float offset[3], scale[3];
};

// kWriteCells cells per CTA: their bounds into shared memory, then the CTA writes the cells' 216 floats each as one
// contiguous run.  Bounds follow the reference's float expression ((float)i / gridsz - offset) / scale, each
// operation rounded to nearest.
template <class K>
__global__ void __launch_bounds__(kTB) wire_write_kernel(const K* __restrict__ keys, const uint8_t* __restrict__ lvls,
                                                         long long n, int Lc, WireXf xf, float* __restrict__ out) {
    __shared__ float bb[kWriteCells][6];
    const long long c0 = (long long)blockIdx.x * kWriteCells;
    const int t = threadIdx.x;
    if (t < kWriteCells && c0 + t < n) {
        uint32_t c[3];
        key_corner(keys[c0 + t], Lc, c);
        const int L = lvls[c0 + t];
        const float gs = __uint2float_rn(1u << L);
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const uint32_t i = c[a] >> (Lc - L);
            bb[t][a] = __fdiv_rn(__fsub_rn(__fdiv_rn(__uint2float_rn(i), gs), xf.offset[a]), xf.scale[a]);
            bb[t][3 + a] = __fdiv_rn(__fsub_rn(__fdiv_rn(__uint2float_rn(i + 1), gs), xf.offset[a]), xf.scale[a]);
        }
    }
    __syncthreads();
    const long long left = n - c0;
    const int nf = (int)(left < kWriteCells ? left : kWriteCells) * kCellFloats;
    float* o = out + c0 * kCellFloats;
    for (int i = t; i < nf; i += blockDim.x) {
        const int cell = i / kCellFloats, r = i - cell * kCellFloats, vtx = r / 9, comp = r - vtx * 9;
        float val;
        if (comp < 3) {
            const uint32_t m = comp == 0 ? kSelX : comp == 1 ? kSelY : kSelZ;
            val = bb[cell][3 * ((m >> vtx) & 1u) + comp];
        } else {
            val = comp == 8 ? 1.f : 0.f;   // colour 0,0,0, normal 0,0,1
        }
        o[i] = val;
    }
}

unsigned int blocks_for(long long threads) { return (unsigned int)((threads + kTB - 1) / kTB); }

int clamp_depth(int max_depth) { return std::min(std::max(max_depth, 0), kWireLevels - 2); }

template <class K>
cudaError_t fill_impl(const WireTree& t, const WireLevels& lv, int mm, int Lc, long long n, float* out, cudaStream_t s,
                      int* launches) {
    long long cap = 1;   // frontier size: the most nodes of any depth the walk visits
    for (int l = 1; l <= mm; ++l) cap = std::max(cap, lv.inner[l]);
    K* keys[2] = {nullptr, nullptr};
    uint8_t* lvls[2] = {nullptr, nullptr};
    WireNode* nodes[2] = {nullptr, nullptr};
    unsigned long long* ctr = nullptr;   // {cells, next frontier}
    void* tmp = nullptr;
    size_t tmp_bytes = 0;
    cudaError_t e = cudaSuccess;
    auto alloc = [&](void** p, size_t bytes) {
        if (e == cudaSuccess) e = cudaMallocAsync(p, bytes, s);
    };
    for (int i = 0; i < 2; ++i) {
        alloc((void**)&keys[i], (size_t)n * sizeof(K));
        alloc((void**)&lvls[i], (size_t)n);
        alloc((void**)&nodes[i], (size_t)cap * sizeof(WireNode));
    }
    alloc((void**)&ctr, 2 * sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaMemsetAsync(ctr, 0, 2 * sizeof(unsigned long long), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(nodes[0], 0, sizeof(WireNode), s);   // the root: table 0, corner 0
    long long n_in = 1;
    int cur = 0;
    for (int d = -t.wide_p; e == cudaSuccess; d += kWideLv) {
        if (d > 0) {
            if (d > mm) break;
            n_in = lv.inner[d];
            if (n_in == 0) break;
            e = cudaMemsetAsync(ctr + 1, 0, sizeof(unsigned long long), s);
        }
        if (e != cudaSuccess) break;
        wire_expand_kernel<K, false><<<blocks_for(n_in * kWideEntries), kTB, 0, s>>>(
            t.wide, nodes[cur], n_in, d, t.wide_p, mm, Lc, nodes[cur ^ 1], reinterpret_cast<unsigned int*>(ctr + 1),
            keys[0], lvls[0], ctr, nullptr);
        e = cudaGetLastError();
        ++*launches;
        cur ^= 1;
    }
    if (e == cudaSuccess) {
        if constexpr (std::is_same<K, unsigned long long>::value) {
            e = cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys[0], keys[1], lvls[0], lvls[1], (int)n, 0, 3 * Lc, s);
            alloc(&tmp, tmp_bytes);
            if (e == cudaSuccess)
                e = cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys[0], keys[1], lvls[0], lvls[1], (int)n, 0, 3 * Lc, s);
        } else {
            e = cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys[0], keys[1], lvls[0], lvls[1], (int)n, Key128Bits{}, s);
            alloc(&tmp, tmp_bytes);
            if (e == cudaSuccess)
                e = cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys[0], keys[1], lvls[0], lvls[1], (int)n, Key128Bits{}, s);
        }
        ++*launches;   // counted as one launch, whatever number of passes the sort takes
    }
    if (e == cudaSuccess) {
        WireXf xf;
        for (int a = 0; a < 3; ++a) { xf.offset[a] = t.offset[a]; xf.scale[a] = t.scale[a]; }
        wire_write_kernel<K><<<(unsigned int)((n + kWriteCells - 1) / kWriteCells), kTB, 0, s>>>(keys[1], lvls[1], n, Lc, xf, out);
        e = cudaGetLastError();
        ++*launches;
    }
    for (int i = 0; i < 2; ++i) { cudaFreeAsync(keys[i], s); cudaFreeAsync(lvls[i], s); cudaFreeAsync(nodes[i], s); }
    cudaFreeAsync(ctr, s);
    cudaFreeAsync(tmp, s);
    return e;
}

}  // namespace

cudaError_t wire_levels(const WireTree& t, WireLevels& L, cudaStream_t s, int* launches) {
    memset(&L, 0, sizeof(L));
    WireNode* nodes[2] = {nullptr, nullptr};
    unsigned int* n_next = nullptr;
    unsigned long long* hist = nullptr;
    cudaError_t e = cudaSuccess;
    auto alloc = [&](void** p, size_t bytes) {
        if (e == cudaSuccess) e = cudaMallocAsync(p, bytes, s);
    };
    // no depth holds more tables than the tree
    for (int i = 0; i < 2; ++i) alloc((void**)&nodes[i], (size_t)std::max(t.n_tables, 1LL) * sizeof(WireNode));
    alloc((void**)&n_next, sizeof(unsigned int));
    alloc((void**)&hist, 2 * kWireLevels * sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaMemsetAsync(hist, 0, 2 * kWireLevels * sizeof(unsigned long long), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(nodes[0], 0, sizeof(WireNode), s);
    long long n_in = 1;
    int cur = 0;
    for (int d = -t.wide_p; e == cudaSuccess && n_in > 0; d += kWideLv) {
        e = cudaMemsetAsync(n_next, 0, sizeof(unsigned int), s);
        if (e != cudaSuccess) break;
        wire_expand_kernel<unsigned long long, true><<<blocks_for(n_in * kWideEntries), kTB, 0, s>>>(
            t.wide, nodes[cur], n_in, d, t.wide_p, INT_MAX, 0, nodes[cur ^ 1], n_next, nullptr, nullptr, nullptr, hist);
        e = cudaGetLastError();
        ++*launches;
        unsigned int h = 0;
        if (e == cudaSuccess) e = cudaMemcpyAsync(&h, n_next, sizeof(h), cudaMemcpyDeviceToHost, s);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        n_in = h;
        cur ^= 1;
    }
    unsigned long long h_hist[2 * kWireLevels] = {};
    if (e == cudaSuccess) e = cudaMemcpyAsync(h_hist, hist, sizeof(h_hist), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    for (int l = 0; l < kWireLevels; ++l) {
        L.leaf[l] = (long long)h_hist[l];
        L.inner[l] = (long long)h_hist[kWireLevels + l];
    }
    for (int i = 0; i < 2; ++i) cudaFreeAsync(nodes[i], s);
    cudaFreeAsync(n_next, s);
    cudaFreeAsync(hist, s);
    return e;
}

long long wire_cells(const WireTree& t, const WireLevels& lv, int max_depth) {
    const int L = clamp_depth(max_depth) + 1;
    long long n = 0;
    for (int l = 1; l <= L; ++l) n += lv.leaf[l];
    return n + lv.inner[L];
}

cudaError_t wire_fill(const WireTree& t, const WireLevels& lv, int max_depth, float* out, cudaStream_t s, int* launches) {
    const long long n = wire_cells(t, lv, max_depth);
    if (n <= 0) return cudaSuccess;
    if (n > INT_MAX) return cudaErrorInvalidValue;
    const int mm = clamp_depth(max_depth);
    const int Lc = std::min(mm + 1, t.max_level);
    return Lc <= kKey64Levels ? fill_impl<unsigned long long>(t, lv, mm, Lc, n, out, s, launches)
                              : fill_impl<Key128>(t, lv, mm, Lc, n, out, s, launches);
}

}  // namespace vrb
