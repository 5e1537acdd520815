// vr_wire.cu -- the octree grid as a line mesh: N3Tree::gen_wireframe (reference src/n3tree.cpp:365-434)
// generated on the device from the wide tables, bit for bit.  See DESIGN.md section 9.
//
// The reference walks the host tree depth first and pushes 24 vertices per emitted cell.  Here the cells are
// generated level by level (one thread per table entry, vr_wire_walk.cuh), keyed by their Morton code, sorted (which
// restores the depth-first pre-order), and expanded to vertices.
#include <cub/device/device_radix_sort.cuh>
#include <cuda/std/tuple>

#include <algorithm>
#include <climits>
#include <cstring>
#include <type_traits>

#include "vr_types.h"
#include "vr_wire.h"
#include "vr_wire_walk.cuh"

namespace vrb {
namespace {

constexpr int kWriteCells = 32;        // cells per CTA of the vertex writer
constexpr int kCellFloats = 24 * 9;    // 12 segments = 24 vertices of position, colour, normal
constexpr int kKey64Levels = 21;       // 3 bits per level

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

// The sink of the fill: each emitted cell's key, its corner left-aligned to Lc bits, and its level.
template <class K>
struct WireKeys {
    static constexpr bool kCount = false;
    K* keys;
    uint8_t* lvls;
    unsigned long long* n_cells;
    int Lc;
    __device__ __forceinline__ void operator()(uint32_t, uint32_t, int L, uint32_t x, uint32_t y, uint32_t z) const {
        const int up = Lc - L;
        const uint32_t c[3] = {x << up, y << up, z << up};
        const unsigned long long s = wire_claim(n_cells);
        make_key(keys[s], c, Lc);
        lvls[s] = (uint8_t)L;
    }
};

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
__global__ void __launch_bounds__(kWireTB) wire_write_kernel(const K* __restrict__ keys, const uint8_t* __restrict__ lvls,
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

int clamp_depth(int max_depth) { return std::min(std::max(max_depth, 0), kWireLevels - 2); }

template <class K>
cudaError_t fill_impl(const WireTree& t, const WireLevels& lv, int mm, int Lc, long long n, float* out, cudaStream_t s,
                      int* launches) {
    K* keys[2] = {nullptr, nullptr};
    uint8_t* lvls[2] = {nullptr, nullptr};
    unsigned long long* n_cells = nullptr;
    void* tmp = nullptr;
    size_t tmp_bytes = 0;
    cudaError_t e = cudaSuccess;
    auto alloc = [&](void** p, size_t bytes) {
        if (e == cudaSuccess) e = cudaMallocAsync(p, bytes, s);
    };
    for (int i = 0; i < 2; ++i) {
        alloc((void**)&keys[i], (size_t)n * sizeof(K));
        alloc((void**)&lvls[i], (size_t)n);
    }
    alloc((void**)&n_cells, sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaMemsetAsync(n_cells, 0, sizeof(unsigned long long), s);
    if (e == cudaSuccess) e = wire_walk(t, lv, mm, WireKeys<K>{keys[0], lvls[0], n_cells, Lc}, s, launches);
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
        wire_write_kernel<K><<<(unsigned int)((n + kWriteCells - 1) / kWriteCells), kWireTB, 0, s>>>(keys[1], lvls[1], n, Lc, xf, out);
        e = cudaGetLastError();
        ++*launches;
    }
    for (int i = 0; i < 2; ++i) { cudaFreeAsync(keys[i], s); cudaFreeAsync(lvls[i], s); }
    cudaFreeAsync(n_cells, s);
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
        wire_expand_kernel<WireCount><<<wire_blocks(n_in * kWideEntries), kWireTB, 0, s>>>(
            t.wide, nodes[cur], n_in, d, t.wide_p, INT_MAX, nodes[cur ^ 1], n_next, WireCount{hist});
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
