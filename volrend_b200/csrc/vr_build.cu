// vr_build.cu -- build the canonical N3Tree of a set of voxel cells (vr_tree_build).  DESIGN.md section 21 states the
// definition; the stages are:
//   sort       the key of a cell is the Morton code of its min corner at level 23 (69 bits, x the most significant bit
//              of each triple), then its level: 74 bits, sorted as two stable CUB radix passes (low 64 bits, then the
//              high 10).  A containing cell sorts right before the cells it contains, so a duplicate or overlap always
//              shows up as a cell that contains its sorted successor.
//   merge      (VR_BUILD_MERGE) all-+0 rows are dropped (an unlisted slot holds +0 too), then level by level from 23
//              up to 2 each complete group of 8 sibling cells with bitwise-equal rows becomes its parent cell.  A cell's
//              `span` is the number of array positions it covers once its absorbed descendants are skipped, so a group
//              is walked without compacting the array between levels.  Each pass reads and writes only inside the
//              parent regions its threads own, so no result depends on thread order.
//   count      cell s starts the nodes of levels c+1 .. L_s-1, where c is the deepest level at which its min corner
//              shares a cell with its predecessor's (c = -1 for the first cell: it starts the root); an inclusive
//              scan gives the node count, which the host reads back (the one synchronisation).
//   number     every (level, starting cell) pair is emitted in cell order and stably sorted by level: breadth-first
//              order with the nodes of a level in Morton order.  A node's parent is the last node of the level above
//              whose starting cell is at or before its own (binary search); the node's octant comes from its code.
//   scatter    the outputs are zeroed, then each link and each listed row is written by exactly one thread.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "vr_build.h"

namespace vrb {
namespace {

constexpr int kTB = 256;
constexpr int kDeep = kBuildMaxLevel;
using u128 = unsigned __int128;

// the low 21 bits of v spread to every third bit
__host__ __device__ __forceinline__ uint64_t part3(uint64_t v) {
    v &= 0x1fffffull;
    v = (v | v << 32) & 0x1f00000000ffffull;
    v = (v | v << 16) & 0x1f0000ff0000ffull;
    v = (v | v << 8) & 0x100f00f00f00f00full;
    v = (v | v << 4) & 0x10c30c30c30c30c3ull;
    v = (v | v << 2) & 0x1249249249249249ull;
    return v;
}

// Morton code (69 bits) of the level-23 point (x, y, z), x the most significant bit of each triple
__host__ __device__ __forceinline__ u128 morton(uint32_t x, uint32_t y, uint32_t z) {
    const uint64_t lo = part3(x) << 2 | part3(y) << 1 | part3(z);
    const uint64_t hi = part3(x >> 21) << 2 | part3(y >> 21) << 1 | part3(z >> 21);
    return (u128)hi << 63 | lo;
}

// deepest level (0..23) at which the two codes lie in one cell
__device__ __forceinline__ int common_level(uint64_t alo, uint8_t ahi, uint64_t blo, uint8_t bhi) {
    const uint64_t xh = (uint64_t)(ahi ^ bhi), xl = alo ^ blo;
    if (!xh && !xl) return kDeep;
    const int lz = xh ? __clzll((long long)xh) - 59 : 5 + __clzll((long long)xl);   // leading zeros of 69 bits
    return lz / 3;
}

__device__ __forceinline__ int octant(uint64_t lo, uint8_t hi, int level) {
    const u128 c = (u128)hi << 64 | lo;
    return (int)(c >> (3 * (kDeep - level))) & 7;
}

// The level-23 corner of cell c; an invalid cell sets kBuildBadCell in *bad (when given) and reads as (1, 0, 0, 0)
__device__ __forceinline__ u128 cell_code(const int32_t* __restrict__ cells, long long c, int* level, int* bad) {
    const int32_t* v = cells + 4 * c;
    const int L = v[0], x = v[1], y = v[2], z = v[3];
    const bool ok = L >= 1 && L <= kDeep && x >= 0 && y >= 0 && z >= 0 && x < (1 << L) && y < (1 << L) && z < (1 << L);
    if (!ok) {
        if (bad) atomicOr(bad, 1 << kBuildBadCell);
        *level = 1;
        return 0;
    }
    const int sh = kDeep - L;
    *level = L;
    return morton((uint32_t)x << sh, (uint32_t)y << sh, (uint32_t)z << sh);
}

// Cells in sorted order (struct of arrays)
struct Cells {
    uint64_t* lo;    // Morton code, low 64 bits
    uint8_t* hi;     // Morton code, high 5 bits
    uint8_t* lvl;
    uint32_t* src;   // input index: the cell's row
};

__global__ void __launch_bounds__(kTB) key_lo_kernel(const int32_t* __restrict__ cells, long long n,
                                                     uint64_t* __restrict__ key, uint32_t* __restrict__ idx,
                                                     int* __restrict__ bad) {
    const long long t = (long long)blockIdx.x * kTB + threadIdx.x;
    if (t >= n) return;
    int L;
    const u128 c = cell_code(cells, t, &L, bad);
    key[t] = (uint64_t)(c << 5) | (uint64_t)L;
    idx[t] = (uint32_t)t;
}

__global__ void __launch_bounds__(kTB) key_hi_kernel(const int32_t* __restrict__ cells, long long n,
                                                     const uint32_t* __restrict__ idx, uint32_t* __restrict__ key) {
    const long long t = (long long)blockIdx.x * kTB + threadIdx.x;
    if (t >= n) return;
    int L;
    key[t] = (uint32_t)(cell_code(cells, idx[t], &L, nullptr) >> 59);   // bits 64..73 of code << 5 | level
}

// The sorted cells; the live count (*m) is n; with `flag`, flag[t] = 1 unless the row is all +0 bits
__global__ void __launch_bounds__(kTB) sorted_kernel(const int32_t* __restrict__ cells, const uint16_t* __restrict__ rows,
                                                     long long n, int dd, const uint32_t* __restrict__ perm, Cells out,
                                                     uint32_t* __restrict__ flag, uint32_t* __restrict__ m) {
    const long long t = (long long)blockIdx.x * kTB + threadIdx.x;
    if (t >= n) return;
    if (t == 0) *m = (uint32_t)n;
    const uint32_t c = perm[t];
    int L;
    const u128 code = cell_code(cells, c, &L, nullptr);
    out.lo[t] = (uint64_t)code;
    out.hi[t] = (uint8_t)(code >> 64);
    out.lvl[t] = (uint8_t)L;
    out.src[t] = c;
    if (flag) {
        const uint16_t* r = rows + (size_t)c * dd;
        uint32_t any = 0;
        for (int j = 0; j < dd; ++j) any |= r[j];
        flag[t] = any != 0;
    }
}

// a cell that contains its sorted successor (duplicates included)
__global__ void __launch_bounds__(kTB) overlap_kernel(Cells c, long long n, int* __restrict__ bad) {
    const long long t = (long long)blockIdx.x * kTB + threadIdx.x + 1;
    if (t >= n) return;
    const int la = c.lvl[t - 1];
    if (la <= c.lvl[t] && common_level(c.lo[t - 1], c.hi[t - 1], c.lo[t], c.hi[t]) >= la)
        atomicOr(bad, 1 << kBuildOverlap);
}

// compaction: the flagged cells of `in`, in order, to `out` (excl: exclusive sum of the flags); *m = their number;
// spans start at 1
__global__ void __launch_bounds__(kTB) compact_kernel(Cells in, long long n, const uint32_t* __restrict__ flag,
                                                      const uint32_t* __restrict__ excl, Cells out,
                                                      uint32_t* __restrict__ span, uint32_t* __restrict__ m) {
    const long long t = (long long)blockIdx.x * kTB + threadIdx.x;
    if (t >= n) return;
    if (t == n - 1) *m = excl[t] + flag[t];
    if (!flag[t]) return;
    const uint32_t d = excl[t];
    out.lo[d] = in.lo[t];
    out.hi[d] = in.hi[t];
    out.lvl[d] = in.lvl[t];
    out.src[d] = in.src[t];
    if (span) span[d] = 1;
}

__device__ __forceinline__ bool rows_equal(const uint16_t* __restrict__ rows, int dd, uint32_t a, uint32_t b) {
    const uint16_t* ra = rows + (size_t)a * dd;
    const uint16_t* rb = rows + (size_t)b * dd;
    for (int j = 0; j < dd; ++j)
        if (ra[j] != rb[j]) return false;
    return true;
}

// One level of the merge: a level-L cell of octant 0 whose 7 successors (skipping absorbed cells) are its level-L
// siblings with its row becomes their parent; the siblings are marked dead.  A thread reads the level and span of a
// cell only once the cell is known to lie in its own parent region, which no other thread of the pass writes.
__global__ void __launch_bounds__(kTB) merge_kernel(Cells c, long long n, const uint32_t* __restrict__ m_dev, int L,
                                                    const uint16_t* __restrict__ rows, int dd,
                                                    uint32_t* __restrict__ span, uint8_t* __restrict__ dead) {
    const long long t = (long long)blockIdx.x * kTB + threadIdx.x;
    const uint32_t m = *m_dev;
    if (t >= n || t >= m || c.lvl[t] != L) return;
    const uint64_t lo = c.lo[t];
    const uint8_t hi = c.hi[t];
    if (octant(lo, hi, L) != 0) return;
    uint32_t total = 0;
    long long u = t;
    for (int j = 0; j < 8; ++j) {
        if (u >= m || common_level(lo, hi, c.lo[u], c.hi[u]) < L - 1 || c.lvl[u] != L ||
            octant(c.lo[u], c.hi[u], L) != j || (j > 0 && !rows_equal(rows, dd, c.src[t], c.src[u])))
            return;
        total += span[u];
        u += span[u];
    }
    for (long long v = t + span[t], j = 1; j < 8; ++j) {
        dead[v] = 1;
        v += span[v];
    }
    span[t] = total;
    c.lvl[t] = (uint8_t)(L - 1);
}

__global__ void __launch_bounds__(kTB) live_kernel(long long n, const uint32_t* __restrict__ m_dev,
                                                   const uint8_t* __restrict__ dead, uint32_t* __restrict__ flag) {
    const long long t = (long long)blockIdx.x * kTB + threadIdx.x;
    if (t < n) flag[t] = t < *m_dev && !dead[t];
}

__device__ __forceinline__ int first_level(Cells c, long long t) {
    return t == 0 ? -1 : common_level(c.lo[t - 1], c.hi[t - 1], c.lo[t], c.hi[t]);
}

// nodes started by each cell (0 past the live count)
__global__ void __launch_bounds__(kTB) count_kernel(Cells c, long long n, const uint32_t* __restrict__ m_dev,
                                                    unsigned long long* __restrict__ k) {
    const long long t = (long long)blockIdx.x * kTB + threadIdx.x;
    if (t >= n) return;
    k[t] = t < *m_dev ? (unsigned long long)max(0, (int)c.lvl[t] - 1 - first_level(c, t)) : 0ull;
}

__global__ void __launch_bounds__(kTB) emit_kernel(Cells c, long long m, const unsigned long long* __restrict__ k,
                                                   const unsigned long long* __restrict__ incl,
                                                   uint8_t* __restrict__ rec_lvl, uint32_t* __restrict__ rec_cell) {
    const long long t = (long long)blockIdx.x * kTB + threadIdx.x;
    if (t >= m) return;
    const int n_start = (int)k[t], l0 = first_level(c, t) + 1;
    const unsigned long long o = incl[t] - n_start;
    for (int j = 0; j < n_start; ++j) {
        rec_lvl[o + j] = (uint8_t)(l0 + j);
        rec_cell[o + j] = (uint32_t)t;
    }
}

// base[l] = first node of level l (l = 0 .. 24) in the level-sorted records
__global__ void bases_kernel(const uint8_t* __restrict__ rec_lvl, uint32_t N, uint32_t* __restrict__ base) {
    const int l = threadIdx.x;
    if (l > kDeep + 1) return;
    uint32_t a = 0, b = N;
    while (a < b) {
        const uint32_t mid = (a + b) / 2;
        if (rec_lvl[mid] < l) a = mid + 1;
        else b = mid;
    }
    base[l] = a;
}

// the node of level l whose region holds sorted cell s: the last one started at or before s
__device__ __forceinline__ uint32_t node_at(const uint32_t* __restrict__ base, const uint32_t* __restrict__ rec_cell,
                                            int l, uint32_t s) {
    uint32_t a = base[l], b = base[l + 1];
    while (a < b) {
        const uint32_t mid = (a + b) / 2;
        if (rec_cell[mid] <= s) a = mid + 1;
        else b = mid;
    }
    return a - 1;
}

__global__ void __launch_bounds__(kTB) link_kernel(Cells c, uint32_t N, const uint8_t* __restrict__ rec_lvl,
                                                   const uint32_t* __restrict__ rec_cell, const uint32_t* __restrict__ base,
                                                   int32_t* __restrict__ child) {
    const uint32_t i = blockIdx.x * kTB + threadIdx.x + 1;
    if (i >= N) return;
    const int l = rec_lvl[i];
    const uint32_t s = rec_cell[i];
    const uint32_t p = node_at(base, rec_cell, l - 1, s);
    child[(size_t)p * 8 + octant(c.lo[s], c.hi[s], l)] = (int32_t)(i - p);
}

__global__ void __launch_bounds__(kTB) leaf_kernel(Cells c, long long m, const uint32_t* __restrict__ rec_cell,
                                                   const uint32_t* __restrict__ base, unsigned long long* __restrict__ dst) {
    const long long t = (long long)blockIdx.x * kTB + threadIdx.x;
    if (t >= m) return;
    const int L = c.lvl[t];
    dst[t] = (unsigned long long)node_at(base, rec_cell, L - 1, (uint32_t)t) * 8 + octant(c.lo[t], c.hi[t], L);
}

__global__ void __launch_bounds__(kTB) rows_kernel(const uint32_t* __restrict__ src, const unsigned long long* __restrict__ dst,
                                                   long long m, int dd, const uint16_t* __restrict__ rows,
                                                   uint16_t* __restrict__ data) {
    const long long total = m * dd;
    for (long long e = (long long)blockIdx.x * kTB + threadIdx.x; e < total; e += (long long)gridDim.x * kTB) {
        const long long t = e / dd;
        const int j = (int)(e - t * dd);
        data[dst[t] * dd + j] = rows[(size_t)src[t] * dd + j];
    }
}

unsigned int blocks_for(long long n) { return (unsigned int)std::max(1ll, (n + kTB - 1) / kTB); }

size_t align256(size_t b) { return (b + 255) / 256 * 256; }

// carves consecutive 256-byte-aligned arrays out of one allocation (base nullptr: only measures)
struct Carve {
    unsigned char* base;
    size_t off = 0;
    template <class T>
    T* take(size_t count) {
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += align256(count * sizeof(T));
        return p;
    }
    Cells cells(size_t n) { return Cells{take<uint64_t>(n), take<uint8_t>(n), take<uint8_t>(n), take<uint32_t>(n)}; }
};

}  // namespace

cudaError_t tree_build(const BuildArgs& a, cudaStream_t s, long long* n_nodes, int* reject, int* launches) {
    *reject = kBuildOk;
    *n_nodes = 0;
    const long long n = a.n;
    const int dd = a.data_dim;
    const bool write = a.child != nullptr;
    cudaError_t e;
    if (n == 0) {   // the root alone, with eight +0 leaves
        *n_nodes = 1;
        if (!write) return cudaSuccess;
        if (a.max_nodes < 1) { *reject = kBuildCapacity; return cudaSuccess; }
        if (((e = cudaMemsetAsync(a.child, 0, 8 * sizeof(int32_t), s)) != cudaSuccess ||
                      (e = cudaMemsetAsync(a.data, 0, (size_t)8 * dd * 2, s)) != cudaSuccess))
            return e;
        return cudaSuccess;
    }

    // ---- scratch of the cell stages: sort buffers, two cell sets, flags and scans, node counts
    const int ni = (int)n;
    size_t sort_bytes = 0, sort2_bytes = 0, scan_bytes = 0, scan64_bytes = 0;
    if ((e = cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (uint64_t*)nullptr, (uint64_t*)nullptr, (uint32_t*)nullptr,
                                             (uint32_t*)nullptr, ni, 0, 64, s)) != cudaSuccess ||
        (e = cub::DeviceRadixSort::SortPairs(nullptr, sort2_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                             (uint32_t*)nullptr, ni, 0, 10, s)) != cudaSuccess ||
        (e = cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, ni, s)) != cudaSuccess ||
        (e = cub::DeviceScan::InclusiveSum(nullptr, scan64_bytes, (unsigned long long*)nullptr,
                                           (unsigned long long*)nullptr, ni, s)) != cudaSuccess)
        return e;
    const size_t tmp_bytes = std::max({sort_bytes, sort2_bytes, scan_bytes, scan64_bytes});
    auto layout = [&](unsigned char* base, uint64_t** key, uint32_t** idx, Cells* c0, Cells* c1, uint32_t** flag,
                      uint32_t** excl, uint32_t** span, uint8_t** dead, unsigned long long** k,
                      unsigned long long** kin, int** bad, uint32_t** m, void** tmp) {
        Carve cv{base};
        key[0] = cv.take<uint64_t>(n); key[1] = cv.take<uint64_t>(n);
        idx[0] = cv.take<uint32_t>(n); idx[1] = cv.take<uint32_t>(n);
        *c0 = cv.cells(n);
        *c1 = a.merge ? cv.cells(n) : Cells{};
        *flag = a.merge ? cv.take<uint32_t>(n) : nullptr;
        *excl = a.merge ? cv.take<uint32_t>(n) : nullptr;
        *span = a.merge ? cv.take<uint32_t>(n) : nullptr;
        *dead = a.merge ? cv.take<uint8_t>(n) : nullptr;
        *k = cv.take<unsigned long long>(n);
        *kin = cv.take<unsigned long long>(n);
        *bad = cv.take<int>(1);
        *m = cv.take<uint32_t>(1);
        *tmp = cv.take<unsigned char>(tmp_bytes);
        return cv.off;
    };
    uint64_t* key[2];
    uint32_t *idx[2], *flag, *excl, *span, *m_dev;
    Cells c0, c1;
    uint8_t* dead;
    unsigned long long *k, *kin;
    int* bad;
    void* tmp;
    const size_t bytes1 = layout(nullptr, key, idx, &c0, &c1, &flag, &excl, &span, &dead, &k, &kin, &bad, &m_dev, &tmp);
    unsigned char* s1 = nullptr;
    if ((e = cudaMallocAsync((void**)&s1, bytes1, s)) != cudaSuccess) return e;
    layout(s1, key, idx, &c0, &c1, &flag, &excl, &span, &dead, &k, &kin, &bad, &m_dev, &tmp);
    unsigned char* s2 = nullptr;
    auto done = [&](cudaError_t err) {
        if (s2) cudaFreeAsync(s2, s);
        const cudaError_t e2 = cudaFreeAsync(s1, s);
        return err != cudaSuccess ? err : e2;
    };
    auto launched = [&](int count) {
        *launches += count;
        return cudaGetLastError();
    };

    // ---- sort by (corner, level) and refuse invalid and overlapping cells
    const unsigned nb = blocks_for(n);
    if ((e = cudaMemsetAsync(bad, 0, sizeof(int), s)) != cudaSuccess) return done(e);
    key_lo_kernel<<<nb, kTB, 0, s>>>(a.cells, n, key[0], idx[0], bad);
    if ((e = launched(1)) != cudaSuccess) return done(e);
    {
        cub::DoubleBuffer<uint64_t> kb(key[0], key[1]);
        cub::DoubleBuffer<uint32_t> vb(idx[0], idx[1]);
        if ((e = cub::DeviceRadixSort::SortPairs(tmp, sort_bytes, kb, vb, ni, 0, 64, s)) != cudaSuccess) return done(e);
        // the high key bits into the (now free) key buffers, sorted stably after the low ones
        uint32_t* hk[2] = {reinterpret_cast<uint32_t*>(key[0]), reinterpret_cast<uint32_t*>(key[1])};
        uint32_t* perm = vb.Current();
        key_hi_kernel<<<nb, kTB, 0, s>>>(a.cells, n, perm, hk[0]);
        cub::DoubleBuffer<uint32_t> hb(hk[0], hk[1]);
        cub::DoubleBuffer<uint32_t> pb(perm, vb.Alternate());
        if ((e = launched(2)) != cudaSuccess ||
            (e = cub::DeviceRadixSort::SortPairs(tmp, sort2_bytes, hb, pb, ni, 0, 10, s)) != cudaSuccess)
            return done(e);
        ++*launches;
        sorted_kernel<<<nb, kTB, 0, s>>>(a.cells, a.rows, n, dd, pb.Current(), c0, flag, m_dev);
        overlap_kernel<<<nb, kTB, 0, s>>>(c0, n, bad);
        if ((e = launched(2)) != cudaSuccess) return done(e);
    }

    // ---- merge: drop all-+0 rows, collapse sibling groups level by level, keep the live cells
    if (a.merge) {
        if ((e = cub::DeviceScan::ExclusiveSum(tmp, scan_bytes, flag, excl, ni, s)) != cudaSuccess) return done(e);
        if ((e = cudaMemsetAsync(dead, 0, n, s)) != cudaSuccess) return done(e);
        compact_kernel<<<nb, kTB, 0, s>>>(c0, n, flag, excl, c1, span, m_dev);
        if ((e = launched(2)) != cudaSuccess) return done(e);
        for (int L = kDeep; L >= 2; --L) merge_kernel<<<nb, kTB, 0, s>>>(c1, n, m_dev, L, a.rows, dd, span, dead);
        live_kernel<<<nb, kTB, 0, s>>>(n, m_dev, dead, flag);
        if ((e = launched(kDeep)) != cudaSuccess ||
            (e = cub::DeviceScan::ExclusiveSum(tmp, scan_bytes, flag, excl, ni, s)) != cudaSuccess)
            return done(e);
        compact_kernel<<<nb, kTB, 0, s>>>(c1, n, flag, excl, c0, nullptr, m_dev);
        if ((e = launched(2)) != cudaSuccess) return done(e);
    }

    // ---- node count: the one synchronisation
    count_kernel<<<nb, kTB, 0, s>>>(c0, n, m_dev, k);
    if ((e = launched(1)) != cudaSuccess ||
        (e = cub::DeviceScan::InclusiveSum(tmp, scan64_bytes, k, kin, ni, s)) != cudaSuccess)
        return done(e);
    ++*launches;
    int host_bad = 0;
    uint32_t host_m = 0;
    unsigned long long host_nodes = 0;
    if ((e = cudaMemcpyAsync(&host_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, s)) != cudaSuccess ||
        (e = cudaMemcpyAsync(&host_m, m_dev, sizeof(uint32_t), cudaMemcpyDeviceToHost, s)) != cudaSuccess ||
        (e = cudaMemcpyAsync(&host_nodes, kin + n - 1, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s)) != cudaSuccess ||
        (e = cudaStreamSynchronize(s)) != cudaSuccess)
        return done(e);
    if (host_bad) {
        *reject = (host_bad & (1 << kBuildBadCell)) ? kBuildBadCell : kBuildOverlap;
        return done(cudaSuccess);
    }
    const long long m = host_m;
    const long long N = m > 0 ? (long long)host_nodes : 1;
    *n_nodes = N;
    if (N > a.node_limit) { *reject = kBuildTooLarge; return done(cudaSuccess); }
    if (!write) return done(cudaSuccess);
    if (N > a.max_nodes) { *reject = kBuildCapacity; return done(cudaSuccess); }

    // ---- outputs: zero, then number the nodes and scatter links and rows
    if ((e = cudaMemsetAsync(a.child, 0, (size_t)N * 8 * sizeof(int32_t), s)) != cudaSuccess ||
        (e = cudaMemsetAsync(a.data, 0, (size_t)N * 8 * dd * 2, s)) != cudaSuccess)
        return done(e);
    if (m == 0) return done(cudaSuccess);
    const int Ni = (int)N;
    size_t rec_sort_bytes = 0;
    if ((e = cub::DeviceRadixSort::SortPairs(nullptr, rec_sort_bytes, (uint8_t*)nullptr, (uint8_t*)nullptr,
                                             (uint32_t*)nullptr, (uint32_t*)nullptr, Ni, 0, 5, s)) != cudaSuccess)
        return done(e);
    Carve measure{nullptr};
    measure.take<uint8_t>(N); measure.take<uint8_t>(N); measure.take<uint32_t>(N); measure.take<uint32_t>(N);
    measure.take<uint32_t>(kDeep + 2); measure.take<unsigned char>(rec_sort_bytes);
    if ((e = cudaMallocAsync((void**)&s2, measure.off, s)) != cudaSuccess) return done(e);
    Carve cv{s2};
    uint8_t* rl[2] = {cv.take<uint8_t>(N), cv.take<uint8_t>(N)};
    uint32_t* rc[2] = {cv.take<uint32_t>(N), cv.take<uint32_t>(N)};
    uint32_t* base = cv.take<uint32_t>(kDeep + 2);
    void* rtmp = cv.take<unsigned char>(rec_sort_bytes);
    emit_kernel<<<blocks_for(m), kTB, 0, s>>>(c0, m, k, kin, rl[0], rc[0]);
    if ((e = launched(1)) != cudaSuccess) return done(e);
    cub::DoubleBuffer<uint8_t> lb(rl[0], rl[1]);
    cub::DoubleBuffer<uint32_t> cb(rc[0], rc[1]);
    if ((e = cub::DeviceRadixSort::SortPairs(rtmp, rec_sort_bytes, lb, cb, Ni, 0, 5, s)) != cudaSuccess) return done(e);
    bases_kernel<<<1, 32, 0, s>>>(lb.Current(), (uint32_t)N, base);
    if (N > 1) link_kernel<<<blocks_for(N - 1), kTB, 0, s>>>(c0, (uint32_t)N, lb.Current(), cb.Current(), base, a.child);
    unsigned long long* dst = k;   // the per-cell counts are consumed by emit_kernel
    leaf_kernel<<<blocks_for(m), kTB, 0, s>>>(c0, m, cb.Current(), base, dst);
    rows_kernel<<<(unsigned)std::min<long long>(blocks_for(m * dd), 1 << 20), kTB, 0, s>>>(c0.src, dst, m, dd, a.rows, a.data);
    return done(launched(4 + (N > 1)));
}

}  // namespace vrb
