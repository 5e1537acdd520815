// vr_wire_walk.cuh -- the level-by-level walk of the wide tables that yields every cell of the octree with its table
// entry, level and integer corner.  Shared by the grid wireframe (vr_wire.cu) and the leaf-neighbour table (vr_tv.cu).
#pragma once
#include <cooperative_groups.h>

#include <algorithm>

#include "vr_types.h"
#include "vr_wire.h"

namespace vrb {

constexpr int kWireTB = 256;

// A node the expansion visits: its table id and its integer corner on the grid of its own depth.
struct WireNode {
    uint32_t table, x, y, z;
};

// One slot per calling thread from a global counter, one atomic per group of converged threads.
template <class T>
__device__ __forceinline__ T wire_claim(T* ctr) {
    namespace cg = cooperative_groups;
    cg::coalesced_group grp = cg::coalesced_threads();
    T base = 0;
    if (grp.thread_rank() == 0) base = atomicAdd(ctr, (T)grp.size());
    return grp.shfl(base, 0) + (T)grp.thread_rank();
}

// The count sink: leaves and internal cells by level into hist (2 * kWireLevels counters).
struct WireCount {
    static constexpr bool kCount = true;
    unsigned long long* hist;
};

// One thread per entry of every table in `in` (nodes of depth d).  An entry resolves kWideLv levels below its node:
// at sub-level k it lies in the cell of level d + k + 1 whose node has depth d + k.  That cell ends the walk when it
// is a leaf or when d + k >= max_depth; it is then emitted by the first of the 8^(kWideLv-1-k) entries it covers:
// count sink (WireCount), tallied in hist; any other sink, sink(table, entry, level L, x, y, z) with (x, y, z) the
// cell's corner on the 2^L grid (the entry's leaf slot, when the cell is a leaf, is the slot map's
// table * kWideEntries + entry).  An entry that never ends is the table id of a node of depth d + kWideLv, which joins
// the next frontier.  The root table of wide_p = v sits at depth -v; its first v levels are the virtual root's
// octant 0, so only entries with zero virtual bits are real.
template <class Sink>
__global__ void __launch_bounds__(kWireTB) wire_expand_kernel(const uint32_t* __restrict__ wide,
                                                              const WireNode* __restrict__ in, long long n_in, int d,
                                                              int v, int max_depth, WireNode* __restrict__ next,
                                                              unsigned int* __restrict__ n_next, Sink sink) {
    constexpr int LV = kWideLv;
    constexpr uint32_t M = (1u << LV) - 1u;
    constexpr bool kCount = Sink::kCount;
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
                    if constexpr (kCount) {
                        atomicAdd(&tally[dn + 1], 1u);
                    } else {
                        sink(F.table, e, dn + 1, (F.x << (k + 1)) | (ex >> sh), (F.y << (k + 1)) | (ey >> sh),
                             (F.z << (k + 1)) | (ez >> sh));
                    }
                }
                inner = false;
                break;
            }
            if (kCount && first) atomicAdd(&tally[kWireLevels + dn + 1], 1u);
        }
        if (inner) {
            const unsigned int s = wire_claim(n_next);
            next[s] = WireNode{w, (F.x << LV) | ex, (F.y << LV) | ey, (F.z << LV) | ez};
        }
    }
    if constexpr (kCount) {
        __syncthreads();
        for (int i = threadIdx.x; i < 2 * kWireLevels; i += blockDim.x)
            if (tally[i]) atomicAdd(sink.hist + i, (unsigned long long)tally[i]);
    }
}

inline unsigned int wire_blocks(long long threads) { return (unsigned int)((threads + kWireTB - 1) / kWireTB); }

// The walk from the root down to the nodes of depth mm (lv: the tree's counts, wire_levels), calling `sink` for every
// cell it ends at: the leaves down to level mm + 1 and the internal cells of that level.  Stream-ordered; the frontiers
// come from the stream-ordered allocator.  *launches counts the kernels it ran.
template <class Sink>
cudaError_t wire_walk(const WireTree& t, const WireLevels& lv, int mm, const Sink& sink, cudaStream_t s,
                      int* launches) {
    long long cap = 1;   // frontier size: the most nodes of any depth the walk visits
    for (int l = 1; l <= mm; ++l) cap = std::max(cap, lv.inner[l]);
    WireNode* nodes[2] = {nullptr, nullptr};
    unsigned int* n_next = nullptr;
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < 2 && e == cudaSuccess; ++i) e = cudaMallocAsync((void**)&nodes[i], (size_t)cap * sizeof(WireNode), s);
    if (e == cudaSuccess) e = cudaMallocAsync((void**)&n_next, sizeof(unsigned int), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(nodes[0], 0, sizeof(WireNode), s);   // the root: table 0, corner 0
    long long n_in = 1;
    int cur = 0;
    for (int d = -t.wide_p; e == cudaSuccess; d += kWideLv) {
        if (d > 0) {
            if (d > mm) break;
            n_in = lv.inner[d];
            if (n_in == 0) break;
        }
        e = cudaMemsetAsync(n_next, 0, sizeof(unsigned int), s);
        if (e != cudaSuccess) break;
        wire_expand_kernel<Sink><<<wire_blocks(n_in * kWideEntries), kWireTB, 0, s>>>(
            t.wide, nodes[cur], n_in, d, t.wide_p, mm, nodes[cur ^ 1], n_next, sink);
        e = cudaGetLastError();
        ++*launches;
        cur ^= 1;
    }
    for (int i = 0; i < 2; ++i) cudaFreeAsync(nodes[i], s);
    cudaFreeAsync(n_next, s);
    return e;
}

}  // namespace vrb
