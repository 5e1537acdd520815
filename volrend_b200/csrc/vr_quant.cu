// vr_quant.cu -- median-cut colour quantisation of a PlenOctree into the quant_colors / quant_map format the
// loader decodes (vr_tree_create_quantized).  See DESIGN.md section 12 for the contract these kernels implement.
//
// Stages (all sets at once; point p of the batch belongs to set p / M, its bucket is found from p % M):
//   kept      one thread per slot: sigma > thresh (compared as fp16) and the non-finite check of kept slots
//   compact   CUB exclusive sum of the kept flags; the kept count is read back (it sizes the scratch)
//   gather    one thread per slot: sigma / data_retained outputs and the struct-of-arrays point sets
//   levels    per level: segment bounding boxes (warp-segmented min/max + atomics), a 16-bit key per point
//             (the orderable fp16 value on its segment's widest axis), then a stable segmented sort by that key:
//             one CTA per segment ranking by counting when segments hold <= 512 points, else a two-pass LSD radix
//             sort over tiles of each segment (digit histograms, an exclusive sum, a stable scatter).
//             The contract splits a bucket after a STABLE SORT, and the sorted order of each child decides the
//             ties of every later level, so the split is a full stable segmented sort, not a select + partition.
//   finish    exact integer sums per bucket (two int64 halves, warp-segmented + atomics) and the map scatter,
//             then one thread per codebook row: f64 mean of the exact sum, rounded once to fp16.
// Bucket sizes depend only on M and the path (floor(n/2) to the even child), so a point's segment, and a segment's
// start, are found by walking bits down the levels: no offsets are stored or scanned.  Scratch comes from the
// device's default stream-ordered pool (cudaMallocAsync), which hands it back at the next synchronisation.
#include <cub/device/device_scan.cuh>
#include <cuda_fp16.h>

#include <algorithm>

#include "vr_quant.h"

namespace vrb {
namespace {

constexpr int kTB = 256;
constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ float h2f(uint16_t h) { return __half2float(__ushort_as_half(h)); }

// 16-bit key whose unsigned order is the fp16 order, with -0 folded onto +0 (no NaN reaches here)
__device__ __forceinline__ uint32_t okey(uint16_t h) {
    if (h == 0x8000u) h = 0;
    return (h & 0x8000u) ? (~h & 0xffffu) : (h | 0x8000u);
}
__device__ __forceinline__ uint16_t okey_inv(uint32_t k) {
    return (uint16_t)((k & 0x8000u) ? (k & 0x7fffu) : (~k & 0xffffu));
}

// the fp16 value as an exact integer multiple of 2^-24 (|m| < 2^40)
__device__ __forceinline__ long long mult24(uint16_t h) {
    const int e = (h >> 10) & 31, f = h & 1023;
    const long long m = e == 0 ? (long long)f : (long long)(1024 + f) << (e - 1);
    return (h & 0x8000u) ? -m : m;
}

// bucket of in-set position q after L levels of floor(n/2) / rest splits of M points; *n = its size
__device__ __forceinline__ uint32_t walk(uint32_t q, uint32_t M, int L, uint32_t* n_out) {
    uint32_t n = M, b = 0;
    for (int l = 0; l < L; ++l) {
        const uint32_t half = n >> 1;
        if (q >= half) { q -= half; n -= half; b = 2 * b + 1; }
        else { n = half; b = 2 * b; }
    }
    *n_out = n;
    return b;
}

// global segment (set << L | bucket) of batch position p
__device__ __forceinline__ uint32_t segment_of(uint32_t p, uint32_t M, int L, uint32_t* bucket = nullptr) {
    const uint32_t s = p / M;
    uint32_t n;
    const uint32_t b = walk(p - s * M, M, L, &n);
    if (bucket) *bucket = b;
    return (s << L) | b;
}

// Inclusive segmented scan over a warp whose lanes hold non-decreasing segment ids (positions are contiguous, so
// equal ids are one run); the last lane of each run ends up holding its run's total.
template <typename T, typename Op>
__device__ __forceinline__ void seg_scan(uint32_t seg, int lane, T& v, Op op) {
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const uint32_t os = __shfl_up_sync(kFull, seg, off);
        const T ov = __shfl_up_sync(kFull, v, off);
        if (lane >= off && os == seg) v = op(v, ov);
    }
}

__device__ __forceinline__ bool run_tail(uint32_t seg, int lane) {
    const uint32_t next = __shfl_down_sync(kFull, seg, 1);
    return lane == 31 || next != seg;
}

// kept flag per slot; flags a non-finite quantised coefficient of a kept slot
__global__ void __launch_bounds__(kTB) keep_kernel(const uint16_t* __restrict__ data, long long n_child, int dd,
                                                   int B, int retain, float thresh, uint32_t* __restrict__ flags,
                                                   int* __restrict__ bad) {
    const long long i = (long long)blockIdx.x * kTB + threadIdx.x;
    if (i >= n_child) return;
    const uint16_t* row = data + i * dd;
    const bool keep = h2f(row[dd - 1]) > thresh;   // NaN sigma is not kept
    flags[i] = keep;
    if (!keep) return;
    bool finite = true;
    for (int k = 0; k < 3; ++k)
        for (int j = retain; j < B; ++j) finite &= (row[k * B + j] & 0x7c00u) != 0x7c00u;
    if (!finite) *bad = 1;
}

// sigma / data_retained outputs for every slot, point sets (struct of arrays) and slot index for kept ones
__global__ void __launch_bounds__(kTB) gather_kernel(const uint16_t* __restrict__ data, long long n_child, int dd,
                                                     int B, int retain, const uint32_t* __restrict__ flags,
                                                     const uint32_t* __restrict__ pos, uint32_t M,
                                                     uint16_t* __restrict__ sigma, uint16_t* __restrict__ retained,
                                                     uint16_t* __restrict__ px, uint16_t* __restrict__ py,
                                                     uint16_t* __restrict__ pz, uint32_t* __restrict__ slot_of) {
    const long long i = (long long)blockIdx.x * kTB + threadIdx.x;
    if (i >= n_child) return;
    const uint16_t* row = data + i * dd;
    const bool keep = flags[i] != 0;
    sigma[i] = keep ? row[dd - 1] : (uint16_t)0;
    for (int j = 0; j < retain; ++j)
        for (int k = 0; k < 3; ++k) retained[((size_t)j * n_child + i) * 3 + k] = keep ? row[k * B + j] : (uint16_t)0;
    if (!keep) return;
    const uint32_t c = pos[i];
    slot_of[c] = (uint32_t)i;
    for (int j = retain; j < B; ++j) {
        const size_t o = (size_t)(j - retain) * M + c;
        px[o] = row[j];
        py[o] = row[B + j];
        pz[o] = row[2 * B + j];
    }
}

__global__ void __launch_bounds__(kTB) iota_kernel(uint32_t* __restrict__ v, uint32_t n) {
    const uint32_t p = blockIdx.x * kTB + threadIdx.x;
    if (p < n) v[p] = p;
}

// per-segment min / max of the three orderable keys
__global__ void __launch_bounds__(kTB) bbox_kernel(const uint32_t* __restrict__ vals, const uint16_t* __restrict__ px,
                                                   const uint16_t* __restrict__ py, const uint16_t* __restrict__ pz,
                                                   uint32_t NP, uint32_t M, int L, uint32_t* __restrict__ bmin,
                                                   uint32_t* __restrict__ bmax) {
    const uint32_t p = blockIdx.x * kTB + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const bool ok = p < NP;
    uint32_t seg = 0xffffffffu, k[3] = {0xffffu, 0xffffu, 0xffffu};
    if (ok) {
        seg = segment_of(p, M, L);
        const uint32_t g = vals[p];
        k[0] = okey(px[g]); k[1] = okey(py[g]); k[2] = okey(pz[g]);
    }
    // min and max of one axis packed as (min << 16 | 0xffff - max): both reduce with one unsigned min
    uint32_t mm[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) mm[a] = ok ? (k[a] << 16) | (0xffffu - k[a]) : kFull;
    auto vmin = [](uint32_t x, uint32_t y) { return min(x, y); };
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        // componentwise min of the two 16-bit halves
        uint32_t v = mm[a];
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const uint32_t os = __shfl_up_sync(kFull, seg, off);
            const uint32_t ov = __shfl_up_sync(kFull, v, off);
            if (lane >= off && os == seg) v = (vmin(v >> 16, ov >> 16) << 16) | vmin(v & 0xffffu, ov & 0xffffu);
        }
        mm[a] = v;
    }
    const bool tail = run_tail(seg, lane);
    if (ok && tail)
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            atomicMin(bmin + 3 * (size_t)seg + a, mm[a] >> 16);
            atomicMax(bmax + 3 * (size_t)seg + a, 0xffffu - (mm[a] & 0xffffu));
        }
}

// sort key of each point: the orderable value on its segment's widest axis
__global__ void __launch_bounds__(kTB) key_kernel(const uint32_t* __restrict__ vals, const uint16_t* __restrict__ px,
                                                  const uint16_t* __restrict__ py, const uint16_t* __restrict__ pz,
                                                  uint32_t NP, uint32_t M, int L, const uint32_t* __restrict__ bmin,
                                                  const uint32_t* __restrict__ bmax, uint16_t* __restrict__ keys) {
    const uint32_t p = blockIdx.x * kTB + threadIdx.x;
    if (p >= NP) return;
    const uint32_t seg = segment_of(p, M, L);
    int axis = 0;
    float best = 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float r = __fsub_rn(h2f(okey_inv(bmax[3 * (size_t)seg + a])), h2f(okey_inv(bmin[3 * (size_t)seg + a])));
        if (a == 0 || r > best) { best = r; axis = a; }   // ties keep the lowest axis
    }
    const uint32_t g = vals[p];
    const uint16_t v = axis == 0 ? px[g] : axis == 1 ? py[g] : pz[g];
    keys[p] = (uint16_t)okey(v);
}

// ---- stable segmented sort of (key, val) by the 16-bit key; segments are contiguous and in segment order.
// Segment `seg` (= set << L | bucket) starts at set * M + (offset of the bucket in its set), found by walking the
// bucket's bits; every segment of a level has floor or ceil of M / 2^L points.
__device__ __forceinline__ void segment_range(uint32_t seg, uint32_t M, int L, uint32_t* begin, uint32_t* n_out) {
    const uint32_t set = seg >> L, b = seg & ((1u << L) - 1u);
    uint32_t n = M, off = 0;
    for (int l = L - 1; l >= 0; --l) {
        const uint32_t half = n >> 1;
        if ((b >> l) & 1u) { off += half; n -= half; }
        else n = half;
    }
    *begin = set * M + off;
    *n_out = n;
}

// Small segments (at most kSmallSeg points): one CTA per segment; a point's destination is its stable rank,
// the number of points with a smaller key plus the number with an equal key before it.
constexpr int kSmallSeg = 512;
__global__ void __launch_bounds__(kTB) small_sort_kernel(const uint16_t* __restrict__ keys, const uint32_t* __restrict__ vin,
                                                         uint32_t* __restrict__ vout, uint32_t M, int L) {
    __shared__ uint16_t k[kSmallSeg];
    uint32_t begin, n;
    segment_range(blockIdx.x, M, L, &begin, &n);
    for (uint32_t i = threadIdx.x; i < n; i += kTB) k[i] = keys[begin + i];
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += kTB) {
        const uint16_t ki = k[i];
        uint32_t rank = 0;
        for (uint32_t j = 0; j < n; ++j) rank += (k[j] < ki) | ((k[j] == ki) & (j < i));
        vout[begin + rank] = vin[begin + i];
    }
}

// Large segments: LSD radix sort, two passes of 8-bit digits.  Each segment is cut into `tps` tiles of `tile`
// points (CTA = (segment, tile)).  A pass counts each tile's digits into hist[segment][digit][tile]; an exclusive
// sum over the whole array then gives, for each (segment, digit, tile), where its points go (segments are laid out
// in order, so the sum also carries each segment's start); the scatter places a tile's points chunk by chunk in
// position order, so equal digits keep their order and the pass is stable.
__global__ void __launch_bounds__(kTB) digit_hist_kernel(const uint16_t* __restrict__ keys, uint32_t M, int L,
                                                         uint32_t tile, uint32_t tps, int shift,
                                                         uint32_t* __restrict__ hist) {
    __shared__ uint32_t h[256];
    const uint32_t seg = blockIdx.x / tps, t = blockIdx.x - seg * tps;
    h[threadIdx.x] = 0;
    __syncthreads();
    uint32_t begin, n;
    segment_range(seg, M, L, &begin, &n);
    const uint32_t lo = min(t * tile, n), hi = min(lo + tile, n);
    for (uint32_t i = lo + threadIdx.x; i < hi; i += kTB) atomicAdd(&h[(keys[begin + i] >> shift) & 0xffu], 1u);
    __syncthreads();
    hist[((size_t)seg * 256 + threadIdx.x) * tps + t] = h[threadIdx.x];
}

__global__ void __launch_bounds__(kTB) digit_scatter_kernel(const uint16_t* __restrict__ kin, const uint32_t* __restrict__ vin,
                                                            uint16_t* __restrict__ kout, uint32_t* __restrict__ vout,
                                                            uint32_t M, int L, uint32_t tile, uint32_t tps, int shift,
                                                            const uint32_t* __restrict__ offs) {
    constexpr int kWarps = kTB / 32;
    __shared__ uint32_t next[256];          // destination of the next point of each digit
    __shared__ uint32_t wcnt[kWarps][256];  // this chunk's count of each digit per warp
    const uint32_t seg = blockIdx.x / tps, t = blockIdx.x - seg * tps;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    next[threadIdx.x] = offs[((size_t)seg * 256 + threadIdx.x) * tps + t];
    for (int i = 0; i < kWarps; ++i) wcnt[i][threadIdx.x] = 0;
    __syncthreads();
    uint32_t begin, n;
    segment_range(seg, M, L, &begin, &n);
    const uint32_t lo = min(t * tile, n), hi = min(lo + tile, n);
    for (uint32_t c = lo; c < hi; c += kTB) {
        const uint32_t i = c + threadIdx.x;
        const bool ok = i < hi;
        const uint16_t key = ok ? kin[begin + i] : (uint16_t)0;
        const uint32_t d = ok ? (key >> shift) & 0xffu : 0x100u;
        const unsigned peers = __match_any_sync(kFull, d);
        const uint32_t before = __popc(peers & ((1u << lane) - 1u));
        const bool leader = before == 0;
        if (ok && leader) wcnt[w][d] = __popc(peers);
        __syncthreads();
        if (ok) {
            uint32_t dst = next[d] + before;
            for (int v = 0; v < w; ++v) dst += wcnt[v][d];
            if (kout) kout[dst] = key;
            vout[dst] = vin[begin + i];
        }
        __syncthreads();
        if (ok && leader) {
            atomicAdd(&next[d], (uint32_t)__popc(peers));
            wcnt[w][d] = 0;
        }
        __syncthreads();
    }
}

// exact per-bucket sums (each 2^-24 multiple split as hi * 2^20 + lo, lo in [0, 2^20)) and the map scatter
__global__ void __launch_bounds__(kTB) finish_points_kernel(const uint32_t* __restrict__ vals,
                                                            const uint16_t* __restrict__ px, const uint16_t* __restrict__ py,
                                                            const uint16_t* __restrict__ pz, uint32_t NP, uint32_t M,
                                                            int bits, const uint32_t* __restrict__ slot_of,
                                                            long long n_child, uint16_t* __restrict__ qmap,
                                                            unsigned long long* __restrict__ acc) {
    const uint32_t p = blockIdx.x * kTB + threadIdx.x;
    const int lane = threadIdx.x & 31;
    const bool ok = p < NP;
    uint32_t seg = 0xffffffffu;
    long long s[6] = {0, 0, 0, 0, 0, 0};
    if (ok) {
        uint32_t b;
        seg = segment_of(p, M, bits, &b);
        const uint32_t g = vals[p];
        const uint32_t set = g / M;
        qmap[(size_t)set * n_child + slot_of[g - set * M]] = (uint16_t)b;
        const long long m[3] = {mult24(px[g]), mult24(py[g]), mult24(pz[g])};
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            s[a] = m[a] >> 20;
            s[3 + a] = m[a] & 0xfffff;
        }
    }
    auto add = [](long long x, long long y) { return x + y; };
#pragma unroll
    for (int a = 0; a < 6; ++a) seg_scan(seg, lane, s[a], add);
    const bool tail = run_tail(seg, lane);
    if (ok && tail)
#pragma unroll
        for (int a = 0; a < 6; ++a) atomicAdd(acc + 6 * (size_t)seg + a, (unsigned long long)s[a]);
}

// round-to-nearest-even conversion of a 128-bit integer to double
__device__ __forceinline__ double i128_to_f64_rn(__int128 v) {
    const bool neg = v < 0;
    const unsigned __int128 u = neg ? (unsigned __int128)0 - (unsigned __int128)v : (unsigned __int128)v;
    const unsigned long long hi = (unsigned long long)(u >> 64), lo = (unsigned long long)u;
    double d;
    if (hi == 0) {
        d = __ull2double_rn(lo);
    } else {
        // keep the top 64 bits, OR the shifted-out bits into the lowest one (below the rounding position)
        const int sh = 64 - __clzll((long long)hi);
        const unsigned long long top = (unsigned long long)(u >> sh) | ((lo << (64 - sh)) != 0ull);
        d = scalbn(__ull2double_rn(top), sh);
    }
    return neg ? -d : d;
}

// one thread per codebook row: mean = fp16_rn(f64_rn(S) / n * 2^-24); empty buckets and rows >= 2^bits are +0
__global__ void __launch_bounds__(kTB) codebook_kernel(const unsigned long long* __restrict__ acc, int n_quant, int bits,
                                                       uint32_t M, uint16_t* __restrict__ colors) {
    const uint32_t t = blockIdx.x * kTB + threadIdx.x;
    if (t >= (uint32_t)n_quant << 16) return;
    const uint32_t set = t >> 16, r = t & 0xffffu;
    uint16_t out[3] = {0, 0, 0};
    if (r < (1u << bits)) {
        uint32_t n = M;
        for (int l = bits - 1; l >= 0; --l) {
            const uint32_t half = n >> 1;
            n = ((r >> l) & 1u) ? n - half : half;
        }
        if (n > 0) {
            const unsigned long long* a = acc + 6 * (((size_t)set << bits) | r);
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const __int128 S = (__int128)(long long)a[k] * (1 << 20) + (__int128)(long long)a[3 + k];
                const double mean = __ddiv_rn(i128_to_f64_rn(S), (double)n) * 0x1p-24;
                out[k] = __half_as_ushort(__double2half(mean));
            }
        }
    }
    colors[3 * (size_t)t] = out[0];
    colors[3 * (size_t)t + 1] = out[1];
    colors[3 * (size_t)t + 2] = out[2];
}

unsigned int blocks_for(long long n) { return (unsigned int)((n + kTB - 1) / kTB); }

size_t align256(size_t b) { return (b + 255) / 256 * 256; }

// How a level's segments are sorted: one CTA per segment when they are small, else tiles of a radix pass.
struct SortPlan {
    bool small;
    uint32_t tile, tps;
    size_t n_hist;      // (segment, digit, tile) counters of one radix pass
};

SortPlan sort_plan(uint32_t M, int nq, int L) {
    const uint32_t n_max = (uint32_t)(((unsigned long long)M + (1ull << L) - 1) >> L);   // ceil(M / 2^L)
    SortPlan p{};
    p.small = n_max <= (uint32_t)kSmallSeg;
    if (!p.small) {
        p.tile = std::min<uint32_t>(4096u, (n_max + kTB - 1) / kTB * kTB);
        p.tps = (n_max + p.tile - 1) / p.tile;
        p.n_hist = ((size_t)nq << L) * 256 * p.tps;
    }
    return p;
}

}  // namespace

cudaError_t quant_compress(const QuantArgs& q, cudaStream_t s, long long* n_kept, int* reject, int* launches) {
    *n_kept = 0;
    *reject = kQuantOk;
    const int dd = q.data_dim, B = (dd - 1) / 3, nq = B - q.n_retain, bits = q.bits;
    const long long NC = q.n_child;
    cudaError_t e;

    // ---- kept flags, compaction, kept count (the one synchronisation)
    size_t scan_bytes = 0;
    if ((e = cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)std::max(NC, 1ll), s)) != cudaSuccess)
        return e;
    const size_t slots = align256((size_t)std::max(NC, 1ll) * 4);
    unsigned char* s1 = nullptr;
    if ((e = cudaMallocAsync((void**)&s1, 2 * slots + 256 + align256(scan_bytes), s)) != cudaSuccess) return e;
    uint32_t* flags = reinterpret_cast<uint32_t*>(s1);
    uint32_t* pos = reinterpret_cast<uint32_t*>(s1 + slots);
    int* bad = reinterpret_cast<int*>(s1 + 2 * slots);
    void* scan_tmp = s1 + 2 * slots + 256;
    unsigned char* s2 = nullptr;
    auto done = [&](cudaError_t err) {
        if (s2) cudaFreeAsync(s2, s);
        const cudaError_t e2 = cudaFreeAsync(s1, s);
        return err != cudaSuccess ? err : e2;
    };
    unsigned long long host_tail[2] = {0, 0};   // {last pos, last flag}
    int host_bad = 0;
    if (NC > 0) {
        if ((e = cudaMemsetAsync(bad, 0, sizeof(int), s)) != cudaSuccess) return done(e);
        keep_kernel<<<blocks_for(NC), kTB, 0, s>>>(q.data, NC, dd, B, q.n_retain, q.thresh, flags, bad);
        ++*launches;
        if ((e = cudaGetLastError()) != cudaSuccess) return done(e);
        if ((e = cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, flags, pos, (int)NC, s)) != cudaSuccess) return done(e);
        ++*launches;
        uint32_t tail[2];
        if ((e = cudaMemcpyAsync(&tail[0], pos + NC - 1, 4, cudaMemcpyDeviceToHost, s)) != cudaSuccess ||
            (e = cudaMemcpyAsync(&tail[1], flags + NC - 1, 4, cudaMemcpyDeviceToHost, s)) != cudaSuccess ||
            (e = cudaMemcpyAsync(&host_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, s)) != cudaSuccess ||
            (e = cudaStreamSynchronize(s)) != cudaSuccess)
            return done(e);
        host_tail[0] = tail[0];
        host_tail[1] = tail[1];
    }
    const unsigned long long kept = host_tail[0] + host_tail[1];
    *n_kept = (long long)kept;
    if (host_bad) {
        *reject = kQuantNonFinite;
        return done(cudaSuccess);
    }
    if ((unsigned long long)nq * kept > (unsigned long long)INT32_MAX) {
        *reject = kQuantTooManyPoints;
        return done(cudaSuccess);
    }
    const uint32_t M = (uint32_t)kept;
    const uint32_t NP = (uint32_t)nq * M;

    // ---- scratch sized by the kept count
    size_t n_hist = 0;
    for (int L = 0; L < bits; ++L) n_hist = std::max(n_hist, sort_plan(M, nq, L).n_hist);
    size_t hist_scan_bytes = 0;
    if (n_hist > 0 &&
        (e = cub::DeviceScan::ExclusiveSum(nullptr, hist_scan_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)n_hist, s)) != cudaSuccess)
        return done(e);
    const size_t np1 = std::max(NP, 1u), m1 = std::max(M, 1u);
    const size_t n_box = align256(((size_t)nq << std::max(bits - 1, 0)) * 3 * 4);
    const size_t o_px = 0, o_py = o_px + align256(np1 * 2), o_pz = o_py + align256(np1 * 2);
    const size_t o_slot = o_pz + align256(np1 * 2), o_v0 = o_slot + align256(m1 * 4), o_v1 = o_v0 + align256(np1 * 4);
    const size_t o_k0 = o_v1 + align256(np1 * 4), o_k1 = o_k0 + align256(np1 * 2), o_bmin = o_k1 + align256(np1 * 2);
    const size_t o_bmax = o_bmin + n_box, o_acc = o_bmax + n_box;
    const size_t n_acc = ((size_t)nq << bits) * 6 * 8;
    const size_t o_hist = o_acc + align256(n_acc), o_offs = o_hist + align256(n_hist * 4);
    const size_t o_tmp = o_offs + align256(n_hist * 4), bytes = o_tmp + align256(hist_scan_bytes);
    if ((e = cudaMallocAsync((void**)&s2, bytes, s)) != cudaSuccess) return done(e);
    uint16_t* px = reinterpret_cast<uint16_t*>(s2 + o_px);
    uint16_t* py = reinterpret_cast<uint16_t*>(s2 + o_py);
    uint16_t* pz = reinterpret_cast<uint16_t*>(s2 + o_pz);
    uint32_t* slot_of = reinterpret_cast<uint32_t*>(s2 + o_slot);
    uint32_t* vals = reinterpret_cast<uint32_t*>(s2 + o_v0);
    uint32_t* vtmp = reinterpret_cast<uint32_t*>(s2 + o_v1);
    uint16_t* keys = reinterpret_cast<uint16_t*>(s2 + o_k0);
    uint16_t* ktmp = reinterpret_cast<uint16_t*>(s2 + o_k1);
    uint32_t* bmin = reinterpret_cast<uint32_t*>(s2 + o_bmin);
    uint32_t* bmax = reinterpret_cast<uint32_t*>(s2 + o_bmax);
    unsigned long long* acc = reinterpret_cast<unsigned long long*>(s2 + o_acc);
    uint32_t* hist = reinterpret_cast<uint32_t*>(s2 + o_hist);
    uint32_t* offs = reinterpret_cast<uint32_t*>(s2 + o_offs);
    void* hist_tmp = s2 + o_tmp;

    if (NC > 0) {
        gather_kernel<<<blocks_for(NC), kTB, 0, s>>>(q.data, NC, dd, B, q.n_retain, flags, pos, M, q.sigma, q.retained,
                                                     px, py, pz, slot_of);
        ++*launches;
        if ((e = cudaGetLastError()) != cudaSuccess) return done(e);
    }

    // ---- median cut, one level of every set per iteration
    if (NP > 0) {
        iota_kernel<<<blocks_for(NP), kTB, 0, s>>>(vals, NP);
        ++*launches;
        if ((e = cudaGetLastError()) != cudaSuccess) return done(e);
    }
    for (int L = 0; L < bits && NP > 0; ++L) {
        const unsigned nseg = (unsigned)nq << L;
        const size_t segs3 = (size_t)nseg * 3 * 4;
        if ((e = cudaMemsetAsync(bmin, 0xff, segs3, s)) != cudaSuccess || (e = cudaMemsetAsync(bmax, 0, segs3, s)) != cudaSuccess)
            return done(e);
        bbox_kernel<<<blocks_for(NP), kTB, 0, s>>>(vals, px, py, pz, NP, M, L, bmin, bmax);
        key_kernel<<<blocks_for(NP), kTB, 0, s>>>(vals, px, py, pz, NP, M, L, bmin, bmax, keys);
        *launches += 2;
        if ((e = cudaGetLastError()) != cudaSuccess) return done(e);
        // stable sort of every segment by its key: equal values keep their current order
        const SortPlan p = sort_plan(M, nq, L);
        if (p.small) {
            small_sort_kernel<<<nseg, kTB, 0, s>>>(keys, vals, vtmp, M, L);
            ++*launches;
            std::swap(vals, vtmp);
        } else {
            // low digit: keys and vals to the spare buffers; high digit: vals back (keys are no longer needed)
            for (int pass = 0; pass < 2 && e == cudaSuccess; ++pass) {
                const int shift = 8 * pass;
                const uint16_t* kin = pass == 0 ? keys : ktmp;
                digit_hist_kernel<<<nseg * p.tps, kTB, 0, s>>>(kin, M, L, p.tile, p.tps, shift, hist);
                if ((e = cub::DeviceScan::ExclusiveSum(hist_tmp, hist_scan_bytes, hist, offs, (int)p.n_hist, s)) != cudaSuccess)
                    break;
                digit_scatter_kernel<<<nseg * p.tps, kTB, 0, s>>>(kin, pass == 0 ? vals : vtmp, pass == 0 ? ktmp : nullptr,
                                                                  pass == 0 ? vtmp : vals, M, L, p.tile, p.tps, shift, offs);
                *launches += 3;
            }
        }
        if (e != cudaSuccess || (e = cudaGetLastError()) != cudaSuccess) return done(e);
    }

    // ---- means and map
    if ((e = cudaMemsetAsync(q.qmap, 0, (size_t)nq * NC * 2, s)) != cudaSuccess ||
        (e = cudaMemsetAsync(acc, 0, n_acc, s)) != cudaSuccess)
        return done(e);
    if (NP > 0) {
        finish_points_kernel<<<blocks_for(NP), kTB, 0, s>>>(vals, px, py, pz, NP, M, bits, slot_of, NC, q.qmap, acc);
        ++*launches;
    }
    codebook_kernel<<<blocks_for((long long)nq << 16), kTB, 0, s>>>(acc, nq, bits, M, q.colors);
    ++*launches;
    if ((e = cudaGetLastError()) != cudaSuccess) return done(e);
    return done(cudaSuccess);
}

}  // namespace vrb
