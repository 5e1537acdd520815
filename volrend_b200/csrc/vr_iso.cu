// vr_iso.cu -- marching cubes over the leaf sigma of a device tree (vr_tree_isosurface).  DESIGN.md section 23 states
// the definition bit for bit; the triangle table is generated (vr_iso_table.h, tools/gen_iso_table.py).
//
// The lattice is (R + 2)^3 points, R = 2^L, stored padded: index g = i + 1 along each axis, so that padding sits at
// g = 0 and g = R + 1.  It is processed in slabs of S x-planes, so that scratch stays bounded at L = 11.  A slab owns
// the vertices of planes [g0, g0 + S) and the cubes whose lower corner lies there; its last cubes read vertex ids of
// plane g0 + S, whose x-edges look at plane g0 + S + 1, so the slab holds sigma for S + 2 planes (the last two are
// carried over to the next slab by a copy instead of sampled again) and scans vertex counts over S + 1 planes.
//   sample    one thread per run of kRun consecutive points of a z-row: descend_wide, restarted at the deepest table
//             the previous point of the run also went through (as query_kernel restarts)
//   classify  per point its crossing edges (bit d: the edge along axis d to the next point crosses) and, per cube, its
//             case and triangle count
//   scan      CUB exclusive sums of the vertex and triangle counts; the running totals of the slabs before stay on the
//             device and are added by the emit kernels
//   emit      each vertex from the thread of its owner point, each face from the thread of its cube: every output
//             element has exactly one writer, so the mesh is bit-reproducible
// The colour pass (iso_color) runs after the normals: it descends again from the root to the inside endpoint, whose
// lattice index the fill leaves in the vertex's colour slots.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cub/device/device_scan.cuh>

#include "vr_iso.h"
#include "vr_iso_table.h"
#include "vr_lumisphere.cuh"
#include "vr_probe.h"

namespace vrb {
namespace {

constexpr int kIsoBlock = 256;
constexpr int kRun = 16;                      // points per sampling thread
constexpr int kSteps = 24 / kWideLv;          // table fetches on the deepest root-to-leaf path
constexpr long long kSlabPoints = 1ll << 25;  // scratch budget: points of the S + 2 sigma planes of a slab

struct Slab {
    int R, n1;            // cells per axis, points per axis (R + 2)
    long long P;          // points per plane
    int g0;               // global plane of slab plane 0
    int S;                // owned planes
};

// The leaf sigma as the lattice reads it: NaN -> 0, +-inf -> +-65504.
__device__ __forceinline__ float lattice_sigma(uint32_t wl) {
    const float s = __half2float(__ushort_as_half((unsigned short)(wl & 0xffffu)));
    return s != s ? 0.f : fminf(fmaxf(s, -65504.f), 65504.f);
}

__global__ void __launch_bounds__(kIsoBlock) iso_sample_kernel(const TreeDev tree, const Slab sl, int rel_lo, int rel_hi,
                                                               int sh, float* __restrict__ sig) {
    __shared__ uint32_t s_tab[kSteps][kIsoBlock];
    const int chunks = (sl.R + kRun - 1) / kRun;
    const long long per_plane = (long long)sl.n1 * chunks;
    const long long item = (long long)blockIdx.x * kIsoBlock + threadIdx.x;
    if (item >= (long long)(rel_hi - rel_lo) * per_plane) return;
    const int rel = rel_lo + (int)(item / per_plane);
    const long long rem = item % per_plane;
    const int h = (int)(rem / chunks), ch = (int)(rem % chunks);
    const int g = sl.g0 + rel;
    float* row = sig + rel * sl.P + (long long)h * sl.n1;
    const int l0 = 1 + ch * kRun, l1 = min(sl.R, ch * kRun + kRun);   // interior points l0 .. l1
    if (ch == 0) row[0] = 0.f;
    if (l1 == sl.R) row[sl.R + 1] = 0.f;
    if (g == 0 || g > sl.R || h == 0 || h > sl.R) {
        for (int l = l0; l <= l1; ++l) row[l] = 0.f;
        return;
    }
    uint32_t u[3], pu[3] = {0u, 0u, 0u};
    u[0] = (uint32_t)(2 * g - 1) << sh;
    u[1] = (uint32_t)(2 * h - 1) << sh;
    int pstep = -1;
    for (int l = l0; l <= l1; ++l) {
        u[2] = (uint32_t)(2 * l - 1) << sh;
        int j = 0;
        if (pstep >= 0) {
            const uint32_t diff = (u[0] ^ pu[0]) | (u[1] ^ pu[1]) | (u[2] ^ pu[2]);
            j = min((__clz(diff) - 8) / kWideLv, pstep);
        }
        const uint32_t T = j > 0 ? s_tab[j][threadIdx.x] : 0u;
        uint32_t wl = 0;
        descend_wide(tree, u, j, T, wl, &s_tab[0][threadIdx.x], kIsoBlock);
        pu[0] = u[0]; pu[1] = u[1]; pu[2] = u[2];
        pstep = j;
        row[l] = lattice_sigma(wl);
    }
}

__global__ void __launch_bounds__(kIsoBlock) iso_classify_kernel(const Slab sl, float level, const float* __restrict__ sig,
                                                                 uint32_t* __restrict__ vcnt, uint8_t* __restrict__ vmask,
                                                                 uint32_t* __restrict__ tcnt, uint8_t* __restrict__ tcase) {
    const long long p = (long long)blockIdx.x * kIsoBlock + threadIdx.x;
    if (p >= (long long)(sl.S + 1) * sl.P) return;
    const int rel = (int)(p / sl.P);
    const long long rem = p % sl.P;
    const int h = (int)(rem / sl.n1), l = (int)(rem % sl.n1);
    const int g = sl.g0 + rel, last = sl.R + 1;
    uint32_t m = 0;
    if (g <= last) {
        const bool in0 = sig[p] > level;
        if (g < last && (sig[p + sl.P] > level) != in0) m |= 1u;
        if (h < last && (sig[p + sl.n1] > level) != in0) m |= 2u;
        if (l < last && (sig[p + 1] > level) != in0) m |= 4u;
    }
    vcnt[p] = __popc(m);
    vmask[p] = (uint8_t)m;
    if (rel < sl.S) {
        uint32_t c = 0;
        if (g < last && h < last && l < last) {
#pragma unroll
            for (int k = 0; k < 8; ++k)
                c |= (uint32_t)(sig[p + (k & 1) * sl.P + ((k >> 1) & 1) * sl.n1 + ((k >> 2) & 1)] > level) << k;
        }
        tcnt[p] = kIsoTriCount[c];
        tcase[p] = (uint8_t)c;
    }
}

__global__ void __launch_bounds__(kIsoBlock) iso_vert_kernel(const Slab sl, float level, float3 off, float3 scale,
                                                             bool color, const float* __restrict__ sig,
                                                             const uint32_t* __restrict__ vexcl,
                                                             const uint8_t* __restrict__ vmask,
                                                             const unsigned long long* __restrict__ base,
                                                             float* __restrict__ vert) {
    const long long p = (long long)blockIdx.x * kIsoBlock + threadIdx.x;
    if (p >= (long long)sl.S * sl.P) return;
    const uint32_t m = vmask[p];
    if (!m) return;
    const long long rem = p % sl.P;
    const int a[3] = {sl.g0 + (int)(p / sl.P) - 1, (int)(rem / sl.n1) - 1, (int)(rem % sl.n1) - 1};   // lattice index
    const long long stride[3] = {sl.P, sl.n1, 1};
    const float o[3] = {off.x, off.y, off.z}, sc[3] = {scale.x, scale.y, scale.z};
    const float fR = (float)sl.R;
    unsigned long long v = base[0] + vexcl[p];
    const float sa = sig[p];
    for (int d = 0; d < 3; ++d) {
        if (!((m >> d) & 1u)) continue;
        const float sb = sig[p + stride[d]];
        const float t = __fdiv_rn(__fsub_rn(level, sa), __fsub_rn(sb, sa));
        float* out = vert + 9 * v;
#pragma unroll
        for (int e = 0; e < 3; ++e) {
            float c = __fadd_rn((float)a[e], 0.5f);
            if (e == d) c = __fadd_rn(c, t);
            out[e] = __fdiv_rn(__fsub_rn(__fdiv_rn(c, fR), o[e]), sc[e]);
        }
        if (color) {   // the inside endpoint, read back by iso_color
            const bool a_in = sa > level;
#pragma unroll
            for (int e = 0; e < 3; ++e) out[3 + e] = __int_as_float(a[e] + (!a_in && e == d ? 1 : 0));
        } else {
            out[3] = 1.f; out[4] = 1.f; out[5] = 1.f;
        }
        out[6] = 0.f; out[7] = 0.f; out[8] = 0.f;
        ++v;
    }
}

__global__ void __launch_bounds__(kIsoBlock) iso_face_kernel(const Slab sl, const uint32_t* __restrict__ vexcl,
                                                             const uint8_t* __restrict__ vmask,
                                                             const uint32_t* __restrict__ tcnt,
                                                             const uint32_t* __restrict__ texcl,
                                                             const uint8_t* __restrict__ tcase,
                                                             const unsigned long long* __restrict__ base,
                                                             uint32_t* __restrict__ faces) {
    const long long p = (long long)blockIdx.x * kIsoBlock + threadIdx.x;
    if (p >= (long long)sl.S * sl.P) return;
    const uint32_t n = tcnt[p];
    if (!n) return;
    const int c = tcase[p];
    const unsigned long long f0 = base[1] + texcl[p];
    const uint32_t v0 = (uint32_t)base[0];
    for (uint32_t t = 0; t < n; ++t)
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int e = kIsoTris[c][3 * t + k], cn = kIsoEdgeCorner[e], d = e >> 2;
            const long long q = p + (cn & 1) * sl.P + ((cn >> 1) & 1) * sl.n1 + ((cn >> 2) & 1);
            faces[3 * (f0 + t) + k] = v0 + vexcl[q] + __popc(vmask[q] & ((1u << d) - 1u));
        }
}

// running totals: + the vertices of the S owned planes and the triangles of their cubes
__global__ void iso_advance_kernel(const Slab sl, const uint32_t* __restrict__ vexcl, const uint32_t* __restrict__ tcnt,
                                   const uint32_t* __restrict__ texcl, unsigned long long* base) {
    const long long n = (long long)sl.S * sl.P;
    base[0] += vexcl[n];
    base[1] += (unsigned long long)texcl[n - 1] + tcnt[n - 1];
}

template <int KBD>
__global__ void __launch_bounds__(kIsoBlock) iso_color_kernel(const TreeDev tree, int sh, float* __restrict__ vert,
                                                              long long n, int bmin, int bmax) {
    const long long i = (long long)blockIdx.x * kIsoBlock + threadIdx.x;
    if (i >= n) return;
    float* v = vert + 9 * i;
    uint32_t u[3];
#pragma unroll
    for (int e = 0; e < 3; ++e) u[e] = (2u * (uint32_t)__float_as_int(v[3 + e]) + 1u) << sh;
    int j = 0;
    uint32_t wl = 0;
    const uint32_t idx = descend_wide(tree, u, j, 0u, wl, nullptr, 0);
    uint32_t rw[RecWords<KBD>::n];
    load_rec<KBD>(rec_addr(tree.wrecs, idx, RecBytes<KBD>::n), rw);
    float out[3];
    lumisphere_rgb<KBD>(tree, -v[6], -v[7], -v[8], bmin, bmax,
                        [&](int k) { return __half2float(__ushort_as_half((unsigned short)((rw[k >> 1] >> (16 * (k & 1))) & 0xffffu))); },
                        out);
    v[3] = out[0]; v[4] = out[1]; v[5] = out[2];
}

unsigned grid_of(long long n) { return (unsigned)((n + kIsoBlock - 1) / kIsoBlock); }

}  // namespace

cudaError_t iso_run(const IsoArgs& a, bool fill, cudaStream_t s, long long* n_verts, long long* n_faces, int* launches) {
    Slab sl{};
    sl.R = 1 << a.depth;
    sl.n1 = sl.R + 2;
    sl.P = (long long)sl.n1 * sl.n1;
    int S = a.slab_planes > 0 ? a.slab_planes : (int)(kSlabPoints / sl.P) - 2;
    S = max(2, min(S, sl.n1));
    const int sh = 23 - a.depth - a.tree.wide_p;
    const long long nv = (long long)(S + 1) * sl.P, nt = (long long)S * sl.P;
    size_t scan_bytes = 0;
    cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, nv, s);
    if (e != cudaSuccess) return e;
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t o_sig = 0, o_vcnt = o_sig + al((S + 2) * sl.P * 4), o_vexcl = o_vcnt + al(nv * 4),
                 o_vmask = o_vexcl + al(nv * 4), o_tcnt = o_vmask + al(nv), o_texcl = o_tcnt + al(nt * 4),
                 o_tcase = o_texcl + al(nt * 4), o_base = o_tcase + al(nt), o_tmp = o_base + 256,
                 bytes = o_tmp + al(scan_bytes);
    unsigned char* scratch = nullptr;
    if ((e = cudaMallocAsync((void**)&scratch, bytes, s)) != cudaSuccess) return e;
    float* sig = reinterpret_cast<float*>(scratch + o_sig);
    uint32_t* vcnt = reinterpret_cast<uint32_t*>(scratch + o_vcnt);
    uint32_t* vexcl = reinterpret_cast<uint32_t*>(scratch + o_vexcl);
    uint8_t* vmask = scratch + o_vmask;
    uint32_t* tcnt = reinterpret_cast<uint32_t*>(scratch + o_tcnt);
    uint32_t* texcl = reinterpret_cast<uint32_t*>(scratch + o_texcl);
    uint8_t* tcase = scratch + o_tcase;
    unsigned long long* base = reinterpret_cast<unsigned long long*>(scratch + o_base);
    void* tmp = scratch + o_tmp;
    auto done = [&](cudaError_t err) {
        const cudaError_t e2 = cudaFreeAsync(scratch, s);
        return err != cudaSuccess ? err : e2;
    };
    int n_launch = 0;
    if ((e = cudaMemsetAsync(base, 0, 2 * sizeof(unsigned long long), s)) != cudaSuccess) return done(e);
    const float3 off = make_float3(a.tree.offset[0], a.tree.offset[1], a.tree.offset[2]);
    const float3 scale = make_float3(a.tree.scale[0], a.tree.scale[1], a.tree.scale[2]);
    const long long chunks = (sl.R + kRun - 1) / kRun;
    for (int g0 = 0; g0 < sl.n1; g0 += S) {
        const int prev_S = sl.S;
        sl.g0 = g0;
        sl.S = min(S, sl.n1 - g0);
        int rel_lo = 0;
        if (g0 > 0) {   // planes g0, g0 + 1 were the previous slab's planes S, S + 1
            if ((e = cudaMemcpyAsync(sig, sig + prev_S * sl.P, 2 * sl.P * sizeof(float), cudaMemcpyDeviceToDevice, s)) !=
                cudaSuccess)
                return done(e);
            rel_lo = 2;
        }
        const int rel_hi = sl.S + 2;
        iso_sample_kernel<<<grid_of((rel_hi - rel_lo) * sl.n1 * chunks), kIsoBlock, 0, s>>>(a.tree, sl, rel_lo, rel_hi,
                                                                                            sh, sig);
        iso_classify_kernel<<<grid_of((long long)(sl.S + 1) * sl.P), kIsoBlock, 0, s>>>(sl, a.level, sig, vcnt, vmask,
                                                                                         tcnt, tcase);
        if ((e = cudaGetLastError()) != cudaSuccess) return done(e);
        const long long snv = (long long)(sl.S + 1) * sl.P, snt = (long long)sl.S * sl.P;
        if ((e = cub::DeviceScan::ExclusiveSum(tmp, scan_bytes, vcnt, vexcl, snv, s)) != cudaSuccess ||
            (e = cub::DeviceScan::ExclusiveSum(tmp, scan_bytes, tcnt, texcl, snt, s)) != cudaSuccess)
            return done(e);
        n_launch += 4;
        if (fill) {
            iso_vert_kernel<<<grid_of(snt), kIsoBlock, 0, s>>>(sl, a.level, off, scale, a.color, sig, vexcl, vmask,
                                                               base, a.vert);
            iso_face_kernel<<<grid_of(snt), kIsoBlock, 0, s>>>(sl, vexcl, vmask, tcnt, texcl, tcase, base, a.faces);
            n_launch += 2;
        }
        iso_advance_kernel<<<1, 1, 0, s>>>(sl, vexcl, tcnt, texcl, base);
        n_launch += 1;
        if ((e = cudaGetLastError()) != cudaSuccess) return done(e);
    }
    *launches += n_launch;
    if (!fill) {
        unsigned long long h[2] = {0, 0};
        if ((e = cudaMemcpyAsync(h, base, sizeof(h), cudaMemcpyDeviceToHost, s)) != cudaSuccess) return done(e);
        if ((e = done(cudaSuccess)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(s)) != cudaSuccess) return e;
        *n_verts = (long long)h[0];
        *n_faces = (long long)h[1];
        return cudaSuccess;
    }
    return done(cudaSuccess);
}

cudaError_t iso_color(const TreeDev& tree, int depth, float* vert, long long n, int32_t bmin, int32_t bmax,
                      cudaStream_t s, int* launches) {
    if (n == 0) return cudaSuccess;
    const int sh = 23 - depth - tree.wide_p;
    switch (tree.kbd) {
        case -1: iso_color_kernel<-1><<<grid_of(n), kIsoBlock, 0, s>>>(tree, sh, vert, n, bmin, bmax); break;
        case 1: iso_color_kernel<1><<<grid_of(n), kIsoBlock, 0, s>>>(tree, sh, vert, n, bmin, bmax); break;
        case 4: iso_color_kernel<4><<<grid_of(n), kIsoBlock, 0, s>>>(tree, sh, vert, n, bmin, bmax); break;
        case 9: iso_color_kernel<9><<<grid_of(n), kIsoBlock, 0, s>>>(tree, sh, vert, n, bmin, bmax); break;
        case 16: iso_color_kernel<16><<<grid_of(n), kIsoBlock, 0, s>>>(tree, sh, vert, n, bmin, bmax); break;
        case 25: iso_color_kernel<25><<<grid_of(n), kIsoBlock, 0, s>>>(tree, sh, vert, n, bmin, bmax); break;
        default: return cudaErrorInvalidValue;
    }
    *launches += 1;
    return cudaGetLastError();
}

}  // namespace vrb
