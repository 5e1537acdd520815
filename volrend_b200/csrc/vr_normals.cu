// vr_normals.cu -- per-vertex normals of a triangle mesh: estimate_normals (reference src/mesh.cpp:63-97) on the
// device, bit for bit.  See DESIGN.md section 11.
//
// The reference adds each face's cross product into its three corners' vertices, serially in face order, starting
// from +0.f, then normalises.  A vertex's normal is therefore an ordered fp32 chain over its incident faces.  Here
// the corners are sorted by vertex with a stable radix sort (face order survives inside each vertex's segment), and
// one thread per vertex adds its segment in that order.  Parallelism is across vertices only: a vertex shared by
// many faces is a long serial chain, exactly as in the reference.  Every float operation is an explicitly rounded
// intrinsic, so nothing is contracted into an FMA (the reference is built for x86-64 without -march).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "vr_normals.h"
#include "vr_raster.h"

namespace vrb {
namespace {

constexpr int kTB = 256;

struct Cross {
    float x, y, z;
};

// mesh.cpp:82-86: a = v1 - v0, b = v2 - v0, cross(a, b) (_cross3, mesh.cpp:42-46)
__device__ __forceinline__ Cross face_cross(const float* __restrict__ vert, uint32_t i0, uint32_t i1, uint32_t i2) {
    const float* p0 = vert + 9 * (size_t)i0;
    const float* p1 = vert + 9 * (size_t)i1;
    const float* p2 = vert + 9 * (size_t)i2;
    float a[3], b[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const float o = __ldg(p0 + j);
        a[j] = __fsub_rn(__ldg(p1 + j), o);
        b[j] = __fsub_rn(__ldg(p2 + j), o);
    }
    return {__fsub_rn(__fmul_rn(a[1], b[2]), __fmul_rn(a[2], b[1])),
            __fsub_rn(__fmul_rn(a[2], b[0]), __fmul_rn(a[0], b[2])),
            __fsub_rn(__fmul_rn(a[0], b[1]), __fmul_rn(a[1], b[0]))};
}

// _normalize (mesh.cpp:48-61): sqrtf((x*x + y*y) + z*z), divide only when norm > 1e-6 (a double literal, so the
// comparison is in double).  A vertex without faces keeps 0, 0, 0.
__device__ __forceinline__ void store_normal(float* __restrict__ v, float x, float y, float z) {
    const float norm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
    if ((double)norm > 1e-6) {
        x = __fdiv_rn(x, norm);
        y = __fdiv_rn(y, norm);
        z = __fdiv_rn(z, norm);
    }
    v[6] = x;
    v[7] = y;
    v[8] = z;
}

// Triangle soup (no index buffer): vertex v is corner v % 3 of face v / 3, its only face, so its sum is the one
// term +0.f + cross.  Vertices past the last whole face (n_verts % 3 of them) get 0, 0, 0.  One thread per vertex.
__global__ void __launch_bounds__(kTB) soup_normals_kernel(float* __restrict__ vert, int n_verts, int n_faces) {
    const int v = blockIdx.x * kTB + threadIdx.x;
    if (v >= n_verts) return;
    const int f = v / 3;
    float x = 0.f, y = 0.f, z = 0.f;
    if (f < n_faces) {
        const Cross c = face_cross(vert, 3 * f, 3 * f + 1, 3 * f + 2);
        x = __fadd_rn(0.f, c.x);
        y = __fadd_rn(0.f, c.y);
        z = __fadd_rn(0.f, c.z);
    }
    store_normal(vert + 9 * (size_t)v, x, y, z);
}

// One thread per face: its cross product, and its three corners as (vertex, face) pairs for the sort.  A face with
// an index >= n_verts contributes nothing: its corners get the key n_verts, which sorts after every real vertex and
// is never counted.
__global__ void __launch_bounds__(kTB) face_corners_kernel(const float* __restrict__ vert, const uint32_t* __restrict__ faces,
                                                           int n_faces, uint32_t n_verts, Cross* __restrict__ cross,
                                                           uint32_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                           uint32_t* __restrict__ count) {
    const int f = blockIdx.x * kTB + threadIdx.x;
    if (f >= n_faces) return;
    const size_t c = 3 * (size_t)f;
    const uint32_t i0 = faces[c], i1 = faces[c + 1], i2 = faces[c + 2];
    const bool ok = i0 < n_verts && i1 < n_verts && i2 < n_verts;
    keys[c] = ok ? i0 : n_verts;
    keys[c + 1] = ok ? i1 : n_verts;
    keys[c + 2] = ok ? i2 : n_verts;
    vals[c] = vals[c + 1] = vals[c + 2] = (uint32_t)f;
    if (!ok) return;
    cross[f] = face_cross(vert, i0, i1, i2);
    // a repeated index is counted (and later added) once per corner, as the reference adds it
    atomicAdd(count + i0, 1u);
    atomicAdd(count + i1, 1u);
    atomicAdd(count + i2, 1u);
}

// One thread per vertex: the ordered sum over its sorted segment (incident faces in face order), then normalise.
__global__ void __launch_bounds__(kTB) vertex_normals_kernel(float* __restrict__ vert, int n_verts,
                                                             const uint32_t* __restrict__ offs,
                                                             const uint32_t* __restrict__ count,
                                                             const uint32_t* __restrict__ face_of,
                                                             const Cross* __restrict__ cross) {
    const int v = blockIdx.x * kTB + threadIdx.x;
    if (v >= n_verts) return;
    const uint32_t b = offs[v], e = b + count[v];
    float x = 0.f, y = 0.f, z = 0.f;   // +0.f, as mesh.cpp:68-70 zeroes it: +0.f + (-0.f) is +0.f
    for (uint32_t k = b; k < e; ++k) {
        const Cross c = cross[face_of[k]];
        x = __fadd_rn(x, c.x);
        y = __fadd_rn(y, c.y);
        z = __fadd_rn(z, c.z);
    }
    store_normal(vert + 9 * (size_t)v, x, y, z);
}

unsigned int blocks_for(long long n) { return (unsigned int)((n + kTB - 1) / kTB); }

size_t align256(size_t b) { return (b + 255) / 256 * 256; }

}  // namespace

cudaError_t normals_estimate(float* vert, long long n_verts, const uint32_t* faces, long long n_faces,
                             cudaStream_t s, int* launches) {
    if (n_verts <= 0) return cudaSuccess;
    const int V = (int)n_verts;
    if (!faces || n_faces == 0) {
        // mesh.cpp:65-66: without faces the vertices are a triangle soup; an empty index list here means no faces
        soup_normals_kernel<<<blocks_for(V), kTB, 0, s>>>(vert, V, faces ? 0 : V / 3);
        ++*launches;
        return cudaGetLastError();
    }
    const int F = (int)n_faces, C = 3 * F;
    // keys the sort needs: vertex ids 0 .. V-1 and the skipped-face key V
    const int key_bits = 32 - __builtin_clz((unsigned)V);
    size_t sort_bytes = 0, scan_bytes = 0;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                                    (uint32_t*)nullptr, (uint32_t*)nullptr, C, 0, key_bits, s);
    if (e == cudaSuccess)
        e = cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, V, s);
    if (e != cudaSuccess) return e;
    const size_t corners = align256((size_t)C * 4), verts = align256((size_t)V * 4);
    const size_t o_keys = 0, o_vals = 2 * corners, o_cross = 4 * corners;
    const size_t o_count = o_cross + align256((size_t)F * sizeof(Cross)), o_offs = o_count + verts;
    const size_t o_tmp = o_offs + verts, bytes = o_tmp + align256(std::max(sort_bytes, scan_bytes));
    cudaMemPool_t pool;
    if ((e = scratch_pool(&pool)) != cudaSuccess) return e;
    unsigned char* scratch = nullptr;
    if ((e = cudaMallocFromPoolAsync((void**)&scratch, bytes, pool, s)) != cudaSuccess) return e;
    uint32_t* keys[2] = {reinterpret_cast<uint32_t*>(scratch + o_keys), reinterpret_cast<uint32_t*>(scratch + o_keys + corners)};
    uint32_t* vals[2] = {reinterpret_cast<uint32_t*>(scratch + o_vals), reinterpret_cast<uint32_t*>(scratch + o_vals + corners)};
    Cross* cross = reinterpret_cast<Cross*>(scratch + o_cross);
    uint32_t* count = reinterpret_cast<uint32_t*>(scratch + o_count);
    uint32_t* offs = reinterpret_cast<uint32_t*>(scratch + o_offs);
    void* tmp = scratch + o_tmp;
    if ((e = cudaMemsetAsync(count, 0, (size_t)V * 4, s)) == cudaSuccess) {
        face_corners_kernel<<<blocks_for(F), kTB, 0, s>>>(vert, faces, F, (uint32_t)V, cross, keys[0], vals[0], count);
        ++*launches;
        e = cudaGetLastError();
    }
    // LSD radix sort is stable: each vertex's corners stay in face order
    if (e == cudaSuccess) {
        e = cub::DeviceRadixSort::SortPairs(tmp, sort_bytes, keys[0], keys[1], vals[0], vals[1], C, 0, key_bits, s);
        ++*launches;   // counted as one launch, whatever number of passes the sort takes
    }
    if (e == cudaSuccess) {
        e = cub::DeviceScan::ExclusiveSum(tmp, scan_bytes, count, offs, V, s);
        ++*launches;
    }
    if (e == cudaSuccess) {
        vertex_normals_kernel<<<blocks_for(V), kTB, 0, s>>>(vert, V, offs, count, vals[1], cross);
        ++*launches;
        e = cudaGetLastError();
    }
    const cudaError_t e2 = cudaFreeAsync(scratch, s);
    return e != cudaSuccess ? e : e2;
}

}  // namespace vrb
