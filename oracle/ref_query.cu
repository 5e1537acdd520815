// ref_query.cu -- C-ABI around the UNMODIFIED reference's query_single_from_root (test infrastructure).
//
// Built only where the reference sources exist (oracle/Makefile.query), into oracle/_ref/libref_query.so.  It
// includes the reference's own include/volrend/internal/n3tree_query.hpp and data_spec.hpp and loads trees with the
// reference's unchanged N3Tree loader (which uploads them); no reference source is copied.
//
//   ref_query_tree_open / _close -> N3Tree(path)
//   ref_query                    -> one thread per point: cen = offset + scale * xyz as retrieve_cursor_lumisphere_kernel
//                                   computes it (volrend.cu:180-182), then internal::query_single_from_root; copies
//                                   the data row the reference's `out` points at, cube_sz and the in-cell xyz back
#include <cstdint>
#include <string>

#include <cuda_fp16.h>

#include "volrend/internal/n3tree_query.hpp"
#include "volrend/n3tree.hpp"

using namespace volrend;

namespace {

__global__ void ref_query_kernel(internal::TreeSpec tree, const float* xyz, long long n, uint16_t* data, float* cube,
                                 float* local) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float cen[3];
    for (int k = 0; k < 3; ++k) cen[k] = tree.offset[k] + tree.scale[k] * xyz[3 * i + k];
    float cube_sz;
    const half* val;
    internal::query_single_from_root(tree, cen, &val, &cube_sz);
    const uint16_t* v = reinterpret_cast<const uint16_t*>(val);
    for (int c = 0; c < tree.data_dim; ++c) data[i * tree.data_dim + c] = v[c];
    cube[i] = cube_sz;
    for (int k = 0; k < 3; ++k) local[3 * i + k] = cen[k];
}

}  // namespace

extern "C" {

void* ref_query_tree_open(const char* npz_path) {
    N3Tree* t = new N3Tree(std::string(npz_path));
    if (!t->is_data_loaded()) { delete t; return nullptr; }
    return t;
}
void ref_query_tree_close(void* t) { delete static_cast<N3Tree*>(t); }
int ref_query_data_dim(void* t) { return static_cast<N3Tree*>(t)->data_dim; }

// n host points -> host outputs (data: n * data_dim halves).  *ms (if not NULL): device time of the kernel, averaged
// over `reps` launches (CUDA events).
int ref_query(void* tp, const float* xyz, long long n, uint16_t* data, float* cube, float* local, int reps, float* ms) {
    N3Tree& tree = *static_cast<N3Tree*>(tp);
    internal::TreeSpec spec(tree);
    const int dd = tree.data_dim;
    float *dx = nullptr, *dc = nullptr, *dl = nullptr;
    uint16_t* dd_ = nullptr;
    cudaMalloc(&dx, sizeof(float) * 3 * (size_t)(n ? n : 1));
    cudaMalloc(&dc, sizeof(float) * (size_t)(n ? n : 1));
    cudaMalloc(&dl, sizeof(float) * 3 * (size_t)(n ? n : 1));
    cudaMalloc(&dd_, sizeof(uint16_t) * (size_t)dd * (size_t)(n ? n : 1));
    cudaMemcpy(dx, xyz, sizeof(float) * 3 * (size_t)n, cudaMemcpyHostToDevice);
    const unsigned grid = (unsigned)((n + 255) / 256);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    if (n > 0) ref_query_kernel<<<grid, 256>>>(spec, dx, n, dd_, dc, dl);   // warm-up / result
    cudaEventRecord(e0);
    for (int r = 0; r < reps && n > 0; ++r) ref_query_kernel<<<grid, 256>>>(spec, dx, n, dd_, dc, dl);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    if (ms) {
        float t = 0.f;
        cudaEventElapsedTime(&t, e0, e1);
        *ms = reps > 0 ? t / reps : 0.f;
    }
    if (data) cudaMemcpy(data, dd_, sizeof(uint16_t) * (size_t)dd * (size_t)n, cudaMemcpyDeviceToHost);
    if (cube) cudaMemcpy(cube, dc, sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost);
    if (local) cudaMemcpy(local, dl, sizeof(float) * 3 * (size_t)n, cudaMemcpyDeviceToHost);
    const cudaError_t e = cudaGetLastError();
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaFree(dx); cudaFree(dc); cudaFree(dl); cudaFree(dd_);
    return e == cudaSuccess ? 0 : -(int)e;
}

}  // extern "C"
