// vr_query.cu -- point queries of a device tree: the leaf a world point falls in (query_single_from_root,
// n3tree_query.hpp:13-48), its data row, cube size and in-cell coordinates (vr_tree_query), and its colour along a
// direction as the probe disc shows it (vr_tree_eval, volrend.cu:111-128).
//
// One persistent grid-stride kernel per call.  A warp owns runs of kGroups groups of 32 consecutive points; lane l
// takes point l of each group, so a thread's points are 32 apart and a warp's 32 points of one group are adjacent.
//   descent   descend_wide (vr_probe.h), restarted at the deepest table the thread's previous point also went
//             through: the tables of a descent are kept in shared memory, and the first position bit in which the
//             two points differ bounds how far down the old path is still valid.
//   records   read like the march reads them (load_rec: plain read-only loads).
//   rows      a data row is 3*B+1 halves (98 bytes for SH16, 26 for SH4): the warp stages its 32 rows in shared
//             memory and writes them as one contiguous span of 16-byte stores.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "vr_lumisphere.cuh"
#include "vr_probe.h"
#include "vr_query.h"

namespace vrb {
namespace {

constexpr int kQBlock = 128, kQWarps = kQBlock / 32;
constexpr int kQSteps = 24 / kWideLv;   // table fetches on the deepest root-to-leaf path
constexpr int kGroups = 8;              // 32-point groups per warp run

__device__ __forceinline__ uint32_t rec_half(const uint32_t* w, int c) { return (w[c >> 1] >> (16 * (c & 1))) & 0xffffu; }

template <int KBD, bool EVAL>
__global__ void __launch_bounds__(kQBlock) query_kernel(const QueryLaunch Q) {
    constexpr int kRow = 3 * BasisCount<KBD>::n + 1;   // halves of a data row
    constexpr int kStage = EVAL ? 8 : ((32 * kRow + 7) / 8) * 8;
    __shared__ uint32_t s_tab[kQSteps][kQBlock];
    __shared__ __align__(16) unsigned short s_row[kQWarps][kStage];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool need_rec = EVAL ? Q.rgb != nullptr : (Q.data != nullptr || Q.coef != nullptr);
    const bool row16 = !EVAL && ((reinterpret_cast<uintptr_t>(Q.data) & 15u) == 0);
    const long long n_runs = ((Q.n + 31) / 32 + kGroups - 1) / kGroups;
    for (long long run = (long long)blockIdx.x * kQWarps + warp; run < n_runs; run += (long long)gridDim.x * kQWarps) {
        uint32_t pu[3] = {0u, 0u, 0u};
        int pstep = -1;   // leaf step of this thread's previous point (-1: none)
        for (int g = 0; g < kGroups; ++g) {
            const long long p0 = (run * kGroups + g) * 32;
            if (p0 >= Q.n) break;
            const long long i = p0 + lane;
            const bool live = i < Q.n;
            uint32_t rw[RecWords<KBD>::n];
            uint32_t wl = 0;
            if (live) {
                float p[3];
                uint32_t u[3];
                if (Q.xyz) probe_position(Q.tree, Q.xyz[3 * i], Q.xyz[3 * i + 1], Q.xyz[3 * i + 2], p, u);
                else probe_position(Q.tree, Q.point[0], Q.point[1], Q.point[2], p, u);
                // the table of step k is selected by position bits 23 .. 24 - kWideLv*k: it is the previous point's
                // table while no bit from there up differs
                int j = 0;
                if (pstep >= 0) {
                    const uint32_t diff = (u[0] ^ pu[0]) | (u[1] ^ pu[1]) | (u[2] ^ pu[2]);
                    j = min((__clz(diff) - 8) / kWideLv, pstep);
                }
                const uint32_t T = j > 0 ? s_tab[j][threadIdx.x] : 0u;
                const uint32_t e = descend_wide(Q.tree, u, j, T, wl, &s_tab[0][threadIdx.x], kQBlock);
                pu[0] = u[0]; pu[1] = u[1]; pu[2] = u[2];
                pstep = j;
                if (need_rec) load_rec<KBD>(rec_addr(Q.tree.wrecs, e, RecBytes<KBD>::n), rw);
                if constexpr (EVAL) {
                    if (Q.sigma) Q.sigma[i] = __half2float(__ushort_as_half((unsigned short)(wl & 0xffffu)));
                    if (Q.rgb) {
                        float out[3];
                        lumisphere_rgb<KBD>(Q.tree, Q.dir[3 * i], Q.dir[3 * i + 1], Q.dir[3 * i + 2], Q.bmin, Q.bmax,
                                            [&](int k) { return __half2float(__ushort_as_half((unsigned short)rec_half(rw, k))); },
                                            out);
                        Q.rgb[3 * i] = out[0]; Q.rgb[3 * i + 1] = out[1]; Q.rgb[3 * i + 2] = out[2];
                    }
                } else {
                    // leaf word bits 23..30 = 103 + leaf depth + wide_p; cube_sz = 2^depth
                    const float cube = __uint_as_float((wl & 0x7f800000u) + ((uint32_t)(24 - Q.tree.wide_p) << 23));
                    if (Q.cube) Q.cube[i] = cube;
                    if (Q.local) {
#pragma unroll
                        for (int k = 0; k < 3; ++k) {   // frac(p * 2^depth): exact, as the reference's per-level x*N - floor
                            const float t = __fmul_rn(p[k], cube);
                            Q.local[3 * i + k] = __fsub_rn(t, floorf(t));
                        }
                    }
                    if (Q.coef)
#pragma unroll
                        for (int k = 0; k < kRow - 1; ++k)
                            if (k < Q.n_coef) Q.coef[i * Q.n_coef + k] = __half2float(__ushort_as_half((unsigned short)rec_half(rw, k)));
                    if (Q.data) {
                        unsigned short* r = &s_row[warp][lane * kRow];
#pragma unroll
                        for (int k = 0; k < kRow - 1; ++k) r[k] = (unsigned short)rec_half(rw, k);
                        r[kRow - 1] = (unsigned short)(wl & 0xffffu);
                    }
                }
            }
            if constexpr (!EVAL) {
                if (Q.data) {
                    __syncwarp();
                    const long long live_n = Q.n - p0 < 32 ? Q.n - p0 : 32;
                    uint16_t* dst = Q.data + (size_t)p0 * kRow;
                    if (live_n == 32 && row16) {   // 32 * kRow halves = 4 * kRow 16-byte chunks, 16-byte aligned
                        const uint4* src = reinterpret_cast<const uint4*>(s_row[warp]);
                        for (int c = lane; c < 4 * kRow; c += 32) reinterpret_cast<uint4*>(dst)[c] = src[c];
                    } else {
                        for (int c = lane; c < live_n * kRow; c += 32) dst[c] = s_row[warp][c];
                    }
                    __syncwarp();
                }
            }
        }
    }
}

template <int KBD, bool EVAL>
cudaError_t launch(const QueryLaunch& Q, int num_sms, cudaStream_t stream) {
    int per_sm = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, query_kernel<KBD, EVAL>, kQBlock, 0);
    if (e != cudaSuccess) return e;
    const long long runs = ((Q.n + 31) / 32 + kGroups - 1) / kGroups;
    long long grid = (long long)(per_sm > 0 ? per_sm : 1) * num_sms;
    const long long need = (runs + kQWarps - 1) / kQWarps;
    if (grid > need) grid = need;
    query_kernel<KBD, EVAL><<<(unsigned)grid, kQBlock, 0, stream>>>(Q);
    return cudaGetLastError();
}

template <bool EVAL>
cudaError_t dispatch(const QueryLaunch& Q, int kbd, int num_sms, cudaStream_t stream) {
    switch (kbd) {
        case -1: return launch<-1, EVAL>(Q, num_sms, stream);
        case 1: return launch<1, EVAL>(Q, num_sms, stream);
        case 4: return launch<4, EVAL>(Q, num_sms, stream);
        case 9: return launch<9, EVAL>(Q, num_sms, stream);
        case 16: return launch<16, EVAL>(Q, num_sms, stream);
        case 25: return launch<25, EVAL>(Q, num_sms, stream);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace

cudaError_t query_launch(const QueryLaunch& Q, int kbd, bool eval, int num_sms, cudaStream_t stream) {
    return eval ? dispatch<true>(Q, kbd, num_sms, stream) : dispatch<false>(Q, kbd, num_sms, stream);
}

}  // namespace vrb
