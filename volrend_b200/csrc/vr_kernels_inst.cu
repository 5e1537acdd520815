// vr_kernels_inst.cu -- instantiates the march kernels for one basis size (-DVR_KBD=...).
// Compiled six times (RGBA, SH/SG/ASG 1, 4, 9, 16, 25) so the builds run in parallel.
//
// The two kernels:
//   variant 7          march_queue_kernel (vr_march_q.cuh): default for single-frame launches with 4, 9 or 16 basis
//                      functions (launch_renderer, the CLI), selectable for batches and for 25
//   variant 3 + 16*193 march_persistent_kernel with inline shading (vr_march.cuh): default for batches and for
//                      RGBA / 1 / 25 basis functions, and the A/B partner of the queue kernel in the parity tests
//                      and the bench
// Both also come as kOutViewOpts instantiations (plain and counting), which read each view's options from
// LaunchDev::opts: batches with options per view.  The VR_KBD=1 object also holds the weights pass
// (march_persistent_kernel<0, *, kOutWeights>, vr_tree_leaf_weights) and the error pass (<0, *, kOutError>,
// vr_tree_leaf_error), one kernel each for every basis size, and every object the gradient pass of its basis size
// (march_persistent_kernel<VR_KBD, false, kOutGrads>, vr_tree_leaf_grads).
#include <mutex>

#include "vr_kernels.h"
#include "vr_march_q.cuh"

#ifndef VR_KBD
#error "compile with -DVR_KBD=<-1|1|4|9|16|25>"
#endif

namespace vrb {

namespace {

// Resident CTAs of a persistent kernel, cached per (device, kernel, dynamic shared memory).
template <typename K>
int resident_ctas(K kernel, size_t smem, int num_sms) {
    struct Entry { int device; const void* fn; size_t smem; int per_sm; };
    static std::mutex mu;
    static Entry cache[32];
    static int n_cache = 0;
    int dev = 0;
    cudaGetDevice(&dev);
    const void* fn = reinterpret_cast<const void*>(kernel);
    std::lock_guard<std::mutex> lk(mu);
    for (int i = 0; i < n_cache; ++i)
        if (cache[i].device == dev && cache[i].fn == fn && cache[i].smem == smem) return cache[i].per_sm * num_sms;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kBlock, smem) != cudaSuccess || per_sm < 1) {
        cudaGetLastError();
        per_sm = 1;
    }
    if (n_cache < 32) cache[n_cache++] = Entry{dev, fn, smem, per_sm};
    return per_sm * num_sms;
}

// blocks: whether the kernel understands SM-local tile blocks (the product kernels do)
void set_work(LaunchDev& P, const LaunchCfg& cfg, bool blocks = true) {
    P.tiles_x = (P.w + kTW - 1) / kTW;
    P.tiles_y = (P.h + kTH - 1) / kTH;
    P.work_counter = cfg.work_counter;
    // Batches have the queue hand out blocks of 64 tiles, the warps of an SM sharing a block (vr_march.cuh next_item).
    // Up to 16 basis functions: 4x4 tiles of 4 consecutive views, view innermost, so that the colour records
    // neighbouring poses share are read from the SM's L1 instead of from L2 (DESIGN.md 4: modelled record L1 hit rate
    // 7 % -> 43 %; config 2 +0.2 to +4.8 % over three H100 sessions).  25 basis functions (160-byte records,
    // config 4): 8x8 tiles of one view, which measured 1-2 % faster there than the 4-view blocks.  A block needs
    // enough blocks per SM to balance (a block is ~20 us of an SM), so single frames and small batches keep one tile
    // per item.
    const int gs = P.tree.kbd == 25 ? 0 : 2, ws = P.tree.kbd == 25 ? 3 : 2;
    const int G = 1 << gs, bw = 1 << ws, bh = kBlkTiles / (G * bw);
    const long long bx = (P.tiles_x + bw - 1) / bw, by = (P.tiles_y + bh - 1) / bh, ng = (P.n_views + G - 1) / G;
    const long long nb = bx * by * ng;
    const bool want = P.n_views >= G && P.n_views >= 2 && nb >= 16LL * cfg.num_sms;
    if (blocks && want && nb * kBlkTiles <= 0x7fffffffLL) {
        P.blk_mode = 1; P.blocks_x = (int)bx; P.n_blocks = (int)nb;
        P.blk_gshift = gs; P.blk_wshift = ws; P.blk_groups = (int)ng;
        P.n_tiles = (int)(nb * kBlkTiles);   // item ids (block * 64 + index), incl. the tiles beyond the image edge
        set_div((uint32_t)bx, P.div_row_mul, P.div_row_shift);   // block -> (block row, view group) pair
        set_div((uint32_t)ng, P.div_view_mul, P.div_view_shift);
        return;
    }
    P.blk_mode = 0; P.blocks_x = 0; P.n_blocks = 0; P.blk_gshift = 0; P.blk_wshift = 0; P.blk_groups = 0;
    P.n_tiles = P.tiles_x * P.tiles_y * P.n_views;
    set_div((uint32_t)P.tiles_x, P.div_row_mul, P.div_row_shift);    // item -> (tile row, view) pair (decode_item)
    set_div((uint32_t)P.n_views, P.div_view_mul, P.div_view_shift);
}

template <typename K>
cudaError_t launch_persistent_grid(K kernel, size_t smem, LaunchDev& P, const LaunchCfg& cfg, bool blocks = true) {
    set_work(P, cfg, blocks);
    int grid = resident_ctas(kernel, smem, cfg.num_sms);
    const int need = (P.n_tiles + (kBlock / 32) - 1) / (kBlock / 32);
    if (grid > need) grid = need;
    if (grid < 1) grid = 1;
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(grid); lc.blockDim = dim3(kBlock); lc.dynamicSmemBytes = smem; lc.stream = cfg.stream;
    cudaLaunchAttribute attr[1];   // programmatic dependent launch: see pdl_wait_predecessor() in vr_march.cuh
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    lc.attrs = attr; lc.numAttrs = cfg.pdl ? 1 : 0;
    return cudaLaunchKernelEx(&lc, kernel, P);
}

template <int KBD, bool COUNT, int OUT>
cudaError_t launch_persistent(LaunchDev& P, const LaunchCfg& cfg) {
    const size_t smem = march_smem_bytes(P.tree.max_depth) + basis_smem_bytes<KBD>();
    return launch_persistent_grid(march_persistent_kernel<KBD, COUNT, OUT>, smem, P, cfg);
}

template <int KBD, bool COUNT, int OUT>
cudaError_t launch_queue(LaunchDev& P, const LaunchCfg& cfg) {
    if constexpr (KBD >= 4) {
        const size_t smem = queue_smem_bytes<KBD>(P.tree.max_depth);
        return launch_persistent_grid(march_queue_kernel<KBD, COUNT, OUT>, smem, P, cfg, false);   // tile queue only
    } else {
        return cudaErrorInvalidValue;
    }
}

}  // namespace

template <int KBD>
cudaError_t launch_march(LaunchDev& P, const LaunchCfg& cfg) {
    if (P.opts) {   // options per view (vr_render_batch_opts): no surface output
        if (cfg.surface) return cudaErrorInvalidValue;
        if (cfg.count)
            return cfg.queue ? launch_queue<KBD, true, kOutViewOpts>(P, cfg) : launch_persistent<KBD, true, kOutViewOpts>(P, cfg);
        return cfg.queue ? launch_queue<KBD, false, kOutViewOpts>(P, cfg) : launch_persistent<KBD, false, kOutViewOpts>(P, cfg);
    }
    if (cfg.surface) {  // drop-in launch_renderer path writing the caller's cudaArray
        return cfg.queue ? launch_queue<KBD, false, kOutSurface>(P, cfg) : launch_persistent<KBD, false, kOutSurface>(P, cfg);
    }
    if (cfg.count) {  // instrumented builds
        return cfg.queue ? launch_queue<KBD, true, kOutLinear>(P, cfg) : launch_persistent<KBD, true, kOutLinear>(P, cfg);
    }
    return cfg.queue ? launch_queue<KBD, false, kOutLinear>(P, cfg) : launch_persistent<KBD, false, kOutLinear>(P, cfg);
}

template cudaError_t launch_march<VR_KBD>(LaunchDev&, const LaunchCfg&);

// no parked ray constants: the gradient march keeps its ray in registers
template <int KBD>
cudaError_t launch_grads(LaunchDev& P, const LaunchCfg& cfg) {
    return launch_persistent_grid(march_persistent_kernel<KBD, false, kOutGrads>, march_smem_bytes(P.tree.max_depth), P, cfg);
}

template cudaError_t launch_grads<VR_KBD>(LaunchDev&, const LaunchCfg&);

#if VR_KBD == 1
// KBD 0: no basis set-up and no parked ray constants (the weights march reads no record)
cudaError_t launch_weights(LaunchDev& P, const LaunchCfg& cfg) {
    const size_t smem = march_smem_bytes(P.tree.max_depth);
    if (cfg.count) return launch_persistent_grid(march_persistent_kernel<0, true, kOutWeights>, smem, P, cfg);
    return launch_persistent_grid(march_persistent_kernel<0, false, kOutWeights>, smem, P, cfg);
}

cudaError_t launch_error(LaunchDev& P, const LaunchCfg& cfg) {
    const size_t smem = march_smem_bytes(P.tree.max_depth);
    if (cfg.count) return launch_persistent_grid(march_persistent_kernel<0, true, kOutError>, smem, P, cfg);
    return launch_persistent_grid(march_persistent_kernel<0, false, kOutError>, smem, P, cfg);
}
#endif

}  // namespace vrb
