// vr_types.h -- device-side parameter blocks shared by the C-ABI and the kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "volrend_b200.h"

namespace vrb {

// Leaf flag of a node word; the low 16 bits then hold sigma as fp16 bits.
constexpr uint32_t kLeafBit = 0x80000000u;
// Deepest leaf we accept: positions are 24-bit fixed point (fp32 mantissa).
constexpr int kMaxTreeDepth = 23;
// Octree levels resolved per table fetch: 64-entry tables.
constexpr int kWideLv = 2;
constexpr int kWideEntries = 1 << (3 * kWideLv);
// tables on a root-to-leaf path (the ancestor stack of the march kernels)
inline __host__ __device__ int wide_table_levels(int max_depth) { return (max_depth + kWideLv - 2) / kWideLv + 1; }

// Device copy of one N3Tree, re-laid-out at upload (vr_tree_create).
struct TreeDev {
    // two-levels-per-step view of the octree: one 64-entry table per internal node whose depth has
    // parity wide_p (plus the root); entry = table id of the grandchild, or leaf word:
    //   kLeafBit | (103 + leaf depth) << 23 | sigma   (bits 23..30 = fp32 exponent of the cube size)
    const uint32_t* wide;
    // colour records indexed by table entry: coefficients only (sigma is in the leaf word), channel-major fp16,
    // padded to a 16-byte multiple (8 bytes for one coefficient per channel)
    const unsigned char* wrecs;
    const float* extra;
    float offset[3];
    float scale[3];
    float ndc_width, ndc_height, ndc_focal;
    int32_t N;          // 0: nothing to draw (background only)
    int32_t format;     // VR_FMT_*
    int32_t basis_dim;  // reference basis_dim (-1 RGBA)
    int32_t kbd;        // kernel basis: -1 RGBA, 1, 4, 9, 16, 25 (others collapse to 1)
    int32_t rec_bytes;
    int32_t max_depth;
    int32_t wide_p;     // v in [0, kWideLv): internal nodes of depth d with (d + v) % kWideLv == 0 own a table (+ the root)
    uint32_t wide_entries;  // number of table entries (64 per table): bound of every record / table index
    // With wide_p = 1 the tables behave as if the octree hung one level below a virtual root (octant 0): leaf words
    // carry depth + wide_p, and the march keeps positions on a 2^(24 - wide_p) grid.  The three constants below are
    // all the kernel needs of the parity -- no per-sample arithmetic on it.
    float pos_scale;        // 2^(24 - wide_p)
    float pos_hi;           // (1 - 1e-6f) * pos_scale: upper clamp of a position (n3tree_query.hpp:17-19)
    uint32_t icube_bias;    // 0x73000000 + (wide_p << 23): 1/2^depth = bits(icube_bias - (w & 0x7f800000))
};

struct CamDev {
    int32_t width, height;
    float fx, fy;
    float c2w[12];
};

struct OptDev {
    float step_size, sigma_thresh, stop_thresh, background_brightness;
    float render_bbox[6];
    int32_t basis_min, basis_max;
    float rot_dirs[3];
    int32_t render_depth;
};

// Magic numbers for n / d, exact for 0 <= n < 2^31 (d >= 1): with 2^(s-1) < d <= 2^s and
// m = ceil(2^(31+s) / d) < 2^32, floor(n*m / 2^(31+s)) = floor(n/d) because the excess
// n*(m*d - 2^(31+s)) / (d*2^(31+s)) stays below 1/d.
inline void set_div(uint32_t d, uint32_t& mul, int32_t& shift) {
    if (d <= 1) { mul = 0; shift = -1; return; }
    int s = 0;
    while ((1ull << s) < d) ++s;
    mul = (uint32_t)(((1ull << (31 + s)) + d - 1) / d);
    shift = s - 1;
}

// Work queue of the persistent kernels.  One slot per launch in flight: {head, done CTAs}, then per SM id (mod 256) a
// 64-bit block state and a 32-bit lock (SM-local tile blocks, vr_march.cuh next_item).
constexpr int kBlkShift = 6, kBlkTiles = 1 << kBlkShift;   // a block = 64 warp tiles: views x tiles wide x tiles high
constexpr uint32_t kBlkDone = 0xfffffffdu, kBlkInvalid = 0xffffffffu;
constexpr unsigned long long kBlkIdle = 0x80000000ull;             // low word of a state that holds no tiles
constexpr int kQueueSlotBytes = 4096, kQueueStateOff = 64, kQueueLockOff = 64 + 256 * 8;

struct LaunchDev {
    TreeDev tree;
    OptDev opt;
    CamDev cam;            // used when cams == nullptr
    const CamDev* cams;    // device array for batches
    int32_t n_views;
    int32_t x0, y0, w, h;  // tile inside the cam.width x cam.height frame (h = rows of the output buffer)
    int32_t band_h, band_parts, band_part;  // ray-tile sharding: output row r is frame row
                                            // y0 + ((r/band_h)*band_parts + band_part)*band_h + r%band_h
    uint8_t* rgba8;        // linear tile-sized RGBA8 per view (or nullptr)
    float4* rgbaf;         // linear tile-sized float4 per view (or nullptr)
    const float* depth_in; // composite mode: per-pixel t limit (world units)
    vr_counters* counters; // device counters (instrumented kernels only)
    cudaSurfaceObject_t surf, dsurf;
    int32_t composite;     // 1: read existing colour from rgba8/surf + depth limit
    int32_t tiles_x, tiles_y, n_tiles;  // persistent kernels: work decomposition
    // division of a work item (< 2^31) by tiles_x and of the quotient by n_views as multiply-high + shift
    // (set_div): q = shift < 0 ? n : umulhi(n, mul) >> shift
    uint32_t div_view_mul, div_row_mul;
    int32_t div_view_shift, div_row_shift;
    unsigned int* work_counter;         // persistent kernels: global work queue {head, done CTAs} (start of a queue slot)
    // SM-local tile blocks (batches, vr_march.cuh next_item): the queue hands out BLOCKS of 64 warp tiles -- the same
    // 2^blk_wshift x 2^(6 - blk_gshift - blk_wshift) tiles of 2^blk_gshift consecutive views --, the warps of one SM
    // share a block, so that neighbouring tiles of neighbouring poses -- same tables, same records -- are marched at the
    // same time on the same L1.  blk_mode 0: one tile per queue item (single frames: finest balance).
    int32_t blk_mode, blocks_x, n_blocks, blk_gshift, blk_wshift, blk_groups;   // blk_groups: view groups of the batch
    unsigned long long* trace;          // diagnostics: per work item {start ns, end ns, smid, warp}
    // per-view options (vr_render_batch_opts): device array of n_views entries, read only by the kOutViewOpts
    // instantiations; nullptr = every view uses `opt`.  Last field, so the other fields keep their offsets.
    const OptDev* opts;
    // leaf weights (vr_tree_leaf_weights), read only by the kOutWeights instantiations: the tree's table entry -> slot
    // map, the caller's per-slot maximum weights and the per-pixel alpha output (or nullptr).  After `opts`, so that
    // every other field keeps its offset.
    const uint32_t* wslot;
    float* weights;
    float* alpha;
    // leaf gradients (vr_tree_leaf_grads), read only by the kOutGrads instantiations, which also use wslot and rgbaf:
    // dL/d(pixel) per pixel, the caller's gradient rows of grad_dim (= data_dim) floats per slot.  Last, as above.
    const float4* dpix;
    float* grad;
    int32_t grad_dim;
    // leaf error (vr_tree_leaf_error), read only by the kOutError instantiations, which also use wslot: the per-pixel
    // error and the caller's per-slot sums.  Last, as above.
    const float* err;
    float* score;
};

}  // namespace vrb
