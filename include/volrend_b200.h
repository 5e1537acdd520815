/*
 * volrend_b200.h -- thin C-ABI of the H100-native PlenOctree ray-marcher.
 *
 * This is the drop-in boundary for volrend's CUDA backend (reference paths relative to the
 * reference's root).  Everything the reference's `src/cuda/*` exports is re-expressed
 * here with plain pointers and sizes -- no torch, glm, cnpy or CUDA types:
 *
 *   vr_tree_create / vr_tree_destroy   replace N3Tree::load_cuda / free_cuda
 *                                      (src/cuda/n3tree.cu:9-41, :43-49; the struct
 *                                      N3Tree::device, include/volrend/n3tree.hpp:72-78)
 *   vr_render                          replaces launch_renderer(..., offscreen=true)
 *                                      (include/volrend/cuda/renderer_kernel.hpp:9-12,
 *                                      src/cuda/volrend.cu:195-245) and the device side
 *                                      render_kernel (volrend.cu:78-173) + trace_ray
 *                                      (include/volrend/cuda/rt_core.cuh:66-196)
 *   vr_render_composite                replaces launch_renderer(..., offscreen=false):
 *                                      colour + depth inputs (volrend.cu:92-96,143-146)
 *   vr_render_batch                    the per-pose loop of main_headless.cpp:208-223 as
 *                                      one call (same per-view semantics)
 *   vr_render_batch_opts               the same with one RenderOptions per view (the frames of
 *                                      main_anim.cpp:1252-1262, whose options change per frame)
 *   vr_render_frames_host              main_headless.cpp:208-223 with `-o`: renders and
 *                                      copies every frame to host memory (:216-219)
 *   vr_probe_lumisphere                retrieve_cursor_lumisphere_kernel (volrend.cu:175-191)
 *   vr_draw_probe                      the enable_probe disc of render_kernel (volrend.cu:100-134),
 *                                      drawn over frames the calls above have written
 *   vr_last_error                      replaces the abort-on-error cuda_assert
 *                                      (src/cuda/common.cu:8-21) -- the C-ABI never aborts;
 *                                      the C++ shim (volrend_b200/csrc/shim) restores it.
 *
 * All calls return 0 on success or a negative VR_E* code; vr_last_error() gives the text.
 * Device buffers are caller-owned; rendering is asynchronous on the given CUDA stream
 * (passed as void* == cudaStream_t).  One vr_tree lives on the device that was current at
 * creation.  There is NO CPU fallback: without a CUDA device every call fails with
 * VR_ENODEVICE.
 */
#ifndef VOLREND_B200_H_
#define VOLREND_B200_H_
#include <stddef.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VR_BASIS_MAX 25 /* VOLREND_GLOBAL_BASIS_MAX, include/volrend/render_options.hpp:6 */

enum { VR_OK = 0, VR_EINVAL = -1, VR_ENODEVICE = -2, VR_ECUDA = -3, VR_ENOMEM = -4, VR_EUNSUPPORTED = -5 };

/* DataFormat::format, include/volrend/data_format.hpp:9-15 */
enum { VR_FMT_RGBA = 0, VR_FMT_SH = 1, VR_FMT_SG = 2, VR_FMT_ASG = 3 };

typedef struct vr_tree vr_tree; /* opaque: re-laid-out device copy of one N3Tree */

/* Host-side view of a loaded N3Tree (fields of include/volrend/n3tree.hpp:33-85). */
typedef struct {
    const int32_t* child;   /* N3Tree::child_  int32 [capacity*N^3], relative offsets, 0 = leaf */
    const uint16_t* data;   /* N3Tree::data_   fp16  [capacity*N^3*data_dim] */
    const float* extra;     /* N3Tree::extra_  SG: [basis_dim*4], ASG: [basis_dim*11], else NULL */
    int64_t capacity;       /* N3Tree::capacity */
    int32_t N;              /* N3Tree::N (only 2 is supported, as in the reference) */
    int32_t data_dim;       /* N3Tree::data_dim */
    int32_t format;         /* N3Tree::data_format.format (VR_FMT_*) */
    int32_t basis_dim;      /* N3Tree::data_format.basis_dim (-1 for RGBA) */
    float offset[3];        /* N3Tree::offset */
    float scale[3];         /* N3Tree::scale */
    int32_t use_ndc;        /* N3Tree::use_ndc */
    float ndc_width, ndc_height, ndc_focal;
} vr_tree_desc;

/* Camera (include/volrend/camera.hpp:31-48); c2w by value, no device copy needed. */
typedef struct {
    int32_t width, height;
    float fx, fy;
    float c2w[12];          /* glm::mat4x3 Camera::transform, column-major */
} vr_camera;

/* RenderOptions (include/volrend/render_options.hpp:11-53), ray-march subset. */
typedef struct {
    float step_size, sigma_thresh, stop_thresh, background_brightness;
    float render_bbox[6];
    int32_t basis_minmax[2];
    float rot_dirs[3];
    int32_t render_depth;
} vr_options;

typedef struct { int32_t x0, y0, w, h; } vr_rect;

/* Work counters (device-resident, accumulated with atomics when requested). */
typedef struct {
    unsigned long long samples;      /* S        march-loop iterations (rt_core.cuh:108) */
    unsigned long long child_loads;  /* sum d_s  child[] reads the reference algorithm makes */
    unsigned long long shaded;       /* S_shaded samples with sigma > sigma_thresh */
    unsigned long long rays_hit;     /* rays entering the march */
    unsigned long long node_fetches; /* node words this implementation actually loaded */
} vr_counters;

typedef struct {
    int64_t capacity;
    int32_t max_depth;               /* deepest leaf (root children = 1) */
    int32_t rec_bytes;               /* padded leaf-record stride */
    int64_t node_bytes, rec_total_bytes, top_bytes; /* sizes of the slot-indexed layout (node words, records,
                                                       a 16^3 top grid); never resident */
    int32_t kernel_basis;            /* -1 RGBA, 1, 4, 9, 16, 25 */
    int32_t wide_parity;             /* v: internal nodes of depth d with (d + v) % 2 == 0 own a 64-entry table (+ the root);
                                        the v with fewer tables is chosen per tree */
    int64_t n_tables;
    int64_t wide_bytes, wrecs_bytes; /* 64-entry tables; colour records indexed by table entry */
    int64_t kernel_bytes;            /* what the render kernels can touch: wide_bytes + wrecs_bytes + grid_bytes */
    int64_t device_bytes;            /* everything the tree keeps resident */
    int64_t grid_bytes;              /* coarse max-sigma grid (32^3 cells) that batch renders cull ray tiles with */
} vr_tree_info;

/* Compressed N3Tree as written by scripts/compress_octree.py:93-118 (keys quant_colors, quant_map,
 * sigma, data_retained).  The reference decodes it on the CPU with a scalar loop at load time
 * (src/n3tree.cpp:279-340); vr_tree_create_quantized uploads the compressed arrays and decodes on
 * the GPU straight into the device layout (same resulting tree, bit for bit). */
typedef struct {
    vr_tree_desc base;             /* child + header fields; base.data must be NULL */
    const uint16_t* quant_colors;  /* fp16 [n_quant][65536][3] codebooks */
    const uint16_t* quant_map;     /* u16  [n_quant][capacity*N^3] codebook indices */
    const uint16_t* sigma;         /* fp16 [capacity*N^3] */
    const uint16_t* data_retained; /* fp16 [n_retain][capacity*N^3][3] or NULL */
    int32_t n_quant;               /* quantised basis functions */
    int32_t n_retain;              /* un-quantised leading basis functions (n_quant+n_retain == basis_dim) */
} vr_tree_quant_desc;

void vr_default_options(vr_options* o);

int vr_tree_create(const vr_tree_desc* desc, vr_tree** out);
int vr_tree_create_quantized(const vr_tree_quant_desc* desc, vr_tree** out);
/* The same with creation flags; flags = 0 is vr_tree_create / vr_tree_create_quantized, other bits are VR_EINVAL.
 * VR_TREE_SLOT_MAP keeps the table entry -> slot map the upload builds (one u32 per table entry: node * 8 + octant of
 * the entry's leaf in the source child / data arrays, or 0xffffffff for an entry that is not a leaf), which
 * vr_tree_leaf_weights needs.  With it, device_bytes includes the map (4 bytes per table entry); kernel_bytes and the
 * march kernels are the same. */
#define VR_TREE_SLOT_MAP 1u
int vr_tree_create_ex(const vr_tree_desc* desc, uint32_t flags, vr_tree** out);
int vr_tree_create_quantized_ex(const vr_tree_quant_desc* desc, uint32_t flags, vr_tree** out);
void vr_tree_destroy(vr_tree* tree);
int vr_tree_get_info(const vr_tree* tree, vr_tree_info* info);

/* Offscreen render of `tile` (NULL = full frame) of view `cam`.  rgba8_dev: tile-sized
 * linear RGBA8 (pitch 4*tile.w) or NULL; rgba32f_dev: tile-sized float4 or NULL;
 * counters_dev: device vr_counters to accumulate into, or NULL. */
int vr_render(const vr_tree* tree, const vr_camera* cam, const vr_options* opt, const vr_rect* tile,
              uint8_t* rgba8_dev, float* rgba32f_dev, vr_counters* counters_dev, void* stream);

/* n_views cameras (host array), outputs are n_views consecutive tile-sized images. */
int vr_render_batch(const vr_tree* tree, const vr_camera* cams, int n_views, const vr_options* opt,
                    const vr_rect* tile, uint8_t* rgba8_dev, float* rgba32f_dev,
                    vr_counters* counters_dev, void* stream);

/* Same, with options per view: view i is rendered with opts[i] (n_views entries), as vr_render would render it.
 * Output layout, tile, counters, the one-image-size rule and the splitting of very large batches are those of
 * vr_render_batch; NULL opts with n_views > 0 is VR_EINVAL.  The options travel through a device ring beside the
 * camera ring (allocated by the first such call on a (tree, stream)).
 * Used by the animator (volrend_anim, main_anim.cpp:268-307), whose interpolated options change every frame. */
int vr_render_batch_opts(const vr_tree* tree, const vr_camera* cams, int n_views, const vr_options* opts,
                         const vr_rect* tile, uint8_t* rgba8_dev, float* rgba32f_dev, vr_counters* counters_dev,
                         void* stream);

/* Maximum compositing weight per leaf over n_views views (the weight-based pruning of the PlenOctree conversion).
 * Every shaded sample (sigma > sigma_thresh) of every pixel of `tile` (NULL = full frame) of every view sets
 *   weight_dev[slot] = max(weight_dev[slot], T * (1 - att))
 * with the weight computed by exactly the operations of vr_render_batch's march; slot = node * 8 + octant of the
 * sample's leaf in the source arrays.  weight_dev: capacity * 8 floats on the tree's device, initialised by the caller
 * (e.g. to -inf), so that calls accumulate and one call over a set of views equals several calls over any split of it.
 * The maximum is taken in the total order of floats with -0 < +0 (negative weights arise when sigma_thresh < 0 lets
 * sigma <= 0 through); NaN weights are not recorded.  Of `opt`, step_size, sigma_thresh, stop_thresh and render_bbox
 * act as in vr_render_batch (so do NDC and early termination); render_depth, basis_minmax, rot_dirs and
 * background_brightness have no effect.  alpha_dev (NULL, or tile-sized floats per view) receives each ray's alpha,
 * the alpha channel of vr_render_batch's float output; counters_dev accumulates the usual counters.  Asynchronous on
 * stream.  VR_EUNSUPPORTED for a tree created without VR_TREE_SLOT_MAP; otherwise validated as vr_render_batch. */
int vr_tree_leaf_weights(const vr_tree* tree, const vr_camera* cams, int n_views, const vr_options* opt,
                         const vr_rect* tile, float* weight_dev, float* alpha_dev, vr_counters* counters_dev,
                         void* stream);

/* Per-leaf sum of compositing weight x pixel error over n_views views (choosing the leaves to split when refining a
 * fitted tree).  Every shaded sample (sigma > sigma_thresh) of every pixel of `tile` (NULL = full frame) of every view
 * adds  w_i * err[view][pixel]  to score_dev[slot] (slot = node*8 + octant in the source arrays), w_i = T_i (1 - att_i)
 * computed by exactly the operations of vr_tree_leaf_weights' weights.  err_dev: tile-sized floats per view;
 * score_dev: capacity*8 floats, ACCUMULATED into (caller initialises, e.g. to 0).  Every ray is marched whatever its
 * err (an err of 0 adds zeros), so counters_dev accumulates exactly the counters of vr_tree_leaf_weights.  One
 * atomicAdd per shaded sample: the sums depend on the order of the atomics and are not bit-reproducible from run to
 * run.  Of `opt`, the same fields act as in vr_tree_leaf_weights.  VR_EUNSUPPORTED for a tree created without
 * VR_TREE_SLOT_MAP; VR_EINVAL for NULL err_dev / score_dev or buffers that are not device memory of the tree's
 * device; otherwise validated as vr_render_batch.  Asynchronous on stream. */
int vr_tree_leaf_error(const vr_tree* tree, const vr_camera* cams, int n_views, const vr_options* opt,
                       const vr_rect* tile, const float* err_dev, float* score_dev, vr_counters* counters_dev,
                       void* stream);

/* Gradient of the float output of vr_render_batch w.r.t. every leaf's data row (fitting leaf values to images).
 * dpix_dev: tile-sized float4 per view (dL/d{r,g,b,alpha} of the rgba32f output); grad_dev: capacity*8*data_dim floats
 * on the tree's device, slot-major like N3Tree::data_ (slot = node*8 + octant), ACCUMULATED into (caller initialises,
 * e.g. to 0).  rgba32f_dev: NULL, or receives the float output of the forward replay (bit-identical to
 * vr_render_batch's).  The samples are vr_render_batch's; every shaded sample adds its terms with one atomicAdd each
 * (formulas in DESIGN.md 18), so the sums depend on the order of the atomics and are not bit-reproducible from run to
 * run.  Columns the device does not keep (coefficients k >= 1 of a basis size without its own kernel, columns between
 * the colour coefficients and sigma) get nothing, nor do internal and free slots.  render_depth is VR_EINVAL, a tree
 * created without VR_TREE_SLOT_MAP VR_EUNSUPPORTED; otherwise validated as vr_render_batch.  Asynchronous on stream. */
int vr_tree_leaf_grads(const vr_tree* tree, const vr_camera* cams, int n_views, const vr_options* opt,
                       const vr_rect* tile, const float* dpix_dev, float* grad_dev, float* rgba32f_dev, void* stream);

/* Replace the leaf values of a tree created with VR_TREE_SLOT_MAP: data_dev is fp16 [capacity*8*data_dim] on the
 * tree's device, laid out as vr_tree_desc::data.  Every table entry whose wslot names a leaf gets that slot's colour
 * record and the sigma bits of its leaf word rewritten (under table parity 1 several entries name one slot: all are
 * written); structure, parity, tables and sizes (vr_tree_get_info) do not change, and renders, vr_tree_query,
 * vr_tree_eval and vr_probe_lumisphere read the new values.  VR_EUNSUPPORTED without the slot map, VR_EINVAL for NULL
 * data or data on another device.  Asynchronous on stream: ordering against launches on other streams that read the
 * tree is the caller's job. */
int vr_tree_update_data(vr_tree* tree, const uint16_t* data_dev, void* stream);

/* Forward neighbours of every leaf (the total-variation prior of vr_tree_leaf_tv).  A reachable leaf slot at depth d
 * (root's slots: 1) with integer cell i in [0, 2^d)^3 of the tree's unit cube has, along axis a, the neighbour
 * n_a = the leaf whose cell holds the point (i + e_a) 2^-d, found by a descent from the root: the leaf that covers a
 * coarser or equal region across the +a face, the leaf at the min-corner octant of a finer one; none when
 * i_a + 1 = 2^d.  nbr_dev: capacity*8*3 int32 on the tree's device, nbr[slot*3 + a] = n_a or -1; internal, free and
 * unreachable slots get -1 in all three.  Cell counts are taken on the first call for a tree (shared with
 * vr_tree_wireframe; that call synchronises stream).  VR_EUNSUPPORTED for a tree created without VR_TREE_SLOT_MAP,
 * VR_EINVAL for a NULL buffer or one that is not device memory of the tree's device.  Asynchronous on stream. */
int vr_tree_leaf_neighbors(const vr_tree* tree, int32_t* nbr_dev, void* stream);

/* Total variation between neighbouring leaves (DESIGN.md 20), on the fp32 rows data_dev [capacity*8*data_dim]:
 *   E = sum_G (lambda_G / N_leaf) sum_{leaf s} sum_{c in G} sqrt(1e-8 + sum_{a: n_a(s) exists} (v[n_a, c] - v[s, c])^2)
 * over the groups G = sigma (column data_dim - 1) and colour (the coefficient columns vr_tree_leaf_grads writes);
 * N_leaf is the number of reachable leaf slots and n_a comes from nbr_dev, vr_tree_leaf_neighbors' table of this
 * tree.  dE/dv is ACCUMULATED into grad_dev (capacity*8*data_dim floats, e.g. vr_tree_leaf_grads' buffer) and E added
 * to *energy_dev (one double on the device; NULL: not computed).  Other columns and non-leaf slots get nothing; a
 * group whose weight is 0 is skipped, and with both weights 0 nothing is launched.  The gradient terms are float
 * atomicAdds: the sums depend on the order of the atomics and are not bit-reproducible from run to run.  VR_EINVAL for
 * a negative or non-finite weight, NULL nbr / data / grad or buffers that are not device memory of the tree's device;
 * VR_EUNSUPPORTED without the slot map.  Asynchronous on stream (the first call for a tree may synchronise it, as in
 * vr_tree_leaf_neighbors). */
int vr_tree_leaf_tv(const vr_tree* tree, const int32_t* nbr_dev, const float* data_dev, float lambda_sigma,
                    float lambda_color, float* grad_dev, double* energy_dev, void* stream);

/* launch_renderer(offscreen=false): rgba8_dev is read (existing colour) and overwritten;
 * depth_dev holds the per-pixel ray-distance limit (world units), both tile-sized. */
int vr_render_composite(const vr_tree* tree, const vr_camera* cam, const vr_options* opt,
                        const vr_rect* tile, uint8_t* rgba8_dev, const float* depth_dev,
                        float* rgba32f_dev, void* stream);
/* vr_render_composite for n_views views: view i's colour, depth limit and float output are the i-th tile-sized
 * frames of rgba8_dev, depth_dev and rgba32f_dev, and its bytes equal vr_render_composite of cams[i].  Tile, the
 * one-image-size rule and the splitting of very large batches are those of vr_render_batch; _opts renders view i
 * with opts[i]. */
int vr_render_composite_batch(const vr_tree* tree, const vr_camera* cams, int n_views, const vr_options* opt,
                              const vr_rect* tile, uint8_t* rgba8_dev, const float* depth_dev, float* rgba32f_dev,
                              void* stream);
int vr_render_composite_batch_opts(const vr_tree* tree, const vr_camera* cams, int n_views, const vr_options* opts,
                                   const vr_rect* tile, uint8_t* rgba8_dev, const float* depth_dev,
                                   float* rgba32f_dev, void* stream);

/* Same, writing a CUDA surface object over an RGBA8 cudaArray (what the reference's
 * caller owns, main_headless.cpp:190-199); depth_surf = 0 => offscreen. */
int vr_render_surface(const vr_tree* tree, const vr_camera* cam, const vr_options* opt,
                      unsigned long long rgba8_surf, unsigned long long depth_surf, void* stream);

/* Ray-tile sharding of one frame across n_parts GPUs (SURVEY.md 8e): this call renders every
 * n_parts-th band of band_h rows (bands part, part+n_parts, ...) of the full frame and writes them
 * compactly, band after band, into rgba8_dev / rgba32f_dev (vr_band_rows() rows of cam->width
 * pixels).  One launch per GPU per frame; the caller gathers the compact buffers. */
int vr_render_bands(const vr_tree* tree, const vr_camera* cam, const vr_options* opt, int band_h, int n_parts,
                    int part, uint8_t* rgba8_dev, float* rgba32f_dev, void* stream);
int vr_band_rows(int height, int band_h, int n_parts, int part);
/* Same for n_views cameras in ONE launch: view i's bands land at rgba8_dev + i * 4*width*vr_band_rows(). */
int vr_render_bands_batch(const vr_tree* tree, const vr_camera* cams, int n_views, const vr_options* opt, int band_h,
                          int n_parts, int part, uint8_t* rgba8_dev, float* rgba32f_dev, void* stream);

/* Host-buffer entry point: renders n_views full frames and copies each to
 * rgba8_host + i*4*w*h (pinned or pageable); returns after the last copy completed. */
int vr_render_frames_host(const vr_tree* tree, const vr_camera* cams, int n_views,
                          const vr_options* opt, uint8_t* rgba8_host);

/* Image egress (main_headless.cpp:216-222 with -o + src/imwrite.cpp:14-79): PNG files, 8-bit RGBA,
 * compression level 0 / filter NONE like the reference, written without libpng (stored deflate
 * blocks + CRC-32/Adler-32).  vr_render_frames_png renders, copies out and encodes n_views frames,
 * overlapping the three stages; paths[i] receives view i. */
int vr_write_png(const char* path, const uint8_t* rgba8_host, int width, int height);
int vr_render_frames_png(const vr_tree* tree, const vr_camera* cams, int n_views, const vr_options* opt,
                         const char* const* paths, int n_threads);
/* The same pipeline with options per view (opts[i] for view i, as vr_render_batch_opts). */
int vr_render_frames_png_opts(const vr_tree* tree, const vr_camera* cams, int n_views, const vr_options* opts,
                              const char* const* paths, int n_threads);

/* Copies the colour coefficients of the leaf containing world point xyz into out_dev as floats
 * (retrieve_cursor_lumisphere_kernel): min(data_dim-1, 3*basis_dim) values (3 for RGBA). */
int vr_probe_lumisphere(const vr_tree* tree, const float xyz_world[3], float* out_dev, void* stream);

/* RenderOptions::enable_probe (volrend.cu:100-134): draws the lumisphere probe disc of the leaf containing world point
 * probe_xyz over n_views frames that vr_render / vr_render_batch / vr_render_composite / vr_render_surface already
 * wrote with the same cams, tile and layout (one launch, stream-ordered after them).  disp_size is probe_disp_size:
 * the disc spans the top-right disp_size x disp_size pixels of the full frame, 5 pixels in from the right and down
 * from the top edge; of a `tile` only the part inside it is written, at tile-relative positions.  A disc pixel gets
 * the leaf's colour seen along the direction the disc point faces (the camera rotation applied to the point of the
 * unit hemisphere behind it), alpha 1: sigmoid of the basis sum for SH/SG/ASG trees, the raw RGB for RGBA trees; the
 * byte and float outputs hold what the reference's render_kernel stores there.  Pixels outside the disc are left as
 * they are.  Of `opt` only basis_minmax is read, clamped to the tree's basis (the reference reads past the
 * coefficients when the range reaches beyond basis_dim - 1).  rgba8_surf != 0 selects the surface form: one view,
 * tile NULL, rgba8_dev and rgba32f_dev NULL.  disp_size <= 0 draws nothing.  VR_EUNSUPPORTED for the trees
 * vr_probe_lumisphere refuses. */
int vr_draw_probe(const vr_tree* tree, const vr_camera* cams, int n_views, const vr_options* opt,
                  const float probe_xyz[3], int disp_size, const vr_rect* tile,
                  uint8_t* rgba8_dev, float* rgba32f_dev, unsigned long long rgba8_surf, void* stream);

/* ---- point queries (volrend_b200/csrc/vr_query.cu) --------------------------------------------------------
 * query_single_from_root (n3tree_query.hpp:13-48) for n points given in world coordinates (the tree maps them with
 * offset + scale * xyz, as retrieve_cursor_lumisphere_kernel does, volrend.cu:180-182, and clamps them to
 * [0, 1-1e-6] with fminf / fmaxf: a NaN coordinate ends up at 1-1e-6).
 *   data_dev  fp16 [n][data_dim]: the leaf's data row, bit for bit what the reference's `out` points at (colour
 *             coefficients channel-major, sigma last), or NULL
 *   cube_dev  float [n]: the reference's cube_sz (N^depth, root children = N), or NULL
 *   local_dev float [n][3]: the in-cell coordinates the reference leaves in xyz, or NULL
 * Asynchronous on stream.  VR_EUNSUPPORTED when data_dev != NULL for trees whose basis size keeps only coefficient 0
 * on the device (the ones vr_probe_lumisphere refuses) or whose data_dim exceeds 3 * basis_dim + 1 (4 for RGBA);
 * VR_EINVAL for n < 0, NULL xyz_dev with n > 0, or a buffer that is not device memory of the tree's device
 * (pageable host memory, another device's allocation). */
int vr_tree_query(const vr_tree* tree, const float* xyz_dev, int64_t n,
                  uint16_t* data_dev, float* cube_dev, float* local_dev, void* stream);

/* The colour the probe disc of render_kernel gives a leaf seen along dir (volrend.cu:111-128), for n (point,
 * direction) pairs: rgb_dev float [n][3] = sigmoid(sum over basis_minmax of basis(dir) * coeff) per channel
 * (SH/SG/ASG), raw RGB for RGBA trees; sigma_dev float [n] = the leaf's sigma.  Directions are used as given (not
 * normalised, as the probe uses the rotated unit vector).  Of opt only basis_minmax is read, clamped as vr_draw_probe
 * clamps it (opt NULL: the whole basis).  Either output may be NULL.  VR_EUNSUPPORTED when rgb_dev != NULL for the
 * trees vr_probe_lumisphere refuses; VR_EINVAL as vr_tree_query, and for NULL dir_dev with rgb_dev and n > 0. */
int vr_tree_eval(const vr_tree* tree, const float* xyz_dev, const float* dir_dev, int64_t n,
                 const vr_options* opt, float* rgb_dev, float* sigma_dev, void* stream);

/* Diagnostics: one full-frame render with the instrumented kernel that also records, per 8x4-pixel
 * work item (row-major tiles of 8x4), {start ns, end ns, SM id, global warp id} into
 * trace_dev[4 * n_items] (n_items = ceil(w/8)*ceil(h/4)). */
int vr_debug_trace(const vr_tree* tree, const vr_camera* cam, const vr_options* opt, uint8_t* rgba8_dev,
                   vr_counters* counters_dev, unsigned long long* trace_dev, void* stream);

/* Kernel variant selection for measurement.  0 = default: the inline-shading kernel (3 + 16*193) for batches, the
 * shading-queue kernel (7) for single-view launches on trees with 4, 9 or 16 basis functions (measured, DESIGN.md 4;
 * both produce identical bits).  vr_get_variant returns the process-wide setting (0 unless changed), vr_tree_variant
 * the variant a BATCH launch on `tree` resolves to (-1 if the setting is not available for its basis size), vr_variant_supported whether `variant` is
 * built into this library for a kernel basis of -1 (RGBA), 1, 4, 9, 16 or 25. */
int vr_set_variant(int variant);
int vr_get_variant(void);
int vr_tree_variant(const vr_tree* tree);
int vr_variant_supported(int kernel_basis, int variant);
/* Multi-GPU plumbing without SM-resident collectives: finished RGBA8 frames / bands are moved to the
 * gathering GPU by the copy engines over NVLink (cudaMemcpyAsync between peer-mapped buffers), so the
 * persistent march kernel keeps every SM.  vr_dev_alloc returns plain cudaMalloc memory (the base
 * address an IPC handle needs); vr_ipc_export writes the 64-byte cudaIpcMemHandle_t of such a buffer,
 * vr_ipc_open maps a peer process's buffer into this process (enabling peer access when possible),
 * vr_copy_async is a stream-ordered device/peer/host copy (kind inferred from the pointers). */
int vr_dev_alloc(size_t bytes, void** ptr);
int vr_dev_free(void* ptr);
int vr_ipc_export(void* dev_ptr, unsigned char handle_out[64]);
int vr_ipc_open(const unsigned char handle[64], void** ptr_out);
int vr_ipc_close(void* ptr);
int vr_copy_async(void* dst, const void* src, size_t bytes, void* stream);
/* 2-D variant (cudaMemcpy2DAsync, kind inferred): scatters a rank's compact bands into their interleaved rows
 * of a frame that lives in a peer-mapped buffer. */
int vr_copy2d_async(void* dst, size_t dst_pitch, const void* src, size_t src_pitch, size_t width_bytes, size_t rows,
                    void* stream);

/* ---- multi-GPU, one process driving N devices (volrend_b200/csrc/vr_mg.cu) ------------------------------
 * What a multi-GPU main_headless.cpp needs (the reference is single-GPU: main_headless.cpp:118-121 picks ONE
 * device): the tree replicated on `devices`, poses or ray tiles sharded over them, finished RGBA8 frames
 * gathered on devices[0] by the copy engines over NVLink (peer copies, no SM-resident collective).
 *   VR_MG_VIEWS  view i -> device i % n            VR_MG_TILES  band b (band_h rows) of every frame -> device b % n
 * vr_mg_render is synchronous: on return n_views frames are in rgba8_dev0 (device memory on devices[0]; NULL =
 * an internal buffer, see vr_mg_frames_dev0) and, when rgba8_host != NULL, in host memory.  `batch` = views per
 * kernel launch per device (<= 0: all).  *ms_out = device time of the whole job, max over devices (CUDA events;
 * all devices start idle). */
typedef struct vr_mg vr_mg;
enum { VR_MG_VIEWS = 0, VR_MG_TILES = 1 };
int vr_mg_create(const vr_tree_desc* desc, const int* devices, int n_devices, vr_mg** out);
void vr_mg_destroy(vr_mg* mg);
int vr_mg_device_count(const vr_mg* mg);
int vr_mg_device(const vr_mg* mg, int index);
vr_tree* vr_mg_tree(const vr_mg* mg, int index);
int vr_mg_render(vr_mg* mg, const vr_camera* cams, int n_views, const vr_options* opt, int mode, int band_h, int batch,
                 uint8_t* rgba8_dev0, uint8_t* rgba8_host, float* ms_out);
const uint8_t* vr_mg_frames_dev0(const vr_mg* mg);
const char* vr_mg_last_error(const vr_mg* mg);
/* How many of this library's kernels were launched by this process.  One exception: a batch render's tile-coverage
 * pass (the kernel that decides which ray tiles of the batch can shade) is not counted on its own but with the march
 * launch it prepares, so a batch march still counts as one launch. */
unsigned long long vr_launch_count(void);

const char* vr_last_error(void);
const char* vr_version(void);

/* ---- meshes (volrend_b200/csrc/vr_raster.cu) --------------------------------------------------------------
 * The GL mesh pass of cuda_renderer.cpp:83-113 (Mesh::draw, src/mesh.cpp:98-160,366-396) as a CUDA rasterizer.
 * A vertex is 9 floats: position, colour, normal (mesh.cpp:26).  face_size 3 / 2 / 1 = triangles / lines /
 * points (4x4 pixels); with faces_dev NULL the primitives are consecutive vertices, n_verts / face_size of
 * them, and n_faces is ignored.  A primitive with an index >= n_verts is not drawn.  unlit != 0 writes the
 * vertex colour, otherwise the reference's fixed three-light Phong shader (mesh.cpp:137-156). */
typedef struct {
    const float* vert_dev;      /* n_verts * 9 floats, device (caller-owned, like every buffer here) */
    const uint32_t* faces_dev;  /* n_faces * face_size indices, or NULL = consecutive vertices */
    int32_t n_verts, n_faces, face_size, unlit;
    float model[16];            /* column-major model matrix (host computes it from rotation/translation/scale) */
} vr_mesh_desc;
/* Draws meshes in order over the existing rgba8_dev (W*H*4) and depth_dev (W*H float, ray distance in world
 * units), GL depth test LESS against an internal z-buffer initialised from depth_dev; asynchronous on stream.
 * Where a fragment wins, rgba8_dev receives its colour (alpha included) and depth_dev its ray distance
 * length(camera-space position), ready for vr_render_composite.  depth_dev must be >= 0 (1e9 = empty). */
int vr_draw_meshes(const vr_camera* cam, const vr_mesh_desc* meshes, int n_meshes,
                   uint8_t* rgba8_dev, float* depth_dev, void* stream);
/* n_views frames of one size (every cams[i] has the same width and height), stored one after another in rgba8_dev
 * (4*W*H bytes each) and depth_dev (W*H floats each).  View i draws meshes[mesh_off[i] .. mesh_off[i+1]) in that
 * order.  Its bytes equal
 *   vr_draw_meshes(&cams[i], meshes + mesh_off[i], mesh_off[i+1] - mesh_off[i], rgba8_dev + i*4*W*H, depth_dev + i*W*H)
 * exactly (colour and depth).  mesh_off has n_views + 1 entries, non-decreasing, starting at 0.  n_views == 0 and
 * views without primitives write nothing.  The views with primitives are drawn in launch groups of four launches
 * each: a group's scratch (8 B of z-buffer per pixel, 16 B per possible large sub-primitive, i.e. 6 per triangle and
 * 1 per line or point) stays within 256 MiB, unless a single view needs more by itself, and its primitives below
 * 2^29.  Each view is validated as vr_draw_meshes validates its camera and meshes; views of different sizes, a
 * NULL, decreasing or non-zero-based mesh_off and a negative n_views are VR_EINVAL. */
int vr_draw_meshes_batch(const vr_camera* cams, int n_views, const vr_mesh_desc* meshes, const int32_t* mesh_off,
                         uint8_t* rgba8_dev, float* depth_dev, void* stream);

/* ---- octree grid (volrend_b200/csrc/vr_wire.cu) -----------------------------------------------------------
 * N3Tree::gen_wireframe (src/n3tree.cpp:365-434) generated from the device tree, byte for byte.  Starting at the
 * root (depth 0), a cell of a node of depth d is emitted when it is a leaf or d >= max_depth, else the walk descends
 * into it; so max_depth <= 0 gives the root's 8 cells and max_depth >= the tree's depth every leaf.  Each cell
 * becomes 12 line segments = 24 vertices of 9 floats (position, colour 0,0,0, normal 0,0,1), cells in the
 * reference's depth-first order, ready for a vr_mesh_desc with face_size 2.  vert_dev NULL: only *n_verts_out is
 * written.  Otherwise max_verts is the buffer's capacity in vertices (VR_EINVAL, nothing written, if the wireframe
 * needs more).  The first call on a tree counts its cells per level and synchronises `stream`; later calls are
 * stream-ordered and take their scratch memory from the stream-ordered allocator. */
int vr_tree_wireframe(const vr_tree* tree, int max_depth, float* vert_dev, int64_t max_verts,
                      int64_t* n_verts_out, void* stream);

/* ---- mesh normals (volrend_b200/csrc/vr_normals.cu) ------------------------------------------------------
 * Mesh estimate_normals (src/mesh.cpp:63-97), byte for byte: overwrites floats 6..8 (the normal) of each 9-float
 * vertex of vert_dev with the normalised sum of the cross products of its incident triangles, added in face order
 * from +0.f (vertices without faces get 0,0,0); every other float is left alone.  faces_dev NULL: a triangle soup,
 * n_verts / 3 faces of consecutive vertex triples (n_faces is ignored).  Otherwise n_faces triangles of 3 indices;
 * a face with an index >= n_verts contributes nothing.  Asynchronous on stream; scratch comes from the
 * rasterizer's stream-ordered pool.  VR_EINVAL for negative counts, NULL vert_dev with n_verts > 0, or more than
 * 2^31-1 vertices or face corners. */
int vr_mesh_estimate_normals(float* vert_dev, int64_t n_verts, const uint32_t* faces_dev, int64_t n_faces,
                             void* stream);

/* ---- tree compression (volrend_b200/csrc/vr_quant.cu) ----------------------------------------------------
 * Median-cut colour quantisation of a tree into the arrays vr_tree_quant_desc consumes (the format of the
 * reference's scripts/compress_octree.py, with codebooks always 65536 rows); DESIGN.md section 12 states the
 * algorithm bit for bit.  data_dev: fp16 [n_child][data_dim], channel-major coefficients (coefficient j of channel
 * k at k*B + j, B = (data_dim-1)/3), sigma last.  A slot is kept iff sigma > fp16_rn(sigma_thresh), compared as
 * fp16 (NaN is not kept).  The first n_retain basis functions are copied; each of the other B - n_retain is cut
 * into 2^bits buckets of its kept slots' RGB triples.  Outputs (device, caller-owned): quant_colors_dev fp16
 * [B-n_retain][65536][3] (bucket means, +0 for empty buckets and rows >= 2^bits), quant_map_dev u16
 * [B-n_retain][n_child] (0 for slots not kept), sigma_dev fp16 [n_child] (+0 where not kept), data_retained_dev fp16
 * [n_retain][n_child][3] (0 where not kept; NULL iff n_retain == 0); *n_kept_out = kept slots.  The kept count
 * sizes the scratch, so the call synchronises `stream` once; the rest is stream-ordered, with scratch from the
 * device's default stream-ordered pool (returned to it at the next synchronisation).  VR_EINVAL for bits outside
 * [1, 16], n_retain < 0, no basis function left to quantise, data_dim != 3B+1, n_child outside [0, INT32_MAX], and,
 * with no output written, for an Inf / NaN quantised coefficient in a kept slot or more than INT32_MAX points in
 * all (kept slots x (B - n_retain)). */
int vr_tree_compress(const uint16_t* data_dev, int64_t n_child, int32_t data_dim, float sigma_thresh, int32_t n_retain,
                     int32_t bits, uint16_t* quant_colors_dev, uint16_t* quant_map_dev, uint16_t* sigma_dev,
                     uint16_t* data_retained_dev, int64_t* n_kept_out, void* stream);

/* ---- tree construction (volrend_b200/csrc/vr_build.cu) ----------------------------------------------------
 * The canonical N3Tree of a set of voxel cells; DESIGN.md section 21 states it bit for bit.  cells_dev: int32 [n][4],
 * (level, i, j, k), the cube [i, i+1) x [j, j+1) x [k, k+1) * 2^-level of the tree's unit cube with 1 <= level <= 23
 * and 0 <= i, j, k < 2^level (i along x, the first axis of child[node, x, y, z]); rows_dev: fp16 [n][data_dim], laid
 * out as a row of N3Tree::data_.  The tree holds the root and one node per cell of level >= 1 that strictly contains a
 * listed cell; listed slots hold their rows bit for bit, every other slot +0.  Nodes are numbered breadth first, the
 * nodes of a level in Morton order (x the most significant bit), links are positive offsets: the output depends only
 * on the set of cells.  With VR_BUILD_MERGE, bottom-up, a node whose 8 slots are leaves with bitwise-equal rows (an
 * unlisted slot reads +0) becomes a leaf of its parent with that row; the root stays.
 * child_dev and data_dev both NULL: only *n_nodes_out is written.  Otherwise child_dev int32 [max_nodes*8] and data_dev
 * fp16 [max_nodes*8*data_dim] (caller-owned) receive the tree's first n_nodes nodes.  The node count synchronises
 * `stream` once; the rest is stream-ordered, with scratch from the device's default stream-ordered pool.  VR_EINVAL,
 * with nothing written, for: a level outside [1, 23], a coordinate outside [0, 2^level), a duplicate or overlapping
 * cell, n outside [0, INT32_MAX], data_dim < 1, NULL cells_dev / rows_dev with n > 0, NULL n_nodes_out, only one of
 * child_dev / data_dev NULL, a buffer that is not device memory of the current device, more than 0xffffffff / 8 nodes
 * (the int32 links and the u32 slot map) and more nodes than max_nodes. */
#define VR_BUILD_MERGE 1u
int vr_tree_build(const int32_t* cells_dev, const uint16_t* rows_dev, int64_t n, int32_t data_dim, uint32_t flags,
                  int32_t* child_dev, uint16_t* data_dev, int64_t max_nodes, int64_t* n_nodes_out, void* stream);

/* ---- image quality (volrend_b200/csrc/vr_ssim.cu) ------------------------------------------------------
 * Per-view SSIM of x against y, JaxNeRF's compute_ssim (DESIGN.md section 22): an 11-tap Gaussian (sigma 1.5,
 * normalised) applied separably with valid filtering to x, y, x^2, y^2 and xy of each of channels 0..2, clipped
 * variances and covariance, C1 = 0.01^2, C2 = 0.03^2, max_val 1, no clamping; ssim_dev[v] (double) is the mean over the
 * 3 channels and the (height-10) x (width-10) valid pixels of view v, overwritten.  x_dev: float32
 * [n_views][height][width][x_channels], y_dev the same with y_channels; channels 3 or 4 (only 0..2 are read).  dx_dev
 * NULL: forward only; otherwise x's layout, and dx += dx_scale * d ssim_v / dx on channels 0..2 of every view (other
 * elements untouched).  Bit-reproducible from run to run (no atomics).  Asynchronous on stream, with scratch from the
 * device's default stream-ordered pool.  n_views = 0 launches nothing.  VR_EINVAL for n_views < 0, height or width
 * below 11, channels other than 3 or 4, a non-finite dx_scale, NULL x_dev, y_dev or ssim_dev, and buffers that are not
 * device memory of the current device. */
int vr_image_ssim(const float* x_dev, int x_channels, const float* y_dev, int y_channels, int n_views, int height,
                  int width, double* ssim_dev, float* dx_dev, float dx_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif
