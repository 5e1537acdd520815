// vr_api.cu -- C-ABI of the H100 PlenOctree ray-marcher (declared in include/volrend_b200.h).
//
// Owns the launch logic (launch_renderer, reference src/cuda/volrend.cu:195-245) and the entry points; the device
// layout of a tree (N3Tree::load_cuda) and vr_tree_create / vr_tree_destroy are in vr_tree.cu.
// There is no CPU path in this library: every entry point needs a CUDA device.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <type_traits>
#include <vector>

#include "vr_build.h"
#include "vr_frames.h"
#include "vr_iso.h"
#include "vr_kernels.h"
#include "vr_normals.h"
#include "vr_probe.h"
#include "vr_quant.h"
#include "vr_query.h"
#include "vr_raster.h"
#include "vr_ssim.h"
#include "vr_tree.h"
#include "vr_tv.h"
#include "vr_wire.h"

using namespace vrb;

// ------------------------------------------------------------------------------------ errors
std::atomic<unsigned long long> vrb::g_launches{0};

namespace {
thread_local std::string g_err;
std::atomic<int> g_variant{0};
constexpr int kQueueSlots = 256;
constexpr int kCamRing = 8192;  // device ring of per-view cameras for batched launches
}  // namespace

int vrb::fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

int vrb::need_device(const vr_tree* t) {
    int dev = -1, ndev = 0;
    const bool ok = t ? cudaGetDevice(&dev) == cudaSuccess
                      : cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0 && cudaGetDevice(&dev) == cudaSuccess;
    if (!ok) {
        cudaGetLastError();
        return fail(VR_ENODEVICE, "no CUDA device: volrend_b200 has no CPU fallback");
    }
    if (t && dev != t->device) return fail(VR_EINVAL, "tree lives on device %d but device %d is current", t->device, dev);
    return VR_OK;
}

int vrb::buffer_check(const vr_tree* t, const void* p, const char* what) {
    if (!p) return VR_OK;
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
        cudaGetLastError();
        return fail(VR_EINVAL, "%s is not a CUDA allocation", what);
    }
    if (a.type == cudaMemoryTypeUnregistered) return fail(VR_EINVAL, "%s is not device memory", what);
    if (a.type == cudaMemoryTypeDevice && a.device != t->device)
        return fail(VR_EINVAL, "%s lives on device %d, the tree on device %d", what, a.device, t->device);
    return VR_OK;
}

int vrb::need_slot_map(const vr_tree* t, const char* what) {
    if (t->wslot) return VR_OK;
    return fail(VR_EUNSUPPORTED, "%s needs the slot map: create the tree with VR_TREE_SLOT_MAP", what);
}

namespace {
// f(std::integral_constant<int, K>{}) for the kernel bases K the march kernels are built for (kbd_built); `otherwise`
// for any other kbd.
template <class R, class F>
R with_kbd(int kbd, R otherwise, F f) {
    switch (kbd) {
        case -1: return f(std::integral_constant<int, -1>{});
        case 1: return f(std::integral_constant<int, 1>{});
        case 4: return f(std::integral_constant<int, 4>{});
        case 9: return f(std::integral_constant<int, 9>{});
        case 16: return f(std::integral_constant<int, 16>{});
        case 25: return f(std::integral_constant<int, 25>{});
        default: return otherwise;
    }
}

// All views of a batch have view 0's image size.
int same_size(const vr_camera* cams, int n_views) {
    for (int v = 1; v < n_views; ++v)
        if (cams[v].width != cams[0].width || cams[v].height != cams[0].height)
            return fail(VR_EINVAL, "view %d is %dx%d, view 0 %dx%d: all views of a batch must share one image size", v,
                        cams[v].width, cams[v].height, cams[0].width, cams[0].height);
    return VR_OK;
}

// Calls f(v0, nv) for consecutive chunks [v0, v0 + nv) of at most max_views views; stops at the first error.
template <class F>
int for_chunks(int n_views, int max_views, F f) {
    for (int v0 = 0; v0 < n_views; v0 += max_views)
        if (int rc = f(v0, std::min(max_views, n_views - v0))) return rc;
    return VR_OK;
}

// p advanced by n elements; a null (absent) output stays null.
template <class T>
T* skip(T* p, size_t n) { return p ? p + n : p; }

// The tree's basis has no kernel of its own (kernel_basis): the device keeps only coefficient 0 of each channel.
bool coef0_only(const vr_tree* t) { return t->dev.kbd > 0 && t->dev.kbd != t->dev.basis_dim; }

// opt's basis_minmax clamped to the tree's basis, as the march clamps it (NULL opt: the whole basis).  The reference
// sums basis_minmax[0]..[1] and reads past the coefficients when the range leaves the tree's basis.
void basis_range(const vr_tree* t, const vr_options* opt, int32_t* bmin, int32_t* bmax) {
    const int nb = t->dev.kbd > 0 ? t->dev.kbd : 1;
    *bmin = opt ? std::max(opt->basis_minmax[0], 0) : 0;
    *bmax = opt ? std::min(opt->basis_minmax[1], nb - 1) : nb - 1;
}

// one block per queue slot: {head, done} = 0, every SM's block state = "no block", locks free (vr_march.cuh next_item)
__global__ void queue_init_kernel(unsigned char* slots) {
    unsigned char* slot = slots + (size_t)blockIdx.x * kQueueSlotBytes;
    const int i = threadIdx.x;
    if (i < 2) reinterpret_cast<unsigned int*>(slot)[i] = 0u;
    reinterpret_cast<unsigned long long*>(slot + kQueueStateOff)[i] = ((unsigned long long)kBlkInvalid << 32) | kBlkIdle;
    reinterpret_cast<unsigned int*>(slot + kQueueLockOff)[i] = 0u;
}

}  // namespace

// ------------------------------------------------------------------------------------ launch plumbing
namespace {

void fill_opt(OptDev& o, const vr_options* s) {
    o.step_size = s->step_size; o.sigma_thresh = s->sigma_thresh; o.stop_thresh = s->stop_thresh;
    o.background_brightness = s->background_brightness;
    for (int i = 0; i < 6; ++i) o.render_bbox[i] = s->render_bbox[i];
    o.basis_min = s->basis_minmax[0]; o.basis_max = s->basis_minmax[1];
    for (int i = 0; i < 3; ++i) o.rot_dirs[i] = s->rot_dirs[i];
    o.render_depth = s->render_depth;
}
void fill_cam(CamDev& c, const vr_camera* s) {
    c.width = s->width; c.height = s->height; c.fx = s->fx; c.fy = s->fy;
    memcpy(c.c2w, s->c2w, sizeof(c.c2w));
}

// Launch resources of (tree, stream); created on the first launch on that stream.
int stream_res(vr_tree* t, cudaStream_t stream, StreamRes*& out) {
    std::lock_guard<std::mutex> lk(t->res_mu);
    auto it = t->res.find(stream);
    if (it == t->res.end()) {
        StreamRes r;
        VR_CUDA(cudaMalloc(&r.queues, (size_t)kQueueSlots * kQueueSlotBytes));
        cudaError_t e = cudaMalloc(&r.cam_ring, kCamRing * sizeof(CamDev));
        if (e == cudaSuccess) {   // legacy stream: ordered before later launches
            queue_init_kernel<<<kQueueSlots, 256>>>(reinterpret_cast<unsigned char*>(r.queues));
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
        if (e != cudaSuccess) {
            cudaFree(r.queues); cudaFree(r.cam_ring);
            return fail(VR_ECUDA, "stream resources: %s", cudaGetErrorString(e));
        }
        it = t->res.emplace(stream, r).first;
    }
    out = &it->second;
    return VR_OK;
}

// What a march launch computes: the render, the weights or error pass (one kernel for every basis size) or the
// gradient pass (one kernel per basis size); the passes ignore the variant setting.
enum class Pass { kRender, kWeights, kGrads, kError };

// One launch of P.n_views views, on the kernel march_kernel() picks.
int dispatch(const vr_tree* t, LaunchDev& P, bool count, bool surface, cudaStream_t stream, Pass pass = Pass::kRender) {
    const int variant = vr_get_variant();
    const MarchKernel kernel = march_kernel(t->dev.kbd, variant, P.n_views);
    if (pass == Pass::kRender && kernel == MarchKernel::kNotBuilt)
        return fail(VR_EUNSUPPORTED, "kernel variant %d is not available for kernel basis %d", variant, t->dev.kbd);
    LaunchCfg cfg;
    cfg.queue = kernel == MarchKernel::kQueue;
    cfg.count = count; cfg.surface = surface; cfg.num_sms = t->num_sms; cfg.stream = stream;
    vr_tree* mt = const_cast<vr_tree*>(t);
    StreamRes* sr = nullptr;
    if (int rc = stream_res(mt, stream, sr)) return rc;
    {
        std::lock_guard<std::mutex> lk(mt->res_mu);
        cfg.work_counter = reinterpret_cast<unsigned int*>(reinterpret_cast<unsigned char*>(sr->queues) + (size_t)(sr->next_queue++ % kQueueSlots) * kQueueSlotBytes);
        // The kernels read the tree before griddepcontrol.wait, and only that wait makes the predecessor's writes
        // visible.  So the first launch on a stream after vr_tree_update_data rewrote the tree waits for its
        // predecessor in full; later launches overlap again (the tree is not written between them).
        cfg.pdl = sr->data_gen == mt->data_gen;
        sr->data_gen = mt->data_gen;
    }
    // Batches on the inline kernel march only the tiles the coverage pass marks (vr_cull.cu); the instrumented
    // kernels march every ray, so they need no mask.
    if (pass == Pass::kRender && !count && kernel == MarchKernel::kInline && P.cams)
        if (int rc = launch_tile_mask(mt, P, stream)) return rc;
    // march_kernel above has rejected every kbd without kernels
    const cudaError_t e = pass == Pass::kWeights ? launch_weights(P, cfg) : pass == Pass::kError ? launch_error(P, cfg) : with_kbd(t->dev.kbd, cudaErrorInvalidValue, [&](auto k) {
        return pass == Pass::kGrads ? launch_grads<decltype(k)::value>(P, cfg) : launch_march<decltype(k)::value>(P, cfg);
    });
    if (e != cudaSuccess) return fail(VR_ECUDA, "kernel launch failed: %s", cudaGetErrorString(e));
    g_launches += 1;
    return VR_OK;
}

// Upper bound of the warp tiles of one view for every tile shape the kernels are built with
// (2x16, 4x8, 8x4 pixels): the persistent kernels index tiles of a whole batch with 31 bits.
long long tile_bound(const vr_rect& r) { return ((long long)r.w / 2 + 1) * ((long long)r.h / 4 + 1); }

int check_common(const vr_tree* t, const vr_camera* cam, const vr_options* opt, const vr_rect* tile, vr_rect& r) {
    if (!t || !cam || !opt) return fail(VR_EINVAL, "null argument");
    if (cam->width <= 0 || cam->height <= 0) return fail(VR_EINVAL, "bad camera size %dx%d", cam->width, cam->height);
    if (tile) {
        r = *tile;
        if (r.w < 0 || r.h < 0 || r.x0 < 0 || r.y0 < 0 || r.x0 + r.w > cam->width || r.y0 + r.h > cam->height)
            return fail(VR_EINVAL, "tile (%d,%d,%d,%d) outside %dx%d frame", r.x0, r.y0, r.w, r.h, cam->width, cam->height);
    } else {
        r.x0 = r.y0 = 0; r.w = cam->width; r.h = cam->height;
    }
    if (tile_bound(r) > 0x7fffffffLL)
        return fail(VR_EUNSUPPORTED, "%dx%d pixels: more tiles than the 31-bit work queue can index", r.w, r.h);
    return need_device(t);
}

// The opening checks of the batch entry points: n_views >= 0, and for a non-empty batch check_common (r: the tile or
// the full frame of view 0) and one image size for every view.  An empty batch is VR_OK before any pointer is read;
// callers return once it is checked.
int check_batch(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt, const vr_rect* tile,
                vr_rect& r) {
    if (n_views < 0) return fail(VR_EINVAL, "n_views < 0");
    if (n_views == 0) return VR_OK;
    if (int rc = check_common(t, cams, opt, tile, r)) return rc;
    return same_size(cams, n_views);
}

// Cameras of a batch go through a device ring owned by (tree, stream): no allocation on the launch path (a
// stream-ordered pool would hand memory back to the OS at every synchronisation), and a slot is rewritten
// only by a copy that is stream-ordered behind the launch that read it.  n_views <= kCamRing.
// opts != nullptr: n_views options, one per view, staged the same way into the option ring, slot for slot beside
// the cameras (the ring is allocated here on first use: callers that never pass per-view options pay nothing).
int stage_cams(const vr_tree* t, const vr_camera* cams, int n_views, cudaStream_t stream, LaunchDev& P,
               const vr_options* opts = nullptr) {
    if (n_views <= 1) return VR_OK;
    vr_tree* mt = const_cast<vr_tree*>(t);
    StreamRes* sr = nullptr;
    if (int rc = stream_res(mt, stream, sr)) return rc;
    unsigned int slot;
    {
        std::lock_guard<std::mutex> lk(mt->res_mu);
        if (opts && !sr->opt_ring) VR_CUDA(cudaMalloc(&sr->opt_ring, kCamRing * sizeof(OptDev)));
        if (sr->cam_pos + (unsigned int)n_views > (unsigned int)kCamRing) sr->cam_pos = 0;  // no wrap inside a batch
        slot = sr->cam_pos;
        sr->cam_pos += (unsigned int)n_views;
    }
    std::vector<CamDev> h(n_views);
    for (int i = 0; i < n_views; ++i) fill_cam(h[i], &cams[i]);
    CamDev* dcams = sr->cam_ring + slot;
    VR_CUDA(cudaMemcpyAsync(dcams, h.data(), sizeof(CamDev) * n_views, cudaMemcpyHostToDevice, stream));
    // pageable source: the copy has been staged when cudaMemcpyAsync returns
    P.cams = dcams;
    if (opts) {
        std::vector<OptDev> ho(n_views);
        for (int i = 0; i < n_views; ++i) fill_opt(ho[i], &opts[i]);
        OptDev* dopts = sr->opt_ring + slot;
        VR_CUDA(cudaMemcpyAsync(dopts, ho.data(), sizeof(OptDev) * n_views, cudaMemcpyHostToDevice, stream));
        P.opts = dopts;
    }
    return VR_OK;
}

// The march launches of every render entry point.  P holds the outputs and the rect (x0, y0, w, h; the output buffers
// hold h rows of w pixels per view); this adds the tree, the cameras and the options, and launches the views in chunks
// that fit the camera ring and the 31-bit tile index, the output pointers advanced to each chunk's first view.
// opt_stride as in vr_frames.h; a chunk of one view is an ordinary single-view launch with that view's options.
// pass: the weights, gradient or error pass, P.alpha, P.dpix and P.err advanced like the outputs.
int march(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt, int opt_stride,
          const LaunchDev& P, bool surface, cudaStream_t stream, Pass pass = Pass::kRender) {
    const long long tb = tile_bound(vr_rect{P.x0, P.y0, P.w, P.h});
    const int max_views = tb * kCamRing > 0x7fffffffLL ? (int)(0x7fffffffLL / tb) : kCamRing;
    const size_t px = (size_t)P.w * P.h;
    return for_chunks(n_views, max_views, [&](int v0, int nv) {
        const vr_options* o = opt + (size_t)opt_stride * v0;
        LaunchDev C = P;
        C.tree = t->dev;
        fill_opt(C.opt, o);
        fill_cam(C.cam, &cams[v0]);
        C.n_views = nv;
        C.rgba8 = skip(P.rgba8, 4 * px * v0);
        C.rgbaf = skip(P.rgbaf, px * v0);
        C.depth_in = skip(P.depth_in, px * v0);
        C.alpha = skip(P.alpha, px * v0);
        C.dpix = skip(P.dpix, px * v0);
        C.err = skip(P.err, px * v0);
        if (int rc = stage_cams(t, cams + v0, nv, stream, C, opt_stride ? o : nullptr)) return rc;
        return dispatch(t, C, P.counters != nullptr, surface, stream, pass);
    });
}

// vr_render_composite_batch (opt_stride 0) and vr_render_composite_batch_opts (opt_stride 1)
int render_composite_batch(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt, int opt_stride,
                           const vr_rect* tile, uint8_t* rgba8_dev, const float* depth_dev, float* rgba32f_dev,
                           void* stream) {
    if (n_views > 0 && (!rgba8_dev || !depth_dev)) return fail(VR_EINVAL, "composite mode needs colour and depth inputs");
    return render_batch(t, cams, n_views, opt, opt_stride, tile, rgba8_dev, rgba32f_dev, nullptr, stream, depth_dev);
}

// A buffer of a leaf pass, its name in the errors, and whether the pass needs it.
struct PassBuf { const void* p; const char* name; bool required = false; };

// The march-based leaf passes (vr_tree_leaf_weights, _error, _grads), `what` naming the pass.  The checks run in this
// order: a required buffer that is NULL is VR_EINVAL; check_batch (an empty batch is VR_OK before any pointer is
// read); `refuse(opt)`, the pass's own refusals; the slot map; buffer_check of every buffer; an empty rect is VR_OK.
// P holds the pass's buffers; the rect, the slot map and the gradient row width are added here.
int leaf_pass(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt, const vr_rect* tile,
              void* stream, Pass pass, const char* what, LaunchDev P, std::initializer_list<PassBuf> bufs,
              int (*refuse)(const vr_options*) = nullptr) {
    if (n_views > 0)
        for (const PassBuf& b : bufs)
            if (b.required && !b.p) return fail(VR_EINVAL, "%s: null %s", what, b.name);
    vr_rect r;
    int rc = check_batch(t, cams, n_views, opt, tile, r);
    if (rc || n_views == 0) return rc;
    if ((refuse && (rc = refuse(opt))) || (rc = need_slot_map(t, what))) return rc;
    for (const PassBuf& b : bufs)
        if ((rc = buffer_check(t, b.p, b.name))) return rc;
    if (r.w == 0 || r.h == 0) return VR_OK;
    P.x0 = r.x0; P.y0 = r.y0; P.w = r.w; P.h = r.h;
    P.wslot = t->wslot;
    P.grad_dim = t->data_dim;
    return march(t, cams, n_views, opt, 0, P, false, (cudaStream_t)stream, pass);
}
}  // namespace

// vr_render_batch (opt_stride 0: one options struct for every view) and vr_render_batch_opts (opt_stride 1: view i
// uses opt[i]).
int vrb::render_batch(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt, int opt_stride,
                      const vr_rect* tile, uint8_t* rgba8_dev, float* rgba32f_dev, vr_counters* counters_dev,
                      void* stream, const float* depth_dev) {
    vr_rect r;
    const int rc = check_batch(t, cams, n_views, opt, tile, r);
    if (rc || n_views == 0) return rc;
    if (depth_dev && !rgba8_dev) return fail(VR_EINVAL, "composite mode needs colour and depth inputs");
    if (r.w == 0 || r.h == 0) return VR_OK;
    LaunchDev P{};
    P.x0 = r.x0; P.y0 = r.y0; P.w = r.w; P.h = r.h;
    P.rgba8 = rgba8_dev; P.rgbaf = reinterpret_cast<float4*>(rgba32f_dev);
    P.counters = counters_dev;
    P.depth_in = depth_dev; P.composite = depth_dev != nullptr;
    return march(t, cams, n_views, opt, opt_stride, P, false, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------ C-ABI
extern "C" {

const char* vr_last_error(void) { return g_err.c_str(); }
const char* vr_version(void) { return "volrend_b200 0.2 (sm_90a)"; }
int vr_variant_supported(int kernel_basis, int variant) {
    return march_kernel(kernel_basis, variant, 1) != MarchKernel::kNotBuilt ? 1 : 0;
}
int vr_set_variant(int variant) {
    // accepted when at least one basis size has it; a tree whose basis size lacks it fails at launch
    for (int kbd = -1; kbd <= VR_BASIS_MAX; ++kbd)
        if (vr_variant_supported(kbd, variant)) { g_variant.store(variant); return VR_OK; }
    return fail(VR_EINVAL, "kernel variant %d is not built into this library", variant);
}
int vr_get_variant(void) { return g_variant.load(); }
int vr_tree_variant(const vr_tree* t) {
    if (!t) return -1;
    const MarchKernel k = march_kernel(t->dev.kbd, g_variant.load(), 2);   // two views: a batch
    return k == MarchKernel::kQueue ? kVariantQueue : k == MarchKernel::kInline ? kVariantInline : -1;
}
unsigned long long vr_launch_count(void) { return g_launches.load(); }

void vr_default_options(vr_options* o) {
    if (!o) return;
    memset(o, 0, sizeof(*o));
    o->step_size = 1e-4f; o->sigma_thresh = 1e-2f; o->stop_thresh = 1e-2f;  // render_options.hpp:14-23
    o->background_brightness = 1.f;
    o->render_bbox[3] = o->render_bbox[4] = o->render_bbox[5] = 1.f;
    o->basis_minmax[0] = 0; o->basis_minmax[1] = VR_BASIS_MAX - 1;
}

int vr_render_batch(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt, const vr_rect* tile,
                    uint8_t* rgba8_dev, float* rgba32f_dev, vr_counters* counters_dev, void* stream) {
    return render_batch(t, cams, n_views, opt, 0, tile, rgba8_dev, rgba32f_dev, counters_dev, stream);
}

int vr_render_batch_opts(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opts,
                         const vr_rect* tile, uint8_t* rgba8_dev, float* rgba32f_dev, vr_counters* counters_dev,
                         void* stream) {
    return render_batch(t, cams, n_views, opts, 1, tile, rgba8_dev, rgba32f_dev, counters_dev, stream);
}

int vr_tree_leaf_weights(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt,
                         const vr_rect* tile, float* weight_dev, float* alpha_dev, vr_counters* counters_dev,
                         void* stream) {
    LaunchDev P{};
    P.weights = weight_dev; P.alpha = alpha_dev; P.counters = counters_dev;
    return leaf_pass(t, cams, n_views, opt, tile, stream, Pass::kWeights, "vr_tree_leaf_weights", P,
                     {{weight_dev, "weight_dev", true}, {alpha_dev, "alpha_dev"}, {counters_dev, "counters_dev"}});
}

int vr_tree_leaf_error(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt,
                       const vr_rect* tile, const float* err_dev, float* score_dev, vr_counters* counters_dev,
                       void* stream) {
    LaunchDev P{};
    P.err = err_dev; P.score = score_dev; P.counters = counters_dev;
    return leaf_pass(t, cams, n_views, opt, tile, stream, Pass::kError, "vr_tree_leaf_error", P,
                     {{err_dev, "err_dev", true}, {score_dev, "score_dev", true}, {counters_dev, "counters_dev"}});
}

int vr_tree_leaf_grads(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt,
                       const vr_rect* tile, const float* dpix_dev, float* grad_dev, float* rgba32f_dev, void* stream) {
    LaunchDev P{};
    P.dpix = reinterpret_cast<const float4*>(dpix_dev); P.grad = grad_dev;
    P.rgbaf = reinterpret_cast<float4*>(rgba32f_dev);
    return leaf_pass(t, cams, n_views, opt, tile, stream, Pass::kGrads, "vr_tree_leaf_grads", P,
                     {{dpix_dev, "dpix_dev", true}, {grad_dev, "grad_dev", true}, {rgba32f_dev, "rgba32f_dev"}},
                     [](const vr_options* o) {
                         return o->render_depth ? fail(VR_EINVAL, "leaf gradients are of the colour output: "
                                                                  "render_depth is not supported")
                                                : VR_OK;
                     });
}

int vr_render_composite_batch(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt,
                              const vr_rect* tile, uint8_t* rgba8_dev, const float* depth_dev, float* rgba32f_dev,
                              void* stream) {
    return render_composite_batch(t, cams, n_views, opt, 0, tile, rgba8_dev, depth_dev, rgba32f_dev, stream);
}

int vr_render_composite_batch_opts(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opts,
                                   const vr_rect* tile, uint8_t* rgba8_dev, const float* depth_dev,
                                   float* rgba32f_dev, void* stream) {
    return render_composite_batch(t, cams, n_views, opts, 1, tile, rgba8_dev, depth_dev, rgba32f_dev, stream);
}

int vr_render_bands_batch(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt, int band_h,
                          int n_parts, int part, uint8_t* rgba8_dev, float* rgba32f_dev, void* stream) {
    vr_rect r;
    const int rc = check_batch(t, cams, n_views, opt, nullptr, r);
    if (rc || n_views == 0) return rc;
    if (band_h < 4 || band_h % 4 || n_parts < 1 || part < 0 || part >= n_parts)
        return fail(VR_EINVAL, "bands: band_h must be a positive multiple of 4 and 0 <= part < n_parts");
    const int rows = vr_band_rows(cams[0].height, band_h, n_parts, part);
    if (rows == 0) return VR_OK;
    LaunchDev P{};
    P.w = r.w; P.h = rows;
    P.band_h = band_h; P.band_parts = n_parts; P.band_part = part;
    P.rgba8 = rgba8_dev; P.rgbaf = reinterpret_cast<float4*>(rgba32f_dev);
    return march(t, cams, n_views, opt, 0, P, false, (cudaStream_t)stream);
}

int vr_render_bands(const vr_tree* t, const vr_camera* cam, const vr_options* opt, int band_h, int n_parts,
                    int part, uint8_t* rgba8_dev, float* rgba32f_dev, void* stream_) {
    return vr_render_bands_batch(t, cam, 1, opt, band_h, n_parts, part, rgba8_dev, rgba32f_dev, stream_);
}

int vr_band_rows(int height, int band_h, int n_parts, int part) {
    if (height <= 0 || band_h <= 0 || n_parts <= 0 || part < 0 || part >= n_parts) return 0;
    const int n_bands = (height + band_h - 1) / band_h;
    int rows = 0;
    for (int b = part; b < n_bands; b += n_parts) {
        const int y = b * band_h;
        rows += (height - y < band_h) ? height - y : band_h;
    }
    return rows;
}

int vr_debug_trace(const vr_tree* t, const vr_camera* cam, const vr_options* opt, uint8_t* rgba8_dev,
                   vr_counters* counters_dev, unsigned long long* trace_dev, void* stream) {
    vr_rect r;
    int rc = check_common(t, cam, opt, nullptr, r);
    if (rc) return rc;
    if (!counters_dev || !trace_dev) return fail(VR_EINVAL, "trace needs counters and a trace buffer");
    LaunchDev P{};
    P.w = r.w; P.h = r.h;
    P.rgba8 = rgba8_dev; P.counters = counters_dev; P.trace = trace_dev;
    return march(t, cam, 1, opt, 0, P, false, (cudaStream_t)stream);
}

int vr_render(const vr_tree* t, const vr_camera* cam, const vr_options* opt, const vr_rect* tile, uint8_t* rgba8_dev,
              float* rgba32f_dev, vr_counters* counters_dev, void* stream) {
    return vr_render_batch(t, cam, 1, opt, tile, rgba8_dev, rgba32f_dev, counters_dev, stream);
}

int vr_render_composite(const vr_tree* t, const vr_camera* cam, const vr_options* opt, const vr_rect* tile,
                        uint8_t* rgba8_dev, const float* depth_dev, float* rgba32f_dev, void* stream) {
    return vr_render_composite_batch(t, cam, 1, opt, tile, rgba8_dev, depth_dev, rgba32f_dev, stream);
}

int vr_render_surface(const vr_tree* t, const vr_camera* cam, const vr_options* opt, unsigned long long rgba8_surf,
                      unsigned long long depth_surf, void* stream) {
    vr_rect r;
    int rc = check_common(t, cam, opt, nullptr, r);
    if (rc) return rc;
    if (!rgba8_surf) return fail(VR_EINVAL, "null surface");
    LaunchDev P{};
    P.w = r.w; P.h = r.h;
    P.surf = (cudaSurfaceObject_t)rgba8_surf; P.dsurf = (cudaSurfaceObject_t)depth_surf;
    P.composite = depth_surf != 0;
    return march(t, cam, 1, opt, 0, P, true, (cudaStream_t)stream);
}

}  // extern "C"

int vrb::render_frames_host(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt,
                            int opt_stride, uint8_t* rgba8_host) {
    // main_headless.cpp:208-223 with -o: every frame goes back to host memory.  Frames are
    // rendered in chunks of a few views per launch on two alternating streams (the tail of
    // one chunk overlaps the head of the next) and copied out on a third stream while the
    // following chunks render.
    if (n_views > 0 && !rgba8_host) return fail(VR_EINVAL, "null host buffer");
    vr_rect r;
    int rc = check_batch(t, cams, n_views, opt, nullptr, r);
    if (rc || n_views == 0) return rc;
    const size_t frame = (size_t)4 * r.w * r.h;
    const int chunk = std::min(8, n_views);
    vr_tree* mt = const_cast<vr_tree*>(t);
    std::lock_guard<std::mutex> host_lock(mt->host_mu);   // one host-path sweep per tree at a time
    vr_tree::HostPath& R = mt->host;
    constexpr int kRing = vr_tree::HostPath::kRing;
    if (!R.ready) {
        VR_CUDA(cudaStreamCreateWithFlags(&R.sr[0], cudaStreamNonBlocking));
        VR_CUDA(cudaStreamCreateWithFlags(&R.sr[1], cudaStreamNonBlocking));
        VR_CUDA(cudaStreamCreateWithFlags(&R.sc, cudaStreamNonBlocking));
        for (int i = 0; i < kRing; ++i) {
            VR_CUDA(cudaEventCreateWithFlags(&R.rendered[i], cudaEventDisableTiming));
            VR_CUDA(cudaEventCreateWithFlags(&R.copied[i], cudaEventDisableTiming));
        }
        R.ready = true;
    }
    if (R.buf_bytes < frame * chunk) {
        for (int i = 0; i < kRing; ++i) { cudaFree(R.buf[i]); R.buf[i] = nullptr; }
        R.buf_bytes = 0;
        for (int i = 0; i < kRing; ++i) VR_CUDA(cudaMalloc(&R.buf[i], frame * chunk));
        R.buf_bytes = frame * chunk;
    }
    int c = 0;
    for (int v0 = 0; v0 < n_views; v0 += chunk, ++c) {
        const int nv = n_views - v0 < chunk ? n_views - v0 : chunk;
        const int s = c % kRing;
        cudaStream_t sr = R.sr[c & 1];
        if (c >= kRing) VR_CUDA(cudaStreamWaitEvent(sr, R.copied[s], 0));
        rc = render_batch(t, cams + v0, nv, opt + (size_t)opt_stride * v0, opt_stride, nullptr, R.buf[s], nullptr,
                          nullptr, sr);
        if (rc) return rc;
        VR_CUDA(cudaEventRecord(R.rendered[s], sr));
        VR_CUDA(cudaStreamWaitEvent(R.sc, R.rendered[s], 0));
        VR_CUDA(cudaMemcpyAsync(rgba8_host + (size_t)v0 * frame, R.buf[s], frame * nv, cudaMemcpyDeviceToHost, R.sc));
        VR_CUDA(cudaEventRecord(R.copied[s], R.sc));
    }
    VR_CUDA(cudaStreamSynchronize(R.sc));
    VR_CUDA(cudaStreamSynchronize(R.sr[0]));
    VR_CUDA(cudaStreamSynchronize(R.sr[1]));
    return VR_OK;
}

extern "C" {

int vr_render_frames_host(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt,
                          uint8_t* rgba8_host) {
    return render_frames_host(t, cams, n_views, opt, 0, rgba8_host);
}

int vr_dev_alloc(size_t bytes, void** ptr) {
    if (!ptr) return fail(VR_EINVAL, "null argument");
    *ptr = nullptr;
    VR_CUDA(cudaMalloc(ptr, bytes ? bytes : 1));
    return VR_OK;
}
int vr_dev_free(void* ptr) {
    VR_CUDA(cudaFree(ptr));
    return VR_OK;
}
int vr_ipc_export(void* dev_ptr, unsigned char handle_out[64]) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    if (!dev_ptr || !handle_out) return fail(VR_EINVAL, "null argument");
    cudaIpcMemHandle_t h;
    VR_CUDA(cudaIpcGetMemHandle(&h, dev_ptr));
    memcpy(handle_out, &h, 64);
    return VR_OK;
}
int vr_ipc_open(const unsigned char handle[64], void** ptr_out) {
    if (!handle || !ptr_out) return fail(VR_EINVAL, "null argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    VR_CUDA(cudaIpcOpenMemHandle(ptr_out, h, cudaIpcMemLazyEnablePeerAccess));
    return VR_OK;
}
int vr_ipc_close(void* ptr) {
    VR_CUDA(cudaIpcCloseMemHandle(ptr));
    return VR_OK;
}
int vr_copy_async(void* dst, const void* src, size_t bytes, void* stream) {
    if (bytes == 0) return VR_OK;
    if (!dst || !src) return fail(VR_EINVAL, "null argument");
    VR_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, (cudaStream_t)stream));
    return VR_OK;
}

int vr_copy2d_async(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width_bytes, size_t rows, void* stream) {
    if (width_bytes == 0 || rows == 0) return VR_OK;
    if (!dst || !src) return fail(VR_EINVAL, "null argument");
    VR_CUDA(cudaMemcpy2DAsync(dst, dpitch, src, spitch, width_bytes, rows, cudaMemcpyDefault, (cudaStream_t)stream));
    return VR_OK;
}

int vr_probe_lumisphere(const vr_tree* t, const float xyz[3], float* out_dev, void* stream_) {
    if (!t || !xyz || !out_dev) return fail(VR_EINVAL, "null argument");
    if (int rc = need_device(t)) return rc;
    if (coef0_only(t))
        return fail(VR_EUNSUPPORTED, "probe unavailable for basis_dim %d (only coefficient 0 is resident)", t->dev.basis_dim);
    // the resident record holds the colour coefficients only: 3 per RGBA leaf, 3*basis_dim otherwise
    // (extra trailing channels of an over-wide data_dim are not kept)
    const int resident = t->dev.kbd < 0 ? 3 : 3 * t->dev.kbd;
    QueryLaunch Q{};
    Q.tree = t->dev;
    Q.n = 1;
    for (int i = 0; i < 3; ++i) Q.point[i] = xyz[i];
    Q.coef = out_dev;
    Q.n_coef = t->data_dim - 1 < resident ? t->data_dim - 1 : resident;
    VR_CUDA(query_launch(Q, t->dev.kbd, false, t->num_sms, (cudaStream_t)stream_));
    g_launches += 1;
    return VR_OK;
}

// Checks shared by vr_tree_query and vr_tree_eval; *full: the device keeps the tree's whole data row (every colour
// coefficient, and no halves between them and sigma that the records drop).
static int query_check(const vr_tree* t, const float* xyz, int64_t n, bool* full) {
    if (!t) return fail(VR_EINVAL, "null tree");
    if (n < 0) return fail(VR_EINVAL, "n = %lld < 0", (long long)n);
    if (!xyz && n > 0) return fail(VR_EINVAL, "null points with n = %lld", (long long)n);
    if (int rc = need_device(t)) return rc;
    const int nb = t->dev.kbd > 0 ? t->dev.kbd : 1;
    *full = !coef0_only(t) && t->data_dim == 3 * nb + 1;
    return VR_OK;
}

// query_single_from_root (n3tree_query.hpp:13-48) for n world points (kernel: vr_query.cu).
int vr_tree_query(const vr_tree* t, const float* xyz_dev, int64_t n, uint16_t* data_dev, float* cube_dev,
                  float* local_dev, void* stream_) {
    bool full = false;
    const int rc = query_check(t, xyz_dev, n, &full);
    if (rc) return rc;
    if (data_dev && !full)
        return fail(VR_EUNSUPPORTED, "data rows unavailable for basis_dim %d, data_dim %d (the device keeps %s)",
                    t->dev.basis_dim, t->data_dim,
                    coef0_only(t) ? "only coefficient 0" : "the colour coefficients and sigma only");
    if (n == 0 || (!data_dev && !cube_dev && !local_dev)) return VR_OK;
    int bc;
    if ((bc = buffer_check(t, xyz_dev, "xyz_dev")) || (bc = buffer_check(t, data_dev, "data_dev")) ||
        (bc = buffer_check(t, cube_dev, "cube_dev")) || (bc = buffer_check(t, local_dev, "local_dev")))
        return bc;
    QueryLaunch Q{};
    Q.tree = t->dev;
    Q.xyz = xyz_dev; Q.n = n;
    Q.data = data_dev; Q.cube = cube_dev; Q.local = local_dev;
    VR_CUDA(query_launch(Q, t->dev.kbd, false, t->num_sms, (cudaStream_t)stream_));
    g_launches += 1;
    return VR_OK;
}

// The probe disc's colour (volrend.cu:111-128) of the leaves of n world points along n directions (kernel: vr_query.cu).
int vr_tree_eval(const vr_tree* t, const float* xyz_dev, const float* dir_dev, int64_t n, const vr_options* opt,
                 float* rgb_dev, float* sigma_dev, void* stream_) {
    bool full = false;
    const int rc = query_check(t, xyz_dev, n, &full);
    if (rc) return rc;
    if (rgb_dev && !dir_dev && n > 0) return fail(VR_EINVAL, "null directions with n = %lld", (long long)n);
    if (rgb_dev && coef0_only(t))
        return fail(VR_EUNSUPPORTED, "eval unavailable for basis_dim %d (only coefficient 0 is resident)", t->dev.basis_dim);
    if (n == 0 || (!rgb_dev && !sigma_dev)) return VR_OK;
    int bc;
    if ((bc = buffer_check(t, xyz_dev, "xyz_dev")) || (rgb_dev && (bc = buffer_check(t, dir_dev, "dir_dev"))) ||
        (bc = buffer_check(t, rgb_dev, "rgb_dev")) || (bc = buffer_check(t, sigma_dev, "sigma_dev")))
        return bc;
    QueryLaunch Q{};
    Q.tree = t->dev;
    Q.xyz = xyz_dev; Q.dir = dir_dev; Q.n = n;
    Q.rgb = rgb_dev; Q.sigma = sigma_dev;
    basis_range(t, opt, &Q.bmin, &Q.bmax);
    VR_CUDA(query_launch(Q, t->dev.kbd, true, t->num_sms, (cudaStream_t)stream_));
    g_launches += 1;
    return VR_OK;
}

// The probe disc of render_kernel (volrend.cu:100-134) over frames the march has written (kernel: vr_probe.cu).
int vr_draw_probe(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt, const float probe_xyz[3],
                  int disp_size, const vr_rect* tile, uint8_t* rgba8_dev, float* rgba32f_dev,
                  unsigned long long rgba8_surf, void* stream_) {
    if (!probe_xyz) return fail(VR_EINVAL, "null probe position");
    if (rgba8_surf) {
        if (n_views != 1 || tile || rgba8_dev || rgba32f_dev)
            return fail(VR_EINVAL, "the surface form draws one full frame and no linear or float output");
    } else if (!rgba8_dev && !rgba32f_dev) {
        return fail(VR_EINVAL, "no output to draw into");
    }
    vr_rect r;
    const int rc = check_batch(t, cams, n_views, opt, tile, r);
    if (rc || n_views == 0) return rc;
    if (coef0_only(t))
        return fail(VR_EUNSUPPORTED, "probe unavailable for basis_dim %d (only coefficient 0 is resident)", t->dev.basis_dim);
    if (disp_size <= 0) return VR_OK;   // the reference's candidate pixels then all lie outside the disc
    // candidate corner, volrend.cu:100-101: y < S + 5 && x >= W - S - 5, in the 32-bit wrapping adds of the SASS
    const int W = cams[0].width, H = cams[0].height;
    const int y_end = (int)((uint32_t)disp_size + 5u), x_beg = (int)((uint32_t)W - (uint32_t)disp_size - 5u);
    const int cx0 = std::max(std::max(x_beg, 0), r.x0), cx1 = std::min(W, r.x0 + r.w);
    const int cy0 = r.y0, cy1 = std::min(std::min(y_end, H), r.y0 + r.h);
    if (cx0 >= cx1 || cy0 >= cy1) return VR_OK;
    const cudaStream_t stream = (cudaStream_t)stream_;
    ProbeLaunch P{};
    P.tree = t->dev;
    for (int i = 0; i < 3; ++i) P.probe[i] = probe_xyz[i];
    P.disp = disp_size;
    basis_range(t, opt, &P.bmin, &P.bmax);
    P.x0 = r.x0; P.y0 = r.y0; P.w = r.w; P.h = r.h;
    P.cx0 = cx0; P.cy0 = cy0; P.cw = cx1 - cx0; P.ch = cy1 - cy0;
    P.surf = (cudaSurfaceObject_t)rgba8_surf;
    const size_t px = (size_t)r.w * r.h;
    return for_chunks(n_views, kCamRing, [&](int v0, int nv) -> int {
        ProbeLaunch C = P;
        fill_cam(C.cam, &cams[v0]);
        C.n_views = nv;
        C.rgba8 = skip(rgba8_dev, 4 * px * v0);
        C.rgbaf = skip(reinterpret_cast<float4*>(rgba32f_dev), px * v0);
        LaunchDev L{};
        if (int rc = stage_cams(t, cams + v0, nv, stream, L)) return rc;
        C.cams = nv > 1 ? L.cams : nullptr;
        const cudaError_t e = probe_draw(C, t->dev.kbd, stream);
        if (e != cudaSuccess) return fail(VR_ECUDA, "probe overlay launch failed: %s", cudaGetErrorString(e));
        g_launches += 1;
        return VR_OK;
    });
}

// Mesh pass of cuda_renderer.cpp:103-112 without GL (kernels: vr_raster.cu).  The view matrix is
// w2c = affineInverse(c2w) (camera.cpp:65), folded with each model matrix in double on the host.
int vr_draw_meshes(const vr_camera* cam, const vr_mesh_desc* meshes, int n_meshes, uint8_t* rgba8_dev,
                   float* depth_dev, void* stream) {
    if (n_meshes < 0) return fail(VR_EINVAL, "negative mesh count %d", n_meshes);
    const int32_t off[2] = {0, n_meshes};
    return vr_draw_meshes_batch(cam, 1, meshes, off, rgba8_dev, depth_dev, stream);
}

// The views are drawn in launch groups: consecutive views with primitives, as many as keep the group's scratch
// within kRasterScratchBytes, its primitives below kRasterMaxPrims and its views within kRasterMaxViews.
int vr_draw_meshes_batch(const vr_camera* cams, int n_views, const vr_mesh_desc* meshes, const int32_t* mesh_off,
                         uint8_t* rgba8_dev, float* depth_dev, void* stream) {
    if (n_views < 0) return fail(VR_EINVAL, "negative view count %d", n_views);
    if (n_views == 0) return VR_OK;
    if (!cams) return fail(VR_EINVAL, "null camera");
    if (!mesh_off) return fail(VR_EINVAL, "null mesh_off");
    if (mesh_off[0] != 0) return fail(VR_EINVAL, "mesh_off[0] = %d, not 0", mesh_off[0]);
    for (int v = 0; v < n_views; ++v)
        if (mesh_off[v + 1] < mesh_off[v])
            return fail(VR_EINVAL, "mesh_off decreases at view %d (%d < %d)", v, mesh_off[v + 1], mesh_off[v]);
    if (mesh_off[n_views] > 0 && !meshes) return fail(VR_EINVAL, "null mesh array");
    if (!rgba8_dev || !depth_dev) return fail(VR_EINVAL, "mesh drawing needs colour and depth buffers");
    const int W = cams[0].width, H = cams[0].height;
    if (W <= 0 || H <= 0) return fail(VR_EINVAL, "zero-size frame %dx%d", W, H);
    if (W > kRasterMaxSide || H > kRasterMaxSide)
        return fail(VR_EINVAL, "frame %dx%d exceeds %d pixels per side", W, H, kRasterMaxSide);
    if (int rc = same_size(cams, n_views)) return rc;
    const long long npx = (long long)W * H;
    std::vector<RasterMesh> rm;
    std::vector<RasterFrame> rf;
    std::vector<long long> prims, caps;     // per entry of rf
    std::vector<size_t> first;              // per entry of rf: its first mesh in rm
    for (int v = 0; v < n_views; ++v) {
        const vr_camera* cam = &cams[v];
        const float* c = cam->c2w;  // column-major 3x4: R[r][k] = c[3k + r], translation c[9..11]
        double R[3][3], inv[3][3];
        for (int r = 0; r < 3; ++r)
            for (int k = 0; k < 3; ++k) R[r][k] = c[3 * k + r];
        const double det = R[0][0] * (R[1][1] * R[2][2] - R[1][2] * R[2][1]) + R[0][1] * (R[1][2] * R[2][0] - R[1][0] * R[2][2]) +
                           R[0][2] * (R[1][0] * R[2][1] - R[1][1] * R[2][0]);
        if (!(det != 0.0) || !std::isfinite(det)) return fail(VR_EINVAL, "view %d: camera rotation is singular", v);
        inv[0][0] = (R[1][1] * R[2][2] - R[1][2] * R[2][1]) / det;
        inv[0][1] = (R[0][2] * R[2][1] - R[0][1] * R[2][2]) / det;
        inv[0][2] = (R[0][1] * R[1][2] - R[0][2] * R[1][1]) / det;
        inv[1][0] = (R[1][2] * R[2][0] - R[1][0] * R[2][2]) / det;
        inv[1][1] = (R[0][0] * R[2][2] - R[0][2] * R[2][0]) / det;
        inv[1][2] = (R[0][2] * R[1][0] - R[0][0] * R[1][2]) / det;
        inv[2][0] = (R[1][0] * R[2][1] - R[1][1] * R[2][0]) / det;
        inv[2][1] = (R[0][1] * R[2][0] - R[0][0] * R[2][1]) / det;
        inv[2][2] = (R[0][0] * R[1][1] - R[0][1] * R[1][0]) / det;
        double V[3][4];  // w2c rows
        for (int r = 0; r < 3; ++r) {
            for (int k = 0; k < 3; ++k) V[r][k] = inv[r][k];
            V[r][3] = -((inv[r][0] * c[9] + inv[r][1] * c[10]) + inv[r][2] * c[11]);
        }
        const size_t m0 = rm.size();
        long long total = 0, large_cap = 0;
        for (int i = mesh_off[v]; i < mesh_off[v + 1]; ++i) {
            const vr_mesh_desc& d = meshes[i];
            if (d.face_size < 1 || d.face_size > 3)
                return fail(VR_EINVAL, "mesh %d: face_size %d (1 = points, 2 = lines, 3 = triangles)", i, d.face_size);
            if (d.n_verts < 0 || d.n_faces < 0)
                return fail(VR_EINVAL, "mesh %d: negative count (n_verts %d, n_faces %d)", i, d.n_verts, d.n_faces);
            if (!d.vert_dev && d.n_verts > 0) return fail(VR_EINVAL, "mesh %d: null vert_dev with %d vertices", i, d.n_verts);
            const long long np = d.faces_dev ? d.n_faces : d.n_verts / d.face_size;
            if (np == 0) continue;
            RasterMesh m{};
            m.vert = d.vert_dev; m.faces = d.faces_dev;
            m.n_verts = d.n_verts; m.face_size = d.face_size; m.unlit = d.unlit != 0;
            const float* M = d.model;  // column-major 4x4: M[r][k] = model[4k + r]
            for (int k = 0; k < 4; ++k)
                for (int r = 0; r < 3; ++r)
                    m.mv[3 * k + r] = (float)(((V[r][0] * M[4 * k] + V[r][1] * M[4 * k + 1]) + V[r][2] * M[4 * k + 2]) +
                                              V[r][3] * M[4 * k + 3]);
            for (int k = 0; k < 3; ++k)
                for (int r = 0; r < 3; ++r) m.m3[3 * k + r] = M[4 * k + r];
            m.base = total; m.n_prims = np;     // view-relative here; made launch-wide below
            total += np;
            large_cap += np * (d.face_size == 3 ? 6 : 1);
            if (total >= kRasterMaxPrims)
                return fail(VR_EINVAL, "view %d: more than %lld primitives", v, kRasterMaxPrims - 1);
            rm.push_back(m);
        }
        if (total == 0) continue;   // nothing to draw: the view's colour and depth stay
        RasterFrame f{};
        f.W = W; f.H = H; f.fx = cam->fx; f.fy = cam->fy;
        f.cx = 0.5f * W; f.cy = 0.5f * H;
        // camPos = -transpose(mat3(V)) * V[3] (mesh.cpp:376): the eye only when the rotation is orthonormal; a
        // rotation scaled by s gives t / s^2
        for (int k = 0; k < 3; ++k)
            f.cam_pos[k] = (float)-((V[0][k] * V[0][3] + V[1][k] * V[1][3]) + V[2][k] * V[2][3]);
        f.rgba8 = rgba8_dev + (size_t)v * 4 * npx;
        f.depth = depth_dev + (size_t)v * npx;
        rf.push_back(f);
        prims.push_back(total);
        caps.push_back(large_cap);
        first.push_back(m0);
    }
    if (int rc = need_device(nullptr)) return rc;
    first.push_back(rm.size());
    for (size_t g0 = 0; g0 < rf.size();) {
        // grow the group while it stays within the bounds; a first view that exceeds kRasterScratchBytes alone
        // still runs, alone
        size_t g1 = g0 + 1;
        long long total = prims[g0];
        size_t bytes = raster_view_bytes(npx, caps[g0]);
        while (g1 < rf.size() && g1 - g0 < (size_t)kRasterMaxViews && total + prims[g1] < kRasterMaxPrims &&
               bytes + raster_view_bytes(npx, caps[g1]) <= kRasterScratchBytes) {
            total += prims[g1];
            bytes += raster_view_bytes(npx, caps[g1]);
            ++g1;
        }
        long long base = 0, large_off = 0;
        for (size_t k = g0; k < g1; ++k) {
            rf[k].large_off = large_off;
            large_off += caps[k];
            for (size_t i = first[k]; i < first[k + 1]; ++i) {
                rm[i].view = (int)(k - g0);
                rm[i].base = base;
                base += rm[i].n_prims;
            }
        }
        VR_CUDA(raster_draw(rf.data() + g0, (int)(g1 - g0), rm.data() + first[g0], (int)(first[g1] - first[g0]), total,
                            large_off, (cudaStream_t)stream));
        g_launches += kRasterLaunches;
        g0 = g1;
    }
    return VR_OK;
}

}  // extern "C"

namespace {
// The tree as the wireframe walk reads it.
WireTree wire_tree(const vr_tree* t) {
    WireTree w{};
    w.wide = t->wide; w.n_tables = t->n_tables; w.wide_p = t->dev.wide_p; w.max_level = t->dev.max_depth;
    for (int i = 0; i < 3; ++i) { w.offset[i] = t->dev.offset[i]; w.scale[i] = t->dev.scale[i]; }
    return w;
}

// The tree's cells per level (t->wire_levels), counted on the first call (which synchronises `stream`).
int ensure_wire_levels(const vr_tree* t, const WireTree& w, cudaStream_t stream) {
    vr_tree* mt = const_cast<vr_tree*>(t);
    std::lock_guard<std::mutex> lk(mt->wire_mu);
    if (!mt->wire_ready) {
        int launches = 0;
        const cudaError_t e = wire_levels(w, mt->wire_levels, stream, &launches);
        g_launches += launches;
        if (e != cudaSuccess) return cuda_fail(e, "wireframe cell count");
        mt->wire_ready = true;
    }
    return VR_OK;
}
// VR_EINVAL unless every non-null buffer is device (or managed) memory of the current device.
struct NamedBuffer {
    const void* p;
    const char* name;
};
int current_device_buffers(std::initializer_list<NamedBuffer> bufs) {
    int dev = 0;
    VR_CUDA(cudaGetDevice(&dev));
    for (const auto& b : bufs) {
        if (!b.p) continue;
        cudaPointerAttributes pa{};
        if (cudaPointerGetAttributes(&pa, b.p) != cudaSuccess) {
            cudaGetLastError();
            return fail(VR_EINVAL, "%s is not a CUDA allocation", b.name);
        }
        if ((pa.type != cudaMemoryTypeDevice && pa.type != cudaMemoryTypeManaged) || pa.device != dev)
            return fail(VR_EINVAL, "%s is not device memory of the current device %d", b.name, dev);
    }
    return VR_OK;
}
}  // namespace

extern "C" {

// N3Tree::gen_wireframe (n3tree.cpp:365-434) from the device tables (kernels: vr_wire.cu).
int vr_tree_wireframe(const vr_tree* t, int max_depth, float* vert_dev, int64_t max_verts, int64_t* n_verts_out,
                      void* stream_) {
    if (!t || !n_verts_out) return fail(VR_EINVAL, "null argument");
    if (int rc = need_device(t)) return rc;
    cudaStream_t stream = (cudaStream_t)stream_;
    const WireTree w = wire_tree(t);
    if (int rc = ensure_wire_levels(t, w, stream)) return rc;
    const long long n = 24 * wire_cells(w, t->wire_levels, max_depth);
    *n_verts_out = n;
    if (!vert_dev) return VR_OK;
    if (max_verts < n) return fail(VR_EINVAL, "the wireframe at max_depth %d has %lld vertices, the buffer holds %lld", max_depth, n, (long long)max_verts);
    int launches = 0;
    const cudaError_t e = wire_fill(w, t->wire_levels, max_depth, vert_dev, stream, &launches);
    g_launches += launches;
    if (e != cudaSuccess) return cuda_fail(e, "wireframe");
    return VR_OK;
}

// Forward neighbours of every leaf slot (kernels: vr_tv.cu, on the wireframe's walk).
int vr_tree_leaf_neighbors(const vr_tree* t, int32_t* nbr_dev, void* stream_) {
    if (!t) return fail(VR_EINVAL, "null tree");
    int rc = need_device(t);
    if (rc) return rc;
    if ((rc = need_slot_map(t, "vr_tree_leaf_neighbors"))) return rc;
    if (!nbr_dev) return fail(VR_EINVAL, "null neighbour buffer");
    if ((rc = buffer_check(t, nbr_dev, "nbr_dev"))) return rc;
    cudaStream_t stream = (cudaStream_t)stream_;
    const WireTree w = wire_tree(t);
    if ((rc = ensure_wire_levels(t, w, stream))) return rc;
    int launches = 0;
    const cudaError_t e = tv_neighbors(w, t->wire_levels, t->dev, t->wslot, t->info.capacity * 8, nbr_dev, stream,
                                       &launches);
    g_launches += launches;
    if (e != cudaSuccess) return cuda_fail(e, "leaf neighbours");
    return VR_OK;
}

// Total variation between neighbouring leaves, its gradient added to grad_dev (kernels: vr_tv.cu).
int vr_tree_leaf_tv(const vr_tree* t, const int32_t* nbr_dev, const float* data_dev, float lambda_sigma,
                    float lambda_color, float* grad_dev, double* energy_dev, void* stream_) {
    if (!t) return fail(VR_EINVAL, "null tree");
    int rc = need_device(t);
    if (rc) return rc;
    if (!(lambda_sigma >= 0.f) || !(lambda_color >= 0.f) || std::isinf(lambda_sigma) || std::isinf(lambda_color))
        return fail(VR_EINVAL, "TV weights must be finite and >= 0 (sigma %g, colour %g)", lambda_sigma, lambda_color);
    if ((rc = need_slot_map(t, "vr_tree_leaf_tv"))) return rc;
    if (!nbr_dev || !data_dev || !grad_dev) return fail(VR_EINVAL, "null neighbour, data or gradient buffer");
    if ((rc = buffer_check(t, nbr_dev, "nbr_dev")) || (rc = buffer_check(t, data_dev, "data_dev")) ||
        (rc = buffer_check(t, grad_dev, "grad_dev")) || (rc = buffer_check(t, energy_dev, "energy_dev")))
        return rc;
    if (lambda_sigma == 0.f && lambda_color == 0.f) return VR_OK;
    cudaStream_t stream = (cudaStream_t)stream_;
    const WireTree w = wire_tree(t);
    if ((rc = ensure_wire_levels(t, w, stream))) return rc;
    long long n_leaf = 0;
    for (int l = 0; l < kWireLevels; ++l) n_leaf += t->wire_levels.leaf[l];
    // the columns of vr_tree_leaf_grads: RGBA channels 0..2, or coefficient k < kbd of channel c at c * basis_dim + k
    TvColumns cols;
    cols.data_dim = t->data_dim;
    cols.n_coef = t->dev.kbd > 0 ? t->dev.kbd : 1;
    cols.coef_stride = t->dev.kbd > 0 ? t->dev.basis_dim : 1;
    int launches = 0;
    const cudaError_t e = tv_pass(data_dev, nbr_dev, t->info.capacity * 8, cols, (double)lambda_sigma / n_leaf,
                                  (double)lambda_color / n_leaf, grad_dev, energy_dev, stream, &launches);
    g_launches += launches;
    if (e != cudaSuccess) return cuda_fail(e, "leaf TV");
    return VR_OK;
}

// estimate_normals (mesh.cpp:63-97) on a device vertex buffer (kernels: vr_normals.cu).
int vr_mesh_estimate_normals(float* vert_dev, int64_t n_verts, const uint32_t* faces_dev, int64_t n_faces,
                             void* stream) {
    if (n_verts < 0 || n_faces < 0)
        return fail(VR_EINVAL, "negative count (n_verts %lld, n_faces %lld)", (long long)n_verts, (long long)n_faces);
    if (!vert_dev && n_verts > 0) return fail(VR_EINVAL, "null vert_dev with %lld vertices", (long long)n_verts);
    if (n_verts > INT32_MAX) return fail(VR_EINVAL, "%lld vertices: at most %d", (long long)n_verts, INT32_MAX);
    if (faces_dev && n_faces > INT32_MAX / 3)
        return fail(VR_EINVAL, "%lld faces: at most %d face corners", (long long)n_faces, INT32_MAX);
    if (int rc = need_device(nullptr)) return rc;
    int launches = 0;
    const cudaError_t e = normals_estimate(vert_dev, n_verts, faces_dev, n_faces, (cudaStream_t)stream, &launches);
    g_launches += launches;
    if (e != cudaSuccess) return cuda_fail(e, "mesh normals");
    return VR_OK;
}

// Median-cut compression into the quant_colors / quant_map format (kernels: vr_quant.cu).
int vr_tree_compress(const uint16_t* data_dev, int64_t n_child, int32_t data_dim, float sigma_thresh, int32_t n_retain,
                     int32_t bits, uint16_t* quant_colors_dev, uint16_t* quant_map_dev, uint16_t* sigma_dev,
                     uint16_t* data_retained_dev, int64_t* n_kept_out, void* stream) {
    if (!n_kept_out) return fail(VR_EINVAL, "null n_kept_out");
    *n_kept_out = 0;
    if (bits < 1 || bits > 16) return fail(VR_EINVAL, "bits %d outside [1, 16]", bits);
    if (n_retain < 0) return fail(VR_EINVAL, "retain %d < 0", n_retain);
    if (data_dim < 4 || (data_dim - 1) % 3 != 0)
        return fail(VR_EINVAL, "data_dim %d is not 3 * basis_dim + 1", data_dim);
    const int basis = (data_dim - 1) / 3, n_quant = basis - n_retain;
    if (n_quant < 1)
        return fail(VR_EINVAL, "retain %d leaves no basis function to quantise (the tree has %d)", n_retain, basis);
    if (n_child < 0 || n_child > INT32_MAX)
        return fail(VR_EINVAL, "n_child %lld outside [0, %d]", (long long)n_child, INT32_MAX);
    if ((!data_dev && n_child > 0) || !quant_colors_dev || (!quant_map_dev && n_child > 0) || (!sigma_dev && n_child > 0))
        return fail(VR_EINVAL, "null argument");
    if ((n_retain > 0) != (data_retained_dev != nullptr))
        return fail(VR_EINVAL, "data_retained_dev must be NULL exactly when n_retain == 0");
    if (int rc = need_device(nullptr)) return rc;
    QuantArgs a{};
    a.data = data_dev; a.n_child = n_child; a.data_dim = data_dim; a.n_retain = n_retain; a.bits = bits;
    a.thresh = __half2float(__float2half_rn(sigma_thresh));   // sigma > thresh compared as fp16
    a.colors = quant_colors_dev; a.qmap = quant_map_dev; a.sigma = sigma_dev; a.retained = data_retained_dev;
    long long kept = 0;
    int reject = kQuantOk, launches = 0;
    const cudaError_t e = quant_compress(a, (cudaStream_t)stream, &kept, &reject, &launches);
    g_launches += launches;
    if (e != cudaSuccess) return cuda_fail(e, "tree compress");
    if (reject == kQuantNonFinite) return fail(VR_EINVAL, "a quantised coefficient of a kept voxel is Inf or NaN");
    if (reject == kQuantTooManyPoints)
        return fail(VR_EINVAL, "%lld kept voxels x %d quantised basis functions exceed %d points", kept, n_quant, INT32_MAX);
    *n_kept_out = kept;
    return VR_OK;
}

// Canonical tree of a set of voxel cells (kernels: vr_build.cu).
int vr_tree_build(const int32_t* cells_dev, const uint16_t* rows_dev, int64_t n, int32_t data_dim, uint32_t flags,
                  int32_t* child_dev, uint16_t* data_dev, int64_t max_nodes, int64_t* n_nodes_out, void* stream) {
    if (!n_nodes_out) return fail(VR_EINVAL, "null n_nodes_out");
    if (n < 0 || n > INT32_MAX) return fail(VR_EINVAL, "n %lld outside [0, %d]", (long long)n, INT32_MAX);
    if (data_dim < 1) return fail(VR_EINVAL, "data_dim %d < 1", data_dim);
    if (flags & ~VR_BUILD_MERGE) return fail(VR_EINVAL, "unknown flags 0x%x", flags);
    if (n > 0 && (!cells_dev || !rows_dev)) return fail(VR_EINVAL, "null cells_dev or rows_dev with n = %lld", (long long)n);
    if ((child_dev == nullptr) != (data_dev == nullptr))
        return fail(VR_EINVAL, "child_dev and data_dev must both be NULL (count only) or both be given");
    if (int rc = need_device(nullptr)) return rc;
    if (int rc = current_device_buffers({{cells_dev, "cells_dev"}, {rows_dev, "rows_dev"}, {child_dev, "child_dev"},
                                         {data_dev, "data_dev"}}))
        return rc;
    BuildArgs a{};
    a.cells = cells_dev; a.rows = rows_dev; a.n = n; a.data_dim = data_dim; a.merge = (flags & VR_BUILD_MERGE) != 0;
    a.child = child_dev; a.data = data_dev; a.max_nodes = max_nodes; a.node_limit = 0xffffffffll / 8;
    long long nodes = 0;
    int reject = kBuildOk, launches = 0;
    const cudaError_t e = tree_build(a, (cudaStream_t)stream, &nodes, &reject, &launches);
    g_launches += launches;
    if (e != cudaSuccess) return cuda_fail(e, "tree build");
    switch (reject) {
        case kBuildBadCell: return fail(VR_EINVAL, "a cell has a level outside [1, 23] or a coordinate outside [0, 2^level)");
        case kBuildOverlap: return fail(VR_EINVAL, "two cells are equal or one contains the other");
        case kBuildTooLarge:
            return fail(VR_EINVAL, "the tree has %lld nodes: more than the %lld the int32 links and the u32 slot map address",
                        nodes, a.node_limit);
        case kBuildCapacity: return fail(VR_EINVAL, "the tree has %lld nodes, the outputs room for %lld", nodes, (long long)max_nodes);
        default: break;
    }
    *n_nodes_out = nodes;
    return VR_OK;
}

// Marching cubes over the tree's leaf sigma on a level-`depth` lattice (kernels: vr_iso.cu, normals: vr_normals.cu).
int vr_tree_isosurface(const vr_tree* t, int32_t depth, float level, const vr_options* opt, uint32_t flags,
                       float* vert_dev, int64_t max_verts, uint32_t* faces_dev, int64_t max_faces, int64_t* n_verts_out,
                       int64_t* n_faces_out, void* stream_) {
    if (!t) return fail(VR_EINVAL, "null tree");
    if (!n_verts_out || !n_faces_out) return fail(VR_EINVAL, "null n_verts_out or n_faces_out");
    if (depth < 1 || depth > kIsoMaxDepth) return fail(VR_EINVAL, "depth %d outside [1, %d]", depth, kIsoMaxDepth);
    if (!std::isfinite(level) || !(level > 0.f)) return fail(VR_EINVAL, "level %g must be finite and > 0", level);
    if (flags & ~VR_ISO_COLOR) return fail(VR_EINVAL, "unknown flags 0x%x", flags);
    if ((vert_dev == nullptr) != (faces_dev == nullptr))
        return fail(VR_EINVAL, "vert_dev and faces_dev must both be NULL (count only) or both be given");
    if (int rc = need_device(t)) return rc;
    if (t->dev.ndc_width > 0.f) return fail(VR_EUNSUPPORTED, "isosurfaces of NDC trees are not supported");
    const bool color = (flags & VR_ISO_COLOR) != 0;
    if (color && coef0_only(t))
        return fail(VR_EUNSUPPORTED, "colours unavailable for basis_dim %d (only coefficient 0 is resident)",
                    t->dev.basis_dim);
    int rc;
    if ((rc = buffer_check(t, vert_dev, "vert_dev")) || (rc = buffer_check(t, faces_dev, "faces_dev"))) return rc;
    cudaStream_t stream = (cudaStream_t)stream_;
    IsoArgs a{};
    a.tree = t->dev; a.depth = depth; a.level = level; a.vert = vert_dev; a.faces = faces_dev; a.color = color;
    if (const char* e = getenv("VR_ISO_SLAB_PLANES")) a.slab_planes = atoi(e);
    long long nv = 0, nf = 0;
    int launches = 0;
    cudaError_t e = iso_run(a, false, stream, &nv, &nf, &launches);
    g_launches += launches;
    if (e != cudaSuccess) return cuda_fail(e, "isosurface count");
    *n_verts_out = nv;
    *n_faces_out = nf;
    if (nv > INT32_MAX || nf > INT32_MAX / 3)
        return fail(VR_EUNSUPPORTED, "the mesh has %lld vertices and %lld faces: at most %d vertices and face corners",
                    nv, nf, INT32_MAX);
    if (!vert_dev) return VR_OK;
    if (max_verts < nv || max_faces < nf)
        return fail(VR_EINVAL, "the mesh has %lld vertices and %lld faces, the outputs room for %lld and %lld", nv, nf,
                    (long long)max_verts, (long long)max_faces);
    launches = 0;
    e = iso_run(a, true, stream, &nv, &nf, &launches);
    if (e == cudaSuccess) e = normals_estimate(vert_dev, nv, faces_dev, nf, stream, &launches);
    if (e == cudaSuccess && color) {
        int32_t bmin, bmax;
        basis_range(t, opt, &bmin, &bmax);
        e = iso_color(t->dev, depth, vert_dev, nv, bmin, bmax, stream, &launches);
    }
    g_launches += launches;
    if (e != cudaSuccess) return cuda_fail(e, "isosurface");
    return VR_OK;
}

// Per-view SSIM and its gradient (kernels: vr_ssim.cu).
int vr_image_ssim(const float* x_dev, int x_channels, const float* y_dev, int y_channels, int n_views, int height,
                  int width, double* ssim_dev, float* dx_dev, float dx_scale, void* stream) {
    if (n_views < 0) return fail(VR_EINVAL, "n_views %d < 0", n_views);
    if (height < 11 || width < 11) return fail(VR_EINVAL, "images are %dx%d: SSIM needs at least 11x11", width, height);
    if ((x_channels != 3 && x_channels != 4) || (y_channels != 3 && y_channels != 4))
        return fail(VR_EINVAL, "channels %d and %d: each must be 3 or 4", x_channels, y_channels);
    if (!std::isfinite(dx_scale)) return fail(VR_EINVAL, "dx_scale %g is not finite", dx_scale);
    if (!x_dev || !y_dev || !ssim_dev) return fail(VR_EINVAL, "null x_dev, y_dev or ssim_dev");
    if (int rc = need_device(nullptr)) return rc;
    if (int rc = current_device_buffers({{x_dev, "x_dev"}, {y_dev, "y_dev"}, {ssim_dev, "ssim_dev"}, {dx_dev, "dx_dev"}}))
        return rc;
    int launches = 0;
    const cudaError_t e = ssim_pass(x_dev, x_channels, y_dev, y_channels, n_views, height, width, ssim_dev, dx_dev,
                                    dx_scale, (cudaStream_t)stream, &launches);
    g_launches += launches;
    if (e != cudaSuccess) return cuda_fail(e, "image SSIM");
    return VR_OK;
}

}  // extern "C"
