// volrend_backend.cu -- C++ drop-in for volrend's CUDA backend, over the volrend_b200 C-ABI.
//
// Link this (plus libvolrend_b200.so) INSTEAD of the reference's src/cuda/volrend.cu,
// src/cuda/n3tree.cu, src/cuda/common.cu and src/cuda_renderer.cpp.  The reference's loader,
// camera, option parsing and CLI (src/n3tree.cpp, src/camera.cpp, src/opts.cpp,
// main_headless.cpp) and all of its headers are used unchanged; this file only defines the
// symbols those callers expect:
//   volrend::launch_renderer         include/volrend/cuda/renderer_kernel.hpp:9-12
//   volrend::N3Tree::load_cuda/free_cuda   include/volrend/n3tree.hpp:101-105 (called from
//                                    src/n3tree.cpp:107,150-152,168-170)
//   volrend::cuda_assert             include/volrend/cuda/common.cuh:78-79 (abort-on-error
//                                    semantics of src/cuda/common.cu:8-21 are preserved here;
//                                    the C-ABI underneath never aborts)
//   volrend::VolumeRenderer          include/volrend/renderer.hpp:11-42, GL-free offscreen Impl
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <unordered_map>

#include "volrend/common.hpp"
#include "volrend/cuda/common.cuh"
#include "volrend/cuda/renderer_kernel.hpp"
#include "volrend/n3tree.hpp"
#include "volrend/renderer.hpp"

#include "volrend_b200.h"
#include "volrend_b200_shim.hpp"

namespace volrend {

// ---------------------------------------------------------------- cuda_assert
cudaError_t cuda_assert(const cudaError_t code, const char* const file, const int line, const bool abort) {
    if (code != cudaSuccess) {
        fprintf(stderr, "cuda_assert: %s %s %d\n", cudaGetErrorString(code), file, line);
        if (abort) {
            cudaDeviceReset();
            exit(code);
        }
    }
    return code;
}

namespace {

[[noreturn]] void die(const char* what, int rc) {
    // same contract as cuda(...): print, reset, exit
    fprintf(stderr, "volrend_b200: %s failed (%d): %s\n", what, rc, vr_last_error());
    cudaDeviceReset();
    exit(rc < 0 ? -rc : 1);
}

std::mutex g_mu;
std::unordered_map<const N3Tree*, vr_tree*> g_trees;   // N3Tree -> re-laid-out device tree

struct SurfKey { cudaArray_t arr; };
struct SurfEntry { cudaSurfaceObject_t surf; size_t w, h; int fmt_x; };
std::unordered_map<cudaArray_t, SurfEntry> g_surfs;    // caller-owned cudaArray -> surface object

cudaSurfaceObject_t surface_for(cudaArray_t arr) {
    cudaChannelFormatDesc desc;
    cudaExtent ext;
    unsigned int flags = 0;
    cuda(ArrayGetInfo(&desc, &ext, &flags, arr));
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_surfs.find(arr);
    if (it != g_surfs.end()) {
        if (it->second.w == ext.width && it->second.h == ext.height && it->second.fmt_x == desc.x)
            return it->second.surf;
        cudaDestroySurfaceObject(it->second.surf);   // the array was re-created with a new shape
        g_surfs.erase(it);
    }
    cudaResourceDesc res;
    memset(&res, 0, sizeof(res));
    res.resType = cudaResourceTypeArray;
    res.res.array.array = arr;
    cudaSurfaceObject_t s = 0;
    cuda(CreateSurfaceObject(&s, &res));
    g_surfs[arr] = SurfEntry{s, ext.width, ext.height, desc.x};
    return s;
}

vr_tree* device_tree(const N3Tree& tree) {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_trees.find(&tree);
    return it == g_trees.end() ? nullptr : it->second;
}

void to_c(const Camera& cam, vr_camera& c) {
    c.width = cam.width; c.height = cam.height; c.fx = cam.fx; c.fy = cam.fy;
    // glm::mat4x3 is 4 columns of vec3 = 12 contiguous floats, column-major (camera.cpp:52-55)
    memcpy(c.c2w, &cam.transform[0][0], 12 * sizeof(float));
}
void to_c(const RenderOptions& o, vr_options& c) {
    c.step_size = o.step_size; c.sigma_thresh = o.sigma_thresh; c.stop_thresh = o.stop_thresh;
    c.background_brightness = o.background_brightness;
    for (int i = 0; i < 6; ++i) c.render_bbox[i] = o.render_bbox[i];
    c.basis_minmax[0] = o.basis_minmax[0]; c.basis_minmax[1] = o.basis_minmax[1];
    for (int i = 0; i < 3; ++i) c.rot_dirs[i] = o.rot_dirs[i];
    c.render_depth = o.render_depth ? 1 : 0;
}

}  // namespace

// ---------------------------------------------------------------- N3Tree device side
void N3Tree::load_cuda() {
    free_cuda();
    vr_tree_desc d;
    memset(&d, 0, sizeof(d));
    d.child = child_.data<int32_t>();
    d.data = reinterpret_cast<const uint16_t*>(data_.data<__half>());
    d.extra = extra_.data_holder.size() ? extra_.data<float>() : nullptr;
    d.capacity = capacity; d.N = N; d.data_dim = data_dim;
    d.format = (int)data_format.format; d.basis_dim = data_format.basis_dim;
    for (int i = 0; i < 3; ++i) { d.offset[i] = offset[i]; d.scale[i] = scale[i]; }
    d.use_ndc = use_ndc ? 1 : 0;
    d.ndc_width = ndc_width; d.ndc_height = ndc_height; d.ndc_focal = ndc_focal;
    vr_tree* t = nullptr;
    const int rc = vr_tree_create(&d, &t);
    if (rc != VR_OK) die("vr_tree_create", rc);
    {
        std::lock_guard<std::mutex> lk(g_mu);
        g_trees[this] = t;
    }
    cuda_loaded_ = true;
}

void N3Tree::free_cuda() {
    vr_tree* t = nullptr;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        auto it = g_trees.find(this);
        if (it != g_trees.end()) { t = it->second; g_trees.erase(it); }
    }
    if (t) vr_tree_destroy(t);
}

// ---------------------------------------------------------------- launch_renderer
__host__ void launch_renderer(const N3Tree& tree, const Camera& cam, const RenderOptions& options,
                              cudaArray_t& image_arr, cudaArray_t& depth_arr, cudaStream_t stream,
                              bool offscreen) {
    vr_tree* t = device_tree(tree);
    if (!t) {
        fprintf(stderr, "volrend_b200: launch_renderer on a tree that is not on the device\n");
        return;
    }
    vr_camera c;
    vr_options o;
    to_c(cam, c);
    to_c(options, o);
    if (tree.use_ndc) {
        // NDC parameters are filled in by N3Tree::open after load_cuda ran (n3tree.cpp:130-152
        // computes them before load_cuda, but callers may toggle use_ndc) -- nothing to do here.
    }
    const cudaSurfaceObject_t surf = surface_for(image_arr);
    cudaSurfaceObject_t dsurf = 0;
    if (!offscreen) {
        if (!depth_arr) {
            fprintf(stderr, "volrend_b200: launch_renderer(offscreen=false) needs a depth array\n");
            return;
        }
        dsurf = surface_for(depth_arr);
    }
    const int rc = vr_render_surface(t, &c, &o, (unsigned long long)surf, (unsigned long long)dsurf, (void*)stream);
    if (rc != VR_OK) die("vr_render_surface", rc);
    if (options.enable_probe) {   // the lumisphere probe disc of volrend.cu:100-134
        const int prc = vr_draw_probe(t, &c, 1, &o, options.probe, options.probe_disp_size, nullptr, nullptr, nullptr,
                                      (unsigned long long)surf, (void*)stream);
        if (prc == VR_EUNSUPPORTED) {
            static bool warned = false;
            if (!warned) { fprintf(stderr, "volrend_b200: enable_probe disc not drawn: %s\n", vr_last_error()); warned = true; }
        } else if (prc != VR_OK) {
            die("vr_draw_probe", prc);
        }
    }
}

// ---------------------------------------------------------------- VolumeRenderer (GL-free)
namespace {
struct OffscreenTarget {   // what volrend_b200_read_pixels needs to see of an Impl
    cudaArray_t array = nullptr;
    cudaStream_t stream = nullptr;
    int w = 0, h = 0;
};
}  // namespace

struct VolumeRenderer::Impl : OffscreenTarget {
    Impl(Camera& camera, RenderOptions& options) : camera(camera), options(options) {
        cuda(StreamCreateWithFlags(&stream, cudaStreamDefault));
    }
    ~Impl() {
        if (array) cudaFreeArray(array);
        cudaStreamDestroy(stream);
    }
    void resize(int width, int height) {
        if (array && width == w && height == h) return;
        if (array) cuda(FreeArray(array));
        cudaChannelFormatDesc cd = cudaCreateChannelDesc(8, 8, 8, 8, cudaChannelFormatKindUnsigned);
        cuda(MallocArray(&array, &cd, width, height, cudaArraySurfaceLoadStore));
        w = width; h = height;
    }
    void render() {
        camera._update();
        if (!array) resize(camera.width, camera.height);
        if (tree == nullptr || !tree->is_cuda_loaded()) return;
        cudaArray_t depth = nullptr;
        launch_renderer(*tree, camera, options, array, depth, stream, true);
    }
    Camera& camera;
    RenderOptions& options;
    N3Tree* tree = nullptr;
};

namespace {
std::unordered_map<const VolumeRenderer*, OffscreenTarget*>& impls() {
    static std::unordered_map<const VolumeRenderer*, OffscreenTarget*> m;
    return m;
}
}  // namespace

VolumeRenderer::VolumeRenderer() : impl_(std::make_unique<Impl>(camera, options)) {
    std::lock_guard<std::mutex> lk(g_mu);
    impls()[this] = impl_.get();
}
VolumeRenderer::~VolumeRenderer() {
    std::lock_guard<std::mutex> lk(g_mu);
    impls().erase(this);
}
void VolumeRenderer::render() { impl_->render(); }
void VolumeRenderer::set(N3Tree& tree) {
    impl_->tree = &tree;
    // cuda_renderer.cpp:176-177
    options.basis_minmax[0] = 0;
    options.basis_minmax[1] = std::max(tree.data_format.basis_dim - 1, 0);
}
void VolumeRenderer::clear() { impl_->tree = nullptr; }
void VolumeRenderer::resize(int width, int height) {
    camera.width = width;
    camera.height = height;
    impl_->resize(width, height);
}
const char* VolumeRenderer::get_backend() { return "CUDA"; }

}  // namespace volrend

// ---------------------------------------------------------------- offscreen read-back helper
bool volrend_b200_read_pixels(volrend::VolumeRenderer& r, uint8_t* rgba_host) {
    volrend::OffscreenTarget* impl = nullptr;
    {
        std::lock_guard<std::mutex> lk(volrend::g_mu);
        auto it = volrend::impls().find(&r);
        if (it != volrend::impls().end()) impl = it->second;
    }
    if (!impl || !impl->array) return false;
    return cudaMemcpy2DFromArrayAsync(rgba_host, 4 * impl->w, impl->array, 0, 0, 4 * impl->w, impl->h,
                                      cudaMemcpyDeviceToHost, impl->stream) == cudaSuccess &&
           cudaStreamSynchronize(impl->stream) == cudaSuccess;
}
