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
//   volrend::VolumeRenderer          include/volrend/renderer.hpp:11-42, GL-free Impl: the offscreen march, or
//                                    with meshes, the probe cube or the grid the mesh pass of
//                                    cuda_renderer.cpp:83-126 (volrend::Mesh: mesh_b200.cpp)
#include <algorithm>
#include <cmath>
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
#include "mesh_pass_b200.hpp"

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

// GL's clear of the mesh framebuffer: colour (bg, bg, bg, 255) and ray distance 1e9
__global__ void clear_mesh_target(uint32_t* rgba, float* depth, size_t n, uint32_t rgba_word) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        rgba[i] = rgba_word;
        depth[i] = 1e9f;
    }
}
}  // namespace

struct VolumeRenderer::Impl : OffscreenTarget {
    Impl(Camera& camera, RenderOptions& options, std::vector<Mesh>& meshes)
        : camera(camera), options(options), meshes(meshes) {
        cuda(StreamCreateWithFlags(&stream, cudaStreamDefault));
        // the probe marker of cuda_renderer.cpp:25-38: black, faces -z/+z blue, -y/+y green, -x/+x red
        probe_ = Mesh::Cube(glm::vec3(0.f));
        probe_.name = "_probe_cube";
        probe_.visible = false;
        probe_.scale = 0.05f;
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 12; ++j) probe_.vert[(size_t)(12 * i + j) * 9 + 3 + 2 - i] = 1.f;
        probe_.unlit = true;
        probe_.update();
    }
    ~Impl() {
        if (array) cudaFreeArray(array);
        if (depth_array_) cudaFreeArray(depth_array_);
        if (rgba_lin_) cudaFree(rgba_lin_);
        if (depth_lin_) cudaFree(depth_lin_);
        if (wire_dev_) cudaFree(wire_dev_);
        cudaStreamDestroy(stream);
    }
    void resize(int width, int height) {
        if (array && width == w && height == h) return;
        if (array) cuda(FreeArray(array));
        cudaChannelFormatDesc cd = cudaCreateChannelDesc(8, 8, 8, 8, cudaChannelFormatKindUnsigned);
        cuda(MallocArray(&array, &cd, width, height, cudaArraySurfaceLoadStore));
        w = width; h = height;
    }
    void set(N3Tree& t) {
        tree = &t;
        probe_.scale = 0.02f / t.scale[0];   // cuda_renderer.cpp:178
        wire_valid_ = false;
    }
    void clear() {
        tree = nullptr;
        wire_valid_ = false;
    }
    void render() {
        camera._update();
        if (!array) resize(camera.width, camera.height);
        probe_.visible = options.enable_probe;   // cuda_renderer.cpp:94-95
        for (int i = 0; i < 3; ++i) probe_.translation[i] = options.probe[i];
        const bool has_tree = tree != nullptr && tree->is_cuda_loaded();
        bool mesh_pass = probe_.visible || (options.show_grid && has_tree);
        for (const Mesh& m : meshes) mesh_pass = mesh_pass || m.visible;
        if (mesh_pass) {
            render_meshes(has_tree);
            return;
        }
        if (!has_tree) return;
        cudaArray_t depth = nullptr;
        launch_renderer(*tree, camera, options, array, depth, stream, true);
    }

    // cuda_renderer.cpp:83-126: clear, draw the meshes, the probe cube and the grid, composite the volume over them
    void render_meshes(bool has_tree) {
        if (camera.width != w || camera.height != h) resize(camera.width, camera.height);
        ensure_mesh_target();
        const double bg = std::min(std::max((double)options.background_brightness, 0.0), 1.0);
        const uint32_t b = (uint32_t)std::nearbyint(bg * 255.0);   // round half to even, as Python's round()
        const size_t n = (size_t)w * h;
        if (n) {
            const int blocks = (int)std::min<size_t>((n + 255) / 256, 4096);
            clear_mesh_target<<<blocks, 256, 0, stream>>>((uint32_t*)rgba_lin_, depth_lin_, n,
                                                          b | (b << 8) | (b << 16) | (0xffu << 24));
            cuda(GetLastError());
        }
        b200::MeshPass pass;
        b200::set_current_mesh_pass(&pass);
        for (const Mesh& mesh : meshes) mesh.draw(camera.w2c, camera.K);
        probe_.draw(camera.w2c, camera.K);
        b200::set_current_mesh_pass(nullptr);
        if (options.show_grid && has_tree) append_grid(pass);
        vr_camera c;
        to_c(camera, c);
        if (!pass.meshes.empty()) {
            const int rc = vr_draw_meshes(&c, pass.meshes.data(), (int)pass.meshes.size(), rgba_lin_, depth_lin_,
                                          (void*)stream);
            if (rc != VR_OK) die("vr_draw_meshes", rc);
        }
        cuda(Memcpy2DToArrayAsync(array, 0, 0, rgba_lin_, 4 * (size_t)w, 4 * (size_t)w, h,
                                  cudaMemcpyDeviceToDevice, stream));
        if (has_tree) {
            cuda(Memcpy2DToArrayAsync(depth_array_, 0, 0, depth_lin_, 4 * (size_t)w, 4 * (size_t)w, h,
                                      cudaMemcpyDeviceToDevice, stream));
            launch_renderer(*tree, camera, options, array, depth_array_, stream, false);
        }
    }

    // RGBA8 and ray-distance buffers for vr_draw_meshes, and the R32F array launch_renderer composites against
    void ensure_mesh_target() {
        if (depth_array_ && target_w_ == w && target_h_ == h) return;
        if (depth_array_) cuda(FreeArray(depth_array_));
        if (rgba_lin_) cuda(Free(rgba_lin_));
        if (depth_lin_) cuda(Free(depth_lin_));
        cudaChannelFormatDesc cd = cudaCreateChannelDesc(32, 0, 0, 0, cudaChannelFormatKindFloat);
        cuda(MallocArray(&depth_array_, &cd, w, h, cudaArraySurfaceLoadStore));
        cuda(Malloc((void**)&rgba_lin_, std::max<size_t>((size_t)4 * w * h, 4)));
        cuda(Malloc((void**)&depth_lin_, std::max<size_t>((size_t)4 * w * h, 4)));
        target_w_ = w;
        target_h_ = h;
    }

    // The octree grid at grid_max_depth (cuda_renderer.cpp:99-111,182-188), generated on the device into a buffer
    // kept until the depth changes or the tree is set or cleared; drawn unlit as lines with the identity model.
    void append_grid(b200::MeshPass& pass) {
        vr_tree* t = device_tree(*tree);
        if (!t) return;
        const int depth = options.grid_max_depth;
        if (!wire_valid_ || wire_depth_ != depth) {
            wire_valid_ = false;
            int64_t n = 0;
            int rc = vr_tree_wireframe(t, depth, nullptr, 0, &n, (void*)stream);
            if (rc != VR_OK) die("vr_tree_wireframe", rc);
            if (n > INT32_MAX) {
                fprintf(stderr, "volrend_b200: grid at depth %d has %lld vertices; a mesh holds at most %d: "
                        "not drawn\n", depth, (long long)n, INT32_MAX);
                return;
            }
            if ((size_t)n * 9 > wire_cap_) {
                if (wire_dev_) cuda(Free(wire_dev_));
                wire_dev_ = nullptr;
                cuda(Malloc((void**)&wire_dev_, (size_t)n * 9 * sizeof(float)));
                wire_cap_ = (size_t)n * 9;
            }
            int64_t got = 0;
            if (n) {
                rc = vr_tree_wireframe(t, depth, wire_dev_, n, &got, (void*)stream);
                if (rc != VR_OK) die("vr_tree_wireframe", rc);
            }
            wire_n_ = n;
            wire_depth_ = depth;
            wire_valid_ = true;
        }
        if (wire_n_ == 0) return;
        vr_mesh_desc d;
        memset(&d, 0, sizeof(d));
        d.vert_dev = wire_dev_;
        d.n_verts = (int32_t)wire_n_;
        d.face_size = 2;
        d.unlit = 1;
        for (int i = 0; i < 4; ++i) d.model[5 * i] = 1.f;
        pass.meshes.push_back(d);
    }

    Camera& camera;
    RenderOptions& options;
    std::vector<Mesh>& meshes;
    N3Tree* tree = nullptr;

    Mesh probe_;
    cudaArray_t depth_array_ = nullptr;   // R32F ray distance for launch_renderer(offscreen=false)
    uint8_t* rgba_lin_ = nullptr;
    float* depth_lin_ = nullptr;
    int target_w_ = 0, target_h_ = 0;
    float* wire_dev_ = nullptr;           // the grid's vertices, wire_n_ of them, for grid_max_depth wire_depth_
    size_t wire_cap_ = 0;
    int64_t wire_n_ = 0;
    int wire_depth_ = 0;
    bool wire_valid_ = false;             // false: no grid generated
};

namespace {
std::unordered_map<const VolumeRenderer*, OffscreenTarget*>& impls() {
    static std::unordered_map<const VolumeRenderer*, OffscreenTarget*> m;
    return m;
}
}  // namespace

VolumeRenderer::VolumeRenderer() : impl_(std::make_unique<Impl>(camera, options, meshes)) {
    std::lock_guard<std::mutex> lk(g_mu);
    impls()[this] = impl_.get();
}
VolumeRenderer::~VolumeRenderer() {
    std::lock_guard<std::mutex> lk(g_mu);
    impls().erase(this);
}
void VolumeRenderer::render() { impl_->render(); }
void VolumeRenderer::set(N3Tree& tree) {
    impl_->set(tree);
    // cuda_renderer.cpp:176-177
    options.basis_minmax[0] = 0;
    options.basis_minmax[1] = std::max(tree.data_format.basis_dim - 1, 0);
}
void VolumeRenderer::clear() { impl_->clear(); }
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
