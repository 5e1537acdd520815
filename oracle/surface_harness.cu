// surface_harness.cu -- test infrastructure: one RGBA8 cudaArray (and optionally one R32F cudaArray) with their
// surface objects, so that tests can run vr_render_surface and the surface form of vr_draw_probe the way the C++
// drop-in launch_renderer does: into a cudaArray the caller owns.
//
// The harness does not link libvolrend_b200.so.  The caller passes the entry points it has already loaded as function
// pointers, so that the variant setting, vr_last_error and the launch counter the test reads are the ones these calls
// change.  Every CUDA error comes back as a nonzero return code (the cudaError_t); an entry point's own return code is
// passed through unchanged.
#include <cstdint>
#include <cstdlib>

#include <cuda_runtime.h>

// vr_render_surface and vr_draw_probe of include/volrend_b200.h, with the argument types the harness does not read
// left opaque
typedef int (*render_surface_fn)(const void* tree, const void* cam, const void* opt, unsigned long long rgba8_surf,
                                 unsigned long long depth_surf, void* stream);
typedef int (*draw_probe_fn)(const void* tree, const void* cams, int n_views, const void* opt, const float probe_xyz[3],
                             int disp_size, const void* tile, uint8_t* rgba8_dev, float* rgba32f_dev,
                             unsigned long long rgba8_surf, void* stream);

struct sh_frame {
    int w, h;
    cudaArray_t colour, depth;          // depth: nullptr when the frame has no depth array
    cudaSurfaceObject_t scolour, sdepth;
};

namespace {

cudaError_t make_array(int w, int h, cudaChannelFormatDesc fmt, cudaArray_t* arr, cudaSurfaceObject_t* surf) {
    cudaError_t e = cudaMallocArray(arr, &fmt, (size_t)w, (size_t)h, cudaArraySurfaceLoadStore);
    if (e != cudaSuccess) { *arr = nullptr; return e; }
    cudaResourceDesc rd{};
    rd.resType = cudaResourceTypeArray;
    rd.res.array.array = *arr;
    return cudaCreateSurfaceObject(surf, &rd);
}

}  // namespace

extern "C" {

// Frees every object of the frame that was created; returns the first error.
int sh_free(sh_frame* f) {
    if (!f) return 0;
    cudaError_t first = cudaSuccess;
    auto keep = [&](cudaError_t e) { if (first == cudaSuccess) first = e; };
    if (f->scolour) keep(cudaDestroySurfaceObject(f->scolour));
    if (f->sdepth) keep(cudaDestroySurfaceObject(f->sdepth));
    if (f->colour) keep(cudaFreeArray(f->colour));
    if (f->depth) keep(cudaFreeArray(f->depth));
    free(f);
    return (int)first;
}

// An RGBA8 array of w x h pixels and, with with_depth, an R32F array of the same size.
int sh_alloc(int w, int h, int with_depth, sh_frame** out) {
    if (!out) return (int)cudaErrorInvalidValue;
    *out = nullptr;
    if (w <= 0 || h <= 0) return (int)cudaErrorInvalidValue;
    sh_frame* f = (sh_frame*)calloc(1, sizeof(sh_frame));
    if (!f) return (int)cudaErrorMemoryAllocation;
    f->w = w; f->h = h;
    cudaError_t e = make_array(w, h, cudaCreateChannelDesc<uchar4>(), &f->colour, &f->scolour);
    if (e == cudaSuccess && with_depth) e = make_array(w, h, cudaCreateChannelDesc<float>(), &f->depth, &f->sdepth);
    if (e != cudaSuccess) {
        sh_free(f);
        return (int)e;
    }
    *out = f;
    return 0;
}

// Host RGBA8 rows of w pixels (and, when the frame has a depth array and depth is given, host float rows) into the
// arrays.  Returns when the copies have landed: a copy from pageable memory may return before its DMA ends, and a
// render on a non-blocking stream would not wait for it.
int sh_upload(sh_frame* f, const uint8_t* rgba8, const float* depth) {
    if (!f || (depth && !f->depth)) return (int)cudaErrorInvalidValue;
    cudaError_t e = cudaSuccess;
    if (rgba8) e = cudaMemcpy2DToArray(f->colour, 0, 0, rgba8, (size_t)f->w * 4, (size_t)f->w * 4, f->h,
                                       cudaMemcpyHostToDevice);
    if (e == cudaSuccess && depth)
        e = cudaMemcpy2DToArray(f->depth, 0, 0, depth, (size_t)f->w * 4, (size_t)f->w * 4, f->h, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return (int)e;
}

// The RGBA8 array into host rows of w pixels, after everything queued on the device has finished.
int sh_download(sh_frame* f, uint8_t* rgba8) {
    if (!f || !rgba8) return (int)cudaErrorInvalidValue;
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess)
        e = cudaMemcpy2DFromArray(rgba8, (size_t)f->w * 4, f->colour, 0, 0, (size_t)f->w * 4, f->h,
                                  cudaMemcpyDeviceToHost);
    return (int)e;
}

// fn(tree, cam, opt, colour surface, depth surface or 0, stream).  use_depth: pass the depth surface (composite).
int sh_render(sh_frame* f, render_surface_fn fn, const void* tree, const void* cam, const void* opt, int use_depth,
              void* stream) {
    if (!f || !fn) return (int)cudaErrorInvalidValue;
    if (use_depth && !f->depth) return (int)cudaErrorInvalidValue;
    return fn(tree, cam, opt, f->scolour, use_depth ? f->sdepth : 0, stream);
}

// The probe disc of one view into the colour surface: fn(tree, cam, 1, opt, xyz, disp, no tile, no linear or float
// output, colour surface, stream).
int sh_probe(sh_frame* f, draw_probe_fn fn, const void* tree, const void* cam, const void* opt, const float xyz[3],
             int disp_size, void* stream) {
    if (!f || !fn) return (int)cudaErrorInvalidValue;
    return fn(tree, cam, 1, opt, xyz, disp_size, nullptr, nullptr, nullptr, f->scolour, stream);
}

// The colour surface object (for calls the helpers above do not make).
unsigned long long sh_colour_surface(const sh_frame* f) { return f ? f->scolour : 0; }

}  // extern "C"
