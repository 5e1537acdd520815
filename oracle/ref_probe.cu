// ref_probe.cu -- C-ABI around the UNMODIFIED reference renderer with the lumisphere probe on (test infrastructure).
//
// Built only where the reference sources exist (oracle/Makefile.probe), into oracle/_ref/libref_probe.so.  Like
// ref_harness.cu it #includes the reference's own src/cuda/volrend.cu, so `volrend::launch_renderer` below is the
// reference's stock code path: render_kernel draws the disc (volrend.cu:100-134) from the coefficients that
// retrieve_cursor_lumisphere_kernel fetched (:175-191, :202-209).  No reference source is copied.
//
//   ref_probe_tree_open / _close -> N3Tree(path) of this library
//   ref_probe_render_u8          -> launch_renderer with enable_probe / probe / probe_disp_size set, offscreen or
//                                   over colour + depth inputs, bytes read back as main_headless.cpp:216-219 does
#include <cstdint>
#include <cstring>
#include <string>

#include "../src/cuda/volrend.cu"  // resolved through -I$(VOLREND_REF)/include/.. (see Makefile.probe)

#include "volrend/camera.hpp"
#include "volrend/n3tree.hpp"

using namespace volrend;

extern "C" {

// RenderOptions fields of the march (same layout as ref_harness.cu's ref_options) plus the probe.
struct ref_probe_options {
    float step_size, sigma_thresh, stop_thresh, background_brightness;
    float render_bbox[6];
    int32_t basis_minmax[2];
    float rot_dirs[3];
    int32_t render_depth;
    float probe[3];
    int32_t probe_disp_size;
};

void* ref_probe_tree_open(const char* npz_path) {
    N3Tree* t = new N3Tree(std::string(npz_path));
    if (!t->is_data_loaded()) { delete t; return nullptr; }
    return t;
}
void ref_probe_tree_close(void* t) { delete static_cast<N3Tree*>(t); }

int ref_probe_render_u8(void* tp, int w, int h, float fx, float fy, const float* c2w12, const ref_probe_options* o,
                        const uint8_t* rgba_in, const float* depth_in, uint8_t* out_host) {
    N3Tree& tree = *static_cast<N3Tree*>(tp);
    Camera cam(w, h, fx, fy);
    for (int c = 0; c < 4; ++c)
        for (int r = 0; r < 3; ++r) cam.transform[c][r] = c2w12[c * 3 + r];
    cam._update(false);
    RenderOptions opt;
    opt.step_size = o->step_size; opt.sigma_thresh = o->sigma_thresh; opt.stop_thresh = o->stop_thresh;
    opt.background_brightness = o->background_brightness;
    for (int i = 0; i < 6; ++i) opt.render_bbox[i] = o->render_bbox[i];
    opt.basis_minmax[0] = o->basis_minmax[0]; opt.basis_minmax[1] = o->basis_minmax[1];
    for (int i = 0; i < 3; ++i) opt.rot_dirs[i] = o->rot_dirs[i];
    opt.render_depth = o->render_depth != 0;
    opt.enable_probe = true;
    for (int i = 0; i < 3; ++i) opt.probe[i] = o->probe[i];
    opt.probe_disp_size = o->probe_disp_size;
    cudaArray_t arr = nullptr, darr = nullptr;
    cudaChannelFormatDesc cd = cudaCreateChannelDesc(8, 8, 8, 8, cudaChannelFormatKindUnsigned);
    cuda(MallocArray(&arr, &cd, w, h, cudaArraySurfaceLoadStore));
    const bool offscreen = rgba_in == nullptr;
    if (!offscreen) {
        cudaChannelFormatDesc dd = cudaCreateChannelDesc(32, 0, 0, 0, cudaChannelFormatKindFloat);
        cuda(MallocArray(&darr, &dd, w, h, cudaArraySurfaceLoadStore));
        cuda(Memcpy2DToArray(arr, 0, 0, rgba_in, 4 * w, 4 * w, h, cudaMemcpyHostToDevice));
        cuda(Memcpy2DToArray(darr, 0, 0, depth_in, 4 * w, 4 * w, h, cudaMemcpyHostToDevice));
    }
    cudaStream_t stream;
    cuda(StreamCreateWithFlags(&stream, cudaStreamDefault));
    launch_renderer(tree, cam, opt, arr, darr, stream, offscreen);
    cuda(Memcpy2DFromArrayAsync(out_host, 4 * w, arr, 0, 0, 4 * w, h, cudaMemcpyDeviceToHost, stream));
    cuda(StreamSynchronize(stream));
    cudaError_t e = cudaGetLastError();
    cuda(StreamDestroy(stream));
    cuda(FreeArray(arr));
    if (darr) cuda(FreeArray(darr));
    return e == cudaSuccess ? 0 : -(int)e;
}

}  // extern "C"
