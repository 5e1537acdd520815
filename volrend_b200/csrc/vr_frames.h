// vr_frames.h -- the batch and host-frame paths behind the C-ABI, with the options as a strided array: opt_stride 0
// renders every view with opt[0] (vr_render_batch, vr_render_frames_host, vr_render_frames_png), opt_stride 1 view
// i with opt[i] (the *_opts entry points).  Shared by vr_api.cu and vr_png.cpp, so that each pipeline exists once.
#pragma once
#include "volrend_b200.h"

namespace vrb {

// depth_dev != nullptr: composite mode (vr_render_composite_batch): rgba8_dev is read and overwritten, depth_dev
// holds each view's ray-distance limits, one tile-sized frame per view.
int render_batch(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt, int opt_stride,
                 const vr_rect* tile, uint8_t* rgba8_dev, float* rgba32f_dev, vr_counters* counters_dev, void* stream,
                 const float* depth_dev = nullptr);

int render_frames_host(const vr_tree* t, const vr_camera* cams, int n_views, const vr_options* opt, int opt_stride,
                       uint8_t* rgba8_host);

}  // namespace vrb
