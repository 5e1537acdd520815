// vr_ssim.h -- internal interface between the C-ABI (vr_api.cu: vr_image_ssim) and the SSIM kernels (vr_ssim.cu).
// See DESIGN.md section 22.
#pragma once
#include <cuda_runtime.h>

namespace vrb {

// Per-view SSIM of x against y (RGB of [n_views][height][width][x_channels / y_channels] float32, channels 3 or 4,
// height and width >= 11) into ssim[n_views], overwritten; with dx (x's layout) not null, dx += dx_scale * dssim/dx on
// channels 0..2.  Scratch for the per-tile partial sums comes from the device's stream-ordered pool.  Stream-ordered
// and bit-reproducible: no atomics, every sum in a fixed order.
cudaError_t ssim_pass(const float* x, int x_channels, const float* y, int y_channels, int n_views, int height, int width,
                      double* ssim, float* dx, float dx_scale, cudaStream_t stream, int* launches);

}  // namespace vrb
