// shim_probe.cpp -- one frame with the lumisphere probe on, through the reference's own launch_renderer signature:
//   shim_probe <tree.npz> <pose.txt> <w> <h> <fx> <px> <py> <pz> <disp_size> <basis_min> <basis_max> <out.rgba>
// Writes the raw RGBA8 frame (main_headless.cpp-style cudaArray read-back).
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <vector>

#include "volrend/common.hpp"
#include "volrend/cuda/common.cuh"
#include "volrend/cuda/renderer_kernel.hpp"
#include "volrend/n3tree.hpp"

using namespace volrend;

int main(int argc, char** argv) {
    if (argc < 13) {
        fprintf(stderr, "usage: shim_probe tree.npz pose.txt w h fx px py pz disp_size basis_min basis_max out.rgba\n");
        return 2;
    }
    const int w = atoi(argv[3]), h = atoi(argv[4]);
    const float fx = (float)atof(argv[5]);
    glm::mat4x3 pose;
    {
        std::ifstream ifs(argv[2]);
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 4; ++c) ifs >> pose[c][r];
        if (!ifs) { fprintf(stderr, "bad pose file\n"); return 2; }
    }
    N3Tree tree(argv[1]);
    if (!tree.is_data_loaded() || !tree.is_cuda_loaded()) { fprintf(stderr, "tree not loaded\n"); return 3; }
    Camera camera(w, h, fx, fx);
    camera.transform = pose;
    camera._update(false);
    RenderOptions options;
    options.enable_probe = true;
    for (int i = 0; i < 3; ++i) options.probe[i] = (float)atof(argv[6 + i]);
    options.probe_disp_size = atoi(argv[9]);
    options.basis_minmax[0] = atoi(argv[10]);
    options.basis_minmax[1] = atoi(argv[11]);
    cudaArray_t array;
    cudaStream_t stream;
    cudaChannelFormatDesc cd = cudaCreateChannelDesc(8, 8, 8, 8, cudaChannelFormatKindUnsigned);
    cuda(MallocArray(&array, &cd, w, h, cudaArraySurfaceLoadStore));
    cuda(StreamCreateWithFlags(&stream, cudaStreamDefault));
    cudaArray_t depth_arr = nullptr;
    launch_renderer(tree, camera, options, array, depth_arr, stream, true);
    std::vector<uint8_t> buf((size_t)4 * w * h);
    cuda(Memcpy2DFromArrayAsync(buf.data(), 4 * w, array, 0, 0, 4 * w, h, cudaMemcpyDeviceToHost, stream));
    cuda(StreamSynchronize(stream));
    FILE* f = fopen(argv[12], "wb");
    if (!f || fwrite(buf.data(), 1, buf.size(), f) != buf.size()) { fprintf(stderr, "cannot write %s\n", argv[12]); return 4; }
    fclose(f);
    cuda(FreeArray(array));
    cuda(StreamDestroy(stream));
    return 0;
}
