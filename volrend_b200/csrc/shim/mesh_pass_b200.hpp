// Between mesh_b200.cpp (volrend::Mesh) and volrend_backend.cu (VolumeRenderer::Impl): the mesh pass that
// Mesh::draw adds to, in the role the bound GL framebuffer plays in the reference.
#pragma once
#include <vector>

#include "volrend_b200.h"

namespace volrend {
namespace b200 {

// The meshes drawn since the pass was opened, in draw order; the renderer flushes them with one vr_draw_meshes call,
// so an earlier mesh wins exact depth ties.
struct MeshPass {
    std::vector<vr_mesh_desc> meshes;
};

// The calling thread's open pass, or nullptr.  VolumeRenderer::render opens one around its draw calls.
MeshPass* current_mesh_pass();
void set_current_mesh_pass(MeshPass* pass);

}  // namespace b200
}  // namespace volrend
