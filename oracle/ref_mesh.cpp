// ref_mesh.cpp -- C-ABI around the UNMODIFIED reference's Mesh loaders and helpers (test infrastructure).
//
// Built only where the reference sources exist (oracle/Makefile.mesh), into oracle/_ref/libref_mesh.so, from the
// reference's own src/mesh.cpp, tiny_obj_loader.cpp and cnpy.cpp.  No reference source is copied.  mesh.cpp is GL
// code: its only GL uses are GLEW function pointers (shader setup in the Mesh constructor, buffer upload in
// Mesh::update) and glDrawArrays/glDrawElements (Mesh::draw, never called here).  They are defined below as no-op
// stubs, with glGetShaderiv/glGetProgramiv reporting success, so the harness needs neither GL nor a GPU.
//
//   ref_mesh_open_drawlist_mem -> Mesh::open_drawlist_mem (src/mesh.cpp:947-951)
//   ref_mesh_load_mem_obj      -> Mesh::load_mem_basic_obj (mesh.cpp:765-767)
//   ref_mesh_lattice           -> Mesh::Lattice (mesh.cpp:493-520)
//   ref_mesh_camera_frustum    -> Mesh::CameraFrustum (mesh.cpp:522-554)
//   ref_mesh_from / _repeat / _apply_transform / _apply_matrix -> Mesh::repeat, Mesh::apply_transform (633-678)
#include <GL/glew.h>

#include <chrono>
#include <cstring>
#include <string>
#include <vector>

#include "volrend/mesh.hpp"

namespace {
template <class F>
struct Stub;
template <class R, class... A>
struct Stub<R(GLAPIENTRY*)(A...)> {
    static R GLAPIENTRY f(A...) { return R(); }
};
void GLAPIENTRY get_iv_ok(GLuint, GLenum, GLint* params) {
    if (params) *params = GL_TRUE;
}
using Meshes = std::vector<volrend::Mesh>;
}  // namespace

#define VR_STUB(name, type) type name = &Stub<type>::f
VR_STUB(__glewAttachShader, PFNGLATTACHSHADERPROC);
VR_STUB(__glewBindAttribLocation, PFNGLBINDATTRIBLOCATIONPROC);
VR_STUB(__glewBindBuffer, PFNGLBINDBUFFERPROC);
VR_STUB(__glewBindVertexArray, PFNGLBINDVERTEXARRAYPROC);
VR_STUB(__glewBufferData, PFNGLBUFFERDATAPROC);
VR_STUB(__glewCompileShader, PFNGLCOMPILESHADERPROC);
VR_STUB(__glewCreateProgram, PFNGLCREATEPROGRAMPROC);
VR_STUB(__glewCreateShader, PFNGLCREATESHADERPROC);
VR_STUB(__glewDeleteShader, PFNGLDELETESHADERPROC);
VR_STUB(__glewEnableVertexAttribArray, PFNGLENABLEVERTEXATTRIBARRAYPROC);
VR_STUB(__glewGenBuffers, PFNGLGENBUFFERSPROC);
VR_STUB(__glewGenVertexArrays, PFNGLGENVERTEXARRAYSPROC);
VR_STUB(__glewGetProgramInfoLog, PFNGLGETPROGRAMINFOLOGPROC);
VR_STUB(__glewGetShaderInfoLog, PFNGLGETSHADERINFOLOGPROC);
VR_STUB(__glewGetUniformLocation, PFNGLGETUNIFORMLOCATIONPROC);
VR_STUB(__glewLinkProgram, PFNGLLINKPROGRAMPROC);
VR_STUB(__glewShaderSource, PFNGLSHADERSOURCEPROC);
VR_STUB(__glewUniform1i, PFNGLUNIFORM1IPROC);
VR_STUB(__glewUniform3fv, PFNGLUNIFORM3FVPROC);
VR_STUB(__glewUniformMatrix4fv, PFNGLUNIFORMMATRIX4FVPROC);
VR_STUB(__glewUseProgram, PFNGLUSEPROGRAMPROC);
VR_STUB(__glewVertexAttribPointer, PFNGLVERTEXATTRIBPOINTERPROC);
PFNGLGETSHADERIVPROC __glewGetShaderiv = &get_iv_ok;
PFNGLGETPROGRAMIVPROC __glewGetProgramiv = &get_iv_ok;
#undef VR_STUB
extern "C" {
void GLAPIENTRY glDrawArrays(GLenum, GLint, GLsizei) {}
void GLAPIENTRY glDrawElements(GLenum, GLsizei, GLenum, const void*) {}

// Each call returns a handle to a list of meshes (free with ref_mesh_free).  *ms (if not NULL) receives the host
// time of the reference call.
void* ref_mesh_open_drawlist_mem(const char* data, unsigned long long size, int default_visible, double* ms) {
    const auto t0 = std::chrono::steady_clock::now();
    Meshes* m = new Meshes(volrend::Mesh::open_drawlist_mem(data, size, default_visible != 0));
    const auto t1 = std::chrono::steady_clock::now();
    if (ms) *ms = std::chrono::duration<double, std::milli>(t1 - t0).count();
    fflush(stdout);
    return m;
}

void* ref_mesh_load_mem_obj(const char* text, unsigned long long size) {
    Meshes* m = new Meshes();
    m->push_back(volrend::Mesh::load_mem_basic_obj(std::string(text, size)));
    fflush(stdout);
    return m;
}

void* ref_mesh_lattice(int reso, const float* color) {
    return new Meshes{volrend::Mesh::Lattice(reso, glm::vec3(color[0], color[1], color[2]))};
}

void* ref_mesh_camera_frustum(float focal_length, float image_width, float image_height, float z, const float* color) {
    return new Meshes{volrend::Mesh::CameraFrustum(focal_length, image_width, image_height, z,
                                                   glm::vec3(color[0], color[1], color[2]))};
}

// A mesh with the given vertices (n_floats floats) and faces, for repeat / apply_transform.
void* ref_mesh_from(const float* vert, long long n_floats, const unsigned* faces, long long n_faces_idx, int face_size) {
    volrend::Mesh m(0, 0, face_size);
    m.vert.assign(vert, vert + n_floats);
    m.faces.assign(faces, faces + n_faces_idx);
    return new Meshes{std::move(m)};
}

void ref_mesh_repeat(void* h, int n) { (*static_cast<Meshes*>(h))[0].repeat(n); }

void ref_mesh_apply_transform(void* h, const float* r, const float* t, int start, int end) {
    (*static_cast<Meshes*>(h))[0].apply_transform(glm::vec3(r[0], r[1], r[2]), glm::vec3(t[0], t[1], t[2]), start, end);
}

// m: column-major 4x4 (glm's layout)
void ref_mesh_apply_matrix(void* h, const float* m, int start, int end) {
    glm::mat4 M;
    for (int c = 0; c < 4; ++c)
        for (int r = 0; r < 4; ++r) M[c][r] = m[4 * c + r];
    (*static_cast<Meshes*>(h))[0].apply_transform(M, start, end);
}

int ref_mesh_count(void* h) { return (int)static_cast<Meshes*>(h)->size(); }

// Sizes of mesh i: sizes[0] = vert floats, sizes[1] = face indices, sizes[2] = name bytes.
void ref_mesh_sizes(void* h, int i, long long* sizes) {
    const volrend::Mesh& m = (*static_cast<Meshes*>(h))[i];
    sizes[0] = (long long)m.vert.size();
    sizes[1] = (long long)m.faces.size();
    sizes[2] = (long long)m.name.size();
}

// Every field of mesh i: vert, faces, name (not terminated), f7 = scale, translation, rotation,
// i4 = face_size, visible, unlit, 0.
void ref_mesh_get(void* h, int i, float* vert, unsigned* faces, char* name, float* f7, int* i4) {
    const volrend::Mesh& m = (*static_cast<Meshes*>(h))[i];
    if (!m.vert.empty()) memcpy(vert, m.vert.data(), m.vert.size() * sizeof(float));
    if (!m.faces.empty()) memcpy(faces, m.faces.data(), m.faces.size() * sizeof(unsigned));
    if (!m.name.empty()) memcpy(name, m.name.data(), m.name.size());
    f7[0] = m.scale;
    for (int k = 0; k < 3; ++k) {
        f7[1 + k] = m.translation[k];
        f7[4 + k] = m.rotation[k];
    }
    i4[0] = m.face_size;
    i4[1] = m.visible;
    i4[2] = m.unlit;
    i4[3] = 0;
}

void ref_mesh_free(void* h) { delete static_cast<Meshes*>(h); }

}  // extern "C"
