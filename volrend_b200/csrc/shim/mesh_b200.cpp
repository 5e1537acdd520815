// mesh_b200.cpp -- GL-free definitions of include/volrend/mesh.hpp (volrend::Mesh) over the volrend_b200 C-ABI.
//
// Build this INSTEAD of the reference's src/mesh.cpp (which is GL code).  Every member the header declares is here:
//   * presets, auto_faces, repeat, apply_transform: host code, byte for byte what volrend_b200/mesh.py computes
//     (float32 in the reference's operation order; compile without FMA contraction);
//   * load_basic_obj / load_mem_basic_obj: tinyobj with the reference's configuration; normals estimated on the
//     device (vr_mesh_estimate_normals) when the file has fewer `vn` than `v`;
//   * open_drawlist / open_drawlist_mem: cnpy, with the drawlist rules of volrend_b200/mesh_io.py (DESIGN §11);
//   * update(): uploads vert and faces to device memory named by a handle in vao_/vbo_/ebo_ (DESIGN §16);
//   * draw(): adds the mesh to the mesh pass VolumeRenderer::render has open (mesh_pass_b200.hpp);
//   * use_shader(): a no-op, there is no GL program.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <map>
#include <mutex>
#include <sstream>
#include <stdexcept>
#include <string>
#include <vector>

#include "cnpy.h"
#include "tiny_obj_loader.h"
#include "volrend/common.hpp"
#include "volrend/cuda/common.cuh"
#include "volrend/mesh.hpp"

#include "mesh_pass_b200.hpp"
#include "volrend_b200.h"

namespace volrend {

namespace b200 {
namespace {
thread_local MeshPass* g_pass = nullptr;
}  // namespace
MeshPass* current_mesh_pass() { return g_pass; }
void set_current_mesh_pass(MeshPass* pass) { g_pass = pass; }
}  // namespace b200

namespace {

constexpr int VERT_SZ = 9;   // position, colour, normal

// ---------------------------------------------------------------- device uploads
// One upload per handle.  Like the GL buffer names of the reference, a handle lives as long as the process: Mesh
// has no destructor to release it, and copies of a Mesh share it.
struct Upload {
    float* vert_dev = nullptr;
    uint32_t* faces_dev = nullptr;
    size_t vert_cap = 0, faces_cap = 0;   // floats / indices allocated
    size_t n_vert_floats = 0, n_face_idx = 0;
};
std::mutex g_up_mu;
std::deque<Upload> g_uploads;             // handle h names g_uploads[h - 1]; a deque keeps references stable

[[noreturn]] void die(const char* what, int rc) {
    // the shim's cuda(...) contract: print, reset, exit
    fprintf(stderr, "volrend_b200: %s failed (%d): %s\n", what, rc, vr_last_error());
    cudaDeviceReset();
    exit(rc < 0 ? -rc : 1);
}

template <class T>
void upload_into(T*& dev, size_t& cap, const T* host, size_t n) {
    if (n > cap) {
        if (dev) cuda(Free(dev));
        dev = nullptr;
        cuda(Malloc((void**)&dev, n * sizeof(T)));
        cap = n;
    }
    if (n) cuda(Memcpy(dev, host, n * sizeof(T), cudaMemcpyHostToDevice));
}

// estimate_normals of the reference, on the device (DESIGN §11): a temporary upload, vr_mesh_estimate_normals, and
// the vertices copied back.
void estimate_normals(std::vector<float>& vert, const std::vector<unsigned int>& faces) {
    const size_t n_verts = vert.size() / VERT_SZ;
    float* vd = nullptr;
    uint32_t* fd = nullptr;
    if (!vert.empty()) {
        cuda(Malloc((void**)&vd, vert.size() * sizeof(float)));
        cuda(Memcpy(vd, vert.data(), vert.size() * sizeof(float), cudaMemcpyHostToDevice));
    }
    if (!faces.empty()) {
        cuda(Malloc((void**)&fd, faces.size() * sizeof(uint32_t)));
        cuda(Memcpy(fd, faces.data(), faces.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    }
    const int rc = vr_mesh_estimate_normals(vd, (int64_t)n_verts, fd, (int64_t)(faces.size() / 3), nullptr);
    if (rc != VR_OK) die("vr_mesh_estimate_normals", rc);
    if (vd) cuda(Memcpy(vert.data(), vd, vert.size() * sizeof(float), cudaMemcpyDeviceToHost));
    if (vd) cuda(Free(vd));
    if (fd) cuda(Free(fd));
}

// ---------------------------------------------------------------- model transforms
// Mesh::draw's model matrix as volrend_b200/mesh.py's model_matrix computes it: double precision, the rotation's
// norm summed (x*x + y*y) + z*z as numpy's r @ r does, rounded once to float.  Column-major, glm's layout.
glm::mat4 model_matrix(const glm::vec3& rotation, const glm::vec3& translation, float scale) {
    const double r0 = rotation[0], r1 = rotation[1], r2 = rotation[2];
    const double norm = std::sqrt((r0 * r0 + r1 * r1) + r2 * r2);
    double m[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};   // m[row][col]
    if (norm >= 1e-3) {
        const double x = r0 / norm, y = r1 / norm, z = r2 / norm;
        const double s = std::sin(norm / 2), c = std::cos(norm / 2);
        const double qw = c, qx = x * s, qy = y * s, qz = z * s;
        m[0][0] = 1 - 2 * (qy * qy + qz * qz);
        m[0][1] = 2 * (qx * qy - qw * qz);
        m[0][2] = 2 * (qx * qz + qw * qy);
        m[1][0] = 2 * (qx * qy + qw * qz);
        m[1][1] = 1 - 2 * (qx * qx + qz * qz);
        m[1][2] = 2 * (qy * qz - qw * qx);
        m[2][0] = 2 * (qx * qz - qw * qy);
        m[2][1] = 2 * (qy * qz + qw * qx);
        m[2][2] = 1 - 2 * (qx * qx + qy * qy);
    }
    glm::mat4 out(1.f);
    for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r) out[c][r] = (float)(m[r][c] * (double)scale);
    for (int r = 0; r < 3; ++r) out[3][r] = translation[r];
    return out;
}

// The matrix apply_transform(r, t) builds: float32, glm's length and 1e-3 test, angleAxis with sinf/cosf, mat4_cast,
// translation in column 3 (mesh.py's _glm_transform).
glm::mat4 axis_angle_matrix(const glm::vec3& r, const glm::vec3& t) {
    glm::mat4 m(1.f);
    const float norm = std::sqrt((r[0] * r[0] + r[1] * r[1]) + r[2] * r[2]);
    if ((double)norm >= 1e-3) {
        const float ax = r[0] / norm, ay = r[1] / norm, az = r[2] / norm;
        const float half = norm * 0.5f;
        const float s = sinf(half), w = cosf(half);
        const float x = ax * s, y = ay * s, z = az * s;
        const float xx = x * x, yy = y * y, zz = z * z, xz = x * z, xy = x * y, yz = y * z;
        const float wx = w * x, wy = w * y, wz = w * z;
        m[0][0] = 1.f - 2.f * (yy + zz); m[0][1] = 2.f * (xy + wz);       m[0][2] = 2.f * (xz - wy);
        m[1][0] = 2.f * (xy - wz);       m[1][1] = 1.f - 2.f * (xx + zz); m[1][2] = 2.f * (yz + wx);
        m[2][0] = 2.f * (xz + wy);       m[2][1] = 2.f * (yz - wx);       m[2][2] = 1.f - 2.f * (xx + yy);
    }
    m[3][0] = t[0]; m[3][1] = t[1]; m[3][2] = t[2];
    return m;
}

void push_vertex(std::vector<float>& v, float x, float y, float z, const glm::vec3& color, float nx, float ny,
                 float nz) {
    const float f[VERT_SZ] = {x, y, z, color[0], color[1], color[2], nx, ny, nz};
    v.insert(v.end(), f, f + VERT_SZ);
}

// Mesh::Points / Mesh::Lines vertices: n points, the given colour, normal (0, 0, 1).
size_t point_vertices(Mesh& m, const std::vector<float>& points, const glm::vec3& color, const char* who) {
    if (points.size() % 3) printf("%s: Number of elements in points must be divisible by 3\n", who);
    const size_t n = points.size() / 3;
    m.vert.clear();
    m.vert.reserve(n * VERT_SZ);
    for (size_t i = 0; i < n; ++i)
        push_vertex(m.vert, points[3 * i], points[3 * i + 1], points[3 * i + 2], color, 0.f, 0.f, 1.f);
    return n;
}

// ---------------------------------------------------------------- drawlist fields (mesh_io.py's _get_*)
float half_to_float(uint16_t h) {
    const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
    uint32_t exp = (h >> 10) & 0x1fu, man = h & 0x3ffu, bits;
    if (exp == 0x1fu) {
        bits = sign | 0x7f800000u | (man << 13);
    } else if (exp == 0) {
        if (man == 0) {
            bits = sign;
        } else {                                  // subnormal: normalise
            int e = -1;
            do { man <<= 1; ++e; } while (!(man & 0x400u));
            bits = sign | ((uint32_t)(127 - 15 - e) << 23) | ((man & 0x3ffu) << 13);
        }
    } else {
        bits = sign | ((exp + 127 - 15) << 23) | (man << 13);
    }
    float f;
    memcpy(&f, &bits, 4);
    return f;
}

using Fields = std::map<std::string, cnpy::NpyArray>;

size_t n_elems(const cnpy::NpyArray& a) { return a.word_size ? a.data_holder.size() / a.word_size : 0; }

bool is_int_size(size_t ws) { return ws == 1 || ws == 2 || ws == 4 || ws == 8; }
bool is_float_size(size_t ws) { return ws == 2 || ws == 4 || ws == 8; }

// Element i read as a signed integer of the array's element size, then kept to 32 bits.
int32_t int_at(const cnpy::NpyArray& a, size_t i) {
    const char* p = a.data_holder.data() + i * a.word_size;
    switch (a.word_size) {
        case 1: { int8_t v; memcpy(&v, p, 1); return v; }
        case 2: { int16_t v; memcpy(&v, p, 2); return v; }
        case 4: { int32_t v; memcpy(&v, p, 4); return v; }
        default: { int64_t v; memcpy(&v, p, 8); return (int32_t)(uint32_t)(uint64_t)v; }
    }
}

// Element i read as a float of the array's element size, rounded to float32.
float float_at(const cnpy::NpyArray& a, size_t i) {
    const char* p = a.data_holder.data() + i * a.word_size;
    switch (a.word_size) {
        case 2: { uint16_t v; memcpy(&v, p, 2); return half_to_float(v); }
        case 4: { float v; memcpy(&v, p, 4); return v; }
        default: { double v; memcpy(&v, p, 8); return (float)v; }
    }
}

int get_int(const Fields& f, const std::string& key, int defval, std::stringstream& errs) {
    auto it = f.find(key);
    if (it == f.end()) return defval;
    if (!is_int_size(it->second.word_size)) {
        errs << "Invalid word size for int " << it->second.word_size << "\n";
        return 0;
    }
    if (n_elems(it->second) < 1) {
        errs << "Field '" << key << "' is empty\n";
        return defval;
    }
    return int_at(it->second, 0);
}

float get_float(const Fields& f, const std::string& key, float defval, std::stringstream& errs) {
    auto it = f.find(key);
    if (it == f.end()) return defval;
    if (!is_float_size(it->second.word_size)) {
        errs << "Invalid word size for float " << it->second.word_size << "\n";
        return 0.f;
    }
    if (n_elems(it->second) < 1) {
        errs << "Field '" << key << "' is empty\n";
        return defval;
    }
    return float_at(it->second, 0);
}

glm::vec3 get_vec3(const Fields& f, const std::string& key, const glm::vec3& defval, std::stringstream& errs) {
    auto it = f.find(key);
    if (it == f.end()) return defval;
    const cnpy::NpyArray& a = it->second;
    if (a.shape.size() != 1 || a.shape[0] != 3) errs << "Invalid shape for float3, must be (3,)";
    if (!is_float_size(a.word_size)) {
        errs << "Invalid word size for float " << a.word_size << "\n";
        return defval;
    }
    if (n_elems(a) < 3) return defval;   // the reference reads past the array here
    return glm::vec3(float_at(a, 0), float_at(a, 1), float_at(a, 2));
}

std::vector<float> get_floatarr(const Fields& f, const std::string& key, std::stringstream& errs) {
    auto it = f.find(key);
    if (it == f.end()) return {};
    const cnpy::NpyArray& a = it->second;
    const size_t n = n_elems(a);
    std::vector<float> out(n, 0.f);
    if (!is_float_size(a.word_size)) {
        errs << "Invalid word size for float " << a.word_size << "\n";
        return out;
    }
    for (size_t i = 0; i < n; ++i) out[i] = float_at(a, i);
    return out;
}

std::vector<unsigned int> get_intarr(const Fields& f, const std::string& key, std::stringstream& errs) {
    auto it = f.find(key);
    if (it == f.end()) return {};
    const cnpy::NpyArray& a = it->second;
    const size_t n = n_elems(a);
    std::vector<unsigned int> out(n, 0u);
    if (!is_int_size(a.word_size)) {
        errs << "Invalid word size for int " << a.word_size << "\n";
        return out;
    }
    for (size_t i = 0; i < n; ++i) out[i] = (unsigned int)int_at(a, i);
    return out;
}

// Split on "__", dropping empty pieces before each separator; in a run of three or more underscores the piece becomes
// the rest of the string (mesh_io.py's _split_by_2underscore).
std::vector<std::string> split_by_2underscore(const std::string& s) {
    std::vector<std::string> r;
    size_t j = 0;
    for (size_t i = 1; i < s.size(); ++i) {
        if (s[i] == '_' && s[i - 1] == '_') {
            if (i - 1 != j) r.push_back(i - 1 > j ? s.substr(j, i - 1 - j) : s.substr(j));
            j = i + 1;
        }
    }
    if (j < s.size()) r.push_back(s.substr(j));
    return r;
}

// The low byte of each 4-byte unit, all but the first lowercased (ASCII).
std::string type_string(const cnpy::NpyArray& a) {
    std::string b(a.data_holder.begin(), a.data_holder.end());
    for (size_t i = 4; i < b.size(); i += 4) {
        const char c = b[i];
        b[i / 4] = (c >= 'A' && c <= 'Z') ? (char)(c - 'A' + 'a') : c;
    }
    b.resize(b.size() / 4);
    return b;
}

// One frustum per (r, t) triple of a camerafrustum entry, optionally connected centre to centre.  A camera `r`
// shorter than `t` reads 0 for the missing values.
void camera_frustums(Mesh& me, const Fields& fields, std::stringstream& errs) {
    const std::vector<float> t = get_floatarr(fields, "t", errs);
    std::vector<float> r = get_floatarr(fields, "r", errs);
    if (r.size() != t.size() || r.size() % 3) errs << "camerafrustums r, t have different sizes or not multiple of 3\n";
    const size_t nv = me.vert.size() / VERT_SZ;
    const size_t n_reps = t.size() / 3;
    if (r.size() < 3 * n_reps) r.resize(3 * n_reps, 0.f);
    me.repeat((int)n_reps);
    for (size_t i = 0; i < n_reps; ++i)
        me.apply_transform(glm::vec3(r[3 * i], r[3 * i + 1], r[3 * i + 2]),
                           glm::vec3(t[3 * i], t[3 * i + 1], t[3 * i + 2]), (int)(nv * i), (int)(nv * (i + 1)));
    if (get_int(fields, "connect", 0, errs) != 0) {
        if (n_reps == 0) throw std::invalid_argument("camerafrustum: 'connect' needs at least one camera in 't'");
        for (size_t i = 0; i + 1 < n_reps; ++i) {
            me.faces.push_back((unsigned int)(nv * i));
            me.faces.push_back((unsigned int)(nv * (i + 1)));
        }
    }
}

// The preset or generic mesh of one drawlist entry; false for an unsupported type.
bool build_entry(const std::string& type, const Fields& fields, Mesh& me, std::stringstream& errs) {
    const glm::vec3 color = get_vec3(fields, "color", glm::vec3(1.0f, 0.5f, 0.2f), errs);
    if (type == "cube") {
        me = Mesh::Cube(color);
    } else if (type == "sphere") {
        const int rings = get_int(fields, "rings", 15, errs);
        const int sectors = get_int(fields, "sectors", 30, errs);
        me = Mesh::Sphere(rings, sectors, color);
    } else if (type == "line") {
        const glm::vec3 a = get_vec3(fields, "a", glm::vec3(0.f, 0.f, 0.f), errs);
        const glm::vec3 b = get_vec3(fields, "b", glm::vec3(0.f, 0.f, 1.f), errs);
        me = Mesh::Line(a, b, color);
    } else if (type == "camerafrustum") {
        const float focal = get_float(fields, "focal_length", 1111.0f, errs);
        const float w = get_float(fields, "image_width", 800.0f, errs);
        const float h = get_float(fields, "image_height", 800.0f, errs);
        const float z = get_float(fields, "z", -0.3f, errs);
        me = Mesh::CameraFrustum(focal, w, h, z, color);
        if (fields.count("t")) camera_frustums(me, fields, errs);
    } else if (type == "lines") {
        me = Mesh::Lines(get_floatarr(fields, "points", errs), color);
        if (fields.count("segs")) me.faces = get_intarr(fields, "segs", errs);
    } else if (type == "points") {
        me = Mesh::Points(get_floatarr(fields, "points", errs), color);
    } else if (type == "mesh") {
        me = Mesh::Points(get_floatarr(fields, "points", errs), color);
        me.face_size = get_int(fields, "face_size", 3, errs);
        if (me.face_size <= 0 || me.face_size > 3) {
            me.face_size = 3;
            errs << "Mesh face size must be one of 1,2,3\n";
        }
        if (fields.count("faces")) {
            std::vector<unsigned int> faces = get_intarr(fields, "faces", errs);
            if (faces.size() % me.face_size) errs << "Faces must have face_size=" << me.face_size << " elements\n";
            me.faces = std::move(faces);
        }
        if (me.face_size == 3) estimate_normals(me.vert, me.faces);
    } else {
        return false;
    }
    return true;
}

std::vector<Mesh> load_npz(const cnpy::npz_t& npz, bool default_visible) {
    printf("INFO: Loading drawlist npz\n");
    std::map<std::string, std::pair<std::string, Fields>> parse;   // std::map: name (byte) order
    for (const auto& kv : npz) {
        const std::vector<std::string> spl = split_by_2underscore(kv.first);
        if (spl.size() == 1) {
            parse[spl[0]].first = type_string(kv.second);
        } else if (spl.size() == 2) {
            parse[spl[0]].second[spl[1]] = kv.second;
        } else {
            printf("Mesh load_npz warning: invalid field '%s', must be of the form <name>=mesh_type or "
                   "<name>__<field>=val\n", kv.first.c_str());
        }
    }
    std::vector<Mesh> meshes;
    std::stringstream errs;
    for (const auto& kv : parse) {
        const std::string& name = kv.first;
        const Fields& fields = kv.second.second;
        Mesh me;
        if (!build_entry(kv.second.first, fields, me, errs)) {
            errs << "Mesh '" << name << "' has unsupported type '" << kv.second.first << "'\n";
            continue;
        }
        if (fields.count("vert_color")) {
            const std::vector<float> vc = get_floatarr(fields, "vert_color", errs);
            if (vc.size() * VERT_SZ != me.vert.size() * 3) {
                errs << "Mesh " << name << " vert_color has invalid size\n";
                continue;
            }
            for (size_t i = 0; i < vc.size() / 3; ++i)
                for (int j = 0; j < 3; ++j) me.vert[i * VERT_SZ + 3 + j] = vc[3 * i + j];
        }
        me.name = name;
        me.scale = get_float(fields, "scale", 1.0f, errs);
        me.translation = get_vec3(fields, "translation", glm::vec3(0.f), errs);
        me.rotation = get_vec3(fields, "rotation", glm::vec3(0.f), errs);
        me.visible = get_int(fields, "visible", default_visible ? 1 : 0, errs) != 0;
        me.unlit = get_int(fields, "unlit", 0, errs) != 0;
        me.update();
        meshes.push_back(std::move(me));
    }
    const std::string e = errs.str();
    if (!e.empty()) printf("Mesh load_npz encountered errors while parsing:\n%s", e.c_str());
    return meshes;
}

// ---------------------------------------------------------------- OBJ
Mesh load_obj(const std::string& path_or_text, bool from_string) {
    Mesh mesh;
    tinyobj::ObjReaderConfig config;
    if (!from_string) config.mtl_search_path = "./";
    config.triangulate = true;
    config.vertex_color = true;
    tinyobj::ObjReader reader;
    const bool ok = from_string ? reader.ParseFromString(path_or_text, "", config)
                                : reader.ParseFromFile(path_or_text, config);
    if (!ok) {
        if (!reader.Error().empty()) printf("ERROR Failed to load OBJ: %s", reader.Error().c_str());
        return mesh;
    }
    const tinyobj::attrib_t& attrib = reader.GetAttrib();
    const size_t nv = attrib.vertices.size() / 3;
    mesh.vert.assign(nv * VERT_SZ, 0.f);
    for (size_t i = 0; i < nv; ++i)
        for (int j = 0; j < 3; ++j) mesh.vert[i * VERT_SZ + j] = attrib.vertices[3 * i + j];
    // only the triangles become faces, in shape and face order
    for (const tinyobj::shape_t& shape : reader.GetShapes()) {
        size_t off = 0;
        for (const auto fv : shape.mesh.num_face_vertices) {
            if (fv == 3)
                for (size_t k = 0; k < 3; ++k) mesh.faces.push_back((unsigned int)shape.mesh.indices[off + k].vertex_index);
            off += fv;
        }
    }
    if (attrib.colors.size() / 3 >= nv)
        for (size_t i = 0; i < nv; ++i)
            for (int j = 0; j < 3; ++j) mesh.vert[i * VERT_SZ + 3 + j] = attrib.colors[3 * i + j];
    if (attrib.normals.size() / 3 >= nv) {
        for (size_t i = 0; i < nv; ++i)   // by vertex index
            for (int j = 0; j < 3; ++j) mesh.vert[i * VERT_SZ + 6 + j] = attrib.normals[3 * i + j];
    } else {
        estimate_normals(mesh.vert, mesh.faces);
    }
    mesh.face_size = 3;
    mesh.name = from_string ? "OBJ" : path_or_text;
    return mesh;
}

}  // namespace

// ---------------------------------------------------------------- Mesh
Mesh::Mesh(int n_verts, int n_faces, int face_size, bool unshaded)
    : vert(VERT_SZ * (size_t)std::max(n_verts, 0), 0.f),
      faces((size_t)std::max(n_faces, 0) * (size_t)std::max(face_size, 0), 0u),
      rotation(0.f),
      translation(0.f),
      transform_(1.f),
      face_size(face_size),
      unlit(unshaded),
      vao_(0),
      vbo_(0),
      ebo_(0) {}

void Mesh::update() {
    std::lock_guard<std::mutex> lk(g_up_mu);
    if (vao_ == 0) {
        g_uploads.emplace_back();
        vao_ = vbo_ = ebo_ = (unsigned int)g_uploads.size();
    }
    Upload& u = g_uploads[vao_ - 1];
    upload_into(u.vert_dev, u.vert_cap, vert.data(), vert.size());
    upload_into(u.faces_dev, u.faces_cap, reinterpret_cast<const uint32_t*>(faces.data()), faces.size());
    u.n_vert_floats = vert.size();
    u.n_face_idx = faces.size();
}

void Mesh::use_shader() {}

void Mesh::draw(const glm::mat4x4& V, glm::mat4x4 K, bool y_up) const {
    (void)V; (void)K; (void)y_up;   // the pass rasterizes with the renderer's camera, whose V and K these are
    if (!visible || vao_ == 0) return;
    b200::MeshPass* pass = b200::current_mesh_pass();
    if (pass == nullptr) {
        fprintf(stderr, "volrend_b200: Mesh::draw('%s') outside VolumeRenderer::render: nothing drawn\n",
                name.c_str());
        return;
    }
    Upload u;
    {
        std::lock_guard<std::mutex> lk(g_up_mu);
        u = g_uploads[vao_ - 1];
    }
    const size_t nv = u.n_vert_floats / VERT_SZ;
    if (nv > (size_t)INT32_MAX || u.n_face_idx / std::max(face_size, 1) > (size_t)INT32_MAX) {
        fprintf(stderr, "volrend_b200: Mesh::draw('%s'): more than 2^31-1 vertices or faces: nothing drawn\n",
                name.c_str());
        return;
    }
    transform_ = model_matrix(rotation, translation, scale);
    vr_mesh_desc d;
    memset(&d, 0, sizeof(d));
    d.vert_dev = nv ? u.vert_dev : nullptr;
    d.faces_dev = u.n_face_idx ? u.faces_dev : nullptr;
    d.n_verts = (int32_t)nv;
    d.n_faces = u.n_face_idx && face_size > 0 ? (int32_t)(u.n_face_idx / face_size) : 0;
    d.face_size = face_size;
    d.unlit = unlit ? 1 : 0;
    memcpy(d.model, &transform_[0][0], 16 * sizeof(float));
    pass->meshes.push_back(d);
}

void Mesh::auto_faces() {
    const size_t nv = vert.size() / VERT_SZ;
    faces.resize(nv);
    for (size_t i = 0; i < nv; ++i) faces[i] = (unsigned int)i;
}

void Mesh::repeat(int n) {
    if (n < 1) return;
    const unsigned int nv = (unsigned int)(vert.size() / VERT_SZ);
    const size_t vs = vert.size(), fs = faces.size();
    vert.resize(vs * n);
    faces.resize(fs * n);
    for (int i = 1; i < n; ++i) {
        std::copy(vert.begin(), vert.begin() + vs, vert.begin() + vs * i);
        for (size_t k = 0; k < fs; ++k) faces[fs * i + k] = faces[k] + (unsigned int)i * nv;
    }
}

void Mesh::apply_transform(glm::vec3 r, glm::vec3 t, int start, int end) {
    apply_transform(axis_angle_matrix(r, t), start, end);
}

void Mesh::apply_transform(glm::mat4 transform, int start, int end) {
    const int nv = (int)(vert.size() / VERT_SZ);
    if (end == -1) end = nv;
    start = std::max(start, 0);
    end = std::min(end, nv);
    for (int i = start; i < end; ++i) {
        float* p = &vert[(size_t)i * VERT_SZ];
        const float x = p[0], y = p[1], z = p[2];
        for (int k = 0; k < 3; ++k)
            p[k] = (transform[0][k] * x + transform[1][k] * y) + (transform[2][k] * z + transform[3][k]);
    }
}

Mesh Mesh::Cube(glm::vec3 color) {
    Mesh m(0, 0, 3);
    // faces -z, +z, -y, +y, -x, +x; two triangles each with corners (a, b) in units of 0.5, where (a, b) is (x, y)
    // on the z faces, (x, z) on the y faces and (z, y) on the x faces
    static const int corners[6][2] = {{-1, -1}, {1, 1}, {1, -1}, {1, 1}, {-1, -1}, {-1, 1}};
    static const int sides[6][2] = {{2, -1}, {2, 1}, {1, -1}, {1, 1}, {0, -1}, {0, 1}};
    for (const auto& as : sides) {
        const int axis = as[0], side = as[1];
        float n[3] = {0.f, 0.f, 0.f};
        n[axis] = (float)side;
        for (const auto& ab : corners) {
            float p[3] = {0.f, 0.f, 0.f};
            p[axis] = 0.5f * side;
            if (axis == 2) { p[0] = 0.5f * ab[0]; p[1] = 0.5f * ab[1]; }
            else if (axis == 1) { p[0] = 0.5f * ab[0]; p[2] = 0.5f * ab[1]; }
            else { p[1] = 0.5f * ab[1]; p[2] = 0.5f * ab[0]; }
            push_vertex(m.vert, p[0], p[1], p[2], color, n[0], n[1], n[2]);
        }
    }
    m.name = "Cube";
    return m;
}

Mesh Mesh::Sphere(int rings, int sectors, glm::vec3 color) {
    Mesh m(0, 0, 3);
    const double R = (float)(M_PI / (double)(float)(rings - 1));
    const double S = (float)(2 * M_PI / (double)(float)sectors);
    m.vert.reserve((size_t)std::max(rings * sectors, 0) * VERT_SZ);
    for (int r = 0; r < rings; ++r) {
        const double rR = (float)(r * R);
        for (int s = 0; s < sectors; ++s) {
            const double sS = (float)(s * S);
            const double z = std::sin(-0.5 * M_PI + rR);
            const double x = std::cos(sS) * std::sin(rR);
            const double y = std::sin(sS) * std::sin(rR);
            push_vertex(m.vert, (float)x, (float)y, (float)z, color, (float)x, (float)y, (float)z);
        }
    }
    for (int r = 0; r + 1 < rings; ++r) {
        const int nr = r + 1;
        for (int s = 0; s < sectors; ++s) {
            const int ns = (s + 1) % sectors;
            const unsigned int f[6] = {(unsigned)(r * sectors + ns), (unsigned)(r * sectors + s),
                                       (unsigned)(nr * sectors + s), (unsigned)(nr * sectors + s),
                                       (unsigned)(nr * sectors + ns), (unsigned)(r * sectors + ns)};
            m.faces.insert(m.faces.end(), f, f + 6);
        }
    }
    m.name = "Sphere";
    return m;
}

Mesh Mesh::Lattice(int reso, glm::vec3 color) {
    Mesh m(0, 0, 1);
    m.vert.reserve((size_t)reso * reso * reso * VERT_SZ);
    for (int i = 0; i < reso; ++i)
        for (int j = 0; j < reso; ++j)
            for (int k = 0; k < reso; ++k)
                push_vertex(m.vert, ((float)i + 0.5f) / (float)reso, ((float)j + 0.5f) / (float)reso,
                            ((float)k + 0.5f) / (float)reso, color, 1.f, 0.f, 0.f);
    m.name = "Lattice";
    m.unlit = true;
    return m;
}

Mesh Mesh::CameraFrustum(float focal_length, float image_width, float image_height, float z, glm::vec3 color) {
    Mesh m(0, 0, 2);
    const float invf = 1.f / focal_length;
    const float hw = image_width * 0.5f, hh = image_height * 0.5f;
    const float corners[4][2] = {{-hw, -hh}, {-hw, hh}, {hw, hh}, {hw, -hh}};
    push_vertex(m.vert, 0.f, 0.f, 0.f, color, 0.f, 0.f, 1.f);
    for (const auto& c : corners) push_vertex(m.vert, (z * c[0]) * invf, (z * c[1]) * invf, z, color, 0.f, 0.f, 1.f);
    m.faces = {0, 1, 0, 2, 0, 3, 0, 4, 1, 2, 2, 3, 3, 4, 4, 1};
    m.name = "CameraFrustum";
    m.unlit = true;
    return m;
}

Mesh Mesh::Line(glm::vec3 a, glm::vec3 b, glm::vec3 color) {
    Mesh m(0, 0, 2);
    push_vertex(m.vert, a[0], a[1], a[2], color, 0.f, 0.f, 1.f);
    push_vertex(m.vert, b[0], b[1], b[2], color, 0.f, 0.f, 1.f);
    m.faces = {0, 1};
    m.name = "Line";
    m.unlit = true;
    return m;
}

Mesh Mesh::Lines(std::vector<float> points, glm::vec3 color) {
    Mesh m(0, 0, 2);
    const size_t n = point_vertices(m, points, color, "Lines");
    for (size_t i = 0; i + 1 < n; ++i) {
        m.faces.push_back((unsigned int)i);
        m.faces.push_back((unsigned int)(i + 1));
    }
    m.name = "Lines";
    m.unlit = true;
    return m;
}

Mesh Mesh::Points(std::vector<float> points, glm::vec3 color) {
    Mesh m(0, 0, 1);
    point_vertices(m, points, color, "Points");
    m.name = "Points";
    m.unlit = true;
    return m;
}

Mesh Mesh::load_basic_obj(const std::string& path) { return load_obj(path, false); }
Mesh Mesh::load_mem_basic_obj(const std::string& str) { return load_obj(str, true); }

std::vector<Mesh> Mesh::open_drawlist(const std::string& path, bool default_visible) {
    return load_npz(cnpy::npz_load(path), default_visible);
}
std::vector<Mesh> Mesh::open_drawlist_mem(const char* data, uint64_t size, bool default_visible) {
    return load_npz(cnpy::npz_load_mem(data, size), default_visible);
}

}  // namespace volrend
