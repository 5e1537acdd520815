// shim_mesh.cpp -- test driver of the C++ volrend::Mesh and of VolumeRenderer with meshes, probe and grid.
//   shim_mesh <script>
// The script holds one command per line ('#' starts a comment).  Meshes live in one list, indexed from 0; after
// `renderer` that list is the renderer's `meshes`.
//   mesh construction (appends):  cube r g b | sphere rings sectors r g b | lattice reso r g b
//       | frustum focal w h z r g b | line ax ay az bx by bz r g b | lines pts.f32 r g b | points pts.f32 r g b
//       | empty n_verts n_faces face_size unlit | from vert.f32 faces.u32 face_size | copy i
//       | obj path | objmem path | drawlist path default_visible | drawlistmem path default_visible
//   mesh edits:  autofaces i | repeat i n | xf i rx ry rz tx ty tz start end | xfm i m0..m15 start end (column-major)
//       | rotation i x y z | translation i x y z | scale i s | visible i b | unlit i b | facesize i n
//       | vert i k value | update i
//   output:  save i dir   (raw arrays in an existing directory: vert.f32, faces.u32, name.u8, f7.f32 = scale,
//                          translation, rotation, i3.i32 = face_size, visible, unlit, transform.f32 = transform_,
//                          column-major)
//   renderer:  renderer | tree path | set | clear | size w h | fx f | pose pose.txt (3x4 c2w, row-major)
//       | bg v | probe enable x y z | grid show max_depth | render out.rgba out_c2w.f32
//   (`render` writes the frame as RGBA8, row 0 = top, and the camera's 4x3 c2w after Camera::_update, 12 floats.)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <memory>
#include <sstream>
#include <string>
#include <vector>

#include "volrend/common.hpp"
#include "volrend/mesh.hpp"
#include "volrend/n3tree.hpp"
#include "volrend/renderer.hpp"
#include "volrend_b200_shim.hpp"

using namespace volrend;

namespace {

std::string read_bytes(const std::string& path) {
    std::ifstream f(path, std::ios::binary);
    if (!f) {
        fprintf(stderr, "shim_mesh: cannot read %s\n", path.c_str());
        exit(2);
    }
    return std::string(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}

template <class T>
std::vector<T> read_array(const std::string& path) {
    const std::string b = read_bytes(path);
    std::vector<T> v(b.size() / sizeof(T));
    if (!v.empty()) memcpy(v.data(), b.data(), v.size() * sizeof(T));
    return v;
}

template <class T>
void save(const std::string& dir, const std::string& key, const T* data, size_t n) {
    const std::string path = dir + "/" + key;
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) {
        fprintf(stderr, "shim_mesh: cannot write %s\n", path.c_str());
        exit(2);
    }
    if (n) fwrite(data, sizeof(T), n, f);
    fclose(f);
}

// Every field of a mesh as a raw little-endian array in `dir` (which must exist), one file per field.
void save_mesh(const Mesh& m, const std::string& dir) {
    save(dir, "vert.f32", m.vert.data(), m.vert.size());
    save(dir, "faces.u32", m.faces.data(), m.faces.size());
    save(dir, "name.u8", m.name.data(), m.name.size());
    const float f7[7] = {m.scale, m.translation[0], m.translation[1], m.translation[2],
                         m.rotation[0], m.rotation[1], m.rotation[2]};
    save(dir, "f7.f32", f7, 7);
    const int32_t i3[3] = {m.face_size, m.visible ? 1 : 0, m.unlit ? 1 : 0};
    save(dir, "i3.i32", i3, 3);
    save(dir, "transform.f32", &m.transform_[0][0], 16);
}

glm::vec3 vec3_at(const std::vector<std::string>& t, size_t i) {
    return glm::vec3(std::stof(t[i]), std::stof(t[i + 1]), std::stof(t[i + 2]));
}

}  // namespace

int main(int argc, char** argv) {
    if (argc < 2) {
        fprintf(stderr, "usage: shim_mesh <script>\n");
        return 2;
    }
    std::ifstream script(argv[1]);
    if (!script) {
        fprintf(stderr, "shim_mesh: cannot open %s\n", argv[1]);
        return 2;
    }
    std::vector<Mesh> local;
    std::vector<Mesh>* ms = &local;
    std::unique_ptr<VolumeRenderer> rend;
    std::unique_ptr<N3Tree> tree;
    std::string line;
    int line_no = 0;
    while (std::getline(script, line)) {
        ++line_no;
        const size_t hash = line.find('#');
        if (hash != std::string::npos) line.resize(hash);
        std::istringstream ss(line);
        std::vector<std::string> t{std::istream_iterator<std::string>(ss), std::istream_iterator<std::string>()};
        if (t.empty()) continue;
        const std::string& c = t[0];
        auto mesh = [&](size_t k) -> Mesh& { return ms->at(std::stoul(t[k])); };
        auto need_rend = [&]() -> VolumeRenderer& {
            if (!rend) {
                fprintf(stderr, "shim_mesh: line %d: '%s' before 'renderer'\n", line_no, c.c_str());
                exit(2);
            }
            return *rend;
        };
        if (c == "cube") {
            ms->push_back(Mesh::Cube(vec3_at(t, 1)));
        } else if (c == "sphere") {
            ms->push_back(Mesh::Sphere(std::stoi(t[1]), std::stoi(t[2]), vec3_at(t, 3)));
        } else if (c == "lattice") {
            ms->push_back(Mesh::Lattice(std::stoi(t[1]), vec3_at(t, 2)));
        } else if (c == "frustum") {
            ms->push_back(Mesh::CameraFrustum(std::stof(t[1]), std::stof(t[2]), std::stof(t[3]), std::stof(t[4]),
                                              vec3_at(t, 5)));
        } else if (c == "line") {
            ms->push_back(Mesh::Line(vec3_at(t, 1), vec3_at(t, 4), vec3_at(t, 7)));
        } else if (c == "lines") {
            ms->push_back(Mesh::Lines(read_array<float>(t[1]), vec3_at(t, 2)));
        } else if (c == "points") {
            ms->push_back(Mesh::Points(read_array<float>(t[1]), vec3_at(t, 2)));
        } else if (c == "empty") {
            ms->push_back(Mesh(std::stoi(t[1]), std::stoi(t[2]), std::stoi(t[3]), std::stoi(t[4]) != 0));
        } else if (c == "from") {
            Mesh m(0, 0, std::stoi(t[3]));
            m.vert = read_array<float>(t[1]);
            m.faces = read_array<unsigned int>(t[2]);
            ms->push_back(std::move(m));
        } else if (c == "copy") {
            const Mesh m = mesh(1);
            ms->push_back(m);
        } else if (c == "obj") {
            ms->push_back(Mesh::load_basic_obj(t[1]));
        } else if (c == "objmem") {
            ms->push_back(Mesh::load_mem_basic_obj(read_bytes(t[1])));
        } else if (c == "drawlist" || c == "drawlistmem") {
            std::vector<Mesh> got;
            if (c == "drawlist") {
                got = Mesh::open_drawlist(t[1], std::stoi(t[2]) != 0);
            } else {
                const std::string b = read_bytes(t[1]);
                got = Mesh::open_drawlist_mem(b.data(), b.size(), std::stoi(t[2]) != 0);
            }
            ms->insert(ms->end(), got.begin(), got.end());
        } else if (c == "autofaces") {
            mesh(1).auto_faces();
        } else if (c == "repeat") {
            mesh(1).repeat(std::stoi(t[2]));
        } else if (c == "xf") {
            mesh(1).apply_transform(vec3_at(t, 2), vec3_at(t, 5), std::stoi(t[8]), std::stoi(t[9]));
        } else if (c == "xfm") {
            glm::mat4 m;
            for (int k = 0; k < 16; ++k) m[k / 4][k % 4] = std::stof(t[2 + k]);
            mesh(1).apply_transform(m, std::stoi(t[18]), std::stoi(t[19]));
        } else if (c == "rotation") {
            mesh(1).rotation = vec3_at(t, 2);
        } else if (c == "translation") {
            mesh(1).translation = vec3_at(t, 2);
        } else if (c == "scale") {
            mesh(1).scale = std::stof(t[2]);
        } else if (c == "visible") {
            mesh(1).visible = std::stoi(t[2]) != 0;
        } else if (c == "unlit") {
            mesh(1).unlit = std::stoi(t[2]) != 0;
        } else if (c == "facesize") {
            mesh(1).face_size = std::stoi(t[2]);
        } else if (c == "vert") {
            mesh(1).vert.at(std::stoul(t[2])) = std::stof(t[3]);
        } else if (c == "update") {
            mesh(1).update();
        } else if (c == "save") {
            save_mesh(mesh(1), t[2]);
        } else if (c == "renderer") {
            rend = std::make_unique<VolumeRenderer>();
            rend->meshes = std::move(local);
            ms = &rend->meshes;
        } else if (c == "tree") {
            tree = std::make_unique<N3Tree>(t[1]);
            if (!tree->is_data_loaded() || !tree->is_cuda_loaded()) {
                fprintf(stderr, "shim_mesh: tree %s not loaded\n", t[1].c_str());
                return 3;
            }
        } else if (c == "set") {
            need_rend().set(*tree);
        } else if (c == "clear") {
            need_rend().clear();
        } else if (c == "size") {
            need_rend().resize(std::stoi(t[1]), std::stoi(t[2]));
        } else if (c == "fx") {
            need_rend().camera.fx = need_rend().camera.fy = std::stof(t[1]);
        } else if (c == "pose") {
            // express the pose through the camera's own pose model (camera.hpp:28-32)
            std::ifstream pf(t[1]);
            glm::mat4x3 p;
            for (int r = 0; r < 3; ++r)
                for (int k = 0; k < 4; ++k) pf >> p[k][r];
            if (!pf) {
                fprintf(stderr, "shim_mesh: bad pose file %s\n", t[1].c_str());
                return 2;
            }
            VolumeRenderer& r = need_rend();
            r.camera.v_back = p[2];
            r.camera.v_world_up = p[1];
            r.camera.center = p[3];
        } else if (c == "bg") {
            need_rend().options.background_brightness = std::stof(t[1]);
        } else if (c == "probe") {
            VolumeRenderer& r = need_rend();
            r.options.enable_probe = std::stoi(t[1]) != 0;
            for (int k = 0; k < 3; ++k) r.options.probe[k] = std::stof(t[2 + k]);
        } else if (c == "grid") {
            VolumeRenderer& r = need_rend();
            r.options.show_grid = std::stoi(t[1]) != 0;
            r.options.grid_max_depth = std::stoi(t[2]);
        } else if (c == "render") {
            VolumeRenderer& r = need_rend();
            r.render();
            std::vector<uint8_t> buf((size_t)4 * r.camera.width * r.camera.height);
            if (!volrend_b200_read_pixels(r, buf.data())) {
                fprintf(stderr, "shim_mesh: read_pixels failed\n");
                return 4;
            }
            FILE* f = fopen(t[1].c_str(), "wb");
            fwrite(buf.data(), 1, buf.size(), f);
            fclose(f);
            f = fopen(t[2].c_str(), "wb");
            fwrite(&r.camera.transform[0][0], sizeof(float), 12, f);
            fclose(f);
        } else {
            fprintf(stderr, "shim_mesh: line %d: unknown command '%s'\n", line_no, c.c_str());
            return 2;
        }
    }
    fflush(stdout);
    return 0;
}
