// vr_png.cpp -- image egress: RGBA8 frames -> PNG files without libpng.
//
// The reference writes 8-bit RGBA, non-interlaced PNGs with compression level 0 and filter NONE
// (src/imwrite.cpp:27-29,45-47) and calls it "a huge bottleneck" (README.md:128).  With level 0 a
// PNG is only a container: signature, IHDR, one IDAT holding a zlib stream of *stored* deflate
// blocks, IEND -- plus CRC-32 per chunk and Adler-32 over the raw scanlines.  That is what this file
// emits (zlib's crc32/adler32 do the checksums), so any PNG reader decodes exactly the bytes
// launch_renderer produced.  vr_render_frames_png overlaps rendering, D2H copies and encoding.
#include <zlib.h>

#include <atomic>
#include <cerrno>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "volrend_b200.h"
#include "vr_frames.h"

namespace {

void put32(std::vector<unsigned char>& v, uint32_t x) {
    v.push_back((unsigned char)(x >> 24)); v.push_back((unsigned char)(x >> 16));
    v.push_back((unsigned char)(x >> 8)); v.push_back((unsigned char)x);
}

void chunk(std::vector<unsigned char>& out, const char type[4], const unsigned char* data, size_t n) {
    put32(out, (uint32_t)n);
    const size_t start = out.size();
    out.insert(out.end(), type, type + 4);
    if (n) out.insert(out.end(), data, data + n);
    const uint32_t crc = (uint32_t)crc32(crc32(0L, Z_NULL, 0), out.data() + start, (uInt)(n + 4));
    put32(out, crc);
}

void encode_png(const uint8_t* rgba, int w, int h, std::vector<unsigned char>& out) {
    const size_t row = (size_t)w * 4, raw_n = (row + 1) * (size_t)h;
    // zlib stream of stored blocks over [0x00 filter byte | row] x h
    std::vector<unsigned char> z;
    z.reserve(raw_n + raw_n / 65535 * 5 + 16);
    z.push_back(0x78); z.push_back(0x01);
    std::vector<unsigned char> raw(raw_n);
    for (int y = 0; y < h; ++y) {
        raw[(row + 1) * y] = 0;  // filter type NONE
        memcpy(&raw[(row + 1) * y + 1], rgba + row * y, row);
    }
    size_t pos = 0;
    while (pos < raw_n) {
        const size_t n = raw_n - pos < 65535 ? raw_n - pos : 65535;
        z.push_back(pos + n == raw_n ? 1 : 0);  // BFINAL, BTYPE=00 (stored)
        z.push_back((unsigned char)(n & 0xff)); z.push_back((unsigned char)(n >> 8));
        z.push_back((unsigned char)(~n & 0xff)); z.push_back((unsigned char)((~n >> 8) & 0xff));
        z.insert(z.end(), raw.begin() + pos, raw.begin() + pos + n);
        pos += n;
    }
    uLong ad = adler32(0L, Z_NULL, 0);
    for (size_t p = 0; p < raw_n; p += (1u << 30)) ad = adler32(ad, raw.data() + p, (uInt)((raw_n - p < (1u << 30)) ? raw_n - p : (1u << 30)));
    put32(z, (uint32_t)ad);

    static const unsigned char sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
    out.clear();
    out.reserve(z.size() + 64);
    out.insert(out.end(), sig, sig + 8);
    std::vector<unsigned char> ihdr;
    put32(ihdr, (uint32_t)w); put32(ihdr, (uint32_t)h);
    ihdr.push_back(8);  // bit depth
    ihdr.push_back(6);  // colour type RGBA
    ihdr.push_back(0); ihdr.push_back(0); ihdr.push_back(0);  // deflate, adaptive filter method, no interlace
    chunk(out, "IHDR", ihdr.data(), ihdr.size());
    chunk(out, "IDAT", z.data(), z.size());
    chunk(out, "IEND", nullptr, 0);
}

}  // namespace

extern "C" {

int vr_write_png(const char* path, const uint8_t* rgba8_host, int width, int height) {
    if (!path) return vrb::fail(VR_EINVAL, "null PNG path");
    if (!rgba8_host) return vrb::fail(VR_EINVAL, "%s: null pixel buffer", path);
    if (width <= 0 || height <= 0) return vrb::fail(VR_EINVAL, "%s: bad image size %dx%d", path, width, height);
    std::vector<unsigned char> png;
    encode_png(rgba8_host, width, height, png);
    FILE* f = fopen(path, "wb");
    if (!f) return vrb::fail(VR_EINVAL, "cannot open %s: %s", path, strerror(errno));
    const bool ok = fwrite(png.data(), 1, png.size(), f) == png.size();
    const int err = errno;
    fclose(f);
    return ok ? VR_OK : vrb::fail(VR_EINVAL, "cannot write %s: %s", path, strerror(err));
}

}  // extern "C"

namespace {

// vr_render_frames_png(_opts): opt_stride as in vr_frames.h
int render_frames_png(const vr_tree* tree, const vr_camera* cams, int n_views, const vr_options* opt, int opt_stride,
                      const char* const* paths, int n_threads) {
    if (n_views < 0) return vrb::fail(VR_EINVAL, "n_views < 0");
    if (n_views == 0) return VR_OK;
    if (!cams) return vrb::fail(VR_EINVAL, "null cameras");
    if (!paths) return vrb::fail(VR_EINVAL, "null PNG paths");
    if (n_threads < 1) n_threads = 1;
    const int w = cams[0].width, h = cams[0].height;
    const size_t frame = (size_t)4 * w * h;
    // render + D2H in slabs of a few dozen frames; encode slab k on the worker threads while slab k+1
    // renders (vr_render_frames_host pipelines launches and copies internally)
    const int slab = 32;
    std::vector<uint8_t> buf[2];
    buf[0].resize(frame * (size_t)(n_views < slab ? n_views : slab));
    buf[1].resize(buf[0].size());
    // vr_write_png sets the message on its worker thread: the first one is kept for the caller's thread
    std::mutex err_mu;
    std::string err;
    auto encode_slab = [&](const uint8_t* base, int v0, int nv) {
        std::atomic<int> next{0};
        std::vector<std::thread> th;
        for (int t = 0; t < n_threads; ++t)
            th.emplace_back([&, base, v0, nv] {
                for (;;) {
                    const int i = next.fetch_add(1);
                    if (i >= nv) break;
                    if (vr_write_png(paths[v0 + i], base + frame * (size_t)i, w, h) != VR_OK) {
                        std::lock_guard<std::mutex> lk(err_mu);
                        if (err.empty()) err = vr_last_error();
                    }
                }
            });
        for (auto& x : th) x.join();
    };
    std::thread pending;
    int k = 0;
    for (int v0 = 0; v0 < n_views; v0 += slab, ++k) {
        const int nv = n_views - v0 < slab ? n_views - v0 : slab;
        uint8_t* dst = buf[k & 1].data();
        const int rc = vrb::render_frames_host(tree, cams + v0, nv, opt + (size_t)opt_stride * v0, opt_stride, dst);
        if (rc != VR_OK) { if (pending.joinable()) pending.join(); return rc; }
        if (pending.joinable()) pending.join();   // previous slab's buffer is free again after this
        pending = std::thread(encode_slab, dst, v0, nv);
        // the next iteration renders into the other buffer while `pending` encodes this one
    }
    if (pending.joinable()) pending.join();
    return err.empty() ? VR_OK : vrb::fail(VR_EINVAL, "%s", err.c_str());
}

}  // namespace

extern "C" {

int vr_render_frames_png(const vr_tree* tree, const vr_camera* cams, int n_views, const vr_options* opt,
                         const char* const* paths, int n_threads) {
    return render_frames_png(tree, cams, n_views, opt, 0, paths, n_threads);
}

int vr_render_frames_png_opts(const vr_tree* tree, const vr_camera* cams, int n_views, const vr_options* opts,
                              const char* const* paths, int n_threads) {
    return render_frames_png(tree, cams, n_views, opts, 1, paths, n_threads);
}

}  // extern "C"
