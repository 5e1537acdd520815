// vr_raster.cu -- CUDA rasterizer for VolumeRenderer meshes (the GL mesh pass of cuda_renderer.cpp:83-113,
// vertex/fragment shaders src/mesh.cpp:98-160, draw :366-396), GL-free.  DESIGN.md section 8.
//
// Four launches per call, all on the caller's stream, each covering every view of the launch (one z-buffer per view;
// a single-view draw is a launch of one view; DESIGN.md section 15):
//   z_init      z-buffer key per pixel = (bits(depth_dev), 0)
//   raster      one thread per primitive of any view: transform, clip, snap; sub-primitives whose pixel bounding
//               box is at most kSmallPixels are rasterized by that thread, larger ones go to its view's list
//   raster_big  one CTA per (view, 32x32 tile) walks that view's list (a frame-filling triangle is spread
//               over every CTA of its view instead of one thread)
//   resolve     one thread per pixel re-evaluates the primitive that won the pixel: perspective-correct
//               attributes, the fixed three-light Phong shader, RGBA8 + ray distance
// Every fragment does one 64-bit atomicMin on (ray-distance bits << 32 | draw sequence number); the
// minimum does not depend on atomic order, so the output is bit-reproducible.
//
// All float arithmetic that decides coverage, depth or the winner uses explicitly rounded operations
// (no FMA contraction) so that oracle/mesh_oracle.py, a numpy restatement, reproduces it bit for bit.
#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>
#include <vector>
#include <string.h>

#include "vr_raster.h"

namespace vrb {
namespace {

constexpr float kNear = 1e-3f;         // CLIP_NEAR (camera.cpp:58); the far plane is at infinity
constexpr float kGuard = 1048576.f;    // guard band: clip where |window - centre| > 2^20 pixels
constexpr float kMaxWin = 4194304.f;   // window coordinates beyond 2^22 (only NaN/inf inputs) drop the primitive
constexpr int kSmallPixels = 256;      // bounding boxes up to 16x16 pixels stay with their setup thread
constexpr int kTile = 32;              // raster_big tile side
constexpr int kMaxPoly = 8;            // triangle clipped by 5 planes

__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fs(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fd(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float dot3(const float* a, const float* b) {
    return fa(fa(fm(a[0], b[0]), fm(a[1], b[1])), fm(a[2], b[2]));
}
__device__ __forceinline__ long long floor_div(long long a, long long b) {  // b > 0
    return a >= 0 ? a / b : -((-a + b - 1) / b);
}
__device__ __forceinline__ long long ceil_div(long long a, long long b) { return -floor_div(-a, b); }

// Clipped polygon: camera-space positions and weights of the primitive's original vertices.
struct Poly {
    int n;
    float q[kMaxPoly][3];
    float w[kMaxPoly][3];
};

// One rasterizable sub-primitive (kind = vertex count: 1 point, 2 line, 3 triangle).
struct Sub {
    int kind;
    long long X[3], Y[3];  // window coordinates, 8 sub-pixel bits
    long long A;           // triangles: twice the area (> 0); lines: major-axis length (> 0)
    bool xmajor;
    float q[3][3], d[3], w[3][3];
    int x0, y0, x1, y1;    // pixel bounding box, clamped to the frame (empty when x0 > x1 or y0 > y1)
    long long ox, oy;      // points: first covered column / row (unclamped)
};

__device__ int find_mesh(const RasterMesh* M, int n, long long g) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (M[mid].base <= g) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// Signed distance to clip plane i (>= 0 inside): near plane, then the four guard-band planes.
__device__ float plane(const RasterFrame& f, int i, const float* q) {
    const float d = -q[2];
    switch (i) {
        case 0: return fs(d, kNear);
        case 1: return fs(fm(kGuard, d), fm(f.fx, q[0]));
        case 2: return fa(fm(kGuard, d), fm(f.fx, q[0]));
        case 3: return fs(fm(kGuard, d), fm(f.fy, q[1]));
        default: return fa(fm(kGuard, d), fm(f.fy, q[1]));
    }
}

// Intersection on the edge from an inside vertex to an outside one (always in that direction, so two
// triangles that share a clipped edge get the same new vertex).
__device__ void clip_lerp(const float* qi, const float* wi, float di, const float* qo, const float* wo, float dout,
                          float* qr, float* wr) {
    const float t = fd(di, fs(di, dout));
    for (int k = 0; k < 3; ++k) {
        qr[k] = fa(qi[k], fm(t, fs(qo[k], qi[k])));
        wr[k] = fa(wi[k], fm(t, fs(wo[k], wi[k])));
    }
}

// Vertex shader position (mesh.cpp:115): FragPos = MV * aPos.
__device__ void xform(const RasterMesh& m, uint32_t vi, float* q) {
    const float* v = m.vert + (size_t)vi * 9;
    const float p0 = __ldg(v), p1 = __ldg(v + 1), p2 = __ldg(v + 2);
    for (int k = 0; k < 3; ++k)
        q[k] = fa(fa(fa(fm(m.mv[k], p0), fm(m.mv[3 + k], p1)), fm(m.mv[6 + k], p2)), m.mv[9 + k]);
}

// Fetches primitive lp of m, transforms and clips it.  Returns the number of sub-primitives (0: culled,
// or an index >= n_verts).  idx receives the original vertex indices.
__device__ __forceinline__ int clip_prim(const RasterMesh& m, long long lp, const RasterFrame& f, Poly& P, uint32_t* idx) {
    const int fsz = m.face_size;
    for (int j = 0; j < fsz; ++j) {
        const long long k = lp * fsz + j;
        const uint32_t vi = m.faces ? __ldg(m.faces + k) : (uint32_t)k;
        if (vi >= (uint32_t)m.n_verts) return 0;
        idx[j] = vi;
        xform(m, vi, P.q[j]);
        for (int i = 0; i < 3; ++i) P.w[j][i] = i == j ? 1.f : 0.f;
    }
    P.n = fsz;
    for (int pl = 0; pl < 5; ++pl) {
        float dist[kMaxPoly];
        bool all_in = true, any_in = false;
        for (int v = 0; v < P.n; ++v) {
            dist[v] = plane(f, pl, P.q[v]);
            const bool in = dist[v] >= 0.f;  // NaN counts as outside
            all_in &= in;
            any_in |= in;
        }
        if (all_in) continue;
        if (!any_in || fsz == 1) return 0;  // points are dropped when their centre is clipped
        if (fsz == 2) {
            const int o = dist[0] >= 0.f ? 1 : 0, i = 1 - o;
            clip_lerp(P.q[i], P.w[i], dist[i], P.q[o], P.w[o], dist[o], P.q[o], P.w[o]);
            continue;
        }
        Poly out;
        out.n = 0;
        for (int v = 0; v < P.n; ++v) {  // Sutherland-Hodgman
            const int u = v == 0 ? P.n - 1 : v - 1;
            const bool vin = dist[v] >= 0.f, uin = dist[u] >= 0.f;
            if (vin != uin) {
                const int a = vin ? v : u, b = vin ? u : v;
                clip_lerp(P.q[a], P.w[a], dist[a], P.q[b], P.w[b], dist[b], out.q[out.n], out.w[out.n]);
                ++out.n;
            }
            if (vin) {
                for (int k = 0; k < 3; ++k) { out.q[out.n][k] = P.q[v][k]; out.w[out.n][k] = P.w[v][k]; }
                ++out.n;
            }
        }
        P = out;
    }
    return fsz == 3 ? (P.n >= 3 ? P.n - 2 : 0) : 1;
}

template <class T>
__device__ __forceinline__ void swp(T& a, T& b) { T t = a; a = b; b = t; }

__device__ void swap_vert(Sub& S, int a, int b) {
    swp(S.X[a], S.X[b]); swp(S.Y[a], S.Y[b]); swp(S.d[a], S.d[b]);
    for (int k = 0; k < 3; ++k) { swp(S.q[a][k], S.q[b][k]); swp(S.w[a][k], S.w[b][k]); }
}

// Projects sub-primitive s of the clipped polygon (triangles: fan around vertex 0) and snaps it.
// Returns false for a degenerate primitive (zero area, zero length) or non-finite coordinates.
__device__ __forceinline__ bool make_sub(int kind, const Poly& P, int s, const RasterFrame& f, Sub& S) {
    S.kind = kind;
    for (int j = 0; j < kind; ++j) {
        const int v = j == 0 ? 0 : s + j;
        for (int k = 0; k < 3; ++k) { S.q[j][k] = P.q[v][k]; S.w[j][k] = P.w[v][k]; }
        const float d = -S.q[j][2];
        S.d[j] = d;
        // K (camera.cpp:60-63) + viewport: window x = W/2 + fx x / d, window y = H/2 - fy y / d; row 0 of
        // the output is window y in [0, 1), the top of the image, as in the march.
        const float xw = fa(f.cx, fd(fm(f.fx, S.q[j][0]), d));
        const float yw = fs(f.cy, fd(fm(f.fy, S.q[j][1]), d));
        if (!(fabsf(xw) <= kMaxWin) || !(fabsf(yw) <= kMaxWin)) return false;
        S.X[j] = __float2ll_rn(fm(xw, 256.f));
        S.Y[j] = __float2ll_rn(fm(yw, 256.f));
    }
    long long xlo, xhi, ylo, yhi;
    if (kind == 3) {
        long long A = (S.X[1] - S.X[0]) * (S.Y[2] - S.Y[0]) - (S.X[2] - S.X[0]) * (S.Y[1] - S.Y[0]);
        if (A == 0) return false;
        if (A < 0) { swap_vert(S, 1, 2); A = -A; }  // no face culling (main.cpp:628): both windings draw
        S.A = A;
        const long long mnx = min(S.X[0], min(S.X[1], S.X[2])), mxx = max(S.X[0], max(S.X[1], S.X[2]));
        const long long mny = min(S.Y[0], min(S.Y[1], S.Y[2])), mxy = max(S.Y[0], max(S.Y[1], S.Y[2]));
        xlo = ceil_div(mnx - 128, 256); xhi = floor_div(mxx - 128, 256);
        ylo = ceil_div(mny - 128, 256); yhi = floor_div(mxy - 128, 256);
    } else if (kind == 2) {
        const long long dX = S.X[1] - S.X[0], dY = S.Y[1] - S.Y[0];
        if (dX == 0 && dY == 0) return false;
        S.xmajor = (dX < 0 ? -dX : dX) >= (dY < 0 ? -dY : dY);
        if ((S.xmajor && dX < 0) || (!S.xmajor && dY < 0)) swap_vert(S, 0, 1);
        const long long* M0 = S.xmajor ? S.X : S.Y;
        const long long* N0 = S.xmajor ? S.Y : S.X;
        S.A = M0[1] - M0[0];
        const long long mlo = ceil_div(M0[0] - 128, 256), mhi = ceil_div(M0[1] - 128, 256) - 1;
        const long long nlo = floor_div(min(N0[0], N0[1]), 256), nhi = floor_div(max(N0[0], N0[1]), 256);
        if (S.xmajor) { xlo = mlo; xhi = mhi; ylo = nlo; yhi = nhi; }
        else { ylo = mlo; yhi = mhi; xlo = nlo; xhi = nhi; }
    } else {
        S.ox = ceil_div(S.X[0] - 640, 256);  // 4x4 pixels: centres within [X - 2, X + 2)
        S.oy = ceil_div(S.Y[0] - 640, 256);
        xlo = S.ox; xhi = S.ox + 3; ylo = S.oy; yhi = S.oy + 3;
    }
    S.x0 = (int)max(xlo, 0LL); S.x1 = (int)min(xhi, (long long)f.W - 1);
    S.y0 = (int)max(ylo, 0LL); S.y1 = (int)min(yhi, (long long)f.H - 1);
    return true;
}

__device__ __forceinline__ long long edge(long long Xa, long long Ya, long long Xb, long long Yb, long long PX,
                                          long long PY) {
    return (Xb - Xa) * (PY - Ya) - (Yb - Ya) * (PX - Xa);
}
// Top-left rule: a pixel centre exactly on an edge belongs to the triangle when the edge is a "left" edge
// (dy < 0) or a horizontal "top" edge (dy == 0, dx < 0); of two triangles sharing the edge, exactly one.
__device__ __forceinline__ bool edge_in(long long e, long long dx, long long dy) {
    return e > 0 || (e == 0 && (dy < 0 || (dy == 0 && dx < 0)));
}

// Whether the sub-primitive covers pixel (px, py) (sample at the pixel centre, as GL does).
__device__ __forceinline__ bool covers(const Sub& S, int px, int py) {
    const long long PX = (long long)px * 256 + 128, PY = (long long)py * 256 + 128;
    if (S.kind == 3) {
        return edge_in(edge(S.X[1], S.Y[1], S.X[2], S.Y[2], PX, PY), S.X[2] - S.X[1], S.Y[2] - S.Y[1]) &&
               edge_in(edge(S.X[2], S.Y[2], S.X[0], S.Y[0], PX, PY), S.X[0] - S.X[2], S.Y[0] - S.Y[2]) &&
               edge_in(edge(S.X[0], S.Y[0], S.X[1], S.Y[1], PX, PY), S.X[1] - S.X[0], S.Y[1] - S.Y[0]);
    }
    if (S.kind == 2) {
        // One pixel per column (x-major) or row (y-major) whose centre lies in [start, end): the pixel
        // containing the line's position at that centre.
        const long long* M0 = S.xmajor ? S.X : S.Y;
        const long long* N0 = S.xmajor ? S.Y : S.X;
        const long long P = S.xmajor ? PX : PY;
        if (P < M0[0] || P >= M0[1]) return false;
        const long long n = N0[0] + floor_div((P - M0[0]) * (N0[1] - N0[0]), S.A);
        return floor_div(n, 256) == (S.xmajor ? py : px);
    }
    return px >= S.ox && px <= S.ox + 3 && py >= S.oy && py <= S.oy + 3;
}

// Perspective-correct weights of the sub-primitive's vertices at pixel (px, py).
__device__ __forceinline__ void weights(const Sub& S, int px, int py, float* lam) {
    const long long PX = (long long)px * 256 + 128, PY = (long long)py * 256 + 128;
    if (S.kind == 3) {
        const long long E[3] = {edge(S.X[1], S.Y[1], S.X[2], S.Y[2], PX, PY),
                                edge(S.X[2], S.Y[2], S.X[0], S.Y[0], PX, PY),
                                edge(S.X[0], S.Y[0], S.X[1], S.Y[1], PX, PY)};
        const double Ad = __ll2double_rn(S.A);
        float r[3];
        for (int j = 0; j < 3; ++j) r[j] = fd(__double2float_rn(__ddiv_rn(__ll2double_rn(E[j]), Ad)), S.d[j]);
        const float s = fa(fa(r[0], r[1]), r[2]);
        for (int j = 0; j < 3; ++j) lam[j] = fd(r[j], s);
    } else if (S.kind == 2) {
        const long long P = S.xmajor ? PX : PY, M0 = S.xmajor ? S.X[0] : S.Y[0];
        const float t = __double2float_rn(__ddiv_rn(__ll2double_rn(P - M0), __ll2double_rn(S.A)));
        const float r0 = fd(fs(1.f, t), S.d[0]), r1 = fd(t, S.d[1]);
        const float s = fa(r0, r1);
        lam[0] = fd(r0, s); lam[1] = fd(r1, s); lam[2] = 0.f;
    } else {
        lam[0] = 1.f; lam[1] = 0.f; lam[2] = 0.f;
    }
}

// Camera-space position (FragPos) at the fragment; returns its length, the shader's Depth output.
__device__ float frag_pos(const Sub& S, const float* lam, float* P) {
    for (int k = 0; k < 3; ++k) {
        float acc = fm(lam[0], S.q[0][k]);
        for (int j = 1; j < S.kind; ++j) acc = fa(acc, fm(lam[j], S.q[j][k]));
        P[k] = acc;
    }
    return __fsqrt_rn(dot3(P, P));
}

__device__ __forceinline__ unsigned long long frag_key(float depth, unsigned int seq) {
    return ((unsigned long long)__float_as_uint(depth) << 32) | seq;
}

__device__ __forceinline__ void fragment(const Sub& S, int px, int py, unsigned int seq, int W,
                                         unsigned long long* zbuf) {
    float lam[3], P[3];
    weights(S, px, py, lam);
    const float depth = frag_pos(S, lam, P);
    if (!(depth <= 3.4e38f)) return;  // NaN / inf never wins
    atomicMin(zbuf + (size_t)py * W + px, frag_key(depth, seq));
}

// Grid: (pixel blocks, views).
__global__ void z_init(const RasterFrame* __restrict__ frames, unsigned long long* __restrict__ zbuf, long long n) {
    const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const float* depth = frames[blockIdx.y].depth;
    // sequence 0: a fragment at the same distance fails (LESS)
    if (i < n) zbuf[blockIdx.y * n + i] = frag_key(depth[i], 0u);
}

__global__ void __launch_bounds__(128) raster(const RasterMesh* __restrict__ meshes, int n_meshes, long long total,
                                              const RasterFrame* __restrict__ frames, unsigned long long* zbuf,
                                              uint4* large, unsigned int* n_large) {
    const long long g = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    if (g >= total) return;
    const RasterMesh& m = meshes[find_mesh(meshes, n_meshes, g)];
    const RasterFrame& f = frames[m.view];
    zbuf += (size_t)m.view * f.W * f.H;
    Poly P;
    uint32_t idx[3];
    const int nsub = clip_prim(m, g - m.base, f, P, idx);
    for (int s = 0; s < nsub; ++s) {
        Sub S;
        if (!make_sub(m.face_size, P, s, f, S) || S.x0 > S.x1 || S.y0 > S.y1) continue;
        const unsigned int seq = (unsigned int)(g * 8 + s + 1);
        if ((long long)(S.x1 - S.x0 + 1) * (S.y1 - S.y0 + 1) > kSmallPixels) {
            const unsigned int slot = atomicAdd(n_large + m.view, 1u);
            large[f.large_off + slot] = make_uint4(seq, (unsigned)S.x0 | ((unsigned)S.y0 << 16),
                                     (unsigned)S.x1 | ((unsigned)S.y1 << 16), 0u);
            continue;
        }
        for (int y = S.y0; y <= S.y1; ++y)
            for (int x = S.x0; x <= S.x1; ++x)
                if (covers(S, x, y)) fragment(S, x, y, seq, f.W, zbuf);
    }
}

__device__ __forceinline__ bool load_sub(const RasterMesh* meshes, int n_meshes, unsigned int seq, const RasterFrame& f, Sub& S,
                         const RasterMesh** mp, uint32_t* idx) {
    const long long g = (seq - 1u) >> 3;
    const int s = (seq - 1u) & 7;
    const RasterMesh& m = meshes[find_mesh(meshes, n_meshes, g)];
    *mp = &m;
    Poly P;
    const int nsub = clip_prim(m, g - m.base, f, P, idx);
    return s < nsub && make_sub(m.face_size, P, s, f, S);
}

// Grid: (tile columns, tile rows, views); a CTA walks its own view's list only.  Three CTAs per SM: without the bound
// the per-view frame pointer raises the kernel to 100 registers (two CTAs).
__global__ void __launch_bounds__(256, 3) raster_big(const RasterMesh* __restrict__ meshes, int n_meshes,
                                                  const RasterFrame* __restrict__ frames, unsigned long long* zbuf,
                                                  const uint4* __restrict__ large,
                                                  const unsigned int* __restrict__ n_large) {
    const RasterFrame& f = frames[blockIdx.z];
    zbuf += (size_t)blockIdx.z * f.W * f.H;
    large += f.large_off;
    const int tx0 = blockIdx.x * kTile, ty0 = blockIdx.y * kTile;
    const int tx1 = min(tx0 + kTile - 1, f.W - 1), ty1 = min(ty0 + kTile - 1, f.H - 1);
    const int px = tx0 + (threadIdx.x & (kTile - 1));
    const unsigned int n = n_large[blockIdx.z];
    for (unsigned int e = 0; e < n; ++e) {
        const uint4 L = large[e];
        const int x0 = L.y & 0xffff, y0 = L.y >> 16, x1 = L.z & 0xffff, y1 = L.z >> 16;
        if (x1 < tx0 || x0 > tx1 || y1 < ty0 || y0 > ty1) continue;  // uniform over the CTA
        Sub S;
        const RasterMesh* m;
        uint32_t idx[3];
        if (!load_sub(meshes, n_meshes, L.x, f, S, &m, idx)) continue;
        if (px < x0 || px > x1) continue;
        for (int py = ty0 + (threadIdx.x >> 5); py <= min(ty1, y1); py += blockDim.x >> 5)
            if (py >= y0 && covers(S, px, py)) fragment(S, px, py, L.x, f.W, zbuf);
    }
}

__device__ void normalize3(float* v) {
    const float len = __fsqrt_rn(dot3(v, v));
    if (len > 0.f)
        for (int k = 0; k < 3; ++k) v[k] = fd(v[k], len);
}

__device__ __forceinline__ uint8_t to_u8(float v) {
    return (uint8_t)__float2int_rn(fm(fminf(fmaxf(v, 0.f), 1.f), 255.f));
}

// Grid: (32-pixel columns, 4-pixel rows, views).
__global__ void __launch_bounds__(128) resolve(const RasterMesh* __restrict__ meshes, int n_meshes,
                                               const RasterFrame* __restrict__ frames,
                                               const unsigned long long* __restrict__ zbuf) {
    const RasterFrame& f = frames[blockIdx.z];
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 4 + (threadIdx.x >> 5);
    if (x >= f.W || y >= f.H) return;
    const unsigned int p = (unsigned int)(y * f.W + x);   // W * H <= 2^30
    const unsigned int seq = (unsigned int)zbuf[(size_t)blockIdx.z * f.W * f.H + p];
    if (seq == 0u) return;  // no fragment beat the incoming depth: colour and depth stay
    Sub S;
    const RasterMesh* mp;
    uint32_t idx[3];
    if (!load_sub(meshes, n_meshes, seq, f, S, &mp, idx)) return;
    const RasterMesh& m = *mp;
    float lam[3], P[3];
    weights(S, x, y, lam);
    const float dist = frag_pos(S, lam, P);
    // Weights of the primitive's original vertices (the sub-primitive's vertices are clip-space blends).
    float om[3];
    for (int i = 0; i < 3; ++i) {
        float acc = fm(lam[0], S.w[0][i]);
        for (int j = 1; j < S.kind; ++j) acc = fa(acc, fm(lam[j], S.w[j][i]));
        om[i] = acc;
    }
    float col[3] = {0.f, 0.f, 0.f}, nrm[3] = {0.f, 0.f, 0.f};
    for (int i = 0; i < m.face_size; ++i) {
        const float* v = m.vert + (size_t)idx[i] * 9;
        float n[3];
        for (int k = 0; k < 3; ++k) {
            n[k] = fa(fa(fm(m.m3[k], __ldg(v + 6)), fm(m.m3[3 + k], __ldg(v + 7))), fm(m.m3[6 + k], __ldg(v + 8)));
        }
        normalize3(n);  // Normal = normalize(mat3x3(M) * aNormal), per vertex (mesh.cpp:118)
        for (int k = 0; k < 3; ++k) {
            const float c = fm(om[i], __ldg(v + 3 + k)), nn = fm(om[i], n[k]);
            col[k] = i == 0 ? c : fa(col[k], c);
            nrm[k] = i == 0 ? nn : fa(nrm[k], nn);
        }
    }
    float out[4];
    if (m.unlit) {
        out[0] = col[0]; out[1] = col[1]; out[2] = col[2]; out[3] = 1.f;
    } else {
        // mesh.cpp:141-156.  The interpolated normal is not renormalized, and viewDir subtracts the
        // camera-space FragPos from the world-space camPos, exactly as the reference shader does.
        float L1[3] = {0.5f, 0.2f, 1.f}, L2[3] = {-0.5f, -1.f, -0.5f};
        normalize3(L1);
        normalize3(L2);
        const float diffuse = fm(0.7f, fmaxf(dot3(L1, nrm), 0.f));
        const float diffuse2 = fm(0.2f, fmaxf(dot3(L2, nrm), 0.f));
        float V[3] = {fs(f.cam_pos[0], P[0]), fs(f.cam_pos[1], P[1]), fs(f.cam_pos[2], P[2])};
        normalize3(V);
        const float I[3] = {-L1[0], -L1[1], -L1[2]};
        const float dNI2 = fm(2.f, dot3(nrm, I));
        const float R[3] = {fs(I[0], fm(dNI2, nrm[0])), fs(I[1], fm(dNI2, nrm[1])), fs(I[2], fm(dNI2, nrm[2]))};
        float sp = fmaxf(dot3(V, R), 0.f);
        for (int k = 0; k < 5; ++k) sp = fm(sp, sp);  // pow(., 32)
        const float sum = fa(fa(fa(0.3f, diffuse), diffuse2), fm(0.6f, sp));
        out[0] = fm(sum, col[0]); out[1] = fm(sum, col[1]); out[2] = fm(sum, col[2]); out[3] = sum;
    }
    uchar4 o;
    o.x = to_u8(out[0]); o.y = to_u8(out[1]); o.z = to_u8(out[2]); o.w = to_u8(out[3]);
    reinterpret_cast<uchar4*>(f.rgba8)[p] = o;
    f.depth[p] = dist;
}

}  // namespace

// Scratch comes from a memory pool of the rasterizer's own per device, which keeps what it has reserved (the
// default pool returns memory at every synchronisation, and re-mapping it cost more than the draw itself).
// Allocation is stream-ordered, so concurrent calls on different streams never share scratch.
cudaError_t scratch_pool(cudaMemPool_t* out) {
    static std::mutex mu;
    static cudaMemPool_t pools[64] = {};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
    std::lock_guard<std::mutex> g(mu);
    if (!pools[dev]) {
        cudaMemPoolProps p{};
        p.allocType = cudaMemAllocationTypePinned;
        p.location.type = cudaMemLocationTypeDevice;
        p.location.id = dev;
        cudaMemPool_t pool;
        if ((e = cudaMemPoolCreate(&pool, &p)) != cudaSuccess) return e;
        uint64_t keep = UINT64_MAX;
        if ((e = cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep)) != cudaSuccess) return e;
        pools[dev] = pool;
    }
    *out = pools[dev];
    return cudaSuccess;
}

cudaError_t raster_draw(const RasterFrame* frames, int n_views, const RasterMesh* meshes, int n, long long total_prims,
                        long long large_total, cudaStream_t st) {
    const int W = frames[0].W, H = frames[0].H;
    const long long npx = (long long)W * H;
    // scratch: z-buffers | meshes | frames | per-view list counters | large-primitive lists
    const size_t z_bytes = (size_t)npx * 8 * n_views, m_bytes = sizeof(RasterMesh) * (size_t)n;
    const size_t f_bytes = sizeof(RasterFrame) * (size_t)n_views, c_bytes = ((size_t)n_views * 4 + 15) / 16 * 16;
    const size_t m_off = z_bytes, f_off = (m_off + m_bytes + 15) / 16 * 16, c_off = (f_off + f_bytes + 15) / 16 * 16;
    const size_t l_off = c_off + c_bytes;
    const size_t bytes = l_off + (size_t)large_total * sizeof(uint4);
    cudaMemPool_t pool;
    cudaError_t e = scratch_pool(&pool);
    if (e != cudaSuccess) return e;
    unsigned char* scratch = nullptr;
    if ((e = cudaMallocFromPoolAsync((void**)&scratch, bytes, pool, st)) != cudaSuccess) return e;
    unsigned long long* zbuf = reinterpret_cast<unsigned long long*>(scratch);
    RasterMesh* dmesh = reinterpret_cast<RasterMesh*>(scratch + m_off);
    RasterFrame* dframe = reinterpret_cast<RasterFrame*>(scratch + f_off);
    unsigned int* n_large = reinterpret_cast<unsigned int*>(scratch + c_off);
    uint4* large = reinterpret_cast<uint4*>(scratch + l_off);
    // meshes and frames in one copy, counters zeroed behind them; pageable source: the copy has been staged when
    // cudaMemcpyAsync returns
    std::vector<unsigned char> h(c_off + c_bytes - m_off, 0);
    memcpy(h.data(), meshes, m_bytes);
    memcpy(h.data() + (f_off - m_off), frames, f_bytes);
    if ((e = cudaMemcpyAsync(dmesh, h.data(), h.size(), cudaMemcpyHostToDevice, st)) == cudaSuccess) {
        z_init<<<dim3((unsigned)((npx + 255) / 256), n_views), 256, 0, st>>>(dframe, zbuf, npx);
        raster<<<(unsigned)((total_prims + 127) / 128), 128, 0, st>>>(dmesh, n, total_prims, dframe, zbuf, large,
                                                                      n_large);
        raster_big<<<dim3((W + kTile - 1) / kTile, (H + kTile - 1) / kTile, n_views), 256, 0, st>>>(
            dmesh, n, dframe, zbuf, large, n_large);
        resolve<<<dim3((W + 31) / 32, (H + 3) / 4, n_views), 128, 0, st>>>(dmesh, n, dframe, zbuf);
        e = cudaGetLastError();
    }
    const cudaError_t e2 = cudaFreeAsync(scratch, st);
    return e != cudaSuccess ? e : e2;
}

}  // namespace vrb
