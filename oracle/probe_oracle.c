/*
 * probe_oracle.c -- CPU restatement of the lumisphere probe disc (enable_probe) of the reference's render_kernel.
 *
 * TEST INFRASTRUCTURE ONLY, built into oracle/libprobe_oracle.so.  It is the march oracle (march_oracle.c, included
 * unchanged so that its tree, basis and quantisation helpers are the same code) plus one exported function that
 * applies the disc to a frame the oracle marched.  Paths are relative to the reference's root.
 *
 * The disc code is src/cuda/volrend.cu:100-134; the operations follow the SASS nvcc 12.9 emits for it (sm_90, -O3):
 *   h = float(S) * 0.5;  a = xx / h - 1;  b = yy / h - 1;  c = fma(a, a, b * b)          (cen[0] = -a, cen[1] = b)
 *   c <= 1:  s = sqrt(1 - c);  dir[i] = fma(-m[6+i], s, fma(b, m[3+i], -(a * m[i])))      (_mv3, cen[2] = -s)
 *   tmp = fma(coeff[i], basis[i], tmp) over basis_minmax;  out = 1 / (1 + expf(-tmp))
 * with the integer candidate test in wrapping 32-bit adds.  The colour differs from the GPU only through expf ulps
 * (glibc vs libdevice), as in march_oracle.c.
 */
#include "march_oracle.c"

/* include/volrend/internal/n3tree_query.hpp:13-48 from the root: the data of the leaf holding tree point p. */
static const uint16_t* probe_leaf(const orc_tree* tree, const float* p_in) {
    const float fN = (float)tree->N;
    const int64_t N3 = (int64_t)tree->N * tree->N * tree->N;
    float pos[3];
    for (int i = 0; i < 3; ++i) pos[i] = fmaxf(fminf(p_in[i], 1.f - 1e-6f), 0.f);
    int64_t ptr = 0, sub_ptr;
    for (;;) {
        float index = 0.f;
        for (int i = 0; i < 3; ++i) {
            pos[i] = pos[i] * fN;
            const float k = floorf(pos[i]);
            index = fmaf(index, fN, k);
            pos[i] = pos[i] - k;
        }
        sub_ptr = ptr + (int32_t)index;
        const int64_t skip = tree->child[sub_ptr];
        if (skip == 0) break;
        ptr += skip * N3;
    }
    return tree->data + sub_ptr * tree->data_dim;
}

/* maybe_precalc_basis (lumisphere.hpp:9-87) as the disc's instance in render_kernel computes it: the march
 * oracle's basis, except that this instance fuses -y*y into 4zz - xx - yy (SH B[11], B[13]) and the ASG exponent
 * into fma(-dx, dx*a, -(dy*(dy*b))). */
static void disc_basis(const orc_tree* tree, const float* dir, float* out) {
    const int bd = tree->basis_dim;
    precalc_basis(tree, dir, out);
    const float x = dir[0], y = dir[1], z = dir[2];
    if (tree->format == ORC_FMT_SH && bd >= 16) {
        const float z4 = fmaf(-y, y, fmaf(z * z, 4.f, -(x * x)));
        out[11] = (float)(((double)y * -0.4570457994644658) * (double)z4);
        out[13] = (float)((double)z4 * ((double)x * -0.4570457994644658));
    } else if (tree->format == ORC_FMT_ASG) {
        const float* p = tree->extra;
        for (int i = 0; i < bd; ++i) {
            const float S = dot3(dir, p + 8), dx = dot3(dir, p + 2), dy = dot3(dir, p + 5);
            out[i] = S * expf(fmaf(-dx, dx * p[0], -(dy * (dy * p[1])))) / (float)bd;
            p += 11;
        }
    }
}

/* Applies the probe disc of world point probe[3] (disp = probe_disp_size) to the tile [x0,x0+w) x [y0,y0+h) of a
 * frame: where a pixel lies in the disc, rgba_f32 / rgba8 (tile-sized, either may be NULL) receive the disc colour
 * and mask (tile-sized bytes, or NULL) receives 1; other pixels are left as they are (mask 0).  The basis range is
 * basis_minmax clamped to [0, basis_dim - 1].  Returns 0, or -1 for bad arguments. */
int orc_probe_overlay(const orc_tree* tree, const orc_camera* cam, const orc_options* opt, const float* probe,
                      int disp, int x0, int y0, int w, int h, float* rgba_f32, uint8_t* rgba8, uint8_t* mask) {
    if (!tree || !cam || !opt || !probe || w < 0 || h < 0 || tree->N != 2) return -1;
    pthread_once(&g_h2f_once, init_h2f);
    if (mask) memset(mask, 0, (size_t)w * h);
    float pt[3], coef[3 * ORC_BASIS_MAX];
    for (int i = 0; i < 3; ++i) pt[i] = fmaf(tree->scale[i], probe[i], tree->offset[i]);   /* volrend.cu:180-182 */
    const uint16_t* leaf = probe_leaf(tree, pt);
    const int n_coef = tree->basis_dim < 0 ? 3 : 3 * tree->basis_dim;
    for (int i = 0; i < n_coef && i < tree->data_dim - 1; ++i) coef[i] = h2f(leaf[i]);          /* :188-190 */
    const int bd = tree->basis_dim;
    const int lo = opt->basis_minmax[0] > 0 ? opt->basis_minmax[0] : 0;
    const int hi = opt->basis_minmax[1] < bd - 1 ? opt->basis_minmax[1] : bd - 1;
    const int W = cam->width;
    const int32_t y_end = (int32_t)((uint32_t)disp + 5u), x_beg = (int32_t)((uint32_t)W - (uint32_t)disp - 5u);
    for (int r = 0; r < h; ++r) {
        for (int cc = 0; cc < w; ++cc) {
            const int x = x0 + cc, y = y0 + r;
            if (!(y < y_end && x >= x_beg)) continue;                                             /* :100-101 */
            const int32_t xx = (int32_t)((uint32_t)x + 5u - (uint32_t)W + (uint32_t)disp), yy = y - 5;
            const float hs = (float)disp * 0.5f;
            const float a = (float)xx / hs - 1.f, b = (float)yy / hs - 1.f;                       /* :104-107 */
            const float c = fmaf(a, a, b * b);                                                    /* :109 */
            if (!(c <= 1.f)) continue;                                                            /* :110 */
            float out[3];
            if (bd >= 0) {
                const float s = sqrtf(1.f - c);                                                   /* :113 */
                const float* m = cam->c2w;
                float dir[3], B[ORC_BASIS_MAX];
                for (int k = 0; k < 3; ++k) dir[k] = fmaf(-m[6 + k], s, fmaf(b, m[3 + k], -(a * m[k])));   /* :114 */
                memset(B, 0, sizeof(B));
                disc_basis(tree, dir, B);                                                         /* :116 */
                for (int t = 0; t < 3; ++t) {                                                     /* :117-124 */
                    float tmp = 0.f;
                    for (int i = lo; i <= hi; ++i) tmp = fmaf(coef[t * bd + i], B[i], tmp);
                    out[t] = 1.f / (1.f + expf(-tmp));
                }
            } else {
                for (int t = 0; t < 3; ++t) out[t] = coef[t];                                     /* :127-128 */
            }
            const size_t o = (size_t)r * w + cc;
            if (mask) mask[o] = 1;
            for (int t = 0; t < 3; ++t) out[t] = out[t] + 0.f;                                    /* :153-163, alpha 1 */
            if (rgba_f32) {
                float* f = rgba_f32 + 4 * o;
                f[0] = out[0]; f[1] = out[1]; f[2] = out[2]; f[3] = 1.f;
            }
            if (rgba8) {                                                                          /* :166 */
                uint8_t* u = rgba8 + 4 * o;
                u[0] = quant8(out[0]); u[1] = quant8(out[1]); u[2] = quant8(out[2]); u[3] = 255;
            }
        }
    }
    return 0;
}
