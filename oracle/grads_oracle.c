/*
 * grads_oracle.c -- CPU restatement of the leaf-gradient pass (vr_tree_leaf_grads): the gradient of a loss on the
 * offscreen float render w.r.t. every leaf's data row, given dL/d(r, g, b, alpha) of each pixel.
 *
 * TEST INFRASTRUCTURE ONLY, built into oracle/libgrads_oracle.so.  It is the march oracle (march_oracle.c, included
 * unchanged, as weights_oracle.c does) plus one exported function.  The samples, the σ test and the early stop are
 * those of orc_render's trace_ray (include/volrend/cuda/rt_core.cuh:66-196, paths relative to the reference's root),
 * evaluated in float exactly as there; the gradient terms are evaluated in double from the float sample values
 * (Δt, δs, σ, the basis values and the pre-sigmoid channel sums), with double exp.  Per shaded sample i, with
 * Δδ = Δt δs, att = exp(-Δδ σ), w_i = T_i (1 - att), col = sigmoid(x) (RGBA: the raw coefficient), S_c = Σ w col,
 * T the final transmittance, s = 1, K_c = background, dα/dσ = Δδ T when the ray runs to tmax and s = 1 / (1 - T),
 * K_c = pixel colour, dα/dσ = 0 when it stops early:
 *   coefficient k of channel c   g_c s w_i col (1 - col) B_k      (RGBA channel c: g_c s w_i)
 *   σ                            Σ_c g_c s Δδ (T_{i+1} col - (S_c - S_{≤i,c}) - K_c T) + g_α dα/dσ
 * Besides the gradient it returns, per element, A = the sum of the absolute values of the terms added into it (the σ
 * term split into its parts T_{i+1} col, S_c, S_{≤i,c}, K_c T and the alpha part), the scale the GPU's float sums are
 * compared at.
 */
#include "march_oracle.c"

/* Coefficients per channel the device keeps: a basis size with its own kernel keeps all, any other only the first. */
static int kept_coefs(int bd) { return (bd == 4 || bd == 9 || bd == 16 || bd == 25) ? bd : 1; }

typedef struct {
    int64_t slot;
    double dd, tn, w;      /* Δδ, T_{i+1}, w_i */
    double col[3], dcol[3], pre[3];   /* colour, col (1 - col), S_{≤i} */
} gsample;

/* trace_ray of one pixel with the gradient: adds g's terms into grad / A (capacity * 8 * data_dim doubles).  `rgba`
 * receives the float pixel of orc_render. */
static void trace_grads(const orc_tree* tree, float* dir, const float* vdir, const float* cen, const orc_options* opt,
                        const float* g, double* grad, double* A, float* rgba) {
    dir[0] = tree->scale[0] * dir[0];                                 /* _get_delta_scale :52-63 */
    dir[1] = tree->scale[1] * dir[1];
    dir[2] = tree->scale[2] * dir[2];
    const float delta_scale = 1.f / norm3(dir);
    {
        float x = dir[0] * delta_scale, y = delta_scale * dir[1], z = delta_scale * dir[2];
        dir[0] = x; dir[1] = y; dir[2] = z;
    }
    const float tmax_bg = 1e9f / delta_scale;
    float invdir[3];
    for (int i = 0; i < 3; ++i) invdir[i] = (float)(1.0 / ((double)dir[i] + 1e-9)); /* :83 [f64] */
    float tmin = 0.f, tmax = 1e4f;                                    /* _dda_world :18-34 [f64] */
    for (int i = 0; i < 3; ++i) {
        float t1 = (float)((((double)opt->render_bbox[i] + 1e-6) - (double)cen[i]) * (double)invdir[i]);
        float t2 = (float)((((double)opt->render_bbox[i + 3] - 1e-6) - (double)cen[i]) * (double)invdir[i]);
        tmin = fmaxf(tmin, fminf(t1, t2));
        tmax = fminf(tmax, fmaxf(t1, t2));
    }
    tmax = fminf(tmax, tmax_bg);
    const double bg = opt->background_brightness;
    if (tmax < 0.f || tmin > tmax) {                                  /* :88-92 */
        rgba[0] = rgba[1] = rgba[2] = (float)bg; rgba[3] = 0.f;
        return;
    }
    float basis_fn[ORC_BASIS_MAX];
    memset(basis_fn, 0, sizeof(basis_fn));
    precalc_basis(tree, vdir, basis_fn);
    for (int i = 0; i < opt->basis_minmax[0] && i < ORC_BASIS_MAX; ++i) basis_fn[i] = 0.f;  /* :98-100 */
    for (int i = opt->basis_minmax[1] + 1; i < ORC_BASIS_MAX; ++i)                           /* :101-103 */
        if (i >= 0) basis_fn[i] = 0.f;

    const float fN = (float)tree->N;
    const int64_t N3 = (int64_t)tree->N * tree->N * tree->N;
    const int bd = tree->basis_dim, dd = tree->data_dim;
    gsample* smp = NULL;
    size_t n_smp = 0, cap_smp = 0;
    float light = 1.f, out[3] = {0.f, 0.f, 0.f};
    double T = 1.0, S[3] = {0.0, 0.0, 0.0};
    int stopped = 0;
    float t = tmin;
    while (t < tmax) {                                                /* :108 */
        float pos[3];
        for (int i = 0; i < 3; ++i) pos[i] = fmaf(t, dir[i], cen[i]); /* :109-111 */
        for (int i = 0; i < 3; ++i) pos[i] = fmaxf(fminf(pos[i], 1.f - 1e-6f), 0.f);
        int64_t ptr = 0, sub_ptr;
        float cube_sz = fN;
        for (;;) {                                                    /* n3tree_query.hpp:16-47 */
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
            cube_sz = cube_sz * fN;
            ptr += skip * N3;
        }
        const uint16_t* leaf = tree->data + sub_ptr * dd;
        float tsub = 1e4f;                                            /* _dda_unit :37-49 */
        for (int i = 0; i < 3; ++i) {
            float t1 = invdir[i] * -pos[i];
            float t2 = invdir[i] + t1;
            tsub = fminf(tsub, fmaxf(t1, t2));
        }
        const float delta_t = tsub / cube_sz + opt->step_size;        /* :116-117 */
        const float sigma = h2f(leaf[dd - 1]);
        if (sigma > opt->sigma_thresh) {                              /* :118 */
            const float att = expf(((-delta_t) * delta_scale) * sigma);   /* :119 */
            const float weight = light * (1.f - att);                 /* :120 */
            if (n_smp == cap_smp) {
                cap_smp = cap_smp ? 2 * cap_smp : 64;
                smp = (gsample*)realloc(smp, cap_smp * sizeof(gsample));
            }
            gsample* q = &smp[n_smp++];
            q->slot = sub_ptr;
            q->dd = (double)delta_t * (double)delta_scale;
            const double datt = exp(-q->dd * (double)sigma);
            q->w = T * (1.0 - datt);
            T *= datt;
            q->tn = T;
            for (int c = 0; c < 3; ++c) {
                if (bd >= 0) {                                        /* :125-165 */
                    const uint16_t* k = leaf + c * bd;
                    float tmp = basis_fn[0] * h2f(k[0]);
                    if (bd == 25) tmp = tmp + sh_group(basis_fn, k, 16, 24);
                    if (bd == 25 || bd == 16) tmp = tmp + sh_group(basis_fn, k, 9, 15);
                    if (bd == 25 || bd == 16 || bd == 9) tmp = tmp + sh_group(basis_fn, k, 4, 8);
                    if (bd == 25 || bd == 16 || bd == 9 || bd == 4) tmp = tmp + sh_group(basis_fn, k, 1, 3);
                    out[c] = out[c] + weight / (1.f + expf(-tmp));    /* :163 */
                    const double e = exp(-(double)tmp);
                    q->col[c] = 1.0 / (1.0 + e);
                    q->dcol[c] = q->col[c] * (1.0 / (1.0 + 1.0 / e));
                } else {
                    out[c] = fmaf(h2f(leaf[c]), weight, out[c]);     /* :167-171 */
                    q->col[c] = h2f(leaf[c]);
                    q->dcol[c] = 0.0;
                }
                S[c] += q->w * q->col[c];
                q->pre[c] = S[c];
            }
            light = light * att;                                      /* :174 */
            if (light < opt->stop_thresh) { stopped = 1; break; }     /* :176-185 */
        }
        t = t + delta_t;                                              /* :187 */
    }
    /* the float pixel of orc_render (render_pixel's offscreen composite) */
    float alpha = 1.f - light;
    if (stopped) {
        const float scale = 1.f / (1.f - light);
        out[0] *= scale; out[1] *= scale; out[2] *= scale;
        alpha = 1.f;
    }
    const float remain = (1.f - alpha) * opt->background_brightness;
    for (int c = 0; c < 3; ++c) rgba[c] = remain + out[c];
    rgba[3] = alpha;

    const double s = stopped ? 1.0 / (1.0 - T) : 1.0;
    double K[3];
    for (int c = 0; c < 3; ++c) K[c] = stopped ? S[c] * s : bg;
    const int nk = kept_coefs(bd);
    for (size_t i = 0; i < n_smp; ++i) {
        const gsample* q = &smp[i];
        double* gr = grad + q->slot * dd;
        double* ar = A + q->slot * dd;
        double gsig = 0.0, asig = 0.0;
        for (int c = 0; c < 3; ++c) {
            const double gs = (double)g[c] * s;
            const double parts[4] = {gs * q->dd * q->tn * q->col[c], -gs * q->dd * S[c], gs * q->dd * q->pre[c],
                                     -gs * q->dd * K[c] * T};
            for (int j = 0; j < 4; ++j) { gsig += parts[j]; asig += fabs(parts[j]); }
            if (bd < 0) {
                gr[c] += gs * q->w;
                ar[c] += fabs(gs * q->w);
            } else {
                for (int k = 0; k < nk; ++k) {
                    const double v = gs * q->w * q->dcol[c] * (double)basis_fn[k];
                    gr[c * bd + k] += v;
                    ar[c * bd + k] += fabs(v);
                }
            }
        }
        if (!stopped) {
            const double v = (double)g[3] * q->dd * T;
            gsig += v;
            asig += fabs(v);
        }
        gr[dd - 1] += gsig;
        ar[dd - 1] += asig;
    }
    free(smp);
}

typedef struct {
    const orc_tree* tree; const orc_camera* cam; const orc_options* opt;
    int x0, y0, w, h;
    const float* dpix;
    double *grad, *A;      /* this thread's sums */
    float* rgba;
    volatile int* next_row;
} gjob_t;

static void* grads_worker(void* arg) {
    gjob_t* j = (gjob_t*)arg;
    for (;;) {
        int r = __sync_fetch_and_add(j->next_row, 1);
        if (r >= j->h) break;
        for (int c = 0; c < j->w; ++c) {
            const size_t o = (size_t)r * j->w + c;
            float px[4] = {j->opt->background_brightness, j->opt->background_brightness,
                           j->opt->background_brightness, 0.f};
            if (j->tree->N > 0) {                                     /* render_pixel, volrend.cu:136-150 */
                float dir[3], cen[3];
                screen2worlddir(j->x0 + c, j->y0 + r, j->cam, dir, cen);
                float vdir[3] = {dir[0], dir[1], dir[2]};
                maybe_world2ndc(j->tree, dir, cen);
                for (int i = 0; i < 3; ++i) cen[i] = fmaf(j->tree->scale[i], cen[i], j->tree->offset[i]);
                rodrigues(j->opt->rot_dirs, vdir);
                trace_grads(j->tree, dir, vdir, cen, j->opt, j->dpix + 4 * o, j->grad, j->A, px);
            }
            if (j->rgba) memcpy(j->rgba + 4 * o, px, 16);
        }
    }
    return NULL;
}

/* Adds the gradient of the tile [x0,x0+w) x [y0,y0+h) of one view into grad and the absolute terms into A (both
 * capacity * N^3 * data_dim doubles, initialised by the caller).  dpix: tile-sized float4 dL/d(r, g, b, alpha);
 * rgba: tile-sized float4 or NULL, receives orc_render's float output.  render_depth is refused (-1).  Each thread
 * keeps its own sums, added at the end.  Returns 0 on success. */
int orc_leaf_grads(const orc_tree* tree, const orc_camera* cam, const orc_options* opt, int x0, int y0, int w, int h,
                   const float* dpix, double* grad, double* A, float* rgba, int nthreads) {
    if (!tree || !cam || !opt || !dpix || !grad || !A || w < 0 || h < 0 || opt->render_depth) return -1;
    if (tree->N != 0 && tree->N != 2) return -2;
    pthread_once(&g_h2f_once, init_h2f);
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 64) nthreads = 64;
    if (nthreads > h && h > 0) nthreads = h;
    const size_t n = (size_t)tree->capacity * 8 * (size_t)(tree->data_dim > 0 ? tree->data_dim : 1);
    volatile int next_row = 0;
    gjob_t* jobs = (gjob_t*)calloc((size_t)nthreads, sizeof(gjob_t));
    pthread_t* th = (pthread_t*)calloc((size_t)nthreads, sizeof(pthread_t));
    double* local = (double*)calloc(2 * n * (size_t)nthreads + 1, sizeof(double));
    if (!jobs || !th || !local) { free(jobs); free(th); free(local); return -3; }
    for (int i = 0; i < nthreads; ++i) {
        gjob_t* j = &jobs[i];
        j->tree = tree; j->cam = cam; j->opt = opt;
        j->x0 = x0; j->y0 = y0; j->w = w; j->h = h;
        j->dpix = dpix; j->rgba = rgba;
        j->grad = local + 2 * n * (size_t)i;
        j->A = j->grad + n;
        j->next_row = &next_row;
        if (i > 0) pthread_create(&th[i], NULL, grads_worker, j);
    }
    grads_worker(&jobs[0]);
    for (int i = 1; i < nthreads; ++i) pthread_join(th[i], NULL);
    for (int i = 0; i < nthreads; ++i)
        for (size_t k = 0; k < n; ++k) {
            grad[k] += jobs[i].grad[k];
            A[k] += jobs[i].A[k];
        }
    free(jobs); free(th); free(local);
    return 0;
}
