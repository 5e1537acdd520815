/*
 * weights_oracle.c -- CPU restatement of the leaf-weights pass (vr_tree_leaf_weights): per leaf slot, the maximum
 * compositing weight T * (1 - att) of the samples that shade it.
 *
 * TEST INFRASTRUCTURE ONLY, built into oracle/libweights_oracle.so.  It is the march oracle (march_oracle.c, included
 * unchanged so that the ray set-up, the descent and the cell exit are the same code) plus one exported function.  The
 * samples are those of orc_render's trace_ray (include/volrend/cuda/rt_core.cuh:66-196, paths relative to the
 * reference's root); where trace_ray adds the sample's colour this records its weight at the leaf's slot, the offset
 * of query_single_from_root's leaf pointer from the data array divided by data_dim.  The weights differ from the GPU's
 * only through expf ulps (glibc vs libdevice), as the colours of march_oracle.c do; which slots are shaded is exact.
 */
#include <float.h>

#include "march_oracle.c"

/* The order of the weights pass: floats with -0 < +0 (no NaN is ever compared). */
static inline uint32_t weight_key(float w) {
    uint32_t b;
    memcpy(&b, &w, 4);
    return (b & 0x80000000u) ? ~b : b | 0x80000000u;
}
static inline void max_into(float* dst, float w) {
    if (w != w) return;                                               /* NaN weights are not recorded */
    if (weight_key(w) > weight_key(*dst)) *dst = w;
}

/* trace_ray without colour: returns the ray's alpha (out[3] of trace_ray with render_depth off). */
static float trace_weights(const orc_tree* tree, float* dir, const float* cen, const orc_options* opt, float* weights,
                           orc_counters* cnt) {
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
    if (tmax < 0.f || tmin > tmax) return 0.f;                        /* :88-92 */
    if (cnt) cnt->rays_hit += 1;

    const float fN = (float)tree->N;
    const int64_t N3 = (int64_t)tree->N * tree->N * tree->N;
    float light = 1.f;
    float t = tmin;
    while (t < tmax) {                                                /* :108 */
        float pos[3];
        for (int i = 0; i < 3; ++i) pos[i] = fmaf(t, dir[i], cen[i]); /* :109-111 */
        for (int i = 0; i < 3; ++i) pos[i] = fmaxf(fminf(pos[i], 1.f - 1e-6f), 0.f);
        int64_t ptr = 0, sub_ptr;
        float cube_sz = fN;
        uint64_t depth = 0;
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
            ++depth;
            if (skip == 0) break;
            cube_sz = cube_sz * fN;
            ptr += skip * N3;
        }
        const uint16_t* leaf = tree->data + sub_ptr * tree->data_dim;
        if (cnt) { cnt->samples += 1; cnt->child_loads += depth; }
        float tsub = 1e4f;                                            /* _dda_unit :37-49 */
        for (int i = 0; i < 3; ++i) {
            float t1 = invdir[i] * -pos[i];
            float t2 = invdir[i] + t1;
            tsub = fminf(tsub, fmaxf(t1, t2));
        }
        const float delta_t = tsub / cube_sz + opt->step_size;        /* :116-117 */
        const float sigma = h2f(leaf[tree->data_dim - 1]);
        if (sigma > opt->sigma_thresh) {                              /* :118 */
            const float att = expf(((-delta_t) * delta_scale) * sigma);   /* :119 */
            const float weight = light * (1.f - att);                 /* :120 */
            if (cnt) cnt->shaded += 1;
            max_into(weights + (leaf - tree->data) / tree->data_dim, weight);
            light = light * att;                                      /* :174 */
            if (light < opt->stop_thresh) return 1.f;                 /* :176-185 */
        }
        t = t + delta_t;                                              /* :187 */
    }
    return 1.f - light;
}

typedef struct {
    const orc_tree* tree; const orc_camera* cam; const orc_options* opt;
    int x0, y0, w, h;
    float* weights;    /* this thread's capacity * 8 maxima */
    float* alpha;
    orc_counters cnt; int want_cnt;
    volatile int* next_row;
} wjob_t;

static void* weights_worker(void* arg) {
    wjob_t* j = (wjob_t*)arg;
    for (;;) {
        int r = __sync_fetch_and_add(j->next_row, 1);
        if (r >= j->h) break;
        for (int c = 0; c < j->w; ++c) {
            float a = 0.f;
            if (j->tree->N > 0) {                                     /* render_pixel, volrend.cu:136-150 */
                float dir[3], cen[3];
                screen2worlddir(j->x0 + c, j->y0 + r, j->cam, dir, cen);
                maybe_world2ndc(j->tree, dir, cen);
                for (int i = 0; i < 3; ++i) cen[i] = fmaf(j->tree->scale[i], cen[i], j->tree->offset[i]);
                a = trace_weights(j->tree, dir, cen, j->opt, j->weights, j->want_cnt ? &j->cnt : NULL);
            }
            if (j->alpha) j->alpha[(size_t)r * j->w + c] = a;
        }
    }
    return NULL;
}

/* Raises weights[slot] (capacity * N^3 floats, initialised by the caller) to the maximum weight of the samples of the
 * tile [x0,x0+w) x [y0,y0+h) of one view; alpha: tile-sized floats or NULL; counters as orc_render (set, not added).
 * Each thread keeps its own maxima, reduced at the end, so the result does not depend on the thread count.
 * Returns 0 on success. */
int orc_leaf_weights(const orc_tree* tree, const orc_camera* cam, const orc_options* opt, int x0, int y0, int w, int h,
                     float* weights, float* alpha, orc_counters* counters, int nthreads) {
    if (!tree || !cam || !opt || !weights || w < 0 || h < 0) return -1;
    if (tree->N != 0 && tree->N != 2) return -2;
    pthread_once(&g_h2f_once, init_h2f);
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 256) nthreads = 256;
    if (nthreads > h && h > 0) nthreads = h;
    const size_t n_slots = (size_t)tree->capacity * 8;
    volatile int next_row = 0;
    wjob_t* jobs = (wjob_t*)calloc((size_t)nthreads, sizeof(wjob_t));
    pthread_t* th = (pthread_t*)calloc((size_t)nthreads, sizeof(pthread_t));
    float* local = (float*)malloc(sizeof(float) * n_slots * (size_t)nthreads + 1);
    if (!jobs || !th || !local) { free(jobs); free(th); free(local); return -3; }
    for (size_t i = 0; i < n_slots * (size_t)nthreads; ++i) local[i] = -INFINITY;
    for (int i = 0; i < nthreads; ++i) {
        wjob_t* j = &jobs[i];
        j->tree = tree; j->cam = cam; j->opt = opt;
        j->x0 = x0; j->y0 = y0; j->w = w; j->h = h;
        j->weights = local + n_slots * (size_t)i;
        j->alpha = alpha;
        j->want_cnt = counters != NULL; j->next_row = &next_row;
        if (i > 0) pthread_create(&th[i], NULL, weights_worker, j);
    }
    weights_worker(&jobs[0]);
    for (int i = 1; i < nthreads; ++i) pthread_join(th[i], NULL);
    for (int i = 0; i < nthreads; ++i)
        for (size_t s = 0; s < n_slots; ++s) max_into(weights + s, local[n_slots * (size_t)i + s]);
    if (counters) {
        memset(counters, 0, sizeof(*counters));
        for (int i = 0; i < nthreads; ++i) {
            counters->samples += jobs[i].cnt.samples;
            counters->child_loads += jobs[i].cnt.child_loads;
            counters->shaded += jobs[i].cnt.shaded;
            counters->rays_hit += jobs[i].cnt.rays_hit;
        }
    }
    free(jobs); free(th); free(local);
    return 0;
}
