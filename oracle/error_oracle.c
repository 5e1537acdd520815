/*
 * error_oracle.c -- CPU restatement of the leaf-error pass (vr_tree_leaf_error): per leaf slot, the sum over the
 * samples that shade it of their compositing weight T * (1 - att) times their pixel's error.
 *
 * TEST INFRASTRUCTURE ONLY, built into oracle/liberror_oracle.so.  It is the march oracle (march_oracle.c, included
 * unchanged so that the ray set-up, the descent and the cell exit are the same code) plus one exported function.  The
 * samples are those of orc_render's trace_ray (include/volrend/cuda/rt_core.cuh:66-196, paths relative to the
 * reference's root) and of weights_oracle.c; where trace_ray adds the sample's colour this adds weight * err, in
 * double, at the leaf's slot (the offset of query_single_from_root's leaf pointer from the data array divided by
 * data_dim).  It also returns, per slot, the sum of the absolute terms and the number of terms, so that tests can
 * state a tolerance for the GPU's float atomics and compare the set of slots that received terms exactly.
 */
#include "march_oracle.c"

/* trace_ray without colour, adding weight * err to score[slot], |weight * err| to absum[slot], 1 to hits[slot]. */
static void trace_error(const orc_tree* tree, float* dir, const float* cen, const orc_options* opt, float err,
                        double* score, double* absum, uint32_t* hits, orc_counters* cnt) {
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
    if (tmax < 0.f || tmin > tmax) return;                            /* :88-92 */
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
            const size_t slot = (size_t)((leaf - tree->data) / tree->data_dim);
            const double term = (double)weight * (double)err;
            score[slot] += term;
            absum[slot] += fabs(term);
            hits[slot] += 1;
            light = light * att;                                      /* :174 */
            if (light < opt->stop_thresh) return;                     /* :176-185 */
        }
        t = t + delta_t;                                              /* :187 */
    }
}

typedef struct {
    const orc_tree* tree; const orc_camera* cam; const orc_options* opt;
    int x0, y0, w, h;
    const float* err;
    double* score; double* absum; uint32_t* hits;   /* this thread's capacity * 8 sums */
    orc_counters cnt; int want_cnt;
    volatile int* next_row;
} ejob_t;

static void* error_worker(void* arg) {
    ejob_t* j = (ejob_t*)arg;
    for (;;) {
        int r = __sync_fetch_and_add(j->next_row, 1);
        if (r >= j->h) break;
        for (int c = 0; c < j->w; ++c) {
            if (j->tree->N == 0) continue;                            /* render_pixel, volrend.cu:136-150 */
            float dir[3], cen[3];
            screen2worlddir(j->x0 + c, j->y0 + r, j->cam, dir, cen);
            maybe_world2ndc(j->tree, dir, cen);
            for (int i = 0; i < 3; ++i) cen[i] = fmaf(j->tree->scale[i], cen[i], j->tree->offset[i]);
            trace_error(j->tree, dir, cen, j->opt, j->err[(size_t)r * j->w + c], j->score, j->absum, j->hits,
                        j->want_cnt ? &j->cnt : NULL);
        }
    }
    return NULL;
}

/* Adds, for every shaded sample of the tile [x0,x0+w) x [y0,y0+h) of one view, weight * err[pixel] to score[slot],
 * |weight * err[pixel]| to absum[slot] and 1 to hits[slot] (capacity * N^3 each, initialised by the caller; absum and
 * hits may be NULL).  err: tile-sized floats.  Counters as orc_render (set, not added).  Each thread keeps its own
 * sums, added up at the end in thread order, so the result depends on the thread count only through the rounding of
 * the double sums.  Returns 0 on success. */
int orc_leaf_error(const orc_tree* tree, const orc_camera* cam, const orc_options* opt, int x0, int y0, int w, int h,
                   const float* err, double* score, double* absum, uint32_t* hits, orc_counters* counters,
                   int nthreads) {
    if (!tree || !cam || !opt || !err || !score || w < 0 || h < 0) return -1;
    if (tree->N != 0 && tree->N != 2) return -2;
    pthread_once(&g_h2f_once, init_h2f);
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 256) nthreads = 256;
    if (nthreads > h && h > 0) nthreads = h;
    const size_t n_slots = (size_t)tree->capacity * 8, n_all = n_slots * (size_t)nthreads;
    volatile int next_row = 0;
    ejob_t* jobs = (ejob_t*)calloc((size_t)nthreads, sizeof(ejob_t));
    pthread_t* th = (pthread_t*)calloc((size_t)nthreads, sizeof(pthread_t));
    double* ls = (double*)calloc(n_all + 1, sizeof(double));
    double* la = (double*)calloc(n_all + 1, sizeof(double));
    uint32_t* lh = (uint32_t*)calloc(n_all + 1, sizeof(uint32_t));
    if (!jobs || !th || !ls || !la || !lh) { free(jobs); free(th); free(ls); free(la); free(lh); return -3; }
    for (int i = 0; i < nthreads; ++i) {
        ejob_t* j = &jobs[i];
        j->tree = tree; j->cam = cam; j->opt = opt;
        j->x0 = x0; j->y0 = y0; j->w = w; j->h = h;
        j->err = err;
        j->score = ls + n_slots * (size_t)i; j->absum = la + n_slots * (size_t)i; j->hits = lh + n_slots * (size_t)i;
        j->want_cnt = counters != NULL; j->next_row = &next_row;
        if (i > 0) pthread_create(&th[i], NULL, error_worker, j);
    }
    error_worker(&jobs[0]);
    for (int i = 1; i < nthreads; ++i) pthread_join(th[i], NULL);
    for (int i = 0; i < nthreads; ++i)
        for (size_t s = 0; s < n_slots; ++s) {
            score[s] += ls[n_slots * (size_t)i + s];
            if (absum) absum[s] += la[n_slots * (size_t)i + s];
            if (hits) hits[s] += lh[n_slots * (size_t)i + s];
        }
    if (counters) {
        memset(counters, 0, sizeof(*counters));
        for (int i = 0; i < nthreads; ++i) {
            counters->samples += jobs[i].cnt.samples;
            counters->child_loads += jobs[i].cnt.child_loads;
            counters->shaded += jobs[i].cnt.shaded;
            counters->rays_hit += jobs[i].cnt.rays_hit;
        }
    }
    free(jobs); free(th); free(ls); free(la); free(lh);
    return 0;
}
