/* lane_sim.c -- design tool (not product, not a test): replays the exact per-ray sample
 * sequence of a frame (oracle arithmetic) and counts WARP-level instruction issue under
 * different lane-scheduling policies, so that kernel restructurings can be ranked before
 * GPU time is spent on them.
 *
 *   P0  one 4x8 tile per warp pass, inline shading (the round-1 kernel)
 *   P1  P0 + warp-shared shading queue drained 32 items at a time
 *   P2  ray-granular refill from a per-warp pool of set-up rays (threshold = idle lanes) + P1 queue
 *   CULL=1  instead: the tile culling of batch launches (vr_cull.cu) -- tiles and warp instructions it culls, next
 *           to the bound of culling every tile where no ray shades, and a check that no tile with a shading ray
 *           is culled (exit code 1 if one is); THRESH=<sigma_thresh> overrides the default threshold
 *
 * Cost constants (warp instructions) come from the SASS of the round-1 kernel.
 * Usage: lane_sim <dump.bin> ; the dump is written by tools/lane_sim.py.
 */
#include "../oracle/march_oracle.c"

#include <stdio.h>

typedef struct {
    uint32_t off;   /* first sample in the trace */
    uint32_t n;     /* samples */
    uint32_t koff;  /* MEM mode: first key in g_keys */
    uint8_t hit;
} ray_t;

static double g_act_hist[33];
static const int g_p3_theta[6] = {4, 8, 12, 8, 8, 4}, g_p3_pat[6] = {1, 1, 1, 8, 16, 16};
static int g_b[32];   /* cumulative levels resolved after table k */
static uint8_t* g_trace;  /* per sample: fetches (low 4 bits) | shaded << 7 */
static size_t g_trace_n, g_trace_cap;
/* MEM mode: per sample its `fetches` table-word sector keys, then (if shaded) its record key; ray_t::off indexes both
   streams' first sample / key through g_koff */
static uint32_t* g_keys;
static size_t g_keys_n, g_keys_cap;
static int g_mem;

static void push(uint8_t v) {
    if (g_trace_n == g_trace_cap) {
        g_trace_cap = g_trace_cap ? g_trace_cap * 2 : (1u << 24);
        g_trace = (uint8_t*)realloc(g_trace, g_trace_cap);
    }
    g_trace[g_trace_n++] = v;
}

static void push_key(uint64_t k) {
    if (k >= (1ull << 32)) { fprintf(stderr, "key overflow\n"); exit(1); }
    if (g_keys_n == g_keys_cap) {
        g_keys_cap = g_keys_cap ? g_keys_cap * 2 : (1u << 24);
        g_keys = (uint32_t*)realloc(g_keys, g_keys_cap * 4);
    }
    g_keys[g_keys_n++] = (uint32_t)k;
}

/* the march of trace_ray() above without colours; records wide-table fetch counts */
static void trace_one(const orc_tree* tree, const orc_camera* cam, const orc_options* opt, int x, int y, ray_t* R) {
    float dir[3], cen[3];
    R->off = (uint32_t)g_trace_n; R->n = 0; R->hit = 0; R->koff = (uint32_t)g_keys_n;
    screen2worlddir(x, y, cam, dir, cen);
    maybe_world2ndc(tree, dir, cen);
    for (int i = 0; i < 3; ++i) cen[i] = fmaf(tree->scale[i], cen[i], tree->offset[i]);
    float ds;
    {
        for (int i = 0; i < 3; ++i) dir[i] = tree->scale[i] * dir[i];
        ds = 1.f / norm3(dir);
        float a = dir[0] * ds, b = ds * dir[1], c = ds * dir[2];
        dir[0] = a; dir[1] = b; dir[2] = c;
    }
    float invdir[3];
    for (int i = 0; i < 3; ++i) invdir[i] = (float)(1.0 / ((double)dir[i] + 1e-9));
    float tmin = 0.f, tmax = 1e4f;
    for (int i = 0; i < 3; ++i) {
        float t1 = (float)((((double)opt->render_bbox[i] + 1e-6) - (double)cen[i]) * (double)invdir[i]);
        float t2 = (float)((((double)opt->render_bbox[i + 3] - 1e-6) - (double)cen[i]) * (double)invdir[i]);
        tmin = fmaxf(tmin, fminf(t1, t2));
        tmax = fminf(tmax, fmaxf(t1, t2));
    }
    tmax = fminf(tmax, 1e9f / ds);
    if (tmax < 0.f || tmin > tmax) return;
    R->hit = 1;
    float light = 1.f, t = tmin;
    uint32_t pu[3] = {0, 0, 0};
    int pdepth = 1;
    while (t < tmax) {
        float pos[3];
        uint32_t u[3];
        for (int i = 0; i < 3; ++i) {
            pos[i] = fmaf(t, dir[i], cen[i]);
            pos[i] = fmaxf(fminf(pos[i], 1.f - 1e-6f), 0.f);
            u[i] = (uint32_t)(pos[i] * 16777216.f);
        }
        int64_t ptr = 0, sub;
        float cube = 2.f;
        int depth = 0;
        int64_t node_at[32];   /* node id at each depth of the path (its children start at child[8 * id]) */
        for (;;) {
            node_at[depth] = ptr >> 3;
            float index = 0.f;
            for (int i = 0; i < 3; ++i) {
                pos[i] = pos[i] * 2.f;
                const float k = floorf(pos[i]);
                index = fmaf(index, 2.f, k);
                pos[i] -= k;
            }
            sub = ptr + (int32_t)index;
            const int64_t skip = tree->child[sub];
            ++depth;
            if (!skip) break;
            cube *= 2.f;
            ptr += skip * 8;
        }
        /* wide-table fetches (vr_march.cuh find_leaf_wide) */
        const uint32_t diff = (u[0] ^ pu[0]) | (u[1] ^ pu[1]) | (u[2] ^ pu[2]);
        int common = diff ? (__builtin_clz(diff) - 8) : 24;
        /* table k covers the levels (g_b[k-1], g_b[k]] and hangs off a node of depth g_b[k-1] (LEVELS / PHASE env) */
        int shared = common < pdepth - 1 ? common : pdepth - 1;   /* deepest node depth shared and on the previous path */
        int j0 = 0, jl = 0;
        while (g_b[j0] <= shared) ++j0;        /* table j0 is rooted at depth g_b[j0-1] <= shared */
        while (g_b[jl] < depth) ++jl;
        int fetches = jl - j0 + 1;
        if (fetches < 1) fetches = 1;
        if (j0 > jl) j0 = jl;
        uint64_t entry = 0;
        for (int k = j0; g_mem && k <= jl; ++k) {
            /* table k hangs off the path's node of depth g_b[k-1] and is indexed by the x | y | z bits of its levels
               (vr_march.cuh find_leaf_wide); a table is 64 words = 8 sectors, so only the 32-byte sector matters */
            const int rd = k ? g_b[k - 1] : 0, lv = g_b[k] - rd, sh = 24 - g_b[k];
            const uint32_t m = (1u << lv) - 1;
            entry = (uint64_t)node_at[rd] * 64 + ((((u[0] >> sh) & m) << (2 * lv)) | (((u[1] >> sh) & m) << lv) | ((u[2] >> sh) & m));
            push_key(entry >> 3);
        }
        pu[0] = u[0]; pu[1] = u[1]; pu[2] = u[2]; pdepth = depth;
        float tsub = 1e4f;
        for (int i = 0; i < 3; ++i) {
            float t1 = invdir[i] * -pos[i];
            float t2 = invdir[i] + t1;
            tsub = fminf(tsub, fmaxf(t1, t2));
        }
        const float dt = tsub / cube + opt->step_size;
        const float sigma = h2f(tree->data[sub]);  /* data here = sigma only (data_dim 1) */
        int shaded = 0, stop = 0;
        if (sigma > opt->sigma_thresh) {
            shaded = 1;
            const float att = expf(((-dt) * ds) * sigma);
            light *= att;
            if (light < opt->stop_thresh) stop = 1;
        }
        push((uint8_t)(fetches | (shaded << 7)));
        if (g_mem && shaded) push_key(entry);   /* records are indexed by the leaf's table entry */
        R->n++;
        if (stop) break;
        t += dt;
    }
}

/* ---- cost model (warp instructions) */
/* C_BODY / C_FETCH / C_SHADE: SASS of the batch kernel march_persistent_kernel<16, .., 193> as tools/sass_blocks.py
   counts it (body 77, fetch 19, shade 202 before the funnel-shift table index; 72 / 14 / 199 after).  C_SETUP is
   an estimate, not a SASS count.  Each constant can be overridden from the environment (C_BODY=77 ...). */
static double C_SETUP = 330, C_OUT = 25, C_BODY = 72, C_FETCH = 14, C_SHADE = 199;
static double C_ENQ = 55, C_DRAIN = 250, C_ACC = 10, C_VOTE = 4, C_REFILL = 90, C_BATCH_EXTRA = 40, C_TILE = 30;

typedef struct { double instr, body_iters, body_lanes, shade_iters, shade_lanes, fetch_iters, fetch_lanes; } stats_t;

/* P0 / P1: tiles of 4x8 pixels */
static void sim_tiles(const ray_t* rays, int W, int H, int shared_queue, stats_t* S) {
    const int TW = 4, TH = 8;
    for (int ty = 0; ty < (H + TH - 1) / TH; ++ty)
        for (int tx = 0; tx < (W + TW - 1) / TW; ++tx) {
            const ray_t* lane[32];
            uint32_t pos[32];
            int alive = 0;
            for (int l = 0; l < 32; ++l) {
                int x = tx * TW + l % TW, y = ty * TH + l / TW;
                lane[l] = (x < W && y < H) ? &rays[(size_t)y * W + x] : NULL;
                pos[l] = 0;
                if (lane[l] && lane[l]->n) ++alive;
            }
            S->instr += C_TILE + C_SETUP + C_OUT;
            int q = 0;
            while (alive) {
                int act = 0, maxf = 0, nsh = 0;
                int fl[8] = {0};
                for (int l = 0; l < 32; ++l) {
                    if (!lane[l] || pos[l] >= lane[l]->n) continue;
                    uint8_t v = g_trace[lane[l]->off + pos[l]++];
                    int f = v & 15;
                    ++act;
                    if (f > maxf) maxf = f;
                    for (int k = 1; k < f && k < 8; ++k) fl[k]++;
                    if (v & 128) ++nsh;
                    if (pos[l] >= lane[l]->n) --alive;
                }
                S->instr += C_BODY + C_FETCH * (maxf - 1);
                S->body_iters += 1; S->body_lanes += act;
                if (!shared_queue) g_act_hist[act]++;
                for (int k = 1; k < maxf; ++k) { S->fetch_iters += 1; S->fetch_lanes += fl[k]; }
                if (nsh) {
                    if (!shared_queue) {
                        S->instr += C_SHADE; S->shade_iters += 1; S->shade_lanes += nsh;
                    } else {
                        S->instr += C_ENQ;
                        q += nsh;
                        if (q >= 32) { S->instr += C_DRAIN + 2 * C_ACC; S->shade_iters += 1; S->shade_lanes += 32; q -= 32; }
                    }
                }
            }
            if (shared_queue && q) { S->instr += C_DRAIN + 2 * C_ACC; S->shade_iters += 1; S->shade_lanes += q; }
        }
}

/* P2: per-warp pool of set-up rays, refill when idle lanes >= theta.  A warp handles `run`
 * consecutive tiles (stand-in for the dynamic global queue). */
static void sim_refill(const ray_t* rays, int W, int H, int theta, int run, int shared_queue, stats_t* S) {
    const int TW = 4, TH = 8;
    const int ntx = (W + TW - 1) / TW, nty = (H + TH - 1) / TH, ntiles = ntx * nty;
    for (int t0 = 0; t0 < ntiles; t0 += run) {
        int tnext = t0, tend = t0 + run < ntiles ? t0 + run : ntiles;
        const ray_t* pool[128];
        int npool = 0;
        const ray_t* lane[32] = {0};
        uint32_t pos[32] = {0};
        int alive = 0, q = 0;
        S->instr += C_TILE;
        for (;;) {
            int idle = 32 - alive;
            if (idle >= theta || alive == 0) {
                /* top the pool up with full-warp batch set-ups */
                while (npool < idle && tnext < tend) {
                    int tx = tnext % ntx, ty = tnext / ntx;
                    ++tnext;
                    S->instr += C_SETUP + C_BATCH_EXTRA + C_OUT;  /* misses are written here */
                    for (int l = 0; l < 32; ++l) {
                        int x = tx * TW + l % TW, y = ty * TH + l / TW;
                        if (x < W && y < H && rays[(size_t)y * W + x].n) pool[npool++] = &rays[(size_t)y * W + x];
                    }
                }
                if (npool == 0 && alive == 0) break;
                if (npool && idle) {
                    /* finished rays need their queued colours before they are written */
                    if (shared_queue && q) { S->instr += C_DRAIN + 2 * C_ACC; S->shade_iters += 1; S->shade_lanes += q; q = 0; }
                    S->instr += C_REFILL + C_OUT;
                    for (int l = 0; l < 32 && npool; ++l)
                        if (!lane[l] || pos[l] >= lane[l]->n) { lane[l] = pool[--npool]; pos[l] = 0; ++alive; }
                }
            }
            if (!alive) continue;
            int act = 0, maxf = 0, nsh = 0;
            int fl[8] = {0};
            for (int l = 0; l < 32; ++l) {
                if (!lane[l] || pos[l] >= lane[l]->n) continue;
                uint8_t v = g_trace[lane[l]->off + pos[l]++];
                int f = v & 15;
                ++act;
                if (f > maxf) maxf = f;
                for (int k = 1; k < f && k < 8; ++k) fl[k]++;
                if (v & 128) ++nsh;
                if (pos[l] >= lane[l]->n) --alive;
            }
            S->instr += C_BODY + C_VOTE + C_FETCH * (maxf - 1);
            S->body_iters += 1; S->body_lanes += act;
            for (int k = 1; k < maxf; ++k) { S->fetch_iters += 1; S->fetch_lanes += fl[k]; }
            if (nsh) {
                if (!shared_queue) { S->instr += C_SHADE; S->shade_iters += 1; S->shade_lanes += nsh; }
                else {
                    S->instr += C_ENQ;
                    q += nsh;
                    if (q >= 32) { S->instr += C_DRAIN + 2 * C_ACC; S->shade_iters += 1; S->shade_lanes += 32; q -= 32; }
                }
            }
        }
        if (shared_queue && q) { S->instr += C_DRAIN + 2 * C_ACC + C_OUT; S->shade_iters += 1; S->shade_lanes += q; }
    }
}

/* P3: P1 + tail parking.  When a tile has had <= theta rays alive for `patience` iterations, the warp flushes its
 * shading queue, parks the surviving rays in a pool and takes the next tile; whenever 32 rays are parked some warp
 * marches them as a dense pass (which may park its own tail again while the pool is not empty). */
static double C_PARK = 70, C_RESUME = 70;
static double g_park_events[16], g_park_rays[16], g_pool_passes[16];
static int g_p3_cur;
static void sim_park(const ray_t* rays, int W, int H, int theta, int patience, stats_t* S) {
    const int TW = 4, TH = 8;
    static const ray_t* pool[1 << 16];
    static uint32_t pool_pos[1 << 16];
    int npool = 0;
    const int ntx = (W + TW - 1) / TW, nty = (H + TH - 1) / TH;
    int tile = 0;
    const int ntiles = ntx * nty;
    for (;;) {
        const ray_t* lane[32];
        uint32_t pos[32];
        int alive = 0, from_pool = 0;
        if (npool >= 32 || (tile >= ntiles && npool > 0)) {
            from_pool = 1;
            S->instr += C_RESUME;
            g_pool_passes[g_p3_cur] += 1;
            for (int l = 0; l < 32; ++l) {
                if (npool) { --npool; lane[l] = pool[npool]; pos[l] = pool_pos[npool]; ++alive; }
                else { lane[l] = NULL; pos[l] = 0; }
            }
        } else if (tile < ntiles) {
            const int tx = tile % ntx, ty = tile / ntx;
            ++tile;
            for (int l = 0; l < 32; ++l) {
                int x = tx * TW + l % TW, y = ty * TH + l / TW;
                lane[l] = (x < W && y < H) ? &rays[(size_t)y * W + x] : NULL;
                pos[l] = 0;
                if (lane[l] && lane[l]->n) ++alive;
            }
            S->instr += C_TILE + C_SETUP + C_OUT;
        } else break;
        int q = 0, low = 0;
        while (alive) {
            int act = 0, maxf = 0, nsh = 0;
            int fl[8] = {0};
            for (int l = 0; l < 32; ++l) {
                if (!lane[l] || pos[l] >= lane[l]->n) continue;
                uint8_t v = g_trace[lane[l]->off + pos[l]++];
                int f = v & 15;
                ++act;
                if (f > maxf) maxf = f;
                for (int k = 1; k < f && k < 8; ++k) fl[k]++;
                if (v & 128) ++nsh;
                if (pos[l] >= lane[l]->n) --alive;
            }
            S->instr += C_BODY + C_FETCH * (maxf - 1);
            S->body_iters += 1; S->body_lanes += act;
            for (int k = 1; k < maxf; ++k) { S->fetch_iters += 1; S->fetch_lanes += fl[k]; }
            if (nsh) {
                S->instr += C_ENQ;
                q += nsh;
                if (q >= 32) { S->instr += C_DRAIN + 2 * C_ACC; S->shade_iters += 1; S->shade_lanes += 32; q -= 32; }
            }
            low = (alive <= theta) ? low + 1 : 0;
            const int more_work = tile < ntiles || npool > 0;
            if (alive && low >= patience && more_work) {   /* park the tail */
                if (q) { S->instr += C_DRAIN + 2 * C_ACC; S->shade_iters += 1; S->shade_lanes += q; q = 0; }
                S->instr += C_PARK + (from_pool ? 0 : 0);
                g_park_events[g_p3_cur] += 1; g_park_rays[g_p3_cur] += alive;
                for (int l = 0; l < 32; ++l)
                    if (lane[l] && pos[l] < lane[l]->n) { pool[npool] = lane[l]; pool_pos[npool] = pos[l]; ++npool; }
                alive = 0;
            }
        }
        if (q) { S->instr += C_DRAIN + 2 * C_ACC; S->shade_iters += 1; S->shade_lanes += q; }
        if (from_pool) S->instr += C_OUT;
    }
}

/* ---- MEM mode: DRAM traffic of a work order.  The tiles of all views are handed out in queue order to NW warps (a
 * warp takes the next tile when its current one ends); all busy warps advance one march iteration per round, and every
 * table-word fetch (a 32-byte sector of its table) and every shaded sample's 96-byte record (3 sectors, keyed by its
 * table entry) goes through an LRU model of its SM's L1 (L1KB per SM, 0 = none) and, on a miss, of the L2, both in
 * 32-byte sectors.  Warp w runs on SM (w / 4) mod NSM.  No associativity, no cache hints. */
typedef struct {
    uint64_t* key;    /* hash table: key + 1 (0 = empty), linear probing */
    int32_t* slot;
    uint64_t* skey;   /* LRU list over slots */
    int32_t *prev, *next;
    uint64_t mask;
    int32_t cap, n, head, tail;
} lru_t;

static inline uint64_t hmix(uint64_t k) { k *= 0x9E3779B97F4A7C15ull; return k ^ (k >> 29); }

static void lru_init(lru_t* L, int cap) {
    uint64_t hs = 1;
    while (hs < (uint64_t)cap * 2) hs <<= 1;
    L->key = (uint64_t*)calloc(hs, 8); L->slot = (int32_t*)malloc(hs * 4); L->mask = hs - 1;
    L->skey = (uint64_t*)malloc((size_t)cap * 8);
    L->prev = (int32_t*)malloc((size_t)cap * 4); L->next = (int32_t*)malloc((size_t)cap * 4);
    L->cap = cap; L->n = 0; L->head = L->tail = -1;
}
static void lru_free(lru_t* L) { free(L->key); free(L->slot); free(L->skey); free(L->prev); free(L->next); }
static inline void lru_unlink(lru_t* L, int s) {
    if (L->prev[s] >= 0) L->next[L->prev[s]] = L->next[s]; else L->head = L->next[s];
    if (L->next[s] >= 0) L->prev[L->next[s]] = L->prev[s]; else L->tail = L->prev[s];
}
static inline void lru_front(lru_t* L, int s) {
    L->prev[s] = -1; L->next[s] = L->head;
    if (L->head >= 0) L->prev[L->head] = s;
    L->head = s;
    if (L->tail < 0) L->tail = s;
}
static void hash_del(lru_t* L, uint64_t k) {   /* backward-shift deletion */
    uint64_t i = hmix(k) & L->mask;
    while (L->key[i] != k + 1) i = (i + 1) & L->mask;
    for (;;) {
        uint64_t j = i;
        for (;;) {
            j = (j + 1) & L->mask;
            if (!L->key[j]) { L->key[i] = 0; return; }
            const uint64_t h = hmix(L->key[j] - 1) & L->mask;   /* j's entry may fill i unless its home is in (i, j] */
            if (i <= j ? (h <= i || h > j) : (h <= i && h > j)) break;
        }
        L->key[i] = L->key[j]; L->slot[i] = L->slot[j];
        i = j;
    }
}
static inline int lru_touch(lru_t* L, uint64_t k) {   /* 1 on a miss */
    uint64_t i = hmix(k) & L->mask;
    while (L->key[i]) {
        if (L->key[i] == k + 1) {
            const int s = L->slot[i];
            if (L->head != s) { lru_unlink(L, s); lru_front(L, s); }
            return 0;
        }
        i = (i + 1) & L->mask;
    }
    int s;
    if (L->n < L->cap) {
        s = L->n++;
    } else {
        s = L->tail;
        lru_unlink(L, s);
        hash_del(L, L->skey[s]);
        i = hmix(k) & L->mask;
        while (L->key[i]) i = (i + 1) & L->mask;
    }
    L->key[i] = k + 1; L->slot[i] = s; L->skey[s] = k;
    lru_front(L, s);
    return 1;
}

/* A work order: the queue items in order, each (view, tx, ty); view -1 = an item with no pixel (past the last view
   of a view group).  blk = 0: every warp takes the next item of the launch.  blk = n: SM-affine blocks of n items
   (vr_march.cuh next_item, blk_mode): the warps of one SM take the items of their SM's current block, and the warp
   that finds it exhausted claims the next block of the launch for its SM. */
typedef struct {
    const char* name;
    const ray_t* const* vrays;    /* rays of each view */
    int32_t* tiles;               /* (view, tx, ty) per queue item */
    int ntiles, blk, W, H, nw, nsm, cap, l1cap;
    double tbl_acc, tbl_l1miss, tbl_miss, rec_acc, rec_l1miss, rec_miss, rounds;
    double sm_max, sm_min, sm_mean, sm_last, sm_first;   /* per-SM samples; round of each SM's last sample */
} replay_t;

/* L1 of the SM (when modelled), then L2; returns the DRAM misses and counts the L1 misses */
static inline int touch2(lru_t* L1, lru_t* L2, uint64_t k, double* l1miss) {
    if (L1 && !lru_touch(L1, k)) return 0;
    *l1miss += 1;
    return lru_touch(L2, k);
}

static void* replay(void* arg) {
    replay_t* J = (replay_t*)arg;
    const int TW = 4, TH = 8;
    const uint64_t kRec = 1ull << 40;   /* record sectors: their own address range */
    lru_t L;
    lru_init(&L, J->cap);
    lru_t* L1 = NULL;
    if (J->l1cap > 0) {
        L1 = (lru_t*)malloc((size_t)J->nsm * sizeof(lru_t));
        for (int s = 0; s < J->nsm; ++s) lru_init(&L1[s], J->l1cap);
    }
    const ray_t** lane = (const ray_t**)calloc((size_t)J->nw * 32, sizeof(ray_t*));
    uint32_t* pos = (uint32_t*)calloc((size_t)J->nw * 32, 4);
    uint32_t* kp = (uint32_t*)calloc((size_t)J->nw * 32, 4);
    int* alive = (int*)calloc(J->nw, sizeof(int));
    char* busy = (char*)calloc(J->nw, 1);
    int* sm_blk = (int*)malloc((size_t)J->nsm * sizeof(int));   /* SM's block: next item, end */
    int* sm_end = (int*)calloc(J->nsm, sizeof(int));
    double* sm_work = (double*)calloc(J->nsm, sizeof(double));
    double* sm_last = (double*)calloc(J->nsm, sizeof(double));
    for (int s = 0; s < J->nsm; ++s) sm_blk[s] = 0;
    int next = 0;
    for (;;) {
        int any = 0;
        for (int w = 0; w < J->nw; ++w) {
            const ray_t** ln = lane + (size_t)w * 32;
            uint32_t* ps = pos + (size_t)w * 32;
            uint32_t* kq = kp + (size_t)w * 32;
            const int sm = (w / 4) % J->nsm;   /* 4 warps per CTA, CTAs spread round-robin over the SMs */
            if (!busy[w]) {
                int item;
                if (!J->blk) {
                    if (next >= J->ntiles) continue;
                    item = next++;
                } else {
                    if (sm_blk[sm] >= sm_end[sm]) {
                        if (next >= J->ntiles) continue;
                        sm_blk[sm] = next; sm_end[sm] = next + J->blk; next += J->blk;
                    }
                    item = sm_blk[sm]++;
                }
                const int32_t* t = J->tiles + 3 * (size_t)item;
                alive[w] = 0;
                const ray_t* rays = t[0] >= 0 ? J->vrays[t[0]] : NULL;
                for (int l = 0; l < 32; ++l) {
                    const int x = t[1] * TW + l % TW, y = t[2] * TH + l / TW;
                    ln[l] = (rays && x < J->W && y < J->H) ? &rays[(size_t)y * J->W + x] : NULL;
                    ps[l] = 0;
                    if (ln[l]) { kq[l] = ln[l]->koff; if (ln[l]->n) ++alive[w]; }
                }
                busy[w] = 1;
            }
            any = 1;
            lru_t* l1 = L1 ? &L1[sm] : NULL;
            for (int l = 0; l < 32; ++l) {
                if (!ln[l] || ps[l] >= ln[l]->n) continue;
                const uint8_t v = g_trace[ln[l]->off + ps[l]++];
                sm_work[sm] += 1; sm_last[sm] = J->rounds;
                for (int f = v & 15; f > 0; --f) { J->tbl_acc += 1; J->tbl_miss += touch2(l1, &L, g_keys[kq[l]++], &J->tbl_l1miss); }
                if (v & 128) {
                    const uint64_t r = (uint64_t)g_keys[kq[l]++] * 3;
                    J->rec_acc += 1;
                    for (int s = 0; s < 3; ++s) J->rec_miss += touch2(l1, &L, kRec + r + s, &J->rec_l1miss);
                }
                if (ps[l] >= ln[l]->n) --alive[w];
            }
            if (alive[w] <= 0) busy[w] = 0;
        }
        if (!any) break;
        J->rounds += 1;
    }
    J->sm_max = J->sm_min = sm_work[0]; J->sm_last = J->sm_first = sm_last[0]; J->sm_mean = 0;
    for (int s = 0; s < J->nsm; ++s) {
        J->sm_mean += sm_work[s] / J->nsm;
        if (sm_work[s] > J->sm_max) J->sm_max = sm_work[s];
        if (sm_work[s] < J->sm_min) J->sm_min = sm_work[s];
        if (sm_last[s] > J->sm_last) J->sm_last = sm_last[s];
        if (sm_last[s] < J->sm_first) J->sm_first = sm_last[s];
    }
    free(lane); free(pos); free(kp); free(alive); free(busy); free(sm_blk); free(sm_end); free(sm_work); free(sm_last);
    if (L1) { for (int s = 0; s < J->nsm; ++s) lru_free(&L1[s]); free(L1); }
    lru_free(&L);
    return NULL;
}

static inline int centre_out(int r, int rows) {   /* vr_march.cuh decode_item */
    const int half = rows >> 1;
    return r < 2 * half ? ((r & 1) ? half + (r >> 1) : half - 1 - (r >> 1)) : r;
}

/* group = 0: view-major (all tiles of view 0, then view 1, ...); group = g: tile rows outermost inside each group of
   g consecutive views, views inside rows, tx innermost (g >= ncam: one group, row-major across the whole launch) */
static int32_t* make_order(int ncam, int ntx, int nty, int group) {
    int32_t* t = (int32_t*)malloc((size_t)ncam * ntx * nty * 3 * 4);
    size_t k = 0;
    if (!group) {
        for (int v = 0; v < ncam; ++v)
            for (int r = 0; r < nty; ++r)
                for (int x = 0; x < ntx; ++x) { t[k++] = v; t[k++] = x; t[k++] = centre_out(r, nty); }
        return t;
    }
    for (int g0 = 0; g0 < ncam; g0 += group)
        for (int r = 0; r < nty; ++r)
            for (int v = g0; v < g0 + group && v < ncam; ++v)
                for (int x = 0; x < ntx; ++x) { t[k++] = v; t[k++] = x; t[k++] = centre_out(r, nty); }
    return t;
}

/* SM-affine blocks of bw x bh tiles of g consecutive views at the same position, in the order (block row, view group,
   block x) (vr_march.cuh decode_item, blk_mode); inside a block the view is innermost (view_inner) or the tile is.
   Every block has bw * bh * g items; those past the image edge or the last view have no pixel.  *n = items. */
static int32_t* make_blocks(int ncam, int ntx, int nty, int bw, int bh, int g, int view_inner, int* n) {
    const int bx = (ntx + bw - 1) / bw, by = (nty + bh - 1) / bh, ng = (ncam + g - 1) / g, nbt = bw * bh * g;
    *n = bx * by * ng * nbt;
    int32_t* t = (int32_t*)malloc((size_t)*n * 3 * 4);
    size_t k = 0;
    for (int r = 0; r < by; ++r)
        for (int gi = 0; gi < ng; ++gi)
            for (int x = 0; x < bx; ++x)
                for (int i = 0; i < nbt; ++i) {
                    const int v = view_inner ? i % g : i / (bw * bh), tl = view_inner ? i / g : i % (bw * bh);
                    const int view = gi * g + v;
                    t[k++] = view < ncam ? view : -1; t[k++] = x * bw + tl % bw; t[k++] = r * bh + tl / bw;
                }
    return t;
}

/* every (view, tile) exactly once */
static int check_order(const int32_t* t, int n, int ncam, int ntx, int nty) {
    char* seen = (char*)calloc((size_t)ncam * ntx * nty, 1);
    int bad = 0;
    for (int i = 0; i < n; ++i) {
        const int v = t[3 * i], x = t[3 * i + 1], y = t[3 * i + 2];
        if (v < 0 || x >= ntx || y >= nty) continue;
        if (seen[((size_t)v * nty + y) * ntx + x]++) bad = 1;
    }
    for (size_t i = 0; i < (size_t)ncam * ntx * nty; ++i) if (seen[i] != 1) bad = 1;
    free(seen);
    return bad;
}

typedef struct { const char* name; int group, bw, bh, g, view_inner; } order_t;
static const order_t g_orders[] = {
    {"view-major (before 3c9fce8)", 0, 0, 0, 0, 0},
    {"rows across all views (current)", -1, 0, 0, 0, 0},
    {"blocks 8x8 tiles x 1 view", 0, 8, 8, 1, 0},
    {"blocks 4x4 tiles x 1 view", 0, 4, 4, 1, 0},
    {"blocks 16x8 tiles x 1 view", 0, 16, 8, 1, 0},
    {"blocks 8x8 x 2 views, view inner", 0, 8, 8, 2, 1},
    {"blocks 8x8 x 2 views, tile inner", 0, 8, 8, 2, 0},
    {"blocks 8x8 x 4 views, view inner", 0, 8, 8, 4, 1},
    {"blocks 8x8 x 4 views, tile inner", 0, 8, 8, 4, 0},
    {"blocks 8x8 x 8 views, view inner", 0, 8, 8, 8, 1},
    {"blocks 8x8 x 8 views, tile inner", 0, 8, 8, 8, 0},
    {"blocks 4x4 x 4 views, view inner", 0, 4, 4, 4, 1},
    {"blocks 4x4 x 4 views, tile inner", 0, 4, 4, 4, 0},
    {"blocks 4x2 x 8 views, view inner", 0, 4, 2, 8, 1},
};
enum { kOrders = sizeof(g_orders) / sizeof(g_orders[0]) };

/* lane_sim --check-orders <views> <W> <H>: checks that every order of the MEM replay visits every (view, tile)
   exactly once; exit status 1 if one does not */
static int check_orders(int ncam, int W, int H) {
    const int ntx = (W + 3) / 4, nty = (H + 7) / 8;
    int bad = 0;
    for (int k = 0; k < kOrders; ++k) {
        const order_t* o = &g_orders[k];
        int n = ncam * ntx * nty;
        int32_t* t = o->bw ? make_blocks(ncam, ntx, nty, o->bw, o->bh, o->g, o->view_inner, &n)
                           : make_order(ncam, ntx, nty, o->group < 0 ? ncam : o->group);
        const int b = check_order(t, n, ncam, ntx, nty);
        printf("%-36s %s\n", o->name, b ? "BAD" : "ok");
        bad |= b;
        free(t);
    }
    return bad;
}

static void mem_main(const orc_tree* tree, const orc_camera* cams, int ncam, int W, int H) {
    const int nw = getenv("NWARPS") ? atoi(getenv("NWARPS")) : 4224;   /* 8 CTAs x 4 warps x 132 SMs */
    const int nsm = getenv("NSM") ? atoi(getenv("NSM")) : 132;
    const double l2mb = getenv("L2MB") ? atof(getenv("L2MB")) : 50.0;
    /* L1 per SM: 256 KB less the 100 KB shared-memory carve-out that 8 CTAs x (9.2 KB + 1 KB reserved) need */
    const double l1kb = getenv("L1KB") ? atof(getenv("L1KB")) : 156.0;
    const int cap = (int)(l2mb * 1024 * 1024 / 32), l1cap = (int)(l1kb * 1024 / 32);
    const int ntx = (W + 3) / 4, nty = (H + 7) / 8;
    orc_options opt;
    orc_default_options(&opt);
    ray_t** vrays = (ray_t**)malloc((size_t)ncam * sizeof(ray_t*));
    double nshade = 0;
    for (int c = 0; c < ncam; ++c) {
        vrays[c] = (ray_t*)malloc((size_t)W * H * sizeof(ray_t));
        const size_t s0 = g_trace_n;
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x) trace_one(tree, &cams[c], &opt, x, y, &vrays[c][(size_t)y * W + x]);
        for (size_t i = s0; i < g_trace_n; ++i) nshade += g_trace[i] >> 7;
    }
    printf("MEM: %d views %dx%d, %d warps in flight, L2 %.0f MB (%d sectors); %.2fM samples, %.3fM shaded per view\n",
           ncam, W, H, nw, l2mb, cap, g_trace_n / 1e6 / ncam, nshade / 1e6 / ncam);
    printf("L1 per SM %.0f KB (%d sectors, 0 = no L1 model), %d SMs, warp w on SM (w / 4) mod %d\n", l1kb, l1cap, nsm, nsm);
    replay_t J[kOrders];
    pthread_t th[kOrders];
    for (int k = 0; k < kOrders; ++k) {
        const order_t* o = &g_orders[k];
        memset(&J[k], 0, sizeof(J[k]));
        J[k].name = o->name; J[k].vrays = (const ray_t* const*)vrays;
        J[k].ntiles = ncam * ntx * nty;
        if (o->bw) {
            J[k].tiles = make_blocks(ncam, ntx, nty, o->bw, o->bh, o->g, o->view_inner, &J[k].ntiles);
            J[k].blk = o->bw * o->bh * o->g;
        } else {
            J[k].tiles = make_order(ncam, ntx, nty, o->group < 0 ? ncam : o->group);
        }
        J[k].W = W; J[k].H = H; J[k].nw = nw; J[k].nsm = nsm; J[k].cap = cap; J[k].l1cap = l1cap;
        pthread_create(&th[k], NULL, replay, &J[k]);
    }
    /* hit rates per access (tables: one 32-byte sector, records: 3 sectors); "rec L2 hit" is of the L1 misses;
       SM samples: most / fewest per SM over the mean; tail: rounds between the first and the last SM running dry,
       over all rounds of the launch */
    printf("%-36s %8s %8s %8s %10s %10s %9s %9s %6s\n", "order", "tbl L1", "rec L1", "rec L2", "tbl MB/fr",
           "DRAM MB/fr", "SM max", "SM min", "tail");
    for (int k = 0; k < kOrders; ++k) {
        pthread_join(th[k], NULL);
        const double tb = J[k].tbl_miss * 32 / 1e6 / ncam, rb = J[k].rec_miss * 32 / 1e6 / ncam;
        printf("%-36s %7.1f%% %7.1f%% %7.1f%% %10.1f %10.1f %9.3f %9.3f %5.1f%%\n", J[k].name,
               100 * (1 - J[k].tbl_l1miss / (J[k].tbl_acc + 1e-9)), 100 * (1 - J[k].rec_l1miss / (3 * J[k].rec_acc + 1e-9)),
               100 * (1 - J[k].rec_miss / (J[k].rec_l1miss + 1e-9)), tb, tb + rb, J[k].sm_max / J[k].sm_mean,
               J[k].sm_min / J[k].sm_mean, 100 * (J[k].sm_last - J[k].sm_first) / (J[k].rounds + 1e-9));
        free(J[k].tiles);
    }
}

/* ---- tile culling of batch launches: the policy of volrend_b200/csrc/vr_cull.cu restated on the CPU, with the
   same grid level (32^3 cells of the largest sigma of the reachable leaves), the same dilation (eps in tree space,
   dpx in pixels) and the same granularity (one bit per 4x8 tile).  No NDC trees, no bands, no render_bbox other than
   the unit cube here: the kernel marks whole views for those. */
#define CULL_LV 5
#define CULL_N (1 << CULL_LV)
#define CULL_CELL_TILES_MAX 1024   /* kCellTilesMax: a larger cell marks the whole view */
static float g_cgrid[CULL_N * CULL_N * CULL_N];
static float g_csmin;

static void cull_visit(const orc_tree* tree, int64_t node, int depth, uint32_t ox, uint32_t oy, uint32_t oz) {
    const int sh = 23 - depth;   /* children of a node of depth `depth` have cubes of 2^(24 - depth - 1) units */
    for (int oct = 0; oct < 8; ++oct) {
        const uint32_t x = ox | ((uint32_t)(oct >> 2 & 1) << sh), y = oy | ((uint32_t)(oct >> 1 & 1) << sh),
                       z = oz | ((uint32_t)(oct & 1) << sh);
        const int64_t s = node * 8 + oct;
        const int32_t skip = tree->child[s];
        if (skip) { cull_visit(tree, node + skip, depth + 1, x, y, z); continue; }
        const float sg = h2f(tree->data[(size_t)s * tree->data_dim + tree->data_dim - 1]);
        if (sg != sg) continue;
        if (sg < g_csmin) g_csmin = sg;
        const int cs = 24 - CULL_LV;
        const uint32_t span = (1u << sh) - 1u;
        for (uint32_t cx = x >> cs; cx <= (x + span) >> cs; ++cx)
            for (uint32_t cy = y >> cs; cy <= (y + span) >> cs; ++cy)
                for (uint32_t cz = z >> cs; cz <= (z + span) >> cs; ++cz) {
                    float* c = &g_cgrid[(cx * CULL_N + cy) * CULL_N + cz];
                    if (sg > *c) *c = sg;
                }
    }
}

static void cull_grid(const orc_tree* tree) {
    for (int i = 0; i < CULL_N * CULL_N * CULL_N; ++i) g_cgrid[i] = -INFINITY;
    g_csmin = INFINITY;
    cull_visit(tree, 0, 0, 0, 0, 0);
}

/* mask[ty * tiles_x + tx] = 1: the tile may hold a ray that shades (vr_cull.cu tile_mask_kernel) */
static void cull_mask(const orc_tree* tree, const orc_camera* cam, const orc_options* opt, uint8_t* mask) {
    const int W = cam->width, H = cam->height, ntx = (W + 3) / 4, nty = (H + 7) / 8;
    memset(mask, 0, (size_t)ntx * nty);
    const float* c2w = cam->c2w;
    const double M[9] = {c2w[0], c2w[3], -(double)c2w[6], c2w[1], c2w[4], -(double)c2w[7], c2w[2], c2w[5], -(double)c2w[8]};
    const double a0 = M[4] * M[8] - M[5] * M[7], a1 = M[5] * M[6] - M[3] * M[8], a2 = M[3] * M[7] - M[4] * M[6];
    const double det = M[0] * a0 + M[1] * a1 + M[2] * a2;
    int all = tree->ndc_width > 0.f || opt->sigma_thresh < g_csmin || !(fabs(det) > 0.0);
    for (int i = 0; i < 3; ++i) all |= !(opt->render_bbox[i] >= 0.f && opt->render_bbox[i + 3] <= 1.f);
    double m[9] = {0}, c[3] = {0}, l1 = 0.0;
    if (!all) {
        const double id = 1.0 / det;
        m[0] = a0 * id; m[1] = (M[2] * M[7] - M[1] * M[8]) * id; m[2] = (M[1] * M[5] - M[2] * M[4]) * id;
        m[3] = a1 * id; m[4] = (M[0] * M[8] - M[2] * M[6]) * id; m[5] = (M[2] * M[3] - M[0] * M[5]) * id;
        m[6] = a2 * id; m[7] = (M[1] * M[6] - M[0] * M[7]) * id; m[8] = (M[0] * M[4] - M[1] * M[3]) * id;
        for (int i = 0; i < 3; ++i) { c[i] = c2w[9 + i]; l1 += fabs((double)tree->scale[i] * c2w[9 + i] + tree->offset[i]); }
    }
    const double eps = 1e-5 * (4.0 + l1), sdpx = 1e-5 * (fabs((double)cam->fx) + fabs((double)cam->fy));
    for (int cell = 0; !all && cell < CULL_N * CULL_N * CULL_N; ++cell) {
        if (!(g_cgrid[cell] > opt->sigma_thresh)) continue;
        const int ci[3] = {cell >> (2 * CULL_LV), (cell >> CULL_LV) & (CULL_N - 1), cell & (CULL_N - 1)};
        double lo[3], hi[3];
        for (int i = 0; i < 3; ++i) {
            const double a = ((double)ci[i] / CULL_N - eps - tree->offset[i]) / tree->scale[i];
            const double b = ((double)(ci[i] + 1) / CULL_N + eps - tree->offset[i]) / tree->scale[i];
            lo[i] = fmin(a, b) - c[i]; hi[i] = fmax(a, b) - c[i];
        }
        double wmin = INFINITY, wmax = -INFINITY, xmin = INFINITY, xmax = -INFINITY, ymin = INFINITY, ymax = -INFINITY,
               vmax = 0.0;
        for (int k = 0; k < 8; ++k) {
            const double q0 = (k & 4) ? hi[0] : lo[0], q1 = (k & 2) ? hi[1] : lo[1], q2 = (k & 1) ? hi[2] : lo[2];
            const double u = m[0] * q0 + m[1] * q1 + m[2] * q2, v = m[3] * q0 + m[4] * q1 + m[5] * q2,
                         w = m[6] * q0 + m[7] * q1 + m[8] * q2;
            wmin = fmin(wmin, w); wmax = fmax(wmax, w);
            const double vx = u / w, vy = v / w;
            vmax = fmax(vmax, fabs(vx) + fabs(vy));
            const double px = vx * cam->fx + 0.5 * W, py = 0.5 * H - vy * cam->fy;
            xmin = fmin(xmin, px); xmax = fmax(xmax, px); ymin = fmin(ymin, py); ymax = fmax(ymax, py);
        }
        if (wmax < 0.0) continue;
        if (!(wmin > 0.0)) { all = 1; break; }
        const double d = 1.0 + sdpx * (1.0 + vmax) * (1.0 + vmax);
        const double fx0 = ceil(xmin - d), fx1 = floor(xmax + d), fy0 = ceil(ymin - d), fy1 = floor(ymax + d);
        if (!(isfinite(fx0) && isfinite(fx1) && isfinite(fy0) && isfinite(fy1))) { all = 1; break; }
        if (fx1 < 0 || fx0 > W - 1 || fy1 < 0 || fy0 > H - 1) continue;
        const int tx0 = (int)fmax(fx0, 0.0) / 4, tx1 = (int)fmin(fx1, W - 1.0) / 4;
        const int ty0 = (int)fmax(fy0, 0.0) / 8, ty1 = (int)fmin(fy1, H - 1.0) / 8;
        if ((long long)(ty1 - ty0 + 1) * (tx1 - tx0 + 1) > CULL_CELL_TILES_MAX) { all = 1; break; }
        for (int ty = ty0; ty <= ty1; ++ty)
            for (int tx = tx0; tx <= tx1; ++tx) mask[ty * ntx + tx] = 1;
    }
    if (all) memset(mask, 1, (size_t)ntx * nty);
}

/* --cull: per view, the tiles the policy leaves unmarked although a ray in them shades (must be none), the tiles it
   marks that never shade, and the share of warp body iterations and of warp instructions (cost model P0) it culls
   next to the bound of culling exactly the tiles where no ray shades. */
static int cull_main(const orc_tree* tree, const orc_camera* cams, int ncam, const orc_options* opt) {
    const int W = cams[0].width, H = cams[0].height, ntx = (W + 3) / 4, nty = (H + 7) / 8;
    ray_t* rays = (ray_t*)malloc((size_t)W * H * sizeof(ray_t));
    uint8_t* mask = (uint8_t*)malloc((size_t)ntx * nty);
    cull_grid(tree);
    double T[7] = {0};   /* tiles, marked, shading, marked never shading, body, body culled, body bound */
    stats_t sf = {0}, sc = {0}, sb = {0};
    long long bad = 0;
    for (int v = 0; v < ncam; ++v) {
        g_trace_n = 0;
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x) trace_one(tree, &cams[v], opt, x, y, &rays[(size_t)y * W + x]);
        cull_mask(tree, &cams[v], opt, mask);
        long long vt[4] = {0, 0, 0, 0}, vbad = 0;
        ray_t* cut = (ray_t*)malloc((size_t)W * H * sizeof(ray_t));
        ray_t* ideal = (ray_t*)malloc((size_t)W * H * sizeof(ray_t));
        memcpy(cut, rays, (size_t)W * H * sizeof(ray_t));
        memcpy(ideal, rays, (size_t)W * H * sizeof(ray_t));
        for (int ty = 0; ty < nty; ++ty)
            for (int tx = 0; tx < ntx; ++tx) {
                int shades = 0;
                uint32_t body = 0;
                for (int l = 0; l < 32; ++l) {
                    const int x = tx * 4 + l % 4, y = ty * 8 + l / 4;
                    if (x >= W || y >= H) continue;
                    const ray_t* r = &rays[(size_t)y * W + x];
                    if (r->n > body) body = r->n;
                    for (uint32_t k = 0; k < r->n && !shades; ++k) shades = g_trace[r->off + k] >> 7;
                }
                const int mk = mask[ty * ntx + tx];
                vt[0] += 1; vt[1] += mk; vt[2] += shades; vt[3] += mk && !shades;
                if (shades && !mk) ++vbad;
                T[4] += body; T[5] += mk ? 0 : body; T[6] += shades ? 0 : body;
                for (int l = 0; l < 32; ++l) {
                    const int x = tx * 4 + l % 4, y = ty * 8 + l / 4;
                    if (x >= W || y >= H) continue;
                    if (!mk) cut[(size_t)y * W + x].n = 0;
                    if (!shades) ideal[(size_t)y * W + x].n = 0;
                }
            }
        sim_tiles(rays, W, H, 0, &sf);
        sim_tiles(cut, W, H, 0, &sc);
        sim_tiles(ideal, W, H, 0, &sb);
        free(cut); free(ideal);
        printf("cull view %d: tiles %lld marked %lld shading %lld unmarked_shading %lld marked_never_shading %lld\n", v,
               vt[0], vt[1], vt[2], vbad, vt[3]);
        for (int k = 0; k < 4; ++k) T[k] += vt[k];
        bad += vbad;
    }
    /* a culled tile skips its ray set-up too (C_SETUP of every tile in sim_tiles) */
    const double setup_c = C_SETUP * (T[0] - T[1]), setup_b = C_SETUP * (T[0] - T[2]);
    printf("cull total: views %d tiles %.0f unmarked_shading %lld tiles_culled %.4f (bound %.4f) marked_never_shading "
           "%.4f body_culled %.4f (bound %.4f) instr_culled %.4f (bound %.4f)\n", ncam, T[0], bad, 1 - T[1] / T[0],
           1 - T[2] / T[0], T[3] / T[0], T[5] / T[4], T[6] / T[4], 1 - (sc.instr - setup_c) / sf.instr,
           1 - (sb.instr - setup_b) / sf.instr);
    free(rays); free(mask);
    return bad ? 1 : 0;
}

static void report(const char* name, const stats_t* S, int frames) {
    printf("%-34s %7.2f Minstr/frame  body %5.1f/32 (%6.2fM it)  fetch+ %5.1f/32 (%5.2fM)  shade %5.1f/32 (%5.3fM it)\n", name,
           S->instr / frames / 1e6, S->body_lanes / (S->body_iters + 1e-9), S->body_iters / frames / 1e6,
           S->fetch_lanes / (S->fetch_iters + 1e-9), S->fetch_iters / frames / 1e6,
           S->shade_lanes / (S->shade_iters + 1e-9), S->shade_iters / frames / 1e6);
}

int main(int argc, char** argv) {
    if (argc == 5 && !strcmp(argv[1], "--check-orders")) return check_orders(atoi(argv[2]), atoi(argv[3]), atoi(argv[4]));
    if (argc < 2) { fprintf(stderr, "usage: lane_sim dump.bin | lane_sim --check-orders views W H\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) { perror("open"); return 1; }
    int64_t hdr[4];  /* capacity, W, H, n_cams */
    if (fread(hdr, 8, 4, f) != 4) return 1;
    const int64_t cap = hdr[0];
    const int W = (int)hdr[1], H = (int)hdr[2], ncam = (int)hdr[3];
    float meta[8];  /* offset[3], scale[3], fx, fy */
    if (fread(meta, 4, 8, f) != 8) return 1;
    int32_t* child = (int32_t*)malloc((size_t)cap * 8 * 4);
    uint16_t* sigma = (uint16_t*)malloc((size_t)cap * 8 * 2);
    float* cams = (float*)malloc((size_t)ncam * 12 * 4);
    if (fread(child, 4, (size_t)cap * 8, f) != (size_t)cap * 8) return 1;
    if (fread(sigma, 2, (size_t)cap * 8, f) != (size_t)cap * 8) return 1;
    if (fread(cams, 4, (size_t)ncam * 12, f) != (size_t)ncam * 12) return 1;
    fclose(f);
    {
        const int lv = getenv("LEVELS") ? atoi(getenv("LEVELS")) : 2, g0 = getenv("PHASE") ? atoi(getenv("PHASE")) : lv;
        for (int k = 0; k < 32; ++k) g_b[k] = g0 + k * lv;
        printf("tables: %d levels per step, root table resolves %d\n", lv, g0);
    }
    {
        struct { const char* name; double* v; } cs[] = {{"C_SETUP", &C_SETUP}, {"C_BODY", &C_BODY}, {"C_FETCH", &C_FETCH},
                                                        {"C_SHADE", &C_SHADE}};
        for (int k = 0; k < 4; ++k)
            if (getenv(cs[k].name)) *cs[k].v = atof(getenv(cs[k].name));
        printf("cost model: C_SETUP %g, C_BODY %g, C_FETCH %g, C_SHADE %g\n", C_SETUP, C_BODY, C_FETCH, C_SHADE);
    }
    pthread_once(&g_h2f_once, init_h2f);
    orc_tree tree;
    memset(&tree, 0, sizeof(tree));
    tree.child = child; tree.data = sigma; tree.capacity = cap; tree.N = 2; tree.data_dim = 1;
    tree.format = ORC_FMT_SH; tree.basis_dim = 16; tree.ndc_width = -1.f;
    for (int i = 0; i < 3; ++i) { tree.offset[i] = meta[i]; tree.scale[i] = meta[3 + i]; }
    orc_options opt;
    orc_default_options(&opt);
    if (getenv("THRESH")) opt.sigma_thresh = (float)atof(getenv("THRESH"));
    if (getenv("CULL") && atoi(getenv("CULL"))) {   /* tile culling of batch launches instead of the lane policies */
        orc_camera* oc = (orc_camera*)calloc(ncam, sizeof(orc_camera));
        for (int c = 0; c < ncam; ++c) {
            oc[c].width = W; oc[c].height = H; oc[c].fx = meta[6]; oc[c].fy = meta[7];
            memcpy(oc[c].c2w, cams + 12 * c, 48);
        }
        return cull_main(&tree, oc, ncam, &opt);
    }
    if (getenv("MEM") && atoi(getenv("MEM"))) {   /* L2 replay of the work orders instead of the lane policies */
        g_mem = 1;
        orc_camera* oc = (orc_camera*)calloc(ncam, sizeof(orc_camera));
        for (int c = 0; c < ncam; ++c) {
            oc[c].width = W; oc[c].height = H; oc[c].fx = meta[6]; oc[c].fy = meta[7];
            memcpy(oc[c].c2w, cams + 12 * c, 48);
        }
        mem_main(&tree, oc, ncam, W, H);
        return 0;
    }

    stats_t P0 = {0}, P1 = {0}, P2a[6], P2b[6], P3[6];
    memset(P3, 0, sizeof(P3));
    memset(P2a, 0, sizeof(P2a)); memset(P2b, 0, sizeof(P2b));
    const int thetas[6] = {4, 8, 12, 16, 24, 32};
    ray_t* rays = (ray_t*)malloc((size_t)W * H * sizeof(ray_t));
    double nsamp = 0, nshade = 0, nhit = 0, nmarch = 0;
    for (int c = 0; c < ncam; ++c) {
        orc_camera cam;
        cam.width = W; cam.height = H; cam.fx = meta[6]; cam.fy = meta[7];
        memcpy(cam.c2w, cams + 12 * c, 48);
        g_trace_n = 0;
        for (int y = 0; y < H; ++y)
            for (int x = 0; x < W; ++x) trace_one(&tree, &cam, &opt, x, y, &rays[(size_t)y * W + x]);
        for (size_t i = 0; i < (size_t)W * H; ++i) { nhit += rays[i].hit; nmarch += rays[i].n > 0; }
        {   /* ray-length distribution (single-frame tail bound) */
            static uint32_t hist[4096];
            memset(hist, 0, sizeof(hist));
            uint32_t mx = 0;
            for (size_t i = 0; i < (size_t)W * H; ++i) { uint32_t n = rays[i].n < 4095 ? rays[i].n : 4095; hist[n]++; if (n > mx) mx = n; }
            size_t acc = 0; const double qs[5] = {0.5, 0.9, 0.99, 0.999, 0.9999}; int qi = 0;
            printf("view %d samples/ray:", c);
            for (uint32_t n = 0; n <= mx && qi < 5; ++n) { acc += hist[n]; while (qi < 5 && acc >= qs[qi] * W * H) { printf(" p%g=%u", qs[qi] * 100, n); ++qi; } }
            printf(" max=%u\n", mx);
        }
        nsamp += g_trace_n;
        for (size_t i = 0; i < g_trace_n; ++i) nshade += g_trace[i] >> 7;
        sim_tiles(rays, W, H, 0, &P0);
        sim_tiles(rays, W, H, 1, &P1);
        for (int k = 0; k < 6; ++k) { g_p3_cur = k; sim_park(rays, W, H, g_p3_theta[k], g_p3_pat[k], &P3[k]); }
        for (int k = 0; k < 6; ++k) {
            sim_refill(rays, W, H, thetas[k], 64, 0, &P2a[k]);
            sim_refill(rays, W, H, thetas[k], 64, 1, &P2b[k]);
        }
    }
    printf("frames %d: samples %.2fM shaded %.3fM per frame, rays hit %.0f, rays with samples %.0f\n", ncam, nsamp / ncam / 1e6,
           nshade / ncam / 1e6, nhit / ncam, nmarch / ncam);
    {
        double tot = 0, cum = 0;
        for (int a = 1; a <= 32; ++a) tot += g_act_hist[a];
        printf("body iterations by active lanes (cumulative %%):");
        for (int a = 1; a <= 32; ++a) { cum += g_act_hist[a]; if (a % 4 == 0) printf(" <=%d:%.1f", a, 100 * cum / tot); }
        printf("\n");
    }
    report("P0 tiles, inline shading", &P0, ncam);
    report("P1 tiles + shared shade queue", &P1, ncam);
    for (int k = 0; k < 6; ++k) {
        char nm[64];
        snprintf(nm, sizeof nm, "P3 queue + tail parking th=%d pat=%d", g_p3_theta[k], g_p3_pat[k]);
        report(nm, &P3[k], ncam);
        printf("      park events %.0f/frame (%.1f rays each), pool passes %.0f/frame\n", g_park_events[k] / ncam, g_park_rays[k] / (g_park_events[k] + 1e-9), g_pool_passes[k] / ncam);
    }
    for (int k = 0; k < 6; ++k) {
        char nm[64];
        snprintf(nm, sizeof nm, "P2 refill theta=%d, inline", thetas[k]);
        report(nm, &P2a[k], ncam);
        snprintf(nm, sizeof nm, "P2 refill theta=%d + queue", thetas[k]);
        report(nm, &P2b[k], ncam);
    }
    return 0;
}
