/*
 * astar_oracle.c — CPU restatement of the reference's differentiable A* hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product package may import, link or
 * call this file; only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs do.
 *
 * Reference being restated (all file:line relative to /root/reference/):
 *   src/neural_astar/planner/differentiable_astar.py
 *     :26-52   get_heuristic          -> heuristic_plus_cost()
 *     :55-74   _st_softmax_noexp      -> select_literal()
 *     :77-93   expand (3x3 stencil)   -> the neighbour loops over kDy / kDx below
 *     :96-125  backtrack              -> backtrack_literal() / backtrack_spec()
 *     :187-252 state machine          -> nastar_oracle_forward_literal()
 *   (autograd of the above; closed form SURVEY.md App. B) -> nastar_oracle_backward()
 *
 * Two restatements are provided and cross-checked by tests/:
 *   LITERAL  dense planes, exp/softmax/first-argmax selection, batch-coupled stop
 *            exactly as the Python loop is written (incl. post-solve steps).
 *   SPEC     the distilled per-map state machine (SURVEY.md App. A.2): selection is
 *            the lexicographic arg-min of (f, flat index) over the open set, per-map
 *            early exit.  This is the form the CUDA engine implements; it equals
 *            LITERAL except when expf()/division rounding merges two distinct f
 *            values into equal softmax weights (measured: 0 in 141k vanilla
 *            selections; see DESIGN.md "selection semantics").
 *
 * Mechanism (NASTAR_MECH_*, include/nastar_b200.h), as DifferentiableAstar(mechanism=) takes it:
 *   MOORE  the 8 neighbours, h = Chebyshev + 0.001 * Euclid (the reference's own search);
 *   NEWS   N, E, W, S only, h = Manhattan + 0.001 * Euclid (the planning-datasets generator's
 *          NorthEastWestSouth, mechanism.py:113-131; get_news_heuristic's fp32 operation order).
 *
 * Parity pinning: both restatements are checked against golden vectors produced by
 * running the reference's own Python (tests/golden/make_golden.py, make_golden_news.py).
 *
 * Arithmetic: IEEE fp32, one rounding per op (compile with -ffp-contract=off).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#include "nastar_b200.h"

#define NASTAR_ORACLE_OK 0
#define NASTAR_ORACLE_EINVAL 1

static int argmax_first(const float *x, int n)
{
    /* torch.max(dim) on CPU returns the first maximal index; NaN is maximal. */
    int best = 0;
    float bv = x[0];
    for (int i = 1; i < n; ++i) {
        if (x[i] > bv || (x[i] != x[i] && bv == bv)) { bv = x[i]; best = i; }
    }
    return best;
}

/* the moves as (dy, dx): N, E, W, S, NE, NW, SE, SW (mechanism.py:58, :140-149); NEWS takes the first 4 */
static const int kDy[8] = {-1, 0, 0, +1, -1, -1, +1, +1};
static const int kDx[8] = {0, +1, -1, 0, +1, -1, +1, -1};

static int mech_ok(int mech) { return mech == NASTAR_MECH_MOORE || mech == NASTAR_MECH_NEWS; }
static int num_moves(int mech) { return mech == NASTAR_MECH_NEWS ? 4 : 8; }

/* differentiable_astar.py:26-52 (Moore) or get_news_heuristic (NEWS), followed by :192 (h = heuristic + cost) */
static void heuristic_plus_cost(const float *cost, int H, int W, int goal, int mech, float *h)
{
    const float gy = (float)(goal / W), gx = (float)(goal % W);
    for (int y = 0; y < H; ++y) {
        for (int x = 0; x < W; ++x) {
            float dy = fabsf((float)y - gy), dx = fabsf((float)x - gx);
            float dist = (mech == NASTAR_MECH_NEWS) ? dy + dx : (dy + dx) - fminf(dy, dx);
            float euc = sqrtf(dy * dy + dx * dx);
            float t = 0.001f * euc;
            float heur = dist + t;
            h[y * W + x] = heur + cost[y * W + x];
        }
    }
}

int nastar_oracle_num_threads(void)
{
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

void nastar_oracle_set_threads(int n)
{
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

/* ------------------------------------------------------------------------- */
/* LITERAL restatement (dense, batch-coupled)                                */
/* ------------------------------------------------------------------------- */

typedef struct {
    float *g, *h, *open, *hist, *parents, *v;
    int goal, start, solved_at;
} lit_map_t;

/* one loop iteration of differentiable_astar.py:206-249 for one map; returns 1 if
 * this map is "unsolved" after the step (is_unsolved, :220). */
static int literal_step(lit_map_t *m, const float *cost, const float *obst, const float *goalmap,
                        int H, int W, int nmoves, float gr, float omg, float sqrtw, int t, int32_t *trace_out)
{
    const int N = H * W;
    float s = 0.0f;
    for (int i = 0; i < N; ++i) {
        float a = gr * m->g[i];
        float b = omg * m->h[i];
        float f = a + b;                           /* :206 */
        float e = expf((-1.0f * f) / sqrtw);       /* :207 */
        m->v[i] = e * m->open[i];                  /* :208 */
        s += m->v[i];
    }
    for (int i = 0; i < N; ++i) m->v[i] = m->v[i] / s; /* :68 */
    const int ind = argmax_first(m->v, N);             /* :69 */
    if (trace_out) *trace_out = ind;
    /* forward value of (y_hard - y).detach() + y is exactly one-hot (SURVEY App. A.2) */
    const float dist_to_goal = goalmap[ind];           /* :219 sum(sel*goal) */
    const float unsolved = (dist_to_goal < 1e-8f) ? 1.0f : 0.0f;
    if (unsolved == 0.0f && m->solved_at < 0) m->solved_at = t;
    /* :222-225 */
    m->hist[ind] = fminf(fmaxf(m->hist[ind] + 1.0f, 0.0f), 1.0f);
    m->open[ind] = fminf(fmaxf(m->open[ind] - unsolved * 1.0f, 0.0f), 1.0f);
    /* :228-249 — only the neighbours of ind under the filter have neighbor_nodes != 0 */
    const int r = ind / W, c = ind % W;
    const float g2 = m->g[ind] + cost[ind];            /* :234 (g+cost)*sel through the stencil */
    for (int k = 0; k < nmoves; ++k) {
        int y = r + kDy[k], x = c + kDx[k];
        if (y < 0 || y >= H || x < 0 || x >= W) continue; /* zero padding, :91 */
        int n = y * W + x;
        float nbr = 1.0f * obst[n];                /* :229 */
        float gt = (m->g[n] > g2) ? 1.0f : 0.0f;
        float idx = ((1.0f - m->open[n]) * (1.0f - m->hist[n]) + m->open[n] * gt) * nbr; /* :235-236 */
        m->g[n] = g2 * idx + m->g[n] * (1.0f - idx);                  /* :238 */
        m->open[n] = fminf(fmaxf(m->open[n] + idx, 0.0f), 1.0f);     /* :242 */
        m->parents[n] = (float)ind * idx + m->parents[n] * (1.0f - idx); /* :249 */
    }
    return unsolved != 0.0f;
}

/* differentiable_astar.py:96-125 */
static void backtrack_literal(const float *parents, int goal, int N, int current_t, int64_t *path)
{
    for (int i = 0; i < N; ++i) path[i] = 0;
    path[goal] = 1;
    long loc = (long)parents[goal];
    for (int k = 0; k < current_t; ++k) {
        path[loc] = 1;
        loc = (long)parents[loc];
    }
}

/*
 * Batch-coupled literal forward.  Planes are [B][H*W] contiguous fp32.
 * T = number of loop iterations allowed (int(Tmax_eff*W*W), :200-202).
 * Outputs: hist [B][N] fp32, paths [B][N] int64, t_solve [B] (first step the goal was
 * selected, -1 if never), trace [B][T] int32 selected index per executed step (or NULL),
 * *T_batch = number of executed loop iterations.  mech: NASTAR_MECH_MOORE or NASTAR_MECH_NEWS.
 */
int nastar_oracle_forward_literal(const float *cost, const float *start, const float *goal,
                                  const float *obst, int B, int H, int W, float g_ratio,
                                  float one_minus_g_ratio, float sqrt_w, int T,
                                  float *hist, int64_t *paths, int32_t *t_solve, int32_t *trace,
                                  int32_t *T_batch, int mech)
{
    if (B <= 0 || H <= 0 || W <= 0 || T <= 0 || !mech_ok(mech)) return NASTAR_ORACLE_EINVAL;
    const int N = H * W, nm = num_moves(mech);
    lit_map_t *maps = (lit_map_t *)calloc((size_t)B, sizeof(lit_map_t));
    float *pool = (float *)calloc((size_t)B * N * 6, sizeof(float));
    for (int b = 0; b < B; ++b) {
        lit_map_t *m = &maps[b];
        float *p = pool + (size_t)b * N * 6;
        m->g = p; m->h = p + N; m->open = p + 2 * N; m->hist = p + 3 * N;
        m->parents = p + 4 * N; m->v = p + 5 * N;
        m->goal = argmax_first(goal + (size_t)b * N, N);   /* :197 */
        m->start = argmax_first(start + (size_t)b * N, N);
        m->solved_at = -1;
        heuristic_plus_cost(cost + (size_t)b * N, H, W, m->goal, mech, m->h); /* :191-192 */
        memcpy(m->open, start + (size_t)b * N, sizeof(float) * N);       /* :187 */
        for (int i = 0; i < N; ++i) m->parents[i] = (float)m->goal;      /* :195-198 */
    }
    int tb = 0;
    if (g_ratio >= 0.5f) {
        /* The reference runs one loop over t for the whole batch and stops when every map is solved
         * (:251-252).  For g_ratio >= 0.5 a solved map keeps re-selecting its goal (SURVEY App. A.4), so
         * maps only interact through the stop step: phase 1 runs each map to its own solve step, T_batch
         * is the maximum, phase 2 replays the post-solve iterations each map would still have executed.
         * (No barrier per step: needed for sane OpenMP scaling of the CPU baseline.) */
        int32_t *done = (int32_t *)calloc((size_t)B, sizeof(int32_t));
#pragma omp parallel for schedule(dynamic, 1)
        for (int b = 0; b < B; ++b) {
            int t = 0;
            for (t = 0; t < T; ++t) {
                int uns = literal_step(&maps[b], cost + (size_t)b * N, obst + (size_t)b * N, goal + (size_t)b * N,
                                       H, W, nm, g_ratio, one_minus_g_ratio, sqrt_w, t,
                                       trace ? trace + (size_t)b * T + t : NULL);
                if (!uns) { ++t; break; }
            }
            done[b] = t; /* iterations executed so far */
        }
        for (int b = 0; b < B; ++b) if (done[b] > tb) tb = done[b];
#pragma omp parallel for schedule(dynamic, 1)
        for (int b = 0; b < B; ++b) {
            for (int t = done[b]; t < tb; ++t)
                literal_step(&maps[b], cost + (size_t)b * N, obst + (size_t)b * N, goal + (size_t)b * N, H, W, nm,
                             g_ratio, one_minus_g_ratio, sqrt_w, t, trace ? trace + (size_t)b * T + t : NULL);
        }
        free(done);
    } else {
        /* g_ratio < 0.5: a solved map may select other nodes again, so the loop is run in lock step and
         * stops at the first iteration in which EVERY map selects its goal (:219-220, :251-252). */
        for (int t = 0; t < T; ++t) {
            int any_unsolved = 0;
#pragma omp parallel for schedule(static) reduction(| : any_unsolved)
            for (int b = 0; b < B; ++b)
                any_unsolved |= literal_step(&maps[b], cost + (size_t)b * N, obst + (size_t)b * N,
                                             goal + (size_t)b * N, H, W, nm, g_ratio, one_minus_g_ratio, sqrt_w, t,
                                             trace ? trace + (size_t)b * T + t : NULL);
            tb = t + 1;
            if (!any_unsolved) break;
        }
    }
    const int last_t = tb - 1;
    for (int b = 0; b < B; ++b) {
        memcpy(hist + (size_t)b * N, maps[b].hist, sizeof(float) * N);
        backtrack_literal(maps[b].parents, maps[b].goal, N, last_t, paths + (size_t)b * N); /* :255 */
        if (t_solve) t_solve[b] = maps[b].solved_at;
    }
    if (T_batch) *T_batch = last_t + 1;
    free(pool);
    free(maps);
    return NASTAR_ORACLE_OK;
}

/* ------------------------------------------------------------------------- */
/* SPEC restatement (SURVEY.md App. A.2): what the CUDA engine must reproduce */
/* ------------------------------------------------------------------------- */

typedef struct {
    float *g, *h;
    uint8_t *open, *closed;
    int32_t *parent;
} spec_map_t;

static inline float spec_f(float gr, float omg, float g, float h)
{
    float a = gr * g, b = omg * h;
    return a + b;
}

/* arg-min of (f, flat index) over the open set; -1 if the open set is empty */
static int spec_select(const spec_map_t *m, int N, float gr, float omg)
{
    int best = -1;
    float bf = 0.0f;
    for (int i = 0; i < N; ++i) {
        if (!m->open[i]) continue;
        float f = spec_f(gr, omg, m->g[i], m->h[i]);
        if (best < 0 || f < bf) { best = i; bf = f; }
    }
    return best;
}

static void spec_expand(spec_map_t *m, const float *cost, const float *obst, int H, int W, int nmoves, int ind)
{
    const int r = ind / W, c = ind % W;
    const float g2 = m->g[ind] + cost[ind];
    for (int k = 0; k < nmoves; ++k) {
        int y = r + kDy[k], x = c + kDx[k];
        if (y < 0 || y >= H || x < 0 || x >= W) continue;
        int n = y * W + x;
        if (obst[n] == 0.0f) continue;
        int upd = (!m->open[n] && !m->closed[n]) || (m->open[n] && m->g[n] > g2);
        if (upd) { m->g[n] = g2; m->open[n] = 1; m->parent[n] = ind; }
    }
}

/*
 * Per-map forward with early exit.  Same plane layout as the literal form.
 * t_solve[b]: step at which the goal was selected; -1 = step cap T reached;
 * -2 = open set exhausted (goal unreachable; the reference crashes there).
 * n_steps[b]: executed selection steps.  trace [B][T] optional.
 */
int nastar_oracle_forward_spec(const float *cost, const float *start, const float *goal,
                               const float *obst, int B, int H, int W, float g_ratio,
                               float one_minus_g_ratio, int T, int no_early_exit, float *hist, int64_t *paths,
                               int32_t *t_solve, int32_t *n_steps, int32_t *trace, int mech)
{
    if (B <= 0 || H <= 0 || W <= 0 || T <= 0 || !mech_ok(mech)) return NASTAR_ORACLE_EINVAL;
    const int N = H * W, nm = num_moves(mech);
#pragma omp parallel for schedule(dynamic, 1)
    for (int b = 0; b < B; ++b) {
        spec_map_t m;
        m.g = (float *)calloc((size_t)N, sizeof(float));
        m.h = (float *)malloc(sizeof(float) * N);
        m.open = (uint8_t *)calloc((size_t)N, 1);
        m.closed = (uint8_t *)calloc((size_t)N, 1);
        m.parent = (int32_t *)malloc(sizeof(int32_t) * N);
        const float *cb = cost + (size_t)b * N, *ob = obst + (size_t)b * N;
        const int gi = argmax_first(goal + (size_t)b * N, N);
        const int si = argmax_first(start + (size_t)b * N, N);
        heuristic_plus_cost(cb, H, W, gi, mech, m.h);
        for (int i = 0; i < N; ++i) m.parent[i] = gi;
        m.open[si] = 1;
        int ts = -1, steps = 0;
        for (int t = 0; t < T; ++t) {
            int ind = spec_select(&m, N, g_ratio, one_minus_g_ratio);
            if (ind < 0) { ts = -2; break; }
            if (trace) trace[(size_t)b * T + t] = ind;
            steps = t + 1;
            m.closed[ind] = 1;
            if (ind != gi) m.open[ind] = 0;       /* the goal, once selected, stays open */
            spec_expand(&m, cb, ob, H, W, nm, ind);
            if (ind == gi && ts < 0) ts = t;
            if (ind == gi && !no_early_exit) break;   /* no_early_exit: exactly T steps, like the batch loop */
        }
        float *hb = hist + (size_t)b * N;
        int64_t *pb = paths + (size_t)b * N;
        for (int i = 0; i < N; ++i) { hb[i] = m.closed[i] ? 1.0f : 0.0f; pb[i] = 0; }
        /* backtrack (App. A.3): solved -> walk to the start; capped -> at most T-1 hops */
        pb[gi] = 1;
        {
            int loc = m.parent[gi];
            int hops = (ts >= 0) ? N : (T - 1);
            for (int k = 0; k < hops; ++k) {
                pb[loc] = 1;
                if (ts >= 0 && loc == si) break;
                loc = m.parent[loc];
            }
        }
        if (t_solve) t_solve[b] = ts;
        if (n_steps) n_steps[b] = steps;
        free(m.g); free(m.h); free(m.open); free(m.closed); free(m.parent);
    }
    return NASTAR_ORACLE_OK;
}

/*
 * Closed-form backward (SURVEY.md App. B), replaying the SPEC state machine with the
 * reference's post-solve semantics for exactly T_batch steps per map:
 *   dL/dcost[p] = sum_t  -(1-g_ratio)/sqrt_w * y_t[p] * ( Gh[p] - <Gh, y_t> )
 * with y_t = softmax over the open set of -f/sqrt_w and Gh = G with the goal cell zeroed
 * when the map was solved before step T_batch-1 (clamp blocks the gradient there,
 * differentiable_astar.py:222-223).  Accumulation and output in double: the caller rounds once.
 *
 * backward_map() does one map.  bound == NULL is nastar_oracle_backward's arithmetic exactly; otherwise it also
 * writes the per-cell bound M of nastar_oracle_backward_bound (derivation there), and model != 0 computes the
 * softmax numerators as the engines do, v = expf(fl32(-f / sqrt_w)) in fp32, instead of in double.
 */
static void backward_map(const float *cb, const float *sb, const float *gb, const float *ob, const float *G,
                         int H, int W, int mech, float g_ratio, float one_minus_g_ratio, float sqrt_w, int T_batch,
                         int model, double *out, double *bound)
{
    const int N = H * W, nm = num_moves(mech);
    spec_map_t m;
    m.g = (float *)calloc((size_t)N, sizeof(float));
    m.h = (float *)malloc(sizeof(float) * N);
    m.open = (uint8_t *)calloc((size_t)N, 1);
    m.closed = (uint8_t *)calloc((size_t)N, 1);
    m.parent = (int32_t *)malloc(sizeof(int32_t) * N);
    double *acc_y = (double *)calloc((size_t)N, sizeof(double));   /* sum_t y_t[p] */
    double *acc_yd = (double *)calloc((size_t)N, sizeof(double));  /* sum_t y_t[p]*<G,y_t> (goal-free part) */
    double *acc_yg = (double *)calloc((size_t)N, sizeof(double));  /* sum_t y_t[p]*y_t[goal] */
    double *y = (double *)malloc(sizeof(double) * N);
    /* bound only: exact softmax ye, relative numerator error e, and M under both goal hypotheses (Gg = G[goal] or 0;
     * which one holds is known only after the last step) */
    double *ye = NULL, *e = NULL, *Mh = NULL;
    if (bound) {
        ye = (double *)malloc(sizeof(double) * N);
        e = (double *)calloc((size_t)N, sizeof(double));
        Mh = (double *)calloc((size_t)N * 2, sizeof(double));
    }
    const int gi = argmax_first(gb, N);
    const int si = argmax_first(sb, N);
    heuristic_plus_cost(cb, H, W, gi, mech, m.h);
    m.open[si] = 1;
    int blocked_goal = 0;
    for (int t = 0; t < T_batch; ++t) {
        /* softmax over the open set */
        double s = 0.0, se = 0.0;
        int ind = -1;
        float bf = 0.0f;
        for (int i = 0; i < N; ++i) {
            y[i] = 0.0;
            if (bound) ye[i] = 0.0;
            if (!m.open[i]) continue;
            float f = spec_f(g_ratio, one_minus_g_ratio, m.g[i], m.h[i]);
            if (ind < 0 || f < bf) { ind = i; bf = f; }
            const double v = exp(-(double)f / (double)sqrt_w);
            y[i] = model ? (double)expf((-f) / sqrt_w) : v;
            s += y[i];
            if (bound) {
                const double x = fabs((double)((-f) / sqrt_w));   /* the engines' rounded quotient */
                ye[i] = v;
                se += v;
                e[i] = (x > 128.0) ? 0x1p-147 / v
                                   : 0x1p-24 * x * (1.0 + 0x1p-17) + (1.0 + 0x1p-16) * fmax(0x1p-22, 0x1p-148 / v);
            }
        }
        if (ind < 0) break;
        double dot_nogoal = 0.0;
        for (int i = 0; i < N; ++i) {
            y[i] /= s;
            if (i != gi) dot_nogoal += (double)G[i] * y[i];
        }
        for (int i = 0; i < N; ++i) {
            acc_y[i] += y[i];
            acc_yd[i] += y[i] * dot_nogoal;
            acc_yg[i] += y[i] * y[gi];
        }
        if (bound) {
            double eb = 0.0, d0 = 0.0;   /* e-bar_t = sum y e; the goal-free parts of d_t and a_t */
            for (int i = 0; i < N; ++i) {
                if (ye[i] == 0.0) continue;
                ye[i] /= se;
                eb += ye[i] * e[i];
                if (i != gi) d0 += (double)G[i] * ye[i];
            }
            double a0 = 0.0;
            for (int i = 0; i < N; ++i)
                if (ye[i] != 0.0 && i != gi) a0 += fabs((double)G[i]) * ye[i] * (e[i] + eb);
            const double inv = 1.0 / (1.0 - eb);
            for (int k = 0; k < 2; ++k) {
                const double Gg = k ? 0.0 : (double)G[gi];
                const double d = d0 + Gg * ye[gi];
                const double a = a0 + ((ye[gi] != 0.0) ? fabs(Gg) * ye[gi] * (e[gi] + eb) : 0.0);
                double *M = Mh + (size_t)k * N;
                for (int i = 0; i < N; ++i) {
                    if (ye[i] == 0.0) continue;
                    const double Gi = (i == gi) ? Gg : (double)G[i];
                    M[i] += (eb < 1.0) ? ye[i] * inv * ((e[i] + eb) * fabs(Gi - d) + (1.0 + e[i]) * a * inv) : INFINITY;
                }
            }
        }
        if (m.closed[ind]) blocked_goal = 1;   /* hist+sel == 2 before the clamp */
        m.closed[ind] = 1;
        if (ind != gi) m.open[ind] = 0;
        spec_expand(&m, cb, ob, H, W, nm, ind);
    }
    const double Gg = blocked_goal ? 0.0 : (double)G[gi];
    const double coef = -(double)one_minus_g_ratio / (double)sqrt_w;
    for (int i = 0; i < N; ++i) {
        double Gi = (i == gi) ? Gg : (double)G[i];
        out[i] = coef * (acc_y[i] * Gi - acc_yd[i] - acc_yg[i] * Gg);
    }
    if (bound) {
        const double *M = Mh + (size_t)blocked_goal * N;
        for (int i = 0; i < N; ++i) {
            const double m0 = fabs(coef) * M[i];
            bound[i] = m0 + 0x1p-24 * (fabs(out[i]) + m0) + 0x1p-150;   /* + the fp32 rounding of the output */
        }
        free(ye); free(e); free(Mh);
    }
    free(m.g); free(m.h); free(m.open); free(m.closed); free(m.parent);
    free(acc_y); free(acc_yd); free(acc_yg); free(y);
}

int nastar_oracle_backward(const float *cost, const float *start, const float *goal,
                           const float *obst, const float *grad_hist, int B, int H, int W,
                           float g_ratio, float one_minus_g_ratio, float sqrt_w, int T_batch,
                           double *grad_cost, int mech)
{
    if (B <= 0 || H <= 0 || W <= 0 || T_batch <= 0 || !mech_ok(mech)) return NASTAR_ORACLE_EINVAL;
    const size_t N = (size_t)H * W;
#pragma omp parallel for schedule(dynamic, 1)
    for (int b = 0; b < B; ++b)
        backward_map(cost + b * N, start + b * N, goal + b * N, obst + b * N, grad_hist + b * N, H, W, mech,
                     g_ratio, one_minus_g_ratio, sqrt_w, T_batch, 0, grad_cost + b * N, NULL);
    return NASTAR_ORACLE_OK;
}

/*
 * The closed form of nastar_oracle_backward (model == 0) or of the engines' rounding (model != 0, see backward_map),
 * and next to it a per-cell bound M on how far an engine's fp32 gradient may lie from the fp64 closed form.
 *
 * The engines' only unavoidable deviation is the fp32 rounding of each softmax numerator.  They use the same fp32 f
 * and sqrt_w as this oracle and compute v'_q = expf(fl32(-f_q / sqrt_w)).  With x_q = f_q / sqrt_w, |delta| <= 2^-24
 * the quotient's rounding, u = |x_q| 2^-24 and |eta| <= the error of expf:
 *   |v'_q / v_q - 1| = |e^(-x_q delta) (1 + eta) - 1| <= (e^u - 1) + e^u |eta|
 *                   <= u (1 + 2^-17) + (1 + 2^-16) |eta|                 for |x_q| <= 128 (u <= 2^-17),
 * and |eta| <= max(2^-22, 2^-148 / v_q): expf is accurate to 2 ulp over its whole range (CUDA C++ Programming Guide,
 * "Mathematical Functions", single precision; the library is built without fast math, so subnormals are kept), which
 * is 2^-22 relative for a normal result and 2^-148 absolute for a subnormal result or one flushed to zero.  That sum
 * is e_q.  Beyond x_q = 128 (v_q < 2^-184) the quotient is above 127.99, so the result is 0 or a subnormal of at most
 * 2 ulp, |v'_q - v_q| <= 2^-148 + v_q <= 2^-147 and e_q = 2^-147 / v_q.
 * S' = sum v'_q is exact in the engines (a double-double sum of fp32 values), so with e-bar_t = sum_q y_q e_q:
 *   |y'_p - y_p| <= y_p (e_p + e-bar_t) / (1 - e-bar_t),   y'_p <= y_p (1 + e_p) / (1 - e-bar_t),
 *   |d'_t - d_t| <= a_t / (1 - e-bar_t),   d_t = sum_q Gh_q y_q,   a_t = sum_q |Gh_q| y_q (e_q + e-bar_t),
 * and the step's term y'_p (Gh_p - d'_t) - y_p (Gh_p - d_t) = (y'_p - y_p)(Gh_p - d_t) - y'_p (d'_t - d_t) gives
 *   M0[p] = |coef| sum_t y_t[p] / (1 - e-bar_t) * [ (e_p + e-bar_t) |Gh_p - d_t| + (1 + e_p) a_t / (1 - e-bar_t) ].
 * The fp32 output adds at most 2^-24 |got| <= 2^-24 (|want| + M0), or 2^-150 below the normal range:
 *   M[p] = M0[p] + 2^-24 (|want_p| + M0[p]) + 2^-150.
 * e-bar_t >= 1 (every open numerator underflows in fp32) makes M infinite on that step's open cells.  The engines' fp64
 * arithmetic (prefix sums, events, the division by S) is left out of M on purpose: it is meant to be negligible, and
 * tests/test_grad_bound_cpu.py and the GPU tests check that claim.  M costs O(N) per step.
 * grad_cost and bound are [B][N] double.
 */
int nastar_oracle_backward_bound(const float *cost, const float *start, const float *goal,
                                 const float *obst, const float *grad_hist, int B, int H, int W,
                                 float g_ratio, float one_minus_g_ratio, float sqrt_w, int T_batch, int model,
                                 double *grad_cost, double *bound, int mech)
{
    if (B <= 0 || H <= 0 || W <= 0 || T_batch <= 0 || !mech_ok(mech) || !bound) return NASTAR_ORACLE_EINVAL;
    const size_t N = (size_t)H * W;
#pragma omp parallel for schedule(dynamic, 1)
    for (int b = 0; b < B; ++b)
        backward_map(cost + b * N, start + b * N, goal + b * N, obst + b * N, grad_hist + b * N, H, W, mech,
                     g_ratio, one_minus_g_ratio, sqrt_w, T_batch, model, grad_cost + b * N, bound + b * N);
    return NASTAR_ORACLE_OK;
}
