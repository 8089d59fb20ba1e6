/* pq_oracle.c — CPU restatement of the reference's heap A* (pq_astar.solve_single) with pqdict 1.2.0's heap moves.
 *
 * TEST / BASELINE INFRASTRUCTURE ONLY: the GPU kernel (csrc/nastar_pq.cuh) is checked against it in bulk and on
 * large maps, where the reference's Python loop would take minutes.  Written from the semantics in DESIGN.md §17, step
 * for step and in the reference's order: the goal's neighbours are expanded before the `goal in close_list` test, as
 * the reference does.  Built with -ffp-contract=off so every fp64 product and sum is rounded once, as NumPy does.
 *
 * Per map: status 0 solved, 1 goal not found (histories and paths zero), 2 start or goal not exactly one non-zero
 * cell (zero too).  Maps run in parallel (OpenMP), each on its own state.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { NEW = -1, CLOSED = -2 };

typedef struct {
    double *f;     /* by heap position */
    int32_t *cell; /* by heap position */
    int32_t *pos;  /* by cell: NEW, CLOSED or heap position */
    int n;
} heap_t;

static void put(heap_t *h, int p, int32_t c, double v) {
    h->f[p] = v;
    h->cell[p] = c;
    h->pos[c] = p;
}

/* pqdict._swim: move parents down while v < f(parent) */
static void swim(heap_t *h, int p, int32_t c, double v) {
    while (p > 0) {
        int q = (p - 1) >> 1;
        if (v < h->f[q]) {
            put(h, p, h->cell[q], h->f[q]);
            p = q;
            continue;
        }
        break;
    }
    put(h, p, c, v);
}

/* pqdict.additem */
static void additem(heap_t *h, int32_t c, double v) {
    h->n += 1;
    swim(h, h->n - 1, c, v);
}

/* pqdict._sink (Floyd): the hole at `top` goes down to a leaf along the right child unless left < right, then the
 * node swims back up, no further than `top` */
static void sink(heap_t *h, int top, int32_t c, double v) {
    int p = top, ch = 2 * top + 1;
    while (ch < h->n) {
        int o = ch + 1;
        if (o < h->n && !(h->f[ch] < h->f[o])) ch = o;
        put(h, p, h->cell[ch], h->f[ch]);
        p = ch;
        ch = 2 * p + 1;
    }
    while (p > top) {
        int q = (p - 1) >> 1;
        if (!(v < h->f[q])) break;
        put(h, p, h->cell[q], h->f[q]);
        p = q;
    }
    put(h, p, c, v);
}

/* pqdict.popitem: the last node to the root, then _sink */
static int32_t popitem(heap_t *h, double *f_out) {
    int32_t root = h->cell[0];
    *f_out = h->f[0];
    h->n -= 1;
    if (h->n > 0) sink(h, 0, h->cell[h->n], h->f[h->n]);
    return root;
}

/* pqdict.__setitem__ on a queued key -> _reheapify: swim below a larger parent, else sink above a smaller child */
static void reheapify(heap_t *h, int p, int32_t c, double v) {
    if (p > 0 && v < h->f[(p - 1) >> 1]) {
        swim(h, p, c, v);
        return;
    }
    int ch = 2 * p + 1;
    if (ch < h->n) {
        if (ch + 1 < h->n && !(h->f[ch] < h->f[ch + 1])) ++ch;
        if (h->f[ch] < v) {
            sink(h, p, c, v);
            return;
        }
    }
    put(h, p, c, v);
}

/* compute_chebyshev_distance */
static double heur(int i, int goal, int W) {
    int64_t dx = llabs((int64_t)(i % W) - goal % W), dy = llabs((int64_t)(i / W) - goal / W);
    int64_t m = dx > dy ? dx : dy;
    return (double)m + 0.001 * sqrt((double)(dx * dx + dy * dy));
}

static int solve_single(const float *cost, const float *sm, const float *gm, const float *mp, int H, int W, double g,
                        float *hist, int64_t *path, int32_t *expansions, heap_t *h, int32_t *parent) {
    const int N = H * W;
    int s = -1, t = -1, ns = 0, ng = 0;
    memset(hist, 0, sizeof(float) * (size_t)N);
    memset(path, 0, sizeof(int64_t) * (size_t)N);
    *expansions = 0;
    for (int i = 0; i < N; ++i) {
        if (sm[i] != 0.0f) { s = i; ++ns; }
        if (gm[i] != 0.0f) { t = i; ++ng; }
    }
    if (ns != 1 || ng != 1) return 2;
    const double omg = 1.0 - g;
    for (int i = 0; i < N; ++i) h->pos[i] = NEW;
    h->n = 0;
    additem(h, s, 0.0);
    parent[s] = -1;
    int steps = 0;
    while (h->pos[t] != CLOSED) {
        if (h->n == 0 || steps >= N) { *expansions = steps; return 1; }
        ++steps;
        double fs;
        const int sel = popitem(h, &fs);
        h->pos[sel] = CLOSED;
        const int x = sel % W, y = sel / W;
        int nbs[8], k = 0;
        if (x - 1 >= 0) nbs[k++] = sel - 1;
        if (x + 1 < W) nbs[k++] = sel + 1;
        if (y - 1 >= 0) nbs[k++] = sel - W;
        if (y + 1 < H) nbs[k++] = sel + W;
        if (x - 1 >= 0 && y - 1 >= 0) nbs[k++] = sel - W - 1;
        if (x + 1 < W && y - 1 >= 0) nbs[k++] = sel - W + 1;
        if (x - 1 >= 0 && y + 1 < H) nbs[k++] = sel + W - 1;
        if (x + 1 < W && y + 1 < H) nbs[k++] = sel + W + 1;
        for (int j = 0; j < k; ++j) {
            const int nb = nbs[j];
            if (!(mp[nb] == 1.0f)) continue;
            double f_new = fs - omg * heur(sel, t, W);
            f_new = f_new + g * (double)cost[nb];
            f_new = f_new + omg * heur(nb, t, W);
            const int32_t p = h->pos[nb];
            if (p == NEW) {
                additem(h, nb, f_new);
                parent[nb] = sel;
            } else if (p >= 0 && h->f[p] > f_new) {
                reheapify(h, p, nb, f_new);
                parent[nb] = sel;
            }
        }
    }
    *expansions = steps;
    for (int i = 0; i < N; ++i) hist[i] = h->pos[i] == CLOSED ? 1.0f : 0.0f;
    int c = t;
    for (int k = 0; k < N && c >= 0; ++k) {
        path[c] = 1;
        c = parent[c];
    }
    return 0;
}

/* Planes fp32 [B][H][W], contiguous.  Returns 0, or -1 when a work buffer cannot be allocated. */
int nastar_oracle_pq_astar(const float *cost, const float *start, const float *goal, const float *map, int B, int H,
                           int W, double g_ratio, float *histories, int64_t *paths, int32_t *status,
                           int32_t *expansions) {
    const int64_t N = (int64_t)H * W;
    int rc = 0;
#pragma omp parallel
    {
        heap_t h;
        h.f = malloc(sizeof(double) * (size_t)N);
        h.cell = malloc(sizeof(int32_t) * (size_t)N);
        h.pos = malloc(sizeof(int32_t) * (size_t)N);
        int32_t *parent = malloc(sizeof(int32_t) * (size_t)N);
        const int ok = h.f && h.cell && h.pos && parent;
#pragma omp for schedule(dynamic, 1)
        for (int b = 0; b < B; ++b) {
            if (!ok) {
#pragma omp atomic write
                rc = -1;
                continue;
            }
            status[b] = solve_single(cost + b * N, start + b * N, goal + b * N, map + b * N, H, W, g_ratio,
                                     histories + b * N, paths + b * N, expansions + b, &h, parent);
        }
        free(h.f);
        free(h.cell);
        free(h.pos);
        free(parent);
    }
    return rc;
}
