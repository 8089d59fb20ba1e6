/*
 * wlabels_oracle.c -- CPU oracle of the vertex-weighted shortest-path labels (TEST INFRASTRUCTURE ONLY; the product
 * package never links it).  Checks nastar_b200_weighted_labels (neural-astar_b200/csrc/nastar_wlabels.cuh), but is
 * written from the semantics (DESIGN.md §11), not from the kernel.  Moves are the 8 actions of Moore or the first 4
 * (N, E, W, S) of NEWS:
 *   cost-to-go  Dijkstra from the goal with a binary heap of (D, cell), lazy deletion.  Settling u relaxes every
 *               in-grid passable neighbour v != goal (the move v->u charges c[u]): fl(D[u] + c[u]).  Compiled with
 *               -ffp-contract=off on an SSE target, every float add is rounded once.  The fold x -> fl(x + c) is
 *               monotone and never decreases x for c >= 0, so this Dijkstra returns the least fold over all paths.
 *   hops        breadth-first search from the goal over optimal moves (fl(D[u] + c[u]) == D[v]).
 *   policy      for every reachable v != goal: the optimal moves into cells with hop one lower; the first of them.
 *   path        the roll-out of that first move from the start (at most H*W moves), start and goal included.
 * Status bits: 1 bad cost on the goal or a passable cell, 2 no goal, 4 a start that cannot reach the goal.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "nastar_b200.h"

static const int kDy[8] = {-1, 0, 0, +1, -1, -1, +1, +1};   /* N, E, W, S, NE, NW, SE, SW; NEWS takes the first 4 */
static const int kDx[8] = {0, +1, -1, 0, +1, -1, +1, -1};

typedef struct {
    float d;
    int32_t v;
} Item;

static void heap_push(Item *h, int *n, Item it) {
    int i = (*n)++;
    while (i > 0) {
        const int p = (i - 1) / 2;
        if (h[p].d < it.d || (h[p].d == it.d && h[p].v <= it.v)) break;
        h[i] = h[p];
        i = p;
    }
    h[i] = it;
}

static Item heap_pop(Item *h, int *n) {
    const Item top = h[0];
    const Item last = h[--(*n)];
    int i = 0;
    for (;;) {
        int c = 2 * i + 1;
        if (c >= *n) break;
        if (c + 1 < *n && (h[c + 1].d < h[c].d || (h[c + 1].d == h[c].d && h[c + 1].v < h[c].v))) ++c;
        if (last.d < h[c].d || (last.d == h[c].d && last.v <= h[c].v)) break;
        h[i] = h[c];
        i = c;
    }
    h[i] = last;
    return top;
}

typedef struct {
    const float *c;
    const uint8_t *pas;
    const float *D;
    const int32_t *hop;
    int H, W, goal, nmoves;
} Map;

/* the move v -> t is allowed: t on the grid and passable or the goal (v's own passability is the caller's) */
static int target(const Map *m, int v, int a) {
    const int y = v / m->W + kDy[a], x = v % m->W + kDx[a];
    if (y < 0 || y >= m->H || x < 0 || x >= m->W) return -1;
    const int t = y * m->W + x;
    return (t == m->goal || m->pas[t]) ? t : -1;
}

static unsigned policy(const Map *m, int v) {
    if (v == m->goal || m->hop[v] < 0) return 0;
    unsigned mask = 0;
    for (int a = 0; a < m->nmoves; ++a) {
        const int t = target(m, v, a);
        if (t >= 0 && m->hop[t] == m->hop[v] - 1 && m->D[t] + m->c[t] == m->D[v]) mask |= 1u << a;
    }
    return mask;
}

static int one_map(const float *c, const float *passable, int goal, const int32_t *start, int H, int W, int nmoves,
                   float *D,
                   uint8_t *pas, Item *heap, int32_t *queue, float *dists, int32_t *hop, uint8_t *act_mask,
                   int8_t *action, float *path, float *path_cost) {
    const int N = H * W;
    int status = 0;
    if (goal < 0 || goal >= N) {
        status |= 2;
        goal = -1;
    }
    for (int i = 0; i < N; ++i) {
        pas[i] = passable ? passable[i] != 0.0f : 1;
        if ((pas[i] || i == goal) && !(isfinite(c[i]) && c[i] >= 0.0f)) status |= 1;
        D[i] = INFINITY;
        hop[i] = -1;
    }
    Map m = {c, pas, D, hop, H, W, goal, nmoves};
    if (status == 0) {
        int n = 0;
        D[goal] = 0.0f;
        heap_push(heap, &n, (Item){0.0f, goal});
        while (n > 0) {
            const Item it = heap_pop(heap, &n);
            const int u = it.v;
            if (it.d != D[u]) continue;   /* stale entry */
            const float via = D[u] + c[u];
            const int uy = u / W, ux = u % W;
            for (int a = 0; a < nmoves; ++a) {   /* v = u - move(a): the cells whose move a enters u */
                const int vy = uy - kDy[a], vx = ux - kDx[a];
                if (vy < 0 || vy >= H || vx < 0 || vx >= W) continue;
                const int v = vy * W + vx;
                if (v == goal || !pas[v]) continue;
                if (via < D[v]) {
                    D[v] = via;
                    heap_push(heap, &n, (Item){via, v});
                }
            }
        }
        int head = 0, tail = 0;
        hop[goal] = 0;
        queue[tail++] = goal;
        while (head < tail) {
            const int u = queue[head++];
            const float via = D[u] + c[u];
            const int uy = u / W, ux = u % W;
            for (int a = 0; a < nmoves; ++a) {
                const int vy = uy - kDy[a], vx = ux - kDx[a];
                if (vy < 0 || vy >= H || vx < 0 || vx >= W) continue;
                const int v = vy * W + vx;
                if (v == goal || !pas[v] || hop[v] >= 0 || D[v] == INFINITY || via != D[v]) continue;
                hop[v] = hop[u] + 1;
                queue[tail++] = v;
            }
        }
    }
    for (int v = 0; v < N; ++v) {
        const unsigned mk = status == 0 ? policy(&m, v) : 0u;
        dists[v] = 0.0f - D[v];
        act_mask[v] = (uint8_t)mk;
        action[v] = mk ? (int8_t)__builtin_ctz(mk) : (int8_t)-1;
    }
    if (!start) return status;
    memset(path, 0, sizeof(float) * (size_t)N);
    *path_cost = INFINITY;
    const int s = *start;
    if (status != 0 || s < 0 || s >= N || D[s] == INFINITY) return status | 4;
    int v = s;
    path[v] = 1.0f;
    for (int k = 0; k < N && v != goal; ++k) {
        const unsigned mk = policy(&m, v);
        if (!mk) break;
        const int a = __builtin_ctz(mk);
        v = (v / W + kDy[a]) * W + v % W + kDx[a];
        path[v] = 1.0f;
    }
    if (v != goal) {   /* cannot happen: every policy move lowers hop by one */
        memset(path, 0, sizeof(float) * (size_t)N);
        return status | 4;
    }
    *path_cost = c[s] + D[s];
    return status;
}

/* cost, passable (or NULL): [B][H*W] fp32; goal_idx, start_idx (or NULL): [B]; outputs [B][H*W] (path_maps) and
 * [B] (path_costs, status); mech: NASTAR_MECH_MOORE or NASTAR_MECH_NEWS.  Returns 0, or 1 on bad arguments /
 * allocation failure. */
int nastar_oracle_weighted_labels(const float *cost, const float *passable, const int32_t *goal_idx,
                                  const int32_t *start_idx, int B, int H, int W, float *dists, int32_t *hops,
                                  uint8_t *act_mask, int8_t *action, float *path_maps, float *path_costs,
                                  int32_t *status, int mech) {
    if (!cost || !goal_idx || !dists || !hops || !act_mask || !action || !status || B <= 0 || H <= 0 || W <= 0)
        return 1;
    if (start_idx && (!path_maps || !path_costs)) return 1;
    if (mech != NASTAR_MECH_MOORE && mech != NASTAR_MECH_NEWS) return 1;
    const int64_t N = (int64_t)H * W;
    const int nmoves = mech == NASTAR_MECH_NEWS ? 4 : 8;
    int fail = 0;
#pragma omp parallel reduction(| : fail)
    {
        float *D = malloc(sizeof(float) * (size_t)N);
        uint8_t *pas = malloc((size_t)N);
        Item *heap = malloc(sizeof(Item) * (size_t)(8 * N + 1));
        int32_t *queue = malloc(sizeof(int32_t) * (size_t)N);
#pragma omp for schedule(dynamic, 4)
        for (int b = 0; b < B; ++b) {
            if (!D || !pas || !heap || !queue) {
                fail = 1;
                continue;
            }
            status[b] = one_map(cost + b * N, passable ? passable + b * N : NULL, goal_idx[b],
                                start_idx ? start_idx + b : NULL, H, W, nmoves, D, pas, heap, queue, dists + b * N,
                                hops + b * N, act_mask + b * N, action + b * N, start_idx ? path_maps + b * N : NULL,
                                start_idx ? path_costs + b : NULL);
        }
        free(D);
        free(pas);
        free(heap);
        free(queue);
    }
    return fail;
}
