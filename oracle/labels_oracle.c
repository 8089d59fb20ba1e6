/*
 * labels_oracle.c -- CPU restatement of the planning-datasets label generator (TEST INFRASTRUCTURE ONLY; the
 * product package never links it).  Checks nastar_b200_opt_labels (neural-astar_b200/csrc/nastar_labels.cuh).
 *
 * Restates, for the Moore or NEWS mechanism with one orientation (planning-datasets/planning_datasets_utils/):
 *   dijkstra_dist   dijkstra.py:120-157  distances start at num_orient*H*W (:122-125); the goal is popped first with 0
 *                                        (:127-128); a popped cell relaxes the targets of invneighbors_func
 *                                        (mechanism.py:221-231) that lie on the grid and are passable,
 *                                        maze != 0.0 (:144-151), with cost +1 (:153-156); returns -dist (:157).
 *                                        Every step costs 1, so the heap order is a FIFO order: a breadth-first
 *                                        search from the goal gives the same distances.  A popped cell that was
 *                                        never reached carries H*W and relaxes nothing (H*W + 1 < H*W is false).
 *   extract_policy  data.py:40-58        for every cell (obstacles included) the values of the 8 neighbors_func
 *                                        targets, or the 4 of NEWS (mechanism.py:80-111, :166-219: a move off the
 *                                        grid or onto a cell whose value is 0.0 stays put) and the set of actions with the maximal value.
 *                                        The reference draws one member at random (:60); here the whole set is
 *                                        returned as a bit mask, plus its lowest member.
 */
#include <stdint.h>
#include <stdlib.h>

#include "nastar_b200.h"

/* mechanism.py:140-149: N, E, W, S, NE, NW, SE, SW; NEWS (mechanism.py:58) takes the first 4 */
static const int kDy[8] = {-1, 0, 0, +1, -1, -1, +1, +1};
static const int kDx[8] = {0, +1, -1, 0, +1, -1, +1, -1};

/* target of action a from (y, x) under the stay rule (mechanism.py:166-207) */
static int move(const float *maze, int H, int W, int y, int x, int a) {
    const int ty = y + kDy[a], tx = x + kDx[a];
    if (ty < 0 || ty >= H || tx < 0 || tx >= W || maze[ty * W + tx] == 0.0f) return y * W + x;
    return ty * W + tx;
}

static void one_map(const float *maze, int goal, int H, int W, int nmoves, int32_t *dist, int32_t *queue,
                    float *dists, uint8_t *act_mask, int8_t *action) {
    const int N = H * W;
    for (int i = 0; i < N; ++i) dist[i] = N;
    int head = 0, tail = 0;
    if (goal >= 0 && goal < N) {
        dist[goal] = 0;
        queue[tail++] = goal;
    }
    while (head < tail) {
        const int p = queue[head++];
        const int py = p / W, px = p - py * W;
        for (int a = 0; a < nmoves; ++a) {
            const int n = move(maze, H, W, py, px, a);
            if (n == p) continue;   /* off the grid or not passable: skipped by dijkstra.py:145-151 */
            if (dist[p] + 1 < dist[n]) {
                dist[n] = dist[p] + 1;
                queue[tail++] = n;
            }
        }
    }
    for (int i = 0; i < N; ++i) dists[i] = (float)(-dist[i]);
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            int best = 0;
            unsigned mask = 0;
            for (int a = 0; a < nmoves; ++a) {
                const int v = -dist[move(maze, H, W, y, x, a)];
                if (a == 0 || v > best) {
                    best = v;
                    mask = 1u << a;
                } else if (v == best) {
                    mask |= 1u << a;
                }
            }
            act_mask[y * W + x] = (uint8_t)mask;
            action[y * W + x] = (int8_t)__builtin_ctz(mask);
        }
}

/* maps: [B][H*W] fp32; goal_idx: [B]; outputs [B][H*W]; mech: NASTAR_MECH_MOORE or NASTAR_MECH_NEWS.  Returns 0,
 * or 1 on bad arguments / allocation failure. */
int nastar_oracle_opt_labels(const float *maps, const int32_t *goal_idx, int B, int H, int W, float *dists,
                             uint8_t *act_mask, int8_t *action, int mech) {
    if (!maps || !goal_idx || !dists || !act_mask || !action || B <= 0 || H <= 0 || W <= 0) return 1;
    if (mech != NASTAR_MECH_MOORE && mech != NASTAR_MECH_NEWS) return 1;
    const int64_t N = (int64_t)H * W;
    const int nmoves = mech == NASTAR_MECH_NEWS ? 4 : 8;
    int fail = 0;
#pragma omp parallel reduction(| : fail)
    {
        int32_t *dist = malloc(sizeof(int32_t) * (size_t)N);
        int32_t *queue = malloc(sizeof(int32_t) * (size_t)N);
#pragma omp for schedule(dynamic, 4)
        for (int b = 0; b < B; ++b) {
            if (!dist || !queue) {
                fail = 1;
                continue;
            }
            one_map(maps + b * N, goal_idx[b], H, W, nmoves, dist, queue, dists + b * N, act_mask + b * N, action + b * N);
        }
        free(dist);
        free(queue);
    }
    return fail;
}
