// nastar_pq.cuh — the reference's heap A* (`pq_astar.solve_single`, use_differentiable_astar=False) on the GPU, with
// its cost convention, pqdict's heap order and its outputs (DESIGN.md §17).
//
// Per map, on fp32 planes with N = H*W cells and flat index i = y*W + x:
//   start / goal  the single non-zero cell of each plane (status 2 when a plane has 0 or >= 2 of them);
//   open list     a binary min-heap of (f, cell), start inserted with f = 0;
//   loop          pop the minimum (sel, f_sel), close sel, and for each neighbour nb in get_neighbor_indices' order
//                 W, E, N, S, NW, NE, SW, SE inside the grid with map[nb] == 1:
//                   f_new = ((f_sel - (1-g) h(sel)) + g c[nb]) + (1-g) h(nb),
//                   h(i)  = max(dx, dy) + 0.001 sqrt(dx^2 + dy^2),
//                 every operation one fp64 rounding (no FMA); insert nb if it is neither open nor closed, lower its key
//                 if open[nb] > f_new, and in both cases parent[nb] = sel.  Stop when the goal is closed (status 0) or
//                 the open list is empty (status 1: histories and paths all zero).
//   heap moves    pqdict 1.2.0 / heapq: insert appends and swims while f < f(parent); pop moves the last entry to the
//                 root and sinks it Floyd's way (hole to a leaf, taking the right child unless left < right, then a
//                 strict-< swim); a key update is _reheapify (a lowered key swims).  Ties are decided by exactly
//                 these moves.
// The reference expands the goal's neighbours before it tests `goal in close_list`; that expansion only touches open
// cells, never a parent on the goal's chain (every such cell is closed), so it is skipped here.
//
// One warp per map, persistent CTAs of one warp taking maps from an atomic counter.  Lanes 0..7 test one neighbour
// each (grid, passable, open / closed, f_new: reads only); lane 0 then applies the inserts and key decreases in
// neighbour order, since each moves heap entries the next one sees, and does the pops.  State per map, 20 B per cell:
// f by heap position (fp64), cell by heap position, heap position by cell (kNew / kClosed / position), parent.  It
// lives in dynamic shared memory when kShared, else in the CTA's slot of the global workspace.
#pragma once
#include <cstdint>

namespace nastar {

constexpr int kPqThreads = 32;
constexpr int kPqMaxCells = 1 << 20;
constexpr int kPqBytesPerCell = 20;
constexpr int32_t kPqNew = -1;
constexpr int32_t kPqClosed = -2;

constexpr int kPqSolved = 0;
constexpr int kPqNotFound = 1;
constexpr int kPqBadEnds = 2;

struct PqArgs {
    const float* cost;  int64_t cost_stride;
    const float* start; int64_t start_stride;
    const float* goal;  int64_t goal_stride;
    const float* map;   int64_t map_stride;
    int B, H, W;
    double g, omg;      // g_ratio and 1 - g_ratio, each one fp64 rounding
    float* histories;   // [B][N]
    int64_t* paths;     // [B][N]
    int32_t* status;    // [B]
    int32_t* expansions;// [B]
    int32_t* queue;     // zeroed before the launch
    unsigned char* slots;   // !kShared: gridDim.x slots of kPqBytesPerCell * N bytes, 8-byte aligned
    int64_t slot_stride;    // bytes from one slot to the next: a multiple of 8 (the fp64 f array leads each slot)
};

// h(i) of pq_astar.compute_chebyshev_distance: integer max(dx, dy) plus 0.001 * sqrt of the integer dx^2 + dy^2
__device__ __forceinline__ double pq_heur(int x, int y, int gx, int gy) {
    const int dx = abs(x - gx), dy = abs(y - gy);
    const double e = __dsqrt_rn(double(int64_t(dx) * dx + int64_t(dy) * dy));
    return __dadd_rn(double(max(dx, dy)), __dmul_rn(0.001, e));
}

struct PqHeap {
    double* f;       // [N] by heap position
    int32_t* cell;   // [N] by heap position
    int32_t* pos;    // [N] by cell: kPqNew, kPqClosed or the heap position
    int32_t* parent; // [N] by cell, -1 = none

    __device__ __forceinline__ void put(int p, int32_t c, double v) {
        f[p] = v;
        cell[p] = c;
        pos[c] = p;
    }
    // pqdict._swim: place (c, v) at hole p after moving parents down while v < f(parent), stopping at `top`
    __device__ void swim(int p, int32_t c, double v, int top = 0) {
        while (p > top) {
            const int q = (p - 1) >> 1;
            const double fq = f[q];
            if (!(v < fq)) break;
            put(p, cell[q], fq);
            p = q;
        }
        put(p, c, v);
    }
    // pqdict._sink on n entries: the hole at `top` goes down to a leaf along the smaller children (the right one unless
    // left < right), then (c, v) swims back up to `top`
    __device__ void sink(int top, int32_t c, double v, int n) {
        int p = top, ch = 2 * top + 1;
        while (ch < n) {
            const int o = ch + 1;
            if (o < n && !(f[ch] < f[o])) ch = o;
            put(p, cell[ch], f[ch]);
            p = ch;
            ch = 2 * p + 1;
        }
        swim(p, c, v, top);
    }
    // pqdict.popitem on n > 0 entries: returns the root, leaves n - 1
    __device__ int32_t pop(int n, double* f_out) {
        const int32_t root = cell[0];
        *f_out = f[0];
        if (n > 1) sink(0, cell[n - 1], f[n - 1], n - 1);
        return root;
    }
    // pqdict._reheapify after cell c at position p took priority v, on n entries.  A lowered key swims; the sink
    // branch is reached only when an earlier NaN priority left a child below its parent.
    __device__ void reheap(int p, int32_t c, double v, int n) {
        if (p > 0 && v < f[(p - 1) >> 1]) { swim(p, c, v); return; }
        int ch = 2 * p + 1;
        if (ch < n) {
            if (ch + 1 < n && !(f[ch] < f[ch + 1])) ++ch;
            if (f[ch] < v) { sink(p, c, v, n); return; }
        }
        put(p, c, v);
    }
};

template <bool kShared>
__global__ void __launch_bounds__(kPqThreads) pq_astar_kernel(const PqArgs a) {
    extern __shared__ __align__(16) unsigned char pq_smem[];
    const int lane = threadIdx.x;
    const int N = a.H * a.W;
    unsigned char* base = kShared ? pq_smem : a.slots + size_t(blockIdx.x) * size_t(a.slot_stride);
    PqHeap h;
    h.f = reinterpret_cast<double*>(base);
    h.cell = reinterpret_cast<int32_t*>(base + size_t(8) * N);
    h.pos = h.cell + N;
    h.parent = h.pos + N;

    for (;;) {
        int b = 0;
        if (lane == 0) b = atomicAdd(a.queue, 1);
        b = __shfl_sync(0xffffffffu, b, 0);
        if (b >= a.B) break;
        const float* cost = a.cost + b * a.cost_stride;
        const float* sm = a.start + b * a.start_stride;
        const float* gm = a.goal + b * a.goal_stride;
        const float* mp = a.map + b * a.map_stride;
        float* hist = a.histories + int64_t(b) * N;
        int64_t* path = a.paths + int64_t(b) * N;

        // start and goal: count the non-zero cells (NaN counts, as np.argwhere does) and keep one index of each
        int ns = 0, ng = 0, s = -1, t = -1;
        for (int i0 = 0; i0 < N; i0 += 32) {
            const int i = i0 + lane;
            const bool ps = i < N && sm[i] != 0.0f, pg = i < N && gm[i] != 0.0f;
            const unsigned bs = __ballot_sync(0xffffffffu, ps), bg = __ballot_sync(0xffffffffu, pg);
            if (bs) s = i0 + __ffs(bs) - 1;
            if (bg) t = i0 + __ffs(bg) - 1;
            ns += __popc(bs);
            ng += __popc(bg);
            if (i < N) h.pos[i] = kPqNew;
        }
        if (ns != 1 || ng != 1) {
            for (int i = lane; i < N; i += 32) { hist[i] = 0.0f; path[i] = 0; }
            if (lane == 0) { a.status[b] = kPqBadEnds; a.expansions[b] = 0; }
            __syncwarp();
            continue;
        }
        const int gx = t % a.W, gy = t / a.W;
        __syncwarp();
        if (lane == 0) {
            h.put(0, s, 0.0);
            h.parent[s] = -1;
        }
        int n = 1, pops = 0;
        bool solved = false;
        // nb of lane k < 8 for cell sel, or -1: get_neighbor_indices' order
        const int ddx = lane == 0 ? -1 : lane == 1 ? 1 : lane == 4 || lane == 6 ? -1 : lane == 5 || lane == 7 ? 1 : 0;
        const int ddy = lane == 2 || lane == 4 || lane == 5 ? -1 : lane == 3 || lane == 6 || lane == 7 ? 1 : 0;
        while (n > 0 && pops < N) {
            int32_t sel = 0;
            double fs = 0.0;
            if (lane == 0) {
                sel = h.pop(n, &fs);
                h.pos[sel] = kPqClosed;
            }
            --n;
            ++pops;
            sel = __shfl_sync(0xffffffffu, sel, 0);
            fs = __shfl_sync(0xffffffffu, fs, 0);
            if (sel == t) { solved = true; break; }
            __syncwarp();
            const int sx = sel % a.W, sy = sel / a.W;
            const int x = sx + ddx, y = sy + ddy;
            int act = 0;   // 1 insert, 2 lower the key
            int nb = -1;
            double fn = 0.0;
            if (lane < 8 && x >= 0 && x < a.W && y >= 0 && y < a.H) {
                nb = y * a.W + x;
                if (mp[nb] == 1.0f) {
                    const double base_f = __dsub_rn(fs, __dmul_rn(a.omg, pq_heur(sx, sy, gx, gy)));
                    fn = __dadd_rn(__dadd_rn(base_f, __dmul_rn(a.g, double(cost[nb]))),
                                   __dmul_rn(a.omg, pq_heur(x, y, gx, gy)));
                    const int32_t p = h.pos[nb];
                    if (p == kPqNew) act = 1;
                    else if (p >= 0 && h.f[p] > fn) act = 2;
                }
            }
            unsigned todo = __ballot_sync(0xffffffffu, act != 0);
            while (todo) {
                const int k = __ffs(todo) - 1;
                todo &= todo - 1;
                const int c = __shfl_sync(0xffffffffu, nb, k);
                const double v = __shfl_sync(0xffffffffu, fn, k);
                const int ak = __shfl_sync(0xffffffffu, act, k);
                if (lane == 0) {
                    if (ak == 1) h.swim(n, c, v);
                    else h.reheap(h.pos[c], c, v, n);   // positions may have moved since lane k read them
                    h.parent[c] = sel;
                }
                n += ak == 1;
            }
            __syncwarp();
        }
        if (lane == 0) {
            a.status[b] = solved ? kPqSolved : kPqNotFound;
            a.expansions[b] = pops;
        }
        __syncwarp();
        for (int i = lane; i < N; i += 32) {
            hist[i] = solved && h.pos[i] == kPqClosed ? 1.0f : 0.0f;
            path[i] = 0;
        }
        __syncwarp();
        if (solved && lane == 0) {
            int c = t;
            for (int k = 0; k < N && c >= 0; ++k) {   // the chain has at most N cells; the cap guards bad state
                path[c] = 1;
                c = h.parent[c];
            }
        }
        __syncwarp();
    }
}

}  // namespace nastar
