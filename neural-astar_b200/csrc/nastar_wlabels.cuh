// nastar_wlabels.cuh — exact vertex-weighted shortest paths for cost maps: optimal costs-to-go, hop counts, the
// optimal policy and optional optimal paths (the weighted counterpart of nastar_labels.cuh).
//
// Semantics, per map (DESIGN.md §11):
//   inputs   cost c fp32 [H,W]; passable (value != 0; no plane = every cell passable); a goal; optionally a start.
//   moves    actions 0..7 = N, E, W, S, NE, NW, SE, SW (the Moore mechanism of nastar_labels.cuh); a diagonal move
//            does not check the orthogonal cells; a move leaves a passable cell and enters an in-grid cell that is
//            passable or is the goal (the goal is always enterable and is the source).  kNews: actions 0..3 = N, E,
//            W, S only (the NEWS mechanism), everything below with "4 moves" for "8 moves".
//   D        cost-to-go: D[goal] = +0, D[v] = min over moves v->t of fl(D[t] + c[t]) (one __fadd_rn per move, no
//            contraction), +inf where the goal cannot be reached.  For c >= 0, x -> fl(x + c) is monotone and never
//            decreases x, so D is the minimum over all paths of the fp32 left fold from the goal: it does not depend
//            on the relaxation order, and a CPU Dijkstra with the same fold gives the same bits.  Stored negated
//            (0 at the goal, -inf where unreachable), like opt_dists.
//   optimal  a move v->t with fl(D[t] + c[t]) == D[v], v reachable and not the goal.  Tiny costs can be absorbed
//            (fl(D + c) == D) and zero costs make cycles of optimal moves, so a first-minimum rule alone could loop.
//   hop      hop[goal] = 0, hop[v] = 1 + min over v's optimal moves t of hop[t] (a BFS over optimal moves); -1 where
//            unreachable.  Finite for every reachable cell: Dijkstra's settling tree consists of optimal moves.
//   policy   act_mask bit a set iff action a is an optimal move into a cell with hop[t] == hop[v] - 1; action = the
//            lowest such bit, -1 (mask 0) at the goal and at unreachable cells.  Following `action` decreases hop by
//            one per move, so a roll-out reaches the goal after exactly hop[start] moves and its fold equals D[start].
//   path     (with a start) the roll-out's cells, start and goal included, as an fp32 mask; path_cost =
//            fl(c[start] + D[start]), the cost of every cell of the path; an unreachable start gives an empty mask
//            and +inf.
//   status   0, or an OR of: 1 the goal or a passable cell has a negative, NaN or infinite cost (every plane is then
//            filled as unreachable); 2 no goal (index outside [0, H*W)); 4 a start was given and cannot reach the goal.
//
// One CTA per map, one launch.  Everything lives in shared memory: D and c (fp32), hop (u16, exact since
// hop < H*W <= 16384), the passable bit plane and three rotating "changed" bit planes (u32 row words).
//   1. D: frontier Bellman-Ford.  A cell is re-evaluated only in the round after one of its 8 (kNews: 4) neighbours
//      changed; a cell that lowers its D marks itself and those neighbours in the next plane.  Updates are in place
//      (D only decreases and every value read is the fold of a real path, so a stale read is only a later
//      re-evaluation).  The loop ends
//      when a round changes nothing (__syncthreads_or); it is capped at H*W + 1 rounds (Bellman-Ford needs at most
//      H*W - 1), so input that skipped validation cannot hang the GPU.
//   2. hop: BFS wavefronts over the optimal-move relation, frontier-driven the same way, capped the same way.
//   3. one thread per cell writes dists, hops, act_mask and action.
//   4. (with a start) one thread walks the policy from the start (at most H*W moves) into a bit plane; then the whole
//      CTA writes the fp32 path plane from it, coalesced.
// Work items of phases 1-2 are 16-cell half row words, so the CTA has 2 * H * ceil(W/32) threads rounded up to a
// warp: one warp at 12x12, 1024 threads at 128x128.
//
// Limits: H, W <= 128 (so H*W <= 16384): 8*N + 2*N + 16*H*ceil(W/32) bytes of shared memory, 168 KB at 128x128.
#pragma once
#include <cstdint>

namespace nastar {

constexpr int kWLabelsMaxSide = 128;
constexpr int kWLabelsMaxCells = 16384;
constexpr int kWLabelsMaxThreads = 1024;
constexpr uint16_t kHopUnset = 0xFFFFu;
// (dy + 1, dx + 1) of action a in bits 2a..2a+1, for a move chosen at run time
constexpr uint32_t kWLMoveDy = 0xa094u, kWLMoveDx = 0x2249u;

struct WLabelsArgs {
    const float* cost;        // [B] maps of H*W fp32 cells, cost_stride elements apart
    int64_t cost_stride;
    const float* passable;    // [B] maps, passable_stride apart; nullptr = every cell passable
    int64_t passable_stride;
    const int32_t* goal_idx;  // [B] flat goal index y*W+x
    const int32_t* start_idx; // [B] flat start index, or nullptr (no paths)
    int B, H, W;
    float* dists;             // [B][H*W]  -D
    int32_t* hops;            // [B][H*W]
    uint8_t* act_mask;        // [B][H*W]
    int8_t* action;           // [B][H*W]
    float* path_maps;         // [B][H*W]  with start_idx
    float* path_costs;        // [B]       with start_idx
    int32_t* status;          // [B]
};

inline int wlabels_words(int H, int W) { return H * ((W + 31) >> 5); }
inline size_t wlabels_smem_bytes(int H, int W) {
    const size_t N = size_t(H) * W;
    return 8 * N + 2 * ((N + 1) & ~size_t(1)) + 16 * size_t(wlabels_words(H, W));
}
inline int wlabels_threads(int H, int W) {
    const int t = (2 * wlabels_words(H, W) + 31) & ~31;
    return t < 32 ? 32 : (t > kWLabelsMaxThreads ? kWLabelsMaxThreads : t);
}

struct WLMap {
    float* D;
    const float* C;
    uint16_t* hop;
    const uint32_t* pas;
    int H, W, nw, goal;

    __device__ bool enterable(int ty, int tx) const {
        const int t = ty * W + tx;
        return t == goal || ((pas[ty * nw + (tx >> 5)] >> (tx & 31)) & 1u);
    }
    // bit a set iff action a is an optimal move from v = (y, x) into a cell one hop closer to the goal
    template <bool kNews>
    __device__ uint32_t policy_mask(int y, int x) const {
        const int v = y * W + x;
        const int hv = hop[v];
        if (v == goal || hv == kHopUnset) return 0u;
        const float dv = D[v];
        constexpr int dys[8] = {-1, 0, 0, +1, -1, -1, +1, +1};
        constexpr int dxs[8] = {0, +1, -1, 0, +1, -1, +1, -1};
        uint32_t m = 0;
#pragma unroll
        for (int a = 0; a < (kNews ? 4 : 8); ++a) {
            const int ty = y + dys[a], tx = x + dxs[a];
            if (ty < 0 || ty >= H || tx < 0 || tx >= W || !enterable(ty, tx)) continue;
            const int t = ty * W + tx;
            if (int(hop[t]) == hv - 1 && __fadd_rn(D[t], C[t]) == dv) m |= 1u << a;
        }
        return m;
    }
};

// mark the 3x3 block around (y, x) in a row-word bit plane; kNews: (y, x) and its 4 neighbours only
template <bool kNews>
__device__ __forceinline__ void wl_mark(uint32_t* plane, int nw, int H, int W, int y, int x) {
    const int lo = x > 0 ? x - 1 : 0, hi = x + 1 < W ? x + 1 : W - 1;
    const int wl = lo >> 5, wh = hi >> 5;
    for (int yy = y - 1; yy <= y + 1; ++yy) {
        if (yy < 0 || yy >= H) continue;
        uint32_t* row = plane + yy * nw;
        if (kNews && yy != y) {
            atomicOr(row + (x >> 5), 1u << (x & 31));
        } else if (wl == wh) {
            atomicOr(row + wl, ((2u << (hi - lo)) - 1u) << (lo & 31));
        } else {
            atomicOr(row + wl, ~0u << (lo & 31));
            atomicOr(row + wh, (2u << (hi & 31)) - 1u);
        }
    }
}

template <bool kNews>
__global__ void __launch_bounds__(kWLabelsMaxThreads) weighted_labels_kernel(WLabelsArgs a) {
    extern __shared__ __align__(16) unsigned char wl_smem[];
    const int H = a.H, W = a.W, N = H * W, nw = (W + 31) >> 5, nwords = H * nw, nseg = 2 * nwords;
    float* D = reinterpret_cast<float*>(wl_smem);
    float* C = D + N;
    uint16_t* hop = reinterpret_cast<uint16_t*>(C + N);
    uint32_t* pas = reinterpret_cast<uint32_t*>(hop + ((N + 1) & ~1));
    uint32_t* P0 = pas + nwords;
    uint32_t* P1 = P0 + nwords;
    uint32_t* P2 = P1 + nwords;
    const int b = blockIdx.x, tid = threadIdx.x, nthr = blockDim.x;
    const int lane = tid & 31, warp = tid >> 5, nwarp = nthr >> 5;
    const float kInf = __int_as_float(0x7f800000);
    const float* cost = a.cost + int64_t(b) * a.cost_stride;
    const float* pmap = a.passable ? a.passable + int64_t(b) * a.passable_stride : nullptr;

    int status = 0;
    int goal = a.goal_idx[b];
    if (goal < 0 || goal >= N) {
        goal = -1;
        status |= 2;
    }

    // load: a warp per row word, a lane per cell; passability by ballot; validate the costs that can be charged
    int bad = 0;
    for (int i = warp; i < nwords; i += nwarp) {
        const int y = i / nw, x = (i - y * nw) * 32 + lane;
        bool p = false;
        if (x < W) {
            const int c = y * W + x;
            const float cv = cost[c];
            p = pmap ? pmap[c] != 0.0f : true;
            C[c] = cv;
            D[c] = kInf;
            hop[c] = kHopUnset;
            if ((p || c == goal) && !(cv >= 0.0f && cv <= 3.402823466e38f)) bad = 1;
        }
        const uint32_t bits = __ballot_sync(0xFFFFFFFFu, p);
        if (lane == 0) {
            pas[i] = bits;
            P0[i] = 0u;
            P1[i] = 0u;
            P2[i] = 0u;
        }
    }
    if (__syncthreads_or(bad)) status |= 1;
    const bool ok = status == 0;   // block-uniform
    const WLMap m{D, C, hop, pas, H, W, nw, goal};
    constexpr int dys[8] = {-1, 0, 0, +1, -1, -1, +1, +1};
    constexpr int dxs[8] = {0, +1, -1, 0, +1, -1, +1, -1};
    constexpr int kMoves = kNews ? 4 : 8;   // the first 4 actions are N, E, W, S
    const int gy = ok ? goal / W : 0, gx = ok ? goal - gy * W : 0;

    if (ok) {
        if (tid == 0) {
            D[goal] = 0.0f;
            hop[goal] = 0;
            wl_mark<kNews>(P0, nw, H, W, gy, gx);
        }
        __syncthreads();
        // 1. cost-to-go
        uint32_t *cur = P0, *nxt = P1, *zro = P2;
        for (int r = 0; r <= N; ++r) {
            int any = 0;
            for (int i = tid; i < nwords; i += nthr) zro[i] = 0u;
            for (int s = tid; s < nseg; s += nthr) {
                const int wi = s >> 1;
                uint32_t cand = cur[wi] & pas[wi] & ((s & 1) ? 0xFFFF0000u : 0x0000FFFFu);
                if (!cand) continue;
                const int y = wi / nw, x0 = (wi - y * nw) * 32;
                while (cand) {
                    const int x = x0 + __ffs(cand) - 1;
                    cand &= cand - 1;
                    const int v = y * W + x;
                    if (v == goal) continue;
                    const float dv = D[v];
                    float best = dv;
#pragma unroll
                    for (int k = 0; k < kMoves; ++k) {
                        const int ty = y + dys[k], tx = x + dxs[k];
                        if (ty < 0 || ty >= H || tx < 0 || tx >= W || !m.enterable(ty, tx)) continue;
                        const int t = ty * W + tx;
                        const float nd = __fadd_rn(D[t], C[t]);
                        if (nd < best) best = nd;
                    }
                    if (best < dv) {
                        D[v] = best;
                        wl_mark<kNews>(nxt, nw, H, W, y, x);
                        any = 1;
                    }
                }
            }
            if (!__syncthreads_or(any)) break;
            uint32_t* t = cur;
            cur = nxt;
            nxt = zro;
            zro = t;
        }
        // 2. hops: wavefront k sets the cells with an optimal move into a cell of hop k - 1
        for (int i = tid; i < nwords; i += nthr) {
            P0[i] = 0u;
            P1[i] = 0u;
            P2[i] = 0u;
        }
        __syncthreads();
        if (tid == 0) wl_mark<kNews>(P0, nw, H, W, gy, gx);
        __syncthreads();
        cur = P0;
        nxt = P1;
        zro = P2;
        for (int k = 1; k <= N + 1; ++k) {
            int any = 0;
            for (int i = tid; i < nwords; i += nthr) zro[i] = 0u;
            for (int s = tid; s < nseg; s += nthr) {
                const int wi = s >> 1;
                uint32_t cand = cur[wi] & pas[wi] & ((s & 1) ? 0xFFFF0000u : 0x0000FFFFu);
                if (!cand) continue;
                const int y = wi / nw, x0 = (wi - y * nw) * 32;
                while (cand) {
                    const int x = x0 + __ffs(cand) - 1;
                    cand &= cand - 1;
                    const int v = y * W + x;
                    const float dv = D[v];
                    if (hop[v] != kHopUnset || dv == kInf) continue;   // the goal has hop 0
                    bool hit = false;
#pragma unroll
                    for (int q = 0; q < kMoves; ++q) {
                        const int ty = y + dys[q], tx = x + dxs[q];
                        if (ty < 0 || ty >= H || tx < 0 || tx >= W || !m.enterable(ty, tx)) continue;
                        const int t = ty * W + tx;
                        hit |= int(hop[t]) == k - 1 && __fadd_rn(D[t], C[t]) == dv;
                    }
                    if (hit) {
                        hop[v] = uint16_t(k);
                        wl_mark<kNews>(nxt, nw, H, W, y, x);
                        any = 1;
                    }
                }
            }
            if (!__syncthreads_or(any)) break;
            uint32_t* t = cur;
            cur = nxt;
            nxt = zro;
            zro = t;
        }
    }

    // 3. per-cell outputs (hop and D are final: every path above ended in a barrier)
    const int64_t base = int64_t(b) * N;
    for (int c = tid; c < N; c += nthr) {
        const int y = c / W, x = c - y * W;
        const uint32_t mk = ok ? m.policy_mask<kNews>(y, x) : 0u;
        const int h = hop[c];
        a.dists[base + c] = __fsub_rn(0.0f, D[c]);
        a.hops[base + c] = h == kHopUnset ? -1 : h;
        a.act_mask[base + c] = uint8_t(mk);
        a.action[base + c] = int8_t(__ffs(mk) - 1);
    }
    if (!a.start_idx) {
        if (tid == 0) a.status[b] = status;
        return;
    }

    // 4. the roll-out from the start into bit plane P0, then the fp32 path plane
    for (int i = tid; i < nwords; i += nthr) P0[i] = 0u;
    __syncthreads();
    if (tid == 0) {
        const int s = a.start_idx[b];
        float pc = kInf;
        if (ok && s >= 0 && s < N && D[s] != kInf) {
            int v = s, y = s / W, x = s - y * W;
            P0[y * nw + (x >> 5)] |= 1u << (x & 31);
            for (int step = 0; step < N && v != goal; ++step) {
                const uint32_t mk = m.policy_mask<kNews>(y, x);
                if (!mk) break;
                const int q = __ffs(mk) - 1;
                y += int((kWLMoveDy >> (2 * q)) & 3u) - 1;
                x += int((kWLMoveDx >> (2 * q)) & 3u) - 1;
                v = y * W + x;
                P0[y * nw + (x >> 5)] |= 1u << (x & 31);
            }
            if (v == goal) {
                pc = __fadd_rn(C[s], D[s]);
            } else {   // not reached for a converged map; keep the outputs consistent anyway
                for (int i = 0; i < nwords; ++i) P0[i] = 0u;
                status |= 4;
            }
        } else {
            status |= 4;
        }
        a.path_costs[b] = pc;
        a.status[b] = status;
    }
    __syncthreads();
    for (int c = tid; c < N; c += nthr) {
        const int y = c / W, x = c - y * W;
        a.path_maps[base + c] = float((P0[y * nw + (x >> 5)] >> (x & 31)) & 1u);
    }
}

}  // namespace nastar
