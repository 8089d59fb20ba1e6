// nastar_labels.cuh — shortest-path training labels for new maps (the planning-datasets generator's labels).
//
// One CTA per map, two phases in one launch:
//   1. optimal distances: a bit-parallel wavefront BFS from the goal over the passable cells.  The map is held as
//      u32 row words in shared memory (passable / visited / frontier x2); one wavefront is
//          next = dilate8(frontier) & passable & ~visited
//      with dilate8 = the OR of each word's left/right shifts (carries from the neighbouring words) over the three
//      neighbouring rows.  Cells first reached in wavefront k get -k, the goal 0, every other cell -(H*W).  The loop
//      ends when a wavefront is empty (__syncthreads_or, no host round trip).
//   2. policy: one thread per cell reads the distances of its 8 move targets (a move that leaves the grid or enters
//      a non-passable cell stays on the cell) and writes the 8-bit mask of the maximal actions and the first of them.
//
// Semantics (Moore mechanism, one orientation) of planning-datasets/planning_datasets_utils:
//   passable iff map value != 0.0 (mechanism.py:166-207); actions 0..7 = N, E, W, S, NE, NW, SE, SW
//   (mechanism.py:140-149, neighbors_func :209-219), no corner-cutting check; unit step cost, distances of
//   dijkstra_dist (dijkstra.py:120-157, stored negated); max set of extract_policy (data.py:40-58).
//
// The NEWS mechanism (mechanism.py:52-131: actions 0..3 = N, E, W, S, the first four Moore actions in the same order)
// is the kMech = kMechNews instantiation: dilate4 = the word's own left/right shifts with carries OR the vertically
// adjacent rows unshifted, and the policy reads 4 targets, so act_mask uses bits 0..3 only.
//
// Limits: H, W <= kLabelsMaxSide (512).  Then H*W <= 2^18, so every distance is exact in fp32, and the four bit
// planes take at most 4 * 512 * 16 * 4 B = 128 KB of shared memory.
#pragma once
#include <cstdint>

namespace nastar {

constexpr int kLabelsMaxSide = 512;
constexpr int kLabelsMaxThreads = 512;
constexpr int kMechMoore = 0;   // NASTAR_MECH_MOORE
constexpr int kMechNews = 1;    // NASTAR_MECH_NEWS

struct LabelsArgs {
    const float* maps;        // [B] maps of H*W fp32 cells, map_stride elements apart
    int64_t map_stride;
    const int32_t* goal_idx;  // [B] flat goal index y*W+x; out of range = no goal (every cell -(H*W))
    int B, H, W;
    float* dists;             // [B][H*W]
    uint8_t* act_mask;        // [B][H*W]
    int8_t* action;           // [B][H*W]
};

inline int labels_words(int H, int W) { return H * ((W + 31) >> 5); }
inline size_t labels_smem_bytes(int H, int W) { return size_t(4) * labels_words(H, W) * sizeof(uint32_t); }
inline int labels_threads(int H, int W) {
    const int t = (labels_words(H, W) + 31) & ~31;
    return t < 32 ? 32 : (t > kLabelsMaxThreads ? kLabelsMaxThreads : t);
}

template <int kMech>
__global__ void __launch_bounds__(kLabelsMaxThreads) opt_labels_kernel(LabelsArgs a) {
    constexpr int kActions = kMech == kMechNews ? 4 : 8;
    extern __shared__ uint32_t lbl_smem[];
    const int H = a.H, W = a.W, nw = (W + 31) >> 5, nwords = H * nw, N = H * W;
    uint32_t* pas = lbl_smem;
    uint32_t* vis = pas + nwords;
    uint32_t* cur = vis + nwords;
    uint32_t* nxt = cur + nwords;
    const int b = blockIdx.x;
    const float* map = a.maps + int64_t(b) * a.map_stride;
    float* dist = a.dists + int64_t(b) * N;
    const float unreached = -float(N);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    int goal = a.goal_idx[b];
    if (goal < 0 || goal >= N) goal = -1;
    const int gy = goal >= 0 ? goal / W : -1, gx = goal >= 0 ? goal - gy * W : 0;

    // passability words (one ballot per 32 cells of a row) and the "never reached" fill of the distance plane
    for (int i = warp; i < nwords; i += nwarp) {
        const int y = i / nw, w = i - y * nw, x = w * 32 + lane;
        bool p = false;
        if (x < W) {
            p = map[y * W + x] != 0.0f;
            dist[y * W + x] = unreached;
        }
        const uint32_t bits = __ballot_sync(0xFFFFFFFFu, p);
        if (lane == 0) {
            const uint32_t g = (y == gy && w == (gx >> 5)) ? (1u << (gx & 31)) : 0u;
            pas[i] = bits;
            vis[i] = g;
            cur[i] = g;
        }
    }
    __syncthreads();
    if (goal >= 0 && threadIdx.x == 0) dist[goal] = 0.0f;   // the goal is the source even when it is not passable

    for (int k = 1;; ++k) {
        int any = 0;
        const float dk = -float(k);
        for (int i = threadIdx.x; i < nwords; i += blockDim.x) {
            const int y = i / nw, w = i - y * nw;
            uint32_t h = 0;
#pragma unroll
            for (int dy = -1; dy <= 1; ++dy) {
                const int yy = y + dy;
                if (yy < 0 || yy >= H) continue;
                const uint32_t* row = cur + yy * nw;
                const uint32_t c = row[w];
                if (kMech == kMechNews && dy != 0) {   // 4-connected: the rows above and below contribute unshifted
                    h |= c;
                    continue;
                }
                const uint32_t l = w > 0 ? row[w - 1] : 0u;
                const uint32_t r = w + 1 < nw ? row[w + 1] : 0u;
                h |= c | (c << 1) | (l >> 31) | (c >> 1) | (r << 31);
            }
            const uint32_t n = h & pas[i] & ~vis[i];
            nxt[i] = n;
            if (n) {
                vis[i] |= n;
                any = 1;
                float* drow = dist + y * W + w * 32;
                for (uint32_t m = n; m; m &= m - 1) drow[__ffs(m) - 1] = dk;
            }
        }
        if (!__syncthreads_or(any)) break;   // also orders this wavefront's writes before the next one's reads
        uint32_t* t = cur;
        cur = nxt;
        nxt = t;
    }

    // policy: max set over the kActions move targets with the stay rule (the distances written above are visible to
    // the whole block after the barrier that ended the loop)
    const int dys[8] = {-1, 0, 0, +1, -1, -1, +1, +1};
    const int dxs[8] = {0, +1, -1, 0, +1, -1, +1, -1};
    for (int c = threadIdx.x; c < N; c += blockDim.x) {
        const int y = c / W, x = c - y * W;
        float best = 0.0f;
        uint32_t mask = 0;
#pragma unroll
        for (int act = 0; act < kActions; ++act) {
            const int ty = y + dys[act], tx = x + dxs[act];
            int t = c;
            if (ty >= 0 && ty < H && tx >= 0 && tx < W && ((pas[ty * nw + (tx >> 5)] >> (tx & 31)) & 1u)) t = ty * W + tx;
            const float v = dist[t];
            if (act == 0 || v > best) {
                best = v;
                mask = 1u << act;
            } else if (v == best) {
                mask |= 1u << act;
            }
        }
        const int64_t o = int64_t(b) * N + c;
        a.act_mask[o] = uint8_t(mask);
        a.action[o] = int8_t(__ffs(mask) - 1);
    }
}

}  // namespace nastar
