// nastar_goals.cuh — goals for new maps drawn on the GPU (the planning-datasets generator's from_largest rule).
//
// One CTA per map, one launch, no host synchronisation.  Per map (DESIGN.md §12):
//   region     the largest 4-connected region of passable cells (value != 0); ties go to the region whose first cell
//              comes first in raster order;
//   candidates the region's cells inside the four e x e corner squares, (y < e || y >= H-e) && (x < e || x >= W-e),
//              when there is one; otherwise the whole region (e == 0 selects no corner cell, so the whole region);
//   draw       candidate k = (d * count) >> 32 in raster order, d = the map's u32 draw.
//
// The region comes from union-find over flat cell indices with union by minimum index, so a region's root is its
// first cell in raster order and the tie rule becomes "smallest root".  All phases work on one u32 plane P (one entry
// per cell), separated by __syncthreads:
//   1. init    P[c] = the first cell of c's horizontal run inside its warp's 32-cell chunk; obstacles kGoalsNone;
//   2. merge   union(c, c-1) across chunk boundaries, union(c, c-W) where c and c-W are passable unless both left
//              neighbours are (those two runs are then already joined through c-1);  hooks are atomicCAS of a root to
//              the smaller root (ECL-CC), finds halve paths with plain stores; every value in P stays an ancestor;
//   3. compress P[c] = its root, found by a read-only walk, so every cell points at its root;
//   4. count   roots become kGoalsRoot | 0, then every cell adds 1 to its root (one atomic per distinct root of a warp);
//   5. select  the root with the largest (count, -root) as one packed 64-bit key, a block max;
//   6. mark    two bit planes of ceil(H*W/32) words (cell c = bit c%32 of word c/32): the region, and the region's
//              corner cells, by ballot; the corner count by popc;
//   7. pick    the k-th set bit of the chosen plane with the sampler's ballot/popc prefix search (warp_kth_set_bit);
//   8. write   goal_idx, status and the fp32 goal plane (one 1.0, zeros elsewhere).
// The result is a function of the map alone: the partition into regions does not depend on the order in which the
// racing unions land, and neither does any minimum, count or prefix taken from it.
//
// Where P lives: in shared memory when P and the two bit planes fit (H*W <= ~54 000 cells, 232x232); above that, in
// the map's own fp32 goal plane, which has exactly one u32 of room per cell and is overwritten by phase 8 anyway.  So
// there is no workspace at any size.  Reads of P are volatile: other threads change it, and in global memory an L1
// line could otherwise hold a value that an atomic at L2 has already replaced.
//
// Every loop is bounded by H*W (a find follows strictly decreasing indices; a failed hook lowers one of its two roots),
// so input that skipped validation cannot hang the GPU.  Status bit kGoalsNoPassable: the map has no passable cell;
// its goal plane is all zero and goal_idx = -1.
//
// Limits: H, W <= kGoalsMaxSide (512), the limit of the label and sampler kernels.  Then H*W <= 2^18, so an index or a
// count fits below the kGoalsRoot bit.
#pragma once
#include <cstdint>

#include "nastar_sampler.cuh"   // warp_kth_set_bit

namespace nastar {

constexpr int kGoalsMaxSide = 512;
constexpr int kGoalsMaxThreads = 512;
constexpr int kGoalsNoPassable = 1;
constexpr uint32_t kGoalsNone = 0xFFFFFFFFu;   // P of an obstacle cell
constexpr uint32_t kGoalsRoot = 0x80000000u;   // P of a root after phase 4: kGoalsRoot | region size
constexpr size_t kGoalsSmemCap = 225 * 1024;  // dynamic shared memory the plane may take (static use stays < 2 KB)

struct GoalsArgs {
    const float* maps;     // [B] maps of H*W fp32 cells, map_stride elements apart
    int64_t map_stride;
    int B, H, W, edge;
    const uint32_t* draws; // [B]
    int plane_in_smem;     // 1: P in shared memory, 0: P in the map's goal plane
    int32_t* goal_idx;     // [B]
    float* goal_maps;      // [B][H*W]
    int32_t* status;       // [B]
};

inline int goals_words(int H, int W) { return (H * W + 31) >> 5; }
inline bool goals_plane_in_smem(int H, int W) {
    return size_t(H) * W * 4 + size_t(goals_words(H, W)) * 8 <= kGoalsSmemCap;
}
inline size_t goals_smem_bytes(int H, int W) {
    return size_t(goals_words(H, W)) * 8 + (goals_plane_in_smem(H, W) ? size_t(H) * W * 4 : 0);
}
inline int goals_threads(int H, int W) {   // about 8 cells per thread
    const int t = ((H * W + 7) / 8 + 31) & ~31;
    return t < 32 ? 32 : (t > kGoalsMaxThreads ? kGoalsMaxThreads : t);
}

// root of c, following strictly decreasing indices and halving the path on the way
__device__ __forceinline__ uint32_t goals_find(volatile uint32_t* P, uint32_t c, int N) {
    uint32_t par = P[c];
    if (par == c) return par;
    uint32_t prev = c, next;
    for (int s = 0; s < N && par > (next = P[par]); ++s) {
        P[prev] = next;
        prev = par;
        par = next;
    }
    return par;
}

__device__ __forceinline__ void goals_union(volatile uint32_t* P, uint32_t a, uint32_t b, int N) {
    uint32_t ra = goals_find(P, a, N), rb = goals_find(P, b, N);
    uint32_t* Pw = const_cast<uint32_t*>(P);
    for (int s = 0; s < N && ra != rb; ++s) {
        // hook the larger root under the smaller; a failed CAS returns the larger one's new parent, which is lower
        if (ra < rb) {
            const uint32_t r = atomicCAS(Pw + rb, rb, ra);
            if (r == rb) break;
            rb = r;
        } else {
            const uint32_t r = atomicCAS(Pw + ra, ra, rb);
            if (r == ra) break;
            ra = r;
        }
    }
}

// root of a passable cell after phase 4 (kGoalsNone for an obstacle)
__device__ __forceinline__ uint32_t goals_root(volatile uint32_t* P, uint32_t c) {
    const uint32_t p = P[c];
    return p == kGoalsNone ? kGoalsNone : (p & kGoalsRoot) ? c : p;
}

__global__ void __launch_bounds__(kGoalsMaxThreads) sample_goals_kernel(GoalsArgs a) {
    extern __shared__ uint32_t goals_smem[];
    __shared__ unsigned long long s_key[kGoalsMaxThreads / 32];
    __shared__ int s_cnt[kGoalsMaxThreads / 32];
    __shared__ unsigned long long s_best;
    __shared__ int s_goal;

    const int b = blockIdx.x, H = a.H, W = a.W, N = H * W, nw = (N + 31) >> 5, e = a.edge;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
    const float* map = a.maps + int64_t(b) * a.map_stride;
    float* out = a.goal_maps + int64_t(b) * N;
    uint32_t* region_bits = goals_smem;
    uint32_t* corner_bits = goals_smem + nw;
    volatile uint32_t* P = a.plane_in_smem ? goals_smem + 2 * nw : reinterpret_cast<uint32_t*>(out);

    // 1. init: every passable cell points at the first cell of its run within the chunk (run starts: a passable cell
    //    whose left neighbour is not passable or is in the previous row, and lane 0)
    for (int c0 = warp * 32; c0 < N; c0 += nwarp * 32) {
        const int c = c0 + lane;
        const bool pas = c < N && map[c] != 0.0f;
        const bool row_start = c < N && c % W == 0;
        const uint32_t pm = __ballot_sync(0xFFFFFFFFu, pas);
        const uint32_t starts = pm & (~(pm << 1) | __ballot_sync(0xFFFFFFFFu, row_start) | 1u);
        if (c < N) P[c] = pas ? uint32_t(c0 + 31 - __clz(starts & (0xFFFFFFFFu >> (31 - lane)))) : kGoalsNone;
    }
    __syncthreads();
    // 2. merge
    for (int c = tid; c < N; c += blockDim.x) {
        if (P[c] == kGoalsNone) continue;
        const int x = c % W;
        const bool left = x > 0 && P[c - 1] != kGoalsNone;
        if (left && (c & 31) == 0) goals_union(P, c, c - 1, N);
        if (c >= W && P[c - W] != kGoalsNone && !(left && P[c - W - 1] != kGoalsNone)) goals_union(P, c, c - W, N);
    }
    __syncthreads();
    // 3. compress: a read-only walk, each thread writing only its own cell (a halving store here could replace an
    //    entry another thread has just pointed at its root with an intermediate ancestor)
    for (int c = tid; c < N; c += blockDim.x) {
        uint32_t r = P[c], next;
        if (r == kGoalsNone) continue;
        for (int s = 0; s < N && r > (next = P[r]); ++s) r = next;
        P[c] = r;
    }
    __syncthreads();
    // 4. count
    for (int c = tid; c < N; c += blockDim.x)
        if (P[c] == uint32_t(c)) P[c] = kGoalsRoot;
    __syncthreads();
    for (int c0 = warp * 32; c0 < N; c0 += nwarp * 32) {
        const int c = c0 + lane;
        const uint32_t r = c < N ? goals_root(P, c) : kGoalsNone;
        const uint32_t same = __match_any_sync(0xFFFFFFFFu, r);
        if (r != kGoalsNone && lane == __ffs(same) - 1) atomicAdd(const_cast<uint32_t*>(P) + r, __popc(same));
    }
    __syncthreads();
    // 5. select: max of (count << 32 | ~root) over the roots; 0 when there is no passable cell
    unsigned long long best = 0;
    for (int c = tid; c < N; c += blockDim.x) {
        const uint32_t p = P[c];
        if (p != kGoalsNone && (p & kGoalsRoot)) {
            const unsigned long long k = (uint64_t(p & ~kGoalsRoot) << 32) | uint32_t(~uint32_t(c));
            best = k > best ? k : best;
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const unsigned long long v = __shfl_xor_sync(0xFFFFFFFFu, best, o);
        best = v > best ? v : best;
    }
    if (lane == 0) s_key[warp] = best;
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < nwarp; ++w) best = s_key[w] > best ? s_key[w] : best;
        s_best = best;
    }
    __syncthreads();
    best = s_best;
    const int count = int(best >> 32);
    const uint32_t root = ~uint32_t(best);
    // 6. mark the region and its corner cells
    int ncorner = 0;
    if (count > 0) {
        for (int w = warp; w < nw; w += nwarp) {
            const int c = w * 32 + lane;
            const bool in = c < N && goals_root(P, c) == root;
            const int y = c / W, x = c - y * W;
            const bool corner = (y < e || y >= H - e) && (x < e || x >= W - e);
            const uint32_t mr = __ballot_sync(0xFFFFFFFFu, in), mc = __ballot_sync(0xFFFFFFFFu, in && corner);
            if (lane == 0) {
                region_bits[w] = mr;
                corner_bits[w] = mc;
                ncorner += __popc(mc);
            }
        }
    }
    if (lane == 0) s_cnt[warp] = ncorner;
    __syncthreads();
    // 7. pick
    if (warp == 0) {
        int nc = lane < nwarp ? s_cnt[lane] : 0;
#pragma unroll
        for (int o = 16; o; o >>= 1) nc += __shfl_xor_sync(0xFFFFFFFFu, nc, o);
        int goal = -1;
        if (count > 0) {
            const int n = nc > 0 ? nc : count;
            const int k = int((uint64_t(a.draws[b]) * uint32_t(n)) >> 32);
            goal = warp_kth_set_bit(nc > 0 ? corner_bits : region_bits, nw, k, lane);
        }
        if (lane == 0) {
            s_goal = goal;
            a.goal_idx[b] = goal;
            a.status[b] = count > 0 ? 0 : kGoalsNoPassable;
        }
    }
    __syncthreads();   // every read of P is done before the goal plane (possibly P itself) is written
    // 8. write
    const int goal = s_goal;
    for (int c = tid; c < N; c += blockDim.x) out[c] = c == goal ? 1.0f : 0.0f;
}

}  // namespace nastar
