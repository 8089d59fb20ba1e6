// nastar_sampler.cuh — training batches drawn on the GPU: start maps and expert trajectories (MazeDataset semantics).
//
// Two kernels:
//   1. sampler_prepare_kernel, once per dataset, one CTA per map.  From the map's opt_dists, one-hot policy and goal
//      map it writes the three percentile bands of MazeDataset._prepared as bit planes (cell c = bit c&31 of word
//      c>>5, raster order), the band sizes, the goal index, the first-max action of every cell packed as 4-bit
//      nibbles (cell c = bits 4*(c&7) of word c>>3), the four thresholds and a status word (kSampler* flags).
//      The thresholds are np.percentile(vals, 100*(1-[p1,p2,p3,1])) with vals = od[od > od.min()], numpy's
//      default "linear" method restated in fp64 with explicit round-to-nearest operations (no FMA contraction):
//          vi = (n-1)*q;  i = floor(vi);  g = vi - i;  d = v[i+1] - v[i]   (fp32, exact: integer distances)
//          th = g >= 0.5 ? v[i+1] - d*(1-g) : v[i] + d*g
//      and, where vi >= n-1, v[n-1] (numpy clamps both neighbours there).  The order statistics v[i] come from a
//      two-pass radix select over the keys -od in [0, 2^18): 9 high bits, then 9 low bits for the eight wanted ranks.
//      Band r = {c : od[c] > od.min(), th[r+1] <= od[c] <= th[r]}, compared in fp64 like NumPy; bands may overlap.
//   2. sampler_sample_kernel, once per batch, one CTA per sample, one launch for all four output planes.  For start
//      s it reads two u32 draws (d0, d1): band r = (d0*3) >> 32, candidate k = (d1*count_r) >> 32 (exact integer
//      arithmetic), finds the k-th set bit of band r with warp ballot / popc prefix counts, and walks the packed
//      action plane (staged in shared memory where it fits) from the start to the goal, marking the visited cells
//      in a shared bit plane.  The planes are then written with float4 stores.
//
// The walk has no error path: preparation flags (kSamplerBadPolicy) any map with a reachable non-goal cell whose
// action does not move, on the grid, to a cell exactly one step closer, and (kSamplerBadGoal) any map whose goal is
// not its only cell at distance 0.  On an accepted map every walk therefore ends at the goal after exactly -od[start]
// moves and visits no cell twice.  A walk is still capped at H*W moves so that unchecked input cannot hang the GPU.
//
// Limits: H, W <= kSamplerMaxSide (512), so H*W <= 2^18 and every key fits the two 9-bit radix passes.
#pragma once
#include <cstdint>

namespace nastar {

constexpr int kSamplerMaxSide = 512;
constexpr int kSamplerPrepThreads = 512;
constexpr int kSamplerThreads = 256;
constexpr int kSamplerMaxChunk = kSamplerThreads / 32;   // starts walked at once (one warp each)
constexpr int kSamplerBins = 512;

// per-map status bits
constexpr int kSamplerBadDist = 1;      // a distance that is not an integer in [-(H*W), 0]
constexpr int kSamplerNoCandidates = 2; // no cell above od.min()
constexpr int kSamplerEmptyBand = 4;    // a band without a cell
constexpr int kSamplerBadPolicy = 8;    // a reachable non-goal cell whose action does not lead one step closer
constexpr int kSamplerBadGoal = 16;     // the goal is not the only cell at distance 0

struct SamplerPrepArgs {
    const float* dists;     // [B][N]
    const float* policies;  // [B][8][N]
    const float* goals;     // [B][N]
    int B, H, W;
    double q[4];            // quantile fractions, as np.percentile divides them
    uint32_t* band_bits;    // [B][3][nw], nw = ceil(N/32)
    int32_t* counts;        // [B][3]
    int32_t* goal_idx;      // [B]
    uint32_t* actions;      // [B][na], na = ceil(N/8)
    double* thresholds;     // [B][4]
    int32_t* status;        // [B]
};

struct SamplerArgs {
    const float* maps;      // [n_maps][N]
    const float* goals;     // [n_maps][N]
    const uint32_t* band_bits;
    const int32_t* counts;
    const int32_t* goal_idx;
    const uint32_t* actions;
    const int64_t* indices; // [B]
    const uint32_t* draws;  // [B][S][2]
    int n_maps, H, W, B, S;
    int chunk;              // starts per pass (<= kSamplerMaxChunk), limited by shared memory
    int stage;              // 1: the action plane is copied to shared memory first
    float* out_maps;        // [B][N]
    float* out_starts;      // [B][S][N]
    float* out_goals;       // [B][N]
    float* out_trajs;       // [B][S][N]
};

inline int sampler_band_words(int H, int W) { return (H * W + 31) >> 5; }
inline int sampler_action_words(int H, int W) { return (H * W + 7) >> 3; }

// Moore moves of MazeDataset's _ACTION_TO_MOVE: N, E, W, S, NE, NW, SE, SW
__device__ __forceinline__ int sampler_dy(int a) { return ((0xA094 >> (2 * a)) & 3) - 1; }   // -1,0,0,1,-1,-1,1,1
__device__ __forceinline__ int sampler_dx(int a) { return ((0x2249 >> (2 * a)) & 3) - 1; }   //  0,1,-1,0,1,-1,1,-1

__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xFFFFFFFFu, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

// (bin, rank within the bin) of the element with 0-based `rank` in a 512-bin histogram; whole warp
__device__ __forceinline__ void warp_select_bin(const int* hist, int rank, int lane, int& bin, int& resid) {
    const int base = lane * (kSamplerBins / 32);
    int s = 0;
#pragma unroll
    for (int k = 0; k < kSamplerBins / 32; ++k) s += hist[base + k];
    const int incl = warp_incl_scan(s, lane);
    const int excl = incl - s;
    const unsigned hit = __ballot_sync(0xFFFFFFFFu, excl <= rank && rank < incl);
    const int src = __ffs(hit) - 1;
    int b = 0, r = 0;
    if (lane == src) {
        int c = excl;
        for (int k = 0; k < kSamplerBins / 32; ++k) {
            const int h = hist[base + k];
            if (rank < c + h) {
                b = base + k;
                r = rank - c;
                break;
            }
            c += h;
        }
    }
    bin = __shfl_sync(0xFFFFFFFFu, b, src);
    resid = __shfl_sync(0xFFFFFFFFu, r, src);
}

// np.argmax's order: NaN first, then the larger value, then the lower index
__device__ __forceinline__ bool argmax_better(float v, int i, float bv, int bi) {
    const bool n = v != v, bn = bv != bv;
    if (n != bn) return n;
    if (!n && v != bv) return v > bv;
    return i < bi;
}

__global__ void __launch_bounds__(kSamplerPrepThreads, 1) sampler_prepare_kernel(SamplerPrepArgs a) {
    __shared__ int hist1[kSamplerBins];
    __shared__ int hist2[8][kSamplerBins];
    __shared__ int red_i[kSamplerPrepThreads / 32][3];
    __shared__ float red_gv[kSamplerPrepThreads / 32];
    __shared__ int red_gi[kSamplerPrepThreads / 32];
    __shared__ int s_maxkey, s_bad, s_zero, s_goal, s_n, s_status, s_cnt[3];
    __shared__ int s_hi[8], s_res[8], s_key[8];
    __shared__ double s_th[4];

    const int b = blockIdx.x, H = a.H, W = a.W, N = H * W, nw = (N + 31) >> 5;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
    const float* od = a.dists + int64_t(b) * N;
    const float* goal_plane = a.goals + int64_t(b) * N;
    const float* pol = a.policies + int64_t(b) * 8 * N;

    for (int i = tid; i < kSamplerBins; i += blockDim.x) {
        hist1[i] = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) hist2[j][i] = 0;
    }
    if (tid < 3) s_cnt[tid] = 0;
    if (tid == 0) s_status = 0;

    // pass 1: validity, od.min() (as the largest key -od), cells at 0, goal = first argmax of the goal plane
    int maxkey = 0, bad = 0, zero = 0, gi = 0x7FFFFFFF;
    float gv = 0.0f;
    for (int c = tid; c < N; c += blockDim.x) {
        const float v = od[c];
        if (!(v >= -float(N) && v <= 0.0f && v == truncf(v))) {
            bad = 1;
        } else {
            maxkey = max(maxkey, int(-v));
            zero += v == 0.0f;
        }
        const float g = goal_plane[c];
        if (gi == 0x7FFFFFFF || argmax_better(g, c, gv, gi)) {
            gv = g;
            gi = c;
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        maxkey = max(maxkey, __shfl_xor_sync(0xFFFFFFFFu, maxkey, o));
        bad |= __shfl_xor_sync(0xFFFFFFFFu, bad, o);
        zero += __shfl_xor_sync(0xFFFFFFFFu, zero, o);
        const float ov = __shfl_xor_sync(0xFFFFFFFFu, gv, o);
        const int oi = __shfl_xor_sync(0xFFFFFFFFu, gi, o);
        if (oi != 0x7FFFFFFF && (gi == 0x7FFFFFFF || argmax_better(ov, oi, gv, gi))) {
            gv = ov;
            gi = oi;
        }
    }
    if (lane == 0) {
        red_i[warp][0] = maxkey;
        red_i[warp][1] = bad;
        red_i[warp][2] = zero;
        red_gv[warp] = gv;
        red_gi[warp] = gi;
    }
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < nwarp; ++w) {
            maxkey = max(maxkey, red_i[w][0]);
            bad |= red_i[w][1];
            zero += red_i[w][2];
            if (red_gi[w] != 0x7FFFFFFF && (gi == 0x7FFFFFFF || argmax_better(red_gv[w], red_gi[w], gv, gi))) {
                gv = red_gv[w];
                gi = red_gi[w];
            }
        }
        s_maxkey = maxkey;
        s_bad = bad;
        s_zero = zero;
        s_goal = gi;
        a.goal_idx[b] = gi;
    }
    __syncthreads();
    maxkey = s_maxkey;
    const int goal = s_goal;
    if (s_bad) {
        if (tid < 3) a.counts[b * 3 + tid] = 0;
        if (tid < 4) a.thresholds[b * 4 + tid] = 0.0;
        if (tid == 0) a.status[b] = kSamplerBadDist;
        return;
    }

    // pass 2: high 9 bits of the candidate keys (candidates: key < maxkey, i.e. od > od.min())
    for (int c = tid; c < N; c += blockDim.x) {
        const int key = int(-od[c]);
        if (key < maxkey) atomicAdd(&hist1[key >> 9], 1);
    }
    __syncthreads();
    if (warp == 0) {
        int s = 0;
        for (int i = lane; i < kSamplerBins; i += 32) s += hist1[i];
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
        if (lane == 0) s_n = s;
    }
    __syncthreads();
    const int n = s_n;
    if (n == 0) {
        if (tid < 3) a.counts[b * 3 + tid] = 0;
        if (tid < 4) a.thresholds[b * 4 + tid] = 0.0;
        if (tid == 0) a.status[b] = kSamplerNoCandidates;
        return;
    }
    // the eight order statistics (ascending od) that the four interpolations read: warp j < 8 takes rank j
    const double vi_max = double(n - 1);
    auto vindex = [&](int j) {   // selects instead of a.q[j]: a dynamic index would copy the parameters to the stack
        return __dmul_rn(vi_max, j == 0 ? a.q[0] : j == 1 ? a.q[1] : j == 2 ? a.q[2] : a.q[3]);
    };
    auto od_rank = [&](int j) -> int {   // j = 2*quantile + {0: lower, 1: upper} neighbour
        const double vi = vindex(j >> 1);
        if (vi >= vi_max) return n - 1;
        const int lo = int(floor(vi));
        return lo + (j & 1);
    };
    if (warp < 8) {
        const int key_rank = n - 1 - od_rank(warp);   // ascending od = descending key
        int bin, resid;
        warp_select_bin(hist1, key_rank, lane, bin, resid);
        if (lane == 0) {
            s_hi[warp] = bin;
            s_res[warp] = resid;
        }
    }
    __syncthreads();
    // pass 3: low 9 bits of the keys in each wanted high bin
    for (int c = tid; c < N; c += blockDim.x) {
        const int key = int(-od[c]);
        if (key < maxkey) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if ((key >> 9) == s_hi[j]) atomicAdd(&hist2[j][key & (kSamplerBins - 1)], 1);
        }
    }
    __syncthreads();
    if (warp < 8) {
        int bin, resid;
        warp_select_bin(hist2[warp], s_res[warp], lane, bin, resid);
        if (lane == 0) s_key[warp] = (s_hi[warp] << 9) | bin;
    }
    __syncthreads();
    if (tid < 4) {
        const int j = tid;
        const double vi = vindex(j);
        const double prev = vi >= vi_max ? -1.0 : floor(vi);
        const double g = __dsub_rn(vi, prev);
        const float lo = float(-s_key[2 * j]), hi = float(-s_key[2 * j + 1]);   // +0.0 at the goal, like od
        const double d = double(__fsub_rn(hi, lo));
        double th = __dadd_rn(double(lo), __dmul_rn(d, g));
        if (g >= 0.5) th = __dsub_rn(double(hi), __dmul_rn(d, __dsub_rn(1.0, g)));
        s_th[j] = th;
        a.thresholds[b * 4 + j] = th;
    }
    __syncthreads();

    // pass 4: band planes, counts, packed actions and the policy check, one warp per 32 cells
    const double th0 = s_th[0], th1 = s_th[1], th2 = s_th[2], th3 = s_th[3];
    uint32_t* bits = a.band_bits + int64_t(b) * 3 * nw;
    uint32_t* acts = a.actions + int64_t(b) * ((N + 7) >> 3);
    int cnt0 = 0, cnt1 = 0, cnt2 = 0;
    int bad_policy = 0;
    for (int w = warp; w < nw; w += nwarp) {
        const int c = w * 32 + lane;
        const bool in = c < N;
        const float v = in ? od[c] : 0.0f;
        const int key = int(-v);
        const bool cand = in && key < maxkey;
        const double dv = double(v);
        const uint32_t m0 = __ballot_sync(0xFFFFFFFFu, cand && th1 <= dv && dv <= th0);
        const uint32_t m1 = __ballot_sync(0xFFFFFFFFu, cand && th2 <= dv && dv <= th1);
        const uint32_t m2 = __ballot_sync(0xFFFFFFFFu, cand && th3 <= dv && dv <= th2);
        if (lane == 0) {
            bits[w] = m0;
            bits[nw + w] = m1;
            bits[2 * nw + w] = m2;
            cnt0 += __popc(m0);
            cnt1 += __popc(m1);
            cnt2 += __popc(m2);
        }
        int act = 0;
        if (in) {
            float best = pol[c];
#pragma unroll
            for (int k = 1; k < 8; ++k) {
                const float p = pol[int64_t(k) * N + c];
                if (argmax_better(p, k, best, act)) {
                    best = p;
                    act = k;
                }
            }
            if (key < N && c != goal) {   // reachable non-goal cell: the move must land one step closer
                const int y = c / W, x = c - y * W;
                const int ty = y + sampler_dy(act), tx = x + sampler_dx(act);
                if (ty < 0 || ty >= H || tx < 0 || tx >= W || od[ty * W + tx] != v + 1.0f) bad_policy = 1;
            }
        }
        uint32_t word = uint32_t(act) << (4 * (lane & 7));
        word |= __shfl_xor_sync(0xFFFFFFFFu, word, 1);
        word |= __shfl_xor_sync(0xFFFFFFFFu, word, 2);
        word |= __shfl_xor_sync(0xFFFFFFFFu, word, 4);
        if ((lane & 7) == 0 && in) acts[c >> 3] = word;
    }
    if (lane == 0) {
        atomicAdd(&s_cnt[0], cnt0);
        atomicAdd(&s_cnt[1], cnt1);
        atomicAdd(&s_cnt[2], cnt2);
    }
    if (__any_sync(0xFFFFFFFFu, bad_policy) && lane == 0) atomicOr(&s_status, kSamplerBadPolicy);
    __syncthreads();
    if (tid == 0) {
        int st = s_status;
        if (s_cnt[0] == 0 || s_cnt[1] == 0 || s_cnt[2] == 0) st |= kSamplerEmptyBand;
        if (s_zero != 1 || od[goal] != 0.0f) st |= kSamplerBadGoal;
        a.counts[b * 3 + 0] = s_cnt[0];
        a.counts[b * 3 + 1] = s_cnt[1];
        a.counts[b * 3 + 2] = s_cnt[2];
        a.status[b] = st;
    }
}

// flat index of the k-th (0-based) set bit of a bit plane of nw words, raster order; whole warp
__device__ __forceinline__ int warp_kth_set_bit(const uint32_t* plane, int nw, int k, int lane) {
    int before = 0;
    for (int w0 = 0; w0 < nw; w0 += 32) {
        const int w = w0 + lane;
        const uint32_t x = w < nw ? plane[w] : 0u;
        const int c = __popc(x);
        const int incl = warp_incl_scan(c, lane);
        const int total = __shfl_sync(0xFFFFFFFFu, incl, 31);
        if (k < before + total) {
            const int src = __ffs(__ballot_sync(0xFFFFFFFFu, before + incl > k)) - 1;
            int pos = 0;
            if (lane == src) {
                uint32_t m = x;
                for (int r = k - (before + incl - c); r > 0; --r) m &= m - 1;
                pos = w * 32 + __ffs(m) - 1;
            }
            return __shfl_sync(0xFFFFFFFFu, pos, src);
        }
        before += total;
    }
    return -1;
}

__device__ __forceinline__ void sampler_copy_plane(float* dst, const float* src, int N, bool vec) {
    if (vec) {
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* d4 = reinterpret_cast<float4*>(dst);
        for (int i = threadIdx.x; i < (N >> 2); i += blockDim.x) d4[i] = s4[i];
    } else {
        for (int i = threadIdx.x; i < N; i += blockDim.x) dst[i] = src[i];
    }
}

__device__ __forceinline__ void sampler_fill_plane(float* dst, int N, bool vec) {
    if (vec) {
        float4* d4 = reinterpret_cast<float4*>(dst);
        for (int i = threadIdx.x; i < (N >> 2); i += blockDim.x) d4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
        for (int i = threadIdx.x; i < N; i += blockDim.x) dst[i] = 0.0f;
    }
}

__global__ void __launch_bounds__(kSamplerThreads) sampler_sample_kernel(SamplerArgs a) {
    extern __shared__ uint32_t smp_smem[];
    __shared__ int s_start[kSamplerMaxChunk];
    __shared__ int s_off[8];
    const int H = a.H, W = a.W, N = H * W, nw = (N + 31) >> 5, na = (N + 7) >> 3, S = a.S;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int i = blockIdx.x;
    const bool vec = (N & 3) == 0;
    float* out_map = a.out_maps + int64_t(i) * N;
    float* out_goal = a.out_goals + int64_t(i) * N;
    const int64_t bi = a.indices[i];
    if (bi < 0 || bi >= a.n_maps) {   // an index outside the dataset: all-zero planes, nothing read
        sampler_fill_plane(out_map, N, vec);
        sampler_fill_plane(out_goal, N, vec);
        for (int s = 0; s < S; ++s) {
            sampler_fill_plane(a.out_starts + (int64_t(i) * S + s) * N, N, vec);
            sampler_fill_plane(a.out_trajs + (int64_t(i) * S + s) * N, N, vec);
        }
        return;
    }
    const int b = int(bi);
    uint32_t* act_s = smp_smem;
    uint32_t* traj_s = smp_smem + (a.stage ? na : 0);
    const uint32_t* act_g = a.actions + int64_t(b) * na;
    if (a.stage)
        for (int j = tid; j < na; j += blockDim.x) act_s[j] = act_g[j];
    const uint32_t* act = a.stage ? act_s : act_g;
    if (tid < 8) s_off[tid] = sampler_dy(tid) * W + sampler_dx(tid);
    sampler_copy_plane(out_map, a.maps + int64_t(b) * N, N, vec);
    sampler_copy_plane(out_goal, a.goals + int64_t(b) * N, N, vec);
    const int goal = a.goal_idx[b];
    const int32_t* cnt = a.counts + int64_t(b) * 3;
    const uint32_t* bits = a.band_bits + int64_t(b) * 3 * nw;

    for (int s0 = 0; s0 < S; s0 += a.chunk) {
        const int ns = min(a.chunk, S - s0);
        for (int j = tid; j < ns * nw; j += blockDim.x) traj_s[j] = 0u;
        __syncthreads();   // also publishes the staged actions and the move offsets
        if (warp < ns) {
            const uint32_t* d = a.draws + (int64_t(i) * S + s0 + warp) * 2;
            const uint32_t r = uint32_t((uint64_t(d[0]) * 3u) >> 32);
            const uint32_t k = uint32_t((uint64_t(d[1]) * uint32_t(cnt[r])) >> 32);
            const int start = warp_kth_set_bit(bits + int64_t(r) * nw, nw, int(k), lane);
            if (lane == 0) {
                s_start[warp] = start;
                uint32_t* t = traj_s + warp * nw;
                int cur = start;
                for (int step = 0; cur >= 0 && cur != goal && step < N; ++step) {
                    t[cur >> 5] |= 1u << (cur & 31);
                    cur += s_off[(act[cur >> 3] >> (4 * (cur & 7))) & 15u];
                    if (cur < 0 || cur >= N) break;
                }
            }
        }
        __syncthreads();
        for (int j = 0; j < ns; ++j) {
            const int64_t o = (int64_t(i) * S + s0 + j) * N;
            const uint32_t* t = traj_s + j * nw;
            const int st = s_start[j];
            if (vec) {
                float4* ps = reinterpret_cast<float4*>(a.out_starts + o);
                float4* pt = reinterpret_cast<float4*>(a.out_trajs + o);
                for (int e = tid; e < (N >> 2); e += blockDim.x) {
                    const int c = e << 2;
                    const uint32_t m = t[c >> 5] >> (c & 31);
                    pt[e] = make_float4(float(m & 1u), float((m >> 1) & 1u), float((m >> 2) & 1u), float((m >> 3) & 1u));
                    ps[e] = make_float4(float(st == c), float(st == c + 1), float(st == c + 2), float(st == c + 3));
                }
            } else {
                for (int c = tid; c < N; c += blockDim.x) {
                    a.out_trajs[o + c] = float((t[c >> 5] >> (c & 31)) & 1u);
                    a.out_starts[o + c] = float(st == c);
                }
            }
        }
        __syncthreads();   // the next chunk clears traj_s
    }
}

}  // namespace nastar
