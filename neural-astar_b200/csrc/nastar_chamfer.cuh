// nastar_chamfer.cuh — directed Chamfer distances between two cell sets per map, exact and deterministic (DESIGN.md §23).
//
// chamfer_kernel: one CTA per map (CTAs loop over maps when the grid is capped).  masks[b] is H*W bytes, bit 0 = set A,
// bit 1 = set B.  For each direction (A -> B, then B -> A) the CTA computes the exact squared Euclidean distance
// transform of the target set in integer arithmetic, Meijster's separable algorithm:
//   columns  g[y][x] = |y - y'| to the nearest target cell of column x (H + W when the column has none), one thread
//            per column, a downward and an upward sweep;
//   rows     the lower envelope of the parabolas (x - i)^2 + g[y][i]^2 over i, one thread per row (its stacks s, t
//            of W entries each), then dt[y][x] = min_i (x - i)^2 + g[y][i]^2 at every x of the row;
// and sums, in a fixed order, the correctly rounded fp64 sqrt(dt) (chamfer_sqrt) over the source set's cells: each row thread from
// x = W-1 down to 0, then thread 0 over the row sums from y = 0 up.  The mean is that sum over the source set's count.
// A map with an empty set gets NaN in both columns.  The column distances (uint16), the stacks (uint16) and the row
// sums live in shared memory when chamfer_layout(H, W).bytes <= kChamferSmemMax, else in a global slot per CTA.
#pragma once
#include <cstdint>

namespace nastar {

constexpr int kChamferThreads = 128;
constexpr int kChamferMaxSide = 1024;
constexpr int64_t kChamferSmemMax = 96 * 1024;

struct ChamferLayout {
    int P, R;                   // pitch of g in elements (odd: rows of the row pass fall in different banks); rows per pass
    int64_t s_off, t_off, rsum_off, bytes;
};

__host__ __device__ inline ChamferLayout chamfer_layout(int H, int W) {
    ChamferLayout L;
    L.P = W | 1;
    L.R = H < kChamferThreads ? H : kChamferThreads;
    L.s_off = int64_t(H) * L.P * 2;
    L.t_off = L.s_off + int64_t(W) * L.R * 2;
    L.rsum_off = (L.t_off + int64_t(W) * L.R * 2 + 7) & ~int64_t(7);
    L.bytes = L.rsum_off + int64_t(H) * 8;
    return L;
}

struct ChamferArgs {
    const uint8_t* masks;
    int B, H, W;
    double* out;             // [B][2]: d(A -> B), d(B -> A)
    unsigned char* slots;    // global slots of slot_bytes, one per CTA; NULL: shared memory
    int64_t slot_bytes;
};

// floor(num / den) for den > 0
__device__ __forceinline__ int chamfer_floor_div(int num, int den) {
    return num >= 0 ? num / den : -((-num + den - 1) / den);
}

// sqrt(v) correctly rounded to fp64, for 0 <= v < 2^22 (squared distances of maps up to 1024 x 1024), without the
// subroutine call of sqrt()'s special-operand path (its saved registers would spill): two Newton steps from rsqrtf give
// y within an ulp u, then y moves by u until -y u < v - y^2 <= y u, which is exactly |sqrt(v) - y| < u / 2 (v - y^2 is
// computed exactly by the fma and is a multiple of u^2, and sqrt(v) is never a midpoint nor within an ulp of a power
// of two, where u would change, unless it is that power).
__device__ __forceinline__ double chamfer_sqrt(int v) {
    if (v == 0) return 0.0;
    const double x = double(v);
    double r = double(rsqrtf(float(v)));
    r = r * (1.5 - 0.5 * x * r * r);
    r = r * (1.5 - 0.5 * x * r * r);
    double y = x * r;
    const double u = __longlong_as_double(__double_as_longlong(y) & 0x7FF0000000000000LL) * 0x1p-52;
    for (int k = 0; k < 2; ++k) {
        const double e = fma(-y, y, x), yu = y * u;
        if (e > yu) y += u;
        else if (e <= -yu) y -= u;
    }
    return y;
}

__global__ void __launch_bounds__(kChamferThreads) chamfer_kernel(ChamferArgs a) {
    extern __shared__ __align__(16) unsigned char cm_smem[];
    __shared__ int count[2];
    const int tid = threadIdx.x, H = a.H, W = a.W;
    const ChamferLayout L = chamfer_layout(H, W);
    const int P = L.P, R = L.R, INF = H + W;
    unsigned char* base = a.slots ? a.slots + int64_t(blockIdx.x) * a.slot_bytes : cm_smem;
    uint16_t* g = reinterpret_cast<uint16_t*>(base);
    uint16_t* sv = reinterpret_cast<uint16_t*>(base + L.s_off);
    uint16_t* tv = reinterpret_cast<uint16_t*>(base + L.t_off);
    double* rsum = reinterpret_cast<double*>(base + L.rsum_off);
    const int64_t N = int64_t(H) * W;
    for (int b = blockIdx.x; b < a.B; b += gridDim.x) {
        const uint8_t* m = a.masks + int64_t(b) * N;
        if (tid < 2) count[tid] = 0;
        __syncthreads();
        int ca = 0, cb = 0;
        for (int64_t i = tid; i < N; i += kChamferThreads) {
            const uint8_t v = m[i];
            ca += v & 1;
            cb += (v >> 1) & 1;
        }
        atomicAdd(&count[0], ca);
        atomicAdd(&count[1], cb);
        __syncthreads();
        double res0 = __longlong_as_double(0x7FF8000000000000LL), res1 = res0;   // NaN
        if (count[0] && count[1]) {
            for (int dir = 0; dir < 2; ++dir) {
                const uint8_t tbit = dir == 0 ? 2 : 1, sbit = dir == 0 ? 1 : 2;   // target set, source set
                for (int x = tid; x < W; x += kChamferThreads) {
                    int d = INF;
                    for (int y = 0; y < H; ++y) {
                        d = (m[int64_t(y) * W + x] & tbit) ? 0 : (d < INF ? d + 1 : INF);
                        g[int64_t(y) * P + x] = uint16_t(d);
                    }
                    d = INF;
                    for (int y = H - 1; y >= 0; --y) {
                        const int here = g[int64_t(y) * P + x];
                        d = here == 0 ? 0 : (d < INF ? d + 1 : INF);
                        if (d < here) g[int64_t(y) * P + x] = uint16_t(d);
                    }
                }
                __syncthreads();
                for (int y0 = 0; y0 < H; y0 += R) {
                    const int y = y0 + tid;
                    if (tid < R && y < H) {
                        const uint16_t* gr = g + int64_t(y) * P;
                        uint16_t* s = sv + tid;   // entry k of this row's stacks at [k * R]
                        uint16_t* t = tv + tid;
                        // f(x, i) = (x - i)^2 + g[i]^2 <= (W - 1)^2 + (H + W)^2 < 2^31
                        auto f = [&](int x, int i) { const int gi = gr[i]; return (x - i) * (x - i) + gi * gi; };
                        int q = 0;
                        s[0] = 0;
                        t[0] = 0;
                        for (int u = 1; u < W; ++u) {
                            while (q >= 0 && f(t[q * R], s[q * R]) > f(t[q * R], u)) --q;
                            if (q < 0) {
                                q = 0;
                                s[0] = uint16_t(u);
                            } else {
                                const int i = s[q * R], gi = gr[i], gu = gr[u];
                                const int w = 1 + chamfer_floor_div(u * u - i * i + gu * gu - gi * gi, 2 * (u - i));
                                if (w < W) {
                                    ++q;
                                    s[q * R] = uint16_t(u);
                                    t[q * R] = uint16_t(w);
                                }
                            }
                        }
                        const uint8_t* mr = m + int64_t(y) * W;
                        double sum = 0.0;
                        for (int u = W - 1; u >= 0; --u) {
                            if (mr[u] & sbit) sum += chamfer_sqrt(f(u, s[q * R]));
                            if (u == t[q * R]) --q;
                        }
                        rsum[y] = sum;
                    }
                }
                __syncthreads();
                if (tid == 0) {
                    double tot = 0.0;
                    for (int y = 0; y < H; ++y) tot += rsum[y];
                    const double r = tot / double(count[dir]);
                    if (dir == 0) res0 = r;
                    else res1 = r;
                }
                __syncthreads();   // g and the row sums are reused
            }
        }
        if (tid == 0) {
            a.out[2 * int64_t(b)] = res0;
            a.out[2 * int64_t(b) + 1] = res1;
        }
        __syncthreads();
    }
}

}  // namespace nastar
