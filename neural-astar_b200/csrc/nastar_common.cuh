// nastar_common.cuh — device helpers shared by the A* engines (sm_90a).
//
// Arithmetic contract (SURVEY.md App. A): every fp32 operation of the reference's loop is a
// separately rounded IEEE op (ATen element-wise kernels; no FMA contraction), so all
// numerics that feed comparisons go through __fmul_rn/__fadd_rn/__fsqrt_rn here.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nastar {

constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr uint32_t kKeyInf = 0xFFFFFFFFu;  // "no open cell" sentinel, above every float key

// Exit mode of a forward search kernel (template parameter kExit):
//   kExitEarly    the map stops at its solve step (per-map early exit, differentiable_astar.py:251-252);
//   kExitNone     NASTAR_FWD_NO_EARLY_EXIT: exactly T steps per map;
//   kExitCoupled1 pass 1 of nastar_b200_forward_coupled: no solve-step exit, but the map stops at its fixed point
//                 (the goal is re-selected and the step changes nothing), and every executed step's at-goal bit
//                 goes to a per-map bitmap (CoupledWs);
//   kExitCoupled2 pass 2: maps that pass 1 stopped after more than *T_batch steps run again for exactly *T_batch
//                 steps; every other map only finishes its counters.
constexpr int kExitEarly = 0, kExitNone = 1, kExitCoupled1 = 2, kExitCoupled2 = 3;
// kExitBlackbox, added to kExitEarly, kExitCoupled1 or kExitCoupled2: the black-box backward
// (nastar_b200_backward_blackbox).  The prologue searches w' = fl(w + fl(lambda * dL/dhistories)) instead of the cost
// plane, and the epilogue writes dL/dw = (closed(w') - histories) / lambda instead of histories and paths.  A bit of
// the exit mode rather than a template parameter of its own, so that the other instantiations keep their names.
constexpr int kExitBlackbox = 8;

// how pass 1 of the coupled forward ended for a map (CoupledWs::end)
constexpr int kEndCapped = 0;      // T steps executed
constexpr int kEndExhausted = 1;   // the open set ran empty: "at goal" is false from then on
constexpr int kEndFixed = 2;       // fixed point: the goal is selected at every later step

// per-map records of the coupled forward, in the caller's workspace (nastar_b200_forward_coupled)
struct CoupledWs {
    int32_t* stop;    // [B] steps pass 1 executed
    int32_t* end;     // [B] kEnd*
    int32_t* first;   // [B] first step that selected the goal, or NASTAR_TS_* (pass 1's t_solve)
    uint32_t* bits;   // [B][words] bit t of word t/32: step t selected the goal; only bits < stop[b] are valid
    int32_t words;    // ceil(T / 32)
};

// the at-goal bits of map b for steps 32w .. 32w+31: the recorded bits below stop, the constant tail above
__device__ __forceinline__ uint32_t coupled_word(const CoupledWs& cw, int b, int w) {
    const int stop = cw.stop[b];
    const uint32_t tail = (cw.end[b] == kEndFixed) ? 0xFFFFFFFFu : 0u;
    const int lo = w << 5;
    if (lo >= stop) return tail;
    const uint32_t v = cw.bits[int64_t(b) * cw.words + w];
    if (stop - lo >= 32) return v;
    const uint32_t m = (1u << (stop - lo)) - 1u;
    return (v & m) | (tail & ~m);
}

// pass 2 for a map that pass 1 already finished (stop <= T_batch): its masks stand; the counters become those of a
// NO_EARLY_EXIT search of T_batch steps.  A map at its fixed point executes all of them; a map whose open set ran
// empty exactly at step T_batch reaches the cap before it can notice.
__device__ __forceinline__ void coupled_keep(const CoupledWs& cw, int b, int Tb, int32_t* t_solve, int32_t* n_steps) {
    const int end = cw.end[b];
    if (end == kEndFixed && n_steps) n_steps[b] = Tb;
    if (end == kEndExhausted && cw.stop[b] == Tb && t_solve) t_solve[b] = -1;   // NASTAR_TS_CAPPED
}

// Order-preserving map float -> uint32 (a < b  <=>  key(a) < key(b) for non-NaN a, b).
__device__ __forceinline__ uint32_t fkey(float f) {
    uint32_t b = __float_as_uint(f);
    return b ^ (static_cast<uint32_t>(static_cast<int32_t>(b) >> 31) | 0x80000000u);
}

// f = g_ratio*g + (1-g_ratio)*h   (differentiable_astar.py:206) — three roundings.
__device__ __forceinline__ float f_value(float gr, float omg, float g, float h) {
    return __fadd_rn(__fmul_rn(gr, g), __fmul_rn(omg, h));
}

// sqrt(dy^2 + dx^2) as get_heuristic computes it: squares and their sum rounded to fp32 one operation at a time.  Below
// 4 096 cells every step is exact; beyond, dx*dx exceeds 2^24 and the sum is rounded twice, which an exactly rounded
// integer sum would not reproduce (at (dy, dx) = (7, 4281) the heuristic would come out one ulp high).
__device__ __forceinline__ float euclid(int ady, int adx) {
    const float fy = static_cast<float>(ady), fx = static_cast<float>(adx);
    return __fsqrt_rn(__fadd_rn(__fmul_rn(fy, fy), __fmul_rn(fx, fx)));
}

// get_heuristic (differentiable_astar.py:26-52): chebyshev + 0.001 * euclid, all in fp32.
__device__ __forceinline__ float heuristic(int y, int x, int gy, int gx) {
    int idy = y - gy, idx = x - gx;
    int ady = idy < 0 ? -idy : idy, adx = idx < 0 ? -idx : idx;
    float cheb = static_cast<float>(ady + adx - (ady < adx ? ady : adx));   // exact
    return __fadd_rn(cheb, __fmul_rn(0.001f, euclid(ady, adx)));
}

// The generator's NorthEastWestSouth.get_heuristic (planning_datasets_utils/mechanism.py:124-131): manhattan +
// 0.001 * euclid, all in fp32.  The manhattan term is an exact integer, like the Chebyshev one above.
__device__ __forceinline__ float heuristic_news(int y, int x, int gy, int gx) {
    int idy = y - gy, idx = x - gx;
    int ady = idy < 0 ? -idy : idy, adx = idx < 0 ? -idx : idx;
    float manh = static_cast<float>(ady + adx);                               // exact
    return __fadd_rn(manh, __fmul_rn(0.001f, euclid(ady, adx)));
}

// heuristic of the search's mechanism: kNews = NASTAR_FWD_NEWS / NASTAR_MECH_NEWS (4-connected), else Moore
template <bool kNews>
__device__ __forceinline__ float heuristic_of(int y, int x, int gy, int gx) {
    return kNews ? heuristic_news(y, x, gy, gx) : heuristic(y, x, gy, gx);
}

// encoder.py:32-34, cost = sigmoid(x) * const, with the operation sequence of ATen's CUDA sigmoid
// (1 / (1 + exp(-x)), full-precision expf and IEEE division) followed by a separately rounded multiply.
__device__ __forceinline__ float sigmoid_scaled(float x, float scale) {
    return __fmul_rn(__fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))), scale);
}

// NASTAR_COST_TAPS: logit(y,x) = bias + sum_k taps[y+ky-1][x+kx-1][k], k = ky*3+kx ascending, zero padding —
// the 9->1 gather that finishes the encoder's single-output-channel 3x3 convolution (planner/encoder.py
// `_conv3x3_single_output`).  taps is one map's [H*W][9] block.
__device__ __forceinline__ float cost_from_taps(const float* __restrict__ taps, int y, int x, int H, int W,
                                                float bias, float scale) {
    float acc = bias;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
        const int yy = y + ky - 1;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const int xx = x + kx - 1;
            if (unsigned(yy) < unsigned(H) && unsigned(xx) < unsigned(W))
                acc = __fadd_rn(acc, __ldg(taps + (int64_t(yy) * W + xx) * 9 + (ky * 3 + kx)));
        }
    }
    return sigmoid_scaled(acc, scale);
}

// one cost value under nastar_fwd_params.cost_kind (include/nastar_b200.h NASTAR_COST_*)
__device__ __forceinline__ float cost_value(int kind, const float* __restrict__ src, int y, int x, int H, int W,
                                            float bias, float scale) {
    if (kind == 0) return __ldg(src + y * W + x);
    if (kind == 1) return sigmoid_scaled(__ldg(src + y * W + x), scale);
    return cost_from_taps(src, y, x, H, W, bias, scale);
}

// Double-double accumulator for the running sums of the event-based backward (S = sum of exp(-f/sqrt(W)) over the
// open set, D = <Gh, v>).  Over a long search S decays by many orders of magnitude (the selected cell is always the
// LARGEST term): a plain fp64 running sum keeps an absolute error of 1e-16 x the early, large values, which becomes
// a large relative error once S has shrunk by 1e-10 or more (cost x10, 64x64 maps).  With an error-free TwoSum the
// pair (hi, lo) carries ~106 bits, so removed terms cancel exactly against the identical values added earlier.
__device__ __forceinline__ void dd_add(double& hi, double& lo, double x) {
    const double s = __dadd_rn(hi, x);
    const double bb = __dadd_rn(s, -hi);
    const double err = __dadd_rn(__dadd_rn(hi, -__dadd_rn(s, -bb)), __dadd_rn(x, -bb));
    lo = __dadd_rn(lo, err);
    const double t = __dadd_rn(s, lo);
    lo = __dadd_rn(lo, -__dadd_rn(t, -s));
    hi = t;
}

// The double-double keeps S exact (its terms are fp32 values), but D's terms Gh * dv are rounded products, so D keeps
// an absolute error of ~1e-16 x the large early terms.  After an exhaustive search (t_solve -2; cost x10, 64x64) the
// last open cells have v ~ e^-40 and that residue is larger than D itself, so b_t = D / S^2 is wrong.  Whenever S has
// fallen below kResumBelow x its largest value since the last resum, both sums are recomputed from the per-cell
// numerators: v = 0 outside the open set, so S = sum v and D = sum Gh * v.  The running error is then at most
// steps x 1e-16 x 2^16 of the current S.  S can only shrink 2^16-fold a handful of times (v >= e^-80 or so), so
// resums are rare.
constexpr double kResumBelow = 1.0 / 65536.0;

// Recompute (S, D) over cells lane, lane + 32, ... < n.  v_at(i) / gh_at(i): the cell's numerator and upstream
// gradient.  The xor butterfly leaves the same sums in every lane.  Warp-uniform; syncs the warp first.
template <class VAt, class GhAt>
__device__ __forceinline__ void bwd_resum(int lane, int n, VAt v_at, GhAt gh_at, double& S, double& Slo, double& D,
                                          double& Dlo, double& Smax) {
    __syncwarp();
    double s = 0.0, d = 0.0;
    for (int i = lane; i < n; i += 32) {
        const float v = v_at(i);
        if (v != 0.f) {
            s += double(v);
            d += double(gh_at(i)) * double(v);
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        s += __shfl_xor_sync(kFull, s, o);
        d += __shfl_xor_sync(kFull, d, o);
    }
    S = s;
    Slo = 0.0;
    D = d;
    Dlo = 0.0;
    Smax = s;
}

// At the top of each backward step: resum when S has shrunk kResumBelow-fold since the last resum, else track its max.
template <class VAt, class GhAt>
__device__ __forceinline__ void bwd_track(int lane, int n, VAt v_at, GhAt gh_at, double& S, double& Slo, double& D,
                                          double& Dlo, double& Smax) {
    const double s = S + Slo;
    if (s < Smax * kResumBelow) bwd_resum(lane, n, v_at, gh_at, S, Slo, D, Dlo, Smax);
    else Smax = fmax(Smax, s);
}

// The prefix sums A = sum 1/S and B = sum D/S^2 only grow, and a cell's term is v * (Gh * (A - a0) - (B - b0)): a
// difference of two prefix sums with an fp64 error of ~1e-16 x A.  When S grows over a search (low g_ratio, where f
// falls as the search nears the goal) the early steps' 1/S dwarf the late ones, and a late interval loses the ratio
// S_late / S_early of its precision (up to e^45 corner to corner at 2048 wide, g_ratio 0).  Whenever A exceeds kRebaseAbove x this
// step's 1/S, every open cell's partial term is folded into its acc and A, B and the cells' a0, b0 restart from 0,
// which leaves every interval's difference within 1e-16 x kRebaseAbove of a single step's term.  While S stays level
// that happens once per kRebaseAbove steps; each rebase is O(N).
constexpr double kRebaseAbove = 65536.0;

// Fold the open cells lane, lane + 32, ... < n into acc and restart the prefix sums.  Warp-uniform; syncs the warp
// before and after.
template <class GhAt>
__device__ __forceinline__ void bwd_rebase(int lane, int n, const float* v, GhAt gh_at, double* acc, double* a0,
                                           double* b0, double& A, double& B) {
    __syncwarp();
    for (int i = lane; i < n; i += 32) {
        const float vi = v[i];
        if (vi != 0.f) {
            acc[i] += double(vi) * (double(gh_at(i)) * (A - a0[i]) - (B - b0[i]));
            a0[i] = 0.0;
            b0[i] = 0.0;
        }
    }
    __syncwarp();
    A = 0.0;
    B = 0.0;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier + 1-D TMA bulk copy (cp.async.bulk -> SASS UBLKCP) -------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}

__device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace nastar
