// nastar_engine.cuh — what the search engines (nastar_warp32.cuh, nastar_warp64.cuh, nastar_generic.cuh, and the
// output stores of nastar_bin16.cuh) share: the kernel arguments, the heuristic tables and the output stores.
//
// The backward's event bookkeeping, the coupled forward's records and the per-map counter stores stay written out in
// each engine.  Moved into __forceinline__ helpers, even a predicate such as the goal clamp makes nvcc canonicalise the
// surrounding code differently and changes the engines' SASS; the step loops are kept instruction for instruction.
#pragma once
#include "../../include/nastar_b200.h"
#include "nastar_common.cuh"

namespace nastar {

// Kernel arguments of every search engine: the forward parameters plus the extra fields of nastar_bwd_params.
struct SearchArgs {
    nastar_fwd_params f;
    // backward only
    float sqrt_w;
    const int32_t* T_batch;     // device scalar: loop iterations the reference would execute
    const int32_t* t_solve_in;  // forward's t_solve[] (goal clamp blocking, App. B)
    const float* grad_hist;
    int64_t grad_stride;
    float* grad_cost;
    // coupled forward only (kExitCoupled1 / kExitCoupled2; pass 2 also reads *T_batch)
    CoupledWs cw;
    // generic engine's forward only, nullable: per-map flags written by the bin16 engine (nastar_bin16.cuh); when
    // given, only maps with redo[b] != 0 are processed (the others were already finished on-chip)
    const int32_t* redo;
    // black-box backward only (kExitBlackbox): grad_hist / grad_stride carry dL/dhistories and grad_cost receives dL/dw
    float bb_lambda;            // lambda > 0
    const float* bb_hist;       // the forward's histories y(w), [B][H*W]
};

// ---- heuristic tables -----------------------------------------------------------------------------------------
constexpr int kCells = 1024;    // padded 32 x 32
constexpr int kCells64 = 4096;  // padded 64 x 64

// heuristic(|dy|, |dx|) for every offset on a 32x32 / 64x64 grid, filled once per device by heur_init_kernel with the
// very same device function the generic engine evaluates inline — the per-map h pass of engines 1 and 4 becomes one
// cached load + one add per cell instead of an IEEE sqrt chain.  The second half of each array holds the NEWS
// heuristic (heuristic_news) the same way; it shares the array so that every kernel keeps its global address table.
__device__ float g_heur32[2 * kCells];
__device__ float g_heur64[2 * kCells64];

template <int kSide, bool kNews>
__global__ void heur_init_kernel() {
    constexpr int kN = kSide * kSide, kShift = (kSide == 32) ? 5 : 6;
    static_assert(kSide == 32 || kSide == 64, "tables exist for 32x32 and 64x64");
    const int i = threadIdx.x + blockIdx.x * blockDim.x;
    float* const table = (kSide == 32) ? g_heur32 : g_heur64;
    if (i < kN) table[(kNews ? kN : 0) + i] = heuristic_of<kNews>(i >> kShift, i & (kSide - 1), 0, 0);
}

// ---- black-box backward -----------------------------------------------------------------------------------------
// cell i of w' = fl(w + fl(lambda * g)): two roundings, no FMA, no clamp (w' may be negative)
__device__ __forceinline__ float bb_cost(const float* cost, const float* grad, int i, float lam) {
    return __fadd_rn(__ldg(cost + i), __fmul_rn(lam, __ldg(grad + i)));
}

// dL/dw of one cell: (y' - y) / lambda, y' = closed after the search on w', y = the forward's histories; exactly 0 or
// +-fl(1/lambda)
__device__ __forceinline__ float bb_grad(bool closed, float y, float lam) {
    return __fdiv_rn((closed ? 1.f : 0.f) - y, lam);
}

// ---- outputs ----------------------------------------------------------------------------------------------------
// cells 4q .. 4q+3 from the low four bits of cb (histories) and pb (paths): one float4 store and two longlong2 stores;
// hist and path must be 16-byte aligned
__device__ __forceinline__ void store_cells4(float* hist, long long* path, int q, uint32_t cb, uint32_t pb) {
    reinterpret_cast<float4*>(hist)[q] = make_float4((cb & 1u) ? 1.f : 0.f, (cb & 2u) ? 1.f : 0.f,
                                                     (cb & 4u) ? 1.f : 0.f, (cb & 8u) ? 1.f : 0.f);
    reinterpret_cast<longlong2*>(path)[2 * q] = make_longlong2((pb & 1u) ? 1ll : 0ll, (pb & 2u) ? 1ll : 0ll);
    reinterpret_cast<longlong2*>(path)[2 * q + 1] = make_longlong2((pb & 4u) ? 1ll : 0ll, (pb & 8u) ? 1ll : 0ll);
}

}  // namespace nastar
