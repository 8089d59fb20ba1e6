// nastar_warp32.cuh — warp-resident engine for maps with H <= 32 and W <= 32 (forward + backward).
//
// Replaces the T-step loop + backtrack of DifferentiableAstar.forward
// (/root/reference/src/neural_astar/planner/differentiable_astar.py:187-255) and the autograd
// through it, one map per warp.  Design (DESIGN.md "warp32 engine"):
//   * the map lives in shared memory in a PADDED 32x32 layout (cell id rc = y*32 + x), so every
//     index is a shift/mask and every plane sits at a compile-time offset;
//   * lane y owns grid row y: passable / open / closed rows are 32-bit masks in registers, and
//     the lane caches its row's best open cell (order-preserving f key, column);
//   * node selection (:206-209; softmax+argmax == arg-min of (f, flat index), SURVEY App. A.2)
//     is two REDUX.MINs over the 32 cached row minima: min key, then min (row<<5|col) among ties;
//   * expansion (:228-249) touches <= 8 cells in rows r-1..r+1: those three lanes relax their
//     <= 3 cells with branch-free mask algebra and fold the new keys into their cached minimum —
//     insertions/decreases never need a rescan;
//   * only row r lost its minimum (the selected cell): all 32 lanes rescan that one row (one
//     conflict-free LDS + two REDUX.MINs), overlapped with the expansion's dependency chain;
//   * planes are staged with 1-D TMA bulk copies (cp.async.bulk + mbarrier) when W == 32 and
//     results leave as coalesced 128-bit stores; the loop itself never touches HBM.
//   kBwd = true replays the same state machine and accumulates the closed-form gradient of the
//   straight-through softmax (SURVEY App. B) — same code path, so the replay cannot drift; the
//   accumulation is event-based (a cell's softmax weight only changes when it is opened, relaxed or
//   closed: per-cell interval bookkeeping against fp64 prefix sums, O(1) per step).
#pragma once
#include "nastar_engine.cuh"

namespace nastar {

// backward-only planes (dynamic shared memory), event-based closed form (see nastar_generic.cuh / DESIGN.md):
struct __align__(16) W32Bwd {
    double acc[kCells];   // closed intervals: sum of v * (Gh * dA - dB)
    double a0[kCells];    // A(t0), B(t0) of the cell's current open interval
    double b0[kCells];
    float v[kCells];      // softmax numerator exp(-f/sqrt(W)) of open cells, else 0
    float gh[kCells];     // upstream gradient (goal zeroed when the clamp blocks it)
};

struct __align__(16) W32Smem {
    float cost[kCells];        // staged cost plane (padded)
    uint32_t key[kCells];      // order-preserving key of f = g_ratio*g + (1-g_ratio)*h, opened cells only
    float2 ghbuf[kCells + 4];  // {g, h} per cell at ghbuf[2 + rc]; 2 guard cells on either side make the
                               // c-1 / c+1 window loads of the first/last cell addressable (16-B aligned body)
    int8_t par[kCells];        // parent link of opened cells as a signed offset: parent = rc - par[rc], in [-33, 33]
    uint32_t open_row[32];     // every lane's open row, refreshed each step (rescan input)
    uint32_t bits_a[32];       // closed rows for the epilogue
    uint32_t bits_b[32];       // path rows for the epilogue
    unsigned long long bar;    // mbarrier for the TMA prologue
};

// kExit (forward only): kExitEarly, kExitNone (NASTAR_FWD_NO_EARLY_EXIT — keep stepping after the solve step, exactly
// T steps) or a pass of the coupled forward, kExitCoupled1 / kExitCoupled2 (nastar_common.cuh).
// kFused (forward only): the prologue may have to finish the encoder (NASTAR_COST_LOGIT / NASTAR_COST_TAPS); kept out
// of the plain instantiation so that its cold instruction footprint stays small.
// kNews: NASTAR_FWD_NEWS / NASTAR_MECH_NEWS — 4-connected expansion (N, E, W, S) and the Manhattan heuristic.
// kMode: kExit, plus kExitBlackbox for the black-box backward (forward search on w', dL/dw in place of the outputs).
template <bool kTrace, bool kBwd, int kMode = kExitEarly, bool kFused = false, bool kNews = false>
__global__ void __launch_bounds__(32, 12) astar_warp32_kernel(const SearchArgs a) {
    // enumerators, not constexpr variables: the instantiations without kExitBlackbox then compile to the code they had
    // before the black-box backward existed
    enum : int { kExit = kMode & ~kExitBlackbox };
    enum : bool { kBB = (kMode & kExitBlackbox) != 0 };
    constexpr bool kContinue = kBwd || (kExit != kExitEarly);   // the loop does not stop at the solve step
    __shared__ W32Smem S;
    extern __shared__ __align__(16) unsigned char bwd_raw[];  // backward only: W32Bwd
    W32Bwd& Bw = *reinterpret_cast<W32Bwd*>(bwd_raw);
    const nastar_fwd_params& p = a.f;
    float2* const sGH = S.ghbuf + 2;
    const int lane = threadIdx.x;
    const int b = blockIdx.x;                    // output slot
    const int H = p.H, W = p.W, N = H * W;
    // NASTAR_FWD_PAIR: CTAs B..2B-1 search the same problems with cost = obstacles (VanillaAstar, astar.py:93-94)
    const bool vanilla_half = !kBwd && (p.flags & NASTAR_FWD_PAIR) && (b >= p.B);
    const int bi = vanilla_half ? (b - p.B) : b;  // input map

    const float* gStart = p.start + int64_t(bi) * p.start_stride;
    const float* gGoal = p.goal + int64_t(bi) * p.goal_stride;
    const float* gObst = p.obst + int64_t(bi) * p.obst_stride;
    const float* gCost = vanilla_half ? gObst : (p.cost + int64_t(bi) * p.cost_stride);
    const int cost_kind = (!kFused || kBwd || vanilla_half) ? NASTAR_COST_PLANE : p.cost_kind;
    const bool cost_plane = (cost_kind == NASTAR_COST_PLANE);
    const bool obst_is_cost = !kBB && cost_plane && (gObst == gCost);   // w' is never the obstacle plane
    if constexpr (kExit == kExitCoupled2) {
        const int Tc = *a.T_batch;
        if (a.cw.stop[b] <= Tc) {   // pass 1's outputs stand
            if (lane == 0) coupled_keep(a.cw, b, Tc, p.t_solve, p.n_steps);
            return;
        }
    }

    // ---------------- prologue: stage planes, build row masks ------------------------------
    uint32_t pass = 0u;
    int start_rc = -1, goal_rc = -1;
    const bool tma = !kBB && (W == 32) && (!cost_plane || aligned16(gCost)) && aligned16(gStart) && aligned16(gGoal) && aligned16(gObst);
    if (tma) {
        // flat layout == padded layout: bulk-copy whole planes (start/goal/obstacles are parked in the
        // f and {g,h} planes, which are not live yet)
        float* tStart = reinterpret_cast<float*>(S.key);
        float* tGoal = reinterpret_cast<float*>(sGH);
        float* tObst = tGoal + kCells;
        uint64_t* bar = reinterpret_cast<uint64_t*>(&S.bar);
        if (lane == 0) {
            mbar_init(bar, 1);
            fence_mbar_init();
            const uint32_t bytes = uint32_t(N) * 4u;
            mbar_expect_tx(bar, bytes * ((obst_is_cost ? 3u : 4u) - (cost_plane ? 0u : 1u)));
            if (cost_plane) tma_load_1d(S.cost, gCost, bytes, bar);
            tma_load_1d(tStart, gStart, bytes, bar);
            tma_load_1d(tGoal, gGoal, bytes, bar);
            if (!obst_is_cost) tma_load_1d(tObst, gObst, bytes, bar);
        }
        __syncwarp();
        if (kFused && !cost_plane) {
            // fused encoder hand-off (SURVEY 8(f)-3): the cost plane is produced here from the encoder's raw
            // output while the TMA copies of the other planes are in flight
#pragma unroll 4      // four rows of gathers in flight: the prologue is a chain of L2 round trips for one warp
            for (int y = 0; y < H; ++y)
                S.cost[(y << 5) + lane] = cost_value(cost_kind, gCost, y, lane, H, W, p.cost_bias, p.cost_scale);
        }
        mbar_wait(bar, 0);
        const float* sObst = obst_is_cost ? S.cost : tObst;
#pragma unroll 4
        for (int y = 0; y < H; ++y) {
            const int i = (y << 5) + lane;
            const uint32_t wo = __ballot_sync(kFull, sObst[i] != 0.f);
            const uint32_t ws = __ballot_sync(kFull, tStart[i] != 0.f);
            const uint32_t wg = __ballot_sync(kFull, tGoal[i] != 0.f);
            if (lane == y) pass = wo;
            if (start_rc < 0 && ws) start_rc = (y << 5) + __ffs(ws) - 1;
            if (goal_rc < 0 && wg) goal_rc = (y << 5) + __ffs(wg) - 1;
        }
    } else {
        // W < 32 (or unaligned planes): rows are shorter than a warp; issue 8 rows of loads per plane
        // before consuming them so that DRAM latency is paid H/8 times, not H times
        const bool in = lane < W;
        constexpr int kRows = 8;
        for (int y0 = 0; y0 < H; y0 += kRows) {
            float vc[kRows], vo[kRows], vs[kRows], vg[kRows];
#pragma unroll
            for (int u = 0; u < kRows; ++u) {
                const bool ok = in && (y0 + u < H);
                const int i = (y0 + u) * W + lane;
                vc[u] = ok ? (kFused ? cost_value(cost_kind, gCost, y0 + u, lane, H, W, p.cost_bias, p.cost_scale)
                                     : kBB ? bb_cost(gCost, a.grad_hist + int64_t(bi) * a.grad_stride, i, a.bb_lambda) : __ldg(gCost + i)) : 0.f;
                vo[u] = obst_is_cost ? vc[u] : (ok ? __ldg(gObst + i) : 0.f);
                vs[u] = ok ? __ldg(gStart + i) : 0.f;
                vg[u] = ok ? __ldg(gGoal + i) : 0.f;
            }
#pragma unroll
            for (int u = 0; u < kRows; ++u) {
                const int y = y0 + u;
                if (y < H) {
                    S.cost[(y << 5) + lane] = vc[u];
                    const uint32_t wo = __ballot_sync(kFull, vo[u] != 0.f);
                    const uint32_t ws = __ballot_sync(kFull, vs[u] != 0.f);
                    const uint32_t wg = __ballot_sync(kFull, vg[u] != 0.f);
                    if (lane == y) pass = wo;
                    if (start_rc < 0 && ws) start_rc = (y << 5) + __ffs(ws) - 1;
                    if (goal_rc < 0 && wg) goal_rc = (y << 5) + __ffs(wg) - 1;
                }
            }
        }
    }
    if (goal_rc < 0) goal_rc = 0;  // argmax of an all-zero plane (differentiable_astar.py:197)
    const int gy = goal_rc >> 5, gx = goal_rc & 31;
    __syncwarp();
    // h = heuristic + cost (:191-192), one row per iteration; overwrites the parked planes
    {
        const int adx = (lane > gx) ? (lane - gx) : (gx - lane);
#pragma unroll 8
        for (int y = 0; y < H; ++y) {
            const int i = (y << 5) + lane;
            const int ady = (y > gy) ? (y - gy) : (gy - y);
            sGH[i] = make_float2(0.f, __fadd_rn(__ldg(&g_heur32[(kNews ? kCells : 0) + ((ady << 5) | adx)]), S.cost[i]));
        }
    }
    __syncwarp();

    const float gr = p.g_ratio, omg = p.one_minus_g_ratio;
    uint32_t open = 0u, closed = 0u;
    uint32_t rm_key = kKeyInf;
    int rm_col = 0;

    // backward: running sums replicated in every lane (S = sum of v over the open set, D = <Gh, v>, A / B = prefix
    // sums of 1/S and D/S^2 over the executed steps)
    double Ssum = 0.0, Slo = 0.0, Dsum = 0.0, Dlo = 0.0, Acum = 0.0, Bcum = 0.0;   // (Ssum,Slo), (Dsum,Dlo): double-double
    double Smax = 0.0;   // largest S since the last resum (bwd_track)
    bool s_zero = false;   // a step at which every open numerator underflowed to 0: the map's gradient is NaN
    int Tb = 0, ts_in = NASTAR_TS_CAPPED;
    if (kBwd) {
        Tb = *a.T_batch;
        ts_in = a.t_solve_in[b];
        const float* gG = a.grad_hist + int64_t(b) * a.grad_stride;
        // clamp(hist + sel) blocks the gradient at a goal that is re-selected after its solve step
        // (pre-clamp value 2, differentiable_astar.py:222-223; SURVEY App. B)
        const bool blocked = (ts_in >= 0) && (ts_in < Tb - 1);
        for (int y = 0; y < 32; ++y) {
            const int i = (y << 5) + lane;
            Bw.acc[i] = 0.0;
            Bw.v[i] = 0.f;
            Bw.gh[i] = (y < H && lane < W && !(blocked && i == goal_rc)) ? __ldg(gG + y * W + lane) : 0.f;
        }
        __syncwarp();
    }
    if constexpr (kExit == kExitCoupled2) Tb = *a.T_batch;   // pass 2 runs T_batch steps
    if (lane == 0) S.par[goal_rc] = 0;  // parents are initialised to the goal (:195-198): a self link at the goal
    if (start_rc >= 0) {
        const float f0 = f_value(gr, omg, 0.f, sGH[start_rc].y);
        if (lane == 0) {
            S.key[start_rc] = fkey(f0);              // g = 0 already (:193)
            if (kBwd) { Bw.v[start_rc] = expf(__fdiv_rn(-f0, a.sqrt_w)); Bw.a0[start_rc] = 0.0; Bw.b0[start_rc] = 0.0; }  // :207
        }
        if (lane == (start_rc >> 5)) {
            open = 1u << (start_rc & 31);            // open_maps = start_maps (:187)
            rm_key = fkey(f0);
            rm_col = start_rc & 31;
        }
    }
    S.open_row[lane] = open;
    __syncwarp();
    if (kBwd && start_rc >= 0) {
        Ssum = double(Bw.v[start_rc]);
        Dsum = double(Bw.gh[start_rc]) * Ssum;
    }

    // ---------------- the search loop (differentiable_astar.py:203-252) --------------------
    const int T = (kBwd || kExit == kExitCoupled2) ? Tb : p.T;
    // post-solve steps are stationary when g_ratio >= 0.5 (the goal keeps being re-selected and
    // nothing changes, SURVEY App. A.4): the backward then adds them in one go
    const bool stationary_ok = (gr >= 0.5f);
    int t_solve = NASTAR_TS_CAPPED;
    int32_t* trace = kTrace ? (p.trace + int64_t(b) * p.T) : nullptr;
    const float2* ghrow = sGH + (lane << 5);      // this lane's row of {g,h}
    uint32_t gbits = 0u;          // pass 1: at-goal bits of the current 32-step word
    int t = 0;
    for (; t < T; ++t) {
        // -- select: lexicographic arg-min of (f key, row, col) with two REDUX.MINs -----------
        const uint32_t m = __reduce_min_sync(kFull, rm_key);
        if (m == kKeyInf) { t_solve = NASTAR_TS_EXHAUSTED; break; }
        double A1 = 0.0, B1 = 0.0;   // prefix sums INCLUDING step t (the events of step t act from t+1 on)
        if (kBwd) {
            bwd_track(lane, kCells, [&](int i) { return Bw.v[i]; }, [&](int i) { return Bw.gh[i]; }, Ssum, Slo, Dsum,
                      Dlo, Smax);
            const double inv = 1.0 / (Ssum + Slo);
            s_zero |= (Ssum + Slo == 0.0);
            const double a_t = inv, b_t = (Dsum + Dlo) * inv * inv;
            if (Acum > kRebaseAbove * a_t)
                bwd_rebase(lane, kCells, Bw.v, [&](int i) { return Bw.gh[i]; }, Bw.acc, Bw.a0, Bw.b0, Acum, Bcum);
            if (stationary_ok && (ts_in >= 0) && (t == ts_in + 1)) {
                // solved: the goal is re-selected with a frozen open set until step T_batch-1 (App. A.4)
                Acum += double(Tb - t) * a_t;
                Bcum += double(Tb - t) * b_t;
                break;
            }
            A1 = Acum + a_t;
            B1 = Bcum + b_t;
        }
        const uint32_t ind = __reduce_min_sync(kFull, (rm_key == m) ? uint32_t((lane << 5) | rm_col) : 0xFFFFFFFFu);
        const int r = int(ind >> 5), c = int(ind & 31u);
        if (kTrace && lane == 0) trace[t] = r * W + c;
        const bool solved = (int(ind) == goal_rc);          // :219-220
        if constexpr (kExit == kExitCoupled1) {
            gbits |= uint32_t(solved) << (t & 31);
            if ((t & 31) == 31) {
                if (lane == 0) a.cw.bits[int64_t(b) * a.cw.words + (t >> 5)] = gbits;
                gbits = 0u;
            }
        }
        const uint32_t m1 = 1u << c;                        // column masks of the 3-wide window;
        const uint32_t m0 = m1 >> 1, m2 = m1 << 1;          // they fall off the row at c == 0 / 31
        // -- rescan inputs for row r (pre-expansion open cells minus the selected one); stale f
        //    values of cells relaxed this step are upper bounds and the fresh keys are merged below
        const uint32_t open_r = (kContinue && solved) ? S.open_row[r] : (S.open_row[r] & ~m1);
        const uint32_t krs = S.key[(r << 5) + lane];
        const uint32_t rs_key = ((open_r >> lane) & 1u) ? krs : kKeyInf;
        // the rescan's two reductions are issued here, ahead of the expansion's ALU chain, so that their latency
        // overlaps it instead of extending the tail of the step (their inputs are pre-step values only)
        const uint32_t mr = __reduce_min_sync(kFull, rs_key);
        const uint32_t mc = __reduce_min_sync(kFull, (rs_key == mr) ? uint32_t(lane) : 0xFFFFFFFFu);
        // -- expansion inputs ----------------------------------------------------------------
        const int dr = lane - r;
        const bool isr = (dr == 0);
        const bool near = (unsigned(dr + 1) <= 2u);
        // only the three row lanes load (rows are 256 B apart = same banks; 32 lanes would serialise)
        float2 n0 = make_float2(0.f, 0.f), n1 = n0, n2 = n0;
        if (near) { n0 = ghrow[c - 1]; n1 = ghrow[c]; n2 = ghrow[c + 1]; }   // guard cells make c-1/c+1 safe
        const float g2 = __fadd_rn(sGH[ind].x, S.cost[ind]);               // :234, cost of the SELECTED node
        __syncwarp();   // every shared-memory read of this step precedes every write below (no intra-warp WAR)
        // -- closed/open update of the selected cell (:222-225) ------------------------------
        if (isr) {
            closed |= m1;
            if (!solved) open &= ~m1;                       // the goal stays open once selected
            rm_key = kKeyInf;                               // this row's minimum is rebuilt below
        }
        // -- expansion (:228-249) as mask algebra on this lane's row ---------------------------
        //    idx = ((1-open)(1-hist) + open*(g > g2)) * neighbours * obstacles   (:235-236)
        //    NEWS: the own row's left/right neighbours, and only column c of the rows above and below
        const uint32_t win = isr ? (m0 | m2) : (kNews ? m1 : (m0 | m1 | m2));
        const uint32_t cand = near ? (win & pass) : 0u;
        const uint32_t gt = ((n0.x > g2) ? m0 : 0u) | ((n1.x > g2) ? m1 : 0u) | ((n2.x > g2) ? m2 : 0u);
        const uint32_t upd = cand & ((open & gt) | ~(open | closed));
        open |= upd;                                        // :242
        const float ag = __fmul_rn(gr, g2);
        const float f0n = __fadd_rn(ag, __fmul_rn(omg, n0.y));
        const float f1n = __fadd_rn(ag, __fmul_rn(omg, n1.y));
        const float f2n = __fadd_rn(ag, __fmul_rn(omg, n2.y));
        const bool u0 = (upd & m0) != 0u, u1 = (upd & m1) != 0u, u2 = (upd & m2) != 0u;
        const int cell = (lane << 5) + c;
        const uint32_t q0 = fkey(f0n), q1 = fkey(f1n), q2 = fkey(f2n);
        const int off = (dr << 5) - 1;                      // (this row, column c-1) minus the selected cell
        if (u0) { sGH[cell - 1].x = g2; S.key[cell - 1] = q0; S.par[cell - 1] = int8_t(off); }       // :238, :246-249
        if (u1) { sGH[cell].x = g2;     S.key[cell] = q1;     S.par[cell] = int8_t(off + 1); }
        if (u2) { sGH[cell + 1].x = g2; S.key[cell + 1] = q2; S.par[cell + 1] = int8_t(off + 2); }
        if (kBwd) {
            double dS = 0.0, dD = 0.0;   // this lane's change of S and D
            auto event = [&](int cl, float v_new) {
                const float v_old = Bw.v[cl];
                const double gh = double(Bw.gh[cl]);
                if (v_old != 0.f) Bw.acc[cl] += double(v_old) * (gh * (A1 - Bw.a0[cl]) - (B1 - Bw.b0[cl]));
                Bw.v[cl] = v_new;
                Bw.a0[cl] = A1;
                Bw.b0[cl] = B1;
                const double dv = double(v_new) - double(v_old);
                dS += dv;
                dD += gh * dv;
            };
            if (u0) event(cell - 1, expf(__fdiv_rn(-f0n, a.sqrt_w)));   // :207
            if (u1) event(cell, expf(__fdiv_rn(-f1n, a.sqrt_w)));
            if (u2) event(cell + 1, expf(__fdiv_rn(-f2n, a.sqrt_w)));
            if (isr && !solved) event(int(ind), 0.f);                    // the selected cell leaves the open set
            // the events sit on the lanes of rows r-1, r, r+1
            const double s0 = __shfl_sync(kFull, dS, max(r - 1, 0)), s1 = __shfl_sync(kFull, dS, r),
                         s2 = __shfl_sync(kFull, dS, min(r + 1, 31));
            const double d0 = __shfl_sync(kFull, dD, max(r - 1, 0)), d1 = __shfl_sync(kFull, dD, r),
                         d2 = __shfl_sync(kFull, dD, min(r + 1, 31));
            dd_add(Ssum, Slo, (r > 0 ? s0 : 0.0) + s1 + (r < 31 ? s2 : 0.0));
            dd_add(Dsum, Dlo, (r > 0 ? d0 : 0.0) + d1 + (r < 31 ? d2 : 0.0));
            Acum = A1;
            Bcum = B1;
        }
        // fold the fresh keys (ascending column, strict < keeps the lowest column on ties)
        const uint32_t k0 = u0 ? q0 : kKeyInf, k1 = u1 ? q1 : kKeyInf, k2 = u2 ? q2 : kKeyInf;
        uint32_t bk = k0;
        int bc = c - 1;
        if (k1 < bk) { bk = k1; bc = c; }
        if (k2 < bk) { bk = k2; bc = c + 1; }
        if ((bk < rm_key) | ((bk == rm_key) & (bc < rm_col))) { rm_key = bk; rm_col = bc; }
        if (solved && t_solve < 0) t_solve = t;             // first step at which the goal was selected
        if (!kContinue && solved) break;                    // :251-252 (per-map early exit, App. A.4)
        if constexpr (kExit == kExitCoupled1) {
            // the goal, closed at an earlier step, is selected again and nothing is opened or relaxed: the state after
            // this step is the state before it, so every later step repeats it (fixed point)
            if (solved && t_solve < t && !__any_sync(kFull, upd != 0u)) { ++t; break; }
        }
        if (near) S.open_row[lane] = open;
        // -- fold the rescan into lane r's cached minimum -------------------------------------
        const bool take = isr & ((mr < rm_key) | ((mr == rm_key) & (int(mc) < rm_col)));
        rm_key = take ? mr : rm_key;
        rm_col = take ? int(mc) : rm_col;
        __syncwarp();
    }
    __syncwarp();
    // selection steps executed: t on exhaustion / cap, t+1 when the loop left through the solve step
    const int steps = (!kContinue && t_solve >= 0) ? (t + 1) : t;
    if constexpr (kExit == kExitCoupled1) if (lane == 0) {
        if (t & 31) a.cw.bits[int64_t(b) * a.cw.words + (t >> 5)] = gbits;   // the last, partial word
        a.cw.stop[b] = t;
        // left before the cap with the goal selected: the fixed point (a fixed point at step T-1 looks capped, which
        // is the same record: no step past the cap is ever read)
        a.cw.end[b] = (t_solve == NASTAR_TS_EXHAUSTED) ? kEndExhausted : ((t < T) ? kEndFixed : kEndCapped);
        a.cw.first[b] = t_solve;
    }

    if constexpr (kBB) {
        // black-box backward: dL/dw = (closed rows of this search on w' - the forward's histories) / lambda
        S.bits_a[lane] = closed;
        __syncwarp();
        const float* gY = a.bb_hist + int64_t(b) * N;
        float* gOut = a.grad_cost + int64_t(b) * N;
        for (int y = 0; y < H; ++y) {
            const int i = y * W + lane;
            if (lane < W) gOut[i] = bb_grad((S.bits_a[y] >> lane) & 1u, __ldg(gY + i), a.bb_lambda);
        }
        return;
    }

    if (kBwd) {
        // close the intervals of the cells still open; dL/dcost = -(1-g_ratio)/sqrt(W) * acc
        // (h = heuristic + cost, f = g_ratio*g + (1-g_ratio)*h)
        const double coef = -double(omg) / double(a.sqrt_w);
        float* gOut = a.grad_cost + int64_t(b) * N;
        for (int y = 0; y < H; ++y) {
            const int i = (y << 5) + lane;
            if (lane < W) {
                double acc = Bw.acc[i];
                const float v = Bw.v[i];
                if (v != 0.f) acc += double(v) * (double(Bw.gh[i]) * (Acum - Bw.a0[i]) - (Bcum - Bw.b0[i]));
                gOut[y * W + lane] = s_zero ? __int_as_float(0x7fc00000) : float(coef * acc);
            }
        }
        return;
    }

    // ---------------- backtrack (differentiable_astar.py:96-125, App. A.3) ------------------
    uint32_t path = 0u;
    {
        if (lane == gy) path |= 1u << gx;
        // the start's parent is the goal in the reference (the initial value); the walk stops at the start
        // before following it, which marks the same cells (App. A.3)
        int loc = goal_rc - S.par[goal_rc];
        const int hops = (t_solve >= 0) ? N : ((kExit == kExitCoupled2 ? T : p.T) - 1);
        for (int k = 0; k < hops; ++k) {
            if (lane == (loc >> 5)) path |= 1u << (loc & 31);
            if (loc == start_rc || loc == goal_rc) break;   // reached the start (or the goal's self link)
            loc -= S.par[loc];
        }
    }

    // ---------------- epilogue: coalesced stores of histories / paths -----------------------
    S.bits_a[lane] = closed;
    S.bits_b[lane] = path;
    __syncwarp();
    float* gHist = p.histories + int64_t(b) * N;
    long long* gPath = reinterpret_cast<long long*>(p.paths) + int64_t(b) * N;
    if (W == 32 && aligned16(gHist) && aligned16(gPath)) {
        const int x = (lane & 7) << 2;
#pragma unroll 4
        for (int j = 0; j < 8; ++j) {
            const int y = (lane >> 3) + 4 * j;
            if (y < H) {
                const int i4 = lane + 32 * j;
                store_cells4(gHist, gPath, i4, S.bits_a[y] >> x, S.bits_b[y] >> x);
            }
        }
    } else {
        for (int y = 0; y < H; ++y) {
            if (lane < W) {
                gHist[y * W + lane] = ((S.bits_a[y] >> lane) & 1u) ? 1.f : 0.f;
                gPath[y * W + lane] = ((S.bits_b[y] >> lane) & 1u) ? 1ll : 0ll;
            }
        }
    }
    // per-map counts for the validation metrics (utils/training.py:71-85): histories.sum(), paths.sum()
    const int n_closed = __reduce_add_sync(kFull, __popc(closed));
    const int n_path = __reduce_add_sync(kFull, __popc(path));
    if (lane == 0) {
        if (p.t_solve) p.t_solve[b] = t_solve;
        if (p.n_steps) p.n_steps[b] = steps;
        if (p.n_closed) p.n_closed[b] = n_closed;
        if (p.path_len) p.path_len[b] = n_path;
    }
}

}  // namespace nastar
