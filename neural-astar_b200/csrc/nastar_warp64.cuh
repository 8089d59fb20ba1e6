// nastar_warp64.cuh — warp-resident forward engine for maps with H <= 64 and W <= 64 (not both <= 32).
//
// Same state machine and step structure as the warp32 engine (nastar_warp32.cuh; replaces the loop +
// backtrack of /root/reference/src/neural_astar/planner/differentiable_astar.py:187-255), scaled to the
// reference's 64x64 inputs (its own test fixture, tests/astar_test.py:5-14, and the all_064 dataset):
//   * padded 64x64 layout in shared memory (cell id rc = y*64 + x), ~70 KB per map, 3 maps per SM;
//   * lane l owns rows l and l+32: two 64-bit passable/open/closed masks and two cached row minima;
//   * selection = local min of the lane's two rows, then the same two REDUX.MINs;
//   * expansion: of a lane's two rows at most one is within r-1..r+1, so the row lanes pick that slot
//     with selects and run the same branch-free 3-cell mask algebra on 64-bit masks;
//   * rescan of row r: every lane checks columns l and l+32.
// kBwd = true replays the same state machine for *T_batch steps and evaluates the closed-form gradient (SURVEY App. B)
// EVENT-BASED, like the generic engine (nastar_generic.cuh): a cell's softmax weight v = exp(-f/sqrt(W)) only changes
// when the cell is opened, relaxed or closed, so its contribution over an interval of constant v is
// v * (Gh * (A(t1)-A(t0)) - (B(t1)-B(t0))) with A, B the prefix sums of 1/S_t and D_t/S_t^2 (S = sum of v over the open
// set, D = <Gh, v>, both maintained in fp64 from the <= 10 events of a step).  Per-cell v / A(t0) / B(t0) / acc and
// the upstream gradient live in shared memory next to the forward state (198 KB per map).
#pragma once
#include "nastar_engine.cuh"

namespace nastar {

struct __align__(16) W64Smem {
    float cost[kCells64];
    uint32_t key[kCells64];         // order-preserving key of f, opened cells only
    float2 ghbuf[kCells64 + 4];     // {g,h} at ghbuf[2 + rc], guard cells on both sides
    int8_t par[kCells64];           // parent = rc - par[rc], offsets in [-65, 65]
    unsigned long long open_row[64];
    unsigned long long bits_a[64];  // closed rows (epilogue)
    unsigned long long bits_b[64];  // path rows (epilogue)
    unsigned long long bar;
};

// backward-only shared-memory planes (dynamic shared memory right behind W64Smem)
struct __align__(16) W64Bwd {
    double acc[kCells64];   // closed intervals: sum of v * (Gh * dA - dB)
    double a0[kCells64];    // A(t0), B(t0) of the cell's current open interval
    double b0[kCells64];
    float v[kCells64];      // current softmax numerator of the cell, 0 if it is not open
    float gh[kCells64];     // upstream gradient dL/dhistories (goal zeroed when the clamp blocks it)
};

// kFused (forward only): the prologue may have to finish the encoder (NASTAR_COST_LOGIT / NASTAR_COST_TAPS), as in the
// 32-wide engine; kept out of the plain instantiations.
// kNews: 4-connected expansion and the Manhattan heuristic, as in the 32-wide engine.
// kMode: exit mode of the forward (kExitEarly, kExitNone, or a pass of the coupled forward), plus kExitBlackbox for the
// black-box backward, as in the 32-wide engine.
template <bool kTrace, int kMode, bool kBwd = false, bool kFused = false, bool kNews = false>
__global__ void __launch_bounds__(32) astar_warp64_kernel(const SearchArgs a) {
    // enumerators, not constexpr variables: the instantiations without kExitBlackbox then compile to the code they had
    // before the black-box backward existed
    enum : int { kExit = kMode & ~kExitBlackbox };
    enum : bool { kBB = (kMode & kExitBlackbox) != 0 };
    constexpr bool kContinue = kBwd || (kExit != kExitEarly);
    const nastar_fwd_params& p = a.f;
    extern __shared__ __align__(16) unsigned char smem64_raw[];
    W64Smem& S = *reinterpret_cast<W64Smem*>(smem64_raw);
    W64Bwd& Bw = *reinterpret_cast<W64Bwd*>(smem64_raw + sizeof(W64Smem));
    float2* const sGH = S.ghbuf + 2;
    const int lane = threadIdx.x;
    const int b = blockIdx.x;
    const int H = p.H, W = p.W, N = H * W;
    typedef unsigned long long u64;

    const float* gCost = p.cost + int64_t(b) * p.cost_stride;
    const float* gStart = p.start + int64_t(b) * p.start_stride;
    const float* gGoal = p.goal + int64_t(b) * p.goal_stride;
    const float* gObst = p.obst + int64_t(b) * p.obst_stride;
    const int cost_kind = (kFused && !kBwd) ? p.cost_kind : NASTAR_COST_PLANE;
    const bool cost_plane = (cost_kind == NASTAR_COST_PLANE);
    const bool obst_is_cost = !kBB && cost_plane && (gObst == gCost);   // w' is never the obstacle plane
    if constexpr (kExit == kExitCoupled2) {
        const int Tc = *a.T_batch;
        if (a.cw.stop[b] <= Tc) {   // pass 1's outputs stand
            if (lane == 0) coupled_keep(a.cw, b, Tc, p.t_solve, p.n_steps);
            return;
        }
    }

    // ---------------- prologue ----------------------------------------------------------------
    u64 pass[2] = {0ull, 0ull};
    int start_rc = -1, goal_rc = -1;
    const bool tma = !kBB && (W == 64) && (!cost_plane || aligned16(gCost)) && aligned16(gStart) && aligned16(gGoal) && aligned16(gObst);
    if (tma) {
        float* tStart = reinterpret_cast<float*>(S.key);
        float* tGoal = reinterpret_cast<float*>(sGH);
        float* tObst = tGoal + kCells64;
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
            // fused encoder hand-off: the cost plane is produced here from the encoder's raw output while the TMA copies
            // of the other planes are in flight
#pragma unroll 2
            for (int y = 0; y < H; ++y) {
                S.cost[(y << 6) + lane] = cost_value(cost_kind, gCost, y, lane, H, W, p.cost_bias, p.cost_scale);
                S.cost[(y << 6) + lane + 32] = cost_value(cost_kind, gCost, y, lane + 32, H, W, p.cost_bias, p.cost_scale);
            }
        }
        mbar_wait(bar, 0);
        const float* sObst = obst_is_cost ? S.cost : tObst;
#pragma unroll 2
        for (int y = 0; y < H; ++y) {
            const int i = (y << 6) + lane;
            const uint32_t wo0 = __ballot_sync(kFull, sObst[i] != 0.f), wo1 = __ballot_sync(kFull, sObst[i + 32] != 0.f);
            const uint32_t ws0 = __ballot_sync(kFull, tStart[i] != 0.f), ws1 = __ballot_sync(kFull, tStart[i + 32] != 0.f);
            const uint32_t wg0 = __ballot_sync(kFull, tGoal[i] != 0.f), wg1 = __ballot_sync(kFull, tGoal[i + 32] != 0.f);
            if (lane == (y & 31)) {
                if (y >> 5) pass[1] = u64(wo0) | (u64(wo1) << 32);
                else pass[0] = u64(wo0) | (u64(wo1) << 32);
            }
            if (start_rc < 0 && (ws0 | ws1)) start_rc = (y << 6) + (ws0 ? __ffs(ws0) - 1 : 32 + __ffs(ws1) - 1);
            if (goal_rc < 0 && (wg0 | wg1)) goal_rc = (y << 6) + (wg0 ? __ffs(wg0) - 1 : 32 + __ffs(wg1) - 1);
        }
    } else {
        const bool in0 = lane < W, in1 = lane + 32 < W;
        constexpr int kRows = 4;
        for (int y0 = 0; y0 < H; y0 += kRows) {
            float vc[kRows][2], vo[kRows][2], vs[kRows][2], vg[kRows][2];
#pragma unroll
            for (int u = 0; u < kRows; ++u) {
#pragma unroll
                for (int hf = 0; hf < 2; ++hf) {
                    const bool ok = (hf ? in1 : in0) && (y0 + u < H);
                    const int i = (y0 + u) * W + lane + 32 * hf;
                    vc[u][hf] = ok ? (kFused ? cost_value(cost_kind, gCost, y0 + u, lane + 32 * hf, H, W, p.cost_bias, p.cost_scale)
                                             : kBB ? bb_cost(gCost, a.grad_hist + int64_t(b) * a.grad_stride, i, a.bb_lambda) : __ldg(gCost + i)) : 0.f;
                    vo[u][hf] = obst_is_cost ? vc[u][hf] : (ok ? __ldg(gObst + i) : 0.f);
                    vs[u][hf] = ok ? __ldg(gStart + i) : 0.f;
                    vg[u][hf] = ok ? __ldg(gGoal + i) : 0.f;
                }
            }
#pragma unroll
            for (int u = 0; u < kRows; ++u) {
                const int y = y0 + u;
                if (y < H) {
                    S.cost[(y << 6) + lane] = vc[u][0];
                    S.cost[(y << 6) + lane + 32] = vc[u][1];
                    const uint32_t wo0 = __ballot_sync(kFull, vo[u][0] != 0.f), wo1 = __ballot_sync(kFull, vo[u][1] != 0.f);
                    const uint32_t ws0 = __ballot_sync(kFull, vs[u][0] != 0.f), ws1 = __ballot_sync(kFull, vs[u][1] != 0.f);
                    const uint32_t wg0 = __ballot_sync(kFull, vg[u][0] != 0.f), wg1 = __ballot_sync(kFull, vg[u][1] != 0.f);
                    if (lane == (y & 31)) {
                        if (y >> 5) pass[1] = u64(wo0) | (u64(wo1) << 32);
                        else pass[0] = u64(wo0) | (u64(wo1) << 32);
                    }
                    if (start_rc < 0 && (ws0 | ws1)) start_rc = (y << 6) + (ws0 ? __ffs(ws0) - 1 : 32 + __ffs(ws1) - 1);
                    if (goal_rc < 0 && (wg0 | wg1)) goal_rc = (y << 6) + (wg0 ? __ffs(wg0) - 1 : 32 + __ffs(wg1) - 1);
                }
            }
        }
    }
    if (goal_rc < 0) goal_rc = 0;
    const int gy = goal_rc >> 6, gx = goal_rc & 63;
    __syncwarp();
    {
        const int adx0 = (lane > gx) ? (lane - gx) : (gx - lane);
        const int adx1 = (lane + 32 > gx) ? (lane + 32 - gx) : (gx - lane - 32);
#pragma unroll 4
        for (int y = 0; y < H; ++y) {
            const int i = (y << 6) + lane;
            const int ady = (y > gy) ? (y - gy) : (gy - y);
            const float* heur = g_heur64 + (kNews ? kCells64 : 0);
            sGH[i] = make_float2(0.f, __fadd_rn(__ldg(&heur[(ady << 6) | adx0]), S.cost[i]));
            sGH[i + 32] = make_float2(0.f, __fadd_rn(__ldg(&heur[(ady << 6) | adx1]), S.cost[i + 32]));
        }
    }
    __syncwarp();

    const float gr = p.g_ratio, omg = p.one_minus_g_ratio;
    u64 open[2] = {0ull, 0ull}, closed[2] = {0ull, 0ull};
    uint32_t rm_key[2] = {kKeyInf, kKeyInf};
    int rm_col[2] = {0, 0};
    if (lane == 0) S.par[goal_rc] = 0;
    if (start_rc >= 0) {
        const float f0 = f_value(gr, omg, 0.f, sGH[start_rc].y);
        const int sy = start_rc >> 6, sx = start_rc & 63;
        if (lane == 0) S.key[start_rc] = fkey(f0);
        if (lane == (sy & 31)) {
            if (sy >> 5) { open[1] = 1ull << sx; rm_key[1] = fkey(f0); rm_col[1] = sx; }
            else         { open[0] = 1ull << sx; rm_key[0] = fkey(f0); rm_col[0] = sx; }
        }
    }
    S.open_row[lane] = open[0];
    S.open_row[lane + 32] = open[1];
    // backward state: running sums replicated in every lane
    double Ssum = 0.0, Slo = 0.0, Dsum = 0.0, Dlo = 0.0, Acum = 0.0, Bcum = 0.0;   // (Ssum,Slo), (Dsum,Dlo): double-double
    double Smax = 0.0;   // largest S since the last resum (bwd_track)
    bool s_zero = false;   // a step at which every open numerator underflowed to 0: the map's gradient is NaN
    int Tb = 0, ts_in = NASTAR_TS_CAPPED;
    if (kBwd) {
        Tb = *a.T_batch;
        ts_in = a.t_solve_in[b];
        // clamp(hist + sel) blocks the gradient at a goal that is re-selected after its solve step
        // (pre-clamp value 2, differentiable_astar.py:222-223; SURVEY App. B)
        const bool blocked = (ts_in >= 0) && (ts_in < Tb - 1);
        const float* gG = a.grad_hist + int64_t(b) * a.grad_stride;
        for (int i = lane; i < kCells64; i += 32) {
            const int y = i >> 6, x = i & 63;
            Bw.acc[i] = 0.0;
            Bw.v[i] = 0.f;
            Bw.gh[i] = (y < H && x < W && !(blocked && i == goal_rc)) ? __ldg(gG + y * W + x) : 0.f;
        }
        __syncwarp();
        if (start_rc >= 0) {
            const float f0 = f_value(gr, omg, 0.f, sGH[start_rc].y);
            const float v0 = expf(__fdiv_rn(-f0, a.sqrt_w));                 // :207
            if (lane == 0) { Bw.v[start_rc] = v0; Bw.a0[start_rc] = 0.0; Bw.b0[start_rc] = 0.0; }
            Ssum = double(v0);
            Dsum = double(Bw.gh[start_rc]) * Ssum;
        }
    }
    if constexpr (kExit == kExitCoupled2) Tb = *a.T_batch;   // pass 2 runs T_batch steps
    __syncwarp();

    // ---------------- search loop --------------------------------------------------------------
    const int T = (kBwd || kExit == kExitCoupled2) ? Tb : p.T;
    const bool stationary_ok = (gr >= 0.5f);   // post-solve steps are stationary (SURVEY App. A.4)
    int t_solve = NASTAR_TS_CAPPED;
    int32_t* trace = kTrace ? (p.trace + int64_t(b) * T) : nullptr;
    uint32_t gbits = 0u;          // pass 1: at-goal bits of the current 32-step word
    int t = 0;
    for (; t < T; ++t) {
        // local best of the lane's two rows (strict <: the lower row wins ties)
        uint32_t bk = rm_key[0];
        int bid = (lane << 6) | rm_col[0];
        if (rm_key[1] < bk) { bk = rm_key[1]; bid = ((lane + 32) << 6) | rm_col[1]; }
        const uint32_t m = __reduce_min_sync(kFull, bk);
        if (m == kKeyInf) { t_solve = NASTAR_TS_EXHAUSTED; break; }
        double A1 = 0.0, B1 = 0.0;   // prefix sums INCLUDING step t (the events of step t act from t+1 on)
        if (kBwd) {
            bwd_track(lane, kCells64, [&](int i) { return Bw.v[i]; }, [&](int i) { return Bw.gh[i]; }, Ssum, Slo, Dsum,
                      Dlo, Smax);
            const double inv = 1.0 / (Ssum + Slo);
            s_zero |= (Ssum + Slo == 0.0);
            const double a_t = inv, b_t = (Dsum + Dlo) * inv * inv;
            if (Acum > kRebaseAbove * a_t)
                bwd_rebase(lane, kCells64, Bw.v, [&](int i) { return Bw.gh[i]; }, Bw.acc, Bw.a0, Bw.b0, Acum, Bcum);
            if (stationary_ok && (ts_in >= 0) && (t == ts_in + 1)) {
                // solved: the goal is re-selected with a frozen open set until step T_batch-1
                Acum += double(Tb - t) * a_t;
                Bcum += double(Tb - t) * b_t;
                break;
            }
            A1 = Acum + a_t;
            B1 = Bcum + b_t;
        }
        const uint32_t ind = __reduce_min_sync(kFull, (bk == m) ? uint32_t(bid) : 0xFFFFFFFFu);
        const int r = int(ind >> 6), c = int(ind & 63u);
        if (kTrace && lane == 0) trace[t] = r * W + c;
        const bool solved = (int(ind) == goal_rc);
        if constexpr (kExit == kExitCoupled1) {
            gbits |= uint32_t(solved) << (t & 31);
            if ((t & 31) == 31) {
                if (lane == 0) a.cw.bits[int64_t(b) * a.cw.words + (t >> 5)] = gbits;
                gbits = 0u;
            }
        }
        const u64 m1 = 1ull << c, m0 = m1 >> 1, m2 = m1 << 1;
        // rescan inputs: columns lane and lane+32 of row r
        const u64 open_r = (kContinue && solved) ? S.open_row[r] : (S.open_row[r] & ~m1);
        const uint32_t ka = S.key[(r << 6) + lane], kb = S.key[(r << 6) + 32 + lane];
        uint32_t rs_key = ((open_r >> lane) & 1ull) ? ka : kKeyInf;
        int rs_col = lane;
        {
            const uint32_t kb2 = ((open_r >> (lane + 32)) & 1ull) ? kb : kKeyInf;
            if (kb2 < rs_key) { rs_key = kb2; rs_col = lane + 32; }
        }
        // which of this lane's rows (if any) is in r-1..r+1
        const int d0 = lane - r, d1 = lane + 32 - r;
        const bool near1 = (unsigned(d1 + 1) <= 2u);
        const bool near = (unsigned(d0 + 1) <= 2u) | near1;
        const int dr = near1 ? d1 : d0;
        const bool isr = near & (dr == 0);
        const int myrow = near1 ? (lane + 32) : lane;
        u64 myopen = near1 ? open[1] : open[0];
        u64 myclosed = near1 ? closed[1] : closed[0];
        const u64 mypass = near1 ? pass[1] : pass[0];
        uint32_t mykey = near1 ? rm_key[1] : rm_key[0];
        int mycol = near1 ? rm_col[1] : rm_col[0];
        const int cell = (myrow << 6) + c;
        float2 n0 = make_float2(0.f, 0.f), n1 = n0, n2 = n0;
        if (near) { n0 = sGH[cell - 1]; n1 = sGH[cell]; n2 = sGH[cell + 1]; }
        const float g2 = __fadd_rn(sGH[ind].x, S.cost[ind]);
        __syncwarp();   // read phase ends
        if (isr) {
            myclosed |= m1;
            if (!solved) myopen &= ~m1;
            mykey = kKeyInf;
        }
        const u64 win = isr ? (m0 | m2) : (kNews ? m1 : (m0 | m1 | m2));   // NEWS: no diagonal neighbours
        const u64 cand = near ? (win & mypass) : 0ull;
        const u64 gt = ((n0.x > g2) ? m0 : 0ull) | ((n1.x > g2) ? m1 : 0ull) | ((n2.x > g2) ? m2 : 0ull);
        const u64 upd = cand & ((myopen & gt) | ~(myopen | myclosed));
        myopen |= upd;
        const float ag = __fmul_rn(gr, g2);
        const float f0n = __fadd_rn(ag, __fmul_rn(omg, n0.y));
        const float f1n = __fadd_rn(ag, __fmul_rn(omg, n1.y));
        const float f2n = __fadd_rn(ag, __fmul_rn(omg, n2.y));
        const bool u0 = (upd & m0) != 0ull, u1 = (upd & m1) != 0ull, u2 = (upd & m2) != 0ull;
        const uint32_t q0 = fkey(f0n), q1 = fkey(f1n), q2 = fkey(f2n);
        const int off = (dr << 6) - 1;
        if (u0) { sGH[cell - 1].x = g2; S.key[cell - 1] = q0; S.par[cell - 1] = int8_t(off); }
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
            if (u0) event(cell - 1, expf(__fdiv_rn(-f0n, a.sqrt_w)));     // :207
            if (u1) event(cell, expf(__fdiv_rn(-f1n, a.sqrt_w)));
            if (u2) event(cell + 1, expf(__fdiv_rn(-f2n, a.sqrt_w)));
            if (isr && !solved) event(int(ind), 0.f);                      // the selected cell leaves the open set
            // the events sit on the (at most three) lanes that own rows r-1, r, r+1
            const int l0 = (r - 1) & 31, l1 = r & 31, l2 = (r + 1) & 31;
            dd_add(Ssum, Slo, __shfl_sync(kFull, dS, l0) + __shfl_sync(kFull, dS, l1) + __shfl_sync(kFull, dS, l2));
            dd_add(Dsum, Dlo, __shfl_sync(kFull, dD, l0) + __shfl_sync(kFull, dD, l1) + __shfl_sync(kFull, dD, l2));
            Acum = A1;
            Bcum = B1;
        }
        const uint32_t k0 = u0 ? q0 : kKeyInf, k1 = u1 ? q1 : kKeyInf, k2 = u2 ? q2 : kKeyInf;
        uint32_t fk = k0;
        int fc = c - 1;
        if (k1 < fk) { fk = k1; fc = c; }
        if (k2 < fk) { fk = k2; fc = c + 1; }
        if ((fk < mykey) | ((fk == mykey) & (fc < mycol))) { mykey = fk; mycol = fc; }
        if (near) {
            if (near1) { open[1] = myopen; closed[1] = myclosed; rm_key[1] = mykey; rm_col[1] = mycol; }
            else       { open[0] = myopen; closed[0] = myclosed; rm_key[0] = mykey; rm_col[0] = mycol; }
            S.open_row[myrow] = myopen;
        }
        if (solved && t_solve < 0) t_solve = t;
        if (!kContinue && solved) break;
        if constexpr (kExit == kExitCoupled1) {
            // fixed point: the goal, closed at an earlier step, is selected again and nothing is opened or relaxed
            // (see the 32-wide engine)
            if (solved && t_solve < t && !__any_sync(kFull, upd != 0ull)) { ++t; break; }
        }
        // fold the rescan into the cached minimum of row r (lane r&31, slot r>>5)
        // (kept AFTER the expansion: hoisting these two reductions above it, as the warp32 engine does, lands them inside
        // the divergent region of the `near` lanes here and REDUX then takes its slow divergent path — 3.6x slower)
        const uint32_t mr = __reduce_min_sync(kFull, rs_key);
        const uint32_t mc = __reduce_min_sync(kFull, (rs_key == mr) ? uint32_t(rs_col) : 0xFFFFFFFFu);
        if (lane == (r & 31)) {
            if (r >> 5) {
                if ((mr < rm_key[1]) | ((mr == rm_key[1]) & (int(mc) < rm_col[1]))) { rm_key[1] = mr; rm_col[1] = int(mc); }
            } else {
                if ((mr < rm_key[0]) | ((mr == rm_key[0]) & (int(mc) < rm_col[0]))) { rm_key[0] = mr; rm_col[0] = int(mc); }
            }
        }
        __syncwarp();
    }
    __syncwarp();
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
        S.bits_a[lane] = closed[0];
        S.bits_a[lane + 32] = closed[1];
        __syncwarp();
        const float* gY = a.bb_hist + int64_t(b) * N;
        float* gOut = a.grad_cost + int64_t(b) * N;
        for (int y = 0; y < H; ++y)
            for (int x = lane; x < W; x += 32)
                gOut[y * W + x] = bb_grad((S.bits_a[y] >> x) & 1ull, __ldg(gY + y * W + x), a.bb_lambda);
        return;
    }

    if (kBwd) {
        // close the intervals of the cells still open, scale: dL/dcost = -(1-g_ratio)/sqrt(W) * acc
        const double coef = -double(omg) / double(a.sqrt_w);
        float* gOut = a.grad_cost + int64_t(b) * N;
        for (int i = lane; i < kCells64; i += 32) {
            const int y = i >> 6, x = i & 63;
            if (y < H && x < W) {
                double acc = Bw.acc[i];
                const float v = Bw.v[i];
                if (v != 0.f) acc += double(v) * (double(Bw.gh[i]) * (Acum - Bw.a0[i]) - (Bcum - Bw.b0[i]));
                gOut[y * W + x] = s_zero ? __int_as_float(0x7fc00000) : float(coef * acc);
            }
        }
        return;
    }

    // ---------------- backtrack ------------------------------------------------------------------
    u64 path0 = 0ull, path1 = 0ull;
    {
        const int myslot_row0 = lane, myslot_row1 = lane + 32;
#define NASTAR_MARK(LOC)                                                   \
        {                                                                  \
            const int y_ = (LOC) >> 6;                                     \
            const u64 bit_ = 1ull << ((LOC) & 63);                         \
            path0 |= (y_ == myslot_row0) ? bit_ : 0ull;                    \
            path1 |= (y_ == myslot_row1) ? bit_ : 0ull;                    \
        }
        NASTAR_MARK(goal_rc)
        int loc = goal_rc - S.par[goal_rc];
        const int hops = (t_solve >= 0) ? N : (T - 1);
        for (int k = 0; k < hops; ++k) {
            NASTAR_MARK(loc)
            if (loc == start_rc || loc == goal_rc) break;
            loc -= S.par[loc];
        }
#undef NASTAR_MARK
    }

    // ---------------- epilogue -------------------------------------------------------------------
    S.bits_a[lane] = closed[0];
    S.bits_a[lane + 32] = closed[1];
    S.bits_b[lane] = path0;
    S.bits_b[lane + 32] = path1;
    __syncwarp();
    float* gHist = p.histories + int64_t(b) * N;
    long long* gPath = reinterpret_cast<long long*>(p.paths) + int64_t(b) * N;
    if (W == 64 && aligned16(gHist) && aligned16(gPath)) {
        const int x = (lane & 15) << 2;
        const int n4 = N >> 2;
        for (int i4 = lane; i4 < n4; i4 += 32) {
            const int y = i4 >> 4;
            store_cells4(gHist, gPath, i4, uint32_t(S.bits_a[y] >> x), uint32_t(S.bits_b[y] >> x));
        }
    } else {
        for (int y = 0; y < H; ++y) {
            for (int x = lane; x < W; x += 32) {
                gHist[y * W + x] = ((S.bits_a[y] >> x) & 1ull) ? 1.f : 0.f;
                gPath[y * W + x] = ((S.bits_b[y] >> x) & 1ull) ? 1ll : 0ll;
            }
        }
    }
    const int n_closed = __reduce_add_sync(kFull, __popcll(closed[0]) + __popcll(closed[1]));
    const int n_path = __reduce_add_sync(kFull, __popcll(path0) + __popcll(path1));
    if (lane == 0) {
        if (p.t_solve) p.t_solve[b] = t_solve;
        if (p.n_steps) p.n_steps[b] = steps;
        if (p.n_closed) p.n_closed[b] = n_closed;
        if (p.path_len) p.path_len[b] = n_path;
    }
}

}  // namespace nastar
