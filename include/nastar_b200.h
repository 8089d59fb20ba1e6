/*
 * nastar_b200.h — C ABI of the H100-native differentiable-A* engine (libnastar_b200.so).
 *
 * This is the drop-in boundary for the reference's hot path.  The reference has no FFI: the
 * seam is the Python attribute `self.astar = DifferentiableAstar(...)`
 * (/root/reference/src/neural_astar/planner/astar.py:41-44,141-144) whose `.forward`
 * (/root/reference/src/neural_astar/planner/differentiable_astar.py:150-267) is replaced.
 * Each entry point below names the reference code it replaces.  All pointers are DEVICE
 * pointers unless stated otherwise; no torch types cross this boundary.
 *
 * Plane layout: every "plane" argument is B maps of H*W contiguous fp32 cells (row-major,
 * flat index = y*W + x, the same flat index the reference uses for `parents`,
 * differentiable_astar.py:195-198).  `*_stride` is the distance between consecutive maps
 * in ELEMENTS (so a [B,C,H,W] tensor's channel 0 is passed with stride C*H*W, matching
 * `cost_maps[:, 0]`, differentiable_astar.py:177-180).
 */
#ifndef NASTAR_B200_H_
#define NASTAR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NASTAR_B200_ABI_VERSION 4

/* status codes (the reference only has Python asserts, differentiable_astar.py:147,172-175) */
enum {
    NASTAR_OK = 0,
    NASTAR_EINVAL = 1,      /* bad shape / null pointer / T < 1 */
    NASTAR_EUNSUPPORTED = 2,/* map shape outside what this build handles */
    NASTAR_ECUDA = 3,       /* a CUDA runtime call failed; see nastar_b200_last_cuda_error() */
    NASTAR_EWORKSPACE = 4   /* workspace too small */
};

/* per-map outcome written to t_solve[] */
#define NASTAR_TS_CAPPED (-1)    /* step cap T reached before the goal was selected */
#define NASTAR_TS_EXHAUSTED (-2) /* open list ran empty: goal unreachable (the reference
                                    produces NaN -> IndexError here, SURVEY.md sec. 5) */

/* nastar_fwd_params.flags */
#define NASTAR_FWD_NO_EARLY_EXIT 1 /* run exactly T steps per map: a solved map keeps stepping (re-selecting its
                                      goal, or other nodes when g_ratio < 0.5) like the reference's batch-synchronous
                                      loop does until the slowest map is solved (differentiable_astar.py:251-252).
                                      Per-map early exit is exact for g_ratio >= 0.5 (SURVEY App. A.4).  For
                                      g_ratio < 0.5 the batch coupling is either decided on the host from a
                                      NO_EARLY_EXIT trace (a full-length search, then a second one of T_batch steps)
                                      or on the device by nastar_b200_forward_coupled() */
#define NASTAR_FWD_PAIR 2          /* validation pair in ONE launch (utils/training.py:63-87 runs the learned-cost
                                      search and VanillaAstar on the same batch): maps 0..B-1 are searched on
                                      `cost` (any cost_kind), maps B..2B-1 are the same problems searched with
                                      cost = obst (astar.py:93-94).  Every output array then holds 2B entries.
                                      Engine-1 shapes (H,W <= 32) run both halves in one kernel launch; other
                                      shapes issue the two halves back to back inside this call */
#define NASTAR_FWD_NEWS 4          /* 4-connected search of the generator's NorthEastWestSouth mechanism
                                      (mechanism.py:113-131): a selected cell opens and relaxes only its N, E, W and S
                                      neighbours, and h = manhattan + 0.001 * euclid to the goal instead of chebyshev
                                      + 0.001 * euclid.  Everything else (selection, cost charged at the selected cell,
                                      early exit, backtrack, t_solve codes) is unchanged.  Without it the search is
                                      Moore (8-connected).  Applies to both halves of NASTAR_FWD_PAIR.  Engines 1, 4,
                                      2 and 3; engine 5 is never used for it */

/* nastar_fwd_params.cost_kind: what `cost` points to (SURVEY.md 8(f)-3, encoder -> search hand-off) */
#define NASTAR_COST_PLANE 0  /* finished cost maps, fp32 [B][H*W] (differentiable_astar.py:150-157) */
#define NASTAR_COST_LOGIT 1  /* the encoder's raw 1-channel output x, fp32 [B][H*W]; the kernel prologue applies
                                encoder.py:32-34: cost = sigmoid(x) * cost_scale */
#define NASTAR_COST_TAPS  2  /* per-pixel partial products of the encoder's last 3x3 conv (one output channel),
                                fp32 [B][H*W][9] (tap k = ky*3+kx innermost): the prologue gathers
                                x[y][x] = cost_bias + sum_k taps[y+ky-1][x+kx-1][k] (zero padding), then
                                cost = sigmoid(x) * cost_scale.  `cost_stride` is in elements of this layout
                                (9*H*W for a dense batch).  LOGIT / TAPS: engines 1 and 4 (H,W <= 64),
                                NASTAR_EUNSUPPORTED for larger shapes */

typedef struct nastar_fwd_params {
    /* inputs — differentiable_astar.py:150-157 (cost_maps, start_maps, goal_maps, obstacles_maps) */
    const float *cost;   int64_t cost_stride;
    const float *start;  int64_t start_stride;
    const float *goal;   int64_t goal_stride;
    const float *obst;   int64_t obst_stride;   /* may alias cost (VanillaAstar, astar.py:93-94) */
    int32_t B, H, W;
    /* scalars prepared on the host exactly as Python does (differentiable_astar.py:206):
       g_ratio and (1 - g_ratio) evaluated in double, then rounded to fp32 */
    float g_ratio;
    float one_minus_g_ratio;
    /* loop bound int(Tmax_eff * W * W), differentiable_astar.py:200-202 */
    int32_t T;
    /* NASTAR_FWD_* flags */
    int32_t flags;
    /* NASTAR_COST_*; cost_scale = the encoder's `const` (encoder.py:25-28,34), cost_bias = folded bias of the
       last conv (NASTAR_COST_TAPS only).  Zero-initialised params mean a plain cost plane */
    int32_t cost_kind;
    float   cost_scale;
    float   cost_bias;
    /* outputs */
    float   *histories;  /* [B][H*W] fp32 in {0,1}   — AstarOutput.histories, :265 */
    int64_t *paths;      /* [B][H*W] int64 in {0,1}  — AstarOutput.paths (backtrack, :96-125) */
    int32_t *t_solve;    /* [B] step at which the goal was selected, or NASTAR_TS_*; nullable */
    int32_t *n_steps;    /* [B] number of selection steps executed for the map; nullable */
    int32_t *trace;      /* [B][T] selected flat index per step (-1 beyond n_steps); nullable.
                            Feeds store_intermediate_results (:210-216) */
    int32_t *n_closed;   /* [B] number of closed cells = histories.sum() per map; nullable.  With path_len it
                            replaces the host-side sums of the validation metrics (utils/training.py:71-85) */
    int32_t *path_len;   /* [B] number of cells on the path = paths.sum() per map; nullable */
    /* scratch for maps whose state does not fit in shared memory; see
       nastar_b200_forward_workspace_bytes().  nullable when that returns 0 */
    void    *workspace;
    size_t   workspace_bytes;
} nastar_fwd_params;

typedef struct nastar_bwd_params {
    /* the forward's inputs again (the backward replays the deterministic search) */
    const float *cost;   int64_t cost_stride;
    const float *start;  int64_t start_stride;
    const float *goal;   int64_t goal_stride;
    const float *obst;   int64_t obst_stride;
    int32_t B, H, W;
    float g_ratio;
    float one_minus_g_ratio;
    float sqrt_w;             /* fl32(sqrt(W)), differentiable_astar.py:207 */
    /* number of loop iterations the reference would have executed for this batch:
       T_batch = min(T, 1 + max_b t_solve[b]) (batch-coupled stop, :251-252).  Read on the
       DEVICE from *T_batch so that no host synchronisation is needed between forward
       and backward */
    const int32_t *T_batch;
    const int32_t *t_solve;   /* [B] the forward's t_solve[] for the same inputs and loop bound.  Used for (a) the
                                 stationary post-solve shortcut when g_ratio >= 0.5 and (b) the goal clamp: the
                                 gradient at a map's goal is blocked iff 0 <= t_solve[b] < T_batch-1 (the goal is
                                 then selected again and clamp(hist+sel) saw 2, differentiable_astar.py:222-223).
                                 For g_ratio < 0.5 a solved map need not re-select its goal: pass 0 for maps
                                 whose goal is selected at least twice within T_batch steps and T_batch otherwise
                                 (the Python module derives this from a NO_EARLY_EXIT trace, or takes the goal_clamp
                                 of nastar_b200_forward_coupled) */
    const float *grad_histories; int64_t grad_stride; /* dL/d histories, [B][H*W] */
    float *grad_cost;                                  /* dL/d cost_maps, [B][H*W], overwritten */
    void  *workspace;
    size_t workspace_bytes;
} nastar_bwd_params;

/* ABI version of the loaded library (== NASTAR_B200_ABI_VERSION at build time). */
int nastar_b200_abi_version(void);

/* Bytes of device scratch nastar_b200_forward needs for this shape: 0 for H,W <= 64 (every 32x32 / 12x12 / 64x64
 * config); larger maps need the work queue + per-map flags of the binary-cost engine and, beyond 128x128, the
 * per-CTA state slots of the generic engine.  Passing less than this but at least the generic engine's own need
 * still works (the binary-cost fast path is then skipped). */
size_t nastar_b200_forward_workspace_bytes(int32_t B, int32_t H, int32_t W);
size_t nastar_b200_backward_workspace_bytes(int32_t B, int32_t H, int32_t W);

/* Replaces DifferentiableAstar.forward's loop + backtrack (differentiable_astar.py:187-255).
 * Asynchronous on `stream` (a cudaStream_t passed as void*). Returns NASTAR_*. */
int nastar_b200_forward(const nastar_fwd_params *p, void *stream);

/* Replaces autograd through the loop (closed form, SURVEY.md App. B): writes dL/dcost.  Moore searches; it is
 * nastar_b200_backward_mech(p, NASTAR_MECH_MOORE, stream). */
int nastar_b200_backward(const nastar_bwd_params *p, void *stream);

/* nastar_b200_backward for the search of either mechanism: NASTAR_MECH_MOORE, or NASTAR_MECH_NEWS to differentiate a
 * forward that ran with NASTAR_FWD_NEWS (the replay then expands 4-connected with the Manhattan heuristic; the
 * closed form itself does not depend on the stencil).  Any other mechanism is NASTAR_EINVAL, before any launch. */
int nastar_b200_backward_mech(const nastar_bwd_params *p, int32_t mechanism, void *stream);

/* Batch-coupled forward for g_ratio < 0.5 (differentiable_astar.py:203-252) with T_batch decided on the device: the
 * reference steps every map until one step has every map selecting its goal, so a map solved early keeps evolving
 * (it need not re-select its goal when g_ratio < 0.5, SURVEY App. A.4).  Writes the outputs of exactly
 *   T_batch = 1 + min{k < T : every map selects its goal at step k}   (T if there is no such k)
 * steps per map, bit-equal to nastar_b200_forward with p->T = T_batch and NASTAR_FWD_NO_EARLY_EXIT (histories, paths,
 * t_solve, n_steps, n_closed, path_len), plus
 *   T_batch[0]     (device int32) that step count, ready for nastar_bwd_params.T_batch;
 *   goal_clamp[b]  (device int32) 0 if map b selects its goal at least twice within T_batch steps, else T_batch: the
 *                  nastar_bwd_params.t_solve encoding of the goal clamp for this case.
 * Three launches on `stream`, no host round trip (CUDA-graph capturable): pass 1 searches without the solve-step exit
 * and stops a map at its fixed point (its goal, already closed, is selected again and nothing is opened or relaxed: every
 * later step repeats that one), when its open set is exhausted, or at T, recording the at-goal bit of every step; a
 * one-CTA reduction computes T_batch and goal_clamp from those bits; pass 2 re-runs, for exactly T_batch steps, only the
 * maps pass 1 stopped later than T_batch.
 * p->T is the cap; p->flags may hold only NASTAR_FWD_NEWS (NO_EARLY_EXIT or PAIR: NASTAR_EINVAL); p->trace must be
 * NULL; any cost_kind (LOGIT / TAPS on engines 1 and 4).  p->workspace must hold
 * nastar_b200_forward_coupled_workspace_bytes(B, H, W, T) bytes, else NASTAR_EWORKSPACE.  Every check precedes the
 * first launch.  Engines 1, 4, 2 and 3; engine 5 is not used. */
size_t nastar_b200_forward_coupled_workspace_bytes(int32_t B, int32_t H, int32_t W, int32_t T);
int nastar_b200_forward_coupled(const nastar_fwd_params *p, int32_t *T_batch, int32_t *goal_clamp, void *stream);

/* Black-box backward of the search (BB-A*: the gradient of Vlastelica et al., ICLR 2020, through a non-differentiable
 * A*).  With w the cost plane of p, g = grad_histories and lambda > 0:
 *   w'        = fl(w + fl(lambda * g))   (two roundings, no FMA, no clamp: w' may be negative);
 *   y'        = the closed set of the same search on w' (p->g_ratio, p->T, mechanism, start / goal / obstacle planes);
 *   grad_cost = (y' - histories) / lambda, every cell exactly 0 or +-fl(1/lambda).
 * Inputs: p's input fields (cost .. flags, cost_kind, workspace); its output fields are neither read nor written.
 * `histories` are the forward's histories y(w), [B][H*W] contiguous; grad_histories [B][H*W] maps grad_stride elements
 * apart.  Output: grad_cost [B][H*W] contiguous, overwritten.
 * T_batch and goal_clamp both NULL: the search on w' stops each map at its solve step, like nastar_b200_forward
 * without flags (exact for g_ratio >= 0.5 or B = 1).  One launch; w' is formed while the costs are staged and y' is
 * compared with `histories` in the epilogue, so neither w' nor y' is ever stored.  Both non-NULL: the batch-coupled
 * search of nastar_b200_forward_coupled with cap p->T on w', which also writes its T_batch[0] and goal_clamp[B]
 * there; the same three launches, with the black-box prologue and epilogue in both search passes.
 * Checks, all before the first launch: a NULL plane, histories, grad_histories or grad_cost, B, H or W <= 0, T < 1,
 * lambda not finite or <= 0, cost_kind other than NASTAR_COST_PLANE, flags other than NASTAR_FWD_NEWS, a trace, or
 * only one of T_batch / goal_clamp give NASTAR_EINVAL; unsupported shapes NASTAR_EUNSUPPORTED.  Workspace: coupled,
 * nastar_b200_forward_coupled_workspace_bytes(B, H, W, T) bytes; otherwise the generic engine's state slots beyond
 * 128x128 (nastar_b200_forward_workspace_bytes(B, H, W) covers them), else NASTAR_EWORKSPACE.  Engines 1, 4, 2 and 3;
 * engine 5 is never used.  Asynchronous on `stream`. */
int nastar_b200_backward_blackbox(const nastar_fwd_params *p, const float *histories, const float *grad_histories,
                                  int64_t grad_stride, float lambda, float *grad_cost, int32_t *T_batch,
                                  int32_t *goal_clamp, void *stream);

/* T_batch[0] = min(T, 1 + max_b n_steps-style stop) computed on the device from the forward's
 * t_solve/n_steps arrays (replaces the host-synchronising torch.all(...) of :251). */
int nastar_b200_batch_steps(const int32_t *t_solve, const int32_t *n_steps, int32_t B, int32_t T,
                            int32_t *T_batch, void *stream);

/* Which forward engine a shape dispatches to: 1 = warp-resident (H,W <= 32), 4 = warp-resident 64-wide
 * (H,W <= 64), 2 = generic warp engine with shared-memory state, 3 = generic with global-memory state,
 * 0 = unsupported.  Engine-2/3 shapes whose cost
 * plane IS the obstacle plane (same pointer and stride: VanillaAstar, astar.py:93-94) are first offered to
 * engine 5, the CTA-per-map binary-cost engine (csrc/nastar_bin16.cuh); maps it cannot take (a cost value
 * outside {0,1}) are re-run by engine 2/3 inside the same call.  Engine 5 is Moore-only: a NASTAR_FWD_NEWS search
 * of such a shape skips it and runs on engine 2/3 alone, in one launch. */
int nastar_b200_engine_for(int32_t H, int32_t W);

/* 1 if engine 5 (binary-cost, whole map in one CTA's shared memory) can hold this shape. */
int nastar_b200_bin16_supported(int32_t H, int32_t W);

/* Encoder input assembly, replaces NeuralAstar.encode's glue (astar.py:172-177): out is the channels-last
 * (NHWC) tensor [B][Hm][Wm][C+1] with channels 0..C-1 = map_designs[b][c] (fp32 NCHW [B][C][Hm][Wm], contiguous)
 * and channel C = (start + goal) nearest-upsampled from [H][W] to [Hm][Wm] (F.interpolate mode="nearest";
 * identity when the sizes agree).  start/goal are [B][H*W] planes with element strides. */
int nastar_b200_pack_inputs(const float *map_designs, int32_t C, int32_t Hm, int32_t Wm,
                            const float *start, int64_t start_stride, const float *goal, int64_t goal_stride,
                            int32_t B, int32_t H, int32_t W, float *out, void *stream);

/* cost = sigmoid(bias + 9-tap gather of `taps`) * scale for every cell, written as a dense [B][H*W] plane — the
 * same arithmetic, in the same order, as nastar_b200_forward's NASTAR_COST_TAPS prologue (so `encode()` and the
 * fused forward agree bit for bit).  taps: fp32 [B][H*W][9]. */
int nastar_b200_cost_from_taps(const float *taps, int32_t B, int32_t H, int32_t W, float bias, float scale,
                               float *cost, void *stream);

/* First encoder layer of the "m+" planners fused with the input assembly (astar.py:172-177 + the first
 * Conv2d(2,32,3,padding=1) + BatchNorm + ReLU of encoder.py:60-78): out[b][y][x][0..31] (channels-last fp32) =
 * relu(bias + conv3x3(cat(map_designs, start + goal))).  map_designs: fp32 [B][H*W] contiguous (one channel);
 * start / goal: [B][H*W] planes with element strides; w_host: HOST pointer, fp32 [9 taps][2 in][32 out] with
 * BatchNorm folded in; bias_host: HOST pointer, fp32 [32] (both copied into the launch's parameter block, i.e. the
 * constant bank — safe to capture in a CUDA graph).  Same spatial size for maps and marks only; B*H*W <= 2^30. */
int nastar_b200_conv1_marks(const float *map_designs, const float *start, int64_t start_stride, const float *goal,
                            int64_t goal_stride, int32_t B, int32_t H, int32_t W, const float *w_host,
                            const float *bias_host, float *out, void *stream);

/* Head of the encoder (its last 3x3 conv has ONE output channel, encoder.py:60-78): taps[p][k] = sum_c x[p][c] *
 * w[c][k] for every pixel p of the channels-last activation x (fp32 [P][C], C in {16,32,64,128,256}), k = ky*3+kx.
 * `w` is a HOST pointer to C*9 floats ([c][k], BatchNorm folded): it is passed to the kernel by value (constant
 * bank), so it may change between calls without any device copy.  The 9-tap spatial gather + bias + sigmoid * const
 * that finish the layer happen in nastar_b200_forward's NASTAR_COST_TAPS prologue (or nastar_b200_cost_from_taps). */
int nastar_b200_head_taps(const float *x, int64_t P, int32_t C, const float *w_host, float *taps, void *stream);

/* Input of a U-Net decoder block (planner/encoder.py Unet): out[b][y][x][:] = concat(dec[b][y/2][x/2][0..Cd-1],
 * skip[b][y][x][0..Cs-1]) for y < 2h, x < 2w, i.e. torch.cat((F.interpolate(dec, scale_factor=2, mode="nearest"),
 * skip), 1) bit for bit.  dec: channels-last fp32 [B][h][w][Cd]; skip: channels-last fp32 [B][2h][2w][Cs], or NULL with
 * Cs = 0 (the last block has no skip); out: channels-last fp32 [B][2h][2w][Cd+Cs].  Every pointer 16-B aligned, Cd > 0
 * and Cs >= 0 multiples of 4, else NASTAR_EINVAL before any launch.  One kernel launch, asynchronous on `stream`. */
int nastar_b200_upsample_concat(const float *dec, int32_t B, int32_t h, int32_t w, int32_t Cd, const float *skip,
                                int32_t Cs, float *out, void *stream);

/* The encoder's last body layer fused with the head products (encoder.py:60-78, the 128 -> 256 conv + BatchNorm + ReLU
 * followed by nastar_b200_head_taps): taps[p][k] = sum_c relu(bias[c] + conv3x3(x, w)[p][c]) * head_w[c][k], pad 1,
 * stride 1, without writing the [P][C_out] activation.  x: channels-last fp32 [B][H][W][C_in], 16-B aligned;
 * w: fp32 [C_out][3][3][C_in] (OIHW in channels-last memory, BatchNorm folded), 16-B aligned; bias: fp32 [C_out];
 * head_w_host: HOST pointer to C_out*9 floats ([c][k], passed by value like nastar_b200_head_taps); taps: fp32
 * [B][H][W][9], the NASTAR_COST_TAPS layout.  The convolution runs on TF32 tensor cores with fp32 accumulation (like
 * cuDNN with TF32 allowed); bias, ReLU and the head products are fp32.  Deterministic.  C_in = 128, C_out = 256 and
 * H, W <= 64 only, else NASTAR_EUNSUPPORTED.  One kernel launch, asynchronous on `stream`. */
int nastar_b200_conv3x3_head_taps(const float *x, int32_t B, int32_t H, int32_t W, int32_t C_in, int32_t C_out,
                                  const float *w, const float *bias, const float *head_w_host, float *taps,
                                  void *stream);

/* Self-test of engine 5's branch-free square root: counts, on the device, the integers i in [0, n) for which it
 * differs in any bit from the IEEE-rounded sqrtf(i) that get_heuristic needs (differentiable_astar.py:47-50).
 * `mismatches` is a device int the caller zeroed.  n = 2*511*511+1 covers every argument a 512-row map can produce. */
int nastar_b200_selftest_sqrt(int32_t n, int32_t *mismatches, void *stream);

/* Shortest-path training labels for new maps (replaces the planning-datasets generator's dijkstra_dist +
 * extract_policy, planning_datasets_utils/dijkstra.py:120-157 and data.py:27-62; Moore mechanism, one orientation).
 * maps: B fp32 maps of H*W cells, map_stride (>= H*W) elements apart; a cell is passable iff its value != 0.0.
 * goal_idx: DEVICE int32 [B], flat goal index y*W+x (an index outside [0, H*W) means no goal: every cell unreached).
 * Writes, for every map, dense [B][H*W] planes:
 *   dists    fp32  0 at the goal, -(number of moves to the goal) for passable cells that reach it, -(H*W) for every
 *                  other cell (obstacles and unreachable regions) -- dijkstra_dist's negated distance, exact in fp32;
 *   act_mask u8    bit a set iff action a (0..7 = N, E, W, S, NE, NW, SE, SW; a move off the grid or into a
 *                  non-passable cell stays put) leads to a cell of maximal dists -- the set extract_policy draws from;
 *   action   i8    the lowest set bit of act_mask (the first maximal action, np.argmax's choice).
 * One kernel launch.  H, W <= 512, else NASTAR_EUNSUPPORTED.  Asynchronous on `stream`. Returns NASTAR_*. */
int nastar_b200_opt_labels(const float *maps, int64_t map_stride, const int32_t *goal_idx, int32_t B, int32_t H,
                           int32_t W, float *dists, uint8_t *act_mask, int8_t *action, void *stream);

/* mechanism of nastar_b200_opt_labels_mech and nastar_b200_weighted_labels_mech: the planning-datasets generator's --mechanism (mechanism.py:267-277) */
#define NASTAR_MECH_MOORE 0   /* 8 actions: N, E, W, S, NE, NW, SE, SW (the labels of nastar_b200_opt_labels) */
#define NASTAR_MECH_NEWS  1   /* 4 actions: N, E, W, S (NorthEastWestSouth, mechanism.py:52-131) */

/* nastar_b200_opt_labels for either mechanism.  NASTAR_MECH_MOORE gives exactly nastar_b200_opt_labels' output.
 * NASTAR_MECH_NEWS: distances are unit-step BFS distances over the 4 neighbours (same fills: 0 at the goal, -(H*W)
 * where the goal is not reached; the goal is the source even when it is not passable); act_mask holds the maximal
 * actions among the 4 targets of N, E, W, S (bits 0..3; bits 4..7 are never set) and action its lowest member.  Every
 * argument is checked before the launch: a mechanism other than these two is NASTAR_EINVAL.  One kernel launch.
 * H, W <= 512, else NASTAR_EUNSUPPORTED.  Asynchronous on `stream`.  Returns NASTAR_*. */
int nastar_b200_opt_labels_mech(const float *maps, int64_t map_stride, const int32_t *goal_idx, int32_t B, int32_t H,
                                int32_t W, int32_t mechanism, float *dists, uint8_t *act_mask, int8_t *action,
                                void *stream);

/* Exact vertex-weighted shortest paths to a goal, for cost maps (the labels of WarCraft-style training and the optimum
 * that learned-cost paths are measured against).  Per map b (DESIGN.md §11):
 *   cost      B fp32 maps of H*W cells, cost_stride (>= H*W) elements apart;
 *   passable  B fp32 maps, passable_stride (>= H*W) apart, a cell is passable iff != 0.0; NULL = every cell passable;
 *   goal_idx  DEVICE int32 [B] flat goal index y*W+x; start_idx DEVICE int32 [B] or NULL (then path_maps and
 *             path_costs must be NULL too, and with a start both are required).
 * Moves: actions 0..7 = N, E, W, S, NE, NW, SE, SW from a passable cell into an in-grid cell that is passable or is
 * the goal (no corner check).  A move charges the cost of the cell it enters: the cost-to-go is D[goal] = +0,
 * D[v] = min over moves v->t of fl(D[t] + c[t]), each add rounded once; the minimum over all paths of that fp32 fold,
 * independent of evaluation order.  A move v->t is optimal iff fl(D[t] + c[t]) == D[v]; hop[v] = 1 + the least hop
 * of v's optimal targets (hop[goal] = 0).  Writes dense [B][H*W] planes:
 *   dists    fp32  -D: 0 at the goal, -inf where the goal is unreachable;
 *   hops     i32   hop, -1 where unreachable;
 *   act_mask u8    bit a set iff action a is optimal and enters a cell with hop one lower (0 at the goal and at
 *                  unreachable cells);
 *   action   i8    the lowest set bit of act_mask, -1 where it is 0;
 *   path_maps fp32 [B][H*W] (with a start) the cells of the roll-out of `action` from the start, start and goal
 *                  included; path_costs fp32 [B] = fl(c[start] + D[start]) (+inf, empty mask if unreachable);
 *   status   i32 [B]  0, or an OR of: 1 the goal or a passable cell has a negative, NaN or infinite cost (the planes
 *                  are then filled as unreachable); 2 goal index outside [0, H*W); 4 a start was given and cannot
 *                  reach the goal.
 * One kernel launch, one CTA per map.  H, W <= 128 (H*W <= 16384), else NASTAR_EUNSUPPORTED.  Asynchronous on
 * `stream`.  Returns NASTAR_*. */
int nastar_b200_weighted_labels(const float *cost, int64_t cost_stride, const float *passable, int64_t passable_stride,
                                const int32_t *goal_idx, const int32_t *start_idx, int32_t B, int32_t H, int32_t W,
                                float *dists, int32_t *hops, uint8_t *act_mask, int8_t *action, float *path_maps,
                                float *path_costs, int32_t *status, void *stream);

/* nastar_b200_weighted_labels for either mechanism.  NASTAR_MECH_MOORE gives exactly nastar_b200_weighted_labels'
 * output.  NASTAR_MECH_NEWS: moves are actions 0..3 = N, E, W, S only (into an in-grid 4-neighbour that is passable or
 * is the goal); D, hops, the policy, the roll-out, path_costs and status follow the same rules over those 4 moves, and
 * act_mask uses bits 0..3 only.  Every argument is checked before the launch: a mechanism other than these two is
 * NASTAR_EINVAL.  One kernel launch, one CTA per map.  H, W <= 128, else NASTAR_EUNSUPPORTED.  Asynchronous on
 * `stream`.  Returns NASTAR_*. */
int nastar_b200_weighted_labels_mech(const float *cost, int64_t cost_stride, const float *passable,
                                     int64_t passable_stride, const int32_t *goal_idx, const int32_t *start_idx,
                                     int32_t B, int32_t H, int32_t W, int32_t mechanism, float *dists, int32_t *hops,
                                     uint8_t *act_mask, int8_t *action, float *path_maps, float *path_costs,
                                     int32_t *status, void *stream);

/* Training-batch sampler, preparation (MazeDataset._prepared's per-map work, once per dataset, one kernel launch).
 * dists fp32 [B][H*W] (opt_dists), policies fp32 [B][8][H*W] (opt_policies; the first maximal action of each cell
 * is used), goal_maps fp32 [B][H*W] (the first maximum is the goal), all dense.  q0..q3: the quantile fractions that
 * np.percentile evaluates, (100*(1 - [pct1, pct2, pct3, 1])) / 100 in double, each in [0, 1].  Writes per map:
 *   band_bits   u32 [B][3][ceil(H*W/32)]  cell c of band r = bit c%32 of word c/32; band r = the cells with
 *               od > min(od) and th[r+1] <= od <= th[r] (bands may share boundary cells);
 *   band_counts i32 [B][3]; goal_idx i32 [B];
 *   actions     u32 [B][ceil(H*W/8)]  first maximal action of cell c in bits 4*(c%8) of word c/8;
 *   thresholds  f64 [B][4]  th = np.percentile(od[od > od.min()], 100*(1 - pcts)), bit for bit;
 *   status      i32 [B]  0, or an OR of: 1 a distance that is not an integer in [-(H*W), 0]; 2 no cell above
 *               min(od); 4 an empty band; 8 a cell with od > -(H*W), not the goal, whose action leaves the grid or
 *               does not reach a cell with od + 1; 16 the goal is not the only cell with od == 0.  Maps with status 0
 *               are the ones nastar_b200_sampler_sample accepts: each of their walks reaches the goal after exactly
 *               -od[start] moves.
 * H, W <= 512, else NASTAR_EUNSUPPORTED.  Asynchronous on `stream`. */
int nastar_b200_sampler_prepare(const float *dists, const float *policies, const float *goal_maps, int32_t B, int32_t H,
                                int32_t W, double q0, double q1, double q2, double q3, uint32_t *band_bits,
                                int32_t *band_counts, int32_t *goal_idx, uint32_t *actions, double *thresholds,
                                int32_t *status, void *stream);

/* Training-batch sampler, one batch in one kernel launch (MazeDataset.__getitem__ for B samples, collated).
 * maps / goal_maps: fp32 [n_maps][H*W], the prepared arrays of nastar_b200_sampler_prepare for the same n_maps
 * maps (all of status 0); indices: i64 [B] map of each sample; draws: [B][S][2] u32 (passed as int32): start s of
 * sample i takes band r = (d0*3) >> 32 and candidate k = (d1*band_counts[r]) >> 32 of that band, in raster order.
 * Writes out_maps [B][H*W] and out_goals [B][H*W] (copies), out_starts [B][S][H*W] (one 1 per plane) and out_trajs
 * [B][S][H*W] (the cells visited by following the actions from the start to the goal: start included, goal
 * excluded), fp32.  An index outside [0, n_maps) gives all-zero planes.  Plane pointers 16-B aligned.  H, W <= 512. */
int nastar_b200_sampler_sample(const float *maps, const float *goal_maps, int32_t n_maps, int32_t H, int32_t W,
                               const uint32_t *band_bits, const int32_t *band_counts, const int32_t *goal_idx,
                               const uint32_t *actions, const int64_t *indices, const int32_t *draws, int32_t B,
                               int32_t S, float *out_maps, float *out_starts, float *out_goals, float *out_trajs,
                               void *stream);

/* Goals for new maps (the planning-datasets generator's from_largest rule, planning_datasets_utils/data.py:128-147,
 * with the random draw supplied by the caller).  maps: B fp32 maps of H*W cells, map_stride (>= H*W) elements apart; a
 * cell is passable iff its value != 0.0.  Per map b:
 *   region      the largest 4-connected region of passable cells; ties go to the region whose first cell comes first
 *               in raster order (scipy.ndimage.label + argmax of the counts);
 *   candidates  with edge_size e > 0, the region's cells with (y < e || y >= H-e) && (x < e || x >= W-e) (the four
 *               e x e corner squares, NumPy's corner[e:-e] slicing for every e) if there is one, else the whole region;
 *               e == 0: the whole region;
 *   goal        candidate k = (draws[b] * count) >> 32 in raster order, draws read as u32 (passed as int32).
 * Writes goal_idx i32 [B] (flat y*W+x), goal_maps fp32 [B][H*W] (dense: 1.0 at the goal, 0 elsewhere) and
 * status i32 [B]: 0, or 1 = the map has no passable cell (then goal_idx = -1 and an all-zero plane).
 * Needs no workspace.  One kernel launch.  edge_size >= 0; H, W <= 512, else NASTAR_EUNSUPPORTED.  Asynchronous on
 * `stream`.  Returns NASTAR_*. */
int nastar_b200_sample_goals(const float *maps, int64_t map_stride, int32_t B, int32_t H, int32_t W, int32_t edge_size,
                             const int32_t *draws, int32_t *goal_idx, float *goal_maps, int32_t *status, void *stream);

/* Planning maps from decoded map images (the planning-datasets generator's load_maze_from_directory:
 * Image.resize((W, H)) + skimage threshold_otsu + image > threshold).  images: B uint8 L images of H0*W0 levels (rows
 * W0 apart), image_stride (>= H0*W0) elements apart.  Per image b:
 *   resized     Pillow's BICUBIC resize to H x W (reducing_gap=None), bit for bit: a horizontal pass into a uint8
 *               intermediate when W != W0, then a vertical pass when H != H0, with Pillow's 22-bit fixed-point weights;
 *   threshold   threshold_otsu (skimage >= 0.19) of the resized levels as float32: the level of a uniform image,
 *               else the center of the first bin that maximises the between-class variance of the 256-bin histogram
 *               over [min, max], with sequential float64 cumulative sums;
 *   map         1.0 where level > threshold, else 0.0.
 * Writes maps fp32 [B][H*W], resized uint8 [B][H*W] (optional: NULL skips it), thresholds fp32 [B] and status i32 [B]:
 * 0, or 1 = uniform resized image (all-zero map).  Needs no workspace.  One kernel launch.  H, W <= 512 and H0, W0 <=
 * 2048, else NASTAR_EUNSUPPORTED.  Asynchronous on `stream`.  Returns NASTAR_*. */
int nastar_b200_maps_from_images(const uint8_t *images, int64_t image_stride, int32_t B, int32_t H0, int32_t W0,
                                 int32_t H, int32_t W, float *maps, uint8_t *resized, float *thresholds,
                                 int32_t *status, void *stream);

/* One-hot policies drawn from maximal action sets.  act_mask: uint8 [B][N] (bit a = action a is maximal, the act_mask
 * of nastar_b200_opt_labels); draws: [B][N] u32 (passed as int32).  Cell c of map b takes set bit k = (d * popc) >> 32
 * of its mask in action order, d = its draw, and writes policies fp32 [B][8][N] one-hot (all zero for an empty mask).
 * One kernel launch.  Asynchronous on `stream`.  Returns NASTAR_*. */
int nastar_b200_draw_policies(const uint8_t *act_mask, const int32_t *draws, int32_t B, int32_t N, float *policies,
                              void *stream);

/* One PNG image of a nastar_b200_decode_png batch.  Offsets and lengths are in bytes. */
typedef struct nastar_png_desc {
    int64_t in_off, in_len;     /* the zlib stream (the IDAT payloads joined) in `data` */
    int64_t plte_off, plte_len; /* the PLTE payload in `data` (plte_len 0: none; palette images only) */
    int64_t out_off;            /* the image's H0*W0 uint8 L plane in `out`, row-major */
    int32_t W0, H0;             /* IHDR width and height */
    int32_t bit_depth, color_type, interlace, reserved;   /* IHDR fields; reserved is ignored */
} nastar_png_desc;

/* PNG images to L planes, bit-equal to Pillow's Image.open(f).convert("L") (DESIGN.md §16).  data: the device bytes
 * the descriptors point into (data_bytes long); desc: the B descriptors in HOST memory, read for the checks; desc_dev:
 * the same B descriptors in device memory, read by the kernel.  Per image: zlib header, inflate (stored, fixed and
 * dynamic Huffman blocks), the exact inflated length that IHDR implies and the Adler-32; the scanline filters; Adam7
 * when interlace = 1; then L: grey 1/2/4 bits scaled to 0..255, 16-bit grey min(v, 255), RGB and RGBA
 * (19595 R + 38470 G + 7471 B + 0x8000) >> 16 of the samples' high bytes, grey+alpha its grey high byte, palette the
 * RGB rule of the PLTE entry ((0, 0, 0) past its end).  Writes out's planes and status i32 [B]: 0, or an OR of
 * 1 bad zlib header, 2 bad block type or Huffman code (over-subscribed, incomplete, or a code that is not used),
 * 4 a distance past the start of the output, 8 the stream ends early or inflates to more or less than IHDR implies,
 * 16 Adler-32 mismatch, 32 a filter byte above 4.  A plane whose status is not 0 is unspecified; a corrupt stream
 * reads and writes nothing outside its own ranges and workspace slot.  Every check precedes the launch: null pointers,
 * B <= 0, a width or height <= 0, an illegal bit depth / colour type pair, interlace not 0 or 1, or a range outside
 * data / out give NASTAR_EINVAL; W0 or H0 > 2048 gives NASTAR_EUNSUPPORTED; a workspace below
 * nastar_b200_decode_png_workspace_bytes gives NASTAR_EWORKSPACE.  One kernel launch (persistent CTAs, one workspace
 * slot each).  Asynchronous on `stream`.  Returns NASTAR_*. */
int nastar_b200_decode_png(const uint8_t *data, int64_t data_bytes, const nastar_png_desc *desc,
                           const nastar_png_desc *desc_dev, int32_t B, uint8_t *out, int64_t out_bytes,
                           int32_t *status, void *workspace, size_t workspace_bytes, void *stream);

/* Workspace of nastar_b200_decode_png for these B host descriptors: a queue counter and one slot of the largest
 * inflated size per persistent CTA, so it grows with the CTAs (at most 8 per SM), not with B.  0 for arguments that
 * nastar_b200_decode_png rejects with NASTAR_EINVAL or NASTAR_EUNSUPPORTED. */
size_t nastar_b200_decode_png_workspace_bytes(const nastar_png_desc *desc, int32_t B);

/* The reference's heap A* (pq_astar.solve_single, use_differentiable_astar=False), exactly (DESIGN.md §17).  Planes
 * fp32 [B][H][W] with map strides in elements: cost, start, goal, map.  Per map: start and goal are the single
 * non-zero cell of their planes; a neighbour (W, E, N, S, NW, NE, SW, SE order) is entered only where map == 1 and is
 * charged f_new = ((f_sel - (1-g) h(sel)) + g cost[nb]) + (1-g) h(nb), h = max(dx, dy) + 0.001 sqrt(dx^2 + dy^2),
 * each operation one fp64 rounding; the open list is a binary heap with pqdict 1.2.0's moves, which decide ties.
 * Writes histories fp32 [B][H*W] (the closed set), paths int64 [B][H*W] (the parent chain from the goal), status
 * i32 [B] (0 solved, 1 goal not found: histories and paths zero, 2 start or goal not exactly one cell: zero too) and
 * expansions i32 [B] (cells closed).  Every check precedes the launch: null pointers, B, H or W <= 0, a stride
 * below H*W or a workspace not 8-byte aligned give NASTAR_EINVAL; H*W > 1048576 gives NASTAR_EUNSUPPORTED; a workspace below
 * nastar_b200_pq_astar_workspace_bytes gives NASTAR_EWORKSPACE.  One kernel launch (persistent one-warp CTAs).
 * Asynchronous on `stream`.  Returns NASTAR_*. */
int nastar_b200_pq_astar(const float *cost, int64_t cost_stride, const float *start, int64_t start_stride,
                         const float *goal, int64_t goal_stride, const float *map, int64_t map_stride, int32_t B,
                         int32_t H, int32_t W, double g_ratio, float *histories, int64_t *paths, int32_t *status,
                         int32_t *expansions, void *workspace, size_t workspace_bytes, void *stream);

/* Workspace of nastar_b200_pq_astar: a work counter, plus, for maps whose state does not fit in shared memory, one
 * 20*H*W-byte slot per persistent CTA (at most 8 per SM and 2 GiB in all, but one per SM always), so it does not grow
 * with B.  0 for shapes that nastar_b200_pq_astar rejects. */
size_t nastar_b200_pq_astar_workspace_bytes(int32_t B, int32_t H, int32_t W);

/* One member of a nastar_b200_deflate batch.  Pointers are device addresses; lengths are in bytes. */
typedef struct nastar_deflate_desc {
    const uint8_t *head; /* compressed as the member's first chunk (the .npy header); may be NULL when head_len is 0 */
    int64_t head_len;    /* at most one chunk, 262144 bytes */
    const uint8_t *data; /* compressed as the member's next ceil(data_len / 262144) chunks; NULL when data_len is 0 */
    int64_t data_len;
    int64_t gap;         /* bytes left untouched in `out` before the member's stream (room for a zip local header) */
    int64_t chunk0;      /* the member's first chunk: the sum of 1 + ceil(data_len / 262144) over earlier members */
} nastar_deflate_desc;

/* Raw deflate streams of M members, byte-equal to oracle/deflate_oracle.c (DESIGN.md §18).  Each member is cut into
 * 256 KiB chunks (its head first, as one chunk of its own), each compressed alone into one dynamic-Huffman block or
 * stored blocks; chunks other than a member's last end with an empty stored block, and the streams are written back
 * to back into `out`, member m at out_off[m] (its gap before it), out_len[m] bytes.  crc[m] is the CRC-32 of the
 * member's raw head || data.  desc: the descriptors in HOST memory, read for the checks; desc_dev: the same M
 * descriptors in device memory, read by the kernel.  Every check precedes the launch: null pointers, M <= 0, a
 * negative length or gap, a head_len above 262144, a chunk0 that is not the running chunk count, or an output array
 * or the workspace overlapping another of them or an input give NASTAR_EINVAL; out_bytes below nastar_b200_deflate_bound or a workspace below
 * nastar_b200_deflate_workspace_bytes gives NASTAR_EWORKSPACE.  One kernel launch (persistent CTAs, one workspace
 * slot each).  Asynchronous on `stream`.  Returns NASTAR_*. */
int nastar_b200_deflate(const nastar_deflate_desc *desc, const nastar_deflate_desc *desc_dev, int32_t M, uint8_t *out,
                        int64_t out_bytes, int64_t *out_off, int64_t *out_len, uint32_t *crc, void *workspace,
                        size_t workspace_bytes, void *stream);

/* The bytes nastar_b200_deflate may write to `out` for these M host descriptors (gaps included), the worst case of
 * every chunk, as zlib's deflateBound; -1 for descriptors that nastar_b200_deflate rejects with NASTAR_EINVAL. */
int64_t nastar_b200_deflate_bound(const nastar_deflate_desc *desc, int32_t M);

/* Workspace of nastar_b200_deflate: a chunk counter, a publication ring and one 2.6 MB slot per persistent CTA (one
 * per SM at most), so it grows with the SMs, not with the input.  0 for descriptors it rejects. */
size_t nastar_b200_deflate_workspace_bytes(const nastar_deflate_desc *desc, int32_t M);

/* One image of a PNG encode batch (DESIGN.md §21).  Pointers are device addresses; offsets are in bytes. */
typedef struct nastar_png_enc_desc {
    const uint8_t *pixels; /* H*W uint8 grey levels, row-major and contiguous */
    int64_t filt_off;      /* the image's filtered stream, H*(W+1) bytes, in `filt` */
    int32_t W, H;          /* 1 .. 2048 each */
} nastar_png_enc_desc;

/* First of the three launches of a PNG encode: filt_off gets each image's filtered scanlines (filter byte, then the
 * row under the filter type 0..4 with the least sum of |byte as int8|, ties to the lowest type; row 0 sees zeros
 * above it) and adler[i] the Adler-32 of those H*(W+1) bytes.  Then nastar_b200_deflate compresses them: member i is
 * head_len 0, data filt + filt_off[i], data_len H*(W+1), gap nastar_b200_png_gap(i), into an `out` of
 * nastar_b200_png_encode_bound bytes.  desc: the descriptors in HOST memory, read for the checks; desc_dev: the same B
 * descriptors in device memory, read by the kernel.  Every check precedes the launch: null pointers (a pixels pointer
 * included), B <= 0, a side <= 0 or a negative filt_off give NASTAR_EINVAL; a side above 2048 gives
 * NASTAR_EUNSUPPORTED; a filtered range past filt_bytes gives NASTAR_EWORKSPACE.  One kernel launch (one CTA per
 * image).  Asynchronous on `stream`.  Returns NASTAR_*. */
int nastar_b200_png_filter(const nastar_png_enc_desc *desc, const nastar_png_enc_desc *desc_dev, int32_t B,
                           uint8_t *filt, int64_t filt_bytes, uint32_t *adler, void *stream);

/* Third launch: around image i's deflate stream (out_off[i], out_len[i] from nastar_b200_deflate), the 43 bytes of
 * signature, IHDR (8-bit grey, not interlaced) with its CRC, IDAT length and type and zlib header 78 DA before it,
 * and the 20 bytes of Adler-32, IDAT CRC-32 and an IEND chunk after it, all computed on the device.  File i is then
 * out[out_off[i] - 43, out_off[i] + out_len[i] + 20), and the files lie back to back.  Every check precedes the
 * launch: those of nastar_b200_png_filter (filt_off is not read) and null out_off, out_len, adler or out give
 * NASTAR_EINVAL; out_bytes below nastar_b200_png_encode_bound gives NASTAR_EWORKSPACE.  One kernel launch (one CTA per
 * image).  Asynchronous on `stream`.  Returns NASTAR_*. */
int nastar_b200_png_finish(const nastar_png_enc_desc *desc, const nastar_png_enc_desc *desc_dev, int32_t B,
                           const int64_t *out_off, const int64_t *out_len, const uint32_t *adler, uint8_t *out,
                           int64_t out_bytes, void *stream);

/* The deflate gap before image i's stream: 43 bytes of its head, plus 20 of image i-1's tail when i > 0. */
int64_t nastar_b200_png_gap(int32_t i);

/* The bytes `out` needs for these B host descriptors: nastar_b200_deflate_bound of the members above plus the last
 * image's 20-byte tail; -1 for descriptors nastar_b200_png_filter rejects. */
int64_t nastar_b200_png_encode_bound(const nastar_png_enc_desc *desc, int32_t B);

/* One source image of nastar_b200_crop_resize_rgb.  pixels is a device address. */
typedef struct nastar_rgb_image {
    const uint8_t *pixels; /* H rows of W RGB triples, row y at pixels + y * pitch */
    int64_t pitch;         /* bytes between rows, >= 3 W */
    int32_t W, H;          /* 1 .. 4096 each */
} nastar_rgb_image;

/* One crop of nastar_b200_crop_resize_rgb: the box [x0, x1) x [y0, y1) of image `src` in its pixels, which may extend
 * past any edge, resized into output image `out`. */
typedef struct nastar_rgb_crop {
    int32_t src, out;
    int32_t x0, y0, x1, y1;
} nastar_rgb_crop;

/* RGB crops resized to Wo x Ho, bit-equal to Pillow's np.array(image.crop(box).resize((Wo, Ho))) (BICUBIC,
 * reducing_gap=None) for an RGB image (DESIGN.md §22).  A box pixel outside its source is 0 in every channel; each
 * channel is resized as Pillow resizes an L image: a horizontal pass into a uint8 intermediate when x1 - x0 != Wo,
 * then a vertical pass when y1 - y0 != Ho, with 22-bit fixed-point weights.  Writes out uint8 [N][Ho][Wo][3], crop i
 * to image crops[i].out.  src / crops: the S images and N crops in HOST memory, read for the checks; src_dev /
 * crops_dev: the same descriptors in device memory, read by the kernel.  CTA i takes crops[i], so list the largest
 * boxes first: the long CTAs then start first.  Every check precedes the launch: null pointers (a pixels pointer
 * included), S, N, Ho or Wo <= 0, a side <= 0, a pitch below 3 W, a src outside [0, S), out indices that are not a
 * permutation of 0 .. N-1, or an empty box (x1 <= x0 or y1 <= y0) give NASTAR_EINVAL; a source side or box side above
 * 4096, or Ho or Wo above 1024, gives NASTAR_EUNSUPPORTED.  Needs no workspace.  One kernel launch (one CTA per crop).
 * Asynchronous on `stream`.  Returns NASTAR_*. */
int nastar_b200_crop_resize_rgb(const nastar_rgb_image *src, const nastar_rgb_image *src_dev, int32_t S,
                                const nastar_rgb_crop *crops, const nastar_rgb_crop *crops_dev, int32_t N, int32_t Ho,
                                int32_t Wo, uint8_t *out, void *stream);

/* One zip member of a nastar_b200_inflate batch.  Offsets and lengths are in bytes. */
typedef struct nastar_inflate_desc {
    int64_t in_off, in_len;    /* the member's stored bytes or raw deflate stream in `data` */
    int64_t out_off, out_len;  /* its output range in `out`; out_len is its exact size (the central directory's) */
    int32_t method;            /* the zip compression method: 0 stored, 8 deflated */
    int32_t reserved;          /* ignored */
} nastar_inflate_desc;

/* Bytes of the workspace of nastar_b200_inflate: its queue counter. */
#define NASTAR_INFLATE_WORKSPACE_BYTES 256

/* Zip members to their bytes on the device, each with the CRC-32 of its output: the device half of reading .npz files
 * (utils.data.load_npz_device, DESIGN.md §23), which replaces np.load's zipfile + zlib inflate on the host.  Per
 * member: method 8 inflates the raw deflate stream (stored, fixed and dynamic Huffman blocks, with the block decoder of
 * nastar_b200_decode_png) straight into out[out_off, out_off + out_len), which it must fill exactly; method 0 copies
 * in_len == out_len bytes.  Writes status i32 [M]: 0, or an OR of 2 bad block type or Huffman code, 4 a distance past
 * the start of the output, 8 the stream ends early or inflates to more or less than out_len; and crc u32 [M] (passed as
 * int32), the CRC-32 of the output (unspecified where status is not 0), for the caller to compare with the zip's.  A
 * corrupt stream reads and writes nothing outside its own ranges.  desc: the M descriptors in HOST memory, read for the
 * checks; desc_dev: the same descriptors in device memory, read by the kernel.  Every check precedes the launch: null
 * pointers, M <= 0, a method other than 0 and 8, a negative length, an input range outside data, a stored member whose
 * lengths differ, or output ranges outside out or not in increasing, disjoint order give NASTAR_EINVAL; a workspace
 * below NASTAR_INFLATE_WORKSPACE_BYTES gives NASTAR_EWORKSPACE.  One kernel launch (persistent one-warp CTAs taking
 * members from a queue, so one warp inflates one member: suited to many small members, not to a few huge ones).
 * Asynchronous on `stream`.  Returns NASTAR_*. */
int nastar_b200_inflate(const uint8_t *data, int64_t data_bytes, const nastar_inflate_desc *desc,
                        const nastar_inflate_desc *desc_dev, int32_t M, uint8_t *out, int64_t out_bytes,
                        int32_t *status, uint32_t *crc, void *workspace, size_t workspace_bytes, void *stream);

/* Directed Chamfer distances between two cell sets per map, replacing a host loop over
 * scipy.ndimage.distance_transform_edt (DESIGN.md §23).  masks: uint8 [B][H*W] dense, bit 0 = the cell is in set A,
 * bit 1 = in set B.  Writes out fp64 [B][2]: d(A -> B) and d(B -> A), d(S -> T) the mean over S's cells of the
 * Euclidean distance, in cells, to the nearest cell of T; NaN in both columns of a map where A or B is empty.  The
 * squared distances are exact integers (Meijster's separable transform), each square root is correctly rounded and the
 * sums run in a fixed order, so results are the same from run to run.  Maps whose state does not fit in shared memory
 * use one workspace slot per CTA: nastar_b200_chamfer_workspace_bytes (0 when they all fit; workspace may then be
 * NULL).  Every check precedes the launch: null masks or out, or B, H or W <= 0 give NASTAR_EINVAL; H or W above 1024
 * gives NASTAR_EUNSUPPORTED; a workspace below nastar_b200_chamfer_workspace_bytes gives NASTAR_EWORKSPACE.  One kernel
 * launch, one CTA per map.  Asynchronous on `stream`.  Returns NASTAR_*. */
int nastar_b200_chamfer(const uint8_t *masks, int32_t B, int32_t H, int32_t W, double *out, void *workspace,
                        size_t workspace_bytes, void *stream);
size_t nastar_b200_chamfer_workspace_bytes(int32_t B, int32_t H, int32_t W);

/* Search animations (DESIGN.md §19): G GIFs over a search of B maps, layout NASTAR_GIF_EACH (one GIF per map, G = B)
 * or NASTAR_GIF_GRID (one GIF of all maps in make_grid's layout: 8 per row, 2-pixel border, none for B = 1).  GIF g
 * has T_g steps and T_g + 1 frames, numbered GIF by GIF: frame k < T_g is the closed set before step k and the cell
 * selected at step k, frame T_g the histories and paths.  Planes are contiguous [B, H, W] (channel 0 of [B,1,H,W]). */
#define NASTAR_GIF_EACH 0
#define NASTAR_GIF_GRID 1
#define NASTAR_GIF_STEPS_MAP 0     /* T_g from the map's t_solve (EACH) */
#define NASTAR_GIF_STEPS_BATCH 1   /* T_g = the slowest map's steps, the reference loop's T_batch (GRID) */
#define NASTAR_GIF_STEPS_ALL 2     /* T_g = T: a batch-coupled search that ran exactly T steps (GRID) */

typedef struct nastar_gif_params {
    const float *maps;        /* map designs, grey level uint8(v * 255) with v in [0, 1] */
    const float *histories;   /* the search's outputs */
    const int64_t *paths;
    const float *goal_maps;   /* the goal is the first maximum */
    const int32_t *trace;     /* [B, T]: the cell selected at each step (< H*W, the caller's guarantee: the search
                               * kernels write it so); negative entries stand for the goal */
    const int32_t *t_solve;   /* [B] */
    int32_t B, H, W, T;
    int32_t layout;           /* NASTAR_GIF_EACH or NASTAR_GIF_GRID */
    int32_t steps_mode;       /* NASTAR_GIF_STEPS_* */
    int32_t screen_w, screen_h;   /* the logical screen, each 1 .. 65535 */
    int32_t delay_cs;         /* 0 .. 65535 */
    /* device tables, back to back in this order: int32 xmap[screen_w] and ymap[screen_h] (screen column / row -> image
     * column / row, nondecreasing), int32 xspan[Wi][2] and yspan[Hi][2] (image column / row -> its screen columns /
     * rows [lo, hi)), uint8 lut[G][256] (grey level -> palette index) and uint8 colors[G][2] (number of greys n, LZW
     * minimum code size m): palette indices 0 .. n-1 are the greys, n green, n+1 red, n+2 transparent.  Wi x Hi is the
     * make_grid image. */
    const void *tables;
} nastar_gif_params;

/* Bytes of the tables of nastar_gif_params for these shapes; -1 for parameters nastar_b200_gif_plan rejects. */
int64_t nastar_b200_gif_tables_bytes(const nastar_gif_params *p);

/* First of the two launches: writes steps[G] (T_g) and nbytes[G * (T + 1)] (for frame f < sum(T_g + 1): the bytes of
 * its LZW stream).  Every check precedes the launch: null pointers, B, H, W or T below 1, an unknown layout or
 * steps_mode (STEPS_MAP with GRID, BATCH or ALL with EACH), a screen side outside 1 .. 65535 or delay_cs outside
 * 0 .. 65535 give NASTAR_EINVAL (the tables' contents are the caller's); H * W above 2^24 gives NASTAR_EUNSUPPORTED; a workspace
 * below nastar_b200_gif_workspace_bytes gives NASTAR_EWORKSPACE.  One kernel launch (persistent CTAs).  The same
 * workspace, untouched, goes to nastar_b200_gif_encode.  Asynchronous on `stream`.  Returns NASTAR_*. */
int nastar_b200_gif_plan(const nastar_gif_params *p, int32_t *steps, int32_t *nbytes, void *workspace,
                         size_t workspace_bytes, void *stream);

/* The bytes of one frame's record for an LZW stream of lzw_bytes: graphic control extension (8), image descriptor
 * (10), minimum code size (1), the stream in sub-blocks of at most 255 bytes, terminator (1); -1 for lzw_bytes < 1. */
int64_t nastar_b200_gif_record_bytes(int64_t lzw_bytes);

/* Second launch: every frame's record, frame f at offset[f] of `out`.  p, nbytes and the workspace are those of the
 * plan; nbytes_host and offset_host are the host copies of nbytes[0 .. n_frames) and offset[0 .. n_frames] that the
 * checks read (offset_dev: the same offsets in device memory, read by the kernel).  Every check precedes the launch:
 * the plan's checks, n_frames below 1 or above G * (T + 1), an offset that does not start at 0 or does not advance by
 * nastar_b200_gif_record_bytes(nbytes[f]), or an out_bytes below offset[n_frames] give NASTAR_EINVAL.  n_frames must
 * be the sum of T_g + 1 of the plan.  May run again on the same plan and workspace.  One kernel launch.  Asynchronous
 * on `stream`.  Returns NASTAR_*. */
int nastar_b200_gif_encode(const nastar_gif_params *p, const int32_t *nbytes, const int32_t *nbytes_host,
                           const int64_t *offset_host, const int64_t *offset_dev, int64_t n_frames, uint8_t *out,
                           int64_t out_bytes, void *workspace, size_t workspace_bytes, void *stream);

/* Workspace of the two GIF launches: a control block, per-map goals and first-selection tables (4*H*W bytes each) and
 * per-frame rectangles (16 bytes each); 0 for parameters they reject. */
size_t nastar_b200_gif_workspace_bytes(const nastar_gif_params *p);

/* Number of kernel launches issued by this library since load (bench.py's gpu_launches). */
uint64_t nastar_b200_launch_count(void);

const char *nastar_b200_status_string(int status);
/* cudaGetErrorString of the last failing CUDA call made by this library (thread-unsafe, debug aid) */
const char *nastar_b200_last_cuda_error(void);

#ifdef __cplusplus
}
#endif
#endif /* NASTAR_B200_H_ */
