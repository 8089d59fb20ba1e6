// nastar_api.cu — C-ABI entry points of libnastar_b200.so (see include/nastar_b200.h).
// Host side only validates, picks an engine and launches; no torch types, no CPU fallback.
#include <cuda_runtime.h>
#include <atomic>
#include <cmath>
#include <cstdio>

#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <vector>

#include "../../include/nastar_b200.h"
#include "nastar_bin16.cuh"
#include "nastar_chamfer.cuh"
#include "nastar_convhead.cuh"
#include "nastar_crops.cuh"
#include "nastar_deflate.cuh"
#include "nastar_generic.cuh"
#include "nastar_gif.cuh"
#include "nastar_glue.cuh"
#include "nastar_goals.cuh"
#include "nastar_inflate.cuh"
#include "nastar_labels.cuh"
#include "nastar_maps.cuh"
#include "nastar_png.cuh"
#include "nastar_png_encode.cuh"
#include "nastar_pq.cuh"
#include "nastar_sampler.cuh"
#include "nastar_wlabels.cuh"
#include "nastar_warp32.cuh"
#include "nastar_warp64.cuh"

namespace {
std::atomic<uint64_t> g_launches{0};
cudaError_t g_last_err = cudaSuccess;

constexpr size_t kMaxDynSmem = 232448;  // 227 KB opt-in limit per CTA on sm_90
constexpr int kGlobalCtasPerSm = 8;

int num_sms() {
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
            n = 132;   // H100 SXM
    }
    return n;
}

// grid of a kernel that loops over its work: `want` CTAs, but no more than `ctas_per_sm` per SM
int capped_grid(int64_t want, int ctas_per_sm) {
    const int64_t cap = int64_t(num_sms()) * ctas_per_sm;
    return int(want < cap ? want : cap);
}

inline int cuda_fail(cudaError_t e) {
    g_last_err = e;
    return NASTAR_ECUDA;
}

// the last step of every entry point that launched a kernel: the launch counts once issued, then its error is read
int launched() {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? NASTAR_OK : cuda_fail(e);
}

// opts `kernel` in to `smem` bytes of dynamic shared memory, then launches it; returns the opt-in's error (the launch's
// own error is left for launched())
template <class... P, class... A>
cudaError_t launch_smem(void (*kernel)(P...), int grid, int block, size_t smem, cudaStream_t stream, const A&... args) {
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    if (e == cudaSuccess) kernel<<<grid, block, smem, stream>>>(args...);
    return e;
}

// f(std::bool_constant<flags>...): turns runtime flags into template arguments, one instantiation per combination; a
// flag passed as std::false_type has no `true` instantiation
template <class F>
auto with_flags(F&& f) {
    return f();
}
template <class F, class... Rest>
auto with_flags(F&& f, bool flag, Rest... rest) {
    if (flag) return with_flags([&](auto... t) { return f(std::true_type{}, t...); }, rest...);
    return with_flags([&](auto... t) { return f(std::false_type{}, t...); }, rest...);
}
template <class F, class... Rest>
auto with_flags(F&& f, std::false_type, Rest... rest) {
    return with_flags([&](auto... t) { return f(std::false_type{}, t...); }, rest...);
}

// `flag` where the kernel has a variant for it (kHas), else std::false_type
template <bool kHas>
auto flag_if(bool flag) {
    if constexpr (kHas) return flag;
    else return std::false_type{};
}

// one-time fill of the kSide x kSide heuristic table (g_heur32 / g_heur64, or their NEWS twins) on the current device,
// stream-ordered before first use; each table has its own per-device done mask
template <int kSide, bool kNews>
cudaError_t ensure_heur(cudaStream_t stream) {
    static std::atomic<uint64_t> done_mask{0};
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const uint64_t bit = uint64_t(1) << (dev & 63);
    if (done_mask.load(std::memory_order_acquire) & bit) return cudaSuccess;
    nastar::heur_init_kernel<kSide, kNews><<<kSide * kSide / 256, 256, 0, stream>>>();
    g_launches.fetch_add(1, std::memory_order_relaxed);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    // later launches on OTHER streams must also see the table: finish the fill before publishing
    e = cudaStreamSynchronize(stream);
    if (e != cudaSuccess) return e;
    done_mask.fetch_or(bit, std::memory_order_release);
    return cudaSuccess;
}

// SearchArgs of a backward call: the search inputs in `f` (NASTAR_FWD_NEWS in f.flags for `news`), then the
// backward-only fields
nastar::SearchArgs bwd_kernel_args(const nastar_bwd_params* p, bool news) {
    nastar::SearchArgs a{};
    a.f.cost = p->cost;   a.f.cost_stride = p->cost_stride;
    a.f.start = p->start; a.f.start_stride = p->start_stride;
    a.f.goal = p->goal;   a.f.goal_stride = p->goal_stride;
    a.f.obst = p->obst;   a.f.obst_stride = p->obst_stride;
    a.f.B = p->B; a.f.H = p->H; a.f.W = p->W;
    a.f.g_ratio = p->g_ratio;
    a.f.one_minus_g_ratio = p->one_minus_g_ratio;
    a.f.T = 0;   // the loop bound comes from *T_batch on the device
    a.f.flags = news ? NASTAR_FWD_NEWS : 0;
    a.f.workspace = p->workspace;
    a.f.workspace_bytes = p->workspace_bytes;
    a.sqrt_w = p->sqrt_w;
    a.T_batch = p->T_batch;
    a.t_solve_in = p->t_solve;
    a.grad_hist = p->grad_histories;
    a.grad_stride = p->grad_stride;
    a.grad_cost = p->grad_cost;
    return a;
}

// generic engine variant for a shape: 2 = state in shared memory, 3 = state in the HBM workspace, 0 = too large
int generic_engine_for(int32_t H, int32_t W) {
    if (H <= 0 || W <= 0 || int64_t(H) * W > (int64_t(1) << 30)) return 0;
    const nastar::GenericLayout L(H, W);
    if (L.smem_common() + L.smem_planes() <= kMaxDynSmem) return 2;
    if (L.smem_common() <= kMaxDynSmem) return 3;
    return 0;
}

int generic_slots(int B) { return capped_grid(B, kGlobalCtasPerSm); }

// Launches the search kernel of `engine` (nastar_b200_engine_for) for the problems in a.f, with exit mode kExit, or the
// backward replay (kBwd).  The variant follows a.f: a trace when a.f.trace is set, the fused prologue for cost_kind !=
// NASTAR_COST_PLANE, 4-connected for NASTAR_FWD_NEWS; the 32-wide engine runs 2B CTAs under NASTAR_FWD_PAIR.  The
// generic engine gets one CTA per map, or one per workspace slot when its state or the backward lives in the
// workspace.  Fills the heuristic table first where the engine reads one; the launch is left for launched().
// kExit may carry nastar::kExitBlackbox (the black-box backward: no trace, plain cost plane, no pair).
template <int kExit, bool kBwd>
cudaError_t launch_search(int engine, const nastar::SearchArgs& a, cudaStream_t stream) {
    constexpr bool kMayTrace = !kBwd && (kExit == nastar::kExitEarly || kExit == nastar::kExitNone);
    constexpr bool kBlackbox = (kExit & nastar::kExitBlackbox) != 0;
    const auto trace = flag_if<kMayTrace>(a.f.trace != nullptr);
    const auto fused = flag_if<!kBwd && !kBlackbox>(a.f.cost_kind != NASTAR_COST_PLANE);
    const bool news = (a.f.flags & NASTAR_FWD_NEWS) != 0;
    const int B = a.f.B;
    if (engine == 1 || engine == 4) {
        const cudaError_t e = (engine == 1) ? (news ? ensure_heur<32, true>(stream) : ensure_heur<32, false>(stream))
                                            : (news ? ensure_heur<64, true>(stream) : ensure_heur<64, false>(stream));
        if (e != cudaSuccess) return e;
    }
    if (engine == 1) {
        const int grid = (a.f.flags & NASTAR_FWD_PAIR) ? 2 * B : B;   // output slots
        return with_flags([&](auto kTrace, auto kFused, auto kNews) {
            // the backward's dynamic shared memory is the per-cell interval state of the event-based closed form
            // (W32Bwd, 32 KB); with the 17.4 KB of static planes that is above the 48 KB default, hence the opt-in
            if constexpr (kBwd) {
                return launch_smem(nastar::astar_warp32_kernel<kTrace, true, kExit, kFused, kNews>, grid, 32,
                                   sizeof(nastar::W32Bwd), stream, a);
            } else {
                nastar::astar_warp32_kernel<kTrace, false, kExit, kFused, kNews><<<grid, 32, 0, stream>>>(a);
                return cudaSuccess;
            }
        }, trace, fused, news);
    }
    if (engine == 4) {
        // the backward's event-based closed form keeps its per-cell state next to the forward state in shared memory
        const size_t smem = sizeof(nastar::W64Smem) + (kBwd ? sizeof(nastar::W64Bwd) : 0);
        return with_flags([&](auto kTrace, auto kFused, auto kNews) {
            return launch_smem(nastar::astar_warp64_kernel<kTrace, kExit, kBwd, kFused, kNews>, B, 32, smem, stream, a);
        }, trace, fused, news);
    }
    const nastar::GenericLayout L(a.f.H, a.f.W);
    const bool global = (engine == 3);
    const size_t smem = L.smem_common() + (global ? 0 : L.smem_planes());
    const int grid = (global || kBwd) ? generic_slots(B) : B;
    return with_flags([&](auto kGlobal, auto kTrace, auto kNews) {
        return launch_smem(nastar::astar_generic_kernel<kGlobal, kTrace, kBwd, kExit, kNews>, grid, 32, smem, stream,
                           a);
    }, global, trace, news);
}

// ---- engine 5 (nastar_bin16.cuh): binary-cost maps, one CTA per map --------------------------------------
// NASTAR_B200_BIN16=0 in the environment disables it (A/B measurements against engines 2/3)
bool bin16_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = std::getenv("NASTAR_B200_BIN16");
        v = (e && e[0] == '0') ? 0 : 1;
    }
    return v != 0;
}

bool bin16_shape_ok(int32_t H, int32_t W) {
    if (H <= 0 || W <= 0 || (H <= 64 && W <= 64)) return false;   // engines 1 / 4 keep their shapes
    if (generic_engine_for(H, W) == 0) return false;
    const nastar::Bin16Layout L(H, W);
    return L.supported() && L.smem_bytes() <= kMaxDynSmem;
}

// head of the workspace when engine 5 may run: [0,256) work-queue counter, then B redo flags (256-B granules)
size_t bin16_aux_bytes(int32_t B) { return 256 + ((size_t(B) * 4 + 255) & ~size_t(255)); }

__global__ void batch_steps_kernel(const int32_t* __restrict__ t_solve, const int32_t* __restrict__ n_steps,
                                   int B, int T, int32_t* __restrict__ out) {
    // T_batch = number of iterations of the reference's batch-synchronous loop
    // (differentiable_astar.py:203,251-252): it stops right after the slowest map's solve step,
    // or runs all T iterations if some map never reaches its goal.
    int m = 0;
    for (int i = threadIdx.x; i < B; i += blockDim.x) {
        const int ts = t_solve[i];
        const int v = (ts >= 0) ? (ts + 1) : T;
        m = max(m, v);
        (void)n_steps;
    }
    for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
    __shared__ int sm[32];
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x < 32) {
        m = (threadIdx.x < (blockDim.x >> 5)) ? sm[threadIdx.x] : 0;
        for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
        if (threadIdx.x == 0) out[0] = min(m, T);
    }
}

// ---- batch-coupled forward (nastar_b200_forward_coupled) ------------------------------------------------
inline size_t round256(size_t n) { return (n + 255) & ~size_t(255); }

// head of the coupled forward's workspace: stop / end / first [B] int32 each, then the at-goal bitmaps [B][ceil(T/32)];
// the generic engine's slots (engine 3) follow
size_t coupled_aux_bytes(int32_t B, int32_t T) {
    const size_t words = (size_t(T) + 31) / 32;
    return 3 * round256(size_t(B) * 4) + round256(size_t(B) * words * 4);
}

nastar::CoupledWs coupled_ws(void* workspace, int32_t B, int32_t T) {
    unsigned char* w = static_cast<unsigned char*>(workspace);
    const size_t per_map = round256(size_t(B) * 4);
    nastar::CoupledWs cw;
    cw.stop = reinterpret_cast<int32_t*>(w);
    cw.end = reinterpret_cast<int32_t*>(w + per_map);
    cw.first = reinterpret_cast<int32_t*>(w + 2 * per_map);
    cw.bits = reinterpret_cast<uint32_t*>(w + 3 * per_map);
    cw.words = (T + 31) / 32;
    return cw;
}

constexpr int kCoupledThreads = 512;

template <class Op>
__device__ int block_reduce(int v, Op op, int* red) {
    for (int o = 16; o; o >>= 1) v = op(v, __shfl_xor_sync(0xFFFFFFFFu, v, o));
    __syncthreads();   // red[] may still be read by the previous reduction
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    v = red[0];
    for (int i = 1; i < int(blockDim.x >> 5); ++i) v = op(v, red[i]);
    return v;
}

// T_batch = 1 + min{k < T : every map selects its goal at step k}, or T (differentiable_astar.py:251-252), from the
// at-goal bitmaps of pass 1; then goal_clamp[b] = 0 if map b selects its goal at least twice within T_batch steps,
// else T_batch (the t_solve encoding of nastar_bwd_params).  Integer AND / min / popcount only: deterministic.
__global__ void __launch_bounds__(kCoupledThreads) coupled_reduce_kernel(const nastar::CoupledWs cw, int B, int T,
                                                                         int32_t* __restrict__ T_batch,
                                                                         int32_t* __restrict__ goal_clamp) {
    __shared__ int red[kCoupledThreads / 32];
    auto imax = [](int x, int y) { return max(x, y); };
    auto iand = [](int x, int y) { return x & y; };
    // no step before the last map's first goal selection can have every map at its goal; a map that never selects
    // its goal keeps T_batch at T
    int lo = 0;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const int f = cw.first[b];
        lo = max(lo, f < 0 ? T : f);
    }
    lo = block_reduce(lo, imax, red);
    int Tb = T;
    for (int w = lo >> 5; w < cw.words; ++w) {
        uint32_t all = 0xFFFFFFFFu;
        for (int b = threadIdx.x; b < B; b += blockDim.x) all &= nastar::coupled_word(cw, b, w);
        all = uint32_t(block_reduce(int(all), iand, red));
        if (w == cw.words - 1 && (T & 31)) all &= (1u << (T & 31)) - 1u;
        if (all) { Tb = (w << 5) + __ffs(all); break; }   // block-uniform
    }
    if (threadIdx.x == 0) T_batch[0] = Tb;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const int f = cw.first[b];
        int n = 0;
        if (f >= 0) {
            for (int w = f >> 5; (w << 5) < Tb && n < 2; ++w) {
                uint32_t v = nastar::coupled_word(cw, b, w);
                if (Tb - (w << 5) < 32) v &= (1u << (Tb - (w << 5))) - 1u;
                n += __popc(v);
            }
        }
        goal_clamp[b] = (n >= 2) ? 0 : Tb;
    }
}

// the three launches of a batch-coupled search (nastar_b200_forward_coupled): pass 1 (kExitCoupled1), the reduction,
// pass 2 (kExitCoupled2), each with the extra mode bits kMore (nastar::kExitBlackbox for the black-box backward).
// `a` holds the problems; its records and engine-3 slots are carved from p->workspace here.
template <int kMore>
int run_coupled(int engine, nastar::SearchArgs a, const nastar_fwd_params* p, int32_t* T_batch, int32_t* goal_clamp,
                cudaStream_t stream) {
    a.T_batch = T_batch;
    a.cw = coupled_ws(p->workspace, p->B, p->T);
    if (engine == 2 || engine == 3) {
        const size_t aux = coupled_aux_bytes(p->B, p->T);
        a.f.workspace = static_cast<unsigned char*>(p->workspace) + aux;   // engine 3's slots follow the records
        a.f.workspace_bytes = p->workspace_bytes - aux;
    }
    // no host round trip between the three launches
    cudaError_t e = launch_search<nastar::kExitCoupled1 | kMore, false>(engine, a, stream);
    if (e != cudaSuccess) return cuda_fail(e);
    int st = launched();
    if (st != NASTAR_OK) return st;
    coupled_reduce_kernel<<<1, kCoupledThreads, 0, stream>>>(a.cw, p->B, p->T, T_batch, goal_clamp);
    st = launched();
    if (st != NASTAR_OK) return st;
    e = launch_search<nastar::kExitCoupled2 | kMore, false>(engine, a, stream);
    if (e != cudaSuccess) return cuda_fail(e);
    return launched();
}

// ---- PNG decode (nastar_png.cuh) -----------------------------------------------------------------------------
// NASTAR_OK, or the status nastar_b200_decode_png returns for these descriptors; *max_raw = the largest inflated size
int png_check(const nastar_png_desc* desc, int32_t B, int64_t data_bytes, int64_t out_bytes, int64_t* max_raw) {
    if (!desc || B <= 0) return NASTAR_EINVAL;
    auto inside = [](int64_t off, int64_t len, int64_t total) { return off >= 0 && len >= 0 && len <= total - off; };
    int st = NASTAR_OK;
    *max_raw = 0;
    for (int32_t i = 0; i < B; ++i) {
        const nastar_png_desc& d = desc[i];
        if (d.W0 <= 0 || d.H0 <= 0 || !nastar::png_legal(d.bit_depth, d.color_type) || d.interlace < 0 ||
            d.interlace > 1)
            return NASTAR_EINVAL;
        if (d.W0 > nastar::kPngMaxSide || d.H0 > nastar::kPngMaxSide) {
            st = NASTAR_EUNSUPPORTED;   // a later descriptor may still be invalid, which takes precedence
            continue;
        }
        if (!inside(d.in_off, d.in_len, data_bytes) || !inside(d.plte_off, d.plte_len, data_bytes) ||
            !inside(d.out_off, int64_t(d.W0) * d.H0, out_bytes))
            return NASTAR_EINVAL;
        const int64_t r = nastar::png_raw_bytes(d.W0, d.H0, d.bit_depth, d.color_type, d.interlace);
        *max_raw = r > *max_raw ? r : *max_raw;
    }
    return st;
}

size_t png_slot_bytes(int64_t max_raw) { return round256(size_t(max_raw)); }

// ---- deflate (nastar_deflate.cuh) -----------------------------------------------------------------------------
// the bytes nastar_b200_deflate may write (gaps included) and *chunks, or -1 for descriptors it rejects as EINVAL
int64_t deflate_check(const nastar_deflate_desc* desc, int32_t M, int64_t* chunks) {
    if (!desc || M <= 0) return -1;
    int64_t bound = 0, k = 0;
    for (int32_t i = 0; i < M; ++i) {
        const nastar_deflate_desc& d = desc[i];
        if (d.head_len < 0 || d.head_len > nastar::kDeflateChunk || d.data_len < 0 || d.gap < 0 || d.chunk0 != k)
            return -1;   // the head is one chunk: the slot's buffers hold kDeflateChunk positions
        if ((d.head_len > 0 && !d.head) || (d.data_len > 0 && !d.data)) return -1;
        bound += d.gap + nastar::deflate_member_bound(d.head_len, d.data_len);
        k += nastar::deflate_member_chunks(d.data_len);
    }
    *chunks = k;
    return bound;
}

constexpr size_t kDeflateCtl = 256 + nastar::kDeflateRing * sizeof(nastar::DeflatePub);   // counter, ring

int deflate_grid(int64_t chunks) { return capped_grid(chunks, 1); }

// ---- PNG encode (nastar_png_encode.cuh) -----------------------------------------------------------------------------
// NASTAR_OK, or the status nastar_b200_png_filter returns for these descriptors (filt_bytes < 0: the filtered ranges
// are not checked); *bound = nastar_b200_png_encode_bound
int png_enc_check(const nastar_png_enc_desc* desc, int32_t B, int64_t filt_bytes, int64_t* bound) {
    if (!desc || B <= 0) return NASTAR_EINVAL;
    int st = NASTAR_OK;
    *bound = nastar::kPngEncTail;
    for (int32_t i = 0; i < B; ++i) {
        const nastar_png_enc_desc& d = desc[i];
        if (!d.pixels || d.W <= 0 || d.H <= 0 || d.filt_off < 0) return NASTAR_EINVAL;
        if (d.W > nastar::kPngEncMaxSide || d.H > nastar::kPngEncMaxSide) {
            st = NASTAR_EUNSUPPORTED;   // a later descriptor may still be invalid, which takes precedence
            continue;
        }
        const int64_t n = nastar::png_filtered_bytes(d.W, d.H);
        if (filt_bytes >= 0 && d.filt_off > filt_bytes - n && st == NASTAR_OK) st = NASTAR_EWORKSPACE;
        *bound += nastar::png_gap(i) + nastar::deflate_member_bound(0, n);
    }
    return st;
}

// ---- .npz members (nastar_inflate.cuh) --------------------------------------------------------------------------
// NASTAR_OK or NASTAR_EINVAL for these descriptors: a known method, ranges inside data / out, output ranges in
// increasing, disjoint order, and stored members of equal lengths
int inflate_check(const nastar_inflate_desc* desc, int32_t M, int64_t data_bytes, int64_t out_bytes) {
    if (!desc || M <= 0) return NASTAR_EINVAL;
    auto inside = [](int64_t off, int64_t len, int64_t total) { return off >= 0 && len >= 0 && len <= total - off; };
    int64_t end = 0;
    for (int32_t i = 0; i < M; ++i) {
        const nastar_inflate_desc& d = desc[i];
        if ((d.method != 0 && d.method != 8) || (d.method == 0 && d.in_len != d.out_len)) return NASTAR_EINVAL;
        if (!inside(d.in_off, d.in_len, data_bytes) || !inside(d.out_off, d.out_len, out_bytes) || d.out_off < end)
            return NASTAR_EINVAL;
        end = d.out_off + d.out_len;
    }
    return NASTAR_OK;
}

// ---- Chamfer distances (nastar_chamfer.cuh) ---------------------------------------------------------------------
constexpr size_t kChamferWorkspaceBudget = size_t(256) << 20;   // global slots: at most this much, but one always

bool chamfer_global(int32_t H, int32_t W) { return nastar::chamfer_layout(H, W).bytes > nastar::kChamferSmemMax; }
size_t chamfer_slot_bytes(int32_t H, int32_t W) { return round256(size_t(nastar::chamfer_layout(H, W).bytes)); }
int chamfer_grid(int32_t B, int32_t H, int32_t W) {
    if (!chamfer_global(H, W)) return B;
    const int64_t fit = int64_t(kChamferWorkspaceBudget / chamfer_slot_bytes(H, W));
    const int g = capped_grid(B, 1);
    return int(g < fit ? g : fit > 0 ? fit : 1);
}

// ---- search GIFs (nastar_gif.cuh) ------------------------------------------------------------------------------
struct GifShape {
    int64_t G, Hi, Wi;   // GIFs, make_grid image
    size_t ws_first, ws_rect, ws_bytes;
};

// the shapes of a GIF call, or false for parameters nastar_b200_gif_plan rejects with NASTAR_EINVAL
bool gif_shape(const nastar_gif_params* p, GifShape* s) {
    if (!p || !p->maps || !p->histories || !p->paths || !p->goal_maps || !p->trace || !p->t_solve || !p->tables)
        return false;
    if (p->B <= 0 || p->H <= 0 || p->W <= 0 || p->T <= 0) return false;
    if (p->layout == NASTAR_GIF_EACH ? p->steps_mode != NASTAR_GIF_STEPS_MAP
                                     : p->layout != NASTAR_GIF_GRID || (p->steps_mode != NASTAR_GIF_STEPS_BATCH &&
                                                                        p->steps_mode != NASTAR_GIF_STEPS_ALL))
        return false;
    if (p->screen_w < 1 || p->screen_w > 65535 || p->screen_h < 1 || p->screen_h > 65535) return false;
    if (p->delay_cs < 0 || p->delay_cs > 65535) return false;
    const bool tiled = p->layout == NASTAR_GIF_GRID && p->B > 1;
    const int64_t xmaps = p->B < 8 ? p->B : 8, ymaps = (p->B + xmaps - 1) / xmaps;
    s->G = p->layout == NASTAR_GIF_GRID ? 1 : p->B;
    s->Hi = tiled ? (p->H + 2) * ymaps + 2 : p->H;
    s->Wi = tiled ? (p->W + 2) * xmaps + 2 : p->W;
    const int64_t N = int64_t(p->H) * p->W;
    s->ws_first = round256(size_t(p->B) * 4) + round256(size_t(p->B) * size_t(N) * 4);
    s->ws_rect = round256(size_t(s->G) * size_t(p->T + 1) * 16);
    s->ws_bytes = 256 + 2 * round256(size_t(s->G) * 4) + s->ws_first + s->ws_rect;
    return true;
}

bool gif_supported(const nastar_gif_params* p) { return int64_t(p->H) * p->W <= (int64_t(1) << 24); }

nastar::GifArgs gif_args(const nastar_gif_params* p, const GifShape& s, void* workspace, int32_t* nbytes) {
    nastar::GifArgs a{};
    a.maps = p->maps; a.hist = p->histories; a.paths = p->paths; a.goal = p->goal_maps;
    a.trace = p->trace; a.t_solve = p->t_solve;
    a.B = p->B; a.H = p->H; a.W = p->W; a.T = p->T;
    a.grid = p->layout == NASTAR_GIF_GRID;
    a.steps_mode = p->steps_mode;
    a.Hg = int32_t(s.Hi); a.Wg = int32_t(s.Wi);
    a.SW = p->screen_w; a.SH = p->screen_h;
    const int32_t* t32 = static_cast<const int32_t*>(p->tables);
    a.xmap = t32;
    a.ymap = a.xmap + p->screen_w;
    a.xspan = a.ymap + p->screen_h;
    a.yspan = a.xspan + 2 * s.Wi;
    a.lut = reinterpret_cast<const uint8_t*>(a.yspan + 2 * s.Hi);
    a.ncolors = a.lut + 256 * s.G;
    a.delay_cs = p->delay_cs;
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    a.ctl = reinterpret_cast<nastar::GifCtl*>(ws);
    size_t o = 256;
    a.steps = reinterpret_cast<int32_t*>(ws + o);  o += round256(size_t(s.G) * 4);
    a.frame0 = reinterpret_cast<int32_t*>(ws + o); o += round256(size_t(s.G) * 4);
    a.goal_idx = reinterpret_cast<int32_t*>(ws + o); o += round256(size_t(p->B) * 4);
    a.first = reinterpret_cast<int32_t*>(ws + o);  o += round256(size_t(p->B) * size_t(p->H) * size_t(p->W) * 4);
    a.rect = reinterpret_cast<uint32_t*>(ws + o);
    a.nbytes = nbytes;
    return a;
}

int gif_grid(int64_t items) { return capped_grid(items, 1); }

// ---- heap A* (nastar_pq.cuh) ----------------------------------------------------------------------------------
// Maps whose 20 B/cell state fits in this many bytes keep it in shared memory, larger ones in a global slot per CTA
// (threshold measured on an H100: DESIGN.md §17).
#ifndef NASTAR_PQ_SMEM_MAX_BYTES
#define NASTAR_PQ_SMEM_MAX_BYTES (32 * 1024)
#endif
constexpr size_t kPqWorkspaceBudget = size_t(2) << 30;   // global slots: at most this much, but one CTA per SM always

size_t pq_state_bytes(int32_t H, int32_t W) { return size_t(nastar::kPqBytesPerCell) * size_t(H) * size_t(W); }
bool pq_shared(int32_t H, int32_t W) { return pq_state_bytes(H, W) <= size_t(NASTAR_PQ_SMEM_MAX_BYTES); }
int pq_global_grid(int32_t B, int32_t H, int32_t W) {
    const size_t slot = round256(pq_state_bytes(H, W));
    const int64_t fit = int64_t(kPqWorkspaceBudget / slot);
    const int64_t cap = fit > num_sms() ? fit : num_sms();
    const int g = capped_grid(B, kGlobalCtasPerSm);
    return int(g < cap ? g : cap);
}
bool pq_shape_ok(int32_t B, int32_t H, int32_t W) {
    return B > 0 && H > 0 && W > 0 && int64_t(H) * W <= nastar::kPqMaxCells;
}

template <int C>
void launch_head(const float* x, int64_t P, const float* w_host, float* taps, cudaStream_t stream) {
    nastar::HeadWeights<C> hw;
    for (int i = 0; i < C * 9; ++i) hw.w[i] = w_host[i];
    const int64_t want = ((P + 31) / 32 + nastar::kHeadWarps - 1) / nastar::kHeadWarps;   // one 32-pixel group per warp
    nastar::head_taps_kernel<C><<<capped_grid(want, 16), 32 * nastar::kHeadWarps, 0, stream>>>(x, P, hw, taps);
}
}  // namespace

extern "C" {

int nastar_b200_abi_version(void) { return NASTAR_B200_ABI_VERSION; }

int nastar_b200_engine_for(int32_t H, int32_t W) {
    if (H <= 0 || W <= 0) return 0;
    if (H <= 32 && W <= 32) return 1;
    if (H <= 64 && W <= 64) return 4;   // forward and (event-based) backward on the warp-resident 64-wide engine
    return generic_engine_for(H, W);
}

int nastar_b200_bin16_supported(int32_t H, int32_t W) { return bin16_shape_ok(H, W) ? 1 : 0; }

size_t nastar_b200_forward_workspace_bytes(int32_t B, int32_t H, int32_t W) {
    if (B <= 0) return 0;
    const int engine = nastar_b200_engine_for(H, W);
    if (engine != 2 && engine != 3) return 0;
    size_t n = (engine == 3) ? size_t(generic_slots(B)) * nastar::GenericLayout(H, W).slot_bytes() : 0;
    if (bin16_enabled() && bin16_shape_ok(H, W)) n += bin16_aux_bytes(B);
    return n;
}

size_t nastar_b200_backward_workspace_bytes(int32_t B, int32_t H, int32_t W) {
    if (B <= 0 || nastar_b200_engine_for(H, W) == 1 || nastar_b200_engine_for(H, W) == 4) return 0;
    const int e = generic_engine_for(H, W);
    if (e == 0) return 0;
    return size_t(generic_slots(B)) * nastar::GenericLayout(H, W).slot_total(e == 3, true);
}

int nastar_b200_forward(const nastar_fwd_params* p, void* stream_v) {
    if (!p || !p->cost || !p->start || !p->goal || !p->obst || !p->histories || !p->paths) return NASTAR_EINVAL;
    if (p->B <= 0 || p->H <= 0 || p->W <= 0 || p->T < 1) return NASTAR_EINVAL;
    if (p->cost_kind < NASTAR_COST_PLANE || p->cost_kind > NASTAR_COST_TAPS) return NASTAR_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
    const int engine = nastar_b200_engine_for(p->H, p->W);
    if (engine == 0) return NASTAR_EUNSUPPORTED;
    if (p->cost_kind != NASTAR_COST_PLANE && engine != 1 && engine != 4) return NASTAR_EUNSUPPORTED;   // fused hand-off: H,W <= 64
    const bool pair = (p->flags & NASTAR_FWD_PAIR) != 0;
    if (pair && engine != 1) {
        // two halves back to back: the learned-cost search, then the same problems with cost = obstacles
        const int64_t N = int64_t(p->H) * p->W;
        nastar_fwd_params h = *p;
        h.flags &= ~NASTAR_FWD_PAIR;
        int st = nastar_b200_forward(&h, stream_v);
        if (st != NASTAR_OK) return st;
        h.cost = p->obst;
        h.cost_stride = p->obst_stride;
        h.cost_kind = NASTAR_COST_PLANE;
        h.histories = p->histories + int64_t(p->B) * N;
        h.paths = p->paths + int64_t(p->B) * N;
        if (p->t_solve) h.t_solve = p->t_solve + p->B;
        if (p->n_steps) h.n_steps = p->n_steps + p->B;
        if (p->trace) h.trace = p->trace + int64_t(p->B) * p->T;
        if (p->n_closed) h.n_closed = p->n_closed + p->B;
        if (p->path_len) h.path_len = p->path_len + p->B;
        return nastar_b200_forward(&h, stream_v);
    }
    const int nmaps = pair ? 2 * p->B : p->B;   // output slots (= CTAs of the warp32 engine)
    if (p->trace) {
        cudaError_t e = cudaMemsetAsync(p->trace, 0xFF, size_t(nmaps) * size_t(p->T) * sizeof(int32_t), stream);
        if (e != cudaSuccess) return cuda_fail(e);
    }
    nastar::SearchArgs a{};
    a.f = *p;
    const bool noexit = (p->flags & NASTAR_FWD_NO_EARLY_EXIT) != 0;
    auto launch = [&]() {
        const cudaError_t e = noexit ? launch_search<nastar::kExitNone, false>(engine, a, stream)
                                     : launch_search<nastar::kExitEarly, false>(engine, a, stream);
        return e == cudaSuccess ? launched() : cuda_fail(e);
    };
    if (engine == 1 || engine == 4) return launch();
    const bool global = (engine == 3);
    const size_t slots_bytes =
        global ? size_t(generic_slots(p->B)) * nastar::GenericLayout(p->H, p->W).slot_bytes() : 0;
    if (global && (!p->workspace || p->workspace_bytes < slots_bytes)) return NASTAR_EWORKSPACE;
    // engine 5 first when the cost plane IS the binary obstacle plane (VanillaAstar / Config 5): whole map on
    // chip, one CTA per SM pulling maps from a queue; maps it flags are re-run below by the generic engine.
    // Engine 5 is Moore-only: NEWS searches go straight to the generic engine.
    const bool aliased = (p->obst == p->cost) && (p->obst_stride == p->cost_stride);
    const bool news = (p->flags & NASTAR_FWD_NEWS) != 0;
    const size_t aux = bin16_aux_bytes(p->B);
    if (bin16_enabled() && aliased && !news && !p->trace && p->flags == 0 && bin16_shape_ok(p->H, p->W) && p->workspace &&
        p->workspace_bytes >= aux + slots_bytes) {
        unsigned char* ws = static_cast<unsigned char*>(p->workspace);
        nastar::Bin16Args ba{};
        ba.f = *p;
        ba.queue = reinterpret_cast<int32_t*>(ws);
        ba.redo = reinterpret_cast<int32_t*>(ws + 256);
        cudaError_t e = cudaMemsetAsync(ba.queue, 0, 256, stream);
        if (e != cudaSuccess) return cuda_fail(e);
        const size_t bsmem = nastar::Bin16Layout(p->H, p->W).smem_bytes();
        auto launch16 = [&](auto kernel) -> cudaError_t {
            // the occupancy query needs the shared-memory opt-in, and the grid needs the occupancy
            cudaError_t e2 = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(bsmem));
            if (e2 != cudaSuccess) return e2;
            int per_sm = 1;   // resident CTAs per SM (1 at 256x256, a few for smaller maps)
            e2 = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, nastar::kBin16Threads, bsmem);
            if (e2 != cudaSuccess) return e2;
            kernel<<<capped_grid(p->B, per_sm < 1 ? 1 : per_sm), nastar::kBin16Threads, bsmem, stream>>>(ba);
            return cudaSuccess;
        };
        e = (p->H <= 256) ? launch16(nastar::astar_bin16_kernel<8>) : launch16(nastar::astar_bin16_kernel<16>);
        if (e != cudaSuccess) return cuda_fail(e);
        const int st = launched();
        if (st != NASTAR_OK) return st;
        a.redo = ba.redo;
        a.f.workspace = ws + aux;
        a.f.workspace_bytes = p->workspace_bytes - aux;
    }
    return launch();
}

size_t nastar_b200_forward_coupled_workspace_bytes(int32_t B, int32_t H, int32_t W, int32_t T) {
    if (B <= 0 || T < 1) return 0;
    const int engine = nastar_b200_engine_for(H, W);
    if (engine == 0) return 0;
    const size_t slots = (engine == 3) ? size_t(generic_slots(B)) * nastar::GenericLayout(H, W).slot_bytes() : 0;
    return coupled_aux_bytes(B, T) + slots;
}

int nastar_b200_forward_coupled(const nastar_fwd_params* p, int32_t* T_batch, int32_t* goal_clamp, void* stream_v) {
    if (!p || !T_batch || !goal_clamp || !p->cost || !p->start || !p->goal || !p->obst || !p->histories || !p->paths)
        return NASTAR_EINVAL;
    if (p->B <= 0 || p->H <= 0 || p->W <= 0 || p->T < 1) return NASTAR_EINVAL;
    if (p->cost_kind < NASTAR_COST_PLANE || p->cost_kind > NASTAR_COST_TAPS) return NASTAR_EINVAL;
    if ((p->flags & ~NASTAR_FWD_NEWS) != 0 || p->trace) return NASTAR_EINVAL;
    const int engine = nastar_b200_engine_for(p->H, p->W);
    if (engine == 0) return NASTAR_EUNSUPPORTED;
    if (p->cost_kind != NASTAR_COST_PLANE && engine != 1 && engine != 4) return NASTAR_EUNSUPPORTED;
    const size_t need = nastar_b200_forward_coupled_workspace_bytes(p->B, p->H, p->W, p->T);
    if (!p->workspace || p->workspace_bytes < need) return NASTAR_EWORKSPACE;
    nastar::SearchArgs a{};
    a.f = *p;
    return run_coupled<0>(engine, a, p, T_batch, goal_clamp, static_cast<cudaStream_t>(stream_v));
}

int nastar_b200_backward_blackbox(const nastar_fwd_params* p, const float* histories, const float* grad_histories,
                                  int64_t grad_stride, float lambda, float* grad_cost, int32_t* T_batch,
                                  int32_t* goal_clamp, void* stream_v) {
    if (!p || !p->cost || !p->start || !p->goal || !p->obst || !histories || !grad_histories || !grad_cost)
        return NASTAR_EINVAL;
    if (p->B <= 0 || p->H <= 0 || p->W <= 0 || p->T < 1) return NASTAR_EINVAL;
    if (!std::isfinite(lambda) || !(lambda > 0.f)) return NASTAR_EINVAL;
    if (p->cost_kind != NASTAR_COST_PLANE || (p->flags & ~NASTAR_FWD_NEWS) != 0 || p->trace) return NASTAR_EINVAL;
    if ((T_batch == nullptr) != (goal_clamp == nullptr)) return NASTAR_EINVAL;
    const bool coupled = (T_batch != nullptr);
    const int engine = nastar_b200_engine_for(p->H, p->W);
    if (engine == 0) return NASTAR_EUNSUPPORTED;
    const size_t need = coupled ? nastar_b200_forward_coupled_workspace_bytes(p->B, p->H, p->W, p->T)
                                : (engine == 3 ? size_t(generic_slots(p->B)) * nastar::GenericLayout(p->H, p->W).slot_bytes()
                                               : 0);
    if (need && (!p->workspace || p->workspace_bytes < need)) return NASTAR_EWORKSPACE;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
    nastar::SearchArgs a{};
    a.f = *p;
    // the search's own outputs are never written: its closed set goes straight into dL/dw
    a.f.histories = nullptr;
    a.f.paths = nullptr;
    a.f.t_solve = a.f.n_steps = a.f.n_closed = a.f.path_len = nullptr;
    a.grad_hist = grad_histories;
    a.grad_stride = grad_stride;
    a.grad_cost = grad_cost;
    a.bb_lambda = lambda;
    a.bb_hist = histories;
    if (coupled) return run_coupled<nastar::kExitBlackbox>(engine, a, p, T_batch, goal_clamp, stream);
    const cudaError_t e = launch_search<nastar::kExitEarly | nastar::kExitBlackbox, false>(engine, a, stream);
    return e == cudaSuccess ? launched() : cuda_fail(e);
}

int nastar_b200_backward(const nastar_bwd_params* p, void* stream_v) {
    return nastar_b200_backward_mech(p, NASTAR_MECH_MOORE, stream_v);
}

int nastar_b200_backward_mech(const nastar_bwd_params* p, int32_t mechanism, void* stream_v) {
    if (!p || !p->cost || !p->start || !p->goal || !p->obst || !p->grad_histories || !p->grad_cost || !p->T_batch ||
        !p->t_solve)
        return NASTAR_EINVAL;
    if (p->B <= 0 || p->H <= 0 || p->W <= 0) return NASTAR_EINVAL;
    if (mechanism != NASTAR_MECH_MOORE && mechanism != NASTAR_MECH_NEWS) return NASTAR_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
    const int engine = nastar_b200_engine_for(p->H, p->W);
    if (engine == 0) return NASTAR_EUNSUPPORTED;
    if (engine == 2 || engine == 3) {
        const nastar::GenericLayout L(p->H, p->W);
        const size_t need = size_t(generic_slots(p->B)) * L.slot_total(engine == 3, true);
        if (!p->workspace || p->workspace_bytes < need) return NASTAR_EWORKSPACE;
    }
    const cudaError_t e =
        launch_search<nastar::kExitEarly, true>(engine, bwd_kernel_args(p, mechanism == NASTAR_MECH_NEWS), stream);
    if (e != cudaSuccess) return cuda_fail(e);
    return launched();
}

int nastar_b200_batch_steps(const int32_t* t_solve, const int32_t* n_steps, int32_t B, int32_t T, int32_t* T_batch,
                            void* stream_v) {
    if (!t_solve || !T_batch || B <= 0 || T < 1) return NASTAR_EINVAL;
    batch_steps_kernel<<<1, 256, 0, static_cast<cudaStream_t>(stream_v)>>>(t_solve, n_steps, B, T, T_batch);
    return launched();
}

int nastar_b200_pack_inputs(const float* map_designs, int32_t C, int32_t Hm, int32_t Wm, const float* start,
                            int64_t start_stride, const float* goal, int64_t goal_stride, int32_t B, int32_t H,
                            int32_t W, float* out, void* stream_v) {
    if (!map_designs || !start || !goal || !out || C <= 0 || Hm <= 0 || Wm <= 0 || B <= 0 || H <= 0 || W <= 0)
        return NASTAR_EINVAL;
    if ((C == 1 && (reinterpret_cast<uintptr_t>(out) & 7)) || (C == 3 && (reinterpret_cast<uintptr_t>(out) & 15)))
        return NASTAR_EINVAL;
    const int64_t npix = int64_t(B) * Hm * Wm;
    nastar::pack_inputs_kernel<<<capped_grid((npix + 255) / 256, 16), 256, 0, static_cast<cudaStream_t>(stream_v)>>>(
        map_designs, C, Hm, Wm, start, start_stride, goal, goal_stride, B, H, W, out);
    return launched();
}

int nastar_b200_cost_from_taps(const float* taps, int32_t B, int32_t H, int32_t W, float bias, float scale,
                               float* cost, void* stream_v) {
    if (!taps || !cost || B <= 0 || H <= 0 || W <= 0) return NASTAR_EINVAL;
    const int64_t total = int64_t(B) * H * W;
    nastar::cost_from_taps_kernel<<<capped_grid((total + 255) / 256, 16), 256, 0, static_cast<cudaStream_t>(stream_v)>>>(
        taps, B, H, W, bias, scale, cost);
    return launched();
}

int nastar_b200_conv1_marks(const float* map_designs, const float* start, int64_t start_stride, const float* goal,
                            int64_t goal_stride, int32_t B, int32_t H, int32_t W, const float* w_host,
                            const float* bias_host, float* out, void* stream_v) {
    if (!map_designs || !start || !goal || !w_host || !bias_host || !out || B <= 0 || H <= 0 || W <= 0) return NASTAR_EINVAL;
    if (reinterpret_cast<uintptr_t>(out) & 15) return NASTAR_EINVAL;
    const int64_t n_pix = int64_t(B) * H * W;
    if (n_pix > (int64_t(1) << 30)) return NASTAR_EINVAL;
    nastar::Conv1Weights cw;
    std::memcpy(cw.w, w_host, sizeof(cw.w));
    std::memcpy(cw.b, bias_host, sizeof(cw.b));
    const int64_t want = (n_pix + 32 * nastar::kConv1Warps - 1) / (32 * nastar::kConv1Warps);
    nastar::conv1_marks_kernel<<<capped_grid(want, 8), 32 * nastar::kConv1Warps, 0, static_cast<cudaStream_t>(stream_v)>>>(
        map_designs, start, start_stride, goal, goal_stride, int(n_pix), H, W, cw, out);
    return launched();
}

int nastar_b200_head_taps(const float* x, int64_t P, int32_t C, const float* w_host, float* taps, void* stream_v) {
    if (!x || !w_host || !taps || P <= 0 || (reinterpret_cast<uintptr_t>(x) & 15)) return NASTAR_EINVAL;
    if (P > (int64_t(1) << 31) * 127) return NASTAR_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
    switch (C) {
        case 16: launch_head<16>(x, P, w_host, taps, stream); break;
        case 32: launch_head<32>(x, P, w_host, taps, stream); break;
        case 64: launch_head<64>(x, P, w_host, taps, stream); break;
        case 128: launch_head<128>(x, P, w_host, taps, stream); break;
        case 256: launch_head<256>(x, P, w_host, taps, stream); break;
        default: return NASTAR_EUNSUPPORTED;
    }
    return launched();
}

int nastar_b200_upsample_concat(const float* dec, int32_t B, int32_t h, int32_t w, int32_t Cd, const float* skip,
                                int32_t Cs, float* out, void* stream_v) {
    if (!dec || !out || (Cs > 0 && !skip) || B <= 0 || h <= 0 || w <= 0 || Cd <= 0 || Cs < 0) return NASTAR_EINVAL;
    if ((Cd & 3) || (Cs & 3)) return NASTAR_EINVAL;
    if ((reinterpret_cast<uintptr_t>(dec) | reinterpret_cast<uintptr_t>(skip) | reinterpret_cast<uintptr_t>(out)) & 15)
        return NASTAR_EINVAL;
    if (int64_t(B) * 2 * h > INT32_MAX || int64_t(2) * w > INT32_MAX) return NASTAR_EINVAL;
    const int64_t total = int64_t(B) * h * w * (Cd / 4) + int64_t(B) * 4 * h * w * (Cs / 4);
    nastar::upsample_concat_kernel<<<capped_grid((total + 255) / 256, 16), 256, 0, static_cast<cudaStream_t>(stream_v)>>>(
        reinterpret_cast<const float4*>(dec), B, h, w, Cd / 4, reinterpret_cast<const float4*>(skip), Cs / 4,
        reinterpret_cast<float4*>(out));
    return launched();
}

int nastar_b200_conv3x3_head_taps(const float* x, int32_t B, int32_t H, int32_t W, int32_t C_in, int32_t C_out,
                                  const float* w, const float* bias, const float* head_w_host, float* taps,
                                  void* stream_v) {
    if (!x || !w || !bias || !head_w_host || !taps || B <= 0 || H <= 0 || W <= 0 || C_in <= 0 || C_out <= 0)
        return NASTAR_EINVAL;
    if ((reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(w) & 15)) return NASTAR_EINVAL;
    if (C_in != nastar::kCHCin || C_out != nastar::kCHCout) return NASTAR_EUNSUPPORTED;
    if (H > nastar::kCHMaxSide || W > nastar::kCHMaxSide) return NASTAR_EUNSUPPORTED;
    if (int64_t(B) * H * W > (int64_t(1) << 30)) return NASTAR_EINVAL;
    // the launcher sets up tensor maps and the cluster grid first; any error, the launch's included, comes back here
    cudaError_t e = nastar::conv3x3_head_launch(x, B, H, W, w, bias, head_w_host, taps, static_cast<cudaStream_t>(stream_v));
    if (e != cudaSuccess) return cuda_fail(e);
    return launched();
}

int nastar_b200_selftest_sqrt(int32_t n, int32_t* mismatches, void* stream_v) {
    if (n <= 0 || !mismatches) return NASTAR_EINVAL;
    nastar::sqrt_rn_int_check_kernel<<<num_sms() * 4, 256, 0, static_cast<cudaStream_t>(stream_v)>>>(n, mismatches);
    return launched();
}

int nastar_b200_opt_labels_mech(const float* maps, int64_t map_stride, const int32_t* goal_idx, int32_t B, int32_t H,
                                int32_t W, int32_t mechanism, float* dists, uint8_t* act_mask, int8_t* action,
                                void* stream_v) {
    if (!maps || !goal_idx || !dists || !act_mask || !action || B <= 0 || H <= 0 || W <= 0) return NASTAR_EINVAL;
    if (map_stride < int64_t(H) * W) return NASTAR_EINVAL;
    if (mechanism != NASTAR_MECH_MOORE && mechanism != NASTAR_MECH_NEWS) return NASTAR_EINVAL;
    if (H > nastar::kLabelsMaxSide || W > nastar::kLabelsMaxSide) return NASTAR_EUNSUPPORTED;
    const nastar::LabelsArgs a{maps, map_stride, goal_idx, B, H, W, dists, act_mask, action};
    auto* const kernel = mechanism == NASTAR_MECH_NEWS ? nastar::opt_labels_kernel<nastar::kMechNews>
                                                       : nastar::opt_labels_kernel<nastar::kMechMoore>;
    const cudaError_t e = launch_smem(kernel, B, nastar::labels_threads(H, W), nastar::labels_smem_bytes(H, W),
                                      static_cast<cudaStream_t>(stream_v), a);
    if (e != cudaSuccess) return cuda_fail(e);
    return launched();
}

int nastar_b200_opt_labels(const float* maps, int64_t map_stride, const int32_t* goal_idx, int32_t B, int32_t H,
                           int32_t W, float* dists, uint8_t* act_mask, int8_t* action, void* stream_v) {
    return nastar_b200_opt_labels_mech(maps, map_stride, goal_idx, B, H, W, NASTAR_MECH_MOORE, dists, act_mask, action,
                                       stream_v);
}

int nastar_b200_weighted_labels_mech(const float* cost, int64_t cost_stride, const float* passable,
                                     int64_t passable_stride, const int32_t* goal_idx, const int32_t* start_idx,
                                     int32_t B, int32_t H, int32_t W, int32_t mechanism, float* dists, int32_t* hops,
                                     uint8_t* act_mask, int8_t* action, float* path_maps, float* path_costs,
                                     int32_t* status, void* stream_v) {
    if (!cost || !goal_idx || !dists || !hops || !act_mask || !action || !status || B <= 0 || H <= 0 || W <= 0)
        return NASTAR_EINVAL;
    if (cost_stride < int64_t(H) * W || (passable && passable_stride < int64_t(H) * W)) return NASTAR_EINVAL;
    // paths need a start per map, and a start needs somewhere to put its path
    if (bool(start_idx) != bool(path_maps) || bool(start_idx) != bool(path_costs)) return NASTAR_EINVAL;
    if (mechanism != NASTAR_MECH_MOORE && mechanism != NASTAR_MECH_NEWS) return NASTAR_EINVAL;
    if (H > nastar::kWLabelsMaxSide || W > nastar::kWLabelsMaxSide || int64_t(H) * W > nastar::kWLabelsMaxCells)
        return NASTAR_EUNSUPPORTED;
    const nastar::WLabelsArgs a{cost,   cost_stride, passable,  passable_stride, goal_idx,   start_idx, B,     H, W,
                                dists,  hops,        act_mask,  action,          path_maps,  path_costs, status};
    auto* const kernel = mechanism == NASTAR_MECH_NEWS ? nastar::weighted_labels_kernel<true>
                                                       : nastar::weighted_labels_kernel<false>;
    const cudaError_t e = launch_smem(kernel, B, nastar::wlabels_threads(H, W), nastar::wlabels_smem_bytes(H, W),
                                      static_cast<cudaStream_t>(stream_v), a);
    if (e != cudaSuccess) return cuda_fail(e);
    return launched();
}

int nastar_b200_weighted_labels(const float* cost, int64_t cost_stride, const float* passable, int64_t passable_stride,
                                const int32_t* goal_idx, const int32_t* start_idx, int32_t B, int32_t H, int32_t W,
                                float* dists, int32_t* hops, uint8_t* act_mask, int8_t* action, float* path_maps,
                                float* path_costs, int32_t* status, void* stream_v) {
    return nastar_b200_weighted_labels_mech(cost, cost_stride, passable, passable_stride, goal_idx, start_idx, B, H, W,
                                            NASTAR_MECH_MOORE, dists, hops, act_mask, action, path_maps, path_costs,
                                            status, stream_v);
}

int nastar_b200_sampler_prepare(const float* dists, const float* policies, const float* goal_maps, int32_t B, int32_t H,
                                int32_t W, double q0, double q1, double q2, double q3, uint32_t* band_bits,
                                int32_t* band_counts, int32_t* goal_idx, uint32_t* actions, double* thresholds,
                                int32_t* status, void* stream_v) {
    if (!dists || !policies || !goal_maps || !band_bits || !band_counts || !goal_idx || !actions || !thresholds || !status)
        return NASTAR_EINVAL;
    if (B <= 0 || H <= 0 || W <= 0) return NASTAR_EINVAL;
    const double q[4] = {q0, q1, q2, q3};
    for (double v : q)
        if (!(v >= 0.0 && v <= 1.0)) return NASTAR_EINVAL;
    if (H > nastar::kSamplerMaxSide || W > nastar::kSamplerMaxSide) return NASTAR_EUNSUPPORTED;
    nastar::SamplerPrepArgs a{dists, policies, goal_maps, B, H, W, {q0, q1, q2, q3}, band_bits, band_counts, goal_idx,
                              actions, thresholds, status};
    nastar::sampler_prepare_kernel<<<B, nastar::kSamplerPrepThreads, 0, static_cast<cudaStream_t>(stream_v)>>>(a);
    return launched();
}

int nastar_b200_sampler_sample(const float* maps, const float* goal_maps, int32_t n_maps, int32_t H, int32_t W,
                               const uint32_t* band_bits, const int32_t* band_counts, const int32_t* goal_idx,
                               const uint32_t* actions, const int64_t* indices, const int32_t* draws, int32_t B,
                               int32_t S, float* out_maps, float* out_starts, float* out_goals, float* out_trajs,
                               void* stream_v) {
    if (!maps || !goal_maps || !band_bits || !band_counts || !goal_idx || !actions || !indices || !draws || !out_maps ||
        !out_starts || !out_goals || !out_trajs)
        return NASTAR_EINVAL;
    if (n_maps <= 0 || H <= 0 || W <= 0 || B <= 0 || S <= 0) return NASTAR_EINVAL;
    for (const void* p : {static_cast<const void*>(maps), static_cast<const void*>(goal_maps),
                          static_cast<const void*>(out_maps), static_cast<const void*>(out_starts),
                          static_cast<const void*>(out_goals), static_cast<const void*>(out_trajs)})
        if (reinterpret_cast<uintptr_t>(p) & 15) return NASTAR_EINVAL;   // float4 stores
    if (H > nastar::kSamplerMaxSide || W > nastar::kSamplerMaxSide) return NASTAR_EUNSUPPORTED;
    // shared memory: the walked-cell bit planes of up to 8 starts at a time, plus the action plane where it fits
    const size_t traj = size_t(nastar::sampler_band_words(H, W)) * 4, act = size_t(nastar::sampler_action_words(H, W)) * 4;
    int chunk = S < nastar::kSamplerMaxChunk ? S : nastar::kSamplerMaxChunk;
    while (chunk > 1 && chunk * traj + act > kMaxDynSmem) --chunk;
    const int stage = chunk * traj + act <= kMaxDynSmem ? 1 : 0;
    const size_t smem = chunk * traj + (stage ? act : 0);
    const nastar::SamplerArgs a{maps, goal_maps, band_bits, band_counts, goal_idx, actions, indices,
                                reinterpret_cast<const uint32_t*>(draws), n_maps, H, W, B, S, chunk, stage,
                                out_maps, out_starts, out_goals, out_trajs};
    const cudaError_t e = launch_smem(nastar::sampler_sample_kernel, B, nastar::kSamplerThreads, smem,
                                      static_cast<cudaStream_t>(stream_v), a);
    if (e != cudaSuccess) return cuda_fail(e);
    return launched();
}

int nastar_b200_sample_goals(const float* maps, int64_t map_stride, int32_t B, int32_t H, int32_t W, int32_t edge_size,
                             const int32_t* draws, int32_t* goal_idx, float* goal_maps, int32_t* status, void* stream_v) {
    if (!maps || !draws || !goal_idx || !goal_maps || !status || B <= 0 || H <= 0 || W <= 0 || edge_size < 0)
        return NASTAR_EINVAL;
    if (map_stride < int64_t(H) * W) return NASTAR_EINVAL;
    if (H > nastar::kGoalsMaxSide || W > nastar::kGoalsMaxSide) return NASTAR_EUNSUPPORTED;
    const nastar::GoalsArgs a{maps, map_stride, B, H, W, edge_size, reinterpret_cast<const uint32_t*>(draws),
                              nastar::goals_plane_in_smem(H, W) ? 1 : 0, goal_idx, goal_maps, status};
    const cudaError_t e = launch_smem(nastar::sample_goals_kernel, B, nastar::goals_threads(H, W),
                                      nastar::goals_smem_bytes(H, W), static_cast<cudaStream_t>(stream_v), a);
    if (e != cudaSuccess) return cuda_fail(e);
    return launched();
}

int nastar_b200_maps_from_images(const uint8_t* images, int64_t image_stride, int32_t B, int32_t H0, int32_t W0,
                                 int32_t H, int32_t W, float* maps, uint8_t* resized, float* thresholds,
                                 int32_t* status, void* stream_v) {
    if (!images || !maps || !thresholds || !status || B <= 0 || H0 <= 0 || W0 <= 0 || H <= 0 || W <= 0)
        return NASTAR_EINVAL;
    if (image_stride < int64_t(H0) * W0) return NASTAR_EINVAL;
    if (H > nastar::kMapsMaxSide || W > nastar::kMapsMaxSide || H0 > nastar::kMapsMaxSrcSide ||
        W0 > nastar::kMapsMaxSrcSide)
        return NASTAR_EUNSUPPORTED;
    const size_t smem = nastar::maps_smem_bytes(H0, W0, H, W);
    if (smem > kMaxDynSmem) return NASTAR_EUNSUPPORTED;
    const nastar::MapsArgs a{images, image_stride, B, H0, W0, H, W, nastar::maps_taps(W0, W), nastar::maps_taps(H0, H),
                             nastar::maps_strip_cols(H0, W), maps, resized, thresholds, status};
    const cudaError_t e = launch_smem(nastar::maps_from_images_kernel, B, nastar::kMapsThreads, smem,
                                      static_cast<cudaStream_t>(stream_v), a);
    if (e != cudaSuccess) return cuda_fail(e);
    return launched();
}

int nastar_b200_draw_policies(const uint8_t* act_mask, const int32_t* draws, int32_t B, int32_t N, float* policies,
                              void* stream_v) {
    if (!act_mask || !draws || !policies || B <= 0 || N <= 0) return NASTAR_EINVAL;
    const int64_t total = int64_t(B) * N;
    nastar::draw_policies_kernel<<<capped_grid((total + 255) / 256, 16), 256, 0, static_cast<cudaStream_t>(stream_v)>>>(
        act_mask, reinterpret_cast<const uint32_t*>(draws), B, N, policies);
    return launched();
}

size_t nastar_b200_decode_png_workspace_bytes(const nastar_png_desc* desc, int32_t B) {
    int64_t max_raw = 0;
    if (png_check(desc, B, INT64_MAX, INT64_MAX, &max_raw) != NASTAR_OK) return 0;
    return 256 + size_t(capped_grid(B, kGlobalCtasPerSm)) * png_slot_bytes(max_raw);
}

int nastar_b200_decode_png(const uint8_t* data, int64_t data_bytes, const nastar_png_desc* desc,
                           const nastar_png_desc* desc_dev, int32_t B, uint8_t* out, int64_t out_bytes,
                           int32_t* status, void* workspace, size_t workspace_bytes, void* stream_v) {
    if (!data || !desc_dev || !out || !status) return NASTAR_EINVAL;
    int64_t max_raw = 0;
    const int st = png_check(desc, B, data_bytes, out_bytes, &max_raw);
    if (st != NASTAR_OK) return st;
    const int grid = capped_grid(B, kGlobalCtasPerSm);
    const size_t slot = png_slot_bytes(max_raw);
    if (!workspace || workspace_bytes < 256 + size_t(grid) * slot) return NASTAR_EWORKSPACE;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    const cudaError_t e = cudaMemsetAsync(ws, 0, 256, stream);   // the queue counter
    if (e != cudaSuccess) return cuda_fail(e);
    const nastar::PngArgs a{data, desc_dev, B, out, status, reinterpret_cast<int32_t*>(ws), ws + 256, int64_t(slot)};
    nastar::decode_png_kernel<<<grid, nastar::kPngThreads, 0, stream>>>(a);
    return launched();
}

int64_t nastar_b200_deflate_bound(const nastar_deflate_desc* desc, int32_t M) {
    int64_t chunks = 0;
    return deflate_check(desc, M, &chunks);
}

size_t nastar_b200_deflate_workspace_bytes(const nastar_deflate_desc* desc, int32_t M) {
    int64_t chunks = 0;
    if (deflate_check(desc, M, &chunks) < 0) return 0;
    return kDeflateCtl + size_t(deflate_grid(chunks)) * size_t(nastar::kDeflateSlotBytes);
}

int nastar_b200_deflate(const nastar_deflate_desc* desc, const nastar_deflate_desc* desc_dev, int32_t M, uint8_t* out,
                        int64_t out_bytes, int64_t* out_off, int64_t* out_len, uint32_t* crc, void* workspace,
                        size_t workspace_bytes, void* stream_v) {
    if (!desc_dev || !out || !out_off || !out_len || !crc || out_bytes < 0) return NASTAR_EINVAL;
    int64_t chunks = 0;
    const int64_t bound = deflate_check(desc, M, &chunks);
    if (bound < 0) return NASTAR_EINVAL;
    // the four outputs and the inputs: no two of the ranges may overlap
    auto apart = [](const void* a, int64_t na, const void* b, int64_t nb) {
        const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
        return na <= 0 || nb <= 0 || x + uint64_t(na) <= y || y + uint64_t(nb) <= x;
    };
    const int grid = deflate_grid(chunks);
    const size_t ws_need = kDeflateCtl + size_t(grid) * size_t(nastar::kDeflateSlotBytes);
    const void* outs[5] = {out, out_off, out_len, crc, workspace};
    const int64_t lens[5] = {out_bytes, int64_t(M) * 8, int64_t(M) * 8, int64_t(M) * 4,
                             int64_t(!workspace ? 0 : workspace_bytes < ws_need ? workspace_bytes : ws_need)};
    for (int i = 0; i < 5; ++i) {
        for (int j = i + 1; j < 5; ++j)
            if (!apart(outs[i], lens[i], outs[j], lens[j])) return NASTAR_EINVAL;
        if (!apart(outs[i], lens[i], desc_dev, int64_t(M) * int64_t(sizeof(nastar_deflate_desc)))) return NASTAR_EINVAL;
        for (int32_t m = 0; m < M; ++m)
            if (!apart(outs[i], lens[i], desc[m].head, desc[m].head_len) ||
                !apart(outs[i], lens[i], desc[m].data, desc[m].data_len))
                return NASTAR_EINVAL;
    }
    if (out_bytes < bound) return NASTAR_EWORKSPACE;
    if (!workspace || workspace_bytes < ws_need) return NASTAR_EWORKSPACE;
    if (reinterpret_cast<uintptr_t>(workspace) & 255) return NASTAR_EINVAL;   // the slots' u32 words
    cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    cudaError_t e = cudaMemsetAsync(ws, 0, kDeflateCtl, stream);   // the chunk counter and the ring's tags
    if (e != cudaSuccess) return cuda_fail(e);
    const nastar::DeflateArgs a{desc_dev, M, chunks, out, out_off, out_len, crc, reinterpret_cast<int32_t*>(ws),
                                reinterpret_cast<nastar::DeflatePub*>(ws + 256), ws + kDeflateCtl};
    e = launch_smem(nastar::deflate_kernel, grid, nastar::kDeflateThreads, sizeof(nastar::DeflateSmem), stream, a);
    if (e != cudaSuccess) return cuda_fail(e);
    return launched();
}

size_t nastar_b200_pq_astar_workspace_bytes(int32_t B, int32_t H, int32_t W) {
    if (!pq_shape_ok(B, H, W)) return 0;
    if (pq_shared(H, W)) return 256;
    return 256 + size_t(pq_global_grid(B, H, W)) * round256(pq_state_bytes(H, W));
}

int nastar_b200_pq_astar(const float* cost, int64_t cost_stride, const float* start, int64_t start_stride,
                         const float* goal, int64_t goal_stride, const float* map, int64_t map_stride, int32_t B,
                         int32_t H, int32_t W, double g_ratio, float* histories, int64_t* paths, int32_t* status,
                         int32_t* expansions, void* workspace, size_t workspace_bytes, void* stream_v) {
    if (!cost || !start || !goal || !map || !histories || !paths || !status || !expansions) return NASTAR_EINVAL;
    if (B <= 0 || H <= 0 || W <= 0) return NASTAR_EINVAL;
    const int64_t N = int64_t(H) * W;
    if (cost_stride < N || start_stride < N || goal_stride < N || map_stride < N) return NASTAR_EINVAL;
    if (reinterpret_cast<uintptr_t>(workspace) & 7) return NASTAR_EINVAL;   // the slots' fp64 arrays
    if (!pq_shape_ok(B, H, W)) return NASTAR_EUNSUPPORTED;
    const bool shared = pq_shared(H, W);
    const int ggrid = shared ? 0 : pq_global_grid(B, H, W);
    const size_t slot = round256(pq_state_bytes(H, W));
    if (!workspace || workspace_bytes < 256 + size_t(ggrid) * slot) return NASTAR_EWORKSPACE;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    cudaError_t e = cudaMemsetAsync(ws, 0, 256, stream);   // the work counter
    if (e != cudaSuccess) return cuda_fail(e);
    const nastar::PqArgs a{cost, cost_stride, start, start_stride, goal, goal_stride, map, map_stride, B, H, W, g_ratio,
                           1.0 - g_ratio, histories, paths, status, expansions, reinterpret_cast<int32_t*>(ws), ws + 256,
                           int64_t(slot)};
    if (shared) {
        const size_t smem = pq_state_bytes(H, W);
        e = cudaFuncSetAttribute(nastar::pq_astar_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
        int per_sm = 0;
        if (e == cudaSuccess)
            e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, nastar::pq_astar_kernel<true>, nastar::kPqThreads,
                                                              smem);
        if (e != cudaSuccess) return cuda_fail(e);
        nastar::pq_astar_kernel<true><<<capped_grid(B, per_sm > 0 ? per_sm : 1), nastar::kPqThreads, smem, stream>>>(a);
    } else {
        nastar::pq_astar_kernel<false><<<ggrid, nastar::kPqThreads, 0, stream>>>(a);
    }
    return launched();
}

int64_t nastar_b200_gif_tables_bytes(const nastar_gif_params* p) {
    if (!p) return -1;
    nastar_gif_params q = *p;   // the tables themselves need not exist yet
    q.tables = &q;
    GifShape s;
    if (!gif_shape(&q, &s)) return -1;
    return 4 * (int64_t(p->screen_w) + p->screen_h + 2 * s.Wi + 2 * s.Hi) + 258 * s.G;
}

size_t nastar_b200_gif_workspace_bytes(const nastar_gif_params* p) {
    GifShape s;
    if (!gif_shape(p, &s) || !gif_supported(p)) return 0;
    return s.ws_bytes;
}

int64_t nastar_b200_gif_record_bytes(int64_t n) { return n < 1 ? -1 : 19 + n + (n + 254) / 255 + 1; }

int nastar_b200_gif_plan(const nastar_gif_params* p, int32_t* steps, int32_t* nbytes, void* workspace,
                         size_t workspace_bytes, void* stream_v) {
    GifShape s;
    if (!gif_shape(p, &s) || !steps || !nbytes) return NASTAR_EINVAL;
    if (!gif_supported(p)) return NASTAR_EUNSUPPORTED;
    if (!workspace || workspace_bytes < s.ws_bytes) return NASTAR_EWORKSPACE;
    if (reinterpret_cast<uintptr_t>(workspace) & 255) return NASTAR_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
    nastar::GifArgs a = gif_args(p, s, workspace, nbytes);
    cudaError_t e = cudaMemsetAsync(workspace, 0, 256, stream);   // counters
    if (e == cudaSuccess) e = cudaMemsetAsync(a.rect, 0xFF, s.ws_rect, stream);   // empty rectangles
    if (e != cudaSuccess) return cuda_fail(e);
    const int grid = gif_grid(p->B > 1024 ? p->B : 1024);
    e = launch_smem(nastar::gif_plan_kernel, grid, nastar::kGifThreads, sizeof(nastar::GifWarpSmem) * nastar::kGifWarps,
                    stream, a);
    if (e != cudaSuccess) return cuda_fail(e);
    const int st = launched();
    if (st != NASTAR_OK) return st;
    e = cudaMemcpyAsync(steps, a.steps, size_t(s.G) * 4, cudaMemcpyDeviceToDevice, stream);   // T_g, for the host
    return e == cudaSuccess ? NASTAR_OK : cuda_fail(e);
}

int nastar_b200_gif_encode(const nastar_gif_params* p, const int32_t* nbytes, const int32_t* nbytes_host,
                           const int64_t* offset_host, const int64_t* offset_dev, int64_t n_frames, uint8_t* out,
                           int64_t out_bytes, void* workspace, size_t workspace_bytes, void* stream_v) {
    GifShape s;
    if (!gif_shape(p, &s) || !nbytes || !nbytes_host || !offset_host || !offset_dev || !out) return NASTAR_EINVAL;
    if (n_frames < 1 || n_frames > s.G * (int64_t(p->T) + 1)) return NASTAR_EINVAL;
    if (offset_host[0] != 0) return NASTAR_EINVAL;
    for (int64_t f = 0; f < n_frames; ++f) {
        const int64_t r = nastar_b200_gif_record_bytes(nbytes_host[f]);
        if (r < 0 || offset_host[f + 1] != offset_host[f] + r) return NASTAR_EINVAL;
    }
    if (out_bytes < offset_host[n_frames]) return NASTAR_EINVAL;
    if (!gif_supported(p)) return NASTAR_EUNSUPPORTED;
    if (!workspace || workspace_bytes < s.ws_bytes) return NASTAR_EWORKSPACE;
    if (reinterpret_cast<uintptr_t>(workspace) & 255) return NASTAR_EINVAL;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
    nastar::GifArgs a = gif_args(p, s, workspace, const_cast<int32_t*>(nbytes));
    a.offset = offset_dev;
    a.out = out;
    // the encode's frame counter starts over, so the same plan can be encoded again
    cudaError_t e = cudaMemsetAsync(&a.ctl->encode_next, 0, sizeof(int32_t), stream);
    if (e != cudaSuccess) return cuda_fail(e);
    e = launch_smem(nastar::gif_encode_kernel, gif_grid(n_frames), nastar::kGifThreads,
                                      sizeof(nastar::GifWarpSmem) * nastar::kGifWarps, stream, a);
    if (e != cudaSuccess) return cuda_fail(e);
    return launched();
}

int64_t nastar_b200_png_gap(int32_t i) { return nastar::png_gap(i); }

int64_t nastar_b200_png_encode_bound(const nastar_png_enc_desc* desc, int32_t B) {
    int64_t bound = 0;
    return png_enc_check(desc, B, -1, &bound) == NASTAR_OK ? bound : -1;
}

int nastar_b200_png_filter(const nastar_png_enc_desc* desc, const nastar_png_enc_desc* desc_dev, int32_t B,
                           uint8_t* filt, int64_t filt_bytes, uint32_t* adler, void* stream_v) {
    if (!desc_dev || !filt || !adler || filt_bytes < 0) return NASTAR_EINVAL;
    int64_t bound = 0;
    const int st = png_enc_check(desc, B, filt_bytes, &bound);
    if (st != NASTAR_OK) return st;
    const nastar::PngFilterArgs a{desc_dev, filt, adler};
    const cudaError_t e = launch_smem(nastar::png_filter_kernel, B, nastar::kPngEncThreads, 0,
                                      static_cast<cudaStream_t>(stream_v), a);
    if (e != cudaSuccess) return cuda_fail(e);
    return launched();
}

int nastar_b200_png_finish(const nastar_png_enc_desc* desc, const nastar_png_enc_desc* desc_dev, int32_t B,
                           const int64_t* out_off, const int64_t* out_len, const uint32_t* adler, uint8_t* out,
                           int64_t out_bytes, void* stream_v) {
    if (!desc_dev || !out_off || !out_len || !adler || !out) return NASTAR_EINVAL;
    int64_t bound = 0;
    const int st = png_enc_check(desc, B, -1, &bound);
    if (st != NASTAR_OK) return st;
    if (out_bytes < bound) return NASTAR_EWORKSPACE;
    const nastar::PngFinishArgs a{desc_dev, out_off, out_len, adler, out, out_bytes};
    const cudaError_t e = launch_smem(nastar::png_finish_kernel, B, nastar::kPngEncThreads, 0,
                                      static_cast<cudaStream_t>(stream_v), a);
    if (e != cudaSuccess) return cuda_fail(e);
    return launched();
}

int nastar_b200_crop_resize_rgb(const nastar_rgb_image* src, const nastar_rgb_image* src_dev, int32_t S,
                                const nastar_rgb_crop* crops, const nastar_rgb_crop* crops_dev, int32_t N, int32_t Ho,
                                int32_t Wo, uint8_t* out, void* stream_v) {
    if (!src || !src_dev || !crops || !crops_dev || !out || S <= 0 || N <= 0 || Ho <= 0 || Wo <= 0)
        return NASTAR_EINVAL;
    // an invalid descriptor takes precedence over an unsupported one found earlier
    int st = Ho > nastar::kCropMaxOut || Wo > nastar::kCropMaxOut ? NASTAR_EUNSUPPORTED : NASTAR_OK;
    for (int32_t i = 0; i < S; ++i) {
        const nastar_rgb_image& m = src[i];
        if (!m.pixels || m.W <= 0 || m.H <= 0 || m.pitch < int64_t(m.W) * 3) return NASTAR_EINVAL;
        if (m.W > nastar::kCropMaxSide || m.H > nastar::kCropMaxSide) st = NASTAR_EUNSUPPORTED;
    }
    std::vector<uint8_t> seen(size_t(N), 0);
    size_t smem = nastar::kCropSmemTarget;
    for (int32_t i = 0; i < N; ++i) {
        const nastar_rgb_crop& c = crops[i];
        const int64_t cw = int64_t(c.x1) - c.x0, ch = int64_t(c.y1) - c.y0;
        if (c.src < 0 || c.src >= S || c.out < 0 || c.out >= N || seen[c.out] || cw <= 0 || ch <= 0)
            return NASTAR_EINVAL;
        seen[c.out] = 1;
        if (cw > nastar::kCropMaxSide || ch > nastar::kCropMaxSide) st = NASTAR_EUNSUPPORTED;
        if (st != NASTAR_OK) continue;
        const size_t need = nastar::crop_smem_need(int(cw), int(ch), Ho, Wo);
        smem = need > smem ? need : smem;
    }
    if (st != NASTAR_OK) return st;
    if (smem > kMaxDynSmem) return NASTAR_EUNSUPPORTED;
    const nastar::CropArgs a{src_dev, crops_dev, Ho, Wo, int64_t(smem), out};
    const cudaError_t e = launch_smem(nastar::crop_resize_rgb_kernel, N, nastar::kCropThreads, smem,
                                      static_cast<cudaStream_t>(stream_v), a);
    if (e != cudaSuccess) return cuda_fail(e);
    return launched();
}

int nastar_b200_inflate(const uint8_t* data, int64_t data_bytes, const nastar_inflate_desc* desc,
                        const nastar_inflate_desc* desc_dev, int32_t M, uint8_t* out, int64_t out_bytes,
                        int32_t* status, uint32_t* crc, void* workspace, size_t workspace_bytes, void* stream_v) {
    if (!data || !desc_dev || !out || !status || !crc) return NASTAR_EINVAL;
    const int st = inflate_check(desc, M, data_bytes, out_bytes);
    if (st != NASTAR_OK) return st;
    if (!workspace || workspace_bytes < NASTAR_INFLATE_WORKSPACE_BYTES) return NASTAR_EWORKSPACE;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
    int32_t* queue = static_cast<int32_t*>(workspace);
    const cudaError_t e = cudaMemsetAsync(queue, 0, sizeof(int32_t), stream);
    if (e != cudaSuccess) return cuda_fail(e);
    const nastar::InflateArgs a{data, desc_dev, M, out, status, crc, queue};
    nastar::inflate_kernel<<<capped_grid(M, 16), nastar::kInflateThreads, 0, stream>>>(a);
    return launched();
}

size_t nastar_b200_chamfer_workspace_bytes(int32_t B, int32_t H, int32_t W) {
    if (B <= 0 || H <= 0 || W <= 0 || H > nastar::kChamferMaxSide || W > nastar::kChamferMaxSide) return 0;
    return chamfer_global(H, W) ? size_t(chamfer_grid(B, H, W)) * chamfer_slot_bytes(H, W) : 0;
}

int nastar_b200_chamfer(const uint8_t* masks, int32_t B, int32_t H, int32_t W, double* out, void* workspace,
                        size_t workspace_bytes, void* stream_v) {
    if (!masks || !out || B <= 0 || H <= 0 || W <= 0) return NASTAR_EINVAL;
    if (H > nastar::kChamferMaxSide || W > nastar::kChamferMaxSide) return NASTAR_EUNSUPPORTED;
    const size_t need = nastar_b200_chamfer_workspace_bytes(B, H, W);
    if (need && (!workspace || workspace_bytes < need)) return NASTAR_EWORKSPACE;
    const bool global = chamfer_global(H, W);
    const nastar::ChamferArgs a{masks, B, H, W, out, global ? static_cast<unsigned char*>(workspace) : nullptr,
                                int64_t(chamfer_slot_bytes(H, W))};
    const size_t smem = global ? 0 : size_t(nastar::chamfer_layout(H, W).bytes);
    const cudaError_t e = launch_smem(nastar::chamfer_kernel, chamfer_grid(B, H, W), nastar::kChamferThreads, smem,
                                      static_cast<cudaStream_t>(stream_v), a);
    if (e != cudaSuccess) return cuda_fail(e);
    return launched();
}

uint64_t nastar_b200_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

const char* nastar_b200_status_string(int s) {
    switch (s) {
        case NASTAR_OK: return "ok";
        case NASTAR_EINVAL: return "invalid argument";
        case NASTAR_EUNSUPPORTED: return "unsupported map shape or feature";
        case NASTAR_ECUDA: return "CUDA runtime error";
        case NASTAR_EWORKSPACE: return "workspace too small";
        default: return "unknown status";
    }
}

const char* nastar_b200_last_cuda_error(void) { return cudaGetErrorString(g_last_err); }

}  // extern "C"
