// nastar_convhead.cuh — the encoder's widest 3x3 convolution (128 -> 256 channels, pad 1, stride 1, + folded bias +
// ReLU) fused with the single-output-channel head's per-pixel products, on sm_90a tensor cores.
//
//   taps[p][k] = sum_c relu(bias[c] + sum_{ky,kx,ci} x[p + (ky-1, kx-1)][ci] * w[c][ky][kx][ci]) * hw[c][k]
//
// i.e. cuDNN's TF32 conv4 followed by head_taps_kernel (nastar_glue.cuh) in one launch: the [P][256] fp32 activation
// (105 MB at the flagship batch of 100 maps of 32x32) never leaves the SM.  The output is the [B][H][W][9] layout the
// search's NASTAR_COST_TAPS prologue reads.
//
// GEMM view: M = pixels, N = 256 output channels, K = 9 taps x 128 input channels, both operands K-major (the input
// is channels-last, the folded weights are OIHW in channels-last memory = [cout][ky][kx][cin]), which is what TF32
// wgmma requires.  Operands are TF32: the tensor cores read the top 19 bits of each fp32 operand, i.e. truncate the
// mantissa to 10 bits (observed on an H100 SXM for both operands, tests/test_gpu_encoder_exact.py); products are
// accumulated in fp32: the precision class of cuDNN's TF32 path it replaces.  The epilogue (bias, ReLU, the 9 head
// products and the cross-lane sums) is plain fp32 FFMA in a fixed order, so the same inputs give the same bits
// wherever a map lands in the batch and whatever tile width it gets; there are no atomics.
//
// Tiles: a CTA computes 128 pixels x 256 channels = R image rows of Wp pixels, Wp = W rounded up to 8/16/32/64 and
// R = 128 / Wp (4 rows at W = 32).  Columns x >= W and rows y >= H are computed on zeros and not stored.
//   * A operand: one 4-D TMA box {32 channels, Wp, R + 2 rows, 1 map} per (kx, 32-channel chunk), 128-B swizzled,
//     loaded at x offset kx - 1 and row y0 - 1; TMA's out-of-bounds zero fill is the convolution's padding.  The
//     three ky taps are the same box at offsets of ky * Wp * 128 B (a multiple of the 1 KB swizzle atom), so each
//     input byte is loaded 3 times per tile, not 9.
//   * B operand: the 256 x 32 weight slice of one (ky, kx, chunk), 32 KB, also 128-B swizzled.
//   * Warp roles: warpgroup 0 is the producer (one thread issues every TMA; setmaxnreg drops the group to 48
//     registers), warpgroups 1 and 2 each own 64 pixels x 256 channels (128 fp32 accumulators per thread, two
//     m64n128k8 per k step, one per half of the output channels; setmaxnreg raises them to 192).  Rings: 2 A stages,
//     4 B stages, full/empty mbarriers.
//
// Three properties of the flagship shape (B = 100, 32x32: M = 102 400, N = 256, K = 1 152, 800 tiles):
//   * Weight traffic.  The 1.18 MB of weights stay in L2, but every tile streams all of them: 800 x 1.18 MB =
//     0.94 GB per call from L2, about 6 TB/s at 150 us, more than L2 delivers next to the A traffic.  CTAs run in
//     clusters of 2 along M; each loads half of every weight slice (128 output channels) and TMA multicast writes it
//     into both CTAs' shared memory, so L2 serves 0.47 GB.  A stage's empty barrier therefore counts the consumer
//     warps of both CTAs.  A traffic: 12 boxes of 24 KB per tile = 0.23 GB, mostly L2 hits.
//   * Tail.  The grid is persistent: as many clusters as can be co-resident (66 on 132 SMs), each taking tile pairs
//     round-robin.  800 tiles are 6 full rounds of 132 plus 8 tiles.  Instead of a 7th round for those 8, each of
//     them is split between the two CTAs of one cluster as two 64-pixel half tiles (one consumer warpgroup active
//     each), so the last round costs about half a tile: 6.06 / 6.5 = 0.93 of ideal, against 6.06 / 7 = 0.87.
//   * Co-residency with the search.  The step graph runs the search (astar_warp32_kernel<..., kFused=1>: one
//     32-thread CTA per map, 72 registers, 17 840 B static shared memory) beside this kernel.  Registers are
//     budgeted per SM sub-partition, not per SM: each warp is allocated in one of the four 16 384-register files, and
//     the 12 warps of a CTA put 3 in each.  At 144 registers that is 3 x 144 x 32 = 13 824, leaving 2 560 for a
//     search warp of up to 80 registers; at 160 (61 440 of the SM's 65 536, which looks like room) it is 15 360,
//     leaving 1 024, and a CTA of this kernel cannot start on an SM that still runs a search CTA (on an H100 the
//     pair then costs conv + search instead of about the longer of the two, tools/residency_probe.py).  ptxas needs
//     154 launch registers for an m64n256k8 with fp32 accumulators whatever setmaxnreg grants later, hence the two
//     m64n128k8: each output element is still one k8 step at a time in the same order.  setmaxnreg only moves
//     registers inside the CTA's launch allocation (128 x 48 + 256 x 192 = 55 296 = 384 x 144); 0 spills under
//     -Xptxas -v.  Shared memory: 128 KB (B) + 2 x 24 KB (A at W = 32; 2 x 32 KB at W = 64) + 10.3 KB (bias, head)
//     + barriers = 187 KB at W = 32 and 203 KB at W = 64, which leaves room for the search CTA's 17.4 KB (+1 KB
//     reserved per CTA) in the 228 KB of an SM.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>

#include <atomic>
#include <cstdint>

#include "nastar_common.cuh"

namespace nastar {

constexpr int kCHCin = 128;
constexpr int kCHCout = 256;
constexpr int kCHThreads = 384;            // producer warpgroup + 2 consumer warpgroups
constexpr int kCHTileM = 128;              // pixels per tile (64 per consumer warpgroup)
constexpr int kCHCluster = 2;              // CTAs sharing (multicasting) the weight slices
constexpr int kCHAStages = 2;
constexpr int kCHBStages = 4;
constexpr int kCHChunk = 32;               // input channels per 128-B swizzle row
constexpr int kCHChunks = kCHCin / kCHChunk;
constexpr uint32_t kCHBStageBytes = kCHCout * kCHChunk * 4;          // 32 KB
constexpr uint32_t kCHBSliceRows = kCHCout / kCHCluster;             // output channels each CTA loads
constexpr uint32_t kCHBSliceBytes = kCHBStageBytes / kCHCluster;
constexpr uint32_t kCHBHalfBytes = kCHBStageBytes / 2;           // output channels 128..255 of a stage
constexpr int kCHLaunchRegs = 144;         // __maxnreg__ of the launch: see the co-residency budget above
constexpr int kCHProducerRegs = 48;
constexpr int kCHConsumerRegs = 192;
constexpr int kCHMaxSide = 64;
constexpr int kCHSearchRegs = 80;          // the largest search warp that must fit beside a CTA on every sub-partition
static_assert(kCHCluster == 2, "the tail split gives each CTA of a cluster one half tile");
static_assert(128 * kCHProducerRegs + 256 * kCHConsumerRegs <= kCHThreads * kCHLaunchRegs,
              "setmaxnreg exceeds the launch budget");
// a warp's registers come from one SM sub-partition's 16 384-register file, and a CTA's warps are spread evenly
// over the 4 sub-partitions: each must keep room for one search warp next to its share of this CTA
static_assert(kCHThreads / 32 / 4 * kCHLaunchRegs * 32 + kCHSearchRegs * 32 <= 16384,
              "no room for a search warp on an SM sub-partition");

struct ConvHeadWeights {   // the head's folded [C][9] weights, passed by value (constant bank)
    float w[kCHCout * 9];
};

struct ConvHeadArgs {
    const float* bias;     // [256] folded conv bias (device)
    float* taps;           // [B][H][W][9]
    int B, H, W;
    int Wp, R;             // tile = R rows of Wp pixels, Wp * R = 128
    int tiles_per_map;     // ceil(H / R)
    int T;                 // B * tiles_per_map
    uint32_t a_bytes;      // one A box: (R + 2) * Wp * 128 B
};

// dynamic shared memory: [B ring][A ring][bias][head weights][mbarriers], base aligned to 1 KB (128-B swizzle atom)
struct ConvHeadLayout {
    uint32_t a_bytes;
    __host__ __device__ explicit ConvHeadLayout(uint32_t a) : a_bytes(a) {}
    __host__ __device__ uint32_t a_off() const { return kCHBStages * kCHBStageBytes; }
    __host__ __device__ uint32_t bias_off() const { return a_off() + kCHAStages * a_bytes; }
    __host__ __device__ uint32_t head_off() const { return bias_off() + kCHCout * 4; }
    __host__ __device__ uint32_t bar_off() const { return head_off() + kCHCout * 9 * 4; }
    __host__ __device__ uint32_t bytes() const { return bar_off() + 2 * (kCHAStages + kCHBStages) * 8; }
    __host__ __device__ uint32_t alloc_bytes() const { return bytes() + 1024; }
};

__host__ __device__ inline int convhead_wp(int W) { return W <= 8 ? 8 : W <= 16 ? 16 : W <= 32 ? 32 : 64; }

// ---- inline PTX: cluster, TMA tensor copies, wgmma ------------------------------------------------------------
__device__ __forceinline__ uint32_t ch_cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t ch_cluster_id() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t ch_num_clusters() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void ch_cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\nbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ void ch_arrive_cluster(uint64_t* bar, uint32_t rank) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(rank));
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
__device__ __forceinline__ void ch_arrive_local(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void ch_tma_load_4d(void* dst, const CUtensorMap* map, int c0, int c1, int c2, int c3,
                                               uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3),
        "r"(smem_u32(bar))
        : "memory");
}
// 2-D box written at the same offset into every CTA of `mask`, completing bytes on each CTA's `bar`
__device__ __forceinline__ void ch_tma_load_2d_multicast(void* dst, const CUtensorMap* map, int c0, int c1,
                                                         uint64_t* bar, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster"
        " [%0], [%1, {%2, %3}], [%4], %5;"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar)), "h"(mask)
        : "memory");
}
// wgmma shared-memory descriptor: K-major, 128-B swizzle, 8-row groups 1 KB apart (leading offset unused)
__device__ __forceinline__ uint64_t ch_desc(uint32_t saddr) {
    return uint64_t((saddr & 0x3FFFF) >> 4) | (uint64_t(1) << 16) | (uint64_t(1024 >> 4) << 32) | (uint64_t(1) << 62);
}
__device__ __forceinline__ void ch_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void ch_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void ch_wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ch_fence_operand(float& x) { asm volatile("" : "+f"(x)::"memory"); }

// d[64 x 128] (+)= A[64 x 8] * B[8 x 128]^T, TF32 in, fp32 accumulate; scale_d = 0 overwrites d.  The accumulators
// are d[O .. O + 63] of the m64n256 fragment: O = 64 holds output channels 128..255 when B starts 128 rows further.
template <int O>
__device__ __forceinline__ void ch_wgmma_m64n128k8(float (&d)[128], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
    static_assert(O == 0 || O == 64, "one of the two channel halves");
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1;\n}\n"
        : "+f"(d[O + 0]), "+f"(d[O + 1]), "+f"(d[O + 2]), "+f"(d[O + 3]), "+f"(d[O + 4]), "+f"(d[O + 5]), "+f"(d[O + 6]),
          "+f"(d[O + 7]), "+f"(d[O + 8]), "+f"(d[O + 9]), "+f"(d[O + 10]), "+f"(d[O + 11]), "+f"(d[O + 12]), "+f"(d[O + 13]),
          "+f"(d[O + 14]), "+f"(d[O + 15]), "+f"(d[O + 16]), "+f"(d[O + 17]), "+f"(d[O + 18]), "+f"(d[O + 19]), "+f"(d[O + 20]),
          "+f"(d[O + 21]), "+f"(d[O + 22]), "+f"(d[O + 23]), "+f"(d[O + 24]), "+f"(d[O + 25]), "+f"(d[O + 26]), "+f"(d[O + 27]),
          "+f"(d[O + 28]), "+f"(d[O + 29]), "+f"(d[O + 30]), "+f"(d[O + 31]), "+f"(d[O + 32]), "+f"(d[O + 33]), "+f"(d[O + 34]),
          "+f"(d[O + 35]), "+f"(d[O + 36]), "+f"(d[O + 37]), "+f"(d[O + 38]), "+f"(d[O + 39]), "+f"(d[O + 40]), "+f"(d[O + 41]),
          "+f"(d[O + 42]), "+f"(d[O + 43]), "+f"(d[O + 44]), "+f"(d[O + 45]), "+f"(d[O + 46]), "+f"(d[O + 47]), "+f"(d[O + 48]),
          "+f"(d[O + 49]), "+f"(d[O + 50]), "+f"(d[O + 51]), "+f"(d[O + 52]), "+f"(d[O + 53]), "+f"(d[O + 54]), "+f"(d[O + 55]),
          "+f"(d[O + 56]), "+f"(d[O + 57]), "+f"(d[O + 58]), "+f"(d[O + 59]), "+f"(d[O + 60]), "+f"(d[O + 61]), "+f"(d[O + 62]),
          "+f"(d[O + 63])
        : "l"(desc_a), "l"(desc_b), "r"(scale_d));
}

// Which tile CTA `rank` of cluster `c` works on in round `i`; see the schedule in the header comment.
struct ConvHeadTile {
    int b, y0, rows;
    bool valid, half;
};
__device__ __forceinline__ ConvHeadTile ch_tile(const ConvHeadArgs& a, int i, int nf, bool extra_full, int c, int nC,
                                                int rank) {
    ConvHeadTile t;
    int idx;
    if (i < nf || extra_full) {
        idx = (i * nC + c) * kCHCluster + rank;
        t.half = false;
    } else {
        idx = nf * nC * kCHCluster + c;
        t.half = true;
    }
    t.valid = idx < a.T;
    if (!t.valid) idx = 0;
    t.b = idx / a.tiles_per_map;
    t.y0 = (idx - t.b * a.tiles_per_map) * a.R;
    t.rows = a.R;
    if (t.half) {
        t.rows = a.R / 2;
        t.y0 += rank * t.rows;
    }
    return t;
}

__global__ void __cluster_dims__(kCHCluster, 1, 1) __maxnreg__(kCHLaunchRegs)
conv3x3_head_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_w,
                    const __grid_constant__ ConvHeadArgs a, const __grid_constant__ ConvHeadWeights hw) {
    extern __shared__ unsigned char ch_smem_raw[];
    // offset from the __shared__ array itself (not through an integer), so the compiler keeps the shared address
    // space and the epilogue's bias and head-weight reads are LDS instead of generic loads
    unsigned char* smem = ch_smem_raw + ((1024u - (smem_u32(ch_smem_raw) & 1023u)) & 1023u);
    const ConvHeadLayout L(a.a_bytes);
    unsigned char* sB = smem;
    unsigned char* sA = smem + L.a_off();
    float* s_bias = reinterpret_cast<float*>(smem + L.bias_off());
    float* s_head = reinterpret_cast<float*>(smem + L.head_off());
    uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + L.bar_off());
    uint64_t* a_empty = a_full + kCHAStages;
    uint64_t* b_full = a_empty + kCHAStages;
    uint64_t* b_empty = b_full + kCHBStages;

    const int tid = threadIdx.x;
    const uint32_t rank = ch_cluster_rank();
    for (int i = tid; i < kCHCout; i += kCHThreads) s_bias[i] = __ldg(a.bias + i);
    for (int i = tid; i < kCHCout * 9; i += kCHThreads) s_head[i] = hw.w[i];
    if (tid == 0) {
        for (int s = 0; s < kCHAStages; ++s) {
            mbar_init(&a_full[s], 1);
            mbar_init(&a_empty[s], 2 * 4);                   // every consumer warp of this CTA
        }
        for (int s = 0; s < kCHBStages; ++s) {
            mbar_init(&b_full[s], 1);
            mbar_init(&b_empty[s], kCHCluster * 2 * 4);      // every consumer warp of both CTAs
        }
        fence_mbar_init();
    }
    ch_cluster_sync();   // barriers initialised (and bias / head staged) in both CTAs before any multicast

    const int nC = int(ch_num_clusters());
    const int c = int(ch_cluster_id());
    const int per_round = nC * kCHCluster;
    const int nf = a.T / per_round;
    const int tail = a.T - nf * per_round;
    const bool extra_full = tail > nC;                       // more than half a round left: one more full round
    const int rounds = nf + ((extra_full || c < tail) ? 1 : 0);
    const int wg = __shfl_sync(0xFFFFFFFFu, tid >> 7, 0);   // warp-uniform role

    if (wg == 0) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kCHProducerRegs));
        if (tid == 0) {
            uint32_t ai = 0, bi = 0;
            for (int i = 0; i < rounds; ++i) {
                const ConvHeadTile t = ch_tile(a, i, nf, extra_full, c, nC, int(rank));
                for (int kx = 0; kx < 3; ++kx) {
                    for (int ch = 0; ch < kCHChunks; ++ch, ++ai) {
                        const uint32_t as = ai % kCHAStages;
                        mbar_wait(&a_empty[as], ((ai / kCHAStages) & 1) ^ 1);
                        mbar_expect_tx(&a_full[as], a.a_bytes);
                        ch_tma_load_4d(sA + as * a.a_bytes, &tm_x, ch * kCHChunk, kx - 1, t.y0 - 1, t.b, &a_full[as]);
                        for (int ky = 0; ky < 3; ++ky, ++bi) {
                            const uint32_t bs = bi % kCHBStages;
                            mbar_wait(&b_empty[bs], ((bi / kCHBStages) & 1) ^ 1);
                            mbar_expect_tx(&b_full[bs], kCHBStageBytes);
                            ch_tma_load_2d_multicast(sB + bs * kCHBStageBytes + rank * kCHBSliceBytes, &tm_w,
                                                     (ky * 3 + kx) * kCHCin + ch * kCHChunk, int(rank * kCHBSliceRows),
                                                     &b_full[bs], uint16_t((1u << kCHCluster) - 1));
                        }
                    }
                }
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kCHConsumerRegs));
        const int cw = wg - 1;                  // 64-pixel half of the tile
        const int warp = (tid >> 5) & 3, lane = tid & 31;
        float d[128];
#pragma unroll
        for (int j = 0; j < 128; ++j) d[j] = 0.f;
        uint32_t ai = 0, bi = 0;
        // a consumer warp frees a B stage in both CTAs (the multicast wrote both) and an A stage in its own
        auto release = [&](uint32_t bs, int as) {
            __syncwarp();
            if (lane == 0) {
                for (uint32_t r = 0; r < kCHCluster; ++r) ch_arrive_cluster(&b_empty[bs], r);
                if (as >= 0) ch_arrive_local(&a_empty[as]);
            }
        };
        for (int i = 0; i < rounds; ++i) {
            const ConvHeadTile t = ch_tile(a, i, nf, extra_full, c, nC, int(rank));
            const bool active = __shfl_sync(0xFFFFFFFFu, int(t.valid && (!t.half || cw == 0)), 0) != 0;
            int prev_b = -1, prev_a = -1;
            for (int kx = 0; kx < 3; ++kx) {
                for (int ch = 0; ch < kCHChunks; ++ch, ++ai) {
                    const uint32_t as = ai % kCHAStages;
                    mbar_wait(&a_full[as], (ai / kCHAStages) & 1);
                    const uint32_t a_base = smem_u32(sA + as * a.a_bytes) + uint32_t(cw * 64 * 128);
                    for (int ky = 0; ky < 3; ++ky, ++bi) {
                        const uint32_t bs = bi % kCHBStages;
                        mbar_wait(&b_full[bs], (bi / kCHBStages) & 1);
                        if (active) {
                            const uint32_t ab = a_base + uint32_t(ky * a.Wp * 128);
                            const uint32_t bb = smem_u32(sB + bs * kCHBStageBytes);
                            const uint32_t first = (kx | ch | ky) == 0;
                            ch_wgmma_fence();
#pragma unroll
                            for (int kk = 0; kk < kCHChunk / 8; ++kk) {
                                const uint32_t scale = (first && kk == 0) ? 0u : 1u;
                                ch_wgmma_m64n128k8<0>(d, ch_desc(ab + kk * 32), ch_desc(bb + kk * 32), scale);
                                ch_wgmma_m64n128k8<64>(d, ch_desc(ab + kk * 32), ch_desc(bb + kCHBHalfBytes + kk * 32),
                                                       scale);
                            }
                            ch_wgmma_commit();
                            ch_wgmma_wait<1>();
                        }
                        if (prev_b >= 0) release(uint32_t(prev_b), prev_a);
                        prev_b = int(bs);
                        prev_a = (ky == 2) ? int(as) : -1;
                    }
                }
            }
            if (active) ch_wgmma_wait<0>();
#pragma unroll
            for (int j = 0; j < 128; ++j) ch_fence_operand(d[j]);
            release(uint32_t(prev_b), prev_a);
            if (!active) continue;

            // epilogue: relu(acc + bias) . head weights over this thread's 64 channels, then over the 4 lanes of a row
            const int q = lane & 3;
            float t0[9], t1[9];
#pragma unroll
            for (int k = 0; k < 9; ++k) t0[k] = t1[k] = 0.f;
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                // channels cc0 and cc0 + 1 (cc0 even): their 2 biases and 18 head weights are 8-byte aligned pairs
                const int cc0 = 8 * j + 2 * q;
                const float2 bias2 = *reinterpret_cast<const float2*>(s_bias + cc0);
                float w2[18];
#pragma unroll
                for (int i = 0; i < 9; ++i) {
                    const float2 v = reinterpret_cast<const float2*>(s_head + cc0 * 9)[i];
                    w2[2 * i] = v.x;
                    w2[2 * i + 1] = v.y;
                }
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float bc = e ? bias2.y : bias2.x;
                    const float v0 = fmaxf(d[4 * j + e] + bc, 0.f);
                    const float v1 = fmaxf(d[4 * j + 2 + e] + bc, 0.f);
                    const float* wc = w2 + 9 * e;
#pragma unroll
                    for (int k = 0; k < 9; ++k) {
                        const float wk = wc[k];
                        t0[k] = fmaf(v0, wk, t0[k]);
                        t1[k] = fmaf(v1, wk, t1[k]);
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < 9; ++k) {
                t0[k] += __shfl_xor_sync(0xFFFFFFFFu, t0[k], 1);
                t1[k] += __shfl_xor_sync(0xFFFFFFFFu, t1[k], 1);
                t0[k] += __shfl_xor_sync(0xFFFFFFFFu, t0[k], 2);
                t1[k] += __shfl_xor_sync(0xFFFFFFFFu, t1[k], 2);
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = cw * 64 + warp * 16 + (lane >> 2) + 8 * h;
                const int ry = m / a.Wp, x = m - ry * a.Wp, y = t.y0 + ry;
                if (ry < t.rows && y < a.H && x < a.W) {
                    float* o = a.taps + ((size_t(t.b) * a.H + y) * a.W + x) * 9;
#pragma unroll
                    for (int k = 0; k < 9; ++k)       // lane q stores taps q, q + 4 (and 8)
                        if ((k & 3) == q) o[k] = h ? t1[k] : t0[k];
                }
            }
        }
    }
    ch_cluster_sync();   // the partner may still arrive on this CTA's barriers until it is done
}

// ---- host side ---------------------------------------------------------------------------------------------
inline PFN_cuTensorMapEncodeTiled_v12000 ch_encode_fn() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &p, 12000, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
    }
    return fn;
}

// co-resident clusters for one tile width (cached per device and width)
inline cudaError_t ch_max_clusters(int Wp, size_t smem, int* out) {
    static std::atomic<int> cache[64][4];
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    const int wi = Wp == 8 ? 0 : Wp == 16 ? 1 : Wp == 32 ? 2 : 3;
    int v = cache[dev & 63][wi].load(std::memory_order_relaxed);
    if (v <= 0) {
        e = cudaFuncSetAttribute(conv3x3_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
        if (e != cudaSuccess) return e;
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(kCHCluster, 1, 1);
        cfg.blockDim = dim3(kCHThreads, 1, 1);
        cfg.dynamicSmemBytes = smem;
        e = cudaOccupancyMaxActiveClusters(&v, conv3x3_head_kernel, &cfg);
        if (e != cudaSuccess) return e;
        if (v <= 0) return cudaErrorInvalidConfiguration;
        cache[dev & 63][wi].store(v, std::memory_order_relaxed);
    }
    *out = v;
    return cudaSuccess;
}

// x: channels-last [B][H][W][128]; w: [256][3][3][128]; shapes already validated by the caller
inline cudaError_t conv3x3_head_launch(const float* x, int B, int H, int W, const float* w, const float* bias,
                                       const float* head_w_host, float* taps, cudaStream_t stream) {
    auto encode = ch_encode_fn();
    if (!encode) return cudaErrorNotSupported;
    ConvHeadArgs a{};
    a.bias = bias;
    a.taps = taps;
    a.B = B; a.H = H; a.W = W;
    a.Wp = convhead_wp(W);
    a.R = kCHTileM / a.Wp;
    a.tiles_per_map = (H + a.R - 1) / a.R;
    a.T = B * a.tiles_per_map;
    a.a_bytes = uint32_t(a.R + 2) * uint32_t(a.Wp) * 128u;
    const size_t smem = ConvHeadLayout(a.a_bytes).alloc_bytes();

    CUtensorMap tm_x, tm_w;
    {
        const cuuint64_t dims[4] = {cuuint64_t(kCHCin), cuuint64_t(W), cuuint64_t(H), cuuint64_t(B)};
        const cuuint64_t strides[3] = {cuuint64_t(kCHCin) * 4, cuuint64_t(W) * kCHCin * 4, cuuint64_t(H) * W * kCHCin * 4};
        const cuuint32_t box[4] = {cuuint32_t(kCHChunk), cuuint32_t(a.Wp), cuuint32_t(a.R + 2), 1};
        const cuuint32_t estr[4] = {1, 1, 1, 1};
        if (encode(&tm_x, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(x), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
            return cudaErrorInvalidValue;
    }
    {
        const cuuint64_t dims[2] = {cuuint64_t(9 * kCHCin), cuuint64_t(kCHCout)};
        const cuuint64_t strides[1] = {cuuint64_t(9 * kCHCin) * 4};
        const cuuint32_t box[2] = {cuuint32_t(kCHChunk), kCHBSliceRows};
        const cuuint32_t estr[2] = {1, 1};
        if (encode(&tm_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(w), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
            return cudaErrorInvalidValue;
    }
    ConvHeadWeights hw;
    for (int i = 0; i < kCHCout * 9; ++i) hw.w[i] = head_w_host[i];

    int max_clusters = 0;
    cudaError_t e = ch_max_clusters(a.Wp, smem, &max_clusters);
    if (e != cudaSuccess) return e;
    const int pairs = (a.T + kCHCluster - 1) / kCHCluster;
    const int nC = pairs < max_clusters ? pairs : max_clusters;
    e = cudaFuncSetAttribute(conv3x3_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    if (e != cudaSuccess) return e;
    conv3x3_head_kernel<<<nC * kCHCluster, kCHThreads, smem, stream>>>(tm_x, tm_w, a, hw);
    return cudaGetLastError();
}

}  // namespace nastar
