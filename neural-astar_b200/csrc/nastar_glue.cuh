// nastar_glue.cuh — the two small kernels either side of the encoder CNN (SURVEY.md 8(f)-3).
//
// The encoder itself stays PyTorch/cuDNN (north star); what is replaced here is the element-wise glue of
// NeuralAstar.encode (/root/reference/src/neural_astar/planner/astar.py:172-177: start+goal add, nearest
// upsample, channel concat, plus the NCHW->NHWC conversion cuDNN's tensor-core convs want) and of
// EncoderBase.forward (/root/reference/src/neural_astar/planner/encoder.py:32-34: sigmoid * const) —
// seven ATen launches per forward in round 1, now one kernel in front of the convs and the search
// kernel's own prologue behind them.
#pragma once
#include "../../include/nastar_b200.h"
#include "nastar_common.cuh"

namespace nastar {

// out[b][ym][xm][0..C-1] = map_designs[b][c][ym][xm];  out[b][ym][xm][C] = (start+goal)[b][ys][xs] with the
// source index of F.interpolate(mode="nearest"): min(floor(dst * in/out), in-1), scale evaluated in fp32.
__global__ void __launch_bounds__(256) pack_inputs_kernel(const float* __restrict__ maps, int C, int Hm, int Wm,
                                                          const float* __restrict__ start, int64_t start_stride,
                                                          const float* __restrict__ goal, int64_t goal_stride,
                                                          int B, int H, int W, float* __restrict__ out) {
    const int64_t npix = int64_t(B) * Hm * Wm;
    const float sh = float(H) / float(Hm), sw = float(W) / float(Wm);
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < npix; i += int64_t(gridDim.x) * blockDim.x) {
        const int xm = int(i % Wm);
        const int ym = int((i / Wm) % Hm);
        const int b = int(i / (int64_t(Wm) * Hm));
        int ys = ym, xs = xm;
        if (H != Hm) ys = min(int(floorf(float(ym) * sh)), H - 1);
        if (W != Wm) xs = min(int(floorf(float(xm) * sw)), W - 1);
        const float mark = __fadd_rn(__ldg(start + int64_t(b) * start_stride + ys * W + xs),
                                     __ldg(goal + int64_t(b) * goal_stride + ys * W + xs));
        float* o = out + i * (C + 1);
        const float* m = maps + (int64_t(b) * C * Hm + ym) * Wm + xm;
        if (C == 1) {
            *reinterpret_cast<float2*>(o) = make_float2(__ldg(m), mark);
        } else if (C == 3) {
            *reinterpret_cast<float4*>(o) = make_float4(__ldg(m), __ldg(m + int64_t(Hm) * Wm), __ldg(m + 2 * int64_t(Hm) * Wm), mark);
        } else {
            for (int c = 0; c < C; ++c) o[c] = __ldg(m + c * int64_t(Hm) * Wm);
            o[C] = mark;
        }
    }
}

// dense cost plane from the 9-tap partial products: same device function as the search prologue
__global__ void __launch_bounds__(256) cost_from_taps_kernel(const float* __restrict__ taps, int B, int H, int W,
                                                             float bias, float scale, float* __restrict__ cost) {
    const int N = H * W;
    const int64_t total = int64_t(B) * N;
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int b = int(i / N);
        const int rc = int(i - int64_t(b) * N);
        const int y = rc / W, x = rc - y * W;
        cost[i] = cost_from_taps(taps + int64_t(b) * N * 9, y, x, H, W, bias, scale);
    }
}

// ---- first encoder layer fused with the input assembly ("m+" planners) --------------------------------------------
// conv1 of the CNN encoder has 2 input channels (the map and the start+goal marks, astar.py:172-177) and 32 output
// channels (encoder.py:60-78): 18 multiply-adds per output value — not a contraction worth a tensor core, and cuDNN
// runs it with a generic fp32 kernel on top of a separate pack kernel.  Here one thread owns one pixel: the marks
// channel is formed on the fly (start + goal), the 3x3 / pad 1 window is read straight from the three input planes
// (27 predicated loads, L1-resident: 4 KB per map and plane), the 576 FMAs take their weights from the constant bank
// (the folded weights are a by-value kernel parameter, like the head's), BatchNorm arrives folded into w / b, ReLU is
// applied, and the warp's 32 pixels x 32 channels are transposed through shared memory so the channels-last result
// ([B][H][W][32]) leaves as fully coalesced 128-bit stores.  (A first version with thread = (pixel, 4 channels) and the
// weights in shared memory was load/store-unit bound: 8x the window loads and 18 LDS.128 per thread.)
struct Conv1Weights {
    float w[9][2][32];   // [tap][cin][cout], BatchNorm folded
    float b[32];
};

constexpr int kConv1Warps = 8;
constexpr int kConv1Row = 36;   // floats per staged pixel: 32 channels + 4 pad (keeps 16 B alignment, conflict-free quarter-warps)

__global__ void __launch_bounds__(32 * kConv1Warps) conv1_marks_kernel(const float* __restrict__ maps,
                                                                       const float* __restrict__ start, int64_t start_stride,
                                                                       const float* __restrict__ goal, int64_t goal_stride,
                                                                       int n_pix, int H, int W,
                                                                       const __grid_constant__ Conv1Weights cw,
                                                                       float* __restrict__ out) {
    __shared__ __align__(16) float sT[kConv1Warps][32 * kConv1Row];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int N = H * W;
    float* st = sT[warp];
    for (int base = (blockIdx.x * kConv1Warps + warp) * 32; base < n_pix; base += gridDim.x * kConv1Warps * 32) {
        const int pix = base + lane;
        const bool live = pix < n_pix;
        const int pc = live ? pix : 0;
        const int b = pc / N;
        const int rc = pc - b * N;
        const int y = rc / W, x = rc - y * W;
        const float* pm = maps + int64_t(b) * N;
        const float* ps = start + int64_t(b) * start_stride;
        const float* pg = goal + int64_t(b) * goal_stride;
        float acc[32];
#pragma unroll
        for (int c = 0; c < 32; ++c) acc[c] = cw.b[c];
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            const int yy = y + ky - 1;
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                const int xx = x + kx - 1;
                const bool in = live && unsigned(yy) < unsigned(H) && unsigned(xx) < unsigned(W);
                const int o = in ? yy * W + xx : 0;
                const float m = in ? __ldg(pm + o) : 0.f;
                const float k = in ? __fadd_rn(__ldg(ps + o), __ldg(pg + o)) : 0.f;   // start_maps + goal_maps (:173)
#pragma unroll
                for (int c = 0; c < 32; ++c) acc[c] = fmaf(k, cw.w[ky * 3 + kx][1][c], fmaf(m, cw.w[ky * 3 + kx][0][c], acc[c]));
            }
        }
#pragma unroll
        for (int c = 0; c < 32; c += 4)
            *reinterpret_cast<float4*>(st + lane * kConv1Row + c) =
                make_float4(fmaxf(acc[c], 0.f), fmaxf(acc[c + 1], 0.f), fmaxf(acc[c + 2], 0.f), fmaxf(acc[c + 3], 0.f));
        __syncwarp();
        float4* dst = reinterpret_cast<float4*>(out) + int64_t(base) * 8;     // 8 float4 per pixel
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int v = j * 32 + lane;                                       // float4 index inside the warp's 4 KB tile
            if (base + (v >> 3) < n_pix)
                dst[v] = *reinterpret_cast<const float4*>(st + (v >> 3) * kConv1Row + (v & 7) * 4);
        }
        __syncwarp();
    }
}

// ---- single-output-channel head of the encoder: per-pixel partial products ---------------------------------------
// The encoder's last layer is a 3x3 conv with ONE output channel (encoder.py:60-78, channels [...,256,1]).  Round 1
// already evaluated it as a per-pixel [C] x [C,9] product followed by a 9-tap gather (planner/encoder.py
// `_conv3x3_single_output`); the gather now lives in the search kernel's prologue (NASTAR_COST_TAPS).  The product
// itself is 0.5 GFLOP over a 105 MB activation (b=100, 32x32, C=256): HBM-bound, so the activation is read exactly
// once and never through a generic skinny SGEMM.  Here: one thread per pixel keeps the 9 sums in registers; the C*9 weights arrive as a
// by-value kernel parameter, i.e. in the constant bank, so every FFMA takes its weight operand straight from a uniform
// register — no weight loads at all.  The activation is staged through shared memory: a warp copies its 32 pixels'
// channel slice (32 x 32 floats, one 128-byte line per pixel) with fully coalesced 16-byte cp.async into one of its two
// buffers while it multiplies the slice in the other, and every lane reads its own pixel's row back with conflict-free
// LDS.128 (row stride 36 floats).  Measured at b=100, 32x32, C=256 (105 MB read, tools/head_probe.py) on an H100 SXM at
// 700 W: 51 us with CUDA events = 2.06 TB/s; torch.sum over the same tensor takes 41.5 us.  16-channel slices (20 KB per
// CTA, more CTAs per SM) were measured there too and are slower (62 us).  Dropped earlier: the same staging
// single-buffered with 64-channel slices, each lane streaming its own 1 KB row straight from global memory (every LDG.128
// touches 32 different lines), and a CTA-cooperative version with whole 32 KB tiles in a cp.async ring and one channel
// slice per warp (weights per warp either as 8 separately unrolled constant-bank blocks — instruction-cache thrash — or
// as broadcast LDS.128 from shared memory — MIO-throttled).
// Same FMA order as the first version (ascending channel), so the products are bit-identical to it.
template <int C>
struct HeadWeights {
    float w[C * 9];   // [c][k], k = ky*3+kx, BatchNorm already folded
};

constexpr int kHeadWarps = 4;
// channels staged per pass: 32 (128 contiguous bytes per pixel), or all 16 of the U-Net's depth-5 head
template <int C>
constexpr int kHeadSlice = C < 32 ? C : 32;

template <int C>
__device__ __forceinline__ void head_issue_slice(const float* __restrict__ x, int64_t P, int64_t p0, int s0, uint32_t dst_s,
                                                 int lane) {
    constexpr int kRow = kHeadSlice<C> + 4, kChunks = kHeadSlice<C> / 4;
#pragma unroll
    for (int i = 0; i < kChunks; ++i) {              // 32 lanes x kChunks copies of 16 B = the 32 x kHeadSlice tile
        const int idx = i * 32 + lane;
        const int px = idx / kChunks, ch = idx % kChunks;
        int64_t p = p0 + px;
        p = p < P ? p : P - 1;                       // ragged last group: re-read the last pixel, never stored
        const float* src = x + p * C + s0 + ch * 4;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst_s + uint32_t(px * kRow + ch * 4) * 4u), "l"(src)
                     : "memory");
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

template <int C>
__global__ void __launch_bounds__(32 * kHeadWarps) head_taps_kernel(const float* __restrict__ x, int64_t P,
                                                                    const __grid_constant__ HeadWeights<C> hw,
                                                                    float* __restrict__ out) {
    constexpr int kRow = kHeadSlice<C> + 4;          // padded row (floats): 16 B aligned, quarter-warps hit 32 distinct banks
    constexpr int kChunks = kHeadSlice<C> / 4;       // float4 per pixel and slice
    constexpr int kSlices = C / kHeadSlice<C>;
    __shared__ __align__(16) float sX[kHeadWarps][2][32 * kRow];   // per warp: two slices in flight / in use
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t st_s = uint32_t(__cvta_generic_to_shared(&sX[warp][0][0]));
    const int64_t groups = (P + 31) / 32;
    const int64_t gstride = int64_t(gridDim.x) * kHeadWarps;
    int64_t grp = int64_t(blockIdx.x) * kHeadWarps + warp;
    if (grp >= groups) return;
    int buf = 0;
    head_issue_slice<C>(x, P, grp * 32, 0, st_s, lane);
    for (; grp < groups; grp += gstride) {
        const int64_t p0 = grp * 32;
        float acc[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) acc[k] = 0.f;
#pragma unroll
        for (int sl = 0; sl < kSlices; ++sl) {
            // prefetch the next slice (of this group, or the first slice of the warp's next group) into the other buffer
            const bool last = (sl == kSlices - 1);
            const int64_t gn = last ? grp + gstride : grp;
            if (gn < groups)
                head_issue_slice<C>(x, P, gn * 32, last ? 0 : (sl + 1) * kHeadSlice<C>, st_s + uint32_t((buf ^ 1) * 32 * kRow) * 4u, lane);
            else
                asm volatile("cp.async.commit_group;" ::: "memory");
            asm volatile("cp.async.wait_group 1;" ::: "memory");
            __syncwarp();
            const float* st = &sX[warp][buf][0];
#pragma unroll
            for (int c4 = 0; c4 < kChunks; ++c4) {
                const float4 v = *reinterpret_cast<const float4*>(st + lane * kRow + c4 * 4);
#pragma unroll
                for (int k = 0; k < 9; ++k) {
                    acc[k] = fmaf(v.x, hw.w[(sl * kHeadSlice<C> + 4 * c4 + 0) * 9 + k], acc[k]);
                    acc[k] = fmaf(v.y, hw.w[(sl * kHeadSlice<C> + 4 * c4 + 1) * 9 + k], acc[k]);
                    acc[k] = fmaf(v.z, hw.w[(sl * kHeadSlice<C> + 4 * c4 + 2) * 9 + k], acc[k]);
                    acc[k] = fmaf(v.w, hw.w[(sl * kHeadSlice<C> + 4 * c4 + 3) * 9 + k], acc[k]);
                }
            }
            __syncwarp();                            // all lanes done reading before this buffer is refilled
            buf ^= 1;
        }
        if (p0 + lane < P) {
            float* o = out + (p0 + lane) * 9;
#pragma unroll
            for (int k = 0; k < 9; ++k) o[k] = acc[k];
        }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
}

// ---- U-Net decoder block input: nearest x2 upsample and skip concat (planner/encoder.py Unet) --------------------
// out[b][y][x][0..Cd-1] = dec[b][y/2][x/2][..], out[b][y][x][Cd..Cd+Cs-1] = skip[b][y][x][..]; channels-last fp32,
// out is [B][2h][2w][Cd+Cs].  A pure copy, so the result is bit-equal to cat(interpolate(dec, x2, nearest), skip).
// Two index spaces share one grid-stride loop: the first B*h*w*Cd/4 items each read one float4 of dec and store it to
// the four output pixels it covers, the remaining B*2h*2w*Cs/4 items each move one float4 of skip.  Every input byte is
// read once; consecutive threads read and write consecutive 16-byte vectors of one pixel's channel run.
__global__ void __launch_bounds__(256) upsample_concat_kernel(const float4* __restrict__ dec, int B, int h, int w, int cd4,
                                                              const float4* __restrict__ skip, int cs4,
                                                              float4* __restrict__ out) {
    const int W = 2 * w, co4 = cd4 + cs4;
    const int64_t n_dec = int64_t(B) * h * w * cd4;
    const int64_t total = n_dec + int64_t(B) * 2 * h * W * cs4;
    for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        if (i < n_dec) {
            const int64_t pix = i / cd4;                 // (b*h + yy)*w + xx
            const int c = int(i - pix * cd4);
            const int xx = int(pix % w);
            const int64_t by = pix / w;                  // b*h + yy: output rows 2*by and 2*by+1 of the flattened batch
            const float4 v = __ldg(dec + i);
            float4* o = out + (2 * by * W + 2 * xx) * co4 + c;
            o[0] = v;
            o[co4] = v;
            o[int64_t(W) * co4] = v;
            o[int64_t(W) * co4 + co4] = v;
        } else {
            const int64_t j = i - n_dec;
            const int64_t pix = j / cs4;
            const int c = int(j - pix * cs4);
            out[pix * co4 + cd4 + c] = __ldg(skip + j);
        }
    }
}

}  // namespace nastar
