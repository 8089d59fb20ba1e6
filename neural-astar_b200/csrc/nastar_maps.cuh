// nastar_maps.cuh — planning maps from decoded map images (the planning-datasets generator's load_maze_from_directory),
// and one-hot policies drawn from the maximal action sets of the label kernel.
//
// maps_from_images_kernel: one CTA per image, one launch, no host synchronisation.  Per image (DESIGN.md §13):
//   resize     Pillow's Image.resize((W, H)) of a uint8 L image (BICUBIC, reducing_gap=None): a horizontal pass into a
//              uint8 intermediate when the width changes, then a vertical pass when the height changes.  Per axis,
//              scale = in/out, fs = max(scale, 1), support = 2 fs; output j has center = (j + 0.5) scale, first tap
//              xmin = max(int(center - support + 0.5), 0), taps min(int(center + support + 0.5), in) - xmin, weights
//              cubic((x + xmin - center + 0.5) * (1/fs)) (Keys, a = -0.5) divided by their sequential double sum and
//              quantised to 22 fraction bits; an output is clip8((2^21 + sum pixel * weight) >> 22);
//   otsu       skimage's threshold_otsu of the float32 resized image: a uniform image returns its value; otherwise the
//              256-bin histogram over [lo, hi] (the min and max levels), sequential float64 cumulative sums from
//              both ends, and the center of the first bin that maximises w1 w2 (m1 - m2)^2;
//   map        1.0 where level > threshold, else 0.0.
// The coefficient tables are computed in the kernel with explicitly rounded double operations (__dmul_rn, ...), so no
// multiply-add is contracted into an FMA: they equal Pillow's, which evaluates each operation in IEEE double.
// The levels are integers, so np.histogram's edges lo + i (hi-lo)/256 and centers lo + (2i+1)(hi-lo)/512 are exact in
// float32, and level v falls in bin min((v-lo)*256 / (hi-lo), 255): the kernel histograms the 256 levels and maps
// each level to its bin (tests/test_maps_cpu.py checks the rule against np.histogram for every (lo, hi)).  The
// cumulative sums run sequentially on one thread each (a parallel scan would round differently); the 255 variances
// and their first argmax are computed in parallel, which changes no rounding.
//
// Shared memory: the Otsu arrays, both coefficient tables and a strip of the intermediate, `sw` columns of every
// source row the vertical pass reads.  The strips cover the W output columns in turn (a column of the vertical pass
// reads only its own intermediate column), so no source size needs more than the tables and one strip.  The resized
// levels are parked as floats in the image's own fp32 map plane until the threshold is known, then overwritten there.
//
// Limits: H, W <= kMapsMaxSide (512), the limit of the label, goal and sampler kernels; H0, W0 <= kMapsMaxSrcSide
// (2048).  Tables and strip then take at most ~150 KB.
//
// draw_policies_kernel: one thread per cell.  Of the cell's action mask (bit a = action a is maximal, nastar_labels.cuh)
// it picks set bit k = (d * popc) >> 32 in action order, d = the cell's u32 draw, and writes the one-hot column of 8
// floats; a cell with an empty mask gets an all-zero column.
#pragma once
#include <cmath>
#include <cstdint>

namespace nastar {

constexpr int kMapsMaxSide = 512;
constexpr int kMapsMaxSrcSide = 2048;
constexpr int kMapsThreads = 256;
constexpr int kMapsUniform = 1;
constexpr int kMapsPrecision = 22;
constexpr size_t kMapsStripBytes = 64 * 1024;   // the intermediate strip's budget
constexpr size_t kMapsOtsuBytes = 256 * (8 + 8 + 4 + 4 + 4 + 4);   // cs1, cs2 (double); w1, w2, level and bin counts

struct MapsArgs {
    const uint8_t* images;   // [B] images of H0*W0 uint8 levels (rows W0 apart), image_stride elements apart
    int64_t image_stride;
    int B, H0, W0, H, W;
    int kw, kh;              // taps stride of the horizontal / vertical coefficient tables
    int sw;                  // intermediate columns per strip
    float* maps;             // [B][H*W]
    uint8_t* resized;        // [B][H*W] or nullptr
    float* thresholds;       // [B]
    int32_t* status;         // [B]
};

// taps stride of one axis: Pillow's ksize = 2 ceil(support) + 1, never more than the input size
inline int maps_taps(int in, int out) {
    const double fs = double(in) / out > 1.0 ? double(in) / out : 1.0;
    int k = int(std::ceil(2.0 * fs)) * 2 + 1;
    return k < in ? k : in;
}
inline int maps_strip_cols(int H0, int W) {
    const int sw = int(kMapsStripBytes / size_t(H0));
    return sw < 1 ? 1 : (sw > W ? W : sw);
}
inline size_t maps_smem_bytes(int H0, int W0, int H, int W) {
    const size_t tables = size_t(W) * (maps_taps(W0, W) + 2) + size_t(H) * (maps_taps(H0, H) + 2);
    return kMapsOtsuBytes + tables * 4 + size_t(H0) * maps_strip_cols(H0, W);
}

__device__ __forceinline__ double maps_cubic(double x) {
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(a + 2.0, x), a + 3.0), x), x), 1.0);
    if (x < 2.0) return __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(x, 5.0), x), 8.0), x), 4.0), a);
    return 0.0;
}

// output j of an in -> out axis: first tap, tap count (<= stride) and fixed-point weights kk[0..count)
__device__ void maps_coeffs(int in, int out, int j, int stride, int* kk, int* first, int* count) {
    const double scale = __ddiv_rn(double(in), double(out));
    const double fs = scale > 1.0 ? scale : 1.0;
    const double support = __dmul_rn(2.0, fs);
    const double ss = __ddiv_rn(1.0, fs);
    const double center = __dmul_rn(__dadd_rn(double(j), 0.5), scale);
    int xmin = __double2int_rz(__dadd_rn(__dsub_rn(center, support), 0.5));
    int xmax = __double2int_rz(__dadd_rn(__dadd_rn(center, support), 0.5));
    xmin = xmin < 0 ? 0 : xmin;
    xmax = (xmax > in ? in : xmax) - xmin;
    xmax = xmax > stride ? stride : xmax;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) ww = __dadd_rn(ww, maps_cubic(__dmul_rn(__dadd_rn(__dsub_rn(double(x + xmin), center), 0.5), ss)));
    for (int x = 0; x < xmax; ++x) {
        double w = maps_cubic(__dmul_rn(__dadd_rn(__dsub_rn(double(x + xmin), center), 0.5), ss));
        if (ww != 0.0) w = __ddiv_rn(w, ww);
        const double q = __dmul_rn(w, double(1 << kMapsPrecision));
        kk[x] = __double2int_rz(w < 0.0 ? __dadd_rn(-0.5, q) : __dadd_rn(0.5, q));
    }
    *first = xmin;
    *count = xmax;
}

// center of bin i of the histogram over [lo, lo + d]: lo + (2i+1) d / 512, exact in float32
__device__ __forceinline__ float maps_center(int lo, int d, int i) { return float(lo) + float((2 * i + 1) * d) / 512.0f; }

__device__ __forceinline__ uint32_t maps_clip8(int acc) {
    return acc >= (1 << (kMapsPrecision + 8)) ? 255u : acc <= 0 ? 0u : uint32_t(acc >> kMapsPrecision);
}

__global__ void __launch_bounds__(kMapsThreads) maps_from_images_kernel(MapsArgs a) {
    extern __shared__ double maps_smem[];
    __shared__ double s_var[kMapsThreads / 32];
    __shared__ int s_idx[kMapsThreads / 32];
    __shared__ int s_lo, s_hi;

    const int b = blockIdx.x, H0 = a.H0, W0 = a.W0, H = a.H, W = a.W, N = H * W;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool need_h = W != W0, need_v = H != H0;
    double* cs1 = maps_smem;
    double* cs2 = cs1 + 256;
    int* w1 = reinterpret_cast<int*>(cs2 + 256);
    int* w2 = w1 + 256;
    uint32_t* hist = reinterpret_cast<uint32_t*>(w2 + 256);
    uint32_t* cnt = hist + 256;
    int* kk_h = reinterpret_cast<int*>(cnt + 256);
    int* x_h = kk_h + W * a.kw;
    int* n_h = x_h + W;
    int* kk_v = n_h + W;
    int* x_v = kk_v + H * a.kh;
    int* n_v = x_v + H;
    uint8_t* strip = reinterpret_cast<uint8_t*>(n_v + H);
    const uint8_t* img = a.images + int64_t(b) * a.image_stride;
    float* map = a.maps + int64_t(b) * N;

    // 1. coefficient tables, empty histogram
    for (int i = tid; i < 256; i += blockDim.x) hist[i] = 0;
    if (need_h)
        for (int j = tid; j < W; j += blockDim.x) maps_coeffs(W0, W, j, a.kw, kk_h + j * a.kw, x_h + j, n_h + j);
    if (need_v)
        for (int j = tid; j < H; j += blockDim.x) maps_coeffs(H0, H, j, a.kh, kk_v + j * a.kh, x_v + j, n_v + j);
    __syncthreads();

    // 2. resize, strip by strip: the intermediate rows [r0, r1) of columns [x0, x0 + cols), then their H outputs
    const int r0 = need_v ? x_v[0] : 0, r1 = need_v ? x_v[H - 1] + n_v[H - 1] : H0;
    for (int x0 = 0; x0 < W; x0 += a.sw) {
        const int cols = W - x0 < a.sw ? W - x0 : a.sw;
        for (int i = tid; i < (r1 - r0) * cols; i += blockDim.x) {
            const int r = i / cols, c = i - r * cols, xx = x0 + c;
            const uint8_t* row = img + int64_t(r0 + r) * W0;
            uint32_t v;
            if (need_h) {
                const int* k = kk_h + xx * a.kw;
                const uint8_t* s = row + x_h[xx];
                int acc = 1 << (kMapsPrecision - 1);
                for (int t = 0; t < n_h[xx]; ++t) acc += int(s[t]) * k[t];
                v = maps_clip8(acc);
            } else {
                v = row[xx];
            }
            strip[r * cols + c] = uint8_t(v);
        }
        __syncthreads();
        for (int i = tid; i < H * cols; i += blockDim.x) {
            const int yy = i / cols, c = i - yy * cols;
            uint32_t v;
            if (need_v) {
                const int* k = kk_v + yy * a.kh;
                const uint8_t* s = strip + (x_v[yy] - r0) * cols + c;
                int acc = 1 << (kMapsPrecision - 1);
                for (int t = 0; t < n_v[yy]; ++t) acc += int(s[t * cols]) * k[t];
                v = maps_clip8(acc);
            } else {
                v = strip[yy * cols + c];
            }
            const int cell = yy * W + x0 + c;
            map[cell] = float(v);
            if (a.resized) a.resized[int64_t(b) * N + cell] = uint8_t(v);
            atomicAdd(hist + v, 1u);
        }
        __syncthreads();
    }

    // 3. Otsu: the lowest and highest level present, their bin counts, sequential cumulative sums from each end
    if (warp == 0) {
        int lo = 256, hi = -1;
        for (int k = 0; k < 8; ++k) {
            const uint32_t m = __ballot_sync(0xFFFFFFFFu, hist[k * 32 + lane] != 0);
            if (m && lo == 256) lo = k * 32 + __ffs(m) - 1;
            if (m) hi = k * 32 + 31 - __clz(m);
        }
        if (lane == 0) {
            s_lo = lo;
            s_hi = hi;
        }
    }
    for (int i = tid; i < 256; i += blockDim.x) cnt[i] = 0;
    __syncthreads();
    const int lo = s_lo, hi = s_hi, d = hi - lo;
    const bool uniform = d == 0;
    if (!uniform) {
        for (int v = lo + tid; v <= hi; v += blockDim.x)
            if (hist[v]) cnt[min((v - lo) * 256 / d, 255)] = hist[v];
        __syncthreads();
        if (tid == 0 || tid == 32) {
            const bool fwd = tid == 0;
            int wsum = 0;
            double csum = 0.0;
            for (int s = 0; s < 256; ++s) {
                const int i = fwd ? s : 255 - s;
                wsum += int(cnt[i]);
                csum = __dadd_rn(csum, __dmul_rn(double(cnt[i]), double(maps_center(lo, d, i))));
                (fwd ? w1 : w2)[i] = wsum;
                (fwd ? cs1 : cs2)[i] = csum;
            }
        }
        __syncthreads();
        // variance of split i (classes <= i and > i), i < 255; w1[i] >= cnt[0] > 0 and w2[i+1] >= cnt[255] > 0
        double best = -1.0;
        int bi = 256;
        for (int i = tid; i < 255; i += blockDim.x) {
            const double m1 = __ddiv_rn(cs1[i], double(w1[i])), m2 = __ddiv_rn(cs2[i + 1], double(w2[i + 1]));
            const double dm = __dsub_rn(m1, m2);
            const double v = __dmul_rn(double(int64_t(w1[i]) * w2[i + 1]), __dmul_rn(dm, dm));
            if (v > best) {
                best = v;
                bi = i;
            }
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const double ov = __shfl_xor_sync(0xFFFFFFFFu, best, o);
            const int oi = __shfl_xor_sync(0xFFFFFFFFu, bi, o);
            if (ov > best || (ov == best && oi < bi)) {
                best = ov;
                bi = oi;
            }
        }
        if (lane == 0) {
            s_var[warp] = best;
            s_idx[warp] = bi;
        }
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < int(blockDim.x >> 5); ++w)
                if (s_var[w] > best || (s_var[w] == best && s_idx[w] < bi)) {
                    best = s_var[w];
                    bi = s_idx[w];
                }
            s_idx[0] = bi;
        }
        __syncthreads();
    }
    const float th = uniform ? float(lo) : maps_center(lo, d, s_idx[0]);
    if (tid == 0) {
        a.thresholds[b] = th;
        a.status[b] = uniform ? kMapsUniform : 0;
    }
    // 4. threshold: every cell still holds its level
    for (int c = tid; c < N; c += blockDim.x) map[c] = map[c] > th ? 1.0f : 0.0f;
}

__global__ void draw_policies_kernel(const uint8_t* act_mask, const uint32_t* draws, int64_t B, int N, float* policies) {
    const int64_t total = B * N;
    for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += int64_t(gridDim.x) * blockDim.x) {
        const int64_t b = i / N;
        const int c = int(i - b * N);
        uint32_t m = act_mask[i];
        int pick = -1;
        if (m) {
            for (int k = int((uint64_t(draws[i]) * uint32_t(__popc(m))) >> 32); k; --k) m &= m - 1;
            pick = __ffs(m) - 1;
        }
        float* out = policies + b * 8 * N + c;
#pragma unroll
        for (int act = 0; act < 8; ++act) out[int64_t(act) * N] = act == pick ? 1.0f : 0.0f;
    }
}

}  // namespace nastar
