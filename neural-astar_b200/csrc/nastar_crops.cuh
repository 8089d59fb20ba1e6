// nastar_crops.cuh — RGB crops of scene images resized to Wo x Ho, bit-equal to Pillow's
// np.array(image.crop(box).resize((Wo, Ho))) for an RGB image (the planning-datasets SDD samples, DESIGN.md §22).
//
// crop_resize_rgb_kernel: one CTA per crop, one launch, no host synchronisation.  Per crop (x0, y0, x1, y1):
//   crop       pixel (x, y) of the cw x ch crop (cw = x1 - x0, ch = y1 - y0) is source pixel (x0 + x, y0 + y), or 0 in
//              every channel where that lies outside the source (ImagingCrop fills such a box with zeros first);
//   resize     Pillow's BICUBIC resize of the crop, each channel as an L image: a horizontal pass into a uint8
//              intermediate when cw != Wo, then a vertical pass when ch != Ho, with the coefficient tables of
//              maps_coeffs (nastar_maps.cuh: explicitly rounded doubles, 22-bit fixed-point weights) and maps_clip8.
//              Pillow's RGB resize runs the L arithmetic on each of the three bands with the same weights.
// The horizontal pass computes only the intermediate rows the vertical pass reads, [r0, r1), as Pillow does.
//
// Shared memory: the vertical table (Ho rows of kh + 2 ints) for the whole crop, then, strip by strip, the horizontal
// table of the strip's `sw` output columns (kw + 2 ints each) and the intermediate strip, (r1 - r0) rows of sw RGB
// triples.  The launch's dynamic shared memory is the same for every CTA (the host sizes it for the crop that needs
// the most, and at least kCropSmemTarget); each CTA takes the widest strip that fits it, so small crops run their W
// columns in one strip.
//
// Limits: source and crop sides <= kCropMaxSide (4096), Ho, Wo <= kCropMaxOut (1024).  The vertical table then takes
// at most 4 ch + 5 Ho ints (86 KB) and one strip column 3 ch bytes plus kw + 2 <= 4098 ints, so every crop fits.
#pragma once
#include <cstdint>

#include "../../include/nastar_b200.h"
#include "nastar_maps.cuh"   // maps_coeffs, maps_clip8, kMapsPrecision

namespace nastar {

constexpr int kCropMaxSide = 4096;
constexpr int kCropMaxOut = 1024;
constexpr int kCropThreads = 256;
constexpr size_t kCropSmemTarget = 72 * 1024;   // three CTAs per SM

// taps stride of one axis (maps_taps in integers): Pillow's ksize = 2 ceil(2 max(in/out, 1)) + 1, at most `in`
__host__ __device__ inline int crop_taps(int in, int out) {
    const int k = (in > out ? (2 * in + out - 1) / out : 2) * 2 + 1;
    return k < in ? k : in;
}
// ints of the vertical table, and bytes of one strip column (its horizontal table and intermediate), of one crop
__host__ __device__ inline int64_t crop_vtable_ints(int ch, int Ho) { return ch == Ho ? 0 : int64_t(Ho) * (crop_taps(ch, Ho) + 2); }
__host__ __device__ inline int64_t crop_col_bytes(int cw, int ch, int Wo) {
    return (cw == Wo ? 0 : int64_t(crop_taps(cw, Wo) + 2) * 4) + int64_t(ch) * 3;
}
inline size_t crop_smem_need(int cw, int ch, int Ho, int Wo) {
    return size_t(crop_vtable_ints(ch, Ho) * 4 + crop_col_bytes(cw, ch, Wo));
}

struct CropArgs {
    const nastar_rgb_image* src;
    const nastar_rgb_crop* crops;   // CTA i takes crops[i]
    int Ho, Wo;
    int64_t smem;                   // the launch's dynamic shared memory, bytes
    uint8_t* out;                   // [N][Ho][Wo][3]
};

__global__ void __launch_bounds__(kCropThreads) crop_resize_rgb_kernel(CropArgs a) {
    extern __shared__ int crop_smem[];
    const nastar_rgb_crop c = a.crops[blockIdx.x];
    const nastar_rgb_image s = a.src[c.src];
    const int cw = c.x1 - c.x0, ch = c.y1 - c.y0, Ho = a.Ho, Wo = a.Wo, tid = threadIdx.x;
    const bool need_h = cw != Wo, need_v = ch != Ho;
    const int kw = crop_taps(cw, Wo), kh = crop_taps(ch, Ho);
    const int64_t vt = crop_vtable_ints(ch, Ho);
    int* kk_v = crop_smem;
    int* x_v = kk_v + Ho * kh;
    int* n_v = x_v + Ho;
    uint8_t* out = a.out + int64_t(c.out) * Ho * Wo * 3;

    // 1. the vertical table, and the intermediate rows it reads
    if (need_v)
        for (int j = tid; j < Ho; j += blockDim.x) maps_coeffs(ch, Ho, j, kh, kk_v + j * kh, x_v + j, n_v + j);
    __syncthreads();
    const int r0 = need_v ? x_v[0] : 0, rows = (need_v ? x_v[Ho - 1] + n_v[Ho - 1] : ch) - r0;
    const int64_t col = (need_h ? int64_t(kw + 2) * 4 : 0) + int64_t(rows) * 3;
    const int64_t fit = (a.smem - vt * 4) / col;
    const int sw = fit < Wo ? int(fit) : Wo;   // >= 1: the host sized smem for this crop
    int* kk_h = crop_smem + vt;
    int* x_h = kk_h + sw * kw;
    int* n_h = x_h + sw;
    uint8_t* strip = reinterpret_cast<uint8_t*>(need_h ? n_h + sw : kk_h);

    // 2. strip by strip: the horizontal table of output columns [xo, xo + cols), their intermediate rows, their Ho
    //    output rows
    for (int xo = 0; xo < Wo; xo += sw) {
        const int cols = Wo - xo < sw ? Wo - xo : sw;
        if (need_h) {
            for (int j = tid; j < cols; j += blockDim.x) maps_coeffs(cw, Wo, xo + j, kw, kk_h + j * kw, x_h + j, n_h + j);
            __syncthreads();
        }
        for (int i = tid; i < rows * cols; i += blockDim.x) {
            const int r = i / cols, cc = i - r * cols, sy = c.y0 + r0 + r;
            uint32_t v0 = 0, v1 = 0, v2 = 0;
            if (sy >= 0 && sy < s.H) {
                const uint8_t* row = s.pixels + int64_t(sy) * s.pitch;
                if (need_h) {
                    const int* k = kk_h + cc * kw;
                    const int sx0 = c.x0 + x_h[cc];
                    int acc0 = 1 << (kMapsPrecision - 1), acc1 = acc0, acc2 = acc0;
                    for (int t = 0; t < n_h[cc]; ++t) {
                        const int sx = sx0 + t;
                        if (sx >= 0 && sx < s.W) {
                            const uint8_t* p = row + 3 * sx;
                            acc0 += int(p[0]) * k[t];
                            acc1 += int(p[1]) * k[t];
                            acc2 += int(p[2]) * k[t];
                        }
                    }
                    v0 = maps_clip8(acc0);
                    v1 = maps_clip8(acc1);
                    v2 = maps_clip8(acc2);
                } else {
                    const int sx = c.x0 + xo + cc;
                    if (sx >= 0 && sx < s.W) {
                        const uint8_t* p = row + 3 * sx;
                        v0 = p[0];
                        v1 = p[1];
                        v2 = p[2];
                    }
                }
            }
            uint8_t* q = strip + (r * cols + cc) * 3;
            q[0] = uint8_t(v0);
            q[1] = uint8_t(v1);
            q[2] = uint8_t(v2);
        }
        __syncthreads();
        for (int i = tid; i < Ho * cols; i += blockDim.x) {
            const int yy = i / cols, cc = i - yy * cols;
            uint32_t v0, v1, v2;
            if (need_v) {
                const int* k = kk_v + yy * kh;
                const uint8_t* p = strip + ((x_v[yy] - r0) * cols + cc) * 3;
                int acc0 = 1 << (kMapsPrecision - 1), acc1 = acc0, acc2 = acc0;
                for (int t = 0; t < n_v[yy]; ++t, p += cols * 3) {
                    acc0 += int(p[0]) * k[t];
                    acc1 += int(p[1]) * k[t];
                    acc2 += int(p[2]) * k[t];
                }
                v0 = maps_clip8(acc0);
                v1 = maps_clip8(acc1);
                v2 = maps_clip8(acc2);
            } else {
                const uint8_t* p = strip + (yy * cols + cc) * 3;
                v0 = p[0];
                v1 = p[1];
                v2 = p[2];
            }
            uint8_t* q = out + (int64_t(yy) * Wo + xo + cc) * 3;
            q[0] = uint8_t(v0);
            q[1] = uint8_t(v1);
            q[2] = uint8_t(v2);
        }
        __syncthreads();
    }
}

}  // namespace nastar
