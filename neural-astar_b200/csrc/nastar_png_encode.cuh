// nastar_png_encode.cuh — PNG encode on the GPU (DESIGN.md §21): 8-bit grey, non-interlaced, one IDAT chunk per
// file.  Three launches: png_filter_kernel, then deflate_kernel (nastar_deflate.cuh, unchanged) on the filtered
// streams, then png_finish_kernel around its output.
//
// png_filter_kernel: one CTA per image; each warp takes rows.  A row gets the filter type 0..4 (None, Sub, Up, Average,
// Paeth, one byte per pixel) whose filtered bytes have the least sum of |byte as int8| (libpng's heuristic), ties to
// the lowest type; row 0 sees a row of zeros above it.  The CTA writes filter byte + filtered row per scanline into the
// image's H*(W+1)-byte range of `filt`, and the Adler-32 of that stream: with d_j its byte j of n,
// A = 1 + sum d_j and B = n + sum (n - j) d_j (mod 65521), summed exactly in 64 bits per thread and block-reduced, so
// the result does not depend on the thread count.
//
// png_finish_kernel: one CTA per image, after deflate_kernel wrote image i's raw deflate stream at out_off[i] with the
// gaps of png_gap() before it.  Writes the signature, IHDR and its CRC, the IDAT length and type and the zlib header
// 78 DA into the 43 bytes before the stream, and the Adler-32, the IDAT CRC-32 (over "IDAT", the zlib header, the
// stream and the Adler-32: every thread's share, joined by a tree of crc(A||B) = shift(crc(A), |B|) ^ crc(B)) and an
// IEND chunk into the 20 bytes after it.  File i is then out[out_off[i] - 43, out_off[i] + out_len[i] + 20), and the
// files lie back to back.
#pragma once
#include <cstdint>

#include "../../include/nastar_b200.h"
#include "nastar_deflate.cuh"
#include "nastar_png.cuh"   // png_paeth

namespace nastar {

constexpr int kPngEncThreads = 256;
constexpr int kPngEncMaxSide = 2048;
constexpr int64_t kPngEncHead = 8 + 25 + 8 + 2;   // signature, IHDR chunk, IDAT length and type, zlib header
constexpr int64_t kPngEncTail = 4 + 4 + 12;       // Adler-32, IDAT CRC-32, IEND chunk
constexpr uint32_t kAdlerMod = 65521;

using PngEncDesc = nastar_png_enc_desc;   // one image of an encode batch (include/nastar_b200.h)

// the filtered stream's bytes
__host__ __device__ inline int64_t png_filtered_bytes(int32_t W, int32_t H) { return int64_t(H) * (int64_t(W) + 1); }
// the deflate gap before image i's stream: image i-1's tail, then image i's head
__host__ __device__ inline int64_t png_gap(int64_t i) { return kPngEncHead + (i > 0 ? kPngEncTail : 0); }

// byte x of row `cur` under filter f (prev: the row above, zeros for row 0)
__device__ inline uint8_t png_filter_byte(int f, const uint8_t* cur, const uint8_t* prev, int x) {
    const int v = cur[x], a = x > 0 ? cur[x - 1] : 0, b = prev ? prev[x] : 0, c = (x > 0 && prev) ? prev[x - 1] : 0;
    switch (f) {
        case 1: return uint8_t(v - a);
        case 2: return uint8_t(v - b);
        case 3: return uint8_t(v - ((a + b) >> 1));
        case 4: return uint8_t(v - png_paeth(a, b, c));
        default: return uint8_t(v);
    }
}

__device__ inline uint32_t png_abs8(uint8_t v) { return v < 128 ? v : 256u - v; }

struct PngFilterArgs {
    const PngEncDesc* desc;
    uint8_t* filt;
    uint32_t* adler;
};

__global__ void __launch_bounds__(kPngEncThreads) png_filter_kernel(PngFilterArgs a) {
    __shared__ unsigned long long part[2][kPngEncThreads / 32];
    const PngEncDesc d = a.desc[blockIdx.x];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int W = d.W, H = d.H;
    const int64_t n = png_filtered_bytes(W, H);
    uint8_t* out = a.filt + d.filt_off;
    unsigned long long s1 = 0, s2 = 0;   // sum d_j, sum (n - j) d_j
    for (int y = warp; y < H; y += kPngEncThreads / 32) {
        const uint8_t* cur = d.pixels + int64_t(y) * W;
        const uint8_t* prev = y > 0 ? cur - W : nullptr;
        uint32_t cost[5] = {0, 0, 0, 0, 0};
        for (int x = lane; x < W; x += 32)
            for (int f = 0; f < 5; ++f) cost[f] += png_abs8(png_filter_byte(f, cur, prev, x));
        int best = 0;
        uint32_t best_cost = 0;
        for (int f = 0; f < 5; ++f) {
            uint32_t c = cost[f];
            for (int o = 16; o >= 1; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
            if (f == 0 || c < best_cost) {
                best = f;
                best_cost = c;
            }
        }
        const int64_t row0 = int64_t(y) * (W + 1);
        if (lane == 0) {
            out[row0] = uint8_t(best);
            s1 += uint32_t(best);
            s2 += uint64_t(n - row0) * uint32_t(best);
        }
        for (int x = lane; x < W; x += 32) {
            const uint8_t v = png_filter_byte(best, cur, prev, x);
            const int64_t j = row0 + 1 + x;
            out[j] = v;
            s1 += v;
            s2 += uint64_t(n - j) * v;
        }
    }
    for (int o = 16; o >= 1; o >>= 1) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    if (lane == 0) {
        part[0][warp] = s1;
        part[1][warp] = s2;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t1 = 0, t2 = 0;
        for (int w = 0; w < kPngEncThreads / 32; ++w) {
            t1 += part[0][w];
            t2 += part[1][w];
        }
        const uint32_t A = uint32_t((1 + t1) % kAdlerMod), Bv = uint32_t((uint64_t(n) + t2) % kAdlerMod);
        a.adler[blockIdx.x] = Bv << 16 | A;
    }
}

struct PngFinishArgs {
    const PngEncDesc* desc;
    const int64_t* out_off;
    const int64_t* out_len;
    const uint32_t* adler;
    uint8_t* out;
    int64_t out_bytes;
};

__device__ inline void png_put32(uint8_t* p, uint32_t v) {
    p[0] = uint8_t(v >> 24);
    p[1] = uint8_t(v >> 16);
    p[2] = uint8_t(v >> 8);
    p[3] = uint8_t(v);
}

__global__ void __launch_bounds__(kPngEncThreads) png_finish_kernel(PngFinishArgs a) {
    __shared__ uint32_t crc_table[256];
    __shared__ uint32_t x2n[32];
    __shared__ uint32_t part[kPngEncThreads];
    __shared__ unsigned long long plen[kPngEncThreads];
    const int tid = threadIdx.x;
    const int i = blockIdx.x;
    const PngEncDesc d = a.desc[i];
    const int64_t off = a.out_off[i], len = a.out_len[i];
    // deflate_kernel placed the stream after this image's gap; anything else is not touched
    if (off < kPngEncHead || len < 0 || off + len + kPngEncTail > a.out_bytes) return;
    uint8_t* head = a.out + off - kPngEncHead;
    uint8_t* tail = a.out + off + len;
    for (int k = tid; k < 256; k += kPngEncThreads) {
        uint32_t c = uint32_t(k);
        for (int b = 0; b < 8; ++b) c = (c & 1) ? (c >> 1) ^ 0xEDB88320u : c >> 1;
        crc_table[k] = c;
    }
    if (tid == 0) {
        uint32_t p = 1u << 30;   // x^1
        for (int k = 0; k < 32; ++k) {
            x2n[k] = p;
            p = df_multmodp(p, p);
        }
        const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
        for (int k = 0; k < 8; ++k) head[k] = sig[k];
        uint8_t* ihdr = head + 8;
        png_put32(ihdr, 13);
        ihdr[4] = 'I'; ihdr[5] = 'H'; ihdr[6] = 'D'; ihdr[7] = 'R';
        png_put32(ihdr + 8, uint32_t(d.W));
        png_put32(ihdr + 12, uint32_t(d.H));
        ihdr[16] = 8;   // bit depth
        ihdr[17] = 0;   // grey
        ihdr[18] = 0;   // deflate
        ihdr[19] = 0;   // adaptive filtering
        ihdr[20] = 0;   // not interlaced
        uint8_t* idat = ihdr + 25;
        png_put32(idat, uint32_t(2 + len + 4));
        idat[4] = 'I'; idat[5] = 'D'; idat[6] = 'A'; idat[7] = 'T';
        idat[8] = 0x78;   // CM 8, CINFO 7
        idat[9] = 0xDA;   // FLEVEL 3, FDICT 0, FCHECK: 0x78DA % 31 == 0
        png_put32(tail, a.adler[i]);
        png_put32(tail + 8, 0);
        tail[12] = 'I'; tail[13] = 'E'; tail[14] = 'N'; tail[15] = 'D';
        png_put32(tail + 16, 0xAE426082u);   // CRC-32 of "IEND"
    }
    __syncthreads();
    if (tid == 0) {
        uint32_t c = 0xffffffffu;
        for (int k = 12; k < 12 + 17; ++k) c = crc_table[(c ^ head[k]) & 0xff] ^ (c >> 8);
        png_put32(head + 29, c ^ 0xffffffffu);
    }
    // CRC-32 of IDAT's type and data: out[off - 6, off + len + 4)
    const uint8_t* src = head + kPngEncHead - 6;
    const int64_t total = 6 + len + 4;
    const int64_t share = (total + kPngEncThreads - 1) / kPngEncThreads;
    const int64_t b0 = int64_t(tid) * share < total ? int64_t(tid) * share : total;
    const int64_t b1 = b0 + share < total ? b0 + share : total;
    uint32_t c = 0xffffffffu;
    for (int64_t k = b0; k < b1; ++k) c = crc_table[(c ^ src[k]) & 0xff] ^ (c >> 8);
    part[tid] = c ^ 0xffffffffu;
    plen[tid] = uint64_t(b1 - b0);
    __syncthreads();
    for (int s = 1; s < kPngEncThreads; s <<= 1) {
        if ((tid & (2 * s - 1)) == 0) {
            part[tid] = df_crc_combine(x2n, part[tid], part[tid + s], plen[tid + s]);
            plen[tid] += plen[tid + s];
        }
        __syncthreads();
    }
    if (tid == 0) png_put32(tail + 4, part[0]);
}

}  // namespace nastar
