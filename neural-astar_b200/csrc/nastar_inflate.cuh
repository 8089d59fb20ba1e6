// nastar_inflate.cuh — zip members (stored or raw deflate) to their bytes, with the CRC-32 of each, in one launch: the
// device half of the .npz reader (DESIGN.md §23).
//
// inflate_kernel: persistent one-warp CTAs take members from an atomic queue (as decode_png_kernel takes images).  Per
// member, the whole warp:
//   inflate  method 8: png_inflate_blocks (nastar_png.cuh), straight into the member's output range, which it must
//            fill exactly; matches read back from the output, so no workspace slot is needed.  Method 0: a copy;
//   CRC-32   lane l over the l-th 32nd of the output, joined in lane order with crc(A||B) = shift(crc(A), |B|) ^
//            crc(B) (nastar_deflate.cuh's df_crc_combine).
// Status per member (0 = inflated): the kPngBad* bits of png_inflate_blocks; the first error stops that member, and its
// output and CRC are then unspecified.  Every read stays inside the member's input range, every write inside its
// output range.
#pragma once
#include <cstdint>

#include "../../include/nastar_b200.h"
#include "nastar_deflate.cuh"
#include "nastar_png.cuh"

namespace nastar {

constexpr int kInflateThreads = 32;

using InflateDesc = nastar_inflate_desc;   // one member of an inflate batch (include/nastar_b200.h)

struct InflateArgs {
    const uint8_t* data;
    const InflateDesc* desc;
    int M;
    uint8_t* out;
    int32_t* status;
    uint32_t* crc;
    int32_t* queue;   // zeroed before the launch
};

__global__ void __launch_bounds__(kInflateThreads) inflate_kernel(InflateArgs a) {
    __shared__ PngSmem s;
    __shared__ uint32_t crc_table[256];
    __shared__ uint32_t x2n[32];
    const int lane = threadIdx.x & 31;
    for (int i = lane; i < 256; i += 32) {
        uint32_t c = uint32_t(i);
        for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0xEDB88320u : c >> 1;
        crc_table[i] = c;
    }
    if (lane == 0) {
        uint32_t p = 1u << 30;   // x^1
        for (int k = 0; k < 32; ++k) {
            x2n[k] = p;
            p = df_multmodp(p, p);
        }
    }
    __syncwarp();
    for (;;) {
        int m = 0;
        if (lane == 0) m = atomicAdd(a.queue, 1);
        m = __shfl_sync(0xFFFFFFFFu, m, 0);
        if (m >= a.M) break;
        const InflateDesc d = a.desc[m];
        const uint8_t* src = a.data + d.in_off;
        uint8_t* out = a.out + d.out_off;
        const int64_t n = d.out_len;
        int st = 0;
        if (d.method == 0) {
            for (int64_t i = lane; i < n; i += 32) out[i] = __ldg(src + i);   // in_len == out_len (host check)
        } else {
            PngBits br{src, d.in_len, 0, 0, 0};
            st = png_inflate_blocks(s, br, src, d.in_len, out, n);
        }
        __syncwarp();   // every lane's bytes, and lane 0's literals, are visible to the lane that reads them
        uint32_t crc = 0;
        if (!st) {
            const int64_t per = (n + 31) / 32;
            const int64_t b0 = lane * per < n ? lane * per : n, b1 = b0 + per < n ? b0 + per : n;
            uint32_t c = 0xFFFFFFFFu;
            for (int64_t i = b0; i < b1; ++i) c = crc_table[(c ^ out[i]) & 0xFF] ^ (c >> 8);
            c ^= 0xFFFFFFFFu;
            for (int l = 0; l < 32; ++l) {   // every lane folds the same 32 parts in lane order
                const uint32_t part = __shfl_sync(0xFFFFFFFFu, c, l);
                const int64_t len = __shfl_sync(0xFFFFFFFFu, b1 - b0, l);
                if (len) crc = df_crc_combine(x2n, crc, part, uint64_t(len));
            }
        }
        if (lane == 0) {
            a.status[m] = st;
            a.crc[m] = crc;
        }
        __syncwarp();
    }
}

}  // namespace nastar
