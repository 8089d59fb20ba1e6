// nastar_png.cuh — PNG decode on the GPU: inflate, unfilter, Adam7 and conversion to L in one launch, bit-equal to
// Pillow's Image.open(f).convert("L") (DESIGN.md §16).
//
// decode_png_kernel: persistent one-warp CTAs take images from an atomic queue (as engine 5 does) and own one
// workspace slot each, of the largest inflated size in the batch.  Per image, the whole warp:
//   inflate   zlib header (CM 8, CINFO <= 7, FCHECK, FDICT 0), stored / fixed / dynamic Huffman blocks into the slot,
//             then the exact inflated length (from IHDR) and the Adler-32.  Every lane runs the same symbol decode on
//             the same bits (uniform loads are broadcasts, so this costs what one lane would); the lanes split the
//             byte copies of stored blocks and matches.  A match of distance d copies out[p+i] = out[p-d + i%d], so
//             overlapping matches (d < length) are one parallel pass too.  Literal/length codes of <= 10 bits and
//             distance codes of <= 8 bits decode with one shared-memory lookup; longer codes walk the canonical
//             code counts bit by bit;
//   unfilter  per scanline of each pass: None; Up in parallel; Sub as a mod-256 warp scan with stride bpp; Average
//             and Paeth one lane per byte of a pixel (bpp lanes), sequential along the row;
//   convert   every pixel of every pass to its place in the H0 x W0 plane: grey 1/2/4 bits scaled to 0..255, 16-bit
//             grey min(v, 255), RGB / RGBA (19595 R + 38470 G + 7471 B + 0x8000) >> 16 of the high bytes, grey+alpha
//             the grey high byte, palette the RGB rule of the PLTE entry ((0, 0, 0) past its end).
// Status per image (0 = decoded): an OR of kPngBad* below; the first error stops that image, and its plane is then
// unspecified.  Every read stays inside the image's input range and slot, every write inside its slot and plane.
#pragma once
#include <cstdint>

#include "../../include/nastar_b200.h"

namespace nastar {

constexpr int kPngThreads = 32;
constexpr int kPngMaxSide = 2048;
constexpr int kPngLitBits = 10;   // literal/length lookup: 1024 entries
constexpr int kPngDistBits = 8;   // distance lookup: 256 entries
constexpr uint16_t kPngSlow = 0xFFFF;

constexpr int kPngBadHeader = 1;
constexpr int kPngBadCode = 2;
constexpr int kPngBadDistance = 4;
constexpr int kPngBadLength = 8;
constexpr int kPngBadAdler = 16;
constexpr int kPngBadFilter = 32;

using PngDesc = nastar_png_desc;   // one image of a decode batch (include/nastar_b200.h)

struct PngArgs {
    const uint8_t* data;
    const PngDesc* desc;
    int B;
    uint8_t* out;
    int32_t* status;
    int32_t* queue;        // zeroed before the launch
    uint8_t* slots;        // gridDim.x slots of slot_bytes
    int64_t slot_bytes;
};

__host__ __device__ inline bool png_legal(int depth, int ct) {
    switch (ct) {
        case 0: return depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16;
        case 3: return depth == 1 || depth == 2 || depth == 4 || depth == 8;
        case 2: case 4: case 6: return depth == 8 || depth == 16;
        default: return false;
    }
}
__host__ __device__ inline int png_channels(int ct) { return ct == 2 ? 3 : ct == 4 ? 2 : ct == 6 ? 4 : 1; }
__host__ __device__ inline int64_t png_row_bytes(int64_t w, int depth, int ct) {
    return (w * depth * png_channels(ct) + 7) / 8;
}
// Adam7 pass k of 7 (k = 0 without interlace): first column / row and steps.  Steps dx = 8,8,4,4,2,2,1 and
// dy = 8,8,8,4,4,2,2; odd passes start at column dx/2, even passes after the first at row dy/2.
__host__ __device__ inline void png_pass(int interlace, int k, int* x0, int* y0, int* dx, int* dy) {
    if (!interlace) { *x0 = *y0 = 0; *dx = *dy = 1; return; }
    *dx = 8 >> (k / 2);
    *dy = k == 0 ? 8 : 8 >> ((k - 1) / 2);
    *x0 = (k & 1) ? *dx / 2 : 0;
    *y0 = (k && !(k & 1)) ? *dy / 2 : 0;
}
// bytes of the inflated stream: every row of every non-empty pass, with its filter byte
__host__ __device__ inline int64_t png_raw_bytes(int W, int H, int depth, int ct, int interlace) {
    int64_t n = 0;
    for (int k = 0; k < (interlace ? 7 : 1); ++k) {
        int x0, y0, dx, dy;
        png_pass(interlace, k, &x0, &y0, &dx, &dy);
        const int64_t pw = (W - x0 + dx - 1) / dx, ph = (H - y0 + dy - 1) / dy;
        if (pw > 0 && ph > 0) n += ph * (1 + png_row_bytes(pw, depth, ct));
    }
    return n;
}

// LSB-first bit reader over [p, p + n); past the end it feeds zeros and `overrun()` turns true
struct PngBits {
    const uint8_t* p;
    int64_t n, pos;
    uint64_t buf;
    int cnt;
    __device__ void refill() {
        while (cnt <= 56) {
            buf |= uint64_t(pos < n ? __ldg(p + pos) : 0) << cnt;
            ++pos;
            cnt += 8;
        }
    }
    __device__ uint32_t bits(int k) {   // k <= 32, after refill() when k > cnt
        const uint32_t v = uint32_t(buf & ((uint64_t(1) << k) - 1));
        buf >>= k;
        cnt -= k;
        return v;
    }
    __device__ uint32_t get(int k) { refill(); return bits(k); }
    __device__ bool overrun() const { return pos * 8 - cnt > n * 8; }
    __device__ int64_t byte_pos() const { return pos - cnt / 8; }   // after align(): the next unread byte
    __device__ void align() { bits(cnt & 7); }
    __device__ void seek(int64_t b) { pos = b; buf = 0; cnt = 0; }
};

struct PngHuff {   // canonical code: counts per length, symbols by (length, value)
    int16_t count[16];
    int16_t symbol[288];
};

struct PngSmem {
    uint16_t lit_lut[1 << kPngLitBits];
    uint16_t dist_lut[1 << kPngDistBits];
    PngHuff lit, dist, clen;
    uint8_t lens[320];
    uint8_t pal_l[256];
    int16_t offs[16];
    int err, maxlen;
};

__constant__ uint8_t kPngClenOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
__constant__ uint16_t kPngLenBase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31,
                                         35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t kPngLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t kPngDistBase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385,
                                          513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};

// Builds `h` (and `lut`, when given) from lens[0, n): 0 = complete, 1 = over-subscribed, 2 = incomplete; the longest
// length goes to *maxlen.  Warp-collective.
__device__ int png_build(PngSmem& s, PngHuff& h, const uint8_t* lens, int n, uint16_t* lut, int lut_bits, int* maxlen) {
    const int lane = threadIdx.x & 31;
    if (lane < 16) h.count[lane] = 0;
    __syncwarp();
    if (lane == 0) {
        for (int i = 0; i < n; ++i) ++h.count[lens[i]];
        int left = 1, ml = 0, res = 0;
        for (int l = 1; l < 16; ++l) {
            left = left * 2 - h.count[l];
            if (left < 0) res = 1;
            if (h.count[l]) ml = l;
        }
        if (!res && left > 0) res = 2;
        s.offs[1] = 0;
        for (int l = 1; l < 15; ++l) s.offs[l + 1] = s.offs[l] + h.count[l];
        for (int i = 0; i < n; ++i)
            if (lens[i]) h.symbol[s.offs[lens[i]]++] = int16_t(i);
        // offs[l] is now the end of length l; rewind it to the start
        for (int l = 1; l < 16; ++l) s.offs[l] -= h.count[l];
        s.err = res;
        s.maxlen = ml;
    }
    __syncwarp();
    const int res = s.err, ml = s.maxlen;
    *maxlen = ml;
    if (lut && res != 1) {
        for (int i = lane; i < (1 << lut_bits); i += 32) lut[i] = kPngSlow;
        __syncwarp();
        // symbol j of length l has code first[l] + (j - offs[l]), first[l] = (first[l-1] + count[l-1]) << 1
        int first = 0;
        for (int l = 1; l <= lut_bits; ++l) {
            first = (first + (l > 1 ? h.count[l - 1] : 0)) << (l > 1 ? 1 : 0);
            for (int j = lane; j < h.count[l]; j += 32) {
                const uint32_t code = uint32_t(first + j);
                const uint32_t rev = __brev(code) >> (32 - l);
                const uint16_t e = uint16_t(h.symbol[s.offs[l] + j] | (l << 9));
                for (int k = 0; k < (1 << (lut_bits - l)); ++k) lut[rev | (k << l)] = e;
            }
        }
        __syncwarp();
    }
    return res;
}

// next symbol of code `h`: the lookup when its entry is resolved, else bit by bit; -1 for a code that is not used
__device__ int png_decode(PngBits& br, const PngHuff& h, const uint16_t* lut, int lut_bits) {
    br.refill();
    if (lut) {
        const uint16_t e = lut[br.buf & ((1u << lut_bits) - 1)];
        if (e != kPngSlow) {
            br.bits(e >> 9);
            return e & 511;
        }
    }
    int code = 0, first = 0, index = 0;
    for (int l = 1; l < 16; ++l) {
        code |= int(br.bits(1));
        const int count = h.count[l];
        if (code - count < first) return h.symbol[index + (code - first)];
        index += count;
        first = (first + count) << 1;
        code <<= 1;
    }
    return -1;
}

__device__ __forceinline__ int png_paeth(int a, int b, int c) {
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

__device__ __forceinline__ uint32_t png_rgb_l(uint32_t r, uint32_t g, uint32_t b) {
    return (19595u * r + 38470u * g + 7471u * b + 0x8000u) >> 16;
}

// level of pixel x of an unfiltered row
__device__ __forceinline__ uint32_t png_level(const uint8_t* row, int x, int depth, int ct, const uint8_t* pal_l) {
    if (depth < 8) {
        const int per = 8 / depth;
        const uint32_t v = (row[x / per] >> (8 - depth * (x % per + 1))) & ((1u << depth) - 1);
        return ct == 3 ? pal_l[v] : v * (depth == 1 ? 255u : depth == 2 ? 85u : 17u);
    }
    const int bs = depth >> 3;   // bytes per sample; the first byte is the high byte
    switch (ct) {
        case 0: {
            if (bs == 1) return row[x];
            const uint32_t v = (uint32_t(row[2 * x]) << 8) | row[2 * x + 1];
            return v < 255u ? v : 255u;
        }
        case 3: return pal_l[row[x]];
        case 4: return row[x * 2 * bs];
        default: {
            const uint8_t* p = row + int64_t(x) * png_channels(ct) * bs;
            return png_rgb_l(p[0], p[bs], p[2 * bs]);
        }
    }
}

// the raw deflate blocks (stored, fixed and dynamic Huffman) that `br` reads from src[0, src_len), inflated into
// raw[0, raw_len), which they must fill exactly; returns the status bits.  Matches read back from `raw`, so no other
// buffer is needed.  Shared by the PNG decode (png_inflate adds the zlib framing) and the .npz reader
// (nastar_inflate.cuh).  Warp-collective.
__device__ int png_inflate_blocks(PngSmem& s, PngBits& br, const uint8_t* src, int64_t src_len, uint8_t* raw,
                                  int64_t raw_len) {
    const int lane = threadIdx.x & 31;
    int64_t op = 0;
    bool last = false;
    while (!last) {
        last = br.get(1);
        const uint32_t type = br.get(2);
        if (type == 0) {
            br.align();
            const uint32_t len = br.get(16), nlen = br.get(16);
            if (br.overrun()) return kPngBadLength;
            if ((len ^ 0xFFFFu) != nlen) return kPngBadCode;
            const int64_t at = br.byte_pos();
            if (at + len > src_len) return kPngBadLength;
            if (op + len > raw_len) return kPngBadLength;
            for (int64_t i = lane; i < len; i += 32) raw[op + i] = __ldg(src + at + i);
            op += len;
            br.seek(at + len);
            __syncwarp();
            continue;
        }
        if (type == 3) return kPngBadCode;
        int ml = 0;
        if (type == 1) {
            for (int i = lane; i < 320; i += 32) s.lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : i < 288 ? 8 : 5;
            __syncwarp();
            png_build(s, s.lit, s.lens, 288, s.lit_lut, kPngLitBits, &ml);
            png_build(s, s.dist, s.lens + 288, 30, s.dist_lut, kPngDistBits, &ml);
        } else {
            const int nlen = int(br.get(5)) + 257, ndist = int(br.get(5)) + 1, ncode = int(br.get(4)) + 4;
            if (nlen > 286 || ndist > 30) return kPngBadCode;
            __syncwarp();
            if (lane < 19) s.lens[kPngClenOrder[lane]] = 0;   // the code-length code's 19 lengths
            __syncwarp();
            for (int i = 0; i < ncode; ++i) {
                const uint8_t v = uint8_t(br.get(3));
                if (lane == 0) s.lens[kPngClenOrder[i]] = v;
            }
            __syncwarp();
            if (png_build(s, s.clen, s.lens, 19, nullptr, 0, &ml) != 0) return kPngBadCode;
            // s.clen holds the code now; the lengths it came from make way for the nlen + ndist code lengths
            __syncwarp();
            for (int i = lane; i < 320; i += 32) s.lens[i] = 0;
            __syncwarp();
            int idx = 0;
            while (idx < nlen + ndist) {
                const int sym = png_decode(br, s.clen, nullptr, 0);
                if (sym < 0) return kPngBadCode;
                if (sym < 16) {
                    if (lane == 0) s.lens[idx] = uint8_t(sym);
                    ++idx;
                    continue;
                }
                int rep, val = 0;
                if (sym == 16) {
                    if (idx == 0) return kPngBadCode;
                    __syncwarp();
                    val = s.lens[idx - 1];
                    rep = 3 + int(br.get(2));
                } else {
                    rep = sym == 17 ? 3 + int(br.get(3)) : 11 + int(br.get(7));
                }
                if (idx + rep > nlen + ndist) return kPngBadCode;
                for (int j = lane; j < rep; j += 32) s.lens[idx + j] = uint8_t(val);
                idx += rep;
                if (br.overrun()) return kPngBadLength;
            }
            __syncwarp();
            if (s.lens[256] == 0) return kPngBadCode;   // no end-of-block code
            // zlib's rules: over-subscribed is an error; incomplete only for one code of length 1 (and no distances)
            int r = png_build(s, s.lit, s.lens, nlen, s.lit_lut, kPngLitBits, &ml);
            if (r == 1 || (r == 2 && !(s.lit.count[1] == 1 && ml == 1))) return kPngBadCode;
            // the distance lengths follow the literal ones; move them down to a fresh start
            uint8_t dl = lane < ndist ? s.lens[nlen + lane] : 0;
            __syncwarp();
            if (lane < 30) s.lens[288 + lane] = lane < ndist ? dl : 0;
            __syncwarp();
            r = png_build(s, s.dist, s.lens + 288, ndist, s.dist_lut, kPngDistBits, &ml);
            if (r == 1 || (r == 2 && ml > 1)) return kPngBadCode;
        }
        if (br.overrun()) return kPngBadLength;
        // symbols of this block
        for (;;) {
            const int sym = png_decode(br, s.lit, s.lit_lut, kPngLitBits);
            if (br.overrun()) return kPngBadLength;
            if (sym < 0 || sym > 285) return kPngBadCode;
            if (sym < 256) {
                if (op >= raw_len) return kPngBadLength;
                if (lane == 0) raw[op] = uint8_t(sym);
                ++op;
                continue;
            }
            if (sym == 256) break;
            const int ls = sym - 257;
            const int len = kPngLenBase[ls] + int(br.get(kPngLenExtra[ls]));
            const int ds = png_decode(br, s.dist, s.dist_lut, kPngDistBits);
            if (ds < 0 || ds > 29) return kPngBadCode;
            const int dist = kPngDistBase[ds] + int(br.get(ds < 4 ? 0 : (ds >> 1) - 1));
            if (br.overrun()) return kPngBadLength;
            if (dist > op) return kPngBadDistance;
            if (op + len > raw_len) return kPngBadLength;
            __syncwarp();   // the literals lane 0 wrote, and earlier copies, are visible to every lane
            for (int i = lane; i < len; i += 32) raw[op + i] = raw[op - dist + (i % dist)];
            __syncwarp();
            op += len;
        }
    }
    return op != raw_len ? kPngBadLength : 0;
}

// inflate the zlib stream of `d` into raw[0, raw_len); returns the status bits
__device__ int png_inflate(PngSmem& s, const uint8_t* src, int64_t src_len, uint8_t* raw, int64_t raw_len) {
    const int lane = threadIdx.x & 31;
    PngBits br{src, src_len, 0, 0, 0};
    const uint32_t cmf = br.get(8), flg = br.get(8);
    if (br.overrun() || (cmf & 15) != 8 || (cmf >> 4) > 7 || ((cmf << 8) | flg) % 31 != 0 || (flg & 32))
        return kPngBadHeader;
    const int st = png_inflate_blocks(s, br, src, src_len, raw, raw_len);
    if (st) return st;
    br.align();
    const uint32_t b0 = br.get(8), b1 = br.get(8), b2 = br.get(8), b3 = br.get(8);
    if (br.overrun()) return kPngBadLength;
    const uint32_t want = (b0 << 24) | (b1 << 16) | (b2 << 8) | b3;
    // Adler-32: A = 1 + sum d_i, B = n + sum (n - i) d_i, both mod 65521
    __syncwarp();
    uint64_t a = 0, b = 0;
    for (int64_t i = lane; i < raw_len; i += 32) {
        const uint32_t v = raw[i];
        a += v;
        b += uint64_t(raw_len - i) * v;
    }
    a %= 65521u;
    b %= 65521u;
    for (int o = 16; o; o >>= 1) {
        a += __shfl_xor_sync(0xFFFFFFFFu, a, o);
        b += __shfl_xor_sync(0xFFFFFFFFu, b, o);
    }
    const uint32_t A = uint32_t((1 + a) % 65521u), Bs = uint32_t((uint64_t(raw_len) % 65521u + b) % 65521u);
    return ((Bs << 16) | A) == want ? 0 : kPngBadAdler;
}

// unfilter the rows of one pass in place; returns kPngBadFilter for a filter byte above 4
__device__ int png_unfilter(uint8_t* raw, int64_t rb, int ph, int bpp) {
    const int lane = threadIdx.x & 31;
    for (int y = 0; y < ph; ++y) {
        uint8_t* row = raw + int64_t(y) * (rb + 1);
        const uint8_t* prev = y ? row - rb : nullptr;   // the previous row's bytes (after its filter byte)
        const int f = row[0];
        uint8_t* d = row + 1;
        if (f > 4) return kPngBadFilter;
        // a first row's up neighbours are 0: Up is then None, and Paeth is Sub
        const int g = prev ? f : (f == 2 ? 0 : f == 4 ? 1 : f);
        if (g == 2) {
            for (int64_t i = lane; i < rb; i += 32) d[i] = uint8_t(d[i] + prev[i]);
        } else if (g == 1) {
            // Sub: a mod-256 inclusive scan of each residue class mod bpp, 32 bytes at a time; a lane's carry is the
            // last byte of its class in the previous 32
            for (int64_t c = 0; c < rb; c += 32) {
                const int64_t i = c + lane;
                uint32_t v = i < rb ? d[i] : 0;
                for (int o = bpp; o < 32; o <<= 1) {
                    const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, v, o);
                    if (lane >= o) v += u;
                }
                if (c) v += d[c - bpp + lane % bpp];
                __syncwarp();
                if (i < rb) d[i] = uint8_t(v);
                __syncwarp();
            }
        } else if (g >= 3 && lane < bpp) {
            // Average and Paeth: one lane per byte of a pixel, sequential along the row
            for (int64_t i = lane; i < rb; i += bpp) {
                const int a = i >= bpp ? d[i - bpp] : 0, b = prev ? prev[i] : 0, c = (prev && i >= bpp) ? prev[i - bpp] : 0;
                d[i] = uint8_t(d[i] + (g == 3 ? (a + b) >> 1 : png_paeth(a, b, c)));
            }
        }
        __syncwarp();
    }
    return 0;
}

__global__ void __launch_bounds__(kPngThreads) decode_png_kernel(PngArgs a) {
    __shared__ PngSmem s;
    const int lane = threadIdx.x & 31;
    uint8_t* raw = a.slots + int64_t(blockIdx.x) * a.slot_bytes;
    for (;;) {
        int img = 0;
        if (lane == 0) img = atomicAdd(a.queue, 1);
        img = __shfl_sync(0xFFFFFFFFu, img, 0);
        if (img >= a.B) break;
        const PngDesc d = a.desc[img];
        const int W = d.W0, H = d.H0, depth = d.bit_depth, ct = d.color_type, il = d.interlace;
        const int64_t raw_len = png_raw_bytes(W, H, depth, ct, il);
        int st = png_inflate(s, a.data + d.in_off, d.in_len, raw, raw_len);
        __syncwarp();
        const int bpp = depth * png_channels(ct) >= 8 ? depth * png_channels(ct) / 8 : 1;
        int64_t off = 0;
        for (int k = 0; k < (il ? 7 : 1) && !st; ++k) {
            int x0, y0, dx, dy;
            png_pass(il, k, &x0, &y0, &dx, &dy);
            const int pw = (W - x0 + dx - 1) / dx, ph = (H - y0 + dy - 1) / dy;
            if (pw <= 0 || ph <= 0) continue;
            const int64_t rb = png_row_bytes(pw, depth, ct);
            st = png_unfilter(raw + off, rb, ph, bpp);
            off += ph * (rb + 1);
        }
        if (!st) {
            if (ct == 3) {
                const uint8_t* pal = a.data + d.plte_off;
                const int n = int(d.plte_len < 768 ? d.plte_len : 768) / 3;
                for (int i = lane; i < 256; i += 32)
                    s.pal_l[i] = i < n ? uint8_t(png_rgb_l(pal[3 * i], pal[3 * i + 1], pal[3 * i + 2])) : 0;
            }
            __syncwarp();
            uint8_t* plane = a.out + d.out_off;
            off = 0;
            for (int k = 0; k < (il ? 7 : 1); ++k) {
                int x0, y0, dx, dy;
                png_pass(il, k, &x0, &y0, &dx, &dy);
                const int pw = (W - x0 + dx - 1) / dx, ph = (H - y0 + dy - 1) / dy;
                if (pw <= 0 || ph <= 0) continue;
                const int64_t rb = png_row_bytes(pw, depth, ct);
                for (int64_t p = lane; p < int64_t(pw) * ph; p += 32) {
                    const int y = int(p / pw), x = int(p - int64_t(y) * pw);
                    plane[int64_t(y0 + y * dy) * W + x0 + x * dx] =
                        uint8_t(png_level(raw + off + y * (rb + 1) + 1, x, depth, ct, s.pal_l));
                }
                off += ph * (rb + 1);
            }
        }
        if (lane == 0) a.status[img] = st;
        __syncwarp();
    }
}

}  // namespace nastar
