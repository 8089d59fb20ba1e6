// nastar_deflate.cuh — chunked deflate of .npz members on the GPU (DESIGN.md §18); tests check its bytes against a
// sequential C restatement of every rule below.
//
// A member is its .npy header (one chunk) followed by its data cut into kDeflateChunk-byte chunks.  Each chunk is
// compressed alone: no match reaches before its start, so chunks are independent.  It becomes one dynamic-Huffman
// block, or stored blocks (<= 65 535 bytes each) when those are not larger; a chunk that is not its member's last
// ends with an empty stored block (zlib's Z_FULL_FLUSH), so it ends byte-aligned and the chunks join into one raw
// deflate stream.  Only the member's last chunk sets BFINAL.
//
// deflate_kernel: persistent CTAs claim chunks in order from an atomic counter.  Per chunk, in the CTA's workspace
// slot:
//   chains   warp 0 walks the chunk 32 positions at a time; __match_any_sync finds equal 3-byte hashes inside the
//            step and a shared-memory head table (15-bit hash) the latest one before it; prev[p] = the distance to
//            the previous position with p's hash (0: none within 32 KiB);
//   matches  every thread takes positions: up to kDeflateChain chain candidates, the longest match (<= 258, ties
//            to the nearest), a length-3 match only within 4 KiB;
//   parse    thread 0: lazy, a match is deferred to a literal when the next position has a longer one and this one
//            is shorter than kDeflateLazy; the literal/length and distance histograms on the way;
//   codes    thread 0: Huffman lengths limited to 15 bits (code-length codes to 7), every code set complete;
//   emit     the block's bits: each token's bit count, a block-wide exclusive scan for its bit offset, then atomicOr
//            into the slot's zeroed output words; stored blocks are copied;
//   CRC-32   every thread over its share of the chunk, joined by thread 0 with crc(A||B) = shift(crc(A), |B|) ^ crc(B);
//   place    the CTA waits for the previous chunk's published (end offset, member start, running CRC), copies its
//            bytes to `out` at that offset, and publishes its own.  Chunks are claimed in order, so the chunk a CTA
//            waits for belongs to a CTA that is already running: the wait cannot deadlock.
// Every loop is bounded by the chunk's length; reads stay inside the member's header and data, writes inside the
// slot and the member's output range.
#pragma once
#include <cstdint>
#include <cub/block/block_scan.cuh>

#include "../../include/nastar_b200.h"

namespace nastar {

constexpr int kDeflateThreads = 512;
constexpr int64_t kDeflateChunk = 256 * 1024;   // DESIGN.md §18: 1.005x the single-stream size at zlib level 6
constexpr int kDeflateHashBits = 15;
constexpr int kDeflateWindow = 32768;
constexpr int kDeflateChain = 128;
constexpr int kDeflateLazy = 32;
constexpr int kDeflateTooFar = 4096;
constexpr int kDeflateRing = 64;   // publication ring; any size >= 2 is safe (see deflate_kernel)

using DeflateDesc = nastar_deflate_desc;

// worst case of one chunk of n bytes: its stored form plus the empty stored block
__host__ __device__ inline int64_t deflate_chunk_bound(int64_t n) {
    return n + 5 * (n > 0 ? (n + 65534) / 65535 : 1) + 5;
}
__host__ __device__ inline int64_t deflate_member_chunks(int64_t data_len) {
    return 1 + (data_len + kDeflateChunk - 1) / kDeflateChunk;
}
// worst case of a member's stream: its header chunk and its data chunks
__host__ __device__ inline int64_t deflate_member_bound(int64_t head_len, int64_t data_len) {
    const int64_t full = data_len / kDeflateChunk, rest = data_len % kDeflateChunk;
    return deflate_chunk_bound(head_len) + full * deflate_chunk_bound(kDeflateChunk) +
           (rest ? deflate_chunk_bound(rest) : 0);
}
// bytes of one workspace slot: prev u16, match u32 and token u32 per position, and the output words
constexpr int64_t kDeflateOutWords = (kDeflateChunk + 5 * 5 + 5 + 8) / 4;
constexpr int64_t kDeflateSlotBytes = kDeflateChunk * 10 + kDeflateOutWords * 4;

struct DeflatePub {
    unsigned long long end, mstart;   // end of this chunk's bytes in `out`; start of its member's stream
    uint32_t crc, tag;                // the member's CRC-32 so far; chunk index + 1 once published
};

struct DeflateArgs {
    const DeflateDesc* desc;
    int32_t M;
    int64_t chunks;
    uint8_t* out;
    int64_t* out_off;
    int64_t* out_len;
    uint32_t* crc;
    int32_t* counter;
    DeflatePub* ring;
    unsigned char* slots;
};

struct DeflateSmem {
    int32_t head[1 << kDeflateHashBits];
    uint32_t crc_table[256];
    uint32_t x2n[32];
    uint32_t lf[286], df[30], cf[19];
    uint8_t lens[286 + 30], cll[19];
    uint16_t lc[286], dc[30], clc[19];
    uint32_t items[286 + 30];
    int32_t sym[286], parent[2 * 286], depth[2 * 286];
    unsigned long long w[2 * 286];
    uint32_t part_crc[kDeflateThreads];
    uint32_t warp_bits[kDeflateThreads / 32];
    uint8_t seq[286 + 30];
    int32_t count[16], next[16];
    int64_t T;
    int64_t chunk;
    int32_t nitems, hlit, hdist, hclen, dynamic;
    unsigned long long bits, nbytes, base;
    typename cub::BlockScan<uint32_t, kDeflateThreads>::TempStorage scan;
};

__constant__ int16_t kDfLenBase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31,
                                       35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ int8_t kDfLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5,
                                       0};
__constant__ int16_t kDfDistBase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769,
                                        1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ int8_t kDfDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11,
                                        11, 12, 12, 13, 13};
__constant__ int8_t kDfClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
__constant__ int8_t kDfClExtra[19] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 3, 7};

__device__ inline int df_len_code(int len) {
    int c = 0;
    while (c < 28 && kDfLenBase[c + 1] <= len) ++c;
    return c;
}
__device__ inline int df_dist_code(int dist) {
    int c = 0;
    while (c < 29 && kDfDistBase[c + 1] <= dist) ++c;
    return c;
}
__device__ inline uint32_t df_hash3(const uint8_t* p) {
    const uint32_t v = uint32_t(p[0]) | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16);
    return (v * 2654435761u) >> (32 - kDeflateHashBits);
}

// a * b modulo the CRC-32 polynomial, reflected (bit 31 is x^0)
__device__ inline uint32_t df_multmodp(uint32_t a, uint32_t b) {
    uint32_t m = 1u << 31, p = 0;
    for (int i = 0; i < 32; ++i, m >>= 1) {
        if (a & m) p ^= b;
        b = (b & 1) ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}
// crc(A || B) from crc(A), crc(B) and |B|; x2n[k] = x^(2^k)
__device__ inline uint32_t df_crc_combine(const uint32_t* x2n, uint32_t a, uint32_t b, uint64_t len_b) {
    uint32_t p = 1u << 31;
    for (int k = 3; len_b; len_b >>= 1, ++k)
        if (len_b & 1) p = df_multmodp(x2n[k & 31], p);
    return df_multmodp(p, a) ^ b;
}

// Huffman lengths of freq[0..n) limited to maxbits: symbols ranked by (freq, index), a two-queue tree (a leaf before
// an internal node of equal weight), depths clamped and the Kraft sum repaired by lengthening the deepest code below
// the limit, lengths handed out by rank; fewer than two used symbols: the used one and the lowest unused ones get 1
__device__ __noinline__ void df_build_lengths(DeflateSmem& s, const uint32_t* freq, int n, int maxbits, uint8_t* len) {
    int m = 0;
    for (int i = 0; i < n; ++i) {
        len[i] = 0;
        if (freq[i]) s.sym[m++] = i;
    }
    if (m < 2) {
        for (int i = 0; i < n && m < 2; ++i)
            if (!freq[i]) s.sym[m++] = i;
        len[s.sym[0]] = 1;
        len[s.sym[1]] = 1;
        return;
    }
    for (int i = 1; i < m; ++i) {
        const int sy = s.sym[i];
        int j = i - 1;
        while (j >= 0 && (freq[s.sym[j]] > freq[sy] || (freq[s.sym[j]] == freq[sy] && s.sym[j] > sy))) {
            s.sym[j + 1] = s.sym[j];
            --j;
        }
        s.sym[j + 1] = sy;
    }
    for (int i = 0; i < m; ++i) s.w[i] = freq[s.sym[i]];
    int leaf = 0, node = m, next = m;
    while (next < 2 * m - 1) {
        int pick[2];
        for (int k = 0; k < 2; ++k) {
            if (leaf < m && (node >= next || s.w[leaf] <= s.w[node])) pick[k] = leaf++;
            else pick[k] = node++;
        }
        s.w[next] = s.w[pick[0]] + s.w[pick[1]];
        s.parent[pick[0]] = s.parent[pick[1]] = next;
        ++next;
    }
    s.depth[2 * m - 2] = 0;
    for (int i = 2 * m - 3; i >= 0; --i) s.depth[i] = s.depth[s.parent[i]] + 1;
    int32_t* count = s.count;
    for (int b = 0; b < 16; ++b) count[b] = 0;
    for (int i = 0; i < m; ++i) count[s.depth[i] > maxbits ? maxbits : s.depth[i]]++;
    uint32_t total = 0;
    for (int b = 1; b <= maxbits; ++b) total += uint32_t(count[b]) << (maxbits - b);
    while (total > (1u << maxbits)) {
        count[maxbits]--;
        for (int b = maxbits - 1; b > 0; --b)
            if (count[b]) {
                count[b]--;
                count[b + 1] += 2;
                break;
            }
        total--;
    }
    int r = 0;
    for (int b = maxbits; b >= 1; --b)
        for (int k = 0; k < count[b]; ++k) len[s.sym[r++]] = uint8_t(b);
}

__device__ __noinline__ void df_build_codes(DeflateSmem& s, const uint8_t* len, int n, uint16_t* code) {
    int32_t *count = s.count, *next = s.next;
    for (int b = 0; b < 16; ++b) count[b] = 0;
    for (int i = 0; i < n; ++i) count[len[i]]++;
    count[0] = 0;
    int c = 0;
    next[0] = 0;
    for (int b = 1; b < 16; ++b) {
        c = (c + count[b - 1]) << 1;
        next[b] = c;
    }
    for (int i = 0; i < n; ++i) {
        if (!len[i]) {
            code[i] = 0;
            continue;
        }
        const uint32_t v = uint32_t(next[len[i]]++);
        code[i] = uint16_t(__brev(v) >> (32 - len[i]));
    }
}

// the code lengths' run-length coding (16 repeats a non-zero length, 17 / 18 runs of zeros): items sym | extra << 8
__device__ __noinline__ int df_rle(const uint8_t* L, int total, uint32_t* items) {
    int k = 0, i = 0;
    while (i < total) {
        const int v = L[i];
        int run = 1;
        while (i + run < total && L[i + run] == v) ++run;
        if (v == 0) {
            while (run >= 11) {
                const int r = run > 138 ? 138 : run;
                items[k++] = 18u | uint32_t(r - 11) << 8;
                run -= r;
                i += r;
            }
            if (run >= 3) {
                items[k++] = 17u | uint32_t(run - 3) << 8;
                i += run;
                run = 0;
            }
        } else {
            items[k++] = uint32_t(v);
            ++i;
            --run;
            while (run >= 3) {
                const int r = run > 6 ? 6 : run;
                items[k++] = 16u | uint32_t(r - 3) << 8;
                run -= r;
                i += r;
            }
        }
        for (; run > 0; --run, ++i) items[k++] = uint32_t(v);
    }
    return k;
}

// v (< 2^n, n <= 32) at bit `pos` of the zeroed little-endian words
__device__ inline void df_put(uint32_t* words, uint64_t pos, uint32_t v, int n) {
    if (n == 0) return;
    const uint64_t w = pos >> 5;
    const int sh = int(pos & 31);
    atomicOr(&words[w], v << sh);
    if (sh + n > 32) atomicOr(&words[w + 1], v >> (32 - sh));
}

// bits of token t and its fields: (code, len) of the symbol, the length extra, the distance code, the distance extra
__device__ inline uint32_t df_token_bits(const DeflateSmem& s, uint32_t t) {
    if (!(t & 0x80000000u)) return s.lens[t];
    const int lcode = df_len_code(int((t >> 16) & 0x1ff)), d = df_dist_code(int(t & 0xffff) + 1);
    return s.lens[257 + lcode] + kDfLenExtra[lcode] + s.lens[286 + d] + kDfDistExtra[d];
}
__device__ inline void df_emit_token(const DeflateSmem& s, uint32_t* words, uint64_t pos, uint32_t t) {
    if (!(t & 0x80000000u)) {
        df_put(words, pos, s.lc[t], s.lens[t]);
        return;
    }
    const int len = int((t >> 16) & 0x1ff), dist = int(t & 0xffff) + 1;
    const int lcode = df_len_code(len), d = df_dist_code(dist);
    df_put(words, pos, s.lc[257 + lcode], s.lens[257 + lcode]);
    pos += s.lens[257 + lcode];
    df_put(words, pos, uint32_t(len - kDfLenBase[lcode]), kDfLenExtra[lcode]);
    pos += kDfLenExtra[lcode];
    df_put(words, pos, s.dc[d], s.lens[286 + d]);
    pos += s.lens[286 + d];
    df_put(words, pos, uint32_t(dist - kDfDistBase[d]), kDfDistExtra[d]);
}

__global__ void __launch_bounds__(kDeflateThreads, 1) deflate_kernel(DeflateArgs a) {
    extern __shared__ __align__(16) unsigned char df_smem_raw[];
    DeflateSmem& s = *reinterpret_cast<DeflateSmem*>(df_smem_raw);
    const int tid = threadIdx.x, lane = tid & 31;
    unsigned char* slot = a.slots + int64_t(blockIdx.x) * kDeflateSlotBytes;
    uint16_t* prev = reinterpret_cast<uint16_t*>(slot);
    uint32_t* match = reinterpret_cast<uint32_t*>(slot + kDeflateChunk * 2);
    uint32_t* tok = reinterpret_cast<uint32_t*>(slot + kDeflateChunk * 6);
    uint32_t* words = reinterpret_cast<uint32_t*>(slot + kDeflateChunk * 10);
    uint8_t* obytes = reinterpret_cast<uint8_t*>(words);

    for (int i = tid; i < 256; i += kDeflateThreads) {
        uint32_t c = uint32_t(i);
        for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0xEDB88320u : c >> 1;
        s.crc_table[i] = c;
    }
    if (tid == 0) {
        uint32_t p = 1u << 30;   // x^1
        for (int k = 0; k < 32; ++k) {
            s.x2n[k] = p;
            p = df_multmodp(p, p);
        }
    }
    for (;;) {
        if (tid == 0) s.chunk = atomicAdd(a.counter, 1);
        __syncthreads();
        const int64_t k = s.chunk;
        if (k >= a.chunks) break;
        // the member: the last descriptor whose first chunk is <= k
        int lo = 0, hi = a.M - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (a.desc[mid].chunk0 <= k) lo = mid;
            else hi = mid - 1;
        }
        const DeflateDesc& d = a.desc[lo];
        const int64_t j = k - d.chunk0;
        const bool final = j == deflate_member_chunks(d.data_len) - 1;
        const uint8_t* in;
        int64_t n;
        if (j == 0) {
            in = d.head;
            n = d.head_len;
        } else {
            const int64_t off = (j - 1) * kDeflateChunk;
            in = d.data + off;
            n = d.data_len - off < kDeflateChunk ? d.data_len - off : kDeflateChunk;
        }

        // chains
        for (int i = tid; i < (1 << kDeflateHashBits); i += kDeflateThreads) s.head[i] = -1;
        for (int64_t i = tid; i < kDeflateOutWords; i += kDeflateThreads) words[i] = 0;
        __syncthreads();
        if (tid < 32) {
            for (int64_t base = 0; base + 3 <= n; base += 32) {
                const int64_t p = base + lane;
                const bool valid = p + 3 <= n;
                const uint32_t h = valid ? df_hash3(in + p) : 0;
                const uint32_t key = valid ? h : 0x80000000u | uint32_t(lane);
                const uint32_t peers = __match_any_sync(0xffffffffu, key);
                const uint32_t lower = peers & ((1u << lane) - 1u);
                int64_t q = -1;
                if (valid) q = lower ? base + (31 - __clz(lower)) : s.head[h];
                __syncwarp();
                if (valid) {
                    prev[p] = (q >= 0 && p - q <= kDeflateWindow) ? uint16_t(p - q) : uint16_t(0);
                    if ((peers >> lane) == 1u) s.head[h] = int32_t(p);
                }
                __syncwarp();
            }
        }
        __syncthreads();

        // matches
        for (int64_t p = tid; p < n; p += kDeflateThreads) {
            uint32_t m = 0;
            if (p + 3 <= n) {
                const int lim = n - p < 258 ? int(n - p) : 258;
                int best = 0, bestd = 0;
                int64_t q = p;
                for (int c = 0; c < kDeflateChain && prev[q]; ++c) {
                    q -= prev[q];
                    if (p - q > kDeflateWindow) break;
                    if (in[q + best] != in[p + best]) continue;
                    int l = 0;
                    while (l < lim && in[q + l] == in[p + l]) ++l;
                    if (l > best) {
                        best = l;
                        bestd = int(p - q);
                        if (l == lim) break;
                    }
                }
                if (best >= 3 && !(best == 3 && bestd > kDeflateTooFar)) m = uint32_t(best) << 16 | uint32_t(bestd - 1);
            }
            match[p] = m;
        }
        for (int i = tid; i < 286; i += kDeflateThreads) s.lf[i] = 0;
        if (tid < 30) s.df[tid] = 0;
        if (tid < 19) s.cf[tid] = 0;
        // CRC-32 of this thread's share
        {
            const int64_t share = (n + kDeflateThreads - 1) / kDeflateThreads;
            const int64_t b0 = int64_t(tid) * share < n ? int64_t(tid) * share : n;
            const int64_t b1 = b0 + share < n ? b0 + share : n;
            uint32_t c = 0xffffffffu;
            for (int64_t i = b0; i < b1; ++i) c = s.crc_table[(c ^ in[i]) & 0xff] ^ (c >> 8);
            s.part_crc[tid] = c ^ 0xffffffffu;
        }
        __syncthreads();

        // parse, histograms, codes, header (thread 0)
        if (tid == 0) {
            int64_t T = 0;
            for (int64_t p = 0; p < n;) {
                const uint32_t m = match[p];
                const int l = int(m >> 16);
                if (l >= 3 && !(l < kDeflateLazy && p + 1 < n && int(match[p + 1] >> 16) > l)) {
                    tok[T++] = 0x80000000u | m;
                    s.lf[257 + df_len_code(l)]++;
                    s.df[df_dist_code(int(m & 0xffff) + 1)]++;
                    p += l;
                } else {
                    tok[T++] = in[p];
                    s.lf[in[p]]++;
                    p += 1;
                }
            }
            s.T = T;
            s.lf[256] = 1;
            df_build_lengths(s, s.lf, 286, 15, s.lens);
            df_build_lengths(s, s.df, 30, 15, s.lens + 286);
            int hlit = 286, hdist = 30;
            while (hlit > 257 && !s.lens[hlit - 1]) --hlit;
            while (hdist > 1 && !s.lens[286 + hdist - 1]) --hdist;
            for (int i = 0; i < hlit; ++i) s.seq[i] = s.lens[i];
            for (int i = 0; i < hdist; ++i) s.seq[hlit + i] = s.lens[286 + i];
            const int nitems = df_rle(s.seq, hlit + hdist, s.items);
            for (int i = 0; i < nitems; ++i) s.cf[s.items[i] & 0xff]++;
            df_build_lengths(s, s.cf, 19, 7, s.cll);
            int hclen = 19;
            while (hclen > 4 && !s.cll[kDfClOrder[hclen - 1]]) --hclen;
            df_build_codes(s, s.lens, 286, s.lc);
            df_build_codes(s, s.lens + 286, 30, s.dc);
            df_build_codes(s, s.cll, 19, s.clc);
            uint64_t hbits = 3 + 14 + 3 * uint64_t(hclen);
            for (int i = 0; i < nitems; ++i) hbits += s.cll[s.items[i] & 0xff] + kDfClExtra[s.items[i] & 0xff];
            s.nitems = nitems;
            s.hlit = hlit;
            s.hdist = hdist;
            s.hclen = hclen;
            s.bits = hbits;
        }
        __syncthreads();
        // the tokens' bits
        {
            uint32_t mine = 0;
            for (int64_t t = tid; t < s.T; t += kDeflateThreads) mine += df_token_bits(s, tok[t]);
            for (int w = 16; w >= 1; w >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, w);
            if (lane == 0) s.warp_bits[tid >> 5] = mine;
            __syncthreads();
            if (tid == 0) {
                unsigned long long b = s.bits;
                for (int w = 0; w < kDeflateThreads / 32; ++w) b += s.warp_bits[w];
                b += s.lens[256];
                s.bits = b;
                const int64_t nstored = n > 0 ? (n + 65534) / 65535 : 1;
                const int64_t stored_bytes = n + 5 * nstored + (final ? 0 : 5);
                const int64_t dyn_bytes = final ? int64_t((b + 7) / 8) : int64_t((b + 3 + 7) / 8) + 4;
                s.dynamic = dyn_bytes < stored_bytes;
                s.nbytes = s.dynamic ? dyn_bytes : stored_bytes;
            }
            __syncthreads();
        }
        if (s.dynamic) {
            if (tid == 0) {
                uint64_t pos = 0;
                df_put(words, pos, final ? 1u : 0u, 1); pos += 1;
                df_put(words, pos, 2u, 2); pos += 2;
                df_put(words, pos, uint32_t(s.hlit - 257), 5); pos += 5;
                df_put(words, pos, uint32_t(s.hdist - 1), 5); pos += 5;
                df_put(words, pos, uint32_t(s.hclen - 4), 4); pos += 4;
                for (int i = 0; i < s.hclen; ++i, pos += 3) df_put(words, pos, s.cll[kDfClOrder[i]], 3);
                for (int i = 0; i < s.nitems; ++i) {
                    const int sy = int(s.items[i] & 0xff);
                    df_put(words, pos, s.clc[sy], s.cll[sy]);
                    pos += s.cll[sy];
                    df_put(words, pos, s.items[i] >> 8, kDfClExtra[sy]);
                    pos += kDfClExtra[sy];
                }
                s.base = pos;
            }
            __syncthreads();
            using Scan = cub::BlockScan<uint32_t, kDeflateThreads>;
            for (int64_t t0 = 0; t0 < s.T; t0 += kDeflateThreads) {
                const int64_t t = t0 + tid;
                const uint32_t tk = t < s.T ? tok[t] : 0u;
                const uint32_t nb = t < s.T ? df_token_bits(s, tk) : 0u;
                uint32_t off, tile;
                Scan(s.scan).ExclusiveSum(nb, off, tile);
                const unsigned long long base = s.base;
                if (t < s.T) df_emit_token(s, words, base + off, tk);
                __syncthreads();
                if (tid == 0) s.base = base + tile;
                __syncthreads();
            }
            if (tid == 0) {
                uint64_t pos = s.base;
                df_put(words, pos, s.lc[256], s.lens[256]);
                pos += s.lens[256];
                if (!final) {
                    pos += 3;   // the empty stored block's header: 000
                    pos = (pos + 7) & ~uint64_t(7);
                    df_put(words, pos, 0xffff0000u, 32);
                }
            }
        } else {
            const int64_t nstored = n > 0 ? (n + 65534) / 65535 : 1;
            for (int64_t b = tid; b < nstored; b += kDeflateThreads) {
                const int64_t off = b * 65535, len = n - off < 65535 ? n - off : 65535;
                uint8_t* o = obytes + b * 65540;
                o[0] = (final && b == nstored - 1) ? 1 : 0;
                o[1] = uint8_t(len);
                o[2] = uint8_t(len >> 8);
                o[3] = uint8_t(~len);
                o[4] = uint8_t(~len >> 8);
            }
            for (int64_t i = tid; i < n; i += kDeflateThreads) obytes[(i / 65535) * 65540 + 5 + i % 65535] = in[i];
            if (!final && tid == 0) {
                uint8_t* o = obytes + nstored * 5 + n;
                o[0] = 0;
                o[1] = 0;
                o[2] = 0;
                o[3] = 0xff;
                o[4] = 0xff;
            }
        }
        __syncthreads();

        // place: wait for chunk k-1, copy, publish
        if (tid == 0) {
            uint32_t c = 0;
            for (int i = 0; i < kDeflateThreads; ++i) {
                const int64_t share = (n + kDeflateThreads - 1) / kDeflateThreads;
                const int64_t b0 = int64_t(i) * share < n ? int64_t(i) * share : n;
                const int64_t b1 = b0 + share < n ? b0 + share : n;
                if (b1 > b0) c = df_crc_combine(s.x2n, c, s.part_crc[i], uint64_t(b1 - b0));
            }
            unsigned long long end = 0, mstart = 0;
            uint32_t mcrc = 0;
            if (k > 0) {
                volatile DeflatePub* pub = a.ring + (k - 1) % kDeflateRing;
                while (pub->tag != uint32_t(k)) {
                }
                __threadfence();
                end = pub->end;
                mstart = pub->mstart;
                mcrc = pub->crc;
            }
            if (j == 0) {
                mstart = end + uint64_t(d.gap);
                mcrc = c;
            } else {
                mcrc = df_crc_combine(s.x2n, mcrc, c, uint64_t(n));
            }
            s.base = j == 0 ? mstart : end;
            s.bits = mstart;
            s.part_crc[0] = mcrc;
        }
        __syncthreads();
        const unsigned long long dst = s.base, nb = s.nbytes;
        for (unsigned long long i = tid; i < nb; i += kDeflateThreads) a.out[dst + i] = obytes[i];
        __threadfence();
        __syncthreads();
        if (tid == 0) {
            const unsigned long long mstart = s.bits;
            volatile DeflatePub* pub = a.ring + k % kDeflateRing;
            pub->end = dst + nb;
            pub->mstart = mstart;
            pub->crc = s.part_crc[0];
            if (final) {
                a.out_off[lo] = int64_t(mstart);
                a.out_len[lo] = int64_t(dst + nb - mstart);
                a.crc[lo] = s.part_crc[0];
            }
            __threadfence();
            pub->tag = uint32_t(k + 1);
        }
        __syncthreads();
    }
}

}  // namespace nastar
