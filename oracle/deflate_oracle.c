/* deflate_oracle.c — sequential restatement of the chunked deflate of csrc/nastar_deflate.cuh (DESIGN.md §18).
 *
 * TEST INFRASTRUCTURE ONLY: built by oracle/deflate.py, never linked into the product.  The kernel's output must equal
 * this file's byte for byte, so every rule below (hash, chains, match choice, lazy parse, Huffman construction and
 * length limiting, code-length RLE, block choice, bit layout) is the kernel's rule, written for one CPU thread.
 *
 * A member is cut into chunks of DEFLATE_CHUNK bytes.  Each chunk is compressed alone (no match crosses a chunk
 * start) into one dynamic-Huffman block, or into stored blocks when those are not larger.  A chunk that is not its
 * member's last ends with an empty stored block (zlib's Z_FULL_FLUSH), so every chunk ends byte-aligned and the
 * chunks join into one raw deflate stream; the last chunk's last block has BFINAL set. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define DEFLATE_CHUNK (256 * 1024)
#define HASH_BITS 15
#define WINDOW 32768
#define MAX_CHAIN 128
#define MAX_LAZY 32
#define TOO_FAR 4096

static const int kLenBase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31,
                                 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
static const int kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5,
                                  0};
static const int kDistBase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769,
                                  1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
static const int kDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11,
                                   12, 12, 13, 13};
static const int kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

static int len_code(int len) {   /* 0..28 */
    int c = 0;
    while (c < 28 && kLenBase[c + 1] <= len) ++c;
    return c;
}
static int dist_code(int dist) { /* 0..29 */
    int c = 0;
    while (c < 29 && kDistBase[c + 1] <= dist) ++c;
    return c;
}

static uint32_t hash3(const uint8_t* p) {
    const uint32_t v = (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16);
    return (v * 2654435761u) >> (32 - HASH_BITS);
}

/* Huffman code lengths for freq[0..n) limited to maxbits.  Symbols are ranked by (freq, index); the tree is built
 * with two queues (a leaf is taken before an internal node of equal weight); depths above maxbits are clamped and the
 * Kraft sum repaired by lengthening the deepest code below the limit; lengths are then handed out by rank, longest
 * to the rarest.  Fewer than two used symbols: the used one (if any) and the lowest unused ones get length 1. */
static void build_lengths(const uint32_t* freq, int n, int maxbits, uint8_t* len) {
    int sym[286], m = 0;
    memset(len, 0, (size_t)n);
    for (int i = 0; i < n; ++i)
        if (freq[i]) sym[m++] = i;
    if (m < 2) {
        for (int i = 0; i < n && m < 2; ++i)
            if (!freq[i]) sym[m++] = i;
        len[sym[0]] = 1;
        len[sym[1]] = 1;
        return;
    }
    /* insertion sort by (freq, index): n <= 286 */
    for (int i = 1; i < m; ++i) {
        const int s = sym[i];
        int j = i - 1;
        while (j >= 0 && (freq[sym[j]] > freq[s] || (freq[sym[j]] == freq[s] && sym[j] > s))) {
            sym[j + 1] = sym[j];
            --j;
        }
        sym[j + 1] = s;
    }
    uint64_t w[2 * 286];
    int parent[2 * 286];
    for (int i = 0; i < m; ++i) w[i] = freq[sym[i]];
    int leaf = 0, node = m, next = m;   /* internal nodes m.. in creation order (non-decreasing weight) */
    while (next < 2 * m - 1) {
        int pick[2];
        for (int k = 0; k < 2; ++k) {
            if (leaf < m && (node >= next || w[leaf] <= w[node])) pick[k] = leaf++;
            else pick[k] = node++;
        }
        w[next] = w[pick[0]] + w[pick[1]];
        parent[pick[0]] = parent[pick[1]] = next;
        ++next;
    }
    int depth[2 * 286];
    depth[2 * m - 2] = 0;
    for (int i = 2 * m - 3; i >= 0; --i) depth[i] = depth[parent[i]] + 1;
    int count[16] = {0};
    for (int i = 0; i < m; ++i) count[depth[i] > maxbits ? maxbits : depth[i]]++;
    uint32_t total = 0;
    for (int b = 1; b <= maxbits; ++b) total += (uint32_t)count[b] << (maxbits - b);
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
        for (int k = 0; k < count[b]; ++k) len[sym[r++]] = (uint8_t)b;
}

/* canonical codes, bit-reversed for LSB-first output */
static void build_codes(const uint8_t* len, int n, uint16_t* code) {
    int count[16] = {0}, next[16];
    for (int i = 0; i < n; ++i) count[len[i]]++;
    count[0] = 0;
    int c = 0;
    for (int b = 1; b < 16; ++b) {
        c = (c + count[b - 1]) << 1;
        next[b] = c;
    }
    for (int i = 0; i < n; ++i) {
        if (!len[i]) { code[i] = 0; continue; }
        uint32_t v = (uint32_t)next[len[i]]++, rev = 0;
        for (int b = 0; b < len[i]; ++b) rev |= ((v >> b) & 1u) << (len[i] - 1 - b);
        code[i] = (uint16_t)rev;
    }
}

typedef struct {
    uint8_t* out;
    uint64_t bitpos;
} Bits;

static void put(Bits* b, uint32_t v, int n) {
    for (int i = 0; i < n; ++i) {
        if ((v >> i) & 1u) b->out[b->bitpos >> 3] |= (uint8_t)(1u << (b->bitpos & 7));
        b->bitpos++;
    }
}

/* the run-length coding of the code lengths: each item is sym | extra << 8 */
static int rle_lengths(const uint8_t* L, int total, uint32_t* items) {
    int k = 0, i = 0;
    while (i < total) {
        const int v = L[i];
        int run = 1;
        while (i + run < total && L[i + run] == v) ++run;
        if (v == 0) {
            while (run >= 11) {
                const int r = run > 138 ? 138 : run;
                items[k++] = 18u | (uint32_t)(r - 11) << 8;
                run -= r;
                i += r;
            }
            if (run >= 3) {
                items[k++] = 17u | (uint32_t)(run - 3) << 8;
                i += run;
                run = 0;
            }
        } else {
            items[k++] = (uint32_t)v;
            ++i;
            --run;
            while (run >= 3) {
                const int r = run > 6 ? 6 : run;
                items[k++] = 16u | (uint32_t)(r - 3) << 8;
                run -= r;
                i += r;
            }
        }
        for (; run > 0; --run, ++i) items[k++] = (uint32_t)v;
    }
    return k;
}

static const int kClExtra[19] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2, 3, 7};

/* Compress one chunk of n bytes into out (at most deflate_chunk_bound(n) bytes).  Returns the bytes written. */
int64_t nastar_oracle_deflate_chunk(const uint8_t* in, int64_t n, int final, uint8_t* out) {
    /* matches: best (len, dist) at every position, from the hash chains of this chunk only */
    uint16_t* prev = calloc((size_t)(n > 0 ? n : 1), 2);
    uint32_t* match = calloc((size_t)(n > 0 ? n : 1), 4);
    int32_t* head = malloc(sizeof(int32_t) << HASH_BITS);
    for (int i = 0; i < (1 << HASH_BITS); ++i) head[i] = -1;
    for (int64_t p = 0; p + 3 <= n; ++p) {
        const uint32_t h = hash3(in + p);
        prev[p] = (head[h] >= 0 && p - head[h] <= WINDOW) ? (uint16_t)(p - head[h]) : 0;
        head[h] = (int32_t)p;
    }
    for (int64_t p = 0; p + 3 <= n; ++p) {
        const int64_t lim = n - p < 258 ? n - p : 258;
        int best = 0, bestd = 0;
        int64_t q = p;
        for (int c = 0; c < MAX_CHAIN && prev[q]; ++c) {
            q -= prev[q];
            if (p - q > WINDOW) break;
            if (in[q + best] != in[p + best]) continue;   /* cannot be longer than best (best < lim here) */
            int l = 0;
            while (l < lim && in[q + l] == in[p + l]) ++l;
            if (l > best) {
                best = l;
                bestd = (int)(p - q);
                if (l == lim) break;
            }
        }
        if (best >= 3 && !(best == 3 && bestd > TOO_FAR)) match[p] = (uint32_t)best << 16 | (uint32_t)(bestd - 1);
    }
    /* lazy parse into tokens: a literal b, or 0x80000000 | match */
    uint32_t* tok = malloc(sizeof(uint32_t) * (size_t)(n > 0 ? n : 1));
    int64_t T = 0;
    for (int64_t p = 0; p < n;) {
        const uint32_t m = match[p];
        const int l = (int)(m >> 16);
        if (l >= 3 && !(l < MAX_LAZY && p + 1 < n && (int)(match[p + 1] >> 16) > l)) {
            tok[T++] = 0x80000000u | m;
            p += l;
        } else {
            tok[T++] = in[p];
            p += 1;
        }
    }
    /* codes */
    uint32_t lf[286] = {0}, df[30] = {0};
    for (int64_t t = 0; t < T; ++t) {
        if (tok[t] & 0x80000000u) {
            lf[257 + len_code((int)((tok[t] >> 16) & 0x1ff))]++;
            df[dist_code((int)(tok[t] & 0xffff) + 1)]++;
        } else {
            lf[tok[t]]++;
        }
    }
    lf[256] = 1;
    uint8_t ll[286 + 30], *dl = ll + 286, cll[19];
    uint16_t lc[286], dc[30], clc[19];
    build_lengths(lf, 286, 15, ll);
    build_lengths(df, 30, 15, dl);
    int hlit = 286, hdist = 30;
    while (hlit > 257 && !ll[hlit - 1]) --hlit;
    while (hdist > 1 && !dl[hdist - 1]) --hdist;
    uint8_t seq[286 + 30];
    memcpy(seq, ll, (size_t)hlit);
    memcpy(seq + hlit, dl, (size_t)hdist);
    uint32_t items[286 + 30];
    const int nitems = rle_lengths(seq, hlit + hdist, items);
    uint32_t cf[19] = {0};
    for (int i = 0; i < nitems; ++i) cf[items[i] & 0xff]++;
    build_lengths(cf, 19, 7, cll);
    int hclen = 19;
    while (hclen > 4 && !cll[kClOrder[hclen - 1]]) --hclen;
    build_codes(ll, 286, lc);
    build_codes(dl, 30, dc);
    build_codes(cll, 19, clc);
    uint64_t bits = 3 + 14 + 3 * (uint64_t)hclen;
    for (int i = 0; i < nitems; ++i) bits += cll[items[i] & 0xff] + kClExtra[items[i] & 0xff];
    for (int64_t t = 0; t < T; ++t) {
        if (tok[t] & 0x80000000u) {
            const int lcode = len_code((int)((tok[t] >> 16) & 0x1ff)), d = dist_code((int)(tok[t] & 0xffff) + 1);
            bits += ll[257 + lcode] + kLenExtra[lcode] + dl[d] + kDistExtra[d];
        } else {
            bits += ll[tok[t]];
        }
    }
    bits += ll[256];
    const int64_t nstored = n > 0 ? (n + 65534) / 65535 : 1;
    const int64_t stored_bytes = n + 5 * nstored + (final ? 0 : 5);
    const int64_t dyn_bytes = final ? (int64_t)((bits + 7) / 8) : (int64_t)((bits + 3 + 7) / 8) + 4;
    memset(out, 0, (size_t)(stored_bytes < dyn_bytes ? stored_bytes : dyn_bytes));
    Bits b = {out, 0};
    if (dyn_bytes < stored_bytes) {
        put(&b, final ? 1u : 0u, 1);
        put(&b, 2u, 2);
        put(&b, (uint32_t)(hlit - 257), 5);
        put(&b, (uint32_t)(hdist - 1), 5);
        put(&b, (uint32_t)(hclen - 4), 4);
        for (int i = 0; i < hclen; ++i) put(&b, cll[kClOrder[i]], 3);
        for (int i = 0; i < nitems; ++i) {
            const int s = (int)(items[i] & 0xff);
            put(&b, clc[s], cll[s]);
            put(&b, items[i] >> 8, kClExtra[s]);
        }
        for (int64_t t = 0; t < T; ++t) {
            if (tok[t] & 0x80000000u) {
                const int len = (int)((tok[t] >> 16) & 0x1ff), dist = (int)(tok[t] & 0xffff) + 1;
                const int lcode = len_code(len), d = dist_code(dist);
                put(&b, lc[257 + lcode], ll[257 + lcode]);
                put(&b, (uint32_t)(len - kLenBase[lcode]), kLenExtra[lcode]);
                put(&b, dc[d], dl[d]);
                put(&b, (uint32_t)(dist - kDistBase[d]), kDistExtra[d]);
            } else {
                put(&b, lc[tok[t]], ll[tok[t]]);
            }
        }
        put(&b, lc[256], ll[256]);
        if (!final) put(&b, 0u, 3);
        b.bitpos = (b.bitpos + 7) & ~(uint64_t)7;
        if (!final) put(&b, 0xffff0000u, 32);
    } else {
        for (int64_t k = 0; k < nstored; ++k) {
            const int64_t off = k * 65535, len = n - off < 65535 ? n - off : 65535;
            put(&b, (final && k == nstored - 1) ? 1u : 0u, 3);
            b.bitpos = (b.bitpos + 7) & ~(uint64_t)7;
            put(&b, (uint32_t)len | ((uint32_t)(len ^ 0xffff) << 16), 32);
            memcpy(out + (b.bitpos >> 3), in + off, (size_t)len);
            b.bitpos += (uint64_t)len * 8;
        }
        if (!final) {
            put(&b, 0u, 3);
            b.bitpos = (b.bitpos + 7) & ~(uint64_t)7;
            put(&b, 0xffff0000u, 32);
        }
    }
    free(prev);
    free(match);
    free(head);
    free(tok);
    return (int64_t)(b.bitpos >> 3);
}

int64_t nastar_oracle_deflate_chunk_size(void) { return DEFLATE_CHUNK; }

/* worst case of one chunk of n bytes: its stored form plus the empty stored block */
int64_t nastar_oracle_deflate_chunk_bound(int64_t n) { return n + 5 * (n > 0 ? (n + 65534) / 65535 : 1) + 5; }

/* n bytes as a run of chunks, the last one final (an empty input is one empty final chunk).  Returns the bytes
 * written to out, which holds at least the sum of the chunks' bounds. */
int64_t nastar_oracle_deflate(const uint8_t* in, int64_t n, uint8_t* out) {
    int64_t o = 0;
    for (int64_t off = 0;; off += DEFLATE_CHUNK) {
        const int64_t len = n - off < DEFLATE_CHUNK ? n - off : DEFLATE_CHUNK;
        o += nastar_oracle_deflate_chunk(in + off, len, off + len >= n, out + o);
        if (off + len >= n) break;
    }
    return o;
}
