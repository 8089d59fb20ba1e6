/* CPU oracle of the search GIFs (DESIGN.md §19): one GIF, one thread, written the plain way.
 *
 * TEST INFRASTRUCTURE ONLY.  Every frame is rendered whole as screen-sized palette indices and compared with the
 * previous one to find its rectangle; the LZW keeps its dictionary as a (code, symbol) -> code table.  The kernel
 * instead renders only a frame's changed cells, finds rectangles from the selected cells and hashes its dictionary,
 * so the two share nothing but the format.
 *
 * Frames: for k < steps, a cell is red if trace[k] selects it (negative entries select the goal), else green if some
 * trace[j], j < k, selected it, else its grey; frame `steps` is red on the path, green on the histories, else grey; then
 * `hold` copies of the last frame.  Palette: the sorted grey levels with 0, green, red, transparent, black up to
 * 2^m >= 4 entries.  LZW: a clear code first; greedy longest match; after each emitted code the width grows when the
 * next free code equals 2^width (up to 12) and one entry is added; when the next free code reaches 4096 a clear code
 * follows and the table starts over; the last prefix, then end of information; bits LSB-first.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    uint8_t *out;
    int64_t n, cap;
} Buf;

static void put(Buf *b, const void *p, int64_t n) {
    if (n > 0 && b->n + n <= b->cap) memcpy(b->out + b->n, p, (size_t)n);
    b->n += n;
}
static void put1(Buf *b, int v) {
    uint8_t c = (uint8_t)v;
    put(b, &c, 1);
}
static void put2(Buf *b, int v) {
    put1(b, v & 255);
    put1(b, (v >> 8) & 255);
}

typedef struct {
    Buf *b;
    uint8_t block[255];
    int nblock;
    uint32_t acc;
    int nacc, width;
} Bits;

static void bits_byte(Bits *s, int v) {
    s->block[s->nblock++] = (uint8_t)v;
    if (s->nblock == 255) {
        put1(s->b, 255);
        put(s->b, s->block, 255);
        s->nblock = 0;
    }
}
static void bits_code(Bits *s, int code) {
    s->acc |= (uint32_t)code << s->nacc;
    s->nacc += s->width;
    while (s->nacc >= 8) {
        bits_byte(s, s->acc & 255);
        s->acc >>= 8;
        s->nacc -= 8;
    }
}

/* the LZW stream of n symbols, in sub-blocks, with the minimum code size before and the terminator after */
static void lzw(Buf *b, const uint8_t *sym, int64_t n, int m) {
    /* child[p][c] is the code of string p + c when gen[p][c] is the table's current generation */
    static int32_t child[4096][256];
    static uint32_t gen[4096][256], generation;
    const int clear = 1 << m, eoi = clear + 1;
    Bits s = {b, {0}, 0, 0, 0, m + 1};
    put1(b, m);
    ++generation;
    int next = eoi + 1, prefix = -1;
    bits_code(&s, clear);
    for (int64_t i = 0; i < n; ++i) {
        const int c = sym[i];
        if (prefix < 0) { prefix = c; continue; }
        if (gen[prefix][c] == generation) { prefix = child[prefix][c]; continue; }
        bits_code(&s, prefix);
        if (next == (1 << s.width) && s.width < 12) ++s.width;
        child[prefix][c] = next++;
        gen[prefix][c] = generation;
        if (next == 4096) {
            bits_code(&s, clear);
            ++generation;
            next = eoi + 1;
            s.width = m + 1;
        }
        prefix = c;
    }
    if (prefix >= 0) {
        bits_code(&s, prefix);
        if (next == (1 << s.width) && s.width < 12) ++s.width;
    }
    bits_code(&s, eoi);
    if (s.nacc > 0) bits_byte(&s, s.acc & 255);
    if (s.nblock > 0) {
        put1(b, s.nblock);
        put(b, s.block, s.nblock);
    }
    put1(b, 0);
}

/* One GIF.  grey: [nmaps, H*W] grey levels; hist, path: [nmaps, H*W] 0/1 of the final frame; trace: [nmaps, T];
 * goal: [nmaps].  grid: make_grid's layout (8 per row, 2-pixel black border) when nmaps > 1.  xmap / ymap: screen
 * column / row -> image column / row.  Returns the GIF's size (bytes past cap are counted, not written), or -1 when the
 * palette would exceed 256 entries. */
int64_t nastar_oracle_gif(const uint8_t *grey, const uint8_t *hist, const uint8_t *path, const int32_t *trace,
                          const int32_t *goal, int nmaps, int H, int W, int T, int steps, int grid, int SW, int SH,
                          const int32_t *xmap, const int32_t *ymap, int delay, int hold, int loop, uint8_t *out,
                          int64_t cap) {
    const int64_t N = (int64_t)H * W, npx = (int64_t)SW * SH;
    const int tiled = grid && nmaps > 1;
    const int xmaps = nmaps < 8 ? nmaps : 8, ymaps = (nmaps + xmaps - 1) / xmaps;
    const int Hi = tiled ? (H + 2) * ymaps + 2 : H, Wi = tiled ? (W + 2) * xmaps + 2 : W;
    int present[256] = {0}, index[256];
    present[0] = 1;
    for (int64_t i = 0; i < nmaps * N; ++i) present[grey[i]] = 1;
    int ng = 0;
    for (int v = 0; v < 256; ++v)
        if (present[v]) index[v] = ng++;
    const int green = ng, red = ng + 1, transparent = ng + 2;
    int m = 2;
    while ((1 << m) < ng + 3) ++m;
    if (m > 8) return -1;
    /* image pixel -> (map, cell) or -1 for the border */
    int32_t *owner = malloc(sizeof(int32_t) * (size_t)Hi * Wi);
    for (int y = 0; y < Hi; ++y)
        for (int x = 0; x < Wi; ++x) {
            int32_t o = -1;
            if (!tiled) {
                o = y * W + x;
            } else {
                const int yy = y / (H + 2), ry = y % (H + 2) - 2, xx = x / (W + 2), rx = x % (W + 2) - 2;
                if (ry >= 0 && rx >= 0 && yy * xmaps + xx < nmaps) o = (int32_t)((yy * xmaps + xx) * N + ry * W + rx);
            }
            owner[(int64_t)y * Wi + x] = o;
        }
    uint8_t *closed = calloc((size_t)(nmaps * N), 1), *cell = malloc((size_t)(nmaps * N));
    uint8_t *prev = malloc((size_t)npx), *cur = malloc((size_t)npx), *sym = malloc((size_t)npx);
    Buf b = {out, 0, cap};
    put(&b, "GIF89a", 6);
    put2(&b, SW);
    put2(&b, SH);
    put1(&b, 0x80 | (m - 1) << 4 | (m - 1));
    put1(&b, 0);
    put1(&b, 0);
    for (int e = 0; e < (1 << m); ++e) {
        int r = 0, g = 0, bl = 0;
        if (e < ng) {
            for (int v = 0; v < 256; ++v)
                if (present[v] && index[v] == e) r = g = bl = v;
        } else if (e == green) {
            r = 51; g = 204;
        } else if (e == red) {
            r = 255;
        }
        put1(&b, r); put1(&b, g); put1(&b, bl);
    }
    put(&b, "\x21\xff\x0bNETSCAPE2.0\x03\x01", 16);
    put2(&b, loop);
    put1(&b, 0);
    const int nframes = steps + 1 + hold;
    for (int k = 0; k < nframes; ++k) {
        const int f = k < steps ? k : steps;
        for (int mi = 0; mi < nmaps; ++mi)
            for (int64_t c = 0; c < N; ++c) {
                const int64_t i = mi * N + c;
                int v = index[grey[i]];
                if (f < steps) {
                    int s = trace[(int64_t)mi * T + f];
                    if (s < 0) s = goal[mi];
                    if (s == c) v = red;
                    else if (closed[i]) v = green;
                } else if (path[i]) {
                    v = red;
                } else if (hist[i]) {
                    v = green;
                }
                cell[i] = (uint8_t)v;
            }
        if (f < steps)
            for (int mi = 0; mi < nmaps; ++mi) {
                int s = trace[(int64_t)mi * T + f];
                if (s < 0) s = goal[mi];
                closed[mi * N + s] = 1;   /* closed before the next step */
            }
        for (int Y = 0; Y < SH; ++Y)
            for (int X = 0; X < SW; ++X) {
                const int32_t o = owner[(int64_t)ymap[Y] * Wi + xmap[X]];
                cur[(int64_t)Y * SW + X] = o < 0 ? (uint8_t)index[0] : cell[o];
            }
        int x0 = 0, y0 = 0, x1 = SW, y1 = SH;
        if (k > 0) {
            x0 = SW; y0 = SH; x1 = 0; y1 = 0;
            for (int Y = 0; Y < SH; ++Y)
                for (int X = 0; X < SW; ++X)
                    if (cur[(int64_t)Y * SW + X] != prev[(int64_t)Y * SW + X]) {
                        if (X < x0) x0 = X;
                        if (X + 1 > x1) x1 = X + 1;
                        if (Y < y0) y0 = Y;
                        if (Y + 1 > y1) y1 = Y + 1;
                    }
        }
        int64_t n = 0;
        if (x0 >= x1) {   /* nothing changed: one transparent pixel */
            x0 = y0 = 0; x1 = y1 = 1;
            sym[n++] = (uint8_t)transparent;
        } else {
            for (int Y = y0; Y < y1; ++Y)
                for (int X = x0; X < x1; ++X) {
                    const int64_t i = (int64_t)Y * SW + X;
                    sym[n++] = (uint8_t)(k > 0 && cur[i] == prev[i] ? transparent : cur[i]);
                }
        }
        put(&b, "\x21\xf9\x04", 3);
        put1(&b, k == 0 ? 0x04 : 0x05);
        put2(&b, delay);
        put1(&b, k == 0 ? 0 : transparent);
        put1(&b, 0);
        put1(&b, 0x2C);
        put2(&b, x0); put2(&b, y0); put2(&b, x1 - x0); put2(&b, y1 - y0);
        put1(&b, 0);
        lzw(&b, sym, n, m);
        uint8_t *t = prev; prev = cur; cur = t;
    }
    put1(&b, ';');
    free(owner); free(closed); free(cell); free(prev); free(cur); free(sym);
    return b.n;
}
