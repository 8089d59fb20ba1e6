// Search animations as GIF frames (nastar_b200_gif_plan / nastar_b200_gif_encode, DESIGN.md §19).
//
// A call animates G GIFs over B maps: layout "each" has one map per GIF (G = B), layout "grid" one GIF of all B maps
// tiled like make_grid.  GIF g has T_g search steps and T_g + 1 frames: frame k < T_g shows the closed set before step
// k and the cell selected at step k, frame T_g the search's histories and paths.  Frame 0 covers the screen; frame
// k > 0 covers the smallest rectangle of pixels that differ from frame k-1, unchanged pixels transparent.
//
// Two launches of persistent CTAs:
//  - plan: map items first (one CTA per map, from an atomic counter): the map's first-selection table (scatter-min of
//    the trace), then the screen rectangle of every frame, unioned over the GIF's maps with atomics.  The CTA that
//    finishes the last map item numbers the frames.  Then frame items, one warp each from a second counter: the
//    frame's LZW stream is sized without being written.  A warp waits for the last map item before its first frame;
//    map items are taken before any frame item and wait on nothing, so the wait ends.
//  - encode: the same frames again, each written as a complete record (graphic control extension, image descriptor,
//    LZW minimum code size, sub-blocks, terminator) at the offset the host computed from the sizes.
// A warp renders 256 pixels of its rectangle at a time into shared memory; lane 0 runs the LZW over them with the
// dictionary in a shared-memory hash.  Frame items are ordered full frames first (frame 0 and the final frame of
// every GIF), then the rest.
#pragma once
#include <cstdint>

namespace nastar {

constexpr int kGifWarps = 4;
constexpr int kGifThreads = 32 * kGifWarps;
constexpr int kGifHashSlots = 8192;   // open addressing, at most 4096 entries
constexpr int kGifChunk = 256;        // pixels rendered per warp round
constexpr int kGifMaxCode = 4096;

// per-call control block at the start of the workspace (256 bytes)
struct GifCtl {
    int32_t map_next;     // map-item counter
    int32_t frame_next;   // frame-item counter
    int32_t maps_done;
    int32_t ready;        // 1 once the frames are numbered
    int32_t n_frames;     // sum over GIFs of T_g + 1
    int32_t encode_next;  // frame-item counter of the encode launch
};

struct GifArgs {
    const float* maps;       // [B, H, W] map designs
    const float* hist;       // [B, H, W] histories of the search
    const int64_t* paths;    // [B, H, W]
    const float* goal;       // [B, H, W] goal maps
    const int32_t* trace;    // [B, T] selected cell per step (negative: the goal)
    const int32_t* t_solve;  // [B]
    int32_t B, H, W, T;
    int32_t grid;            // 0: one GIF per map; 1: one GIF of all maps in make_grid's layout
    int32_t steps_mode;      // 0: each map's own steps; 1: the slowest map's (batch); 2: all T steps (coupled)
    int32_t Hg, Wg;          // the unscaled image (make_grid's)
    int32_t SW, SH;          // the logical screen
    const int32_t* xmap;     // [SW] screen column -> image column
    const int32_t* ymap;     // [SH] screen row -> image row
    const int32_t* xspan;    // [Wg, 2] image column -> screen columns [lo, hi)
    const int32_t* yspan;    // [Hg, 2]
    const uint8_t* lut;      // [G, 256] grey level -> palette index; green, red, transparent follow the greys
    const uint8_t* ncolors;  // [G, 2]: number of greys, LZW minimum code size
    int32_t delay_cs;
    // workspace
    GifCtl* ctl;
    int32_t* steps;          // [G] T_g
    int32_t* frame0;         // [G] first frame number of GIF g
    int32_t* goal_idx;       // [B] the goal cell of each map
    int32_t* first;          // [B, H*W] first step selecting each cell (INT32_MAX: never)
    uint32_t* rect;          // [G, T + 1, 4] x0, y0, ~x1, ~y1 (atomicMin; 0xFFFFFFFF: empty)
    int32_t* nbytes;         // [G * (T + 1)] LZW bytes of frame f (plan writes, encode reads)
    // encode only
    const int64_t* offset;   // [F] where each frame's record starts in out
    uint8_t* out;
};

__device__ __forceinline__ int gif_steps(const GifArgs& a, int b, int tmax_batch) {
    if (a.steps_mode == 2) return a.T;
    if (a.steps_mode == 1) return tmax_batch;
    const int ts = a.t_solve[b];
    return ts >= 0 ? min(ts + 1, a.T) : a.T;
}

struct GifCell {   // the map and cell behind an image pixel, or b < 0 for make_grid's border
    int b, c;
};

__device__ __forceinline__ GifCell gif_cell(const GifArgs& a, int g, int iy, int ix) {
    if (!a.grid) return {g, iy * a.W + ix};
    if (a.B == 1) return {0, iy * a.W + ix};
    const int xmaps = a.B < 8 ? a.B : 8;
    const int hh = a.H + 2, ww = a.W + 2;
    const int yy = iy / hh, ry = iy - yy * hh - 2, xx = ix / ww, rx = ix - xx * ww - 2;
    const int b = yy * xmaps + xx;
    if (ry < 0 || rx < 0 || xx >= xmaps || b >= a.B) return {-1, 0};
    return {b, ry * a.W + rx};
}

struct GifColors {
    const uint8_t* lut;
    int green, red, transparent;
};

__device__ __forceinline__ GifColors gif_colors(const GifArgs& a, int g) {
    const int n = a.ncolors[2 * g];
    return {a.lut + 256 * g, n, n + 1, n + 2};
}

__device__ __forceinline__ int gif_grey(const GifArgs& a, const GifColors& pc, int b, int c) {
    const float v = a.maps[int64_t(b) * a.H * a.W + c];
    return pc.lut[uint8_t(int(__fmul_rn(v, 255.0f)))];
}

__device__ __forceinline__ int gif_sel(const GifArgs& a, int b, int k, int goal) {
    const int v = a.trace[int64_t(b) * a.T + k];
    return v < 0 ? goal : v;
}

// palette index of cell c of map b in frame k < T_g (sel = the cell selected at step k)
__device__ __forceinline__ int gif_step_color(const GifArgs& a, const GifColors& pc, int b, int c, int k, int sel) {
    if (c == sel) return pc.red;
    if (__ldcg(a.first + int64_t(b) * a.H * a.W + c) < k) return pc.green;
    return gif_grey(a, pc, b, c);
}

__device__ __forceinline__ int gif_final_color(const GifArgs& a, const GifColors& pc, int b, int c) {
    const int64_t i = int64_t(b) * a.H * a.W + c;
    if (a.paths[i] == 1) return pc.red;
    if (a.hist[i] == 1.0f) return pc.green;
    return gif_grey(a, pc, b, c);
}

// the goal cell: the first maximum of the goal map, as argmax
__device__ int gif_goal(const GifArgs& a, int b) {
    __shared__ float sv[kGifThreads];
    __shared__ int si[kGifThreads];
    const int N = a.H * a.W;
    float best = -__int_as_float(0x7f800000);
    int bi = 0x7fffffff;
    for (int c = threadIdx.x; c < N; c += kGifThreads) {
        const float v = a.goal[int64_t(b) * N + c];
        if (v > best) { best = v; bi = c; }
    }
    sv[threadIdx.x] = best;
    si[threadIdx.x] = bi;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int t = 1; t < kGifThreads; ++t)
            if (sv[t] > sv[0] || (sv[t] == sv[0] && si[t] < si[0])) { sv[0] = sv[t]; si[0] = si[t]; }
    }
    __syncthreads();
    const int r = si[0] == 0x7fffffff ? 0 : si[0];
    __syncthreads();
    return r;
}

__device__ __forceinline__ void gif_union(const GifArgs& a, int g, int k, int iy, int ix) {
    const int x0 = a.xspan[2 * ix], x1 = a.xspan[2 * ix + 1], y0 = a.yspan[2 * iy], y1 = a.yspan[2 * iy + 1];
    if (x0 >= x1 || y0 >= y1) return;   // an image pixel that no screen pixel samples
    uint32_t* r = a.rect + (int64_t(g) * (a.T + 1) + k) * 4;
    atomicMin(r + 0, uint32_t(x0));
    atomicMin(r + 1, uint32_t(y0));
    atomicMin(r + 2, ~uint32_t(x1));
    atomicMin(r + 3, ~uint32_t(y1));
}

// image coordinates of cell c of map b in GIF g
__device__ __forceinline__ void gif_image_xy(const GifArgs& a, int b, int c, int* iy, int* ix) {
    const int r = c / a.W, q = c - r * a.W;
    if (!a.grid || a.B == 1) { *iy = r; *ix = q; return; }
    const int xmaps = a.B < 8 ? a.B : 8;
    *iy = (b / xmaps) * (a.H + 2) + 2 + r;
    *ix = (b % xmaps) * (a.W + 2) + 2 + q;
}

// one map item: steps, first-selection table, the rectangles of the map's changes
__device__ void gif_map_item(const GifArgs& a, int b) {
    const int N = a.H * a.W;
    const int g = a.grid ? 0 : b;
    __shared__ int s_tb;
    if (a.steps_mode == 1) {   // the slowest map's steps: the reference loop's T_batch
        if (threadIdx.x == 0) s_tb = 0;
        __syncthreads();
        int m = 0;
        for (int i = threadIdx.x; i < a.B; i += kGifThreads) {
            const int ts = a.t_solve[i];
            m = max(m, ts >= 0 ? ts + 1 : a.T);
        }
        atomicMax(&s_tb, min(m, a.T));
        __syncthreads();
    }
    const int Tg = gif_steps(a, b, a.steps_mode == 1 ? s_tb : 0);
    const int goal = gif_goal(a, b);
    int32_t* first = a.first + int64_t(b) * N;
    for (int c = threadIdx.x; c < N; c += kGifThreads) first[c] = 0x7fffffff;
    __syncthreads();
    for (int k = threadIdx.x; k < Tg; k += kGifThreads) atomicMin(first + gif_sel(a, b, k, goal), k);
    __syncthreads();
    const GifColors pc = gif_colors(a, g);
    // frames 1 .. Tg-1: only the previously and the newly selected cells can change
    for (int k = 1 + threadIdx.x; k < Tg; k += kGifThreads) {
        const int prev = gif_sel(a, b, k - 1, goal), cur = gif_sel(a, b, k, goal);
        const int cells[2] = {prev, cur};
        for (int j = 0; j < 2; ++j) {
            const int c = cells[j];
            if (j == 1 && c == prev) break;
            if (gif_step_color(a, pc, b, c, k - 1, prev) != gif_step_color(a, pc, b, c, k, cur)) {
                int iy, ix;
                gif_image_xy(a, b, c, &iy, &ix);
                gif_union(a, g, k, iy, ix);
            }
        }
    }
    // the final frame against frame Tg-1
    const int last = gif_sel(a, b, Tg - 1, goal);
    for (int c = threadIdx.x; c < N; c += kGifThreads) {
        if (gif_step_color(a, pc, b, c, Tg - 1, last) != gif_final_color(a, pc, b, c)) {
            int iy, ix;
            gif_image_xy(a, b, c, &iy, &ix);
            gif_union(a, g, Tg, iy, ix);
        }
    }
    if (threadIdx.x == 0) {
        a.goal_idx[b] = goal;
        if (!a.grid || b == 0) a.steps[g] = Tg;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0 && atomicAdd(&a.ctl->maps_done, 1) == a.B - 1) {
        __threadfence();
        const int G = a.grid ? 1 : a.B;
        int f = 0;
        for (int i = 0; i < G; ++i) {
            a.frame0[i] = f;
            f += __ldcg(a.steps + i) + 1;
        }
        a.ctl->n_frames = f;
        __threadfence();
        atomicExch(&a.ctl->ready, 1);
    }
}

// frame item q -> (GIF g, frame k): the 2G full frames first, then the middle frames GIF by GIF
__device__ __forceinline__ void gif_frame_of(const GifArgs& a, int q, int G, int* g, int* k) {
    if (q < 2 * G) {
        *g = q >> 1;
        *k = (q & 1) ? __ldcg(a.steps + *g) : 0;
        return;
    }
    int r = q - 2 * G;   // middle frames before GIF g: frame0[g] - 2g
    int lo = 0, hi = G - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldcg(a.frame0 + mid) - 2 * mid <= r) lo = mid; else hi = mid - 1;
    }
    *g = lo;
    *k = 1 + r - (__ldcg(a.frame0 + lo) - 2 * lo);
}

struct GifWarpSmem {
    uint32_t hash[kGifHashSlots];   // (prefix << 8 | symbol) << 12 | code; 0 = empty
    uint8_t sym[kGifChunk];
};

// LZW state of lane 0: greedy longest match, one entry per emitted code, codes from m+1 bits up to 12, a clear code
// and a fresh table when the next free code reaches 4096; bits LSB-first.
template <bool kWrite>
struct GifLzw {
    uint32_t* hash;
    uint8_t* dst;       // the frame's first data byte (after the minimum code size); sub-block lengths interleaved
    int64_t nbytes;     // final LZW byte count (write pass)
    int64_t pos;        // LZW bytes so far
    uint64_t acc;
    int nacc;
    int m, width, next, prefix;

    __device__ void put_byte(uint8_t v) {
        if constexpr (kWrite) {
            const int64_t blk = pos / 255, in = pos - blk * 255;
            uint8_t* p = dst + blk * 256;
            if (in == 0) p[0] = uint8_t(nbytes - pos < 255 ? nbytes - pos : 255);
            p[1 + in] = v;
        }
        ++pos;
    }
    __device__ void emit(int code) {
        acc |= uint64_t(code) << nacc;
        nacc += width;
        while (nacc >= 8) {
            put_byte(uint8_t(acc));
            acc >>= 8;
            nacc -= 8;
        }
    }
    __device__ void reset_table() {   // mid-stream, after 4094 codes: lane 0 alone
        for (int i = 0; i < kGifHashSlots; ++i) hash[i] = 0;
        next = (1 << m) + 2;
        width = m + 1;
    }
    __device__ void begin() {   // the table was cleared by the whole warp
        acc = 0; nacc = 0; pos = 0; prefix = -1;
        width = m + 1;
        emit(1 << m);
        next = (1 << m) + 2;
    }
    __device__ static uint32_t slot_of(uint32_t key) { return (key * 2654435761u) >> (32 - 13); }
    __device__ void symbol(int c) {
        if (prefix < 0) { prefix = c; return; }
        const uint32_t key = (uint32_t(prefix) << 8) | uint32_t(c);
        uint32_t s = slot_of(key);
        for (;;) {
            const uint32_t v = hash[s];
            if (v == 0) break;
            if ((v >> 12) == key) { prefix = int(v & 4095u); return; }
            s = (s + 1) & (kGifHashSlots - 1);
        }
        emit(prefix);
        if (next == (1 << width) && width < 12) ++width;
        hash[s] = (key << 12) | uint32_t(next);
        ++next;
        if (next == kGifMaxCode) {
            emit(1 << m);
            reset_table();
        }
        prefix = c;
    }
    __device__ void finish() {
        if (prefix >= 0) {
            emit(prefix);
            if (next == (1 << width) && width < 12) ++width;
        }
        emit((1 << m) + 1);
        if (nacc > 0) put_byte(uint8_t(acc));
    }
};

// one frame, by one warp: size it (kWrite false) or write its record
template <bool kWrite>
__device__ void gif_frame(const GifArgs& a, GifWarpSmem& s, int g, int k, int fidx) {
    const int lane = threadIdx.x & 31;
    const int Tg = __ldcg(a.steps + g);
    const GifColors pc = gif_colors(a, g);
    int x0 = 0, y0 = 0, w = a.SW, h = a.SH;
    bool empty = false;
    if (k > 0) {
        const uint32_t* r = a.rect + (int64_t(g) * (a.T + 1) + k) * 4;
        const uint32_t rx0 = __ldcg(r), ry0 = __ldcg(r + 1), rx1 = ~__ldcg(r + 2), ry1 = ~__ldcg(r + 3);
        if (rx0 == 0xFFFFFFFFu) {
            w = h = 1;
            empty = true;
        } else {
            x0 = int(rx0); y0 = int(ry0); w = int(rx1 - rx0); h = int(ry1 - ry0);
        }
    }
    const int m = a.ncolors[2 * g + 1];
    GifLzw<kWrite> z;
    z.hash = s.hash;
    z.m = m;
    uint8_t* rec = nullptr;
    if constexpr (kWrite) {
        rec = a.out + a.offset[fidx];
        z.dst = rec + 19;
        z.nbytes = a.nbytes[fidx];
    }
    for (int i = lane; i < kGifHashSlots; i += 32) s.hash[i] = 0;
    __syncwarp();
    if (lane == 0) z.begin();
    __syncwarp();
    const int64_t npx = int64_t(w) * h;
    for (int64_t base = 0; base < npx; base += kGifChunk) {
        for (int j = lane; j < kGifChunk; j += 32) {
            const int64_t i = base + j;
            if (i >= npx) break;
            int sym = pc.transparent;
            if (!empty) {
                const int Y = y0 + int(i / w), X = x0 + int(i % w);
                const GifCell cell = gif_cell(a, g, __ldg(a.ymap + Y), __ldg(a.xmap + X));
                if (cell.b < 0) {
                    sym = k == 0 ? 0 : pc.transparent;   // make_grid's border: palette index 0 is grey 0
                } else if (k == Tg) {
                    const int goal = __ldcg(a.goal_idx + cell.b);
                    const int last = gif_sel(a, cell.b, Tg - 1, goal);
                    const int nw = gif_final_color(a, pc, cell.b, cell.c);
                    sym = nw == gif_step_color(a, pc, cell.b, cell.c, Tg - 1, last) ? pc.transparent : nw;
                } else {
                    const int goal = __ldcg(a.goal_idx + cell.b);
                    const int cur = gif_sel(a, cell.b, k, goal);
                    if (k == 0) {
                        sym = cell.c == cur ? pc.red : gif_grey(a, pc, cell.b, cell.c);
                    } else {
                        const int prev = gif_sel(a, cell.b, k - 1, goal);
                        if (cell.c == cur || cell.c == prev) {
                            const int nw = gif_step_color(a, pc, cell.b, cell.c, k, cur);
                            sym = nw == gif_step_color(a, pc, cell.b, cell.c, k - 1, prev) ? pc.transparent : nw;
                        }
                    }
                }
            }
            s.sym[j] = uint8_t(sym);
        }
        __syncwarp();
        if (lane == 0) {
            const int n = npx - base < kGifChunk ? int(npx - base) : kGifChunk;
            for (int j = 0; j < n; ++j) z.symbol(s.sym[j]);
        }
        __syncwarp();
    }
    if (lane == 0) {
        z.finish();
        if constexpr (kWrite) {
            const int tr = pc.transparent;
            const uint8_t hdr[19] = {0x21, 0xF9, 0x04, uint8_t(k == 0 ? 0x04 : 0x05), uint8_t(a.delay_cs & 255),
                                     uint8_t(a.delay_cs >> 8), uint8_t(k == 0 ? 0 : tr), 0x00, 0x2C,
                                     uint8_t(x0 & 255), uint8_t(x0 >> 8), uint8_t(y0 & 255), uint8_t(y0 >> 8),
                                     uint8_t(w & 255), uint8_t(w >> 8), uint8_t(h & 255), uint8_t(h >> 8), 0x00,
                                     uint8_t(m)};
            for (int i = 0; i < 19; ++i) rec[i] = hdr[i];
            const int64_t n = z.pos;
            rec[19 + n + (n + 254) / 255] = 0x00;
        } else {
            a.nbytes[fidx] = int32_t(z.pos);
        }
    }
    __syncwarp();
}

// the frame items of a launch, one warp each; the plan's warps first wait for the frames to be numbered
template <bool kWrite>
__device__ void gif_frames(const GifArgs& a, GifWarpSmem& s) {
    const int lane = threadIdx.x & 31;
    if (!kWrite) {
        if (lane == 0)
            while (*reinterpret_cast<volatile int32_t*>(&a.ctl->ready) == 0) __nanosleep(256);
        __syncwarp();
        __threadfence();
    }
    const int G = a.grid ? 1 : a.B;
    const int F = __ldcg(&a.ctl->n_frames);
    int32_t* counter = kWrite ? &a.ctl->encode_next : &a.ctl->frame_next;
    for (;;) {
        int q = 0;
        if (lane == 0) q = atomicAdd(counter, 1);
        q = __shfl_sync(0xFFFFFFFFu, q, 0);
        if (q >= F) break;
        int g, k;
        gif_frame_of(a, q, G, &g, &k);
        gif_frame<kWrite>(a, s, g, k, __ldcg(a.frame0 + g) + k);
    }
}

__global__ void __launch_bounds__(kGifThreads, 1) gif_plan_kernel(GifArgs a) {
    extern __shared__ __align__(16) unsigned char gif_smem[];
    __shared__ int s_item;
    for (;;) {
        if (threadIdx.x == 0) s_item = atomicAdd(&a.ctl->map_next, 1);
        __syncthreads();
        const int b = s_item;
        __syncthreads();
        if (b >= a.B) break;
        gif_map_item(a, b);
    }
    gif_frames<false>(a, reinterpret_cast<GifWarpSmem*>(gif_smem)[threadIdx.x >> 5]);
}

__global__ void __launch_bounds__(kGifThreads, 1) gif_encode_kernel(GifArgs a) {
    extern __shared__ __align__(16) unsigned char gif_smem[];
    gif_frames<true>(a, reinterpret_cast<GifWarpSmem*>(gif_smem)[threadIdx.x >> 5]);
}

}  // namespace nastar
