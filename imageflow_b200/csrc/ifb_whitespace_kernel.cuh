// ifb_whitespace_kernel.cuh -- included by ifb_kernels.cuh inside namespace ifbk (product code, sm_90a).
// Uses only: threadIdx, blockIdx, __shared__, __syncthreads, __ldg, min, max, abs -- tests/test_whitespace_product.py compiles
// this file with g++ under a sequential emulation of those and checks the codes against the CPU oracle.
// graphics/whitespace.rs: the part of detect_content that is the same for every window -- approximate_grayscale (:426-523,
// Bgra32 when alpha is meaningful, else Bgr32) and the per-centre half of sobel_scharr_detect (:525-613) -- for every pixel at
// once.  One byte per pixel (layout in ifb_whitespace.h) for ifb200_batch_whitespace_codes; 32 x 8 pixels per CTA through a 34 x 10
// grayscale tile; 4 bytes read + 1 written per pixel.  detect_content itself (one frame or many) no longer writes this map: the
// second half of the file reduces the codes to per-row summaries and replays the reference's window walk over them on the device.
__device__ __forceinline__ uint32_t ws_gray(uint32_t bgra, bool alpha_meaningful) {
    const uint32_t lum = 233u * (bgra & 0xffu) + 1197u * ((bgra >> 8) & 0xffu) + 610u * ((bgra >> 16) & 0xffu);
    if (!alpha_meaningful) return lum / 2048u;                                    // Bgr32
    const uint32_t v = lum * (bgra >> 24);                                        // Bgra32: weighed by alpha, rounded up, clamped
    return min((v + 524287u) / 524288u, 255u);
}
// The code of the centre whose 3x3 neighbourhood is g[ty .. ty + 2][tx .. tx + 2] (an interior pixel): 0xFF when its Scharr value is
// at most `threshold`, else its local edge box (layout: ifb_whitespace.h).  Shared by whitespace_codes_kernel and
// whitespace_segments_kernel.
__device__ __forceinline__ uint32_t ws_centre_code(const uint8_t (*g)[36], uint32_t ty, uint32_t tx, int threshold) {
    uint32_t code = 0xFFu;
    int m[3][3];
#pragma unroll
    for (int j = 0; j < 3; ++j)
#pragma unroll
        for (int i = 0; i < 3; ++i) m[j][i] = g[ty + j][tx + i];
    const int gx = 3 * m[0][0] + 10 * m[1][0] + 3 * m[2][0] - 3 * m[0][2] - 10 * m[1][2] - 3 * m[2][2];
    const int gy = 3 * m[0][0] + 10 * m[0][1] + 3 * m[0][2] - 3 * m[2][0] - 10 * m[2][1] - 3 * m[2][2];
    if (abs(gx) + abs(gy) > threshold) {
        int lo_x = 2, lo_y = 2, hi_x = 1, hi_y = 1;
#pragma unroll
        for (int j = 0; j < 3; ++j) {                                             // differences along x in row j: :576-591
            const bool e01 = abs(m[j][0] - m[j][1]) > threshold, e12 = abs(m[j][1] - m[j][2]) > threshold;
            if (e01) { lo_x = min(lo_x, 1); hi_x = max(hi_x, 1); }
            if (e12) { lo_x = min(lo_x, 2); hi_x = max(hi_x, 2); }
            if (e01 || e12) { lo_y = min(lo_y, j); hi_y = max(hi_y, j + 1); }
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) {                                             // differences along y in column i: :592-608
            const bool e01 = abs(m[0][i] - m[1][i]) > threshold, e12 = abs(m[1][i] - m[2][i]) > threshold;
            if (e01) { lo_y = min(lo_y, 1); hi_y = max(hi_y, 1); }
            if (e12) { lo_y = min(lo_y, 2); hi_y = max(hi_y, 2); }
            if (e01 || e12) { lo_x = min(lo_x, i); hi_x = max(hi_x, i + 1); }
        }
        code = (uint32_t)lo_x | ((uint32_t)(hi_x - 1) << 2) | ((uint32_t)lo_y << 4) | ((uint32_t)(hi_y - 1) << 6);
    }
    return code;
}
__global__ void __launch_bounds__(256) whitespace_codes_kernel(const uint8_t* __restrict__ px, uint32_t w, uint32_t h, uint32_t stride,
                                                               uint32_t alpha_meaningful, int threshold, uint8_t* __restrict__ codes, uint32_t row0) {
    // row0: first image row of this launch (grid.y is bounded, bitmaps are not: tall ones take several launches)
    __shared__ uint8_t g[10][36];
    const int x0 = (int)blockIdx.x * 32 - 1, y0 = (int)(row0 + blockIdx.y * 8) - 1;       // image position of g[0][0]
    for (int i = threadIdx.y * 32 + threadIdx.x; i < 10 * 34; i += 256) {
        const int ty = i / 34, tx = i - ty * 34, x = x0 + tx, y = y0 + ty;
        uint32_t v = 0;
        if (x >= 0 && y >= 0 && x < (int)w && y < (int)h) v = ws_gray(__ldg(reinterpret_cast<const uint32_t*>(px + (size_t)y * stride) + x), alpha_meaningful != 0);
        g[ty][tx] = (uint8_t)v;
    }
    __syncthreads();
    const int x = (int)blockIdx.x * 32 + threadIdx.x, y = (int)(row0 + blockIdx.y * 8) + threadIdx.y;
    if (x >= (int)w || y >= (int)h) return;
    uint32_t code = 0xFFu;
    if (x > 0 && y > 0 && x + 1 < (int)w && y + 1 < (int)h) code = ws_centre_code(g, threadIdx.y, threadIdx.x, threshold);
    codes[(size_t)y * w + x] = (uint8_t)code;
}


#if defined(__CUDACC__) || defined(IFB_WS_BATCH_EMU)
// ---- ifb200_batch_detect_content_many: the codes reduced to summaries, then the reference's walk replayed over them (DESIGN.md §5.16;
// plan and summary layout: ifb_whitespace.h).  tests/cpu_emu/whitespace_many_emu.cc compiles this part under IFB_WS_BATCH_EMU: the
// segments kernel sequentially, each barrier-separated segment in a pass of its own, and the walk with its 32 lanes on OS threads.
#ifndef IFB_WS_SET                                                  // the CPU emulation gates shared and global stores per pass
#define IFB_WS_SET(lhs, v) ((lhs) = (v))
#endif

// The item of CTA `cta` of a flat launch whose n items begin at CTAs first[0] = 0 < first[1] < ...
__device__ __forceinline__ uint32_t ws_item_of(const uint32_t* first, uint32_t n, uint32_t cta) {
    uint32_t lo = 0, hi = n;                                        // first[lo] <= cta < first[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (first[mid] <= cta) lo = mid; else hi = mid;
    }
    return lo;
}

// One CTA = 32 interior columns (one chunk of a window column) x 8 rows of one frame, every frame of the call in one flat launch.  The
// grayscale tile and each centre's code are whitespace_codes_kernel's; then lane 4 r + f of warp 0 reduces field f of row r over the
// chunk's 32 codes into byte f of that row's summary.  Reads 4 bytes per pixel plus the tile's halo; writes 4 bytes per 32 pixels.
__global__ void __launch_bounds__(ifb::kWsThreads) whitespace_segments_kernel(const ifb::WsSeg* __restrict__ segs, const uint32_t* __restrict__ first,
                                                                             uint32_t n_segs, uint32_t* __restrict__ sums) {
    __shared__ uint8_t g[10][36];
    __shared__ uint8_t cd[ifb::kWsBand][ifb::kWsChunk];
    const uint32_t it = ws_item_of(first, n_segs, blockIdx.x);
    const ifb::WsSeg& s = segs[it];
    const uint32_t c = blockIdx.x - first[it], band = c / s.nch, k = c - band * s.nch;
    const int x0 = (int)(s.xa + k * ifb::kWsChunk) - 1, y0 = (int)(band * ifb::kWsBand) - 1;      // image position of g[0][0]
    const bool am = s.alpha_meaningful != 0;
    for (int i = threadIdx.y * 32 + threadIdx.x; i < 10 * 34; i += ifb::kWsThreads) {
        const int ty = i / 34, tx = i - ty * 34, x = x0 + tx, y = y0 + ty;
        uint32_t v = 0;
        if (x >= 0 && y >= 0 && x < (int)s.w && y < (int)s.h) v = ws_gray(__ldg(reinterpret_cast<const uint32_t*>(s.px + (size_t)y * s.stride) + x), am);
        IFB_WS_SET(g[ty][tx], (uint8_t)v);
    }
    __syncthreads();
    const int x = x0 + 1 + (int)threadIdx.x, y = y0 + 1 + (int)threadIdx.y;
    uint32_t code = 0xFFu;
    if (x < (int)s.xb && x > 0 && y > 0 && x + 1 < (int)s.w && y + 1 < (int)s.h) code = ws_centre_code(g, threadIdx.y, threadIdx.x, s.threshold);
    IFB_WS_SET(cd[threadIdx.y][threadIdx.x], (uint8_t)code);
    __syncthreads();
    if (threadIdx.y == 0) {
        const uint32_t r = threadIdx.x >> 2, f = threadIdx.x & 3, yr = (uint32_t)(y0 + 1) + r;
        if (yr < s.h) {
            // field f of a code is bits 2f + 1 .. 2f; x fields (f < 2) are relative to the centre, so they add its column
            uint32_t lo = 0xFFu, hi = 0u;
            bool any = false;
            for (uint32_t kk = 0; kk < ifb::kWsChunk; ++kk) {
                const uint32_t cc = cd[r][kk];
                if (cc == 0xFFu) continue;
                any = true;
                const uint32_t v = ((cc >> (2 * f)) & 3u) + (f < 2 ? kk + f : 0u);
                if (f & 1) hi = max(hi, v); else lo = min(lo, v);
            }
            uint8_t* out = reinterpret_cast<uint8_t*>(sums + s.sum0 + (uint64_t)yr * s.tch + s.chunk0 + k);
            IFB_WS_SET(out[f], (uint8_t)(!any ? 0xFFu : (f & 1) ? hi : lo));
        }
    }
}

// One warp per frame: Walk::region (ifb_whitespace.cc) for the full scan, window by window in the reference's order.  Window columns
// are the plan's; the box only decides the rows a top-trim takes off a window, so each window is the min / max of the summaries of
// its remaining interior rows.  The summaries of a window row (or of a run of its columns that fills the shared buffer) are loaded by
// all lanes at once before the serial decisions, which every lane makes alike; each window's summaries are then combined across the
// lanes.  res: the rectangle, the window-interior pixels visited and `bad` (DESIGN.md §5.16: a window the summaries cannot replay).
__global__ void __launch_bounds__(32) whitespace_walk_kernel(const ifb::WsJob* __restrict__ jobs, const ifb::WsColumn* __restrict__ cols,
                                                            const uint32_t* __restrict__ sums, ifb::WsResult* __restrict__ res) {
    __shared__ uint32_t buf[ifb::kWsWalkWords];
    const ifb::WsJob jb = jobs[blockIdx.x];
    const ifb::WsColumn* col = cols + jb.col0;
    const uint32_t* S = sums + jb.sum0;
    const uint32_t lane = threadIdx.x, w = jb.w, h = jb.h;
    uint32_t lo_x = w, hi_x = 0, lo_y = h, hi_y = 0, bad = 0;
    uint64_t visited = 0;
    for (uint32_t j = 0; j < jb.rows; ++j) {
        const uint32_t by = jb.y1 + (jb.wh - 2) * j, bh = min(max(3u, jb.y2 - by), jb.wh), ey = by + bh;
        const uint32_t ys = ey > h ? h - bh : by;                  // after the shift back inside the frame (bh <= h)
        const uint32_t R = bh - 2;                                  // interior rows [ys + 1, ys + 1 + R) before a trim
        for (uint32_t ca = 0; ca < jb.ncols;) {
            const uint32_t K0 = col[ca].chunk0;
            uint32_t cb = ca + 1;
            while (cb < jb.ncols && (col[cb].chunk0 + col[cb].nch - K0) * R <= ifb::kWsWalkWords) ++cb;
            const uint32_t span = col[cb - 1].chunk0 + col[cb - 1].nch - K0;
            for (uint32_t e = lane; e < span * R; e += 32) {
                const uint32_t r = e / span;
                IFB_WS_SET(buf[e], S[(uint64_t)(ys + 1 + r) * jb.tch + K0 + (e - r * span)]);
            }
            __syncwarp();
            for (uint32_t i = ca; i < cb; ++i) {
                const ifb::WsColumn cl = col[i];
                const bool in_x = lo_x < cl.bx && hi_x > cl.ex, in_y = lo_y < by && hi_y > ey;
                uint32_t t = 0;                                     // rows a top-trim takes off
                if (in_y || (in_x && lo_y < ey && ey < hi_y)) bad = 1;
                else if (in_x && hi_y > by && by > lo_y) t = min(ey - 3, hi_y) - by;
                visited += (uint64_t)(cl.xb - cl.xa) * (R - t);
                uint32_t a0 = ~0u, a1 = ~0u, a2 = ~0u, a3 = ~0u;    // min lo_x, ~max hi_x, min lo_y, ~max hi_y
                const uint32_t n = (R - t) * cl.nch;
                for (uint32_t e = lane; e < n; e += 32) {
                    const uint32_t q = e / cl.nch, kk = e - q * cl.nch, r = t + q;
                    const uint32_t v = buf[r * span + cl.chunk0 - K0 + kk];
                    if (v == ifb::kWsEmpty) continue;
                    const uint32_t xm = cl.xa + kk * ifb::kWsChunk - 1, y = ys + 1 + r;
                    a0 = min(a0, xm + (v & 0xffu));
                    a1 = min(a1, ~(xm + ((v >> 8) & 0xffu)));
                    a2 = min(a2, y - 1 + ((v >> 16) & 0xffu));
                    a3 = min(a3, ~(y + (v >> 24)));
                }
                a0 = __reduce_min_sync(0xffffffffu, a0); a1 = __reduce_min_sync(0xffffffffu, a1);
                a2 = __reduce_min_sync(0xffffffffu, a2); a3 = __reduce_min_sync(0xffffffffu, a3);
                if (a0 != ~0u) { lo_x = min(lo_x, a0); hi_x = max(hi_x, ~a1); lo_y = min(lo_y, a2); hi_y = max(hi_y, ~a3); }
            }
            __syncwarp();
            ca = cb;
        }
    }
    if (lane == 0) {
        ifb::WsResult o{};
        const bool none = lo_x == w && hi_x == 0 && lo_y == h && hi_y == 0;
        o.rect[0] = none ? 0 : lo_x; o.rect[1] = none ? 0 : lo_y; o.rect[2] = none ? w : hi_x; o.rect[3] = none ? h : hi_y;
        o.visited = visited; o.bad = bad;
        IFB_WS_SET(res[blockIdx.x], o);
    }
}
#endif
