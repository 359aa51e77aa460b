// ifb_whitespace.h -- host half of detect_content (graphics/whitespace.rs:284-421): the reference's window walk, replayed
// over the per-pixel code map that whitespace_codes_kernel produces.  Product code: must not include or link anything from oracle/.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/ifb200.h"

namespace ifb {

// Code of pixel (x, y) as the centre of its 3x3 neighbourhood (whitespace.rs:525-613, the part of sobel_scharr_detect
// that does not depend on the window): 0xFF = border pixel or Scharr value <= threshold; otherwise
// bits 1:0 local_min_x (0..2), 3:2 local_max_x - 1, 5:4 local_min_y, 7:6 local_max_y - 1, relative to (x - 1, y - 1).
constexpr uint8_t kNoEdge = 0xFF;

// detect_content over a w*h code map (row pitch w).  rect = {x1, y1, x2, y2}.  `centres`, if not null, receives the number of
// window-interior pixels visited.  Returns false for an empty or oversized bitmap.
bool detect_content_from_codes(const uint8_t* codes, uint32_t w, uint32_t h, uint32_t rect[4], uint64_t* centres);

// ---- the batched form (ifb200_batch_detect_content_many): planned here, run by whitespace_segments_kernel + whitespace_walk_kernel.
// Of the reference's scans only the full one ever searches (the twelve quick strips are all empty, DESIGN.md §5.16), its windows are
// never skipped and their columns never depend on the bounding box: the box only trims interior rows off a window's top.  So the
// codes are reduced per (row, 32-column chunk of a window column's interior) into summaries, and the walk replays the window order
// over those.  A summary is one word: bytes {lo, hi, lo_dy, hi_dy} = min (x - 1 + local min x) - (x0 - 1), max (x + local max x - 1)
// - (x0 - 1), min local min y, max local max y - 1 over the row's edge centres x in the chunk [x0, x0 + 32); kWsEmpty when it has none.
constexpr uint32_t kWsChunk = 32, kWsBand = 8, kWsThreads = kWsChunk * kWsBand;
constexpr uint32_t kWsEmpty = 0xffffffffu;
constexpr uint32_t kWsWalkWords = 4096;                  // the walk's shared buffer of summaries: a window row, or a run of its columns

// One window column of the full scan: [bx, ex) before the shift back inside the frame (the walk's "already inside the box" test
// reads these) and its interior columns [xa, xb) after it; its chunks are chunk0 .. chunk0 + nch - 1 of a row of summaries.
struct WsColumn { uint32_t bx, ex, xa, xb, chunk0, nch; };

// A frame that needs a walk (w, h >= 3).  Window row j starts at y1 + (wh - 2) j and is min(max(3, y2 - by), wh) rows high; its
// columns are cols[col0 .. col0 + ncols).  Its summaries are sums[sum0 + y * tch + chunk] for every row y < h.
struct WsJob {
    uint32_t w, h, y1, y2, wh, rows, col0, ncols, tch, pad;
    uint64_t sum0;
};
// One (frame, window column) of whitespace_segments_kernel: CTA c of it takes chunk c % nch, rows [kWsBand (c / nch), +kWsBand).
struct WsSeg {
    const uint8_t* px;
    uint32_t w, h, stride, alpha_meaningful;
    int32_t threshold;
    uint32_t xa, xb, chunk0, nch, tch;
    uint64_t sum0;
};
// What the walk leaves per frame: the rectangle, the window-interior pixels visited and 1 in `bad` if a window ever met the box in a
// way the summaries cannot replay (a skip, or a shrink of its columns or bottom), which DESIGN.md §5.16 shows cannot happen.
struct WsResult { uint32_t rect[4]; uint64_t visited; uint32_t bad, pad; };

struct WsWork {
    std::vector<WsJob> jobs;
    std::vector<uint32_t> job_of;                        // job_of[k] = the call's index of jobs[k]
    std::vector<WsColumn> cols;
    std::vector<WsSeg> segs;
    std::vector<uint32_t> first;                         // first[i] = the first CTA of segs[i]; first.back() = the number of CTAs
    uint64_t n_sums = 0;                                 // summary words of the call
    uint64_t ctas() const { return first.empty() ? 0 : first.back(); }
};

// The full scan's grid of a w x h frame (w, h >= 3): window rows and columns as Walk::region lays them out.  Appends the columns to
// cols and fills y1, y2, wh, rows, ncols of job (rows = 0 when the scan has no window).
void whitespace_grid(uint32_t w, uint32_t h, WsJob& job, std::vector<WsColumn>& cols);

// Empty when d is a valid descriptor, else why not (*code = IFB200_ERR_INVALID_ARGUMENT).
std::string detect_content_check(const ifb200_detect_content_desc& d, int* code = nullptr);

// Checks every descriptor (check_each: "detect_content job i: <why>"), then plans every frame of at least 3 x 3 into wk.  The
// rectangles of all frames are set to the whole bitmap in rects (4 per job, may be null) and visited to 0 (may be null); the walk
// overwrites those of the frames in wk.jobs.
std::string detect_content_prepare(const ifb200_detect_content_desc* d, size_t n, WsWork& wk, int* code, uint32_t* rects, uint64_t* visited);

}  // namespace ifb
