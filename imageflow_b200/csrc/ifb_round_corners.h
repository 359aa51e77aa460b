// ifb_round_corners.h -- host planner of flow_bitmap_bgra_clear_around_rounded_corners (graphics/rounded_corners.rs:1-346).
// Product code, plain C++ without CUDA calls (tests/cpu_emu links it unchanged): validation of each descriptor, get_radius and
// plan_quadrants in f32 with the reference's operation order, a cover of every pixel the op can touch as disjoint rectangles, and
// the cut of that cover into CTA tiles of one flat launch.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/ifb200.h"

namespace ifb {

// One quadrant of rounded_corners.rs:161-185 as the kernel reads it (the per-row edges are computed per pixel from these).
struct RcQuad {
    float cx, cy;                                  // centre_x, centre_y
    float roi, ros, raw;                           // radius_of_influence, radius_of_solid, radius_aliasing_width (:256-262)
    float roi2, ros2;                              // their squares
    uint32_t y, bottom;                            // quadrant.y, quadrant.bottom()
    uint32_t start_y, end_y;                       // rows of the arc (:220-227)
    uint32_t clear_from, clear_to;                 // columns cleared on the quadrant's other rows (:242-250; only CIRCLE has any)
    uint32_t is_left;
};

// One job as the kernel reads it.  Quadrants in the reference's loop order: TopLeft, TopRight, BottomLeft, BottomRight.
struct RcJob {
    uint8_t* px; uint32_t w, h, stride;
    uint32_t matte;                                // BGRA8 packed little-endian (b | g << 8 | r << 16 | a << 24)
    uint32_t top_rows;                             // rows [0, top_rows) are filled in the TopLeft step (:209-212; CIRCLE only)
    uint32_t bottom_from;                          // rows [bottom_from, h) are filled in the BottomLeft step (:213-216; CIRCLE only)
    uint32_t pad_;
    RcQuad q[4];
};

// One CTA of round_corners_kernel: pixels [first, first + count) of a cover rectangle of job `job` whose top-left pixel is (x0, y0)
// and width rw, counted row by row.
constexpr uint32_t kRcThreads = 256, kRcTilePixels = 2048;
struct RcTile { uint32_t job, x0, y0, rw, first, count; };

// A rectangle of the cover: columns [x0, x0 + w), rows [y0, y0 + h).  fill_only: every pixel of it is overwritten with the matte
// (so its old contents are never read).
struct RcRect { uint32_t x0, y0, w, h; bool fill_only; };

struct RcWork {
    std::vector<RcJob> jobs; std::vector<RcTile> tiles;
};

// Empty when d is a valid descriptor, else why it is not; *code, when given, = IFB200_ERR_INVALID_ARGUMENT (its only status).
// Degenerate radii are not errors: the plan gives them the reference's meaning.
std::string round_corners_check(const ifb200_round_corners_desc& d, int* code = nullptr);

// Appends the job of a valid descriptor on its bitmap (d.px, d.stride) and the tiles of its cover to `wk`, and the cover itself to
// `*rects` when given.  Nothing for an empty window.
void round_corners_plan(const ifb200_round_corners_desc& d, RcWork& wk, std::vector<RcRect>* rects = nullptr);

// Checks every descriptor of one call, then plans all of them into wk.  Empty on success; else "round corners job i: <why>" for the
// first rejected descriptor, with *code = its status, and nothing planned.
std::string round_corners_prepare(const ifb200_round_corners_desc* d, size_t n, RcWork& wk, int* code);

// Disjoint rectangles that together cover every pixel any step of `job` can write.  Each row's cover is a prefix [0, L) and a
// suffix [R, w) of the row (every step works from the left or the right edge); inside a corner's square the cover also holds the
// pixels within the solid radius, which no step writes.  Appends to `out`.
void round_corners_cover(const RcJob& job, std::vector<RcRect>& out);

}  // namespace ifb
