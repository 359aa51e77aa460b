/*
 * round_corners_oracle.c -- CPU ORACLE of graphics/rounded_corners.rs:1-346 (flow_bitmap_bgra_clear_around_rounded_corners).
 * TEST INFRASTRUCTURE, NOT PRODUCT CODE: tests/round_corners_oracle.py compiles it together with oracle/ifb_oracle.c (whose
 * transfer tables and uchar_clamp_ff it uses, unchanged) into a library in a temporary directory.  The product never links it.
 *
 * A plain sequential transcription: the quadrants in the reference's order, each with its fills, edge clears and arc rows,
 * row by row and column by column.  f32 throughout, in the reference's operation order (no contraction: -ffp-contract=off).
 */
#include <math.h>
#include <string.h>

#include "../oracle/ifb_oracle.h"

static uint8_t g_lut16k[16384];
static float g_t_lin[256];
static int g_tables_ready = 0;
static void ensure_tables(void) {
    if (g_tables_ready) return;
    ifo_linear_to_srgb_table(g_lut16k);
    ifo_byte_to_float_table(1, g_t_lin);
    g_tables_ready = 1;
}
static uint8_t lut16k(float lin) {                            /* lut.rs:4-8 */
    float s = lin * 16383.0f;
    if (!(s > 0.0f)) s = 0.0f;                                /* clamp; NaN -> 0 like `NaN as usize` */
    if (s > 16383.0f) s = 16383.0f;
    return g_lut16k[(int)s];
}

static size_t rc_as_usize(float f) {                          /* `f32 as usize`: saturating, NaN -> 0 */
    if (!(f > 0.0f)) return 0;
    if (f >= 18446744073709551616.0f) return (size_t)-1;
    return (size_t)f;
}
static float rc_clamp(float v, float lo, float hi) {          /* f32::clamp (NaN stays NaN) */
    if (v < lo) v = lo;
    if (v > hi) v = hi;
    return v;
}
static float rc_max(float a, float b) { return a != a ? b : (b != b ? a : (a > b ? a : b)); }   /* f32::max */
static float rc_min(float a, float b) { return a != a ? b : (b != b ? a : (a < b ? a : b)); }   /* f32::min */

typedef struct { int which; uint32_t x, y, width, height; float radius, cx, cy; int is_top, is_left; } rc_quadrant;
enum { RC_TL = 0, RC_TR = 1, RC_BR = 2, RC_BL = 3 };          /* Quadrant (:161-167) */

static void rc_plan_custom(const float r[4], uint32_t w, uint32_t h, rc_quadrant q[4]) {   /* :66-156; r = [tl, tr, bl, br] */
    uint32_t rhw = w / 2, bhh = h / 2, lhw = w - rhw, thh = h - bhh;
    rc_quadrant a = {RC_TL, 0, 0, lhw, thh, r[0], r[0], r[0], 1, 1};
    rc_quadrant b = {RC_TR, lhw, 0, rhw, thh, r[1], (float)w - r[1], r[1], 1, 0};
    rc_quadrant c = {RC_BL, 0, thh, lhw, bhh, r[2], r[2], (float)h - r[2], 0, 1};
    rc_quadrant d = {RC_BR, lhw, thh, rhw, bhh, r[3], (float)w - r[3], (float)h - r[3], 0, 0};
    q[0] = a; q[1] = b; q[2] = c; q[3] = d;
}

static void rc_put(uint8_t* px, uint32_t stride, uint8_t* mask, uint32_t w, size_t x, size_t y, const uint8_t v[4], uint8_t mark) {
    memcpy(px + y * stride + x * 4, v, 4);
    if (mask) mask[y * w + x] = mark;
}
static void rc_fill_rect(uint8_t* px, uint32_t stride, uint8_t* mask, uint32_t w, uint32_t x1, uint32_t y1, uint32_t x2, uint32_t y2,
                         const uint8_t m[4]) {                /* BitmapWindowMut::fill_rectangle(x, y, x2, y2) */
    for (uint32_t y = y1; y < y2; ++y)
        for (uint32_t x = x1; x < x2; ++x) rc_put(px, stride, mask, w, x, y, m, 1);
}

/* mode: RoundCornersMode in declaration order (0 Percentage, 1 Pixels, 2 Circle, 3 PercentageCustom, 4 PixelsCustom); radius[] in
 * the field order top_left, top_right, bottom_right, bottom_left ([0] alone for 0/1; unused for 2).  touched (optional, w * h bytes,
 * row pitch w): for every pixel the op writes, 1 if its last write was the matte, 2 if it was a blend; 0 elsewhere.
 * Returns 0, or IFO_ERR_INVALID_ARGUMENT for an unknown mode. */
int rco_round_corners(uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, int mode, const float radius[4], const uint8_t matte[4],
                      uint8_t* touched) {
    if (mode < 0 || mode > 4) return IFO_ERR_INVALID_ARGUMENT;
    if (w == 0 || h == 0) return IFO_OK;
    ensure_tables();
    const float alpha_to_float = 1.0f / 255.0f;
    const float matte_a = (float)matte[3] * alpha_to_float;
    const float matte_b = g_t_lin[matte[0]], matte_g = g_t_lin[matte[1]], matte_r = g_t_lin[matte[2]];
    const float volumetric_offset = 0.56419f;

    /* get_radius (:5-33): radius[] is in RoundCornersMode field order (tl, tr, br, bl); Custom is [tl, tr, bl, br] */
    const float smallest = (float)(w < h ? w : h);
    float r[4];
    rc_quadrant q[4];
    if (mode == 2) {                                          /* Circle (:46-64) */
        uint32_t s = w < h ? w : h;
        uint32_t offset_x = w > h ? (w - h) / 2 : 0, offset_y = h > w ? (h - w) / 2 : 0;
        float v = smallest / 2.0f;
        r[0] = r[1] = r[2] = r[3] = v;
        rc_plan_custom(r, s, s, q);
        for (int i = 0; i < 4; ++i) {
            q[i].x += offset_x; q[i].y += offset_y;
            q[i].cx += (float)offset_x; q[i].cy += (float)offset_y;
        }
    } else {
        if (mode == 0) { float v = smallest * rc_clamp(radius[0], 0.0f, 100.0f) / 200.0f; r[0] = r[1] = r[2] = r[3] = v; }
        else if (mode == 1) { float v = rc_clamp(radius[0], 0.0f, smallest / 2.0f); r[0] = r[1] = r[2] = r[3] = v; }
        else {
            static const int field[4] = {0, 1, 3, 2};         /* [tl, tr, bl, br] from (tl, tr, br, bl) */
            for (int i = 0; i < 4; ++i)
                r[i] = mode == 3 ? smallest * rc_clamp(radius[field[i]], 0.0f, 100.0f) / 200.0f : rc_clamp(radius[field[i]], 0.0f, smallest / 2.0f);
        }
        rc_plan_custom(r, w, h, q);
    }

    for (int qi = 0; qi < 4; ++qi) {                          /* :204-343 */
        const rc_quadrant* Q = &q[qi];
        const uint32_t bottom = Q->y + Q->height, right = Q->x + Q->width;
        if (Q->y > 0 && Q->which == RC_TL) rc_fill_rect(px, stride, touched, w, 0, 0, w, Q->y, matte);
        if (h > bottom && Q->which == RC_BL) rc_fill_rect(px, stride, touched, w, 0, bottom, w, h, matte);
        const size_t radius_ceil = rc_as_usize(ceilf(Q->radius));
        size_t start_y = Q->is_top ? Q->y : (radius_ceil > bottom ? 0 : bottom - radius_ceil);
        size_t end_y = Q->is_top ? Q->y + radius_ceil : bottom;
        if (end_y > h) end_y = h;                             /* where the reference would index out of bounds */
        const uint32_t clear_x_from = Q->is_left ? 0 : right, clear_x_to = Q->is_left ? Q->x : w;
        if (clear_x_from != clear_x_to) {
            for (size_t y = Q->y; y < start_y; ++y) rc_fill_rect(px, stride, touched, w, clear_x_from, (uint32_t)y, clear_x_to, (uint32_t)y + 1, matte);
            for (size_t y = end_y; y < bottom; ++y) rc_fill_rect(px, stride, touched, w, clear_x_from, (uint32_t)y, clear_x_to, (uint32_t)y + 1, matte);
        }
        const float radius_of_influence = Q->radius + (1.0f - volumetric_offset);
        const float radius_of_solid = Q->radius - volumetric_offset;
        const float radius_aliasing_width = radius_of_influence - radius_of_solid;
        const float radius_of_influence_squared = radius_of_influence * radius_of_influence;
        const float radius_of_solid_squared = radius_of_solid * radius_of_solid;
        for (size_t y = start_y; y < end_y; ++y) {
            uint8_t* row = px + y * stride;
            const float yf = (float)y + 0.5f;
            const float y_dist_from_center = fabsf(Q->cy - yf);
            const float y_dist_squared = y_dist_from_center * y_dist_from_center;
            const float x_dist_from_center_solid = sqrtf(rc_max(radius_of_solid_squared - y_dist_squared, 0.0f));
            const float x_dist_from_center_influenced = sqrtf(rc_max(radius_of_influence_squared - y_dist_squared, 0.0f));
            size_t edge_solid_x1 = rc_as_usize(rc_max(ceilf(Q->cx - x_dist_from_center_solid), 0.0f));
            size_t edge_solid_x2 = rc_as_usize(rc_min(floorf(Q->cx + x_dist_from_center_solid), (float)w));
            size_t edge_influence_x1 = rc_as_usize(rc_max(floorf(Q->cx - x_dist_from_center_influenced), 0.0f));
            size_t edge_influence_x2 = rc_as_usize(rc_min(ceilf(Q->cx + x_dist_from_center_influenced), (float)w));
            if (edge_influence_x1 > w) edge_influence_x1 = w;     /* slice bounds the reference would panic on */
            if (Q->is_left) { for (size_t x = 0; x < edge_influence_x1; ++x) rc_put(px, stride, touched, w, x, y, matte, 1); }
            else { for (size_t x = edge_influence_x2; x < w; ++x) rc_put(px, stride, touched, w, x, y, matte, 1); }
            size_t alias_from = Q->is_left ? edge_influence_x1 : edge_solid_x2;
            size_t alias_to = Q->is_left ? edge_solid_x1 : edge_influence_x2;
            if (alias_to > w) alias_to = w;
            for (size_t x = alias_from; x < alias_to; ++x) {
                const float xf = (float)x + 0.5f;
                const float diff_x = Q->cx - xf;
                const float distance = sqrtf(diff_x * diff_x + y_dist_squared);
                if (distance > radius_of_influence) {
                    rc_put(px, stride, touched, w, x, y, matte, 1);
                } else if (distance > radius_of_solid) {
                    const float intensity = (distance - radius_of_solid) / radius_aliasing_width;
                    uint8_t* p = row + x * 4;
                    const float pixel_a_f32 = (float)(int32_t)p[3] * alpha_to_float * (1.0f - intensity);
                    const float m_a = (1.0f - pixel_a_f32) * matte_a;
                    const float final_a = m_a + pixel_a_f32;
                    uint8_t v[4];
                    v[0] = lut16k((g_t_lin[p[0]] * pixel_a_f32 + matte_b * m_a) / final_a);
                    v[1] = lut16k((g_t_lin[p[1]] * pixel_a_f32 + matte_g * m_a) / final_a);
                    v[2] = lut16k((g_t_lin[p[2]] * pixel_a_f32 + matte_r * m_a) / final_a);
                    v[3] = ifo_uchar_clamp_ff(255.0f * final_a);
                    rc_put(px, stride, touched, w, x, y, v, 2);
                }
            }
        }
    }
    return IFO_OK;
}
