// ifb_ycbcr_kernel.cuh -- included by ifb_kernels.cuh inside namespace ifbk, after ifb_pixel_convert_kernel.cuh (product code,
// sm_90a).  Uses only threadIdx, blockIdx, uint4, __funnelshift_r and pixel_convert's pc_fetch / pc_store / pc_item_of --
// tests/cpu_emu/ycbcr_kernel_emu.cc compiles this file with g++ under a sequential emulation of those and checks it against
// tests/ycbcr_oracle.py.
//
// The JPEG colour stage of ifb200_batch_ycbcr_to_bgra: libjpeg-turbo's fancy upsampling (h2v1 at 4:2:2, h2v2 at 4:2:0; replication for
// chroma planes of one or two columns) and its fixed-point YCbCr -> RGB, into BGRA with alpha 255.  Every job of a call in one flat
// launch over the work items of ifb_ycbcr.h; each CTA finds its item by a binary search over the items' first CTAs.  Each thread owns
// a unit: a 16-byte group of a destination row, aligned to the destination's addresses (4 BGRA pixels), at 4:2:0 in both rows 2j and
// 2j + 1 of a row pair.
//   Luma:   the group's 4 samples, read once, through pc_fetch (aligned words realigned in registers; bytes only at a row's ends).
//   Chroma: an 8-sample window from one column left of the group's first chroma column, through pc_fetch, of the rows the group
//           needs: at 4:2:0 the pair's row j and its halo rows j - 1 and j + 1 (clamped to the plane), read once for both output
//           rows.  Each output row takes the 4 columns it needs from [its first chroma column - 1, +4) out of that window -- a shift
//           inside the plane, a clamp of each column at its edges, so neighbours beyond the edges are the edge samples (libjpeg's
//           repeated edge rows and columns).  At 4:2:0 the column sums 3 near + far are formed once per column.  Nothing outside a
//           plane is read, and no full-resolution chroma is formed.
//   Stores: pc_store: a whole group is one 16-byte store; a group cut by an end of the row stores its words one by one.
// Integer arithmetic only.  Each destination byte is stored once.

// The 8 samples of columns [c0, c0 + 8) of chroma row `row` (bytes outside [0, cw) are 0, never read by yc_quad).  Column indices
// fit an int: a destination row of w pixels is at most 2^32 - 1 bytes, so w < 2^30.
__device__ __forceinline__ uint64_t yc_window(const uint8_t* plane, uint32_t stride, uint32_t row, int c0, int cw) {
    const uintptr_t rs = reinterpret_cast<uintptr_t>(plane) + (size_t)row * stride;
    uint32_t r[2];
    pc_fetch(rs + (intptr_t)c0, max(-c0, 0), min(8, cw - c0), rs, rs + cw, r);
    return (uint64_t)r[1] << 32 | r[0];
}

// The samples of columns cs .. cs + 3, each clamped to [0, cw), out of the window `win` that starts at column c0 (c0 <= cs <= c0 + 2),
// as bytes 0..3.  Inside the plane one shift; at its edges each column is clamped.
__device__ __forceinline__ uint32_t yc_quad(uint64_t win, int c0, int cs, int cw) {
    if (cs >= 0 && cs + 4 <= cw) return (uint32_t)(win >> (8 * (cs - c0)));
    uint32_t q = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) q |= (uint32_t)((win >> (8 * (min(max(cs + k, 0), cw - 1) - c0))) & 0xffu) << (8 * k);
    return q;
}

// byte k of q
__device__ __forceinline__ int yc_b(uint32_t q, int k) { return (int)((q >> (8 * k)) & 0xffu); }

__device__ __forceinline__ uint32_t yc_clamp(int v) { return (uint32_t)min(max(v, 0), 255); }

// jdcolor.c ycc_rgb_convert for one sample triple, as (B, G, R, 255)
__device__ __forceinline__ uint32_t yc_bgra(int y, int cb, int cr) {
    cb -= 128;
    cr -= 128;
    const int r = y + ((91881 * cr + 32768) >> 16);               // FIX(1.40200)
    const int g = y + ((-22554 * cb + 32768 - 46802 * cr) >> 16); // FIX(0.34414), FIX(0.71414)
    const int b = y + ((116130 * cb + 32768) >> 16);              // FIX(1.77200)
    return yc_clamp(b) | yc_clamp(g) << 8 | yc_clamp(r) << 16 | 0xff000000u;
}

// The 4 pixels of a row's group from luma `lum` and the chroma values s[0..3] of columns cs .. cs + 3 (cs = (p0 >> 1) - 1; at 4:2:0
// the column sums), with ODD = p0 & 1: pixel i is column c = (p0 + i) >> 1 = cs + 1 + ((i + ODD) >> 1), its neighbour c - 1 for an
// even x = p0 + i and c + 1 for an odd one, and (a s[c] + b s[nb] + bias) >> SH with bias BE / BO for an even / odd x.
template <int ODD, int SH, int BE, int BO>
__device__ __forceinline__ void yc_pixels(uint32_t lum, const int (&sb)[4], const int (&sr)[4], int a, uint32_t (&out)[4]) {
    const int b = 4 - a;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int k = 1 + ((i + ODD) >> 1), odd = (i + ODD) & 1, n = odd ? k + 1 : k - 1, bias = odd ? BO : BE;
        out[i] = yc_bgra((lum >> (8 * i)) & 0xff, (a * sb[k] + b * sb[n] + bias) >> SH, (a * sr[k] + b * sr[n] + bias) >> SH);
    }
}

// one destination row's group: its 16-byte aligned address G = drow + q0, the bytes [lo, hi) of the row it stores, its first pixel p0
struct YcRow {
    uintptr_t drow;
    int64_t q0, lo, hi, p0;
};

__device__ __forceinline__ YcRow yc_row(const ifb::YcItem& it, uint32_t y, uint32_t g) {
    YcRow r;
    r.drow = reinterpret_cast<uintptr_t>(it.dst) + (size_t)y * it.dst_stride;
    r.q0 = 16 * (int64_t)g - (int64_t)(r.drow & 15);
    r.lo = max(r.q0, (int64_t)0);
    r.hi = min(r.q0 + 16, 4 * (int64_t)it.w);
    r.p0 = r.q0 / 4;                                            // 4-byte aligned rows: q0 is a multiple of 4
    return r;
}

// samples of the row's pixels p0 .. p0 + 3 in a full-resolution plane (bytes of pixels outside the window are 0)
__device__ __forceinline__ uint32_t yc_full(const uint8_t* plane, uint32_t stride, uint32_t y, uint32_t w, const YcRow& r) {
    const uintptr_t rs = reinterpret_cast<uintptr_t>(plane) + (size_t)y * stride;
    uint32_t v[1];
    pc_fetch(rs + r.p0, (int)(r.lo / 4 - r.p0), (int)(r.hi / 4 - r.p0), rs, rs + w, v);
    return v[0];
}

// 4:4:4 and 4:2:2: destination row y, group g
template <int S>
__device__ __forceinline__ void yc_unit_row(const ifb::YcItem& it, uint32_t y, uint32_t g) {
    const YcRow r = yc_row(it, y, g);
    if (r.lo >= r.hi) return;
    const uint32_t lum = yc_full(it.y, it.y_stride, y, it.w, r);
    uint32_t out[4];
    if (S == IFB200_YCBCR_444) {
        const uint32_t cb = yc_full(it.cb, it.cb_stride, y, it.w, r), cr = yc_full(it.cr, it.cr_stride, y, it.w, r);
#pragma unroll
        for (int i = 0; i < 4; ++i) out[i] = yc_bgra((lum >> (8 * i)) & 0xff, (cb >> (8 * i)) & 0xff, (cr >> (8 * i)) & 0xff);
    } else {                                                    // h2v1: (a c[i] + b c[i -/+ 1] + 1 / 2) >> 2
        const int cw = (int)((it.w + 1) / 2), cs = (int)(r.p0 >> 1) - 1;
        const uint32_t qb = yc_quad(yc_window(it.cb, it.cb_stride, y, cs, cw), cs, cs, cw);
        const uint32_t qr = yc_quad(yc_window(it.cr, it.cr_stride, y, cs, cw), cs, cs, cw);
        const int sb[4] = {yc_b(qb, 0), yc_b(qb, 1), yc_b(qb, 2), yc_b(qb, 3)}, sr[4] = {yc_b(qr, 0), yc_b(qr, 1), yc_b(qr, 2), yc_b(qr, 3)};
        const int a = cw > 2 ? 3 : 4;
        if (r.p0 & 1) yc_pixels<1, 2, 1, 2>(lum, sb, sr, a, out);
        else yc_pixels<0, 2, 1, 2>(lum, sb, sr, a, out);
    }
    pc_store(r.drow + r.q0, out, (uint32_t)(r.lo - r.q0), (uint32_t)(r.hi - r.q0));
}

// 4:2:0, one output row of the pair: column sums s = a near + b far over columns cs .. cs + 3 (far = the row above for the pair's
// first row, below for its second), then (a s[i] + b s[i -/+ 1] + 8 / 7) >> 4
__device__ __forceinline__ void yc_420_row(const ifb::YcItem& it, uint32_t y, const YcRow& r, uint64_t nb_, uint64_t fb, uint64_t nr,
                                           uint64_t fr, int c0, int cw, int a) {
    if (r.lo >= r.hi) return;
    const int b = 4 - a, cs = (int)(r.p0 >> 1) - 1;
    const uint32_t qnb = yc_quad(nb_, c0, cs, cw), qfb = yc_quad(fb, c0, cs, cw), qnr = yc_quad(nr, c0, cs, cw), qfr = yc_quad(fr, c0, cs, cw);
    int sb[4], sr[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        sb[k] = a * yc_b(qnb, k) + b * yc_b(qfb, k);
        sr[k] = a * yc_b(qnr, k) + b * yc_b(qfr, k);
    }
    const uint32_t lum = yc_full(it.y, it.y_stride, y, it.w, r);
    uint32_t out[4];
    if (r.p0 & 1) yc_pixels<1, 4, 8, 7>(lum, sb, sr, a, out);
    else yc_pixels<0, 4, 8, 7>(lum, sb, sr, a, out);
    pc_store(r.drow + r.q0, out, (uint32_t)(r.lo - r.q0), (uint32_t)(r.hi - r.q0));
}

// 4:2:0: destination rows 2j and 2j + 1 (when inside the frame), group g of each.  The rows' groups start at most 3 pixels apart, so
// one 8-column window from the left halo of the earlier one holds every chroma column (and neighbour) both need.
__device__ __forceinline__ void yc_unit_420(const ifb::YcItem& it, uint32_t j, uint32_t g) {
    const uint32_t y0 = 2 * j, ch = (it.h + 1) / 2;
    const YcRow r0 = yc_row(it, y0, g), r1 = yc_row(it, y0 + 1, g);
    const bool has1 = y0 + 1 < it.h;
    if (r0.lo >= r0.hi && (!has1 || r1.lo >= r1.hi)) return;
    const int cw = (int)((it.w + 1) / 2), c0 = (int)(min(r0.p0, r1.p0) >> 1) - 1;
    const int a = cw > 2 ? 3 : 4;
    const uint32_t up = j > 0 ? j - 1 : 0, dn = j + 1 < ch ? j + 1 : ch - 1;
    const uint64_t nb_ = yc_window(it.cb, it.cb_stride, j, c0, cw), nr = yc_window(it.cr, it.cr_stride, j, c0, cw);
    const uint64_t ub = yc_window(it.cb, it.cb_stride, up, c0, cw), ur = yc_window(it.cr, it.cr_stride, up, c0, cw);
    yc_420_row(it, y0, r0, nb_, ub, nr, ur, c0, cw, a);
    if (!has1) return;
    const uint64_t db = yc_window(it.cb, it.cb_stride, dn, c0, cw), dr = yc_window(it.cr, it.cr_stride, dn, c0, cw);
    yc_420_row(it, y0 + 1, r1, nb_, db, nr, dr, c0, cw, a);
}

__global__ void __launch_bounds__(256) ycbcr_to_bgra_kernel(const ifb::YcItem* __restrict__ items, const uint32_t* __restrict__ first,
                                                            uint32_t n) {
    const uint32_t i = pc_item_of(first, n);
    const ifb::YcItem it = items[i];
    const uint64_t bands = it.sampling == IFB200_YCBCR_420 ? ((uint64_t)it.h + 1) / 2 : it.h;   // ifb::ycbcr_bands
    const uint64_t total = (uint64_t)it.groups * bands;
    const uint64_t k0 = (uint64_t)(blockIdx.x - first[i]) * ifb::kYcCtaUnits;
    if (k0 >= total) return;
    const uint32_t count = (uint32_t)min(total - k0, (uint64_t)ifb::kYcCtaUnits);
    if (it.sampling == IFB200_YCBCR_420) {
        for (uint32_t t = threadIdx.x; t < count; t += ifb::kYcThreads) {
            const uint32_t k = (uint32_t)k0 + t;
            yc_unit_420(it, k / it.groups, k % it.groups);
        }
    } else if (it.sampling == IFB200_YCBCR_422) {
        for (uint32_t t = threadIdx.x; t < count; t += ifb::kYcThreads) {
            const uint32_t k = (uint32_t)k0 + t;
            yc_unit_row<IFB200_YCBCR_422>(it, k / it.groups, k % it.groups);
        }
    } else {
        for (uint32_t t = threadIdx.x; t < count; t += ifb::kYcThreads) {
            const uint32_t k = (uint32_t)k0 + t;
            yc_unit_row<IFB200_YCBCR_444>(it, k / it.groups, k % it.groups);
        }
    }
}
