// ifb_engine.cu -- host side of libifb200.so: plans, batch object, C ABI (include/ifb200.h).
//
// Mirrors the reference seam graphics/scaling.rs:19-90 (validation + dispatch on the canvas'
// compositing mode) and color_matrix.rs:5-28; the arithmetic runs in ifb_kernels.cuh on the GPU.
// There is deliberately no CPU path in this file: if CUDA is unusable the calls fail.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <thread>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <stdexcept>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "../../include/ifb200.h"
#include "ifb_kernels.cuh"
#include "ifb_weights.h"
#include "ifb_whitespace.h"

namespace {

using namespace ifbk;

struct Err {
    int code; std::string msg;
};
#define IFB_THROW(code_, ...) do { char b_[512]; snprintf(b_, sizeof b_, __VA_ARGS__); throw Err{(code_), std::string(b_)}; } while (0)
#define CUDA_OK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
    int c_ = (e_ == cudaErrorMemoryAllocation) ? IFB200_ERR_OUT_OF_MEMORY : \
             (e_ == cudaErrorNoDevice || e_ == cudaErrorInsufficientDriver || e_ == cudaErrorInvalidDevice) ? IFB200_ERR_NO_DEVICE : IFB200_ERR_CUDA; \
    IFB_THROW(c_, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); } } while (0)

// Makes `dev` the calling thread's current device for the lifetime of the object and restores the caller's device afterwards:
// the library never leaves a caller with a different current device than it came with.
struct DeviceScope {
    int prev = -1;
    explicit DeviceScope(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); prev = -1; }
        cudaError_t e = cudaSetDevice(dev);
        if (e != cudaSuccess) {
            char b[256]; snprintf(b, sizeof b, "cudaSetDevice(%d) failed: %s", dev, cudaGetErrorString(e));
            throw std::runtime_error(b);
        }
    }
    ~DeviceScope() { if (prev >= 0) cudaSetDevice(prev); }
    DeviceScope(const DeviceScope&) = delete;
    DeviceScope& operator=(const DeviceScope&) = delete;
};

// adds the lifetime of the object, in seconds, to `acc` (host-side profile of the enqueue path; inclusive, nesting allowed)
struct Tick {
    double& acc; std::chrono::steady_clock::time_point t0;
    explicit Tick(double& a) : acc(a), t0(std::chrono::steady_clock::now()) {}
    ~Tick() { acc += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(); }
};

void put_err(char* err, size_t cap, const std::string& m) {
    if (!err || cap == 0) return;
    size_t n = std::min(cap - 1, m.size());
    memcpy(err, m.data(), n);
    err[n] = 0;
}

template <class F>
int guarded(char* err, size_t cap, F&& f) {
    try {
        f();
        if (err && cap) err[0] = 0;
        return IFB200_OK;
    } catch (const Err& e) {
        put_err(err, cap, e.msg);
        return e.code;
    } catch (const std::bad_alloc&) {
        put_err(err, cap, "host allocation failed");
        return IFB200_ERR_OUT_OF_MEMORY;
    } catch (const std::runtime_error& e) {                   // DeviceScope: the device could not be made current
        put_err(err, cap, e.what());
        return IFB200_ERR_CUDA;
    } catch (const std::exception& e) {
        put_err(err, cap, e.what());
        return IFB200_ERR_INVALID_STATE;
    } catch (...) {
        put_err(err, cap, "unknown failure");
        return IFB200_ERR_INVALID_STATE;
    }
}

// ------------------------------------------------------------------------------------------------
// device buffer helper
template <class T>
struct DevVec {
    T* p = nullptr; size_t n = 0;
    void upload(const std::vector<T>& h) {
        n = h.size();
        if (!n) return;
        CUDA_OK(cudaMalloc(&p, n * sizeof(T)));
        CUDA_OK(cudaMemcpy(p, h.data(), n * sizeof(T), cudaMemcpyHostToDevice));
    }
    ~DevVec() { if (p) cudaFree(p); }
    DevVec() = default;
    DevVec(const DevVec&) = delete;
    DevVec& operator=(const DevVec&) = delete;
};

// Several host arrays packed into ONE device allocation and ONE asynchronous copy (through pinned staging) on the
// stream that is about to use them.  Streams other than the uploading one wait on `ready` (see use_on()).
struct DevBlob {
    uint8_t* p = nullptr;
    std::vector<uint8_t> host;
    cudaEvent_t ready = nullptr; bool owns_ready = true; bool done = false; cudaStream_t up_stream = nullptr;
    size_t add(const void* src, size_t bytes) {
        const size_t off = (host.size() + 255) / 256 * 256;
        host.resize(off + bytes);
        if (bytes && src) memcpy(host.data() + off, src, bytes);
        return off;
    }
    template <class T> size_t add(const std::vector<T>& v) { return add(v.data(), v.size() * sizeof(T)); }
    // a zero-filled region to be built in place: take the pointer with host_at() AFTER the last add of the group
    size_t add_zeroed(size_t bytes) { return add(nullptr, bytes); }
    template <class T> T* host_at(size_t off) { return reinterpret_cast<T*>(host.data() + off); }
    void reserve(size_t bytes) { host.reserve(bytes); }
    void commit(ifb200_batch* b, cudaStream_t st);
    void use_on(cudaStream_t st) {
        if (done || st == up_stream) return;
        if (cudaEventQuery(ready) == cudaSuccess) { done = true; return; }
        CUDA_OK(cudaStreamWaitEvent(st, ready, 0));
    }
    template <class T> const T* at(size_t off) const { return reinterpret_cast<const T*>(p + off); }
    ~DevBlob() { if (ready && owns_ready) cudaEventDestroy(ready); }     // the memory belongs to the batch's table arena (and a shared event to the batch)
    DevBlob() = default;
    DevBlob(const DevBlob&) = delete;
    DevBlob& operator=(const DevBlob&) = delete;
};

struct AxisOnDev {
    size_t o_left = 0, o_right = 0, o_off = 0, o_w = 0;
    void add_to(DevBlob& blob, const ifb::AxisWeights& a) { o_left = blob.add(a.left); o_right = blob.add(a.right); o_off = blob.add(a.offset); o_w = blob.add(a.w); }
    AxisDev view(const DevBlob& blob) const { return AxisDev{blob.at<uint32_t>(o_left), blob.at<uint32_t>(o_right), blob.at<uint32_t>(o_off), blob.at<float>(o_w)}; }
};

// ------------------------------------------------------------------------------------------------
// Streaming H-then-V ring kernel (ifb_hv_kernel.cuh): host tables of one plan.
struct HvTables {
    int max_cols = 0, n_strips = 0;
    uint32_t hw_stride = 0;             // weight records per strip (the longest pixel stream + the chunk the kernel reads ahead), <= cap
    std::vector<HvStripDev> strips;     // host copy (band choice, tests)
    DevBlob blob;                       // strips, hw, hdone, vw, vdone: one allocation, one asynchronous copy
    size_t o_strips = 0, o_hw = 0, o_hdone = 0, o_vw = 0, o_vdone = 0;
};

struct Plan {
    uint32_t in_w, in_h, out_w, out_h;
    ifb::AxisWeights wv, wh;
    AxisOnDev dv, dh; std::unique_ptr<DevBlob> axes;   // CSR windows on the device: only the tile kernel and the generic pair read them
    // tile kernel (small windows: up-scales, 1:1, mild down-scales)
    bool tile_ok = false; TilePlanDev tile{};
    // per output row: its V window padded with zeros to the six source rows of its quad; per quad: first of those rows + 1 (0 = the
    // quad does not fit); per output column: the H window padded to four taps (ifb_tile2_kernel.cuh)
    std::vector<float> tile_vw, tile_hw; std::vector<uint32_t> tile_vq; size_t o_tile_vw = 0, o_tile_vq = 0, o_tile_hw = 0;
    // ring kernel
    bool hv_ok = false; std::string hv_reason;
    int av = 0;                          // ring depth of the kernel variant: 4 or 6 (both axes)
    std::map<int, std::unique_ptr<HvTables>> by_cols;   // by the largest strip width allowed (IFB200_OPT_STRIP_COLUMNS)
    std::vector<int> cols_failed;        // strip widths at which some column's window does not fit the weight table: not ring
};

bool monotone(const ifb::AxisWeights& a) {
    for (uint32_t i = 1; i < a.out_size; ++i)
        if (a.left[i] < a.left[i - 1] || a.right[i] < a.right[i - 1]) return false;
    return true;
}

// smallest A such that at most A consecutive outputs are open at any source sample: left[y+A] > right[y] for all y
int ring_depth(const ifb::AxisWeights& a) {
    int need = 1;
    for (; need <= 64; ++need) {
        bool ok = true;
        for (uint32_t y = 0; y + need < a.out_size && ok; ++y) ok = a.left[y + need] > a.right[y];
        if (ok) break;
    }
    return need;
}

void build_hv(Plan& p) {
    if (!monotone(p.wv) || !monotone(p.wh)) { p.hv_reason = "non-monotone windows"; return; }
    const int need = std::max(ring_depth(p.wv), ring_depth(p.wh));
    if (need > 6) { p.hv_reason = "ring depth " + std::to_string(need) + " > 6"; return; }
    p.av = need <= 4 ? 4 : 6;
    p.hv_ok = true;
}

// tile kernel: 64 x 32 output pixels per CTA at a time (kTile2W x kTile2H); usable when the source extent of every tile fits in shared memory
void build_tile(Plan& p) {
    if (!monotone(p.wv) || !monotone(p.wh)) return;
    TilePlanDev t{};
    t.in_w = p.in_w; t.in_h = p.in_h; t.out_w = p.out_w; t.out_h = p.out_h;
    t.tow = kTile2W; t.toh = kTile2H;
    t.tiles_x = (int)((p.out_w + t.tow - 1) / t.tow); t.tiles_y = (int)((p.out_h + t.toh - 1) / t.toh);
    for (int tx = 0; tx < t.tiles_x; ++tx) {
        const uint32_t X0 = tx * t.tow, X1 = std::min<uint32_t>(X0 + t.tow, p.out_w);
        t.max_ic = std::max<int>(t.max_ic, (int)(p.wh.right[X1 - 1] - p.wh.left[X0] + 1));
    }
    for (int ty = 0; ty < t.tiles_y; ++ty) {
        const uint32_t Y0 = ty * t.toh, Y1 = std::min<uint32_t>(Y0 + t.toh, p.out_h);
        t.max_ir = std::max<int>(t.max_ir, (int)(p.wv.right[Y1 - 1] - p.wv.left[Y0] + 1));
    }
    if (Tile2Smem::make(t.max_ir, t.max_ic, true).total > 96u * 1024u) return;   // large windows: the ring kernel or the generic pair
    // tables of the register forms (kernel header): everything that depends only on the plan is prepared here
    const int rows_pad = t.tiles_y * kTile2H;
    p.tile_vw.assign((size_t)rows_pad * 8, 0.0f);
    p.tile_vq.assign((size_t)rows_pad / 4, 0u);
    for (int ty = 0; ty < t.tiles_y; ++ty) {
        const uint32_t Y0 = ty * t.toh, Y1 = std::min<uint32_t>(Y0 + t.toh, p.out_h);
        const uint32_t r0 = p.wv.left[Y0], r1 = p.wv.right[Y1 - 1];
        for (uint32_t yq = Y0; yq < Y1; yq += 4) {
            const uint32_t b0 = std::min(p.wv.left[yq], std::max(r1 - std::min<uint32_t>(r1, kTile2Span - 1), r0));
            bool fit = r1 - r0 + 1 >= (uint32_t)kTile2Span;
            for (uint32_t y = yq; y < std::min(yq + 4, Y1); ++y) fit = fit && p.wv.left[y] >= b0 && p.wv.right[y] < b0 + kTile2Span;
            p.tile_vq[yq / 4] = fit ? b0 + 1 : 0u;
            if (!fit) continue;
            for (uint32_t y = yq; y < std::min(yq + 4, Y1); ++y)
                for (uint32_t j = p.wv.left[y]; j <= p.wv.right[y]; ++j) p.tile_vw[(size_t)y * 8 + (j - b0)] = p.wv.w[p.wv.offset[y] + (j - p.wv.left[y])];
        }
    }
    t.h4 = p.wh.max_taps <= 4 ? 1 : 0;
    p.tile_hw.assign(t.h4 ? (size_t)t.tiles_x * kTile2W * 4 : 4, 0.0f);
    if (t.h4)
        for (uint32_t x = 0; x < p.out_w; ++x)
            for (uint32_t j = p.wh.left[x]; j <= p.wh.right[x]; ++j) p.tile_hw[(size_t)x * 4 + (j - p.wh.left[x])] = p.wh.w[p.wh.offset[x] + (j - p.wh.left[x])];
    p.tile = t; p.tile_ok = true;
}

template <class F> void hv_for_av(int av, F&& f) { if (av == 4) f(std::integral_constant<int, 4>{}); else f(std::integral_constant<int, 6>{}); }

// host half: strips, per-strip H weights by ring slot in pixel-stream order, completion counts + V-pass marks, V weights by ring slot
//
// A strip's pixel stream is walked by the kernel in pairs of chunks (eight source columns).  Output columns that complete are parked in
// the warp's exchange buffer (room for cg columns) and the V pass of the parked columns (a "group") runs at the END of a pair that
// carries a mark (bit 7 of the completion byte of the pair's last column): the marks are placed here, as late as the buffer allows,
// and a strip may hold at most ng groups (the kernel keeps one set of vertical accumulators per group in registers).
std::unique_ptr<HvTables> hv_tables_host(const Plan& p, int cols_key) {
    auto ht = std::make_unique<HvTables>();
    const int max_cols = cols_key & 0xffff, ng = cols_key >> 16, cg = 32 / (p.av / 2);   // hv_cols(): widest strip | groups the kernel variant holds << 16; columns per V-pass group
    ht->max_cols = max_cols;
    const auto& h = p.wh; const auto& v = p.wv;
    const int av = p.av, avp = av == 4 ? 4 : 8, cap = 16384 / (avp * 4);
    const uint32_t col_cap = (uint32_t)max_cols;             // the caller has clipped it to what the kernel variant can hold (hv_cols)
    // the pixel stream of a strip starts at a multiple of k0_align source columns (16 bytes: TMA box origins stay 16-byte aligned
    // for bitmaps whose window starts on a 16-byte boundary; IFB200_DEBUG_K0_ALIGN=1 lifts that, for experiments)
    static const uint32_t k0_align = [] { const char* e = getenv("IFB200_DEBUG_K0_ALIGN"); const int v = e ? atoi(e) : 4; return (uint32_t)(v >= 1 && v <= 16 ? v : 4); }();
    auto k0_of = [&](uint32_t X0) { return h.left[X0] / k0_align * k0_align; };
    // V-pass marks of [X0,X1): indices of the chunk PAIRS (eight source columns) after which a V pass runs; returns false if some
    // pair completes more than cg columns or the strip needs more than ng groups
    auto marks_of = [&](uint32_t X0, uint32_t X1, std::vector<uint32_t>* marks) {
        const uint32_t k0 = k0_of(X0);
        uint32_t parked = 0, X = X0, groups = 0;
        const uint32_t npairs = (h.right[X1 - 1] - k0 + 1 + 15) / 16 * 2;
        for (uint32_t c = 0; c < npairs; ++c) {
            uint32_t m = 0;
            while (X < X1 && h.right[X] <= k0 + c * 8 + 7) { ++m; ++X; }
            if (m > (uint32_t)cg) return false;
            if (parked + m > (uint32_t)cg) { if (marks) marks->push_back(c - 1); ++groups; parked = 0; }
            parked += m;
        }
        if (parked) { if (marks) marks->push_back(npairs - 1); ++groups; }
        return groups <= (uint32_t)ng;
    };
    auto fits = [&](uint32_t X0, uint32_t X1) {   // [X0,X1): at most col_cap columns in at most ng groups, and a pixel stream (whole stages of 16, plus the chunk the kernel's pipeline reads ahead) within the table
        return X1 - X0 <= col_cap && (h.right[X1 - 1] - k0_of(X0) + 1 + 15) / 16 * 16 + 16 <= (uint32_t)cap && marks_of(X0, X1, nullptr);
    };
    uint32_t ns = 0;
    for (uint32_t X0 = 0; X0 < h.out_size; ++ns) {
        uint32_t X1 = X0 + 1;
        if (!fits(X0, X1)) IFB_THROW(IFB200_ERR_INVALID_STATE, "ring kernel: one output column reads %u source columns (> %d)", h.right[X0] - h.left[X0] + 1, cap - 16);
        while (X1 < h.out_size && fits(X0, X1 + 1)) ++X1;
        X0 = X1;
    }
    std::vector<HvStripDev>& strips = ht->strips;
    for (;; ++ns) {                                  // balance: equal column counts, if they fit
        strips.clear();
        bool ok = true;
        for (uint32_t s = 0; s < ns && ok; ++s) {
            const uint32_t X0 = (uint32_t)((uint64_t)h.out_size * s / ns), X1 = (uint32_t)((uint64_t)h.out_size * (s + 1) / ns);
            if (X1 <= X0) { ok = false; break; }
            ok = fits(X0, X1);
            HvStripDev sd{};
            sd.X0 = (int)X0; sd.X1 = (int)X1; sd.k0 = (int)k0_of(X0);
            sd.nst = (int)((h.right[X1 - 1] - k0_of(X0) + 1 + 15) / 16);
            sd.Xf = (int)X0; sd.hslot0 = (int)(X0 % (uint32_t)av);     // only the strip's own columns are accumulated: the first to complete is X0
            strips.push_back(sd);
        }
        if (ok) break;
        if (ns > h.out_size) IFB_THROW(IFB200_ERR_INVALID_STATE, "ring kernel: strip partition failed");
    }
    ht->n_strips = (int)ns;
    uint32_t rec = 0;                                        // table rows per strip: what the longest stream needs, not the capacity (a mixed
    for (const auto& sd : strips) rec = std::max<uint32_t>(rec, (uint32_t)sd.nst * 16u + 16u);   // workload uploads thousands of these tables)
    ht->hw_stride = rec;
    const size_t hd_stride = (size_t)rec + 64;
    ht->blob.reserve(ns * (sizeof(HvStripDev) + (size_t)rec * avp * 4 + hd_stride) + ((size_t)p.in_h + 32) * (avp * 4 + 1) + 4096);
    ht->o_strips = ht->blob.add(strips);
    ht->o_hw = ht->blob.add_zeroed((size_t)ns * rec * avp * sizeof(float));
    ht->o_hdone = ht->blob.add_zeroed((size_t)ns * hd_stride);
    ht->o_vw = ht->blob.add_zeroed(((size_t)p.in_h + 32) * avp * sizeof(float));   // 32 rows of zeros behind the last: a row block may end below the bitmap
    ht->o_vdone = ht->blob.add_zeroed((size_t)p.in_h + 32);
    float* const hw = ht->blob.host_at<float>(ht->o_hw);
    uint8_t* const hdone = ht->blob.host_at<uint8_t>(ht->o_hdone);
    float* const vw = ht->blob.host_at<float>(ht->o_vw);
    uint8_t* const vdone = ht->blob.host_at<uint8_t>(ht->o_vdone);
    std::vector<uint32_t> marks;
    for (uint32_t s = 0; s < ns; ++s) {
        const HvStripDev& sd = strips[s];
        const uint32_t k0 = (uint32_t)sd.k0;
        for (uint32_t X = (uint32_t)sd.X0; X < (uint32_t)sd.X1; ++X) {
            const float* w = h.w.data() + h.offset[X];
            const uint32_t slot = X % (uint32_t)av;
            for (uint32_t k = h.left[X]; k <= h.right[X]; ++k) hw[((size_t)s * rec + (k - k0)) * avp + slot] = w[k - h.left[X]];
            uint8_t& d = hdone[(size_t)s * hd_stride + (h.right[X] - k0)];
            if (d == 127) IFB_THROW(IFB200_ERR_INVALID_STATE, "ring kernel: too many columns complete at once");
            ++d;
        }
        marks.clear();
        marks_of((uint32_t)sd.X0, (uint32_t)sd.X1, &marks);
        for (uint32_t c : marks) hdone[(size_t)s * hd_stride + c * 8 + 7] |= 0x80u;
    }
    for (uint32_t y = 0; y < v.out_size; ++y) {
        const float* w = v.w.data() + v.offset[y];
        const uint32_t slot = y % (uint32_t)av;
        for (uint32_t j = v.left[y]; j <= v.right[y]; ++j) vw[(size_t)j * avp + slot] = w[j - v.left[y]];
        uint8_t& d = vdone[v.right[y]];
        if (d == 255) IFB_THROW(IFB200_ERR_INVALID_STATE, "ring kernel: too many rows complete at once");
        ++d;
    }
    return ht;
}

// The host tables of (plan, strip width) exist or can be built.  A geometry whose H windows are wider than the weight table
// (a 3000 -> 1 column down-scale has 1400+ taps) cannot run on the ring kernel: it is remembered as such and the job takes the
// tile kernel or the generic pair instead of failing.
bool hv_host_ready(Plan& p, int max_cols) {
    if (!p.hv_ok) return false;
    if (p.by_cols.count(max_cols)) return true;
    if (std::find(p.cols_failed.begin(), p.cols_failed.end(), max_cols) != p.cols_failed.end()) return false;
    try { p.by_cols.emplace(max_cols, hv_tables_host(p, max_cols)); return true; }
    catch (const Err& e) { p.cols_failed.push_back(max_cols); if (p.hv_reason.empty()) p.hv_reason = e.msg; return false; }
}

// device half: one allocation + one asynchronous copy on the first use; later uses only order their stream after it
HvTables& hv_tables(ifb200_batch* bt, cudaStream_t st, Plan& p, int max_cols) {
    auto it = p.by_cols.find(max_cols);
    if (it == p.by_cols.end()) it = p.by_cols.emplace(max_cols, hv_tables_host(p, max_cols)).first;
    HvTables& ht = *it->second;
    if (!ht.blob.p) ht.blob.commit(bt, st); else ht.blob.use_on(st);
    return ht;
}

// Row bands of one launch (a warp's work item is one band of one strip of one job): output rows split evenly, each band with the
// source rows its windows need.
std::vector<HvBandDev> hv_bands(const Plan& p, int nb) {
    const auto& v = p.wv;
    std::vector<HvBandDev> bands;
    for (int i = 0; i < nb; ++i) {
        const uint32_t Y0 = (uint32_t)((uint64_t)p.out_h * i / nb), Y1 = (uint32_t)((uint64_t)p.out_h * (i + 1) / nb);
        HvBandDev b{};
        if (Y1 > Y0) {
            b.Y0 = (int)Y0; b.Y1 = (int)Y1; b.j0 = (int)v.left[Y0]; b.nrows = (int)(v.right[Y1 - 1] - v.left[Y0] + 1);
            uint32_t Yf = Y0;
            while (Yf > 0 && v.right[Yf - 1] >= v.left[Y0]) --Yf;
            b.Yf = (int)Yf; b.vslot0 = (int)(Yf % (uint32_t)p.av);
        }
        bands.push_back(b);
    }
    return bands;
}
// Bands of a launch.  min_items > 0 (IFB200_OPT_MIN_ITEMS): the smallest count that gives that many work items.  Otherwise:
// enough bands to give every warp of the device one item; and when there is more than one round of items anyway, the count
// whose last round is fullest, counting what the band halos (the V window is re-read at every band edge, and a band's rows are
// walked in blocks of 32) cost.
int hv_pick_bands(const Plan& p, size_t jobs_x_strips, int warps, int min_items) {
    const int max_nb = (int)std::max<uint32_t>(1u, p.out_h / 8u);
    auto need = [&](size_t items) { return (int)std::min<size_t>((size_t)max_nb, std::max<size_t>(1, (items + jobs_x_strips - 1) / jobs_x_strips)); };
    if (min_items > 0) return need((size_t)min_items);
    const int nb0 = need((size_t)warps);
    if (jobs_x_strips * (size_t)nb0 <= (size_t)warps) return nb0;
    int best = nb0; double best_eff = -1.0;
    for (int nb = nb0; nb <= std::min(max_nb, nb0 + 15); ++nb) {
        const double items = (double)jobs_x_strips * nb;
        const double rows = (double)p.in_h / nb + (double)p.wv.max_taps;              // source rows of a band
        const double cost = std::ceil(rows / 32.0) * 32.0 * nb / (double)std::max<uint32_t>(p.in_h, 1u);   // rows walked / rows of the bitmap
        const double eff = items / warps / std::ceil(items / warps) / cost;
        if (eff > best_eff + 1e-9) { best_eff = eff; best = nb; }
    }
    return best;
}
// key of a plan's ring tables: widest strip the kernel variant (ring depth, channels) can hold, clipped by IFB200_OPT_STRIP_COLUMNS,
// | the number of column groups the variant keeps vertical accumulators for << 16
int hv_cols(int av, int ch, int option);

// ------------------------------------------------------------------------------------------------
// ring kernel dispatch table
using HvFn = void (*)(const JobDev*, const HvTmap*, Tables, HvPlanDev, uint32_t, uint32_t*);
// fn[ORI][EPI] reads BGRA frames, rows[SRC - 1][EPI] the rows of ifb200_batch_enqueue_rows (HV_SRC_RGBA, HV_SRC_RGB24),
// rows_ori[SRC - 1][ORI - 1][EPI] those of ifb200_batch_enqueue_rows_oriented; EPI: general, simple + linear, simple + sRGB.  A null
// entry is a form that is not compiled (its jobs take the generic pair).
// prof[PROF - 1][ORI][SRC][EPI - 1]: the forms of ifb200_batch_enqueue_profiled (PF_MATRIX, PF_GRAY), with pthreads / pwarps /
// psmem[PROF - 1] in place of threads / warps / smem.  They exist for the simple store epilogues only: a profiled job with the general
// one takes the generic pair.
struct HvEntry {
    int av, ch; HvFn fn[3][3]; int threads, warps, max_cols, ng; uint32_t (*smem)(uint32_t); HvFn rows[2][3]; HvFn rows_ori[2][2][3];
    HvFn prof[2][3][3][2]; int pthreads, pwarps; uint32_t (*psmem[2])(uint32_t);
};
HvFn hv_form(const HvEntry* e, int ori, int src, int epi, int prof = PF_IDENTITY) {
    if (prof != PF_IDENTITY) return epi == 0 ? nullptr : e->prof[prof - 1][ori][src][epi - 1];
    return src == HV_SRC_BGRA ? e->fn[ori][epi] : ori == HV_ORI_NONE ? e->rows[src - 1][epi] : e->rows_ori[src - 1][ori - 1][epi];
}
template <int AV, int CH, int PROF = PF_IDENTITY> uint32_t hv_smem_bytes(uint32_t sb_low16) { return hv_total_bytes<AV, CH, PROF>(sb_low16); }
#define IFB_HV_EPI(AV_, CH_, O_) {hv_ring_kernel<AV_, CH_, 0, O_>, hv_ring_kernel<AV_, CH_, 1, O_>, hv_ring_kernel<AV_, CH_, 2, O_>}
// The RGB24 form with the general store epilogue at ring depth 6 and three channels spills (one register over the 128 of 16 warps):
// it is not compiled, and its jobs take the generic pair (enqueue_locked)
template <int AV, int CH> constexpr HvFn kRgb24General = hv_ring_kernel<AV, CH, 0, HV_ORI_NONE, HV_SRC_RGB24>;
template <> constexpr HvFn kRgb24General<6, 3> = nullptr;
#define IFB_HV_SRC(AV_, CH_) {{hv_ring_kernel<AV_, CH_, 0, HV_ORI_NONE, HV_SRC_RGBA>, hv_ring_kernel<AV_, CH_, 1, HV_ORI_NONE, HV_SRC_RGBA>, \
                               hv_ring_kernel<AV_, CH_, 2, HV_ORI_NONE, HV_SRC_RGBA>}, \
                              {kRgb24General<AV_, CH_>, hv_ring_kernel<AV_, CH_, 1, HV_ORI_NONE, HV_SRC_RGB24>, hv_ring_kernel<AV_, CH_, 2, HV_ORI_NONE, HV_SRC_RGB24>}}
template <int AV, int CH, int EPI, int ORI, int SRC> constexpr HvFn kRowsOriented = hv_ring_kernel<AV, CH, EPI, ORI, SRC>;
// The RGB24 flip forms at ring depth 6 with three channels spill 4 bytes with the general and the linear store epilogues: not compiled
template <> constexpr HvFn kRowsOriented<6, 3, 0, HV_ORI_FLIP, HV_SRC_RGB24> = nullptr;
template <> constexpr HvFn kRowsOriented<6, 3, 1, HV_ORI_FLIP, HV_SRC_RGB24> = nullptr;
#define IFB_HV_RO(AV_, CH_, O_, S_) {kRowsOriented<AV_, CH_, 0, O_, S_>, kRowsOriented<AV_, CH_, 1, O_, S_>, kRowsOriented<AV_, CH_, 2, O_, S_>}
#define IFB_HV_ROWS_ORI(AV_, CH_) {{IFB_HV_RO(AV_, CH_, HV_ORI_FLIP, HV_SRC_RGBA), IFB_HV_RO(AV_, CH_, HV_ORI_TRANSPOSE, HV_SRC_RGBA)}, \
                                   {IFB_HV_RO(AV_, CH_, HV_ORI_FLIP, HV_SRC_RGB24), IFB_HV_RO(AV_, CH_, HV_ORI_TRANSPOSE, HV_SRC_RGB24)}}
#define IFB_HV_PF_E(AV_, CH_, O_, S_, P_) {hv_ring_profiled_kernel<AV_, CH_, 1, O_, S_, P_>, hv_ring_profiled_kernel<AV_, CH_, 2, O_, S_, P_>}
#define IFB_HV_PF_S(AV_, CH_, O_, P_) {IFB_HV_PF_E(AV_, CH_, O_, HV_SRC_BGRA, P_), IFB_HV_PF_E(AV_, CH_, O_, HV_SRC_RGBA, P_), IFB_HV_PF_E(AV_, CH_, O_, HV_SRC_RGB24, P_)}
#define IFB_HV_PF(AV_, CH_, P_) {IFB_HV_PF_S(AV_, CH_, HV_ORI_NONE, P_), IFB_HV_PF_S(AV_, CH_, HV_ORI_FLIP, P_), IFB_HV_PF_S(AV_, CH_, HV_ORI_TRANSPOSE, P_)}
#define IFB_HV(AV_, CH_) {AV_, CH_, {IFB_HV_EPI(AV_, CH_, HV_ORI_NONE), IFB_HV_EPI(AV_, CH_, HV_ORI_FLIP), IFB_HV_EPI(AV_, CH_, HV_ORI_TRANSPOSE)}, \
                          HvCfg<AV_, CH_>::kThreads, HvCfg<AV_, CH_>::kWarps, HvCfg<AV_, CH_>::kMaxCols, HvCfg<AV_, CH_>::kNG, hv_smem_bytes<AV_, CH_>, \
                          IFB_HV_SRC(AV_, CH_), IFB_HV_ROWS_ORI(AV_, CH_), {IFB_HV_PF(AV_, CH_, PF_MATRIX), IFB_HV_PF(AV_, CH_, PF_GRAY)}, \
                          HvCfg<AV_, CH_, PF_MATRIX>::kThreads, HvCfg<AV_, CH_, PF_MATRIX>::kWarps, \
                          {hv_smem_bytes<AV_, CH_, PF_MATRIX>, hv_smem_bytes<AV_, CH_, PF_GRAY>}}
static_assert(HvCfg<4, 3, PF_MATRIX>::kWarps == HvCfg<4, 3, PF_GRAY>::kWarps && HvCfg<4, 4, PF_MATRIX>::kWarps == HvCfg<4, 4, PF_GRAY>::kWarps, "one warp count per profiled variant");
const HvEntry kHv[] = {IFB_HV(4, 3), IFB_HV(4, 4), IFB_HV(6, 3), IFB_HV(6, 4)};
const HvEntry* find_hv(int av, int ch) {
    for (const auto& e : kHv) if (e.av == av && e.ch == ch) return &e;
    return nullptr;
}
int hv_cols(int av, int ch, int option) { const HvEntry* e = find_hv(av, ch); return std::min(option, e->max_cols) | (e->ng << 16); }

// tile kernel (second form) dispatch: compiled per (channels, working space, compositing mode, colour matrix).
// Without meaningful alpha the compositing mode changes nothing (scaling.rs:227-232, :262), so those share compose 0.
using Tile2Fn = void (*)(const JobDev*, uint32_t, Tables, AxisDev, AxisDev, TilePlanDev);
#define IFB_T2_CM(CH_, LIN_, CO_) {fused_tile2_kernel<CH_, LIN_, CO_, false>, fused_tile2_kernel<CH_, LIN_, CO_, true>}
#define IFB_T2_CO4(LIN_) {IFB_T2_CM(4, LIN_, 0), IFB_T2_CM(4, LIN_, 1), IFB_T2_CM(4, LIN_, 2)}
#define IFB_T2_CO3(LIN_) {IFB_T2_CM(3, LIN_, 0), IFB_T2_CM(3, LIN_, 0), IFB_T2_CM(3, LIN_, 0)}
const Tile2Fn kTile2[2][2][3][2] = {{IFB_T2_CO3(false), IFB_T2_CO3(true)}, {IFB_T2_CO4(false), IFB_T2_CO4(true)}};   // [ch==4][linear][compose][cm]
Tile2Fn find_tile2(int ch, bool linear, int compose, bool cm) { return kTile2[ch == 4][linear][compose][cm]; }

// ------------------------------------------------------------------------------------------------
// SM count the host-only entry points (ifb200_plan_probe, ifb200_hv_plan_tables) plan for, having no device to ask: an H100 SXM's
constexpr int kHostPlanSms = 132;

struct PinnedSlot { void* p = nullptr; size_t cap = 0; cudaEvent_t ev = nullptr; bool used = false; };

// cuTensorMapEncodeTiled, looked up through the runtime (cudaGetDriverEntryPoint): the library does not link libcuda
using TmapEncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
struct TmapKey {
    uintptr_t base; uint32_t w, h, stride; bool transposed;   // transposed: the box of the oriented ring kernel for flags 5..8
    bool bytes;                                                // bytes: RGB24 rows, a UINT8 tensor w bytes wide (RGBA32 shares the u32 map)
    bool operator==(const TmapKey& o) const {
        return base == o.base && w == o.w && h == o.h && stride == o.stride && transposed == o.transposed && bytes == o.bytes;
    }
};
struct TmapKeyHash {
    size_t operator()(const TmapKey& k) const {
        uint64_t x = (uint64_t)k.base * 0x9E3779B97F4A7C15ull;
        x ^= ((uint64_t)k.w << 32 | k.h) * 0xC2B2AE3D27D4EB4Full; x ^= ((uint64_t)k.stride * 4 + k.transposed * 2 + k.bytes) * 0x165667B19E3779F9ull;
        return (size_t)(x ^ (x >> 29));
    }
};

}  // namespace

struct ifb200_batch {
    int device = 0;
    cudaStream_t own_stream = nullptr;
    // An enqueue with many different geometries launches one (small) kernel per geometry: they are spread over a few side
    // streams that fork from and join back into the caller's stream, so that they overlap instead of queueing up.
    static constexpr int kSideStreams = 4;
    cudaStream_t side[kSideStreams] = {};
    cudaEvent_t ev_fork = nullptr, ev_join[kSideStreams] = {};
    std::mutex mu;
    DevVec<float> t_lin, t_srgb; DevVec<uint8_t> lut16k;
    DevVec<uint16_t> idct_to_linear; DevVec<uint8_t> idct_to_srgb;     // block scalers' transfer tables (codecs_jpeg_idct_fast.c:103-300)
    Tables tables{};
    using Key = std::tuple<uint32_t, uint32_t, uint32_t, uint32_t, int, uint32_t>;
    static constexpr size_t kMaxPlans = 4096;
    std::map<Key, std::unique_ptr<Plan>> plans;
    std::vector<PinnedSlot> pinned;
    // options
    bool force_generic = false; int strip_cols = IFB_HV_MAXCOLS4; int min_items = 0;
    int sm_count = 0;                                         // cudaDevAttrMultiProcessorCount, read at creation
    // ring kernel: where dynamic shared memory starts in the shared window (probed once), whether TMA descriptors can be made
    uint32_t smem_base_low16 = 0x400u;
    bool ring_ok = true; std::string ring_reason;
    TmapEncodeFn tmap_encode = nullptr;
    std::unordered_map<TmapKey, HvTmap, TmapKeyHash> tmaps;   // encoded once per (base, width, height, pitch, box shape)
    std::map<std::pair<const void*, size_t>, int> tile_occupancy;   // resident tile-kernel CTAs per SM, by (variant, shared memory)
    std::set<const void*> hv_attr_set;                        // ring-kernel variants whose shared-memory attribute is set
    // counters
    uint64_t launches = 0, fused_jobs = 0, generic_jobs = 0, tile_jobs = 0;
    // where the calling thread spends an enqueue (seconds, inclusive; ifb200_batch_host_profile)
    struct { double enqueue = 0, plans = 0, stage = 0, memcpy_ = 0, upload = 0; uint64_t commits = 0, staged_bytes = 0, pinned_allocs = 0, ring_bands = 0; } prof;

    ~ifb200_batch() {
        cudaSetDevice(device);
        for (auto& s : pinned) { if (s.ev) cudaEventDestroy(s.ev); if (s.p) cudaFreeHost(s.p); }
        for (auto& e : shared_events) cudaEventDestroy(e);
        drop_plans();
        if (own_stream) cudaStreamDestroy(own_stream);
        for (auto& sd : side) if (sd) cudaStreamDestroy(sd);
        if (ev_fork) cudaEventDestroy(ev_fork);
        for (auto& e : ev_join) if (e) cudaEventDestroy(e);
    }

    // Bump allocator for plan tables: thousands of small tables cost one cudaMalloc per 32 MiB, not one each.
    // Freed as a whole together with the plan cache.
    std::vector<uint8_t*> arena_chunks; size_t arena_used = 0, arena_cap = 0;
    std::vector<cudaEvent_t> shared_events;                   // `ready` events of table uploads that were committed together (commit_many)
    void commit_many(cudaStream_t st, const std::vector<DevBlob*>& blobs);
    uint8_t* table_alloc(size_t bytes) {
        bytes = (bytes + 255) / 256 * 256;
        if (arena_chunks.empty() || arena_used + bytes > arena_cap) {
            const size_t cap = std::max<size_t>(bytes, (size_t)32 << 20);
            uint8_t* c = nullptr;
            CUDA_OK(cudaMalloc(&c, cap));
            arena_chunks.push_back(c); arena_used = 0; arena_cap = cap;
        }
        uint8_t* r = arena_chunks.back() + arena_used;
        arena_used += bytes;
        return r;
    }
    void drop_plans() {                                   // callers synchronise the device first
        plans.clear();
        for (uint8_t* c : arena_chunks) cudaFree(c);
        arena_chunks.clear(); arena_used = arena_cap = 0;
    }

    // Pinned staging for asynchronous uploads.  A slot is busy until the event recorded after its copy has completed.  Events are
    // only queried when no free slot is large enough (an enqueue with thousands of cold plans would otherwise query every slot
    // for every plan), and small requests share 1 MiB slots instead of getting a cudaMallocHost each.
    void* stage(size_t bytes, cudaEvent_t* ev_out) {
        Tick tk(prof.stage);
        auto take = [&]() -> PinnedSlot* {
            PinnedSlot* best = nullptr;
            for (auto& s : pinned) if (!s.used && s.cap >= bytes && (!best || s.cap < best->cap)) best = &s;
            return best;
        };
        PinnedSlot* s = take();
        if (!s) {
            for (auto& q : pinned) if (q.used && cudaEventQuery(q.ev) == cudaSuccess) q.used = false;
            s = take();
        }
        if (!s) {
            PinnedSlot n;
            n.cap = std::max<size_t>(bytes, (size_t)1 << 20);
            CUDA_OK(cudaMallocHost(&n.p, n.cap));
            CUDA_OK(cudaEventCreateWithFlags(&n.ev, cudaEventDisableTiming));
            ++prof.pinned_allocs;
            pinned.push_back(n);
            s = &pinned.back();
        }
        s->used = true;
        *ev_out = s->ev;
        return s->p;
    }

    static Key key_of(const ifb200_resample_desc& d) {
        uint32_t sbits; const float sp = d.sharpen_percent > 0.0f ? d.sharpen_percent : 0.0f;
        memcpy(&sbits, &sp, 4);
        return Key{d.in_w, d.in_h, d.w, d.h, d.filter, sbits};
    }
    // Everything of a plan that needs no CUDA call (weights exactly as weights.rs, kernel tables staged for upload);
    // thread-safe, so that an enqueue with many new geometries builds its plans on several host threads.
    static std::unique_ptr<Plan> build_plan_host(const ifb200_resample_desc& d, int strip_cols, int sms) {
        const float sp = d.sharpen_percent > 0.0f ? d.sharpen_percent : 0.0f;
        auto p = std::make_unique<Plan>();
        p->in_w = d.in_w; p->in_h = d.in_h; p->out_w = d.w; p->out_h = d.h;
        const ifb::Lobe lobe = sp > 0.0f ? ifb::Lobe::SharpenPercent : ifb::Lobe::Natural;   // scaling.rs:104-106
        int rc = ifb::compute_axis_weights(d.filter, 1.0, lobe, sp, d.h, d.in_h, p->wv);
        if (rc) IFB_THROW(rc, "vertical weights failed: %s", ifb200_status_name(rc));
        rc = ifb::compute_axis_weights(d.filter, 1.0, lobe, sp, d.w, d.in_w, p->wh);
        if (rc) IFB_THROW(rc, "horizontal weights failed: %s", ifb200_status_name(rc));
        build_hv(*p);
        build_tile(*p);
        if (p->hv_ok)
            for (int ch : {3, 4}) {
                // the strip width enqueue_locked() picks for a call with ONE job of this geometry (narrower strips for small images:
                // see there), so that these tables too are built here, on the builder threads, and not inside the launch loop
                int k = hv_cols(p->av, ch, strip_cols);
                if (!hv_host_ready(*p, k)) continue;
                const size_t max_nb = std::max<uint32_t>(1u, p->out_h / 8u), warps_all = (size_t)sms * 16u;
                for (int c : {32, 16}) {
                    if ((size_t)p->by_cols.at(k)->n_strips * max_nb >= warps_all || c >= strip_cols) break;
                    k = hv_cols(p->av, ch, c);
                    if (!hv_host_ready(*p, k)) break;
                }
            }
        return p;
    }
    Plan& plan_for(const ifb200_resample_desc& d) {
        const Key k = key_of(d);
        auto it = plans.find(k);
        if (it != plans.end()) return *it->second;
        Plan& ref = *(plans[k] = build_plan_host(d, strip_cols, sm_count));
        return ref;
    }
    // build the plans this call needs and the cache lacks, in parallel
    void prebuild_plans(const ifb200_resample_desc* descs, size_t n) {
        std::map<Key, size_t> todo;
        auto collect = [&] {
            todo.clear();
            for (size_t i = 0; i < n; ++i) {
                const Key k = key_of(descs[i]);
                if (!plans.count(k)) todo.emplace(k, i);
            }
        };
        collect();
        if (!plans.empty() && plans.size() + todo.size() > kMaxPlans) {   // bound the cache (mixed workloads: thousands of
            CUDA_OK(cudaDeviceSynchronize());                             // geometries); done before any Plan* of this call is
            drop_plans();                                                 // taken; kernels in flight may still read the old
            collect();                                                    // tables, hence the synchronise
        }
        if (todo.size() < 8) return;                      // a few plans: the serial path in plan_for() is fine
        std::vector<std::pair<Key, size_t>> work(todo.begin(), todo.end());
        std::vector<std::unique_ptr<Plan>> built(work.size());
        std::vector<Err> errs(work.size(), Err{0, ""});
        std::atomic<size_t> next{0};
        const unsigned nthreads = std::max(1u, std::min<unsigned>({std::thread::hardware_concurrency(), 32u, (unsigned)work.size()}));
        const int cta = strip_cols, sms = sm_count;
        auto worker = [&] {
            for (size_t w; (w = next.fetch_add(1)) < work.size();) {
                try { built[w] = build_plan_host(descs[work[w].second], cta, sms); }
                catch (const Err& e) { errs[w] = e; }
                catch (...) { errs[w] = Err{IFB200_ERR_OUT_OF_MEMORY, "plan build failed"}; }
            }
        };
        std::vector<std::thread> pool;
        try { for (unsigned t = 1; t < nthreads; ++t) pool.emplace_back(worker); } catch (...) {}      // fewer threads than wanted: the rest do the work
        worker();
        for (auto& th : pool) th.join();
        for (size_t w = 0; w < work.size(); ++w) {
            if (errs[w].code) throw errs[w];
            plans[work[w].first] = std::move(built[w]);
        }
    }
};

void DevBlob::commit(ifb200_batch* b, cudaStream_t st) {
    const size_t n = host.size();
    if (!n) return;
    Tick tk(b->prof.upload);
    ++b->prof.commits; b->prof.staged_bytes += n;
    if (!ready) CUDA_OK(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
    uint8_t* dst = b->table_alloc(n);
    cudaEvent_t ev;
    void* pin = b->stage(n, &ev);
    { Tick tm(b->prof.memcpy_); memcpy(pin, host.data(), n); }
    CUDA_OK(cudaMemcpyAsync(dst, pin, n, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaEventRecord(ev, st));                     // releases the pinned slot
    CUDA_OK(cudaEventRecord(ready, st));
    p = dst;                                              // only a blob whose upload was enqueued counts as committed
    up_stream = st;
    host.clear(); host.shrink_to_fit();
}

// The tables of many cold plans of one enqueue call: packed into few pinned chunks (<= 32 MiB), ONE asynchronous copy and ONE pair of
// events per chunk instead of one of each per plan (a mixed thumbnail workload brings thousands of new geometries per call, and the
// per-upload cost -- a staging slot, a cudaMemcpyAsync, two event records -- was most of its host time).
void ifb200_batch::commit_many(cudaStream_t st, const std::vector<DevBlob*>& blobs) {
    Tick tk(prof.upload);
    const size_t kChunk = (size_t)32 << 20;
    size_t i = 0;
    while (i < blobs.size()) {
        size_t j = i, bytes = 0;
        while (j < blobs.size() && (j == i || bytes + (blobs[j]->host.size() + 255) / 256 * 256 <= kChunk)) { bytes += (blobs[j]->host.size() + 255) / 256 * 256; ++j; }
        uint8_t* dst = table_alloc(bytes);
        cudaEvent_t slot_ev;
        uint8_t* pin = static_cast<uint8_t*>(stage(bytes, &slot_ev));
        cudaEvent_t ready;
        CUDA_OK(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
        shared_events.push_back(ready);
        size_t off = 0;
        {
            Tick tm(prof.memcpy_);
            for (size_t k = i; k < j; ++k) {
                DevBlob& bl = *blobs[k];
                memcpy(pin + off, bl.host.data(), bl.host.size());
                off += (bl.host.size() + 255) / 256 * 256;
            }
        }
        CUDA_OK(cudaMemcpyAsync(dst, pin, bytes, cudaMemcpyHostToDevice, st));
        CUDA_OK(cudaEventRecord(slot_ev, st));            // releases the pinned slot
        CUDA_OK(cudaEventRecord(ready, st));
        off = 0;
        for (size_t k = i; k < j; ++k) {
            DevBlob& bl = *blobs[k];
            ++prof.commits; prof.staged_bytes += bl.host.size();
            bl.p = dst + off; bl.ready = ready; bl.owns_ready = false; bl.up_stream = st;
            off += (bl.host.size() + 255) / 256 * 256;
            bl.host.clear(); bl.host.shrink_to_fit();
        }
        i = j;
    }
}

namespace {

// CSR windows on the device (tile kernel and generic pair only)
void make_axes_blob(Plan& p) {
    p.axes = std::make_unique<DevBlob>();
    p.dv.add_to(*p.axes, p.wv);
    p.dh.add_to(*p.axes, p.wh);
    if (p.tile_ok) { p.o_tile_vw = p.axes->add(p.tile_vw); p.o_tile_vq = p.axes->add(p.tile_vq); p.o_tile_hw = p.axes->add(p.tile_hw); }
}
void ensure_axes(ifb200_batch* b, cudaStream_t st, Plan& p) {
    if (p.axes) { p.axes->use_on(st); return; }
    make_axes_blob(p);
    p.axes->commit(b, st);
}

void validate(const ifb200_resample_desc& d) {
    int code = 0;
    const std::string why = ifb::resample_check(d, &code);                // ifb_watermark.cc: shared with ifb200_batch_watermark
    if (!why.empty()) IFB_THROW(code, "%s", why.c_str());
}

JobDev make_job(const ifb200_resample_desc& d, const float* t_lin_host, const float* t_srgb_host) {
    JobDev j{};
    j.in = d.in;
    j.out = d.canvas + (size_t)d.y * d.cv_stride + (size_t)d.x * 4;
    j.in_stride = d.in_stride; j.out_stride = d.cv_stride; j.in_xoff = 0;
    j.flags = (d.linear ? JF_LINEAR : 0u) | (d.alpha_meaningful ? JF_ALPHA : 0u) | ((uint32_t)d.compose << JF_COMPOSE_SHIFT);
    if (d.compose == IFB200_BLEND_WITH_MATTE && d.alpha_meaningful) {
        const float* T = d.linear ? t_lin_host : t_srgb_host;
        const float ma = (float)d.matte_bgra[3] * (1.0f / 255.0f);
        j.matte[0] = T[d.matte_bgra[0]] * ma; j.matte[1] = T[d.matte_bgra[1]] * ma; j.matte[2] = T[d.matte_bgra[2]] * ma; j.matte[3] = ma;
    }
    if (d.color_matrix) {
        j.flags |= JF_CM;
        const float* m = d.color_matrix;      // m[row][col]; output channel c = sum_k m[k][c]*in_k + 255*m[4][c]
        for (int c = 0; c < 4; ++c) {
            for (int k = 0; k < 4; ++k) j.cm[c * 5 + k] = m[k * 5 + c];
            j.cm[c * 5 + 4] = m[4 * 5 + c] * 255.0f;
        }
        // r,g,b from r,g,b only, alpha passes through, no bias (sepia, the grayscales, ...): the second tile kernel skips
        // the zero terms, which is exact (see finish_pixel_sm)
        bool rgb3 = j.cm[15] == 0.0f && j.cm[16] == 0.0f && j.cm[17] == 0.0f && j.cm[18] == 1.0f && j.cm[19] == 0.0f;
        for (int c = 0; c < 3; ++c) rgb3 = rgb3 && j.cm[c * 5 + 3] == 0.0f && j.cm[c * 5 + 4] == 0.0f;
        if (rgb3) j.flags |= JF_CM_RGB3;
    }
    return j;
}

float g_t_lin_host[256], g_t_srgb_host[256];
std::once_flag g_tables_once;
void host_tables() {
    std::call_once(g_tables_once, [] { ifb::byte_to_float_table(true, g_t_lin_host); ifb::byte_to_float_table(false, g_t_srgb_host); });
}

// TMA descriptor of one input bitmap for the ring kernel: u32 pixels, box 16 x 32, SWIZZLE_64B, out-of-bounds = 0; `transposed`
// (the oriented kernel of flags 5..8): box 32 x 16, no swizzle.  d is the window as stored.
// The base is aligned down to 16 bytes (a window may start at any pixel: bitmaps.rs:413-431); the kernel adds the 0..3 pixels
// it was moved by to its x coordinates.  `bytes` (RGB24 rows of ifb200_batch_enqueue_rows): u8 elements, the 0..15 bytes between
// the base and d.in plus 3 in_w bytes per row, box 64 x 32, SWIZZLE_64B (both: box 128 bytes x 16 rows, no swizzle); *xoff_out is
// then those 0..15 bytes.
const HvTmap& tmap_for(ifb200_batch* b, const ifb200_resample_desc& d, uint32_t* xoff_out, bool transposed = false, bool bytes = false) {
    const uintptr_t addr = (uintptr_t)d.in;
    const uintptr_t base = addr & ~(uintptr_t)15;
    const uint32_t xoff = bytes ? (uint32_t)(addr - base) : (uint32_t)((addr - base) / 4);
    *xoff_out = xoff;
    const uint32_t w = bytes ? xoff + 3u * d.in_w : d.in_w + xoff;
    const TmapKey key{base, w, d.in_h, d.in_stride, transposed, bytes};
    auto it = b->tmaps.find(key);
    if (it != b->tmaps.end()) return it->second;
    if (b->tmaps.size() > 65536) b->tmaps.clear();
    CUtensorMap tm;
    const cuuint64_t dims[2] = {(cuuint64_t)w, (cuuint64_t)d.in_h};
    const cuuint64_t strides[1] = {(cuuint64_t)d.in_stride};
    const cuuint32_t box[2] = {bytes ? (transposed ? 128u : 64u) : transposed ? 32u : 16u, transposed ? 16u : 32u};
    const cuuint32_t estr[2] = {1u, 1u};
    // L2 promotion: how much of a line a box row pulls into L2 (IFB200_DEBUG_L2_PROMOTION = 0 / 64 / 128 / 256 for experiments).
    // The 64-byte rows of the stored-frame boxes take 128 bytes: the row and the next box's.  With 256 (four boxes' worth) the
    // 4K -> 512 bench line took 19.2 ms, with 128 17.5 ms, with 64 or none 22.7 ms (DESIGN.md section 5.1).  The transposed
    // forms' 128-byte rows keep 256.
    static const int promo_env = [] { const char* e = getenv("IFB200_DEBUG_L2_PROMOTION"); return e ? atoi(e) : -1; }();
    const int promo_bytes = promo_env >= 0 ? promo_env : transposed ? 256 : 128;
    const CUtensorMapL2promotion promo = promo_bytes == 0 ? CU_TENSOR_MAP_L2_PROMOTION_NONE : promo_bytes == 64 ? CU_TENSOR_MAP_L2_PROMOTION_L2_64B
                                       : promo_bytes == 128 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B : CU_TENSOR_MAP_L2_PROMOTION_L2_256B;
    const CUresult r = b->tmap_encode(&tm, bytes ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_UINT32, 2, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                      transposed ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_64B, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) IFB_THROW(IFB200_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) for a %ux%u bitmap, pitch %u", (int)r, d.in_w, d.in_h, d.in_stride);
    HvTmap h;
    static_assert(sizeof(CUtensorMap) == sizeof(h.bytes), "tensor map size");
    memcpy(h.bytes, &tm, sizeof h.bytes);
    return b->tmaps.emplace(key, h).first->second;
}

// frees a stream-ordered allocation on its stream when the scope is left, after the work that uses it has been enqueued or when an
// exception leaves the scope
struct AsyncFree {
    void* p = nullptr; cudaStream_t st = nullptr;
    ~AsyncFree() { if (p) cudaFreeAsync(p, st); }
};

// EXIF flag -> which ring kernel form reads it (HV_ORI_*) and which source axes run backwards (JF_FLIP_X / JF_FLIP_Y): the closed
// form of ifb200_orient_desc (include/ifb200.h)
int ori_class(int flag) { return flag >= 2 && flag <= 4 ? HV_ORI_FLIP : flag >= 5 && flag <= 8 ? HV_ORI_TRANSPOSE : HV_ORI_NONE; }
uint32_t ori_flips(int flag) {
    return ((flag == 2 || flag == 3 || flag == 7 || flag == 8) ? JF_FLIP_X : 0u) | ((flag == 3 || flag == 4 || flag == 6 || flag == 7) ? JF_FLIP_Y : 0u);
}

// ori == nullptr: ifb200_batch_enqueue.  Otherwise (enqueue_oriented_locked) descs[i] is the resample of orient(in, ori[i]) with
// ori[i] in 2..8: in_w x in_h is the ORIENTED size (swapped against the stored window for 5..8), the descriptors have been checked
// as stored, and the plans are those of the oriented geometry.  Oriented jobs take the ring kernel's oriented forms or the generic
// pair with the oriented H pass (there is no oriented tile kernel).
// src != nullptr (enqueue_rows_locked): descs[i].in holds rows of format src[i] (HV_SRC_RGBA / HV_SRC_RGB24), checked by the
// caller; these jobs take the ring kernel's row forms or the generic pair with hpass_rows_kernel (there is no tile-kernel form).
// Both (enqueue_rows_oriented_locked): the ring kernel's oriented row forms or the generic pair with hpass_oriented_kernel<TR, BPP>.
// plan != nullptr (enqueue_profiled_locked): plan[i] is job i's profile plan, null for an identity plan; jobs with a plan take the
// ring kernel's profiled forms (one launch per plan) or the generic pair with hpass_oriented_kernel<TR, BPP, PROF> (flag 1 included).
void enqueue_locked(ifb200_batch* b, const ifb200_resample_desc* descs, size_t n, cudaStream_t st, const int32_t* ori = nullptr,
                    const int32_t* src = nullptr, const ifb200_profile_plan* const* plan = nullptr) {
    if (!descs && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    if (n == 0) return;
    Tick tk_all(b->prof.enqueue);
    host_tables();
    DeviceScope dev_scope_(b->device);
    if (!ori && !src)
        for (size_t i = 0; i < n; ++i) validate(descs[i]);
    { Tick tk(b->prof.plans); b->prebuild_plans(descs, n); }
    // group jobs by (plan, kernel class)
    // kind: 0 generic pair, 1 ring kernel, 3 tile kernel (`variant` = its compile-time case)
    struct Group { Plan* plan; int ch; int kind; bool simple; int variant; int ori; int src; const ifb200_profile_plan* prof; std::vector<size_t> idx; int cols_key = 0;
                   int pk() const { return prof ? prof->kind : PF_IDENTITY; } };
    std::vector<Group> groups;
    for (size_t i = 0; i < n; ++i) {
        Plan* pp; { Tick tk(b->prof.plans); pp = &b->plan_for(descs[i]); }
        Plan& p = *pp;
        const ifb200_resample_desc& d = descs[i];
        // TMA boxes: 16-byte aligned origin (a window that starts at pixel 1..3 of a 16-byte group takes the other kernels) and a
        // pitch that is a multiple of 16 bytes (any Bitmap::create_u8 buffer: 64-byte padded rows)
        bool ring = p.hv_ok && b->ring_ok && !b->force_generic && (d.in_stride % 16 == 0) && ((uintptr_t)d.in % 16 == 0);
        const int ch = d.alpha_meaningful ? 4 : 3;
        const bool upscale = p.out_h >= p.in_h && p.out_w >= p.in_w;
        const int oc = ori ? ori_class(ori[i]) : HV_ORI_NONE;
        if (oc != HV_ORI_NONE && upscale) ring = false;                 // oriented up-scales and 1:1: the generic pair
        // the ring kernel's TMA box origins stay 16-byte aligned: with source x reversed, boxes start at W - 16 - x (flags 2, 3) or
        // W - 32 - y (flags 7, 8), so the stored width W (in_w, or in_h of the oriented plan for 5..8) must be a multiple of four
        if (oc != HV_ORI_NONE && (ori_flips(ori[i]) & JF_FLIP_X) && ((oc == HV_ORI_TRANSPOSE ? p.in_h : p.in_w) & 3u)) ring = false;
        // rows: up-scales and 1:1 take the generic pair; RGB24 rows may start at any byte (the box origins are aligned below the
        // window's first byte), so only the pitch must be a multiple of 16 bytes -- also with source x reversed, for any width
        const int sf = src ? src[i] : HV_SRC_BGRA;
        if (sf != HV_SRC_BGRA) {
            if (sf == HV_SRC_RGB24) ring = p.hv_ok && b->ring_ok && !b->force_generic && (d.in_stride % 16 == 0);
            if (upscale) ring = false;
        }
        const ifb200_profile_plan* const jp = plan ? plan[i] : nullptr;
        const int pk = jp ? jp->kind : PF_IDENTITY;
        if (pk != PF_IDENTITY && upscale) ring = false;                // profiled up-scales and 1:1: the generic pair
        const bool simple = d.compose == IFB200_REPLACE_SELF && !d.color_matrix;   // store epilogue without composite / matrix code
        if (ring && (sf != HV_SRC_BGRA || pk != PF_IDENTITY) && !hv_form(find_hv(p.av, ch), oc, sf, simple ? (d.linear ? 1 : 2) : 0, pk)) ring = false;   // a form not compiled
        if (ring && !(p.tile_ok && upscale) && !hv_host_ready(p, hv_cols(p.av, ch, b->strip_cols))) ring = false;   // windows wider than the weight table
        // the ring kernel streams every source row once and wins whenever rows outnumber outputs (down-scales);
        // for up-scales / 1:1 the tile kernel does less work per source pixel
        const bool prefer_tile = oc == HV_ORI_NONE && sf == HV_SRC_BGRA && pk == PF_IDENTITY && p.tile_ok && !b->force_generic && (!ring || upscale);
        const int kind = prefer_tile ? 3 : (ring ? 1 : 0);
        // the ring kernel keeps ONE transfer table per CTA: jobs of different working spaces go to different launches
        const int variant = kind == 3 ? ((d.linear ? 1 : 0) | ((ch == 4 ? d.compose : 0) << 1) | (d.color_matrix ? 8 : 0)) : kind == 1 ? (d.linear ? 1 : 0) : 0;
        Group* g = nullptr;
        for (auto& gg : groups)
            if (gg.plan == &p && gg.ch == ch && gg.kind == kind && gg.simple == simple && gg.variant == variant && gg.ori == oc && gg.src == sf && gg.prof == jp) { g = &gg; break; }
        if (!g) { groups.push_back(Group{&p, ch, kind, simple, variant, oc, sf, jp, {}}); g = &groups.back(); }
        g->idx.push_back(i);
    }
    // Strip width of every ring group: the widest (least halo) that still gives every warp of the device an item; a launch for one
    // small image is bound by the latency of a warp's walk along its strip, so it gets narrower strips = more, shorter items.
    for (auto& g : groups) {
        if (g.kind != 1) continue;
        Plan& p = *g.plan;
        const HvEntry* he = find_hv(p.av, g.ch);
        const size_t warps_all = (size_t)b->sm_count * (g.prof ? he->pwarps : he->warps);
        const size_t max_nb = std::max<uint32_t>(1u, p.out_h / 8u);
        g.cols_key = hv_cols(p.av, g.ch, b->strip_cols);
        if (b->min_items == 0)
            for (int c : {32, 16}) {
                if (g.idx.size() * (size_t)p.by_cols.at(g.cols_key)->n_strips * max_nb >= warps_all || c >= b->strip_cols) break;
                const int k = hv_cols(p.av, g.ch, c);
                if (!hv_host_ready(p, k)) break;
                g.cols_key = k;
            }
    }
    // tables of the plans this call sees for the first time, in launch order: uploaded in packed slices (commit_many) just ahead
    // of the launches that need them, so that the GPU starts on the first geometries while the host is still preparing the later ones
    std::vector<DevBlob*> cold;
    {
        std::set<DevBlob*> seen;
        for (auto& g : groups) {
            Plan& p = *g.plan;
            DevBlob* bl = nullptr;
            if (g.kind == 1) {
                bl = &p.by_cols.at(g.cols_key)->blob;
            } else {
                if (!p.axes) make_axes_blob(p);
                bl = p.axes.get();
            }
            if (!bl->p && !bl->host.empty() && seen.insert(bl).second) cold.push_back(bl);
        }
    }
    size_t cold_next = 0;
    auto upload_ahead = [&](cudaStream_t up) {                // the next slice of cold tables (<= 128 plans)
        const size_t end = std::min(cold.size(), cold_next + 128);
        if (cold_next < end) { b->commit_many(up, std::vector<DevBlob*>(cold.begin() + cold_next, cold.begin() + end)); cold_next = end; }
    };
    // job array (+ the ring kernel's TMA descriptors, band tables and work counters) -> device (pinned staging, stream ordered)
    struct GroupLayout { size_t jobs = 0, tmaps = 0, bands = 0, counters = 0; int nb = 0, grid = 0; std::vector<HvBandDev> bv; };
    std::vector<GroupLayout> lay(groups.size());
    size_t bytes = 0;
    auto take = [&](size_t nbytes) { const size_t o = (bytes + 127) / 128 * 128; bytes = o + nbytes; return o; };
    for (size_t gi = 0; gi < groups.size(); ++gi) {
        Group& g = groups[gi];
        lay[gi].jobs = take(g.idx.size() * sizeof(JobDev) + (g.prof ? sizeof(ProfDev) : 0));   // a plan follows the job array
        if (g.kind == 1) {
            Plan& p = *g.plan;
            const HvEntry* he = find_hv(p.av, g.ch);
            const HvTables& ht = *p.by_cols.at(g.cols_key);
            const size_t jxs = g.idx.size() * (size_t)ht.n_strips;
            const int warps = g.prof ? he->pwarps : he->warps;
            const int warps_all = b->sm_count * warps;
            const int nb = hv_pick_bands(p, jxs, warps_all, b->min_items);
            lay[gi].bv = hv_bands(p, nb);
            lay[gi].nb = (int)lay[gi].bv.size();
            const size_t items = jxs * nb;
            lay[gi].grid = (int)std::min<size_t>((size_t)b->sm_count, (items + warps - 1) / warps);
            lay[gi].tmaps = take(g.idx.size() * sizeof(HvTmap));
            lay[gi].bands = take(lay[gi].bv.size() * sizeof(HvBandDev));
            lay[gi].counters = take((size_t)ht.n_strips * sizeof(uint32_t));
        }
    }
    cudaEvent_t ev;
    uint8_t* hbuf = static_cast<uint8_t*>(b->stage(bytes, &ev));
    for (size_t gi = 0; gi < groups.size(); ++gi) {
        Group& g = groups[gi];
        JobDev* hj = reinterpret_cast<JobDev*>(hbuf + lay[gi].jobs);
        HvTmap* ht = g.kind == 1 ? reinterpret_cast<HvTmap*>(hbuf + lay[gi].tmaps) : nullptr;
        size_t pos = 0;
        for (size_t i : g.idx) {
            hj[pos] = make_job(descs[i], g_t_lin_host, g_t_srgb_host);
            if (g.ori != HV_ORI_NONE) hj[pos].flags |= ori_flips(ori[i]);
            if (ht) {
                ifb200_resample_desc stored = descs[i];                   // the TMA descriptor describes the window as stored
                if (g.ori == HV_ORI_TRANSPOSE) std::swap(stored.in_w, stored.in_h);
                uint32_t xoff = 0; ht[pos] = tmap_for(b, stored, &xoff, g.ori == HV_ORI_TRANSPOSE, g.src == HV_SRC_RGB24); hj[pos].in_xoff = xoff;
            }
            ++pos;
        }
        if (g.prof) {
            ProfDev* pd = reinterpret_cast<ProfDev*>(hj + pos);
            memcpy(pd->trc, g.prof->trc, sizeof pd->trc); memcpy(pd->m, g.prof->m, sizeof pd->m); memcpy(pd->gray, g.prof->gray, sizeof pd->gray);
        }
        if (g.kind == 1) {
            memcpy(hbuf + lay[gi].bands, lay[gi].bv.data(), lay[gi].bv.size() * sizeof(HvBandDev));
            memset(hbuf + lay[gi].counters, 0, (size_t)g.plan->by_cols.at(g.cols_key)->n_strips * sizeof(uint32_t));
        }
    }
    uint8_t* dbuf = nullptr;
    CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&dbuf), bytes, st));
    AsyncFree dbuf_guard{dbuf, st};
    CUDA_OK(cudaMemcpyAsync(dbuf, hbuf, bytes, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaEventRecord(ev, st));

    // many geometries: one small launch each -> fork onto the side streams (the jobs of one call are independent)
    const bool fork = groups.size() >= 4;
    cudaStream_t const user_stream = st;
    if (fork) {
        CUDA_OK(cudaEventRecord(b->ev_fork, user_stream));
        for (auto& sd : b->side) CUDA_OK(cudaStreamWaitEvent(sd, b->ev_fork, 0));
    }
    struct Join {                                   // the side streams always rejoin the caller's stream, also when a launch throws
        ifb200_batch* b; cudaStream_t user; bool on;
        ~Join() {
            if (!on) return;
            for (int k = 0; k < ifb200_batch::kSideStreams; ++k)
                if (cudaEventRecord(b->ev_join[k], b->side[k]) == cudaSuccess) cudaStreamWaitEvent(user, b->ev_join[k], 0);
        }
    } join{b, user_stream, fork};
    for (size_t gi = 0; gi < groups.size(); ++gi) {
        Group& g = groups[gi];
        Plan& p = *g.plan;
        {
            const DevBlob* need = g.kind == 1 ? &p.by_cols.at(g.cols_key)->blob : p.axes.get();
            while (need && !need->p && cold_next < cold.size()) upload_ahead(user_stream);
        }
        const JobDev* jobs = reinterpret_cast<const JobDev*>(dbuf + lay[gi].jobs);
        const size_t nj = g.idx.size();
        st = fork ? b->side[gi % ifb200_batch::kSideStreams] : user_stream;
        if (g.kind == 3) {
            // persistent CTAs: as many as fit on the device (or one per tile if there are fewer tiles), each walks
            // tiles blockIdx.x, blockIdx.x + gridDim.x, ... of the (job, tile) list
            const TilePlanDev& t = p.tile;
            ensure_axes(b, st, p);
            TilePlanDev tv = t;
            tv.vw = p.axes->at<float>(p.o_tile_vw); tv.vq = p.axes->at<uint32_t>(p.o_tile_vq); tv.hw = p.axes->at<float>(p.o_tile_hw);
            const bool linear = g.variant & 1;
            Tile2Fn fn = find_tile2(g.ch, linear, (g.variant >> 1) & 3, (g.variant & 8) != 0);
            const size_t smem = Tile2Smem::make(t.max_ir, t.max_ic, linear).total;
            int& per_sm = b->tile_occupancy[std::make_pair((const void*)fn, smem)];
            if (per_sm == 0) {
                CUDA_OK(cudaFuncSetAttribute((const void*)fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
                CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)fn, 256, smem));
                per_sm = std::max(per_sm, 1);
            }
            const uint64_t resident = (uint64_t)per_sm * b->sm_count;
            for (size_t off = 0; off < nj; off += 65535) {
                const size_t cnt = std::min<size_t>(65535, nj - off);
                const uint64_t total = (uint64_t)cnt * t.tiles_x * t.tiles_y;
                fn<<<(unsigned)std::min<uint64_t>(total, resident), 256, smem, st>>>(jobs + off, (uint32_t)cnt, b->tables, p.dv.view(*p.axes), p.dh.view(*p.axes), tv);
                CUDA_OK(cudaGetLastError());
                b->launches++;
            }
            b->tile_jobs += nj;
        } else if (g.kind == 1) {
            HvTables& ht = hv_tables(b, st, p, g.cols_key);
            const HvEntry* he = find_hv(p.av, g.ch);
            HvPlanDev pl{};
            pl.in_w = p.in_w; pl.in_h = p.in_h; pl.out_w = p.out_w; pl.out_h = p.out_h;
            pl.n_strips = ht.n_strips; pl.n_bands = lay[gi].nb;
            pl.strips = ht.blob.at<HvStripDev>(ht.o_strips);
            pl.bands = reinterpret_cast<const HvBandDev*>(dbuf + lay[gi].bands);
            pl.hw = ht.blob.at<float>(ht.o_hw); pl.hdone = ht.blob.at<uint8_t>(ht.o_hdone);
            pl.vw = ht.blob.at<float>(ht.o_vw); pl.vdone = ht.blob.at<uint8_t>(ht.o_vdone);
            pl.hw_stride = ht.hw_stride;
            const int epi = g.simple ? ((g.variant & 1) ? 1 : 2) : 0;       // the ring kernel's launches are per working space (variant bit 0 = linear)
            HvFn fn = hv_form(he, g.ori, g.src, epi, g.pk());
            const size_t smem = g.prof ? he->psmem[g.pk() - 1](b->smem_base_low16) : he->smem(b->smem_base_low16);
            if (!b->hv_attr_set.count((const void*)fn)) {
                CUDA_OK(cudaFuncSetAttribute((const void*)fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
                b->hv_attr_set.insert((const void*)fn);
            }
            fn<<<(unsigned)lay[gi].grid, g.prof ? he->pthreads : he->threads, smem, st>>>(jobs, reinterpret_cast<const HvTmap*>(dbuf + lay[gi].tmaps), b->tables, pl, (uint32_t)nj,
                                                                  reinterpret_cast<uint32_t*>(dbuf + lay[gi].counters));
            CUDA_OK(cudaGetLastError());
            b->launches++;
            b->fused_jobs += nj;
            b->prof.ring_bands += (uint64_t)lay[gi].nb;
        } else {
            // generic pair; the float4 intermediate [in_h][out_w] is bounded to ~1 GiB per chunk of jobs
            const size_t per = (size_t)p.in_h * p.out_w * sizeof(float4);
            const size_t chunk = std::max<size_t>(1, std::min<size_t>(std::min<size_t>(nj, 65535), ((size_t)1 << 30) / std::max<size_t>(per, 1)));
            ensure_axes(b, st, p);
            float4* inter = nullptr;
            CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&inter), per * chunk, st));
            AsyncFree inter_guard{inter, st};
            for (size_t off = 0; off < nj; off += chunk) {
                const size_t cnt = std::min(chunk, nj - off);
                if (g.ori == HV_ORI_NONE && g.src != HV_SRC_BGRA && !g.prof) {
                    dim3 gh((p.out_w + 127) / 128, std::min<uint32_t>(p.in_h, 65535u), (unsigned)cnt);
                    if (g.src == HV_SRC_RGB24) hpass_rows_kernel<3><<<gh, 128, 0, st>>>(jobs + off, b->tables, p.dh.view(*p.axes), p.in_h, p.out_w, inter);
                    else hpass_rows_kernel<4><<<gh, 128, 0, st>>>(jobs + off, b->tables, p.dh.view(*p.axes), p.in_h, p.out_w, inter);
                } else if (g.ori == HV_ORI_NONE && !g.prof) {
                    dim3 gh((p.out_w + 127) / 128, std::min<uint32_t>(p.in_h, 65535u), (unsigned)cnt);
                    hpass_generic_kernel<<<gh, 128, 0, st>>>(jobs + off, b->tables, p.dh.view(*p.axes), p.in_h, p.out_w, inter);
                } else {
                    // flips: threads along output columns; transposes: threads along oriented rows = along a source row
                    const bool tr = g.ori == HV_ORI_TRANSPOSE;
                    dim3 gh(((tr ? p.in_h : p.out_w) + 127) / 128, std::min<uint32_t>(tr ? p.out_w : p.in_h, 65535u), (unsigned)cnt);
                    // (profiled jobs: also flag 1, the form without flips; the plan follows the group's job array)
                    using HFn = void (*)(const JobDev*, Tables, AxisDev, uint32_t, uint32_t, uint32_t, float4*, const ProfDev*);
#define IFB_HO(P_) {{hpass_oriented_kernel<false, 0, P_>, hpass_oriented_kernel<false, 4, P_>, hpass_oriented_kernel<false, 3, P_>}, \
                    {hpass_oriented_kernel<true, 0, P_>, hpass_oriented_kernel<true, 4, P_>, hpass_oriented_kernel<true, 3, P_>}}
                    static const HFn kOriented[3][2][3] = {IFB_HO(PF_IDENTITY), IFB_HO(PF_MATRIX), IFB_HO(PF_GRAY)};
#undef IFB_HO
                    const ProfDev* pd = g.prof ? reinterpret_cast<const ProfDev*>(jobs + nj) : nullptr;
                    kOriented[g.pk()][tr][g.src]<<<gh, 128, 0, st>>>(jobs + off, b->tables, p.dh.view(*p.axes), p.in_w, p.in_h, p.out_w, inter, pd);
                }
                CUDA_OK(cudaGetLastError());
                dim3 gv((p.out_w + 127) / 128, std::min<uint32_t>(p.out_h, 65535u), (unsigned)cnt);
                vpass_generic_kernel<<<gv, 128, 0, st>>>(jobs + off, b->tables, p.dv.view(*p.axes), p.in_h, p.out_w, p.out_h, inter);
                CUDA_OK(cudaGetLastError());
                b->launches += 2;
            }
            b->generic_jobs += nj;
        }
    }
    st = user_stream;
}

// The checks of one descriptor of decoder rows (ifb200_batch_enqueue_rows, _rows_oriented), on the rows as stored: its format, the
// resample's own rules (resample_check, with the rows' rules in place of a BGRA row's), then the rows'.  `what` begins every message,
// `bgra_entry` is where a Gray8 / GrayAlpha8 job's BGRA frame goes instead.  Returns the job's HV_SRC_*.
int check_rows(const ifb200_resample_desc& r, int32_t f, size_t i, const char* what, const char* bgra_entry) {
    if (f == IFB200_PIXEL_GRAY_TO_BGRA || f == IFB200_PIXEL_GRAY_ALPHA_TO_BGRA)
        IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "%s job %zu: format %d (%s) has no resample form; convert the rows with "
                  "ifb200_batch_pixel_convert, then resample the BGRA frame with %s", what, i, (int)f,
                  f == IFB200_PIXEL_GRAY_TO_BGRA ? "Gray8" : "GrayAlpha8", bgra_entry);
    if (f != IFB200_PIXEL_RGB24_TO_BGRA && f != IFB200_PIXEL_RGBA_TO_BGRA)
        IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "%s job %zu: format %d is not IFB200_PIXEL_RGB24_TO_BGRA (0) or "
                  "IFB200_PIXEL_RGBA_TO_BGRA (1)", what, i, (int)f);
    ifb200_resample_desc c = r;                                           // every rule but the row's
    c.in_w = r.in_w ? 1u : 0u; c.in_stride = 4u;
    int code = 0;
    const std::string why = ifb::resample_check(c, &code);
    if (!why.empty()) IFB_THROW(code, "%s job %zu: %s", what, i, why.c_str());
    const uint32_t bpp = f == IFB200_PIXEL_RGB24_TO_BGRA ? 3u : 4u;
    if (r.in_stride < (uint64_t)r.in_w * bpp)
        IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "%s job %zu: stride %u smaller than a row of %u %s pixels", what, i, r.in_stride,
                  r.in_w, bpp == 3u ? "RGB24" : "RGBA32");
    if (bpp == 4u && (((uintptr_t)r.in & 3) || (r.in_stride & 3)))
        IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "%s job %zu: RGBA32 rows need a 4-byte aligned pointer and stride", what, i);
    return bpp == 3u ? HV_SRC_RGB24 : HV_SRC_RGBA;
}

// n checked jobs of stored windows (BGRA frames when src is null, else rows of formats src[i]) with EXIF flags orientation[i]
// (null: all identity): every plan -- of the oriented geometry, in_w and in_h swapped for 5..8 -- is built before anything is
// enqueued; then the identity jobs go through enqueue_locked exactly as ifb200_batch_enqueue / _rows send them, and the others
// through its oriented forms.
// plan (enqueue_profiled_locked): the jobs' profile plans, null for an identity plan.
void enqueue_oriented_split(ifb200_batch* b, const ifb200_resample_desc* draws, const int32_t* orientation, const int32_t* src, size_t n,
                            cudaStream_t st, const ifb200_profile_plan* const* plan = nullptr) {
    std::vector<ifb200_resample_desc> plain, turned;
    std::vector<int32_t> flags, plain_src, turned_src;
    std::vector<const ifb200_profile_plan*> plain_plan, turned_plan;
    for (size_t i = 0; i < n; ++i) {
        const int32_t o = orientation ? orientation[i] : 1;
        const int32_t s = src ? src[i] : HV_SRC_BGRA;
        if (ori_class(o) == HV_ORI_NONE) { plain.push_back(draws[i]); plain_src.push_back(s); plain_plan.push_back(plan ? plan[i] : nullptr); continue; }
        ifb200_resample_desc od = draws[i];
        if (ori_class(o) == HV_ORI_TRANSPOSE) std::swap(od.in_w, od.in_h);
        turned.push_back(od);
        turned_src.push_back(s);
        turned_plan.push_back(plan ? plan[i] : nullptr);
        flags.push_back(o);
    }
    {
        Tick tk(b->prof.plans);
        // BGRA identity jobs are checked and planned by enqueue_locked itself, as ifb200_batch_enqueue does it
        if (src) { b->prebuild_plans(plain.data(), plain.size()); for (const auto& r : plain) b->plan_for(r); }   // may throw: nothing enqueued yet
        b->prebuild_plans(turned.data(), turned.size());
        for (const auto& od : turned) b->plan_for(od);
    }
    enqueue_locked(b, plain.data(), plain.size(), st, nullptr, src ? plain_src.data() : nullptr, plan ? plain_plan.data() : nullptr);
    enqueue_locked(b, turned.data(), turned.size(), st, flags.data(), src ? turned_src.data() : nullptr, plan ? turned_plan.data() : nullptr);
}

// ifb200_batch_enqueue_oriented: every descriptor is checked as stored, then enqueue_oriented_split.
void enqueue_oriented_locked(ifb200_batch* b, const ifb200_oriented_resample_desc* d, size_t n, cudaStream_t st) {
    if (!d && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    if (n == 0) return;
    std::vector<ifb200_resample_desc> draws(n);
    std::vector<int32_t> flags(n);
    for (size_t i = 0; i < n; ++i) {
        int code = 0;
        const std::string why = ifb::resample_check(d[i].draw, &code);
        if (!why.empty()) IFB_THROW(code, "oriented resample job %zu: %s", i, why.c_str());
        draws[i] = d[i].draw; flags[i] = d[i].orientation;
    }
    enqueue_oriented_split(b, draws.data(), flags.data(), nullptr, n, st);
}

// ifb200_batch_enqueue_rows: every descriptor is checked (check_rows), then every job goes through enqueue_locked's row forms.
void enqueue_rows_locked(ifb200_batch* b, const ifb200_rows_resample_desc* d, size_t n, cudaStream_t st) {
    if (!d && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    if (n == 0) return;
    std::vector<ifb200_resample_desc> draws(n);
    std::vector<int32_t> src(n);
    for (size_t i = 0; i < n; ++i) {
        src[i] = check_rows(d[i].draw, d[i].format, i, "rows resample", "ifb200_batch_enqueue");
        draws[i] = d[i].draw;
    }
    enqueue_oriented_split(b, draws.data(), nullptr, src.data(), n, st);
}

// ifb200_batch_enqueue_rows_oriented: every descriptor is checked on the stored rows (check_rows), then enqueue_oriented_split.
void enqueue_rows_oriented_locked(ifb200_batch* b, const ifb200_rows_oriented_resample_desc* d, size_t n, cudaStream_t st) {
    if (!d && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    if (n == 0) return;
    std::vector<ifb200_resample_desc> draws(n);
    std::vector<int32_t> src(n), flags(n);
    for (size_t i = 0; i < n; ++i) {
        src[i] = check_rows(d[i].draw, d[i].format, i, "oriented rows resample", "ifb200_batch_enqueue_oriented");
        draws[i] = d[i].draw; flags[i] = d[i].orientation;
    }
    enqueue_oriented_split(b, draws.data(), flags.data(), src.data(), n, st);
}

// ifb200_batch_enqueue_profiled: every descriptor is checked on the source as stored (a BGRA window as ifb200_batch_enqueue_oriented
// checks it, rows with check_rows) and every distinct profile planned once (ifb::ProfilePlans), then enqueue_oriented_split with the
// plans; identity plans run as the matching entry runs them.
void enqueue_profiled_locked(ifb200_batch* b, const ifb200_profiled_resample_desc* d, size_t n, cudaStream_t st) {
    if (!d && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    if (n == 0) return;
    std::vector<ifb200_resample_desc> draws(n);
    std::vector<int32_t> src(n), flags(n);
    std::vector<uint32_t> plan_of(n);
    ifb::ProfilePlans pp;
    for (size_t i = 0; i < n; ++i) {
        if (d[i].format == IFB200_PROFILE_SRC_BGRA) {
            int code = 0;
            const std::string why = ifb::resample_check(d[i].draw, &code);
            if (!why.empty()) IFB_THROW(code, "profiled resample job %zu: %s", i, why.c_str());
            src[i] = HV_SRC_BGRA;
        } else {
            src[i] = check_rows(d[i].draw, d[i].format, i, "profiled resample", "ifb200_batch_enqueue_profiled (IFB200_PROFILE_SRC_BGRA)");
        }
        if (!d[i].profile) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "profiled resample job %zu: null profile pointer", i);
        std::string why;
        const int code = pp.add(*d[i].profile, &plan_of[i], &why);
        if (code != IFB200_OK) IFB_THROW(code, "profiled resample job %zu: %s", i, why.c_str());
        draws[i] = d[i].draw; flags[i] = d[i].orientation;
    }
    std::vector<const ifb200_profile_plan*> plan(n);
    for (size_t i = 0; i < n; ++i) plan[i] = pp.plans[plan_of[i]].kind == IFB200_PLAN_IDENTITY ? nullptr : &pp.plans[plan_of[i]];
    enqueue_oriented_split(b, draws.data(), flags.data(), src.data(), n, st, plan.data());
}

// The argument checks of a BGRA window, shared by the device and the host-buffer form of each operation: a null pointer, or a stride
// below a row or not a multiple of 4, is an argument error.  Returns false for an empty window (nothing to do).
bool bgra_window(const void* px, uint32_t w, uint32_t h, uint32_t stride) {
    if (!px) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null bitmap pointer");
    if (w == 0 || h == 0) return false;
    if (stride < w * 4ull || (stride & 3)) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "stride smaller than a BGRA row or not a multiple of 4");
    return true;
}

// The work lists of one launch: host arrays at 256-byte aligned offsets in ONE stream-ordered device allocation on `st`, filled by ONE
// copy through a pinned staging slot, and `tail` bytes after them that are allocated but not copied.  off[k] is the offset of array k,
// off[number of arrays] that of the tail.  The allocation is freed on `st` when the object goes out of scope, after the launches that
// read it have been enqueued.
struct WorkUpload {
    struct Part { const void* p; size_t bytes; };
    AsyncFree mem;
    std::vector<size_t> off;
    WorkUpload(ifb200_batch* b, cudaStream_t st, std::initializer_list<Part> parts, size_t tail = 0) : mem{nullptr, st} {
        size_t end = 0;
        for (const Part& q : parts) { off.push_back((end + 255) / 256 * 256); end = off.back() + q.bytes; }
        off.push_back((end + 255) / 256 * 256);
        cudaEvent_t ev;
        uint8_t* h = static_cast<uint8_t*>(b->stage(end, &ev));
        const Part* q = parts.begin();
        for (size_t k = 0; k < parts.size(); ++k) if (q[k].bytes) memcpy(h + off[k], q[k].p, q[k].bytes);
        CUDA_OK(cudaMallocAsync(&mem.p, off.back() + tail, st));
        CUDA_OK(cudaMemcpyAsync(mem.p, h, end, cudaMemcpyHostToDevice, st));
        CUDA_OK(cudaEventRecord(ev, st));
    }
    template <class T> T* at(size_t k) const { return reinterpret_cast<T*>(static_cast<uint8_t*>(mem.p) + off[k]); }
};
template <class T> WorkUpload::Part part(const std::vector<T>& v) { return {v.data(), v.size() * sizeof(T)}; }

void color_matrix_locked(ifb200_batch* b, uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride, const float* m, cudaStream_t st) {
    if (!m) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null matrix pointer");
    if (!bgra_window(dev_px, w, h, stride)) return;
    const uint64_t total = (uint64_t)w * h;
    if (total > 0xffffffffull) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "bitmap too large");
    DeviceScope dev_scope_(b->device);
    float hm[20];
    for (int c = 0; c < 4; ++c) {
        for (int k = 0; k < 4; ++k) hm[c * 5 + k] = m[k * 5 + c];
        hm[c * 5 + 4] = m[4 * 5 + c] * 255.0f;                 // color_matrix.rs:9-12
    }
    WorkUpload up(b, st, {{hm, sizeof hm}});
    const unsigned blocks = (unsigned)std::min<uint64_t>((total + 255) / 256, (uint64_t)b->sm_count * 16);
    color_matrix_kernel<<<blocks, 256, 0, st>>>(dev_px, w, h, stride, up.at<const float>(0));
    CUDA_OK(cudaGetLastError());
    b->launches++;
}

void apply_matte_locked(ifb200_batch* b, uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride, const uint8_t* matte, cudaStream_t st) {
    if (!matte) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null matte pointer");
    if (!bgra_window(dev_px, w, h, stride)) return;
    const uint64_t total = (uint64_t)w * h;
    if (total > 0xffffffffull) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "bitmap too large");
    DeviceScope dev_scope_(b->device);
    const uint32_t m = (uint32_t)matte[0] | ((uint32_t)matte[1] << 8) | ((uint32_t)matte[2] << 16) | ((uint32_t)matte[3] << 24);
    const unsigned blocks = (unsigned)std::min<uint64_t>((total + 255) / 256, (uint64_t)b->sm_count * 16);
    apply_matte_kernel<<<blocks, 256, 0, st>>>(dev_px, w, h, stride, m, b->tables);
    CUDA_OK(cudaGetLastError());
    b->launches++;
}

// per-thread context for the host-buffer drop-in calls: a small pipeline of streams, each with its own
// device staging for one input window and one destination rect, so that the upload of call i+1 overlaps the
// kernel of call i and the download of call i-1 when several calls are issued through the batched entry point.
constexpr int kHostSlots = 3;
// transpose.rs:95-121 + the bounds checks of transpose.rs:46-79 (strides in bytes here)
void transpose_locked(ifb200_batch* b, const uint8_t* from, uint32_t from_stride, uint32_t w, uint32_t h, uint8_t* to, uint32_t to_stride,
                      cudaStream_t st) {
    if (!to) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null bitmap pointer");
    if (!bgra_window(from, w, h, from_stride) || !bgra_window(to, h, w, to_stride)) return;      // `to` is h x w: empty when `from` is
    DeviceScope dev_scope_(b->device);
    const uint32_t rows_per_launch = 65535u * 32u;           // grid.y is bounded; bitmaps are not
    for (uint32_t y0 = 0; y0 < h; y0 += rows_per_launch) {
        const uint32_t rows = std::min(rows_per_launch, h - y0);
        dim3 grid((w + 31) / 32, (rows + 31) / 32);
        transpose_bgra8_kernel<<<grid, dim3(32, 8), 0, st>>>(from + (size_t)y0 * from_stride, from_stride, w, rows, to + (size_t)y0 * 4, to_stride);
        CUDA_OK(cudaGetLastError());
        b->launches++;
    }
}
void flip_locked(ifb200_batch* b, bool vertical, uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, cudaStream_t st) {
    if (!bgra_window(px, w, h, stride)) return;
    const bool v4 = (w % 4 == 0) && (stride % 16 == 0) && ((uintptr_t)px % 16 == 0);       // four pixels per access
    const uint32_t we = v4 ? w / 4 : w;
    const uint64_t elems = vertical ? (uint64_t)(h / 2) * we : (uint64_t)(v4 ? (we + 1) / 2 : we / 2) * h;
    if (elems == 0) return;
    DeviceScope dev_scope_(b->device);
    const unsigned blocks = (unsigned)std::min<uint64_t>((elems + 255) / 256, (uint64_t)b->sm_count * 16);
    if (vertical) {
        if (v4) flip_vertical_bgra8_kernel<uint4><<<blocks, 256, 0, st>>>(px, we, h, stride);
        else flip_vertical_bgra8_kernel<uint32_t><<<blocks, 256, 0, st>>>(px, we, h, stride);
    } else {
        if (v4) flip_horizontal_bgra8_v4_kernel<<<blocks, 256, 0, st>>>(px, we, h, stride);
        else flip_horizontal_bgra8_kernel<<<blocks, 256, 0, st>>>(px, w, h, stride);
    }
    CUDA_OK(cudaGetLastError());
    b->launches++;
}

// flow_scale_spatial[_srgb]_NxN over a plane of 8x8 blocks (codecs_jpeg_idct_fast.c; hook: codec_jpeg_wrapper.c:274-340)
void block_scale_locked(ifb200_batch* b, const uint8_t* in, uint32_t in_stride, uint32_t blocks_x, uint32_t blocks_y, uint8_t* out, uint32_t out_stride,
                        int n, int srgb, cudaStream_t st) {
    if (!in || !out) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null plane pointer");
    if (n < 1 || n > 7) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "block scalers exist for 1x1 .. 7x7 (got %d)", n);
    if (blocks_x == 0 || blocks_y == 0) return;
    if (in_stride < blocks_x * 8ull || out_stride < (uint64_t)blocks_x * (uint32_t)n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "stride smaller than a row of blocks");
    DeviceScope dev_scope_(b->device);
    const uint32_t gx = (blocks_x + 31u) / 32u;
    for (uint32_t y0 = 0; y0 < blocks_y; y0 += 65535u) {             // grid.y is bounded; planes are not
        const uint32_t cnt = std::min(65535u, blocks_y - y0);
        idct_block_scale_kernel<<<dim3(gx, cnt), 256, 0, st>>>(in + (size_t)y0 * 8u * in_stride, in_stride, blocks_x, out + (size_t)y0 * (uint32_t)n * out_stride,
                                                              out_stride, n, srgb ? 1 : 0, b->idct_to_linear.p, b->idct_to_srgb.p);
        CUDA_OK(cudaGetLastError());
        b->launches++;
    }
}

// flow/nodes/white_balance.rs:93-121 (WhiteBalanceSrgbMutDef::mutate): histograms, area thresholds, byte maps, remap.
// threshold < 0 stands for None (-> 0.006f32, white_balance.rs:76-77); both thresholds are the same value (:114).
void white_balance_locked(ifb200_batch* b, uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, float threshold, cudaStream_t st) {
    if (!bgra_window(px, w, h, stride)) return;
    if (threshold != threshold) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "threshold is NaN");
    DeviceScope dev_scope_(b->device);
    const double low = (double)(threshold < 0.0f ? 0.006f : threshold);      // f64::from(f32)
    unsigned long long* hist = nullptr;
    CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&hist), 768 * sizeof(unsigned long long) + 768, st));
    uint8_t* maps = reinterpret_cast<uint8_t*>(hist + 768);
    CUDA_OK(cudaMemsetAsync(hist, 0, 768 * sizeof(unsigned long long), st));
    const uint64_t total = (uint64_t)w * h;
    const bool v4 = (w % 4 == 0) && (stride % 16 == 0) && ((uintptr_t)px % 16 == 0);       // four pixels per access
    const uint64_t elems = v4 ? total / 4 : total;
    const unsigned blocks = (unsigned)std::min<uint64_t>((elems + 255) / 256, (uint64_t)b->sm_count * 8);
    if (v4) histogram_bgra8_kernel<true><<<blocks, 256, 0, st>>>(px, w, h, stride, hist);
    else histogram_bgra8_kernel<false><<<blocks, 256, 0, st>>>(px, w, h, stride, hist);
    CUDA_OK(cudaGetLastError());
    white_balance_maps_kernel<<<1, 256, 0, st>>>(hist, (unsigned long long)total, low, maps);
    CUDA_OK(cudaGetLastError());
    if (v4) apply_byte_maps_bgra8_kernel<true><<<blocks, 256, 0, st>>>(px, w, h, stride, maps);
    else apply_byte_maps_bgra8_kernel<false><<<blocks, 256, 0, st>>>(px, w, h, stride, maps);
    CUDA_OK(cudaGetLastError());
    CUDA_OK(cudaFreeAsync(hist, st));
    b->launches += 3;
}

// The limits of the code map's bitmap and threshold (an empty bitmap is an error here)
void whitespace_check(const uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, uint32_t threshold) {
    if (!bgra_window(px, w, h, stride)) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "empty bitmap");
    if (w > 0x7fffffffu || h > 0x7fffffffu) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "oversized bitmap");
    if (threshold > 0x7fffffffu) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "threshold out of range");
}

// The per-pixel code map of detect_content (layout: ifb_whitespace.h) of a DEVICE bitmap into a DEVICE buffer of w*h bytes; asynchronous.
void whitespace_codes_locked(ifb200_batch* b, const uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, int alpha_meaningful,
                             uint32_t threshold, uint8_t* dcodes, cudaStream_t st) {
    if (!dcodes) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null pointer");
    whitespace_check(px, w, h, stride, threshold);
    DeviceScope dev_scope_(b->device);
    // grid.y is bounded: tall bitmaps go in chunks of rows (a chunk's first and last rows look one row up / down: the kernel
    // takes the whole bitmap and the chunk's first row)
    const uint32_t rows_per_launch = 65535u * 8u;
    for (uint32_t y0 = 0; y0 < h; y0 += rows_per_launch) {
        const uint32_t rows = std::min(rows_per_launch, h - y0);
        dim3 grid((w + 31) / 32, (rows + 7) / 8);
        whitespace_codes_kernel<<<grid, dim3(32, 8), 0, st>>>(px, w, h, stride, alpha_meaningful ? 1u : 0u, (int)threshold, dcodes, y0);
        CUDA_OK(cudaGetLastError());
        b->launches++;
    }
}

// detect_content of many DEVICE frames (ifb200_batch_detect_content_many, ifb_whitespace.h): every descriptor is checked before
// anything is launched; then one upload of the plan, ONE launch of whitespace_segments_kernel over every frame of at least 3 x 3 and
// ONE of whitespace_walk_kernel (none when no frame needs a walk), and one copy of the results back.  Synchronises `st`.
void detect_content_many_locked(ifb200_batch* b, const ifb200_detect_content_desc* d, size_t n, uint32_t* rects, uint64_t* visited,
                                cudaStream_t st) {
    if (!d && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    if (!rects && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null rectangle array");
    ifb::WsWork wk;
    int code = 0;
    const std::string why = ifb::detect_content_prepare(d, n, wk, &code, nullptr, nullptr);
    if (!why.empty()) IFB_THROW(code, "%s", why.c_str());
    if (wk.ctas() > 0x7fffffffu || wk.jobs.size() > 0x7fffffffu) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "too many pixels in one call");
    std::vector<ifb::WsResult> res(wk.jobs.size());
    if (!wk.jobs.empty()) {
        DeviceScope dev_scope_(b->device);
        const size_t res_bytes = res.size() * sizeof(ifb::WsResult);
        WorkUpload up(b, st, {part(wk.jobs), part(wk.cols), part(wk.segs), part(wk.first)}, (size_t)wk.n_sums * 4 + 256 + res_bytes);
        uint32_t* sums = up.at<uint32_t>(4);
        ifb::WsResult* dres = reinterpret_cast<ifb::WsResult*>(reinterpret_cast<uint8_t*>(sums) + ((size_t)wk.n_sums * 4 + 255) / 256 * 256);
        if (wk.ctas()) {
            whitespace_segments_kernel<<<(unsigned)wk.ctas(), dim3(ifb::kWsChunk, ifb::kWsBand), 0, st>>>(
                up.at<const ifb::WsSeg>(2), up.at<const uint32_t>(3), (uint32_t)wk.segs.size(), sums);
            CUDA_OK(cudaGetLastError());
            b->launches++;
        }
        whitespace_walk_kernel<<<(unsigned)wk.jobs.size(), 32, 0, st>>>(up.at<const ifb::WsJob>(0), up.at<const ifb::WsColumn>(1), sums, dres);
        CUDA_OK(cudaGetLastError());
        b->launches++;
        cudaEvent_t ev;
        ifb::WsResult* host = static_cast<ifb::WsResult*>(b->stage(res_bytes, &ev));
        CUDA_OK(cudaMemcpyAsync(host, dres, res_bytes, cudaMemcpyDeviceToHost, st));
        CUDA_OK(cudaEventRecord(ev, st));
        CUDA_OK(cudaStreamSynchronize(st));
        memcpy(res.data(), host, res_bytes);
    }
    for (size_t k = 0; k < res.size(); ++k)
        if (res[k].bad) IFB_THROW(IFB200_ERR_INVALID_STATE, "detect_content job %u: the window walk met a window it cannot replay", wk.job_of[k]);
    for (size_t i = 0; i < n; ++i) {
        rects[4 * i] = 0; rects[4 * i + 1] = 0; rects[4 * i + 2] = d[i].w; rects[4 * i + 3] = d[i].h;       // whitespace.rs:288-290
        if (visited) visited[i] = 0;
    }
    for (size_t k = 0; k < res.size(); ++k) {
        const uint32_t i = wk.job_of[k];
        for (int q = 0; q < 4; ++q) rects[4 * i + q] = res[k].rect[q];
        if (visited) visited[i] = res[k].visited;
    }
}

// detect_content (graphics/whitespace.rs:284-331) of one DEVICE bitmap: a one-frame call of detect_content_many_locked, after the
// checks and messages this entry point has always had.  Returns a rectangle, so it synchronises `st`.
void detect_content_locked(ifb200_batch* b, const uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, int alpha_meaningful,
                           uint32_t threshold, cudaStream_t st, uint32_t rect[4]) {
    if (!rect) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null pointer");
    whitespace_check(px, w, h, stride, threshold);
    const ifb200_detect_content_desc d{px, w, h, stride, alpha_meaningful ? 1 : 0, threshold};
    detect_content_many_locked(b, &d, 1, rect, nullptr, st);
}

// ONE launch of round_corners_kernel for every tile of `wk`, asynchronous on `st` (none when no job touches a pixel)
void round_corners_launch(ifb200_batch* b, const ifb::RcWork& wk, cudaStream_t st) {
    if (wk.tiles.empty()) return;
    if (wk.tiles.size() > 0x7fffffffu) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "too many pixels in one call");
    DeviceScope dev_scope_(b->device);
    WorkUpload up(b, st, {part(wk.jobs), part(wk.tiles)});
    round_corners_kernel<<<(unsigned)wk.tiles.size(), ifb::kRcThreads, 0, st>>>(up.at<const ifb::RcJob>(0), up.at<const ifb::RcTile>(1), b->tables);
    CUDA_OK(cudaGetLastError());
    b->launches++;
}

// The rounded corners of ifb200_batch_round_corners (ifb_round_corners.h): every descriptor is checked before anything is planned or
// enqueued, then all jobs run in ONE launch.
void round_corners_locked(ifb200_batch* b, const ifb200_round_corners_desc* d, size_t n, cudaStream_t st) {
    if (!d && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    ifb::RcWork wk;
    int code = 0;
    const std::string why = ifb::round_corners_prepare(d, n, wk, &code);
    if (!why.empty()) IFB_THROW(code, "%s", why.c_str());
    round_corners_launch(b, wk, st);
}

// The canvas operations of ifb200_batch_canvas (ifb_canvas.h): every descriptor is checked before anything is planned or enqueued,
// then all jobs run in ONE launch (none when no job writes a pixel).
void canvas_locked(ifb200_batch* b, const ifb200_canvas_desc* d, size_t n, cudaStream_t st) {
    if (!d && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    ifb::CvWork wk;
    int code = 0;
    const std::string why = ifb::canvas_prepare(d, n, wk, &code);
    if (!why.empty()) IFB_THROW(code, "%s", why.c_str());
    if (wk.tiles.empty()) return;
    if (wk.tiles.size() > 0x7fffffffu) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "too many pixels in one call");
    DeviceScope dev_scope_(b->device);
    WorkUpload up(b, st, {part(wk.items), part(wk.tiles)});
    canvas_kernel<<<(unsigned)wk.tiles.size(), ifb::kCvThreads, 0, st>>>(up.at<const ifb::CvItem>(0), up.at<const ifb::CvTile>(1));
    CUDA_OK(cudaGetLastError());
    b->launches++;
}

// The orientations of ifb200_batch_orient (ifb_orient.h): every descriptor is checked before anything is planned or enqueued, then
// all jobs run in ONE launch (none when no job writes a pixel).  The upload is the items and their first CTAs, O(jobs).
void orient_locked(ifb200_batch* b, const ifb200_orient_desc* d, size_t n, cudaStream_t st) {
    if (!d && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    ifb::OrWork wk;
    int code = 0;
    const std::string why = ifb::orient_prepare(d, n, wk, &code);
    if (!why.empty()) IFB_THROW(code, "%s", why.c_str());
    if (wk.items.empty()) return;
    if (wk.ctas() > 0x7fffffffu) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "too many pixels in one call");
    DeviceScope dev_scope_(b->device);
    WorkUpload up(b, st, {part(wk.items), part(wk.first)});
    orient_kernel<<<(unsigned)wk.ctas(), ifb::kOrThreads, 0, st>>>(up.at<const ifb::OrItem>(0), up.at<const uint32_t>(1), (uint32_t)wk.items.size());
    CUDA_OK(cudaGetLastError());
    b->launches++;
}

// The conversions of ifb200_batch_pixel_convert (ifb_pixel_convert.h): every descriptor is checked before anything is planned or
// enqueued, then all jobs run in ONE launch (none when no job has pixels).  The upload is the items and their first CTAs, O(jobs).
void pixel_convert_locked(ifb200_batch* b, const ifb200_pixel_convert_desc* d, size_t n, cudaStream_t st) {
    if (!d && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    ifb::PcWork wk;
    int code = 0;
    const std::string why = ifb::pixel_convert_prepare(d, n, wk, &code);
    if (!why.empty()) IFB_THROW(code, "%s", why.c_str());
    if (wk.items.empty()) return;
    if (wk.ctas() > 0x7fffffffu) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "too many pixels in one call");
    DeviceScope dev_scope_(b->device);
    WorkUpload up(b, st, {part(wk.items), part(wk.first)});
    pixel_convert_kernel<<<(unsigned)wk.ctas(), ifb::kPcThreads, 0, st>>>(up.at<const ifb::PcItem>(0), up.at<const uint32_t>(1),
                                                                           (uint32_t)wk.items.size());
    CUDA_OK(cudaGetLastError());
    b->launches++;
}

// The JPEG colour stages of ifb200_batch_ycbcr_to_bgra (ifb_ycbcr.h): every descriptor is checked before anything is planned or
// enqueued, then all jobs run in ONE launch (none when no job has pixels).  The upload is the items and their first CTAs, O(jobs).
void ycbcr_locked(ifb200_batch* b, const ifb200_ycbcr_desc* d, size_t n, cudaStream_t st) {
    if (!d && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    ifb::YcWork wk;
    int code = 0;
    const std::string why = ifb::ycbcr_prepare(d, n, wk, &code);
    if (!why.empty()) IFB_THROW(code, "%s", why.c_str());
    if (wk.items.empty()) return;
    if (wk.ctas() > 0x7fffffffu) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "too many pixels in one call");
    DeviceScope dev_scope_(b->device);
    WorkUpload up(b, st, {part(wk.items), part(wk.first)});
    ycbcr_to_bgra_kernel<<<(unsigned)wk.ctas(), ifb::kYcThreads, 0, st>>>(up.at<const ifb::YcItem>(0), up.at<const uint32_t>(1),
                                                                          (uint32_t)wk.items.size());
    CUDA_OK(cudaGetLastError());
    b->launches++;
}

// The JPEG encoder colour stages of ifb200_batch_bgra_to_ycbcr (ifb_ycbcr_enc.h): every descriptor is checked before anything is
// planned or enqueued, then all jobs run in ONE launch (none when no job has pixels).  The upload is the items and their first CTAs,
// O(jobs).
void bgra_to_ycbcr_locked(ifb200_batch* b, const ifb200_bgra_to_ycbcr_desc* d, size_t n, cudaStream_t st) {
    if (!d && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    ifb::YeWork wk;
    int code = 0;
    const std::string why = ifb::bgra_to_ycbcr_prepare(d, n, wk, &code);
    if (!why.empty()) IFB_THROW(code, "%s", why.c_str());
    if (wk.items.empty()) return;
    if (wk.ctas() > 0x7fffffffu) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "too many pixels in one call");
    DeviceScope dev_scope_(b->device);
    WorkUpload up(b, st, {part(wk.items), part(wk.first)});
    bgra_to_ycbcr_kernel<<<(unsigned)wk.ctas(), ifb::kYeThreads, 0, st>>>(up.at<const ifb::YeItem>(0), up.at<const uint32_t>(1),
                                                                          (uint32_t)wk.items.size(), b->tables);
    CUDA_OK(cudaGetLastError());
    b->launches++;
}

// The profile transforms of ifb200_batch_transform_to_srgb (ifb_profile.h): every descriptor is checked and every distinct profile
// planned before anything is enqueued, then all jobs run in ONE launch (none when no job writes a pixel).  The upload is the items,
// their first CTAs and plan indices, and the distinct plans: O(jobs + profiles).
void transform_to_srgb_locked(ifb200_batch* b, const ifb200_to_srgb_desc* d, size_t n, cudaStream_t st) {
    if (!d && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    ifb::PfWork wk;
    int code = 0;
    const std::string why = ifb::transform_to_srgb_prepare(d, n, wk, &code);
    if (!why.empty()) IFB_THROW(code, "%s", why.c_str());
    if (wk.pc.items.empty()) return;
    if (wk.pc.ctas() > 0x7fffffffu) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "too many pixels in one call");
    DeviceScope dev_scope_(b->device);
    WorkUpload up(b, st, {part(wk.pc.items), part(wk.pc.first), part(wk.plan_of), part(wk.plans)});
    transform_to_srgb_kernel<<<(unsigned)wk.pc.ctas(), ifb::kPcThreads, 0, st>>>(up.at<const ifb::PcItem>(0), up.at<const uint32_t>(1),
                                                                                 up.at<const uint32_t>(2), up.at<const ifb200_profile_plan>(3),
                                                                                 b->lut16k.p, (uint32_t)wk.pc.items.size());
    CUDA_OK(cudaGetLastError());
    b->launches++;
}

// The colour chains of ifb200_batch_color_chain (ifb_color.h): every descriptor is checked before anything is planned or enqueued.
// The plan (jobs, prefix sums, segments, tables, matrices) goes up in one copy, O(jobs + steps); then ONE launch, or three when some
// job white-balances (histograms into zeroed counters, byte maps into the jobs' kClWb tables, apply); none when no job writes a pixel.
void color_chain_locked(ifb200_batch* b, const ifb200_color_desc* d, size_t n, cudaStream_t st) {
    if (!d && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    ifb::ClWork wk;
    int code = 0;
    const std::string why = ifb::color_prepare(d, n, wk, &code);
    if (!why.empty()) IFB_THROW(code, "%s", why.c_str());
    if (wk.jobs.empty()) return;
    if (wk.ctas() > 0x7fffffffu || wk.wb_ctas() > 0x7fffffffu) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "too many pixels in one call");
    DeviceScope dev_scope_(b->device);
    const size_t hist_bytes = wk.wb_jobs.size() * 768 * sizeof(unsigned long long);
    WorkUpload up(b, st, {part(wk.jobs), part(wk.first), part(wk.wb_jobs), part(wk.wb_first), part(wk.segs), part(wk.tables), part(wk.mats)},
                  hist_bytes);
    ClDev a{up.at<const ifb::ClJob>(0), up.at<const uint32_t>(1), (uint32_t)wk.jobs.size(), up.at<const ifb::ClSeg>(4), up.at<uint8_t>(5),
            up.at<const float>(6), up.at<unsigned long long>(7)};
    if (!wk.wb_jobs.empty()) {
        ClDev w = a;
        w.jobs = up.at<const ifb::ClJob>(2); w.first = up.at<const uint32_t>(3);
        w.n = (uint32_t)wk.wb_jobs.size();
        CUDA_OK(cudaMemsetAsync(w.hist, 0, hist_bytes, st));
        color_hist_kernel<<<(unsigned)wk.wb_ctas(), ifb::kClThreads, 0, st>>>(w);
        CUDA_OK(cudaGetLastError());
        color_maps_kernel<<<w.n, 256, 0, st>>>(w);
        CUDA_OK(cudaGetLastError());
        b->launches += 2;
    }
    color_apply_kernel<<<(unsigned)wk.ctas(), ifb::kClThreads, 0, st>>>(a);
    CUDA_OK(cudaGetLastError());
    b->launches++;
}

// The watermarks of ifb200_batch_watermark (ifb_watermark.h): every descriptor is checked and every plan built before anything is
// enqueued.  The groups are then cut into chunks of consecutive groups whose F and private copies fit in kWmScratchBytes (one chunk for
// any call whose distinct watermarks need less; a larger group is a chunk alone), and each chunk, on `st`, in turn reuses one pooled
// scratch buffer: its groups with an opacity get a private copy of their window and ONE colour-chain launch over the copies
// (EnableTransparency + the Alpha matrix); each distinct geometry gets the generic H pass and vpass_f_kernel over all its groups; and ONE
// composite launch writes every job of the chunk.  The upload is the groups, the jobs and one JobDev per group, O(jobs + groups).
constexpr size_t kWmScratchBytes = (size_t)1 << 30;

void watermark_locked(ifb200_batch* b, const ifb200_watermark_desc* d, size_t n, cudaStream_t st) {
    if (!d && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
    Tick tk_all(b->prof.enqueue);
    host_tables();
    ifb::WmWork wk;
    int code = 0;
    const std::string why = ifb::watermark_prepare(d, n, g_t_lin_host, g_t_srgb_host, wk, &code);
    if (!why.empty()) IFB_THROW(code, "%s", why.c_str());
    if (wk.groups.empty()) return;
    if (wk.ctas() > 0x7fffffffu) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "too many pixels in one call");
    DeviceScope dev_scope_(b->device);
    const uint32_t ng = (uint32_t)wk.groups.size();
    std::vector<ifb200_resample_desc> reps(ng);
    for (uint32_t g = 0; g < ng; ++g) reps[g] = d[wk.rep[g]].draw;
    { Tick tk(b->prof.plans); b->prebuild_plans(reps.data(), ng); }
    std::vector<Plan*> plan(ng);
    for (uint32_t g = 0; g < ng; ++g) { Tick tk(b->prof.plans); plan[g] = &b->plan_for(reps[g]); }      // may throw: nothing enqueued yet
    auto at = [](size_t x) { return (x + 255) / 256 * 256; };
    auto f_size = [&](uint32_t g) { return (size_t)wk.groups[g].w * wk.groups[g].h * 16u; };
    auto copy_size = [&](uint32_t g) { return wk.opacity[g] < 1.0f ? at((size_t)reps[g].in_w * reps[g].in_h * 4u) : (size_t)0; };
    // chunks; inside a chunk, the groups by geometry in first-seen order, their F consecutive (vpass_f_kernel's blockIdx.z), then the copies
    struct Chunk { uint32_t g0, g1; std::vector<std::pair<Plan*, std::vector<uint32_t>>> geo; };
    std::vector<Chunk> chunks;
    std::vector<size_t> f_off(ng), copy_off(ng, SIZE_MAX);
    size_t scratch_bytes = 0;
    for (uint32_t g = 0; g < ng;) {
        Chunk c{g, g, {}};
        for (size_t bytes = 0; g < ng && (g == c.g0 || bytes + f_size(g) + copy_size(g) <= kWmScratchBytes); ++g) bytes += f_size(g) + copy_size(g);
        c.g1 = g;
        for (uint32_t k = c.g0; k < c.g1; ++k) {
            auto it = std::find_if(c.geo.begin(), c.geo.end(), [&](const auto& e) { return e.first == plan[k]; });
            if (it == c.geo.end()) { c.geo.push_back({plan[k], {}}); it = c.geo.end() - 1; }
            it->second.push_back(k);
        }
        size_t off = 0;
        for (auto& e : c.geo)
            for (uint32_t k : e.second) { f_off[k] = off; off += f_size(k); }
        for (uint32_t k = c.g0; k < c.g1; ++k)
            if (copy_size(k)) { copy_off[k] = off; off += copy_size(k); }
        scratch_bytes = std::max(scratch_bytes, off);
        chunks.push_back(std::move(c));
    }
    uint8_t* scratch = nullptr;
    CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&scratch), scratch_bytes, st));
    AsyncFree scratch_guard{scratch, st};
    // the H pass jobs: one per group, reading the caller's window or its private copy
    std::vector<JobDev> hjobs(ng);
    std::vector<uint32_t> hpos(ng);
    {
        uint32_t k = 0;
        for (auto& c : chunks)
            for (auto& e : c.geo)
                for (uint32_t g : e.second) {
                    ifb200_resample_desc r = reps[g];
                    if (copy_off[g] != SIZE_MAX) { r.in = scratch + copy_off[g]; r.in_stride = r.in_w * 4u; r.alpha_meaningful = 1; }
                    r.compose = IFB200_REPLACE_SELF; r.color_matrix = nullptr;
                    hjobs[k] = make_job(r, g_t_lin_host, g_t_srgb_host);
                    hpos[g] = k++;
                }
    }
    for (uint32_t g = 0; g < ng; ++g) wk.groups[g].f = reinterpret_cast<const float*>(scratch + f_off[g]);
    WorkUpload up(b, st, {part(wk.groups), part(wk.jobs), part(hjobs)});      // the plan goes up in one copy
    std::vector<ifb200_color_step> steps(2 * ng);
    for (const Chunk& c : chunks) {
        // 1. opacity: private copies, then the existing colour chain on them (one launch)
        std::vector<ifb200_color_desc> cds;
        for (uint32_t g = c.g0; g < c.g1; ++g) {
            if (copy_off[g] == SIZE_MAX) continue;
            const ifb200_resample_desc& r = reps[g];
            CUDA_OK(cudaMemcpy2DAsync(scratch + copy_off[g], (size_t)r.in_w * 4u, r.in, r.in_stride, (size_t)r.in_w * 4u, r.in_h, cudaMemcpyDeviceToDevice, st));
            ifb200_color_step* s = &steps[2 * g];
            memset(s, 0, 2 * sizeof(ifb200_color_step));
            s[0].kind = IFB200_COLOR_ENABLE_TRANSPARENCY;
            s[1].kind = IFB200_COLOR_MATRIX;
            ifb::color_filter_matrix(6, wk.opacity[g], s[1].matrix);            // ColorFilterSrgb::Alpha (flow/nodes/color.rs)
            cds.push_back(ifb200_color_desc{scratch + copy_off[g], r.in_w, r.in_h, r.in_w * 4u, r.alpha_meaningful ? 1 : 0, s, 2u});
        }
        if (!cds.empty()) color_chain_locked(b, cds.data(), cds.size(), st);
        // 2. F of every group: the generic H pass + vpass_f_kernel, per geometry, in chunks of at most ~1 GiB of intermediate
        for (auto& e : c.geo) {
            Plan& p = *e.first;
            ensure_axes(b, st, p);
            const uint32_t g0 = e.second.front();
            const size_t nj = e.second.size(), per = (size_t)p.in_h * p.out_w * sizeof(float4);
            const size_t chunk = std::max<size_t>(1, std::min<size_t>(std::min<size_t>(nj, 65535), ((size_t)1 << 30) / std::max<size_t>(per, 1)));
            float4* inter = nullptr;
            CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&inter), per * chunk, st));
            AsyncFree inter_guard{inter, st};
            const JobDev* hj = up.at<const JobDev>(2) + hpos[g0];
            float4* fg = reinterpret_cast<float4*>(scratch + f_off[g0]);
            for (size_t off = 0; off < nj; off += chunk) {
                const size_t cnt = std::min(chunk, nj - off);
                dim3 gh((p.out_w + 127) / 128, std::min<uint32_t>(p.in_h, 65535u), (unsigned)cnt);
                hpass_generic_kernel<<<gh, 128, 0, st>>>(hj + off, b->tables, p.dh.view(*p.axes), p.in_h, p.out_w, inter);
                CUDA_OK(cudaGetLastError());
                dim3 gv((p.out_w + 127) / 128, std::min<uint32_t>(p.out_h, 65535u), (unsigned)cnt);
                vpass_f_kernel<<<gv, 128, 0, st>>>(p.dv.view(*p.axes), p.in_h, p.out_w, p.out_h, inter, fg + off * p.out_h * p.out_w);
                CUDA_OK(cudaGetLastError());
                b->launches += 2;
            }
        }
        // 3. every composite of the chunk in one launch
        const uint32_t cta0 = wk.groups[c.g0].first, cta1 = c.g1 < ng ? wk.groups[c.g1].first : (uint32_t)wk.ctas();
        watermark_composite_kernel<<<cta1 - cta0, ifb::kWmThreads, 0, st>>>(up.at<const ifb::WmGroup>(0) + c.g0, c.g1 - c.g0,
                                                                            up.at<const ifb::WmJob>(1), b->tables, cta0);
        CUDA_OK(cudaGetLastError());
        b->launches++;
    }
}

// Pageable host bitmaps (imageflow's Bitmap buffers are plain Vecs, aligned_buffer.rs:40-43): cudaMemcpy2DAsync from pageable memory
// is staged by the driver on the calling thread (about 10 GB/s, and it does not overlap).  The drop-in path therefore stages such
// bitmaps itself: the rows are copied into a pinned buffer of the pipeline slot by a few host threads in parallel, the pinned buffer
// goes to the GPU with one asynchronous copy; results come back into a pinned buffer and are copied out when the slot is reused.
struct CopyPool {
    struct Task { const uint8_t* src; uint8_t* dst; size_t sp, dp, row_bytes, r0, r1; };
    std::vector<std::thread> th;
    std::mutex m; std::condition_variable cv, cv_done;
    std::vector<Task> q; size_t pending = 0; bool stop = false;
    static void run(const Task& t) {
        if (t.sp == t.row_bytes && t.dp == t.row_bytes) { memcpy(t.dst + t.r0 * t.dp, t.src + t.r0 * t.sp, (t.r1 - t.r0) * t.row_bytes); return; }
        for (size_t r = t.r0; r < t.r1; ++r) memcpy(t.dst + r * t.dp, t.src + r * t.sp, t.row_bytes);
    }
    void start(int n) {
        for (int i = 0; i < n; ++i)
            th.emplace_back([this] {
                for (;;) {
                    Task t;
                    {
                        std::unique_lock<std::mutex> lk(m);
                        cv.wait(lk, [this] { return stop || !q.empty(); });
                        if (stop && q.empty()) return;
                        t = q.back(); q.pop_back();
                    }
                    run(t);
                    { std::lock_guard<std::mutex> lk(m); if (--pending == 0) cv_done.notify_all(); }
                }
            });
    }
    // dst[r][0..row_bytes) = src[r][0..row_bytes) for r < rows, split over the pool's threads and the caller
    void copy2d(uint8_t* dst, size_t dp, const uint8_t* src, size_t sp, size_t row_bytes, size_t rows) {
        const size_t parts = std::min<size_t>(th.size() + 1, std::max<size_t>(1, rows * row_bytes >> 20));   // at least 1 MiB per part
        if (parts <= 1) { run(Task{src, dst, sp, dp, row_bytes, 0, rows}); return; }
        {
            std::lock_guard<std::mutex> lk(m);
            for (size_t k = 1; k < parts; ++k) { q.push_back(Task{src, dst, sp, dp, row_bytes, rows * k / parts, rows * (k + 1) / parts}); ++pending; }
        }
        cv.notify_all();
        run(Task{src, dst, sp, dp, row_bytes, 0, rows / parts});
        std::unique_lock<std::mutex> lk(m);
        cv_done.wait(lk, [this] { return pending == 0; });
    }
    ~CopyPool() {
        { std::lock_guard<std::mutex> lk(m); stop = true; }
        cv.notify_all();
        for (auto& t : th) t.join();
    }
};
struct HostSlot {
    cudaStream_t stream = nullptr;
    uint8_t *d_in = nullptr, *d_cv = nullptr; size_t cap_in = 0, cap_cv = 0;
    uint8_t *h_in = nullptr, *h_cv = nullptr; size_t hcap_in = 0, hcap_cv = 0;     // pinned staging (pageable bitmaps only)
    cudaEvent_t up_done = nullptr;                                                   // the upload from h_in has completed
    // a result waiting in h_cv for its copy to the caller's (pageable) canvas
    uint8_t* out_dst = nullptr; size_t out_stride = 0, out_row_bytes = 0, out_rows = 0, out_pitch = 0;
};
struct HostCtx {
    ifb200_batch* batch = nullptr;
    HostSlot slot[kHostSlots];
    std::unique_ptr<CopyPool> pool;
    ~HostCtx() {
        if (!batch) return;
        cudaSetDevice(batch->device);
        for (auto& s : slot) {
            if (s.stream) { cudaStreamSynchronize(s.stream); cudaStreamDestroy(s.stream); }
            if (s.d_in) cudaFree(s.d_in);
            if (s.d_cv) cudaFree(s.d_cv);
            if (s.h_in) cudaFreeHost(s.h_in);
            if (s.h_cv) cudaFreeHost(s.h_cv);
            if (s.up_done) cudaEventDestroy(s.up_done);
        }
        pool.reset();
        delete batch;
    }
};
thread_local HostCtx t_ctx;

ifb200_batch* create_batch(int device) {
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        IFB_THROW(IFB200_ERR_NO_DEVICE, "no usable CUDA device (%s); libifb200 has no CPU fallback", cudaGetErrorString(e));
    if (device < 0 || device >= ndev) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "device %d out of range (0..%d)", device, ndev - 1);
    DeviceScope dev_scope_(device);
    std::unique_ptr<ifb200_batch> b(new ifb200_batch());
    b->device = device;
    CUDA_OK(cudaStreamCreateWithFlags(&b->own_stream, cudaStreamNonBlocking));
    for (auto& sd : b->side) CUDA_OK(cudaStreamCreateWithFlags(&sd, cudaStreamNonBlocking));
    CUDA_OK(cudaEventCreateWithFlags(&b->ev_fork, cudaEventDisableTiming));
    for (auto& e : b->ev_join) CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    {   // job arrays and the generic path's intermediates come from the stream-ordered pool: keep its memory across
        // synchronisation points (the default threshold of 0 returns it to the OS at every synchronise, and the next
        // call pays tens of milliseconds to get it back)
        cudaMemPool_t pool;
        CUDA_OK(cudaDeviceGetDefaultMemPool(&pool, device));
        uint64_t keep = UINT64_MAX;
        CUDA_OK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
    }
    std::vector<float> tl(256), ts(256); std::vector<uint8_t> lut(16384);
    ifb::byte_to_float_table(true, tl.data()); ifb::byte_to_float_table(false, ts.data()); ifb::linear_to_srgb_table(lut.data());
    b->t_lin.upload(tl); b->t_srgb.upload(ts); b->lut16k.upload(lut);
    b->tables = Tables{b->t_lin.p, b->t_srgb.p, b->lut16k.p};
    b->idct_to_linear.upload(std::vector<uint16_t>(kIdct_lut_srgb_to_linear, kIdct_lut_srgb_to_linear + 256));
    b->idct_to_srgb.upload(std::vector<uint8_t>(kIdct_lut_linear_to_srgb, kIdct_lut_linear_to_srgb + 4096));
    CUDA_OK(cudaMemcpyToSymbol(c_idct, kIdctScalers, sizeof kIdctScalers));
    CUDA_OK(cudaDeviceGetAttribute(&b->sm_count, cudaDevAttrMultiProcessorCount, device));
    {   // the ring kernel lays its shared memory out around a 64 KB-aligned (in the shared window) lookup table: learn where
        // dynamic shared memory starts in the window, and check that every variant then fits
        DevVec<uint32_t> probe; probe.upload(std::vector<uint32_t>(1, 0xffffffffu));
        CUDA_OK(cudaFuncSetAttribute((const void*)smem_base_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
        smem_base_probe_kernel<<<1, 32, 100 * 1024, b->own_stream>>>(probe.p);
        CUDA_OK(cudaGetLastError());
        uint32_t got = 0;
        CUDA_OK(cudaMemcpyAsync(&got, probe.p, 4, cudaMemcpyDeviceToHost, b->own_stream));
        CUDA_OK(cudaStreamSynchronize(b->own_stream));
        b->smem_base_low16 = got & 0xffffu;
        int optin = 0;
        CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
        for (const auto& e : kHv)
            if (e.smem(b->smem_base_low16) > (uint32_t)optin) {
                b->ring_ok = false;
                b->ring_reason = "ring kernel needs " + std::to_string(e.smem(b->smem_base_low16)) + " bytes of shared memory per CTA, the device offers " + std::to_string(optin);
            }
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres = cudaDriverEntryPointSymbolNotFound;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
            cudaGetLastError();
            b->ring_ok = false; b->ring_reason = "cuTensorMapEncodeTiled is not available from this driver";
        }
        b->tmap_encode = reinterpret_cast<TmapEncodeFn>(fn);
    }
    return b.release();
}

std::atomic<int> g_dropin_device{-1};             // ifb200_set_dropin_device(); -1: IFB200_DEVICE, else device 0

HostCtx& host_ctx() {
    if (!t_ctx.batch) {
        int dev = g_dropin_device.load();
        if (dev < 0) { dev = 0; if (const char* s = getenv("IFB200_DEVICE")) dev = atoi(s); }
        t_ctx.batch = create_batch(dev);
        for (auto& sl : t_ctx.slot) CUDA_OK(cudaStreamCreateWithFlags(&sl.stream, cudaStreamNonBlocking));
    }
    return t_ctx;
}

// Staging buffers of the drop-in path grow geometrically (a stream of mixed sizes reallocates O(log) times, not at every new maximum)
size_t grown(size_t cap, size_t need) { return std::max(need, cap + cap / 2); }
void ensure(uint8_t*& p, size_t& cap, size_t need, cudaStream_t st) {
    if (cap >= need) return;
    const size_t want = grown(cap, need);
    CUDA_OK(cudaStreamSynchronize(st));           // nothing may still be using the old buffer
    if (p) CUDA_OK(cudaFree(p));
    p = nullptr; cap = 0;
    if (cudaMalloc(&p, want) != cudaSuccess) { cudaGetLastError(); p = nullptr; CUDA_OK(cudaMalloc(&p, need)); cap = need; return; }
    cap = want;
}

// The body of every ifb200_batch_* operation: failures become a status, a null batch is rejected, and fn runs with the batch locked on
// the caller's stream (IFB200_STREAM_OWN: the batch's own).
template <class F>
int with_batch(ifb200_batch* b, void* stream, char* err, size_t cap, F&& fn) {
    return guarded(err, cap, [&] {
        if (!b) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null batch");
        std::lock_guard<std::mutex> lk(b->mu);
        fn(stream == IFB200_STREAM_OWN ? b->own_stream : static_cast<cudaStream_t>(stream));
    });
}

// The drop-in calls on host buffers, after their argument checks: fn(batch, slot, stream) runs on slot 0 of the calling thread's
// context, with its batch locked and its device current.
template <class F>
void on_host_slot(F&& fn) {
    HostCtx& c = host_ctx();
    std::lock_guard<std::mutex> lk(c.batch->mu);
    DeviceScope dev_scope_(c.batch->device);
    fn(c.batch, c.slot[0], c.slot[0].stream);
}

// A drop-in call that changes a host BGRA window in place: after the window's checks, the window goes to the slot's device image at
// a 64-byte pitch, op(batch, device image, pitch, stream) runs on it, and the window comes back before the call returns.
template <class F>
void in_place_on_host(uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, F&& op) {
    if (!bgra_window(px, w, h, stride)) return;
    on_host_slot([&](ifb200_batch* b, HostSlot& sl, cudaStream_t st) {
        const size_t pitch = ((size_t)w * 4 + 63) / 64 * 64;
        ensure(sl.d_cv, sl.cap_cv, pitch * h, st);
        CUDA_OK(cudaMemcpy2DAsync(sl.d_cv, pitch, px, stride, (size_t)w * 4, h, cudaMemcpyHostToDevice, st));
        op(b, sl.d_cv, (uint32_t)pitch, st);
        CUDA_OK(cudaMemcpy2DAsync(px, stride, sl.d_cv, pitch, (size_t)w * 4, h, cudaMemcpyDeviceToHost, st));
        CUDA_OK(cudaStreamSynchronize(st));
    });
}

}  // namespace

// ================================================================================================
extern "C" {

uint32_t ifb200_abi_version(void) { return (IFB200_ABI_VERSION_MAJOR << 16) | IFB200_ABI_VERSION_MINOR; }

int ifb200_set_dropin_device(int device) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return IFB200_ERR_CUDA; }
    if (device < 0 || device >= n) return IFB200_ERR_INVALID_ARGUMENT;
    g_dropin_device.store(device);
    return IFB200_OK;
}

const char* ifb200_status_name(int s) {
    switch (s) {
    case IFB200_OK: return "Ok";
    case IFB200_ERR_INVALID_ARGUMENT: return "InvalidArgument";
    case IFB200_ERR_NOT_IMPLEMENTED: return "MethodNotImplemented";
    case IFB200_ERR_INVALID_STATE: return "InvalidState";
    case IFB200_ERR_TOTAL_WEIGHT_ZERO: return "TotalWeightZero";
    case IFB200_ERR_SOURCE_COUNT_TOO_LARGE: return "SourcePixelCountTooLarge";
    case IFB200_ERR_NO_PIXEL_INPUTS: return "NoPixelInputs";
    case IFB200_ERR_BAD_FILTER: return "BadFilter";
    case IFB200_ERR_CAPACITY: return "Capacity";
    case IFB200_ERR_NO_DEVICE: return "NoDevice";
    case IFB200_ERR_CUDA: return "CudaError";
    case IFB200_ERR_OUT_OF_MEMORY: return "OutOfMemory";
    default: return "Unknown";
    }
}

int ifb200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int ifb200_weights(int filter, double kws, int lobe_mode, float lobe_value, uint32_t out_size, uint32_t in_size,
                   uint32_t* left, uint32_t* right, uint32_t* offsets, float* weights, size_t cap) {
    try {
        if (!left || !right || !offsets || !weights) return IFB200_ERR_INVALID_ARGUMENT;
        if (lobe_mode < 0 || lobe_mode > 2) return IFB200_ERR_INVALID_ARGUMENT;
        ifb::AxisWeights a;
        int rc = ifb::compute_axis_weights(filter, kws, static_cast<ifb::Lobe>(lobe_mode), lobe_value, out_size, in_size, a);
        if (rc) return rc;
        if (a.w.size() > cap) return IFB200_ERR_CAPACITY;
        memcpy(left, a.left.data(), sizeof(uint32_t) * out_size);
        memcpy(right, a.right.data(), sizeof(uint32_t) * out_size);
        memcpy(offsets, a.offset.data(), sizeof(uint32_t) * ((size_t)out_size + 1));
        memcpy(weights, a.w.data(), sizeof(float) * a.w.size());
        return IFB200_OK;
    } catch (...) { return IFB200_ERR_OUT_OF_MEMORY; }
}

void ifb200_byte_to_float_table(int linear, float out[256]) { ifb::byte_to_float_table(linear != 0, out); }
void ifb200_linear_to_srgb_table(uint8_t out[16384]) { ifb::linear_to_srgb_table(out); }
// Host-side cost of preparing the kernel tables of n geometries: builds the plans (weights as weights.rs, ring / tile
// tables) on `threads` host threads and discards them.  No CUDA call, no cache: what a mixed workload pays per new geometry.
int ifb200_plan_probe(const ifb200_resample_desc* descs, size_t n, int threads, double* seconds, uint64_t* table_bytes, uint64_t* table_hash,
                      char* err, size_t err_cap) {
    return guarded(err, err_cap, [&] {
        if (!descs && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
        for (size_t i = 0; i < n; ++i) {
            const auto& d = descs[i];
            if (d.w == 0 || d.h == 0 || d.in_w == 0 || d.in_h == 0) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "empty bitmap");
            if (d.filter < 1 || d.filter > 31) IFB_THROW(IFB200_ERR_BAD_FILTER, "unknown filter id %d", d.filter);
        }
        std::atomic<size_t> next{0};
        std::atomic<uint64_t> bytes{0};
        std::vector<uint64_t> hashes(table_hash ? n : 0, 0);         // FNV-1a of each plan's staged tables and CSR windows
        auto fnv = [](uint64_t h, const void* p, size_t nb) {
            const uint8_t* b = static_cast<const uint8_t*>(p);
            for (size_t i = 0; i < nb; ++i) { h ^= b[i]; h *= 1099511628211ull; }
            return h;
        };
        std::vector<Err> errs((size_t)std::max(threads, 1), Err{0, ""});
        auto worker = [&](int me) {
            try {
                for (size_t i; (i = next.fetch_add(1)) < n;) {
                    auto p = ifb200_batch::build_plan_host(descs[i], 64, kHostPlanSms);
                    uint64_t b = 0;
                    for (auto& kv : p->by_cols) b += kv.second->blob.host.size();
                    bytes += b;
                    if (table_hash) {
                        uint64_t h = 14695981039346656037ull;
                        for (auto& kv : p->by_cols) h = fnv(h, kv.second->blob.host.data(), kv.second->blob.host.size());
                        for (const ifb::AxisWeights* a : {&p->wv, &p->wh}) {
                            h = fnv(h, a->left.data(), a->left.size() * 4); h = fnv(h, a->right.data(), a->right.size() * 4);
                            h = fnv(h, a->offset.data(), a->offset.size() * 4); h = fnv(h, a->w.data(), a->w.size() * 4);
                        }
                        hashes[i] = h;
                    }
                }
            } catch (const Err& e) { errs[me] = e; }
        };
        const auto t0 = std::chrono::steady_clock::now();
        std::vector<std::thread> pool;
        try { for (int t = 1; t < threads; ++t) pool.emplace_back(worker, t); } catch (...) {}           // fewer threads than wanted: the rest do the work
        worker(0);
        for (auto& th : pool) th.join();
        const double dt = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        for (auto& e : errs) if (e.code) throw e;
        if (seconds) *seconds = dt;
        if (table_bytes) *table_bytes = bytes.load();
        if (table_hash) { uint64_t h = 14695981039346656037ull; *table_hash = fnv(h, hashes.data(), hashes.size() * 8); }
    });
}

// The ring kernel's host tables for one geometry (tests: tests/cpu_emu runs the kernel's source over them on the CPU; no CUDA call).
int ifb200_hv_plan_tables(const ifb200_resample_desc* d, int strip_cols, int n_pairs, ifb200_hv_plan_info* info, uint8_t* buf, size_t cap,
                          char* err, size_t err_cap) {
    return guarded(err, err_cap, [&] {
        if (!d || !info) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null pointer");
        if (strip_cols < 16 || strip_cols > 128 || strip_cols % 16 || n_pairs < 1) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "bad strip width or band count");
        memset(info, 0, sizeof *info);
        auto p = ifb200_batch::build_plan_host(*d, strip_cols, kHostPlanSms);
        if (!p->hv_ok) return;                                            // info->ok stays 0: not a ring-kernel geometry
        const int cols = hv_cols(p->av, d->alpha_meaningful ? 4 : 3, strip_cols);
        if (!p->by_cols.count(cols)) return;
        HvTables& ht = *p->by_cols.at(cols);
        const std::vector<HvBandDev> bands = hv_bands(*p, n_pairs);
        const size_t o_bands = (ht.blob.host.size() + 255) / 256 * 256;
        info->ok = 1; info->av = p->av; info->n_strips = ht.n_strips; info->n_bands = (int32_t)bands.size();
        info->avp = p->av == 4 ? 4 : 8; info->cap_px = (int32_t)ht.hw_stride;       // weight records per strip in hw (hdone: + 64 bytes)
        info->o_strips = ht.o_strips; info->o_hw = ht.o_hw; info->o_hdone = ht.o_hdone; info->o_vw = ht.o_vw; info->o_vdone = ht.o_vdone;
        info->o_bands = o_bands; info->total = o_bands + bands.size() * sizeof(HvBandDev);
        if (!buf) return;
        if (cap < info->total) IFB_THROW(IFB200_ERR_CAPACITY, "buffer of %zu bytes, %llu needed", cap, (unsigned long long)info->total);
        memcpy(buf, ht.blob.host.data(), ht.blob.host.size());
        memcpy(buf + o_bands, bands.data(), bands.size() * sizeof(HvBandDev));
    });
}

int  ifb200_color_filter_matrix(int which, float p, float out[25]) { return out ? ifb::color_filter_matrix(which, p, out) : IFB200_ERR_INVALID_ARGUMENT; }

int ifb200_batch_create(int device, ifb200_batch** out, char* err, size_t cap) {
    return guarded(err, cap, [&] {
        if (!out) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null out pointer");
        *out = nullptr;
        *out = create_batch(device);
    });
}

int ifb200_batch_enqueue(ifb200_batch* b, const ifb200_resample_desc* descs, size_t n, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { enqueue_locked(b, descs, n, st); });
}

int ifb200_batch_enqueue_oriented(ifb200_batch* b, const ifb200_oriented_resample_desc* d, size_t n, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { enqueue_oriented_locked(b, d, n, st); });
}

int ifb200_batch_enqueue_rows(ifb200_batch* b, const ifb200_rows_resample_desc* d, size_t n, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { enqueue_rows_locked(b, d, n, st); });
}

int ifb200_batch_enqueue_rows_oriented(ifb200_batch* b, const ifb200_rows_oriented_resample_desc* d, size_t n, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { enqueue_rows_oriented_locked(b, d, n, st); });
}

int ifb200_batch_enqueue_profiled(ifb200_batch* b, const ifb200_profiled_resample_desc* d, size_t n, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { enqueue_profiled_locked(b, d, n, st); });
}
int ifb200_batch_color_matrix(ifb200_batch* b, uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride, const float m[25],
                              void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { color_matrix_locked(b, dev_px, w, h, stride, m, st); });
}

int ifb200_batch_apply_matte(ifb200_batch* b, uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride, const uint8_t matte_bgra[4],
                             int alpha_meaningful, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) {
        if (alpha_meaningful) apply_matte_locked(b, dev_px, w, h, stride, matte_bgra, st);   // blend.rs:10-13: nothing to do unless alpha is meaningful
    });
}

int ifb200_batch_transpose(ifb200_batch* b, const uint8_t* dev_from, uint32_t from_stride, uint32_t w, uint32_t h, uint8_t* dev_to,
                           uint32_t to_stride, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { transpose_locked(b, dev_from, from_stride, w, h, dev_to, to_stride, st); });
}
int ifb200_batch_flip_vertical(ifb200_batch* b, uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { flip_locked(b, true, dev_px, w, h, stride, st); });
}
int ifb200_batch_flip_horizontal(ifb200_batch* b, uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { flip_locked(b, false, dev_px, w, h, stride, st); });
}

int ifb200_batch_white_balance(ifb200_batch* b, uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride, float threshold, void* stream,
                               char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { white_balance_locked(b, dev_px, w, h, stride, threshold, st); });
}

int ifb200_batch_block_scale(ifb200_batch* b, const uint8_t* dev_in, uint32_t in_stride, uint32_t blocks_x, uint32_t blocks_y, uint8_t* dev_out,
                             uint32_t out_stride, int n, int srgb, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { block_scale_locked(b, dev_in, in_stride, blocks_x, blocks_y, dev_out, out_stride, n, srgb, st); });
}

int ifb200_batch_round_corners(ifb200_batch* b, const ifb200_round_corners_desc* d, size_t n, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { round_corners_locked(b, d, n, st); });
}

int ifb200_batch_canvas(ifb200_batch* b, const ifb200_canvas_desc* d, size_t n, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { canvas_locked(b, d, n, st); });
}

int ifb200_batch_orient(ifb200_batch* b, const ifb200_orient_desc* d, size_t n, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { orient_locked(b, d, n, st); });
}

int ifb200_batch_pixel_convert(ifb200_batch* b, const ifb200_pixel_convert_desc* d, size_t n, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { pixel_convert_locked(b, d, n, st); });
}

int ifb200_batch_ycbcr_to_bgra(ifb200_batch* b, const ifb200_ycbcr_desc* d, size_t n, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { ycbcr_locked(b, d, n, st); });
}

int ifb200_batch_bgra_to_ycbcr(ifb200_batch* b, const ifb200_bgra_to_ycbcr_desc* d, size_t n, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { bgra_to_ycbcr_locked(b, d, n, st); });
}

int ifb200_batch_transform_to_srgb(ifb200_batch* b, const ifb200_to_srgb_desc* d, size_t n, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { transform_to_srgb_locked(b, d, n, st); });
}

int ifb200_source_profile_plan(const ifb200_source_profile* p, ifb200_profile_plan* plan, char* why, size_t cap) {
    return guarded(why, cap, [&] {
        if (!p) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null profile pointer");
        ifb200_profile_plan local;
        std::string reason;
        const int code = ifb::profile_plan(*p, plan ? plan : &local, &reason);
        if (code) IFB_THROW(code, "%s", reason.c_str());
    });
}

int ifb200_batch_color_chain(ifb200_batch* b, const ifb200_color_desc* d, size_t n, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { color_chain_locked(b, d, n, st); });
}

int ifb200_batch_watermark(ifb200_batch* b, const ifb200_watermark_desc* d, size_t n, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { watermark_locked(b, d, n, st); });
}

int ifb200_batch_sync(ifb200_batch* b, char* err, size_t cap) {
    return guarded(err, cap, [&] {
        if (!b) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null batch");
        DeviceScope dev_scope_(b->device);
        CUDA_OK(cudaStreamSynchronize(b->own_stream));
    });
}

void ifb200_batch_destroy(ifb200_batch* b) {
    if (!b) return;
    try { DeviceScope dev_scope_(b->device); cudaDeviceSynchronize(); delete b; } catch (...) {}
}

int ifb200_batch_set_option(ifb200_batch* b, int option, int64_t value) {
    if (!b) return IFB200_ERR_INVALID_ARGUMENT;
    std::lock_guard<std::mutex> lk(b->mu);
    switch (option) {
    case IFB200_OPT_FORCE_GENERIC: b->force_generic = value != 0; return IFB200_OK;
    case IFB200_OPT_STRIP_COLUMNS:
        if (value < 16 || value > 128 || value % 16) return IFB200_ERR_INVALID_ARGUMENT;
        b->strip_cols = (int)value; return IFB200_OK;
    case IFB200_OPT_MIN_ITEMS:
        if (value < 0 || value > (1 << 24)) return IFB200_ERR_INVALID_ARGUMENT;
        b->min_items = (int)value; return IFB200_OK;
    default: return IFB200_ERR_INVALID_ARGUMENT;
    }
}
int ifb200_batch_host_profile(const ifb200_batch* b, double* out, int n) {
    if (!b) return 0;
    const double v[9] = {b->prof.enqueue, b->prof.plans, b->prof.stage, b->prof.memcpy_, b->prof.upload,
                         (double)b->prof.commits, (double)b->prof.staged_bytes, (double)b->prof.pinned_allocs, (double)b->prof.ring_bands};
    for (int i = 0; i < n && i < 9; ++i) if (out) out[i] = v[i];
    return 9;
}
uint64_t ifb200_batch_kernel_launches(const ifb200_batch* b) { return b ? b->launches : 0; }
uint64_t ifb200_batch_fused_jobs(const ifb200_batch* b) { return b ? b->fused_jobs : 0; }
uint64_t ifb200_batch_generic_jobs(const ifb200_batch* b) { return b ? b->generic_jobs : 0; }
uint64_t ifb200_batch_tile_jobs(const ifb200_batch* b) { return b ? b->tile_jobs : 0; }
int ifb200_batch_ring_status(const ifb200_batch* b, char* why, size_t cap) {
    if (!b) return 0;
    put_err(why, cap, b->ring_ok ? std::string() : b->ring_reason);
    return b->ring_ok ? 1 : 0;
}

// ---- drop-in calls with HOST buffers -----------------------------------------------------------
namespace {
bool is_pageable(const void* p) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return true; }
    return a.type == cudaMemoryTypeUnregistered;
}
void ensure_pinned(uint8_t*& p, size_t& cap, size_t need) {
    if (cap >= need) return;
    const size_t want = grown(cap, need);
    if (p) CUDA_OK(cudaFreeHost(p));
    p = nullptr; cap = 0;
    if (cudaMallocHost(&p, want) != cudaSuccess) { cudaGetLastError(); p = nullptr; CUDA_OK(cudaMallocHost(&p, need)); cap = need; return; }
    cap = want;
}
// the result parked in the slot's pinned buffer (if any) goes to the caller's canvas; the slot's stream must have been synchronised
void flush_result(HostCtx& c, HostSlot& sl) {
    if (!sl.out_dst) return;
    c.pool->copy2d(sl.out_dst, sl.out_stride, sl.h_cv, sl.out_pitch, sl.out_row_bytes, sl.out_rows);
    sl.out_dst = nullptr;
}
// one host-buffer job on pipeline slot `sl` (asynchronous; caller synchronises the slot's stream and calls flush_result)
void host_job_async(HostCtx& c, HostSlot& sl, const ifb200_resample_desc& d) {
    ifb200_batch* b = c.batch;
    cudaStream_t st = sl.stream;
    // device images: input window with a 64-byte padded pitch; destination rect only
    const size_t in_pitch = ((size_t)d.in_w * 4 + 63) / 64 * 64;
    const size_t cv_pitch = ((size_t)d.w * 4 + 63) / 64 * 64;
    ensure(sl.d_in, sl.cap_in, in_pitch * d.in_h, st);
    ensure(sl.d_cv, sl.cap_cv, cv_pitch * d.h, st);
    uint8_t* host_rect = d.canvas + (size_t)d.y * d.cv_stride + (size_t)d.x * 4;
    const bool stage_in = is_pageable(d.in), stage_cv = is_pageable(host_rect);
    if (stage_in || stage_cv) {
        if (!c.pool) { c.pool.reset(new CopyPool()); c.pool->start((int)std::min(7u, std::max(1u, std::thread::hardware_concurrency() / 2u))); }
        if (!sl.up_done) CUDA_OK(cudaEventCreateWithFlags(&sl.up_done, cudaEventDisableTiming));
    }
    if (sl.out_dst) { CUDA_OK(cudaStreamSynchronize(st)); flush_result(c, sl); }     // the slot's previous result leaves its pinned buffer
    if (stage_in) {
        if (sl.hcap_in < in_pitch * d.in_h) { CUDA_OK(cudaStreamSynchronize(st)); ensure_pinned(sl.h_in, sl.hcap_in, in_pitch * d.in_h); }
        else CUDA_OK(cudaEventSynchronize(sl.up_done));                              // the previous upload from h_in is through
        c.pool->copy2d(sl.h_in, in_pitch, d.in, d.in_stride, (size_t)d.in_w * 4, d.in_h);
        CUDA_OK(cudaMemcpyAsync(sl.d_in, sl.h_in, in_pitch * d.in_h, cudaMemcpyHostToDevice, st));
        CUDA_OK(cudaEventRecord(sl.up_done, st));
    } else {
        CUDA_OK(cudaMemcpy2DAsync(sl.d_in, in_pitch, d.in, d.in_stride, (size_t)d.in_w * 4, d.in_h, cudaMemcpyHostToDevice, st));
    }
    if (stage_cv && sl.hcap_cv < cv_pitch * d.h) { CUDA_OK(cudaStreamSynchronize(st)); ensure_pinned(sl.h_cv, sl.hcap_cv, cv_pitch * d.h); }
    if (d.compose == IFB200_BLEND_WITH_SELF) {      // the composite reads the canvas (scaling.rs:271-283)
        if (stage_cv) {
            c.pool->copy2d(sl.h_cv, cv_pitch, host_rect, d.cv_stride, (size_t)d.w * 4, d.h);
            CUDA_OK(cudaMemcpyAsync(sl.d_cv, sl.h_cv, cv_pitch * d.h, cudaMemcpyHostToDevice, st));
        } else {
            CUDA_OK(cudaMemcpy2DAsync(sl.d_cv, cv_pitch, host_rect, d.cv_stride, (size_t)d.w * 4, d.h, cudaMemcpyHostToDevice, st));
        }
    }
    ifb200_resample_desc dd = d;
    dd.in = sl.d_in; dd.in_stride = (uint32_t)in_pitch;
    dd.canvas = sl.d_cv; dd.cv_w = d.w; dd.cv_h = d.h; dd.cv_stride = (uint32_t)cv_pitch; dd.x = 0; dd.y = 0;
    enqueue_locked(b, &dd, 1, st);
    if (stage_cv) {
        CUDA_OK(cudaMemcpyAsync(sl.h_cv, sl.d_cv, cv_pitch * d.h, cudaMemcpyDeviceToHost, st));
        sl.out_dst = host_rect; sl.out_stride = d.cv_stride; sl.out_row_bytes = (size_t)d.w * 4; sl.out_rows = d.h; sl.out_pitch = cv_pitch;
    } else {
        CUDA_OK(cudaMemcpy2DAsync(host_rect, d.cv_stride, sl.d_cv, cv_pitch, (size_t)d.w * 4, d.h, cudaMemcpyDeviceToHost, st));
    }
}
}  // namespace

int ifb200_scale_and_render(const ifb200_resample_desc* desc, char* err, size_t cap) {
    return guarded(err, cap, [&] {
        if (!desc) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor");
        validate(*desc);
        HostCtx& c = host_ctx();
        std::lock_guard<std::mutex> lk(c.batch->mu);
        DeviceScope dev_scope_(c.batch->device);
        host_job_async(c, c.slot[0], *desc);
        CUDA_OK(cudaStreamSynchronize(c.slot[0].stream));
        flush_result(c, c.slot[0]);
    });
}

int ifb200_scale_and_render_many(const ifb200_resample_desc* descs, size_t n, char* err, size_t cap) {
    return guarded(err, cap, [&] {
        if (!descs && n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor array");
        for (size_t i = 0; i < n; ++i) validate(descs[i]);      // all-or-nothing argument errors, before any pixel moves
        HostCtx& c = host_ctx();
        std::lock_guard<std::mutex> lk(c.batch->mu);
        DeviceScope dev_scope_(c.batch->device);
        try {
            for (size_t i = 0; i < n; ++i) host_job_async(c, c.slot[i % kHostSlots], descs[i]);
        } catch (...) {
            for (auto& sl : c.slot) { cudaStreamSynchronize(sl.stream); sl.out_dst = nullptr; }
            throw;
        }
        for (auto& sl : c.slot) { CUDA_OK(cudaStreamSynchronize(sl.stream)); flush_result(c, sl); }
    });
}

int ifb200_apply_matte_bgra8(uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, const uint8_t matte_bgra[4], int alpha_meaningful,
                             char* err, size_t cap) {
    return guarded(err, cap, [&] {
        if (!px || !matte_bgra) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null pointer");
        if (!alpha_meaningful) return;                       // blend.rs:10-13
        in_place_on_host(px, w, h, stride, [&](ifb200_batch* b, uint8_t* d, uint32_t pitch, cudaStream_t st) {
            apply_matte_locked(b, d, w, h, pitch, matte_bgra, st);
        });
    });
}

// Only the planned cover travels: each rectangle is one 2D copy into the same place of a device image laid out like the frame, the
// kernel runs on that image, each rectangle comes back with one 2D copy.  Rectangles that are only filled are not uploaded.
int ifb200_round_corners_bgra8(const ifb200_round_corners_desc* d, char* err, size_t cap) {
    return guarded(err, cap, [&] {
        if (!d) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null descriptor");
        int code = 0;
        const std::string why = ifb::round_corners_check(*d, &code);
        if (!why.empty()) IFB_THROW(code, "%s", why.c_str());
        if (d->w == 0 || d->h == 0) return;
        on_host_slot([&](ifb200_batch* b, HostSlot& sl, cudaStream_t st) {
            const size_t pitch = ((size_t)d->w * 4 + 63) / 64 * 64;
            ensure(sl.d_cv, sl.cap_cv, pitch * d->h, st);
            ifb200_round_corners_desc dd = *d;
            dd.px = sl.d_cv; dd.stride = (uint32_t)pitch;
            ifb::RcWork wk;
            std::vector<ifb::RcRect> rects;
            ifb::round_corners_plan(dd, wk, &rects);
            auto dev_at = [&](const ifb::RcRect& r) { return sl.d_cv + (size_t)r.y0 * pitch + (size_t)r.x0 * 4; };
            auto host_at = [&](const ifb::RcRect& r) { return d->px + (size_t)r.y0 * d->stride + (size_t)r.x0 * 4; };
            for (const auto& r : rects)
                if (!r.fill_only) CUDA_OK(cudaMemcpy2DAsync(dev_at(r), pitch, host_at(r), d->stride, (size_t)r.w * 4, r.h, cudaMemcpyHostToDevice, st));
            round_corners_launch(b, wk, st);
            for (const auto& r : rects)
                CUDA_OK(cudaMemcpy2DAsync(host_at(r), d->stride, dev_at(r), pitch, (size_t)r.w * 4, r.h, cudaMemcpyDeviceToHost, st));
            CUDA_OK(cudaStreamSynchronize(st));
        });
    });
}

int ifb200_transpose_bgra8(const uint8_t* from, uint32_t from_stride, uint32_t w, uint32_t h, uint8_t* to, uint32_t to_stride,
                           char* err, size_t cap) {
    return guarded(err, cap, [&] {
        if (!to) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null pointer");
        if (!bgra_window(from, w, h, from_stride) || !bgra_window(to, h, w, to_stride)) return;
        on_host_slot([&](ifb200_batch* b, HostSlot& sl, cudaStream_t st) {
            const size_t pin = ((size_t)w * 4 + 63) / 64 * 64, pout = ((size_t)h * 4 + 63) / 64 * 64;
            ensure(sl.d_in, sl.cap_in, pin * h, st);
            ensure(sl.d_cv, sl.cap_cv, pout * w, st);
            CUDA_OK(cudaMemcpy2DAsync(sl.d_in, pin, from, from_stride, (size_t)w * 4, h, cudaMemcpyHostToDevice, st));
            transpose_locked(b, sl.d_in, (uint32_t)pin, w, h, sl.d_cv, (uint32_t)pout, st);
            CUDA_OK(cudaMemcpy2DAsync(to, to_stride, sl.d_cv, pout, (size_t)h * 4, w, cudaMemcpyDeviceToHost, st));
            CUDA_OK(cudaStreamSynchronize(st));
        });
    });
}

int ifb200_detect_content_from_codes(const uint8_t* codes, uint32_t w, uint32_t h, uint32_t rect[4], uint64_t* centres) {
    return ifb::detect_content_from_codes(codes, w, h, rect, centres) ? IFB200_OK : IFB200_ERR_INVALID_ARGUMENT;
}

int ifb200_batch_detect_content(ifb200_batch* b, const uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride, int alpha_meaningful,
                                uint32_t threshold, uint32_t rect[4], void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { detect_content_locked(b, dev_px, w, h, stride, alpha_meaningful, threshold, st, rect); });
}

int ifb200_batch_detect_content_many(ifb200_batch* b, const ifb200_detect_content_desc* d, size_t n, uint32_t* rects, uint64_t* visited,
                                     void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) { detect_content_many_locked(b, d, n, rects, visited, st); });
}

int ifb200_batch_whitespace_codes(ifb200_batch* b, const uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride, int alpha_meaningful,
                                  uint32_t threshold, uint8_t* dev_codes, void* stream, char* err, size_t cap) {
    return with_batch(b, stream, err, cap, [&](cudaStream_t st) {
        whitespace_codes_locked(b, dev_px, w, h, stride, alpha_meaningful, threshold, dev_codes, st);
    });
}

int ifb200_detect_content_bgra8(const uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, int alpha_meaningful, uint32_t threshold,
                                uint32_t rect[4], char* err, size_t cap) {
    return guarded(err, cap, [&] {
        if (!rect) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null pointer");
        if (!bgra_window(px, w, h, stride)) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "empty bitmap");
        on_host_slot([&](ifb200_batch* b, HostSlot& sl, cudaStream_t st) {
            const size_t pitch = ((size_t)w * 4 + 63) / 64 * 64;
            ensure(sl.d_cv, sl.cap_cv, pitch * h, st);
            CUDA_OK(cudaMemcpy2DAsync(sl.d_cv, pitch, px, stride, (size_t)w * 4, h, cudaMemcpyHostToDevice, st));
            detect_content_locked(b, sl.d_cv, w, h, (uint32_t)pitch, alpha_meaningful, threshold, st, rect);
        });
    });
}

int ifb200_block_scale_u8(const uint8_t* in, uint32_t in_stride, uint32_t blocks_x, uint32_t blocks_y, uint8_t* out, uint32_t out_stride, int n, int srgb,
                          char* err, size_t cap) {
    return guarded(err, cap, [&] {
        if (!in || !out) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null pointer");
        if (n < 1 || n > 7) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "block scalers exist for 1x1 .. 7x7 (got %d)", n);
        if (blocks_x == 0 || blocks_y == 0) return;
        if (in_stride < blocks_x * 8ull || out_stride < (uint64_t)blocks_x * (uint32_t)n) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "stride smaller than a row of blocks");
        on_host_slot([&](ifb200_batch* b, HostSlot& sl, cudaStream_t st) {
            const size_t pin = ((size_t)blocks_x * 8 + 63) / 64 * 64, pout = ((size_t)blocks_x * n + 63) / 64 * 64;
            ensure(sl.d_in, sl.cap_in, pin * blocks_y * 8, st);
            ensure(sl.d_cv, sl.cap_cv, pout * blocks_y * n, st);
            CUDA_OK(cudaMemcpy2DAsync(sl.d_in, pin, in, in_stride, (size_t)blocks_x * 8, (size_t)blocks_y * 8, cudaMemcpyHostToDevice, st));
            block_scale_locked(b, sl.d_in, (uint32_t)pin, blocks_x, blocks_y, sl.d_cv, (uint32_t)pout, n, srgb, st);
            CUDA_OK(cudaMemcpy2DAsync(out, out_stride, sl.d_cv, pout, (size_t)blocks_x * n, (size_t)blocks_y * n, cudaMemcpyDeviceToHost, st));
            CUDA_OK(cudaStreamSynchronize(st));
        });
    });
}

int ifb200_white_balance_srgb_bgra8(uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, float threshold, char* err, size_t cap) {
    return guarded(err, cap, [&] {
        in_place_on_host(px, w, h, stride, [&](ifb200_batch* b, uint8_t* d, uint32_t pitch, cudaStream_t st) {
            white_balance_locked(b, d, w, h, pitch, threshold, st);
        });
    });
}

int ifb200_flip_vertical_bgra8(uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, char* err, size_t cap) {
    return guarded(err, cap, [&] {
        in_place_on_host(px, w, h, stride, [&](ifb200_batch* b, uint8_t* d, uint32_t pitch, cudaStream_t st) { flip_locked(b, true, d, w, h, pitch, st); });
    });
}
int ifb200_flip_horizontal_bgra8(uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, char* err, size_t cap) {
    return guarded(err, cap, [&] {
        in_place_on_host(px, w, h, stride, [&](ifb200_batch* b, uint8_t* d, uint32_t pitch, cudaStream_t st) { flip_locked(b, false, d, w, h, pitch, st); });
    });
}

int ifb200_color_matrix_bgra8(uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, const float m[25], char* err, size_t cap) {
    return guarded(err, cap, [&] {
        if (!m) IFB_THROW(IFB200_ERR_INVALID_ARGUMENT, "null pointer");
        in_place_on_host(px, w, h, stride, [&](ifb200_batch* b, uint8_t* d, uint32_t pitch, cudaStream_t st) {
            color_matrix_locked(b, d, w, h, pitch, m, st);
        });
    });
}

}  // extern "C"
