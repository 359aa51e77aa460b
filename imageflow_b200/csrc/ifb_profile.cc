// ifb_profile.cc -- see ifb_profile.h.  Product code: must not include or link anything from the test oracle.
#include "ifb_profile.h"

#include <cmath>
#include <cstring>

#include "ifb_weights.h"

namespace ifb {
namespace {

using Mat = double[3][3];

// ---------------------------------------------------------------- tone curves
// One channel's curve on [0, 1], evaluated in float64.  A power of a base <= 0 is 0.
struct Trc {
    enum Kind { kIdentity, kPower, kTable, kPara, kBt709, kSmpte240 } kind = kIdentity;
    int para = 0;                                    // kPara: ICC function type 0..4
    double g = 1, a = 1, b = 0, c = 0, d = 0, e = 0, f = 0;
    std::vector<uint16_t> table;                     // kTable: at least 2 entries

    static double pw(double x, double y) { return x > 0 ? std::pow(x, y) : 0.0; }
    double operator()(double x) const {
        switch (kind) {
            case kIdentity: return x;
            case kPower: return pw(x, g);
            case kTable: {
                const double pos = x * (double)(table.size() - 1);
                size_t i = (size_t)std::floor(pos);
                if (i > table.size() - 2) i = table.size() - 2;
                const double t = pos - (double)i;
                return ((double)table[i] + ((double)table[i + 1] - (double)table[i]) * t) / 65535.0;
            }
            case kPara:                              // ICC.1:2010 §10.18, table 65
                switch (para) {
                    case 0: return pw(x, g);
                    case 1: return a * x + b >= 0 ? pw(a * x + b, g) : 0.0;
                    case 2: return a * x + b >= 0 ? pw(a * x + b, g) + c : c;
                    case 3: return x >= d ? pw(a * x + b, g) : c * x;
                    default: return x >= d ? pw(a * x + b, g) + e : c * x + f;
                }
            case kBt709: return x < 4.5 * 0.018 ? x / 4.5 : pw((x + 0.099) / 1.099, 1.0 / 0.45);        // H.273 1, 6, 14, 15
            case kSmpte240: return x < 4.0 * 0.0228 ? x / 4.0 : pw((x + 0.1115) / 1.1115, 1.0 / 0.45);  // H.273 7
        }
        return 0.0;
    }
    static Trc power(double g) { Trc t; t.kind = kPower; t.g = g; return t; }
    static Trc srgb() { Trc t; t.kind = kPara; t.para = 3; t.g = 2.4; t.a = 1 / 1.055; t.b = 0.055 / 1.055; t.c = 1 / 12.92; t.d = 0.04045; return t; }
};

// ---------------------------------------------------------------- colorimetry
void mul(const Mat a, const Mat b, Mat out) {
    Mat r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r[i][j] = a[i][0] * b[0][j] + a[i][1] * b[1][j] + a[i][2] * b[2][j];
    std::memcpy(out, r, sizeof r);
}

bool inverse(const Mat m, Mat out) {
    const double c00 = m[1][1] * m[2][2] - m[1][2] * m[2][1], c01 = m[1][2] * m[2][0] - m[1][0] * m[2][2],
                 c02 = m[1][0] * m[2][1] - m[1][1] * m[2][0];
    const double det = m[0][0] * c00 + m[0][1] * c01 + m[0][2] * c02;
    if (!std::isfinite(det) || std::fabs(det) < 1e-12) return false;
    const Mat r = {{c00 / det, (m[0][2] * m[2][1] - m[0][1] * m[2][2]) / det, (m[0][1] * m[1][2] - m[0][2] * m[1][1]) / det},
                   {c01 / det, (m[0][0] * m[2][2] - m[0][2] * m[2][0]) / det, (m[0][2] * m[1][0] - m[0][0] * m[1][2]) / det},
                   {c02 / det, (m[0][1] * m[2][0] - m[0][0] * m[2][1]) / det, (m[0][0] * m[1][1] - m[0][1] * m[1][0]) / det}};
    std::memcpy(out, r, sizeof r);
    return true;
}

constexpr double kD50[3] = {0.9642, 1.0, 0.8249};   // the ICC PCS illuminant
constexpr double kD65[2] = {0.3127, 0.3290};

// The colorants (columns: the XYZ of red, green, blue) of chromaticities xy = {wx, wy, rx, ry, gx, gy, bx, by}, scaled so that
// (1, 1, 1) is the white point at Y = 1 and then Bradford-adapted from that white to D50.  False when they give no matrix.
bool colorants_d50(const double xy[8], Mat out) {
    for (int i = 0; i < 8; ++i)
        if (!std::isfinite(xy[i])) return false;
    if (!(xy[1] > 0)) return false;
    const double w[3] = {xy[0] / xy[1], 1.0, (1.0 - xy[0] - xy[1]) / xy[1]};
    Mat p, pi;
    for (int k = 0; k < 3; ++k) {
        const double x = xy[2 + 2 * k], y = xy[3 + 2 * k];
        p[0][k] = x; p[1][k] = y; p[2][k] = 1.0 - x - y;
    }
    if (!inverse(p, pi)) return false;
    double s[3];
    for (int i = 0; i < 3; ++i) s[i] = pi[i][0] * w[0] + pi[i][1] * w[1] + pi[i][2] * w[2];
    Mat c;
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k) c[i][k] = p[i][k] * s[k];
    static const Mat kBradford = {{0.8951, 0.2664, -0.1614}, {-0.7502, 1.7135, 0.0367}, {0.0389, -0.0685, 1.0296}};
    Mat bi;
    inverse(kBradford, bi);
    double cs[3], cd[3];
    for (int i = 0; i < 3; ++i) {
        cs[i] = kBradford[i][0] * w[0] + kBradford[i][1] * w[1] + kBradford[i][2] * w[2];
        cd[i] = kBradford[i][0] * kD50[0] + kBradford[i][1] * kD50[1] + kBradford[i][2] * kD50[2];
        if (!(std::fabs(cs[i]) > 1e-12)) return false;
    }
    Mat dg = {{cd[0] / cs[0], 0, 0}, {0, cd[1] / cs[1], 0}, {0, 0, cd[2] / cs[2]}}, a;
    mul(bi, dg, a);
    mul(a, kBradford, a);
    mul(a, c, out);
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k)
            if (!std::isfinite(out[i][k])) return false;
    return true;
}

// T_c and M = f32(S^-1 C) into plan; false when C gives no finite matrix
bool plan_matrix(const Trc trc[3], const Mat c, ifb200_profile_plan* plan) {
    static const double kSrgb[8] = {kD65[0], kD65[1], 0.64, 0.33, 0.30, 0.60, 0.15, 0.06};
    Mat s, si, m;
    colorants_d50(kSrgb, s);
    inverse(s, si);
    mul(si, c, m);
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k) {
            if (!std::isfinite(m[i][k])) return false;
            plan->m[i][k] = (float)m[i][k];
        }
    for (int ch = 0; ch < 3; ++ch)
        for (int v = 0; v < 256; ++v) {
            const double y = trc[ch](v / 255.0);
            plan->trc[ch][v] = (float)(y > 0 ? (y < 1 ? y : 1.0) : 0.0);           // clip01, NaN -> 0
        }
    plan->kind = IFB200_PLAN_MATRIX;
    return true;
}

// the gray byte map: the kernel's encode (ifb_lut.cuh lut_encode) of each T[v], on the host
void plan_gray(const Trc& trc, ifb200_profile_plan* plan) {
    static const std::vector<uint8_t> lut = [] { std::vector<uint8_t> t(16384); linear_to_srgb_table(t.data()); return t; }();
    for (int v = 0; v < 256; ++v) {
        const double y = trc(v / 255.0);
        const float t = (float)(y > 0 ? (y < 1 ? y : 1.0) : 0.0);
        plan->trc[0][v] = t;
        float s = t * 16383.0f;
        s = std::fmin(std::fmax(s, 0.0f), 16383.0f);
        plan->gray[v] = lut[(int)s];
    }
    plan->kind = IFB200_PLAN_GRAY;
}

// ---------------------------------------------------------------- ICC
struct Status {
    int code = IFB200_OK;
    std::string why;
    bool ok() const { return code == IFB200_OK; }
};
Status fail(int code, std::string why) { return Status{code, std::move(why)}; }
Status invalid(std::string why) { return fail(IFB200_ERR_INVALID_ARGUMENT, std::move(why)); }
Status unsupported(std::string why) { return fail(IFB200_ERR_NOT_IMPLEMENTED, std::move(why)); }

uint32_t be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
uint16_t be16(const uint8_t* p) { return (uint16_t)(p[0] << 8 | p[1]); }
double s15f16(const uint8_t* p) { return (double)(int32_t)be32(p) / 65536.0; }
uint32_t sig(const char* s) { return be32(reinterpret_cast<const uint8_t*>(s)); }
std::string sig_name(uint32_t s) {
    std::string r;
    for (int i = 3; i >= 0; --i) {
        const char ch = (char)(s >> (8 * i));
        r += ch >= 32 && ch < 127 ? ch : '?';
    }
    return "'" + r + "'";
}

struct Icc {
    const uint8_t* p = nullptr;
    uint32_t size = 0;                               // the header's size, <= the buffer's length
    struct Tag { uint32_t sig, off, size; };
    std::vector<Tag> tags;

    const Tag* find(uint32_t s) const {
        for (const Tag& t : tags)
            if (t.sig == s) return &t;
        return nullptr;
    }
};

Status parse_header(const uint8_t* bytes, size_t len, Icc& icc) {
    if (!bytes) return invalid("null ICC profile pointer");
    if (len < 132) return invalid("ICC profile truncated: " + std::to_string(len) + " bytes, a header and tag count take 132");
    const uint32_t size = be32(bytes);
    if (size > len) return invalid("ICC profile truncated: the header says " + std::to_string(size) + " bytes, the buffer holds " + std::to_string(len));
    if (size < 132) return invalid("ICC profile size " + std::to_string(size) + " is smaller than its header");
    if (be32(bytes + 36) != sig("acsp")) return invalid("not an ICC profile (no 'acsp' signature)");
    const uint32_t n = be32(bytes + 128);
    if (132 + 12 * (uint64_t)n > size) return invalid("ICC tag table of " + std::to_string(n) + " tags runs past the profile's end");
    icc.p = bytes; icc.size = size;
    for (uint32_t i = 0; i < n; ++i) {
        const uint8_t* e = bytes + 132 + 12 * (size_t)i;
        const Icc::Tag t{be32(e), be32(e + 4), be32(e + 8)};
        if ((uint64_t)t.off + t.size > size) return invalid("ICC tag " + sig_name(t.sig) + " runs past the profile's end");
        icc.tags.push_back(t);
    }
    return {};
}

Status read_xyz(const Icc& icc, const char* name, double out[3]) {
    const Icc::Tag* t = icc.find(sig(name));
    if (!t) return invalid(std::string("ICC profile has no ") + name + " tag");
    if (t->size < 20 || be32(icc.p + t->off) != sig("XYZ ")) return invalid(std::string("ICC ") + name + " tag is not a 20-byte 'XYZ ' value");
    for (int i = 0; i < 3; ++i) out[i] = s15f16(icc.p + t->off + 8 + 4 * i);
    return {};
}

Status read_trc(const Icc& icc, const char* name, Trc& out) {
    const Icc::Tag* t = icc.find(sig(name));
    if (!t) return invalid(std::string("ICC profile has no ") + name + " tag");
    const uint8_t* p = icc.p + t->off;
    if (t->size < 12) return invalid(std::string("ICC ") + name + " tag truncated");
    const uint32_t type = be32(p);
    if (type == sig("curv")) {
        const uint32_t n = be32(p + 8);
        if (12 + 2 * (uint64_t)n > t->size) return invalid(std::string("ICC ") + name + " 'curv' of " + std::to_string(n) + " entries truncated");
        if (n == 0) out = Trc{};
        else if (n == 1) out = Trc::power(be16(p + 12) / 256.0);
        else {
            out = Trc{};
            out.kind = Trc::kTable;
            out.table.resize(n);
            for (uint32_t i = 0; i < n; ++i) out.table[i] = be16(p + 12 + 2 * (size_t)i);
        }
        return {};
    }
    if (type == sig("para")) {
        static const int kParams[5] = {1, 3, 4, 5, 7};
        const uint16_t f = be16(p + 8);
        if (f > 4) return invalid(std::string("ICC ") + name + " 'para' function type " + std::to_string(f) + " (0..4 exist)");
        if (12 + 4 * (uint64_t)kParams[f] > t->size) return invalid(std::string("ICC ") + name + " 'para' truncated");
        double v[7] = {0, 0, 0, 0, 0, 0, 0};
        for (int i = 0; i < kParams[f]; ++i) v[i] = s15f16(p + 12 + 4 * i);
        out = Trc{};
        out.kind = Trc::kPara; out.para = f; out.g = v[0];
        out.a = v[1]; out.b = v[2]; out.c = v[3]; out.d = v[4]; out.e = v[5]; out.f = v[6];
        return {};
    }
    return invalid(std::string("ICC ") + name + " tag has type " + sig_name(type) + ", not 'curv' or 'para'");
}

Status plan_icc(const uint8_t* bytes, size_t len, bool gray, ifb200_profile_plan* plan) {
    Icc icc;
    Status st = parse_header(bytes, len, icc);
    if (!st.ok()) return st;
    const uint8_t major = bytes[8];
    if (major != 2 && major != 4) return unsupported("ICC version " + std::to_string(major) + " (2 and 4 are supported)");
    const uint32_t space = be32(bytes + 16), pcs = be32(bytes + 20);
    if (space == sig("CMYK")) return unsupported("CMYK ICC profile");
    if (space != sig("RGB ") && space != sig("GRAY")) return unsupported("ICC colour space " + sig_name(space));
    static const char* const kLutTags[] = {"A2B0", "A2B1", "A2B2", "B2A0", "B2A1", "B2A2", "D2B0", "D2B1", "D2B2", "D2B3",
                                           "B2D0", "B2D1", "B2D2", "B2D3"};
    static const char* const kLutTypes[] = {"mft1", "mft2", "mAB ", "mBA "};
    for (const Icc::Tag& t : icc.tags) {
        for (const char* s : kLutTags)
            if (t.sig == sig(s)) return unsupported("LUT-based ICC profile (" + sig_name(t.sig) + " tag)");
        if (t.size >= 4)
            for (const char* s : kLutTypes)
                if (be32(bytes + t.off) == sig(s)) return unsupported("LUT-based ICC profile (" + sig_name(t.sig) + " tag of type " + sig_name(sig(s)) + ")");
    }
    if (pcs == sig("Lab ")) return unsupported("ICC profile with a Lab PCS");
    if (pcs != sig("XYZ ")) return invalid("ICC PCS " + sig_name(pcs) + " (neither 'XYZ ' nor 'Lab ')");
    if (gray != (space == sig("GRAY")))
        return invalid(gray ? "an RGB ICC profile given as ICC_GRAY" : "a GRAY ICC profile given as ICC");
    if (gray) {
        Trc k;
        if (!(st = read_trc(icc, "kTRC", k)).ok()) return st;
        plan_gray(k, plan);
        return {};
    }
    Trc trc[3];
    double xyz[3][3];
    const char* const kXyz[3] = {"rXYZ", "gXYZ", "bXYZ"};
    const char* const kTrc[3] = {"rTRC", "gTRC", "bTRC"};
    for (int k = 0; k < 3; ++k) {
        if (!(st = read_xyz(icc, kXyz[k], xyz[k])).ok()) return st;
        if (!(st = read_trc(icc, kTrc[k], trc[k])).ok()) return st;
    }
    Mat c;
    for (int i = 0; i < 3; ++i)
        for (int k = 0; k < 3; ++k) c[i][k] = xyz[k][i];
    if (!plan_matrix(trc, c, plan)) return invalid("ICC colorants give no finite matrix");
    return {};
}

// ---------------------------------------------------------------- CICP (ITU-T H.273)
// table 2: white x, y, then red, green, blue x, y
bool cicp_primaries(int cp, double xy[8]) {
    static const double kC[2] = {0.310, 0.316};
    struct Row { int code; double v[8]; };
    static const Row kRows[] = {
        {1, {kD65[0], kD65[1], 0.640, 0.330, 0.300, 0.600, 0.150, 0.060}},
        {4, {kC[0], kC[1], 0.67, 0.33, 0.21, 0.71, 0.14, 0.08}},
        {5, {kD65[0], kD65[1], 0.64, 0.33, 0.29, 0.60, 0.15, 0.06}},
        {6, {kD65[0], kD65[1], 0.630, 0.340, 0.310, 0.595, 0.155, 0.070}},
        {7, {kD65[0], kD65[1], 0.630, 0.340, 0.310, 0.595, 0.155, 0.070}},
        {8, {kC[0], kC[1], 0.681, 0.319, 0.243, 0.692, 0.145, 0.049}},
        {9, {kD65[0], kD65[1], 0.708, 0.292, 0.170, 0.797, 0.131, 0.046}},
        {10, {1.0 / 3.0, 1.0 / 3.0, 1.0, 0.0, 0.0, 1.0, 0.0, 0.0}},
        {11, {0.314, 0.351, 0.680, 0.320, 0.265, 0.690, 0.150, 0.060}},
        {12, {kD65[0], kD65[1], 0.680, 0.320, 0.265, 0.690, 0.150, 0.060}},
        {22, {kD65[0], kD65[1], 0.630, 0.340, 0.295, 0.605, 0.155, 0.077}},
    };
    for (const Row& r : kRows)
        if (r.code == cp) { std::memcpy(xy, r.v, sizeof r.v); return true; }
    return false;
}

Status plan_cicp(const uint8_t cicp[4], ifb200_profile_plan* plan) {
    const int cp = cicp[0], tc = cicp[1], mc = cicp[2];
    if (cp == 1 && tc == 13) { plan->kind = IFB200_PLAN_IDENTITY; return {}; }
    if (mc != 0) return unsupported("CICP matrix coefficients " + std::to_string(mc) + " (only 0, RGB, is supported)");
    if (!cicp[3]) return unsupported("CICP narrow (video) range");
    if (tc == 16 || tc == 18) return unsupported(std::string("CICP transfer ") + (tc == 16 ? "PQ (16)" : "HLG (18)") + " needs tone mapping");
    Trc t;
    switch (tc) {
        case 1: case 6: case 14: case 15: t.kind = Trc::kBt709; break;
        case 4: t = Trc::power(2.2); break;
        case 5: t = Trc::power(2.8); break;
        case 7: t.kind = Trc::kSmpte240; break;
        case 8: break;
        case 13: t = Trc::srgb(); break;
        default: return unsupported("CICP transfer characteristics " + std::to_string(tc));
    }
    double xy[8];
    if (!cicp_primaries(cp, xy)) return unsupported("CICP colour primaries " + std::to_string(cp));
    Mat c;
    colorants_d50(xy, c);
    const Trc trc[3] = {t, t, t};
    if (!plan_matrix(trc, c, plan)) return invalid("CICP primaries give no finite matrix");
    return {};
}

Status plan_gamma_primaries(double gamma, const double chrm[8], ifb200_profile_plan* plan) {
    if (!(std::isfinite(gamma) && gamma > 0)) return invalid("gAMA " + std::to_string(gamma) + " is not a positive number");
    const double e = (double)(float)(1.0 / gamma);
    if (!std::isfinite(e)) return invalid("gAMA " + std::to_string(gamma) + " gives no finite decoding gamma");
    Mat c;
    if (!colorants_d50(chrm, c)) return invalid("cHRM chromaticities give no finite matrix");
    const Trc t = Trc::power(e), trc[3] = {t, t, t};
    if (!plan_matrix(trc, c, plan)) return invalid("cHRM chromaticities give no finite matrix");
    return {};
}

// the same profile for plan sharing: bytes or parameters compared exactly
bool same_profile(const ifb200_source_profile& a, const ifb200_source_profile& b) {
    if (a.kind != b.kind) return false;
    switch (a.kind) {
        case IFB200_PROFILE_ICC: case IFB200_PROFILE_ICC_GRAY:
            return a.icc_len == b.icc_len && (a.icc == b.icc || (a.icc && b.icc && std::memcmp(a.icc, b.icc, a.icc_len) == 0));
        case IFB200_PROFILE_GAMMA_PRIMARIES:
            return std::memcmp(&a.gamma, &b.gamma, sizeof a.gamma) == 0 && std::memcmp(a.chrm, b.chrm, sizeof a.chrm) == 0;
        case IFB200_PROFILE_CICP: return std::memcmp(a.cicp, b.cicp, 4) == 0;
        default: return true;
    }
}

// the descriptor alone as pixel_convert's (a BGRA source as RGBA_TO_BGRA: the same bytes per pixel and in-place rule)
ifb200_pixel_convert_desc as_pixel_convert(const ifb200_to_srgb_desc& d) {
    ifb200_pixel_convert_desc p{};
    p.op = d.format == IFB200_PROFILE_SRC_BGRA ? IFB200_PIXEL_RGBA_TO_BGRA : d.format;
    p.src = d.src; p.src_stride = d.src_stride; p.dst = d.dst; p.dst_stride = d.dst_stride; p.w = d.w; p.h = d.h;
    return p;
}

std::string check_desc(const ifb200_to_srgb_desc& d, int* code) {
    *code = IFB200_ERR_INVALID_ARGUMENT;
    if (d.format != IFB200_PROFILE_SRC_BGRA && (d.format < IFB200_PIXEL_RGB24_TO_BGRA || d.format > IFB200_PIXEL_GRAY_ALPHA_TO_BGRA))
        return "format " + std::to_string(d.format) + " is neither IFB200_PROFILE_SRC_BGRA nor a *_TO_BGRA pixel op";
    if (!d.profile) return "null profile pointer";
    if (d.profile->kind < IFB200_PROFILE_SRGB || d.profile->kind > IFB200_PROFILE_CICP)
        return "unknown profile kind " + std::to_string(d.profile->kind);
    return pixel_convert_check(as_pixel_convert(d), code);
}

}  // namespace

int profile_plan(const ifb200_source_profile& p, ifb200_profile_plan* plan, std::string* why) {
    std::memset(plan, 0, sizeof *plan);
    Status st;
    switch (p.kind) {
        case IFB200_PROFILE_SRGB: plan->kind = IFB200_PLAN_IDENTITY; break;
        case IFB200_PROFILE_ICC: case IFB200_PROFILE_ICC_GRAY:
            st = plan_icc(p.icc, p.icc_len, p.kind == IFB200_PROFILE_ICC_GRAY, plan);
            break;
        case IFB200_PROFILE_GAMMA_PRIMARIES: st = plan_gamma_primaries(p.gamma, p.chrm, plan); break;
        case IFB200_PROFILE_CICP: st = plan_cicp(p.cicp, plan); break;
        default: st = invalid("unknown profile kind " + std::to_string(p.kind));
    }
    if (!st.ok()) {
        std::memset(plan, 0, sizeof *plan);
        if (why) *why = st.why;
    }
    return st.code;
}

int ProfilePlans::add(const ifb200_source_profile& p, uint32_t* index, std::string* why) {
    size_t k = 0;
    while (k < planned.size() && !same_profile(*planned[k], p)) ++k;
    *index = (uint32_t)k;
    if (k < planned.size()) return IFB200_OK;
    plans.emplace_back();
    planned.push_back(&p);
    return profile_plan(p, &plans.back(), why);
}

std::string transform_to_srgb_prepare(const ifb200_to_srgb_desc* d, size_t n, PfWork& wk, int* code) {
    ProfilePlans pp;
    std::vector<uint32_t> plan_of(n, 0);
    for (size_t i = 0; i < n; ++i) {
        if (d[i].w == 0 || d[i].h == 0) continue;
        std::string why = check_desc(d[i], code);
        if (why.empty()) *code = pp.add(*d[i].profile, &plan_of[i], &why);
        if (!why.empty()) return "transform to srgb job " + std::to_string(i) + ": " + why;
    }
    *code = IFB200_OK;
    for (size_t i = 0; i < n; ++i) {
        if (d[i].w == 0 || d[i].h == 0) continue;
        const bool bgra = d[i].format == IFB200_PROFILE_SRC_BGRA;
        if (bgra && d[i].src == d[i].dst && pp.plans[plan_of[i]].kind == IFB200_PLAN_IDENTITY) continue;   // nothing to write
        pixel_convert_plan(as_pixel_convert(d[i]), wk.pc);
        wk.plan_of.push_back(plan_of[i] | (bgra ? kPfBgra : 0u));
    }
    wk.plans = std::move(pp.plans);
    return "";
}

}  // namespace ifb
