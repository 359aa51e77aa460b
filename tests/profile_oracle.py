"""Colour profiles to sRGB restated for the tests (test oracle; nothing in the product imports it): an ICC writer for the fixture
profiles, an independent parser and float64 restatement of the transform (exact tone curves, exact matrix, exact sRGB encode, round to
nearest), and the numpy fp32 per-pixel oracle in the kernel's order, fed the planner's tables and matrix (read through
imageflow_b200.source_profile_plan).  The semantics are those of include/ifb200.h ifb200_source_profile."""
import struct

import numpy as np

D50 = np.array([0.9642, 1.0, 0.8249])
D65 = (0.3127, 0.3290)
SRGB_XY = (D65[0], D65[1], 0.64, 0.33, 0.30, 0.60, 0.15, 0.06)
P3_XY = (D65[0], D65[1], 0.680, 0.320, 0.265, 0.690, 0.150, 0.060)
ADOBE_XY = (D65[0], D65[1], 0.64, 0.33, 0.21, 0.71, 0.15, 0.06)
PROPHOTO_XY = (0.3457, 0.3585, 0.7347, 0.2653, 0.1596, 0.8404, 0.0366, 0.0001)
BRADFORD = np.array([[0.8951, 0.2664, -0.1614], [-0.7502, 1.7135, 0.0367], [0.0389, -0.0685, 1.0296]])


# ---------------------------------------------------------------- colorimetry (float64)
def colorants_d50(xy):
    """columns = XYZ of red, green, blue for chromaticities (wx, wy, rx, ry, gx, gy, bx, by), white at Y = 1, Bradford-adapted to D50"""
    wx, wy = xy[0], xy[1]
    w = np.array([wx / wy, 1.0, (1 - wx - wy) / wy])
    p = np.array([[xy[2 + 2 * k], xy[3 + 2 * k], 1 - xy[2 + 2 * k] - xy[3 + 2 * k]] for k in range(3)]).T
    c = p * np.linalg.solve(p, w)[None, :]
    cs, cd = BRADFORD @ w, BRADFORD @ D50
    a = np.linalg.inv(BRADFORD) @ np.diag(cd / cs) @ BRADFORD
    return a @ c


SRGB_D50 = colorants_d50(SRGB_XY)


def matrix_of(c):
    """S^-1 C in float64"""
    return np.linalg.solve(SRGB_D50, c)


# ---------------------------------------------------------------- tone curves (float64 on arrays in [0, 1])
def _pw(x, g):
    x = np.asarray(x, np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(x > 0, np.power(np.maximum(x, 1e-300), g), 0.0)


def para(ftype, p):
    g, a, b, c, d, e, f = (list(p) + [0.0] * 7)[:7]
    if ftype == 0:
        return lambda x: _pw(x, g)
    if ftype == 1:
        return lambda x: np.where(a * x + b >= 0, _pw(a * x + b, g), 0.0)
    if ftype == 2:
        return lambda x: np.where(a * x + b >= 0, _pw(a * x + b, g) + c, c)
    if ftype == 3:
        return lambda x: np.where(x >= d, _pw(a * x + b, g), c * x)
    return lambda x: np.where(x >= d, _pw(a * x + b, g) + e, c * x + f)


def curv(table):
    t = np.asarray(table, np.float64)
    if t.size == 0:
        return lambda x: np.asarray(x, np.float64)
    if t.size == 1:
        return lambda x: _pw(x, t[0] / 256.0)

    def f(x):
        pos = np.asarray(x, np.float64) * (t.size - 1)
        i = np.minimum(np.floor(pos).astype(np.int64), t.size - 2)
        return (t[i] + (t[i + 1] - t[i]) * (pos - i)) / 65535.0
    return f


SRGB_PARA = (2.4, 1 / 1.055, 0.055 / 1.055, 1 / 12.92, 0.04045)


def cicp_transfer(tc):
    if tc in (1, 6, 14, 15):
        return lambda x: np.where(x < 4.5 * 0.018, x / 4.5, _pw((x + 0.099) / 1.099, 1 / 0.45))
    if tc == 4:
        return lambda x: _pw(x, 2.2)
    if tc == 5:
        return lambda x: _pw(x, 2.8)
    if tc == 7:
        return lambda x: np.where(x < 4 * 0.0228, x / 4, _pw((x + 0.1115) / 1.1115, 1 / 0.45))
    if tc == 8:
        return lambda x: np.asarray(x, np.float64)
    if tc == 13:
        return para(3, SRGB_PARA)
    raise KeyError(tc)


CICP_PRIMARIES = {1: SRGB_XY, 4: (0.310, 0.316, 0.67, 0.33, 0.21, 0.71, 0.14, 0.08), 5: (D65[0], D65[1], 0.64, 0.33, 0.29, 0.60, 0.15, 0.06),
                  6: (D65[0], D65[1], 0.630, 0.340, 0.310, 0.595, 0.155, 0.070), 7: (D65[0], D65[1], 0.630, 0.340, 0.310, 0.595, 0.155, 0.070),
                  8: (0.310, 0.316, 0.681, 0.319, 0.243, 0.692, 0.145, 0.049), 9: (D65[0], D65[1], 0.708, 0.292, 0.170, 0.797, 0.131, 0.046),
                  10: (1 / 3, 1 / 3, 1.0, 0.0, 0.0, 1.0, 0.0, 0.0), 11: (0.314, 0.351, 0.680, 0.320, 0.265, 0.690, 0.150, 0.060),
                  12: P3_XY, 22: (D65[0], D65[1], 0.630, 0.340, 0.295, 0.605, 0.155, 0.077)}


# ---------------------------------------------------------------- ICC writer
def s15(v):
    return struct.pack(">i", int(round(v * 65536)))


def xyz_tag(xyz):
    return b"XYZ " + b"\0" * 4 + b"".join(s15(v) for v in xyz)


def curv_tag(entries):
    """entries: [] identity, [gamma_u8f8] a gamma, else a u16 table"""
    return b"curv" + b"\0" * 4 + struct.pack(">I", len(entries)) + b"".join(struct.pack(">H", int(e)) for e in entries)


def para_tag(ftype, params):
    return b"para" + b"\0" * 4 + struct.pack(">HH", ftype, 0) + b"".join(s15(v) for v in params)


def write_icc(space, tags, version=4, pcs=b"XYZ ", cls=b"mntr"):
    """an ICC profile of colour space `space` (b'RGB ', b'GRAY', ...) with tags [(signature, data)]; each data block padded to 4"""
    n = len(tags)
    off = 132 + 12 * n
    table, blob = b"", b""
    for sig, data in tags:
        table += sig + struct.pack(">II", off + len(blob), len(data))
        blob += data + b"\0" * (-len(data) % 4)
    hdr = bytearray(128)
    size = 132 + 12 * n + len(blob)
    struct.pack_into(">I", hdr, 0, size)
    hdr[8] = version
    hdr[12:16], hdr[16:20], hdr[20:24], hdr[36:40] = cls, space, pcs, b"acsp"
    hdr[68:80] = s15(0.9642) + s15(1.0) + s15(0.8249)
    return bytes(hdr) + struct.pack(">I", n) + table + blob


def rgb_profile(xy, trcs, version=4, extra=()):
    """a matrix/TRC profile: colorants from chromaticities adapted to D50, quantised to s15Fixed16 as a profile stores them"""
    c = colorants_d50(xy)
    tags = [(b"rXYZ", xyz_tag(c[:, 0])), (b"gXYZ", xyz_tag(c[:, 1])), (b"bXYZ", xyz_tag(c[:, 2]))]
    tags += [(s, t) for s, t in zip((b"rTRC", b"gTRC", b"bTRC"), trcs)]
    return write_icc(b"RGB ", tags + list(extra), version)


def fixtures():
    """name -> (kind 'icc' / 'icc_gray', bytes) of the synthesised fixture profiles"""
    p3 = para_tag(3, SRGB_PARA)
    srgb_table = [round(65535 * float(para(3, SRGB_PARA)(np.array(i / 1023.0)))) for i in range(1024)]
    p4 = para_tag(4, (2.2, 0.95, 0.05, 1 / 10.0, 0.05, 0.01, 0.002))
    return {
        "display_p3_v4": ("icc", rgb_profile(P3_XY, [p3] * 3, 4)),
        "adobe_rgb_v2": ("icc", rgb_profile(ADOBE_XY, [curv_tag([563])] * 3, 2)),
        "prophoto_v2": ("icc", rgb_profile(PROPHOTO_XY, [curv_tag([round(1.8 * 256)])] * 3, 2)),
        "srgb_curv1024_v2": ("icc", rgb_profile(SRGB_XY, [curv_tag(srgb_table)] * 3, 2)),
        "srgb_para3_v4": ("icc", rgb_profile(SRGB_XY, [p3] * 3, 4)),
        "para4_v4": ("icc", rgb_profile(P3_XY, [p4, para_tag(0, (1.8,)), curv_tag([])], 4)),
        "gray22_v2": ("icc_gray", write_icc(b"GRAY", [(b"kTRC", curv_tag([round(2.2 * 256)]))], 2)),
    }


def lut_profile(space=b"CMYK", pcs=b"Lab "):
    """a small LUT profile header (A2B0 of type mft2, truncated table) standing in for the reference's 557 KB cmyk.icc"""
    return write_icc(space, [(b"A2B0", b"mft2" + b"\0" * 48)], 2, pcs=pcs, cls=b"prtr")


# ---------------------------------------------------------------- independent ICC parser
def parse_icc(data):
    """-> ('rgb', [trc fn x3], C) or ('gray', trc fn); raises ValueError on what the product refuses"""
    be32 = lambda o: struct.unpack_from(">I", data, o)[0]
    size = be32(0)
    space, pcs = data[16:20], data[20:24]
    tags = {}
    for i in range(be32(128)):
        s, o, n = struct.unpack_from(">4sII", data, 132 + 12 * i)
        tags.setdefault(s, data[o:o + n])

    def trc(t):
        if t[:4] == b"curv":
            n = struct.unpack_from(">I", t, 8)[0]
            return curv(struct.unpack_from(f">{n}H", t, 12))
        f = struct.unpack_from(">H", t, 8)[0]
        k = (1, 3, 4, 5, 7)[f]
        return para(f, [v / 65536.0 for v in struct.unpack_from(f">{k}i", t, 12)])
    assert size <= len(data)
    if space == b"GRAY":
        return "gray", trc(tags[b"kTRC"])
    c = np.array([[v / 65536.0 for v in struct.unpack_from(">3i", tags[s], 8)] for s in (b"rXYZ", b"gXYZ", b"bXYZ")]).T
    return "rgb", [trc(tags[s]) for s in (b"rTRC", b"gTRC", b"bTRC")], c


def restate(profile):
    """(trcs, M) in float64 of an imageflow_b200.SourceProfile of kind ICC, GAMMA_PRIMARIES or CICP; ('gray', trc) for ICC_GRAY"""
    from imageflow_b200 import SourceProfile as SP
    if profile.kind in (SP.ICC, SP.ICC_GRAY):
        r = parse_icc(profile.icc_bytes)
        if r[0] == "gray":
            return "gray", r[1]
        return r[1], matrix_of(r[2])
    if profile.kind == SP.GAMMA_PRIMARIES:
        e = float(np.float32(1.0 / profile.gamma))
        t = lambda x: _pw(x, e)
        return [t] * 3, matrix_of(colorants_d50(profile.chrm))
    cp, tc = profile.cicp_codes[:2]
    t = cicp_transfer(tc)
    return [t] * 3, matrix_of(colorants_d50(CICP_PRIMARIES[cp]))


def clip01(x):
    x = np.asarray(x, np.float64)
    return np.where(x > 0, np.minimum(x, 1.0), 0.0)


def tables_f64(trcs):
    v = np.arange(256) / 255.0
    return np.stack([clip01(t(v)) for t in trcs])


def srgb_encode_f64(lin):
    lin = clip01(lin)
    return np.where(lin <= 0.0031308, 12.92 * lin, 1.055 * np.power(lin, 1 / 2.4) - 0.055)


def exact_bgr(trcs, m, b, g, r):
    """float64 restatement of B, G, R bytes (uint8 arrays) -> output B, G, R bytes (int arrays): exact curves, matrix and encode"""
    t = tables_f64(trcs)
    lin = np.stack([t[0][r], t[1][g], t[2][b]])                          # R, G, B
    o = np.tensordot(m, lin, axes=(1, 0))
    enc = np.rint(255.0 * srgb_encode_f64(o)).astype(np.int64)
    return enc[2], enc[1], enc[0]


def exact_gray(trc, v):
    return np.rint(255.0 * srgb_encode_f64(clip01(trc(np.asarray(v) / 255.0)))).astype(np.int64)


# ---------------------------------------------------------------- the fp32 oracle, in the kernel's order
def encode_f32(lut16k, o):
    s = np.float32(o) * np.float32(16383.0) if np.isscalar(o) else o.astype(np.float32) * np.float32(16383.0)
    s = np.where(np.isnan(s), np.float32(0), s)
    s = np.clip(s, np.float32(0), np.float32(16383.0))
    return lut16k[s.astype(np.int32)]


def apply_plan(plan, lut16k, bgra):
    """(..., 4) uint8 BGRA -> (..., 4) uint8: plan (imageflow_b200.ProfilePlanResult) applied as transform_to_srgb_kernel does"""
    bgra = np.asarray(bgra, np.uint8)
    out = bgra.copy()
    if plan.kind == 0:
        return out
    if plan.kind == 2:
        v = plan.gray[bgra[..., 0]]
        out[..., 0] = out[..., 1] = out[..., 2] = v
        return out
    t = plan.trc.astype(np.float32)
    m = plan.m.astype(np.float32)
    R, G, B = t[0][bgra[..., 2]], t[1][bgra[..., 1]], t[2][bgra[..., 0]]
    for c, pos in ((0, 2), (1, 1), (2, 0)):
        o = (m[c, 0] * R + m[c, 1] * G) + m[c, 2] * B                  # f32 products and sums, left to right
        out[..., pos] = encode_f32(lut16k, o)
    return out


def all_triples():
    """a 4096 x 4096 x 3 uint8 frame (B, G, R) holding every RGB triple once"""
    i = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(i & 255).astype(np.uint8), ((i >> 8) & 255).astype(np.uint8), (i >> 16).astype(np.uint8)], -1).reshape(4096, 4096, 3)
