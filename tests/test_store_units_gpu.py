"""The store epilogue's arithmetic as compiled for sm_90a, held to exact references on the GPU.

The three resample kernels compute the store epilogue (DESIGN.md section 3, step 4) with different instructions and claim the
same bits: the tile kernel divides with a shared reciprocal (t2_rcp_inrange + t2_div3), clamps with a round-toward-zero add
(uchar_clamp_ff_rz) and indexes the linear->sRGB table with a saturating conversion (encode_sm); the ring kernel indexes it
through __saturatef; the generic pair uses __fdiv_rn, uchar_clamp_ff and lut_encode.  An image test sees a one-ulp misrounding
only when the quotient sits next to a byte boundary, so these tests call the product's device functions themselves
(tests/gpu_units/units_probe.cu, built with the product's nvcc flags):
  * scalar units over their whole domain (every float pattern, or every guarded divisor), counted on the device against float64;
  * every compiled store epilogue on one adversarial input set, bit-exact against tests/watermark_oracle.composite followed by
    oracle.color_matrix."""
import time

import numpy as np
import pytest

import oracle
from tests import watermark_oracle as wo

pytestmark = pytest.mark.gpu

F32 = np.float32
N_GUARD = 1 << 29                 # divisors 2^-31 <= d < 2^33
N_EXCLUDED = 64                   # of which the significand is all ones (t2_div3 sends those to __fdiv_rn)


@pytest.fixture(scope="module", autouse=True)
def wall_time():
    t0 = time.perf_counter()
    yield
    print(f"\ntest_store_units_gpu: {time.perf_counter() - t0:.1f} s wall")


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope="module")
def units(torch_mod):
    from tests import gpu_units
    gpu_units.lib()                                   # fails (does not skip) when the probe library was not built
    return gpu_units


@pytest.fixture(scope="module")
def index_luts(torch_mod):
    """linear->sRGB tables that hold their own index: i & 255 and i >> 8"""
    i = np.arange(16384)
    return (torch_mod.from_numpy((i & 255).astype(np.uint8)).cuda(), torch_mod.from_numpy((i >> 8).astype(np.uint8)).cuda())


def _verdict(name, rep, expect_trials=None, assert_zero=True):
    trials, bad, ex = rep
    print(f"{name}: {trials} trials, {bad} mismatches")
    for a, b, got, want in ex:
        print(f"    a={a:#010x} b={b:#010x} got={got:#010x} expected={want:#010x}")
    if expect_trials is not None:
        assert trials == expect_trials, (name, trials, expect_trials)
    assert trials > 0, name
    if assert_zero:
        assert bad == 0, f"{name}: {bad} mismatches, first: {[tuple(hex(v) for v in e) for e in ex]}"


# ---------------------------------------------------------------------------------------------------------------- scalar units
def test_reciprocal_every_guarded_divisor(torch_mod, units):
    """t2_rcp_inrange(d) (rcp.approx.ftz + one Newton step) == RN(1/d) for all 2^29 divisors of the guard"""
    r = units.Reports(torch_mod, 2)
    units.check(units.lib().ifbu_rcp(r.ptr(0), r.ptr(1)), "ifbu_rcp")
    guarded, excluded = r.read()
    _verdict("t2_rcp_inrange, guarded divisors", guarded, N_GUARD - N_EXCLUDED)
    _verdict("t2_rcp_inrange, significand-all-ones divisors (excluded by the guard, not asserted)", excluded, N_EXCLUDED, assert_zero=False)


def _quotient_every_guarded_divisor(torch_mod, units, mode, name):
    """t2_div3 == RN(x / d) for every guarded divisor with three numerators each"""
    r = units.Reports(torch_mod, 1)
    units.check(units.lib().ifbu_div3(mode, r.ptr(), 0x5EED0 + mode, None, None), "ifbu_div3")
    rep = r.read()[0]
    _verdict(f"t2_div3, {name}", rep)
    assert rep[0] >= 0.999 * 3 * (N_GUARD - N_EXCLUDED), rep[0]          # all but the few numerators that round out of range


def test_quotient_near_midpoints_every_guarded_divisor(torch_mod, units):
    """numerators RN((q + ulp(q)/2) d) and their two neighbours, for a random quotient q per divisor"""
    _quotient_every_guarded_divisor(torch_mod, units, 0, "numerators next to a rounding midpoint")


def test_quotient_random_numerators_every_guarded_divisor(torch_mod, units):
    """three random numerators per divisor, 2^-100 <= |x| < 2^64, both signs"""
    _quotient_every_guarded_divisor(torch_mod, units, 1, "random numerators in [2^-100, 2^64)")


def test_quotient_tiny_numerators_encode_alike(torch_mod, units, index_luts):
    """|x| < 2^-100 (residual possibly inexact): the sRGB byte and the table index equal those of __fdiv_rn"""
    r = units.Reports(torch_mod, 1)
    lo, hi = index_luts
    units.check(units.lib().ifbu_div3(2, r.ptr(), 0x717, lo.data_ptr(), hi.data_ptr()), "ifbu_div3")
    _verdict("t2_div3, |x| < 2^-100, encoded bytes", r.read()[0], 3 * (N_GUARD - N_EXCLUDED))


def _neighbours(v, k):
    v = F32(v)
    out = [v]
    up = dn = v
    for _ in range(k):
        up = np.nextafter(up, F32(np.inf), dtype=F32); dn = np.nextafter(dn, F32(-np.inf), dtype=F32)
        out += [up, dn]
    return out


def _guarded(d) -> bool:
    """t2_div3's guard (ifb_tile2_kernel.cuh): 2^-31 <= d < 2^33, significand not all ones"""
    db = int(np.array([d], F32).view(np.uint32)[0])
    return (db - 0x30000000) & 0xFFFFFFFF < 0x20000000 and (db & 0x7FFFFF) != 0x7FFFFF


def test_quotient_edges_equal_library_division(torch_mod, units):
    """divisors on both sides of each guard edge, the significand-all-ones ones, d <= 0, -0, subnormals, inf and NaN: t2_div3
    equals __fdiv_rn (for NaN only NaN-ness is compared).  Divisors inside the guard get numerators of t2_div3's domain (+0 and
    2^-100 <= |x| < 2^64: what the store can divide); the others, which take __fdiv_rn, also get -0, huge, inf and NaN numerators."""
    u = lambda b: np.array([b], np.uint32).view(F32)[0]
    ds = []
    for edge in (2.0 ** -31, 2.0 ** 33):
        ds += _neighbours(edge, 3)
    ds += [u(0x3f7fffff), u(0x307fffff), u(0x4fffffff), u(0x3fffffff), u(0x3effffff)]          # significand all ones
    ds += [F32(0), F32(-0.0), u(1), u(0x007fffff), u(0x00400000), u(0x80000001), F32(-1), F32(-0.5), F32(-3e38),
           F32(np.inf), F32(-np.inf), F32(np.nan), u(0x7fc00001), u(0xffc00000), F32(1e-38), F32(1e-45), F32(3e38), F32(2.0 ** 40)]
    rng = np.random.default_rng(5)
    wide = rng.uniform(0.5, 1, 64) * 2.0 ** rng.integers(-99, 64, 64) * rng.choice([-1, 1], 64)
    xs_in = [F32(0), F32(1), F32(-1), F32(0.5), F32(1e-30), F32(2.0 ** -100), -F32(2.0 ** -100), np.nextafter(F32(2.0 ** 64), F32(0))]
    xs_in += list(rng.uniform(-2, 2, 64).astype(F32)) + list(wide.astype(F32))
    xs_any = xs_in + [F32(-0.0), F32(3e38), F32(-3e38), F32(np.inf), F32(-np.inf), F32(np.nan), u(1), u(0x807fffff)]
    r = units.Reports(torch_mod, 1)
    trials = 0
    for dl, xl in (([d for d in ds if _guarded(d)], xs_in), ([d for d in ds if not _guarded(d)], xs_any)):
        dt = torch_mod.from_numpy(np.array(dl, F32)).cuda()
        xt = torch_mod.from_numpy(np.array(xl, F32)).cuda()
        units.check(units.lib().ifbu_div3_edges(r.ptr(), dt.data_ptr(), len(dl), xt.data_ptr(), len(xl)), "ifbu_div3_edges")
        trials += 3 * len(dl) * len(xl)
    assert sum(_guarded(d) for d in ds) == 6                          # the edge neighbours inside the guard
    _verdict("t2_div3, edge divisors vs __fdiv_rn", r.read()[0], trials)


def test_clamps_every_float(torch_mod, units):
    """uchar_clamp_ff and uchar_clamp_ff_rz == trunc(x + 0.5) saturated to [0, 255], NaN -> 0, for all 2^32 float patterns"""
    r = units.Reports(torch_mod, 2)
    units.check(units.lib().ifbu_clamp(r.ptr(0), r.ptr(1)), "ifbu_clamp")
    ff, rz = r.read()
    _verdict("uchar_clamp_ff", ff, 1 << 32)
    _verdict("uchar_clamp_ff_rz", rz, 1 << 32)


def test_encoders_every_float(torch_mod, units, index_luts):
    """linear: the table index of lut_encode, the ring kernel's encode and encode_sm<true> == clamp(RN32(v * 16383), 0, 16383)
    truncated, NaN -> 0; sRGB: encode(false), the ring kernel's and encode_sm<false> == uchar_clamp_ff(RN32(255 v)); all 2^32 v"""
    r = units.Reports(torch_mod, 6)
    lo, hi = index_luts
    t_any = torch_mod.zeros(256, dtype=torch_mod.float32, device="cuda")
    units.check(units.lib().ifbu_encode(r.ptr(), lo.data_ptr(), hi.data_ptr(), t_any.data_ptr()), "ifbu_encode")
    names = ["lut_encode (index)", "ring kernel linear encode (index)", "encode_sm<true> (index)",
             "encode(false) = uchar_clamp_ff(255 v)", "ring kernel sRGB encode", "encode_sm<false>"]
    for name, rep in zip(names, r.read()):
        _verdict(name, rep, 1 << 32)


# ---------------------------------------------------------------------------------------------------------------- store epilogues
MATTES = [(40, 200, 90, 0), (40, 200, 90, 128), (40, 200, 90, 255)]     # BGRA; matte alpha 0, 128 and 255


def _matrices():
    sepia = oracle.color_filter_matrix(0).astype(F32)
    general = np.array([[0.9, 0.1, -0.05, 0.2, 0], [0.2, 0.7, 0.1, -0.1, 0], [-0.1, 0.05, 1.1, 0.3, 0],
                        [0.05, 0.1, 0.02, 0.8, 0], [0.03, -0.02, 0.05, 0.1, 1]], F32)
    neg0 = np.where(sepia == 0, F32(-0.0), sepia).astype(F32)
    assert np.signbit(neg0[3, 0]) and neg0[3, 0] == 0
    return {"none": None, "sepia": sepia, "general": general, "sepia-0": neg0}


def _alphas():
    u = lambda b: np.array([b], np.uint32).view(F32)[0]
    inv = F32(1.0 / 255.0)
    a = [F32(0), F32(-0.0), u(1), u(0x00400000), F32(1e-4), F32(253) * inv, F32(254) * inv, F32(1.3), F32(-0.25)]
    a += _neighbours(2.0 ** -31, 1) + _neighbours(0.994, 2) + _neighbours(1.0, 1)
    return np.array(a, F32)


def _targets():
    """quotients within +-2 ulps of every LUT index boundary k/16383 and every sRGB half-way point (k + 0.5)/255"""
    q = [np.float64(np.arange(1, 16384)) / 16383.0, (np.arange(255) + 0.5) / 255.0]
    q = np.concatenate(q).astype(F32)
    out = [q]
    up = dn = q
    for _ in range(2):
        up = np.nextafter(up, F32(np.inf), dtype=F32); dn = np.nextafter(dn, F32(-np.inf), dtype=F32)
        out += [up, dn]
    return np.concatenate(out)


def _input_set():
    """(F (n, 4) float32 premultiplied b, g, r, a; canvas (n, 4) uint8 BGRA)"""
    rng = np.random.default_rng(2024)
    A = _alphas()
    Q = _targets()
    n3 = -(-len(Q) // 3)
    Qp = np.resize(Q, n3 * 3).reshape(n3, 3)
    Fs, Cs = [], []
    # P: the quotient itself with alpha 1 (every path divides by 1 or does not divide)
    Fs.append(np.concatenate([Qp, np.ones((n3, 1), F32)], 1))
    Cs.append(rng.integers(0, 256, (n3, 4), dtype=np.uint8))
    # R: numerators RN(q * a), so that the un-premultiply c / a lands next to a boundary
    pos = A[A > 0]
    a = np.resize(pos, n3)
    Fs.append(np.concatenate([Qp * a[:, None], a[:, None]], 1).astype(F32))
    Cs.append(rng.integers(0, 256, (n3, 4), dtype=np.uint8))
    # B: BlendWithSelf over a canvas pixel with zero colour: numerators RN(q * fa), fa = the composite's divisor
    ab = np.resize(pos[pos <= F32(0.994)], n3)
    da = np.arange(n3) % 256
    with np.errstate(all="ignore"):
        dc = (F32(1) - ab) * ((F32(1.0 / 255.0) * da.astype(F32)) + F32(0))
        fa = (ab + dc).astype(F32)
    Fs.append(np.concatenate([Qp * fa[:, None], ab[:, None]], 1).astype(F32))
    cv = np.zeros((n3, 4), np.uint8)
    cv[:, 3] = da
    Cs.append(cv)
    # X: every alpha over every canvas alpha byte, with a few colours (zero, proportional, random and out of range)
    aa, dd = np.meshgrid(A, np.arange(256), indexing="ij")
    aa, dd = aa.ravel(), dd.ravel()
    for cols in (np.zeros((aa.size, 3), F32), aa[:, None] * np.array([0.5, 0.25, 1.0], F32),
                 aa[:, None] * rng.uniform(-0.2, 1.3, (aa.size, 3)).astype(F32)):
        Fs.append(np.concatenate([cols.astype(F32), aa[:, None]], 1).astype(F32))
        cv = rng.integers(0, 256, (aa.size, 4), dtype=np.uint8)
        cv[:, 3] = dd
        Cs.append(cv)
    return np.ascontiguousarray(np.concatenate(Fs), F32), np.ascontiguousarray(np.concatenate(Cs))


def _job(linear, am, compose, matte, m):
    """flags, matte[4] and cm[20] as the engine's make_job writes them (ifb_engine.cu)"""
    flags = (1 if linear else 0) | (2 if am else 0) | (compose << 2)
    mt = np.zeros(4, F32)
    if compose == wo.BLEND_WITH_MATTE and am:
        T = oracle.byte_to_float_table(linear)
        ma = F32(matte[3]) * F32(1.0 / 255.0)
        mt[:] = [T[matte[0]] * ma, T[matte[1]] * ma, T[matte[2]] * ma, ma]
    cm = np.zeros(20, F32)
    if m is not None:
        flags |= 16
        for c in range(4):
            for k in range(4):
                cm[c * 5 + k] = m[k, c]
            cm[c * 5 + 4] = F32(m[4, c]) * F32(255)
        rgb3 = all(cm[i] == 0 for i in (15, 16, 17, 19)) and cm[18] == 1 and all(cm[c * 5 + 3] == 0 and cm[c * 5 + 4] == 0 for c in range(3))
        if rgb3:
            flags |= 32
    return flags, mt, cm


def _variants():
    """(label, family, a, b, c, d, linear, am, compose, matte, matrix name) for every compiled store epilogue.
    family 0 finish_pixel<SIMPLE = a>; 1 hv_finish_pixel<EPI = a, CH = b>; 2 finish_pixel_sm<CH = b, LINEAR = c, COMPOSE = a, CM = d>"""
    mats = list(_matrices())
    out = []

    def cases(am):
        for compose in (0, 1, 2):
            for mi, matte in enumerate(MATTES if (compose == 2 and am) else MATTES[:1]):
                for mname in mats:
                    yield compose, matte, mname
    for linear in (False, True):
        for am in (False, True):
            ch = 4 if am else 3
            out.append((f"finish_pixel<true> lin={linear} am={am}", 0, 1, 0, 0, 0, linear, am, 0, MATTES[0], "none"))
            out.append((f"hv_finish_pixel<{2 - linear},{ch}>", 1, 2 - int(linear), ch, 0, 0, linear, am, 0, MATTES[0], "none"))
            for compose, matte, mname in cases(am):
                tag = f"lin={linear} am={am} compose={compose} matte={matte[3]} cm={mname}"
                out.append((f"finish_pixel<false> {tag}", 0, 0, 0, 0, 0, linear, am, compose, matte, mname))
                out.append((f"hv_finish_pixel<0,{ch}> {tag}", 1, 0, ch, 0, 0, linear, am, compose, matte, mname))
                if am or compose == 0:          # without alpha the engine runs the compose-0 instantiation for every mode
                    out.append((f"finish_pixel_sm<{ch},{int(linear)},{compose if am else 0},{int(mname != 'none')}> {tag}", 2,
                                compose if am else 0, ch, int(linear), int(mname != "none"), linear, am, compose, matte, mname))
    return out


def test_every_store_epilogue_on_adversarial_inputs(torch_mod, units):
    torch = torch_mod
    import imageflow_b200
    L = imageflow_b200.lib()
    import ctypes as C
    tabs = {}
    for lin in (0, 1):
        t = np.zeros(256, F32)
        L.ifb200_byte_to_float_table(lin, t.ctypes.data_as(C.POINTER(C.c_float)))
        tabs[lin] = torch.from_numpy(t).cuda()
    lut = np.zeros(16384, np.uint8)
    L.ifb200_linear_to_srgb_table(lut.ctypes.data_as(C.POINTER(C.c_uint8)))
    lut_d = torch.from_numpy(lut).cuda()

    F, canvas = _input_set()
    n = F.shape[0]
    print(f"store epilogues: {n} input pixels")
    Fd = torch.from_numpy(F).cuda()
    cv_words = torch.from_numpy(canvas.view(np.int32).reshape(n)).cuda()
    mats = _matrices()
    expected = {}
    failures = []
    variants = _variants()
    rgb3_seen = set()
    for label, fam, a, b, c, d, linear, am, compose, matte, mname in variants:
        m = mats[mname]
        key = (linear, am, compose, matte if (compose == 2 and am) else None, mname)
        if key not in expected:
            e = wo.composite(F[None], canvas[None], linear=linear, am=am, compose=compose, matte=matte)
            if m is not None:
                oracle.color_matrix(e, m)
            expected[key] = e[0]
        flags, mt, cm = _job(linear, am, compose, matte, m)
        if fam == 2 and d:
            rgb3_seen.add((mname, bool(flags & 32)))
        px = cv_words.clone()
        units.check(units.lib().ifbu_epilogue(fam, a, b, c, d, Fd.data_ptr(), px.data_ptr(), n, flags, mt.ctypes.data, cm.ctypes.data,
                                              tabs[1].data_ptr(), tabs[0].data_ptr(), lut_d.data_ptr()), label)
        got = px.cpu().numpy().view(np.uint8).reshape(n, 4)
        bad = np.nonzero((got != expected[key]).any(1))[0]
        if bad.size:
            i = bad[0]
            failures.append(f"{label}: {bad.size} pixels differ; first #{i}: F={F[i].tolist()} ({F[i].view(np.uint32).tolist()}) "
                            f"canvas={canvas[i].tolist()} got={got[i].tolist()} expected={expected[key][i].tolist()}")
    print(f"store epilogues: {len(variants)} (form, flags, matte, matrix) combinations x {n} pixels, {len(failures)} with mismatches")
    # the tile kernel's 3x3 form ran for sepia (also with -0.0 coefficients), the general form for the matrix with a bias
    assert {("sepia", True), ("sepia-0", True), ("general", False)} <= rgb3_seen, rgb3_seen
    assert not failures, "\n".join(failures[:20])
