"""The profiled resample on the GPU (Batch.scale_and_render_profiled -> ifb200_batch_enqueue_profiled), bit for bit against both the
two-step route on the device (Batch.transform_to_srgb into a BGRA scratch frame, then Batch.scale_and_render_oriented) and the oracle
(tests/profile_oracle.apply_plan, then tests/orient_oracle.gather, then oracle.scale_and_render): every EXIF flag -1..9 for BGRA,
RGBA32 and RGB24 sources under matrix, gray and CICP plans on the ring kernel's profiled forms and on the generic pair (the counters
confirm which ran); identity plans running exactly as the existing entries; one mixed call with one ring launch per (geometry, form,
plan); cut-out alpha and the general store epilogue; widths that are not a multiple of four with source x reversed; up-scales, 1:1
and 1x1; a refused profile and every rejected descriptor writing nothing; the struct layout; a 1024-job call; and back-to-back calls
on one Batch on two streams."""
import ctypes as C

import numpy as np
import pytest

import oracle
from imageflow_b200 import synth
from tests import orient_oracle
from tests import profile_oracle as pf
from tests.test_rows_resample_gpu import MATTE, _assert_same, _canvas, _device_rows, _ifb, _params, _rows_np, to_bgra

pytestmark = pytest.mark.gpu
FLAGS = list(range(-1, 10))


@pytest.fixture(scope="module")
def lut16k():
    from tests import cpu_emu
    return cpu_emu.transfer_tables(_ifb())[2]


def _profile(name):
    ifb = _ifb()
    if name == "cicp_9_1":
        return ifb.SourceProfile.cicp(9, 1)
    if name == "srgb":
        return ifb.SourceProfile.srgb()
    if name == "cicp_1_13":
        return ifb.SourceProfile.cicp(1, 13)
    kind, data = pf.fixtures()[name]
    return ifb.SourceProfile.icc(data) if kind == "icc" else ifb.SourceProfile.icc_gray(data)


def _source(img, fmt, pad=None, phase=0):
    """(device source as the entry takes it, its BGRA as to_bgra gives it, alpha_meaningful); img: (h, w, 4) RGBA rows"""
    import torch
    ifb = _ifb()
    if fmt == "bgra":
        bgra = to_bgra(img)
        h, w = bgra.shape[:2]
        pitch = (w * 4 + 63) // 64 * 64
        buf = torch.zeros((h, pitch), dtype=torch.uint8, device="cuda")
        buf[:, :w * 4] = torch.from_numpy(bgra.reshape(h, w * 4)).cuda()
        return ifb.BitmapWindow(buf.data_ptr(), w, h, pitch, alpha_meaningful=False, _keep=buf), bgra, False
    rows = np.ascontiguousarray(img[..., :3] if fmt == "rgb24" else img)
    c = rows.shape[2]
    if pad is None:
        pad = (16 - (phase + rows.shape[1] * c) % 16) % 16
    return _device_rows(rows, phase, pad), to_bgra(rows), c == 4


def _case(b, img, fmt, profile, ow, oh, flag, lut, *, filter=2, linear=True, compose=0, cm=None, sharpen=0.0, pad=None, phase=0,
          alpha=None, stream="own"):
    """(fused, two-step, oracle) results of one job and the (ring kernel, generic pair) job counts of the profiled call"""
    import torch
    ifb = _ifb()
    src, bgra, am = _source(img, fmt, pad, phase)
    if alpha is not None:
        am = alpha
    cv = synth.noise_np(ow + 3, oh + 2, seed=11, alpha_mode="mixed")
    p = _params(ow, oh, 1, 1, filter, linear, sharpen)
    fused = _canvas(cv, compose)
    f0, g0 = b.fused_jobs, b.generic_jobs
    b.scale_and_render_profiled([(src, fused, p, profile, flag, cm, am)], stream=stream)
    path = (b.fused_jobs - f0, b.generic_jobs - g0)
    h, w = bgra.shape[:2]
    scratch = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
    win = ifb.BitmapWindow.from_torch(scratch)
    b.transform_to_srgb([(src, win, profile)], stream=stream)
    win.alpha_meaningful = am
    two = _canvas(cv, compose)
    b.scale_and_render_oriented([(win, two, p, flag, cm)], stream=stream)
    b.sync()
    if stream != "own":
        torch.cuda.synchronize()
    srgb = pf.apply_plan(ifb.source_profile_plan(profile), lut, bgra)
    want = cv.copy()
    oracle.scale_and_render(np.ascontiguousarray(orient_oracle.gather(srgb, flag)), want, x=1, y=1, w=ow, h=oh, filter=filter,
                            alpha_meaningful=am, linear=linear, compose=compose, matte=MATTE, color_matrix=cm, sharpen=sharpen)
    return fused._keep.cpu().numpy(), two._keep.cpu().numpy(), want, path


def _check(b, img, fmt, profile, ow, oh, flag, lut, **kw):
    fused, two, want, path = _case(b, img, fmt, profile, ow, oh, flag, lut, **kw)
    _assert_same(fused, want, ("oracle", fmt, img.shape, ow, oh, flag, kw))
    _assert_same(fused, two, ("two-step", fmt, img.shape, ow, oh, flag, kw))
    return path


@pytest.mark.parametrize("force_generic", [0, 1])
@pytest.mark.parametrize("name", ["display_p3_v4", "adobe_rgb_v2", "gray22_v2", "cicp_9_1"])
@pytest.mark.parametrize("fmt", ["bgra", "rgba", "rgb24"])
def test_every_flag_on_the_ring_kernel_and_the_generic_pair(fmt, name, force_generic, lut16k):
    ifb = _ifb()
    b = ifb.Batch(0)
    b.set_option(ifb.Batch.OPT_FORCE_GENERIC, force_generic)
    img = _rows_np(480, 352, 4, seed=5)
    for flag in FLAGS:
        linear = flag % 2 == 0
        path = _check(b, img, fmt, _profile(name), 96, 80, flag, lut16k, linear=linear)
        assert path == ((0, 1) if force_generic else (1, 0)), (fmt, name, flag)


@pytest.mark.parametrize("name", ["srgb", "cicp_1_13"])
@pytest.mark.parametrize("fmt", ["bgra", "rgb24"])
def test_identity_plans_run_as_the_existing_entries(fmt, name):
    """same outputs and the same counters as scale_and_render_oriented / _rows_oriented without a profile"""
    ifb = _ifb()
    img = _rows_np(480, 352, 4, seed=6)
    outs = []
    for profiled in (True, False):
        b = ifb.Batch(0)
        src, _, am = _source(img, fmt)
        cv = np.zeros((82, 100, 4), np.uint8)
        jobs, canv = [], []
        for flag in (1, 6, 3):
            c = _canvas(cv, 0)
            canv.append(c)
            jobs.append((src, c, _params(96, 80, 1, 1, 2, True, 0.0), flag))
        if profiled:
            b.scale_and_render_profiled([(j[0], j[1], j[2], _profile(name), j[3], None, am) for j in jobs], stream="own")
        elif fmt == "bgra":
            b.scale_and_render_oriented(jobs, stream="own")
        else:
            b.scale_and_render_rows_oriented([(j[0], j[1], j[2], j[3], None, am) for j in jobs], stream="own")
        b.sync()
        outs.append(([c._keep.cpu().numpy() for c in canv], b.kernel_launches, b.fused_jobs, b.generic_jobs, b.tile_jobs))
        b.close()
    for g, w in zip(outs[0][0], outs[1][0]):
        _assert_same(g, w, (fmt, name))
    assert outs[0][1:] == outs[1][1:]


def test_one_mixed_call_is_one_ring_launch_per_geometry_form_and_plan(lut16k):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    img = _rows_np(480, 352, 4, seed=7)
    p3, adobe = _profile("display_p3_v4"), _profile("adobe_rgb_v2")
    jobs, expect = [], []
    specs = [("rgb24", p3, 6), ("rgb24", p3, 6), ("rgb24", adobe, 6), ("rgb24", p3, 1), ("bgra", p3, 1), ("rgba", adobe, 8),
             ("rgb24", _profile("srgb"), 6)]
    for fmt, prof, flag in specs:
        src, bgra, am = _source(img, fmt)
        c = _canvas(np.zeros((82, 100, 4), np.uint8), 0)
        jobs.append((src, c, _params(96, 80, 1, 1, 2, True, 0.0), prof, flag, None, am))
        srgb = pf.apply_plan(ifb.source_profile_plan(prof), lut16k, bgra)
        want = np.zeros((82, 100, 4), np.uint8)
        oracle.scale_and_render(np.ascontiguousarray(orient_oracle.gather(srgb, flag)), want, x=1, y=1, w=96, h=80, filter=2,
                                alpha_meaningful=am, linear=True)
        expect.append(want)
    n0, f0 = b.kernel_launches, b.fused_jobs
    b.scale_and_render_profiled(jobs, stream="own")
    b.sync()
    # (rgb24, p3, 6) x2, (rgb24, adobe, 6), (rgb24, p3, 1), (bgra, p3, 1), (rgba, adobe, 8), (rgb24, identity, 6): six launches
    assert b.kernel_launches - n0 == 6 and b.fused_jobs - f0 == len(specs)
    for j, want in zip(jobs, expect):
        _assert_same(j[1]._keep.cpu().numpy(), want, "mixed")
    del torch


@pytest.mark.parametrize("compose", [0, 1, 2])
def test_cutout_alpha_and_the_general_store_epilogue(compose, lut16k):
    """RGBA32 and BGRA with cut-out alpha (CH = 4), every compositing mode, a colour matrix and sharpen"""
    ifb = _ifb()
    b = ifb.Batch(0)
    img = _rows_np(480, 352, 4, seed=8, content="cutout")
    for fmt in ("rgba", "bgra"):
        for flag, cm, sharpen in ((1, None, 0.0), (6, ifb.color_filter_matrix(0), 0.0), (3, None, 40.0)):
            path = _check(b, img, fmt, _profile("display_p3_v4"), 96, 80, flag, lut16k, compose=compose, cm=cm, sharpen=sharpen, alpha=True)
            simple = compose == 0 and cm is None
            assert path == ((1, 0) if simple else (0, 1)), (fmt, compose, flag)


@pytest.mark.parametrize("fmt", ["bgra", "rgba", "rgb24"])
def test_widths_not_a_multiple_of_four_and_rgb24_phases(fmt, lut16k):
    ifb = _ifb()
    b = ifb.Batch(0)
    img = _rows_np(482, 351, 4, seed=9)
    for flag in (2, 3, 7, 8):
        _check(b, img, fmt, _profile("display_p3_v4"), 97, 81, flag, lut16k)
    if fmt == "rgb24":
        for phase in (1, 5, 14):
            assert _check(b, img, fmt, _profile("adobe_rgb_v2"), 97, 81, 6, lut16k, phase=phase) == (1, 0)


@pytest.mark.parametrize("fmt", ["bgra", "rgb24"])
def test_upscales_one_to_one_and_one_pixel(fmt, lut16k):
    ifb = _ifb()
    b = ifb.Batch(0)
    for (w, h), (ow, oh) in (((40, 30), (97, 71)), ((64, 48), (64, 48)), ((1, 1), (1, 1)), ((1, 1), (5, 3))):
        img = _rows_np(w, h, 4, seed=10)
        for flag in (1, 5, 8):
            oww, ohh = (oh, ow) if flag >= 5 and (w, h) == (64, 48) else (ow, oh)
            assert _check(b, img, fmt, _profile("display_p3_v4"), oww, ohh, flag, lut16k)[1] == 1


def test_refused_profile_and_rejected_descriptors_write_nothing():
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    img = _rows_np(200, 100, 4, seed=12)
    src, _, am = _source(img, "rgb24")
    cv = torch.full((40, 40, 4), 7, dtype=torch.uint8, device="cuda")
    canvas = ifb.BitmapWindow.from_torch(cv)
    p = _params(32, 32, 0, 0, 2, True, 0.0)
    good = (src, canvas, p, _profile("display_p3_v4"), 6)
    with pytest.raises(ifb.FlowError, match="profiled resample job 1: .*CMYK") as e:
        b.scale_and_render_profiled([good, (src, canvas, p, ifb.SourceProfile.icc(pf.lut_profile()), 6)], stream="own")
    assert e.value.kind == ifb.ErrorKind.MethodNotImplemented
    gray_rows = torch.zeros((100, 200, 1), dtype=torch.uint8, device="cuda")
    with pytest.raises(ifb.FlowError, match="profiled resample job 1: format 2"):
        b.scale_and_render_profiled([good, (gray_rows, canvas, p, _profile("display_p3_v4"), 1)], stream="own")
    with pytest.raises(ifb.FlowError, match="profiled resample job 0: not a SourceProfile"):
        b.scale_and_render_profiled([(src, canvas, p, None, 1)], stream="own")
    d, keep = b.make_profiled_descs([good, good])
    d[1].profile = None
    buf = C.create_string_buffer(512)
    assert ifb.lib().ifb200_batch_enqueue_profiled(b._h, d, 2, ifb.Batch.STREAM_OWN, buf, 512) != 0
    assert b"profiled resample job 1: null profile pointer" in buf.value
    d[1].profile = d[0].profile
    d[1].format = 7
    assert ifb.lib().ifb200_batch_enqueue_profiled(b._h, d, 2, ifb.Batch.STREAM_OWN, buf, 512) != 0
    assert b"profiled resample job 1: format 7" in buf.value
    d[1].format = 16
    d[1].draw.in_stride = 4
    assert ifb.lib().ifb200_batch_enqueue_profiled(b._h, d, 2, ifb.Batch.STREAM_OWN, buf, 512) != 0
    assert b"profiled resample job 1:" in buf.value
    b.sync()
    assert bool((cv == 7).all())


def test_struct_layout():
    ifb = _ifb()
    from imageflow_b200._lib import ProfiledResampleDesc, ResampleDesc
    assert ProfiledResampleDesc.format.offset == C.sizeof(ResampleDesc)
    assert ProfiledResampleDesc.orientation.offset == C.sizeof(ResampleDesc) + 4
    assert ProfiledResampleDesc.profile.offset == C.sizeof(ResampleDesc) + 8
    assert C.sizeof(ProfiledResampleDesc) == C.sizeof(ResampleDesc) + 16
    assert ifb.lib().ifb200_batch_enqueue_profiled


def test_1024_jobs_in_one_call(lut16k):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    img = _rows_np(256, 192, 3, seed=13)
    src = _device_rows(img, 0, (16 - 256 * 3 % 16) % 16)
    prof = _profile("display_p3_v4")
    out = torch.zeros((1024, 48, 64, 4), dtype=torch.uint8, device="cuda")
    p = _params(64, 48, 0, 0, 2, True, 0.0)
    jobs = [(src, ifb.BitmapWindow.from_torch(out[i]), p, prof, 1 + i % 8) for i in range(1024)]
    n0 = b.kernel_launches
    b.scale_and_render_profiled(jobs, stream="own")
    b.sync()
    # three (geometry, form, plan) groups: flag 1, the flips 2..4 and the transposes 5..8
    assert b.fused_jobs == 1024 and b.kernel_launches - n0 == 3
    srgb = pf.apply_plan(ifb.source_profile_plan(prof), lut16k, to_bgra(img))
    got = out.cpu().numpy()
    for flag in range(1, 9):
        ow, oh = 64, 48
        want = np.zeros((48, 64, 4), np.uint8)
        oracle.scale_and_render(np.ascontiguousarray(orient_oracle.gather(srgb, flag)), want, w=ow, h=oh, filter=2, linear=True)
        for i in range(flag - 1, 1024, 8):
            _assert_same(got[i], want, ("1024", i, flag))


def test_back_to_back_calls_on_two_streams(lut16k):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    img = _rows_np(480, 352, 4, seed=14)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    for k in range(3):
        for s, flag in ((s1, 6), (s2, 3)):
            fused, two, want, path = _case(b, img, "rgb24", _profile("display_p3_v4" if k % 2 else "adobe_rgb_v2"), 96, 80, flag, lut16k,
                                           stream=s.cuda_stream)
            _assert_same(fused, want, ("streams", k, flag))
            _assert_same(fused, two, ("streams", k, flag))
            assert path == (1, 0)
