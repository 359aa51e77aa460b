"""The store epilogue's alpha edges on the GPU: cut-out content (synth.cutout_*) through every resample path, bit-exact against the
oracle and inside the float64 ranges of tests/resample_f64.py.

Noise content averages alpha to mid-grey on a down-scale, so it never reaches the branches that transparent PNGs take on every
pixel: a == 0 (no un-premultiply), a < 0 and a > 1 (clamped A), tiny a (division by it), a next to BlendWithSelf's 0.994, and
fa == 0 / fa < 0 over an alpha-0 canvas pixel (tests/test_alpha_edges_oracle.py checks that this content reaches all of them).
Also: input windows that start inside a larger bitmap (any pixel of a 16-byte group, padded and unpadded pitches) written into a
canvas sub-rect, with the kernel that ran checked against the engine's rule (the ring kernel needs 16-byte aligned TMA boxes)."""
import numpy as np
import pytest

import oracle
from imageflow_b200 import synth
from tests import resample_f64, util
from tests.test_alpha_edges_oracle import MATTE, check_inside_ranges

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ifb():
    import imageflow_b200
    assert imageflow_b200.device_count() > 0, "CUDA extension loaded but no device: GPU tests cannot fall back"
    return imageflow_b200


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    assert torch.cuda.is_available()
    return torch


def _up(torch, a, pitch=None):
    """device copy of an (h, w, 4) array in rows of `pitch` bytes (default: padded to 64 like Bitmap::create_u8)"""
    hh, ww, _ = a.shape
    pitch = (ww * 4 + 63) // 64 * 64 if pitch is None else pitch
    t = torch.zeros((hh, pitch), dtype=torch.uint8, device="cuda")
    v = t.as_strided((hh, ww, 4), (pitch, 4, 1))
    v.copy_(torch.from_numpy(np.ascontiguousarray(a)))
    return v


def _params(ifb, ow, oh, *, x=0, y=0, filter=2, linear=True, sharpen=0.0):
    return ifb.ScaleAndRenderParams(x=x, y=y, w=ow, h=oh, sharpen_percent_goal=sharpen, interpolation_filter=ifb.Filter(filter),
                                    scale_in_colorspace=ifb.WorkingFloatspace(int(linear)))


def _run(ifb, torch, jobs, force_generic=False):
    """jobs: (input window tensor, canvas tensor, alpha, compose, params, colour matrix) -> counters"""
    b = ifb.Batch(0)
    assert b.ring_status()[0], b.ring_status()[1]
    b.set_option(ifb.Batch.OPT_FORCE_GENERIC, int(force_generic))
    b.scale_and_render_many([(ifb.BitmapWindow.from_torch(ti, alpha_meaningful=alpha),
                              ifb.BitmapWindow.from_torch(tc, compose=ifb.BitmapCompositing(compose), matte_bgra=MATTE), p, cm)
                             for (ti, tc, alpha, compose, p, cm) in jobs], stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    cnt = dict(fused=b.fused_jobs, tile=b.tile_jobs, generic=b.generic_jobs)
    b.close()
    return cnt


# (in_w, in_h, out_w, out_h, filter, the kernel the engine picks)
PATH_CASES = [
    (640, 480, 200, 150, 2, "fused"),          # Robidoux 3.2x: ring depth 4
    (960, 540, 128, 128, 6, "fused"),          # Lanczos3 at config-2 ratios: ring depth 6
    (512, 384, 128, 96, 2, "fused"),
    (100, 60, 333, 200, 14, "tile"),           # Mitchell 3.3x up-scale
    (300, 200, 300, 200, 2, "tile"),           # 1:1
]


@pytest.mark.parametrize("case", PATH_CASES, ids=lambda c: "x".join(map(str, c[:5])))
def test_cutout_every_path_and_epilogue(ifb, torch_mod, case):
    """both channel counts x three compositing modes x linear / sRGB space x with / without a colour matrix, through the
    kernel the engine picks and through the generic pair: bit-exact against the oracle, and inside the f64 ranges"""
    torch = torch_mod
    iw, ih, ow, oh, flt, kind = case
    sepia = ifb.color_filter_matrix(0)
    inp = synth.cutout_np(iw, ih, seed=iw + oh)
    canvas = synth.cutout_canvas_np(ow + 5, oh + 3, seed=4)
    ti = _up(torch, inp)
    for alpha in (False, True):
        for compose in (0, 1, 2):
            for linear in (True, False):
                for cm in (None, sepia):
                    kw = dict(x=2, y=1, w=ow, h=oh, filter=flt, linear=linear, alpha_meaningful=alpha, compose=compose, matte=MATTE, color_matrix=cm)
                    exp = canvas.copy()
                    oracle.scale_and_render(inp, exp, **kw)
                    lo, hi = resample_f64.byte_ranges(inp, canvas, **kw)
                    what = (alpha, compose, linear, cm is not None)
                    for force in (False, True):
                        tc = _up(torch, canvas)
                        cnt = _run(ifb, torch, [(ti, tc, alpha, compose, _params(ifb, ow, oh, x=2, y=1, filter=flt, linear=linear), cm)], force)
                        assert cnt[("generic" if force else kind)] == 1, (what, force, cnt)
                        got = tc.cpu().numpy()
                        assert np.array_equal(got, exp), (what, force, util.diff_stats(got, exp))
                        check_inside_ranges(got[1:1 + oh, 2:2 + ow], lo, hi)


@pytest.mark.parametrize("flt", [2, 6], ids=["robidoux", "lanczos3"])
def test_config2_cutout_frames(ifb, torch_mod, flt):
    """3840x2160 -> 512x512 with meaningful alpha: the first frame against the oracle, a batch of 8 against the generic pair"""
    torch = torch_mod
    n = 8
    ins = [synth.cutout_torch(3840, 2160, seed=700 + i) for i in range(n)]
    p = _params(ifb, 512, 512, filter=flt)
    outs = {}
    for force in (False, True):
        cvs = [torch.zeros((512, 512, 4), dtype=torch.uint8, device="cuda") for _ in range(n)]
        cnt = _run(ifb, torch, [(ins[i], cvs[i], True, 0, p, None) for i in range(n)], force)
        assert cnt["generic" if force else "fused"] == n, cnt
        outs[force] = cvs
    for i in range(n):
        assert torch.equal(outs[False][i], outs[True][i]), i
    exp = np.zeros((512, 512, 4), np.uint8)
    oracle.scale_and_render(ins[0].cpu().numpy(), exp, filter=flt, alpha_meaningful=True)
    got = outs[False][0].cpu().numpy()
    assert np.array_equal(got, exp), util.diff_stats(got, exp)
    assert (got[..., 3] == 0).any() and (got[..., 3] == 255).any()            # transparent and opaque output pixels both occur


def test_one_call_mixes_cutout_and_noise_jobs(ifb, torch_mod):
    torch = torch_mod
    sepia = ifb.color_filter_matrix(0)
    spec = [  # (content, in_w, in_h, out_w, out_h, filter, alpha, compose, linear, matrix)
        ("cutout", 640, 480, 200, 150, 2, True, 1, True, None), ("noise", 640, 480, 200, 150, 2, True, 1, True, None),
        ("cutout", 960, 540, 128, 128, 6, True, 0, True, None), ("noise", 960, 540, 128, 128, 6, False, 0, True, None),
        ("cutout", 100, 60, 333, 200, 14, True, 2, False, sepia), ("noise", 512, 384, 128, 96, 14, True, 2, True, None),
        ("cutout", 512, 384, 128, 96, 2, True, 1, False, sepia), ("cutout", 300, 200, 300, 200, 2, True, 1, True, None),
    ]
    jobs, checks = [], []
    for i, (content, iw, ih, ow, oh, flt, alpha, compose, linear, cm) in enumerate(spec):
        inp = synth.cutout_np(iw, ih, seed=i) if content == "cutout" else util.noise(iw, ih, seed=i, alpha_mode="mixed")
        canvas = synth.cutout_canvas_np(ow, oh, seed=10 + i)
        exp = canvas.copy()
        oracle.scale_and_render(inp, exp, filter=flt, linear=linear, alpha_meaningful=alpha, compose=compose, matte=MATTE, color_matrix=cm)
        tc = _up(torch, canvas)
        jobs.append((_up(torch, inp), tc, alpha, compose, _params(ifb, ow, oh, filter=flt, linear=linear), cm))
        checks.append((tc, exp))
    cnt = _run(ifb, torch, jobs)
    assert cnt["fused"] == 6 and cnt["tile"] == 2 and cnt["generic"] == 0, cnt
    for i, (tc, exp) in enumerate(checks):
        got = tc.cpu().numpy()
        assert np.array_equal(got, exp), (i, spec[i], util.diff_stats(got, exp))


@pytest.mark.parametrize("pitch_kind", ["pad64", "odd"])
@pytest.mark.parametrize("x0", [0, 1, 2, 3])
def test_cropped_input_window(ifb, torch_mod, x0, pitch_kind):
    """a 640x480 cut-out window at (x0 + 64, 5) of an opaque noise bitmap -> a sub-rect of a larger canvas.  The ring kernel
    runs only for a 16-byte aligned window origin and pitch; every byte outside the rect (row padding included) is unchanged."""
    torch = torch_mod
    iw, ih, ow, oh = 640, 480, 200, 150
    X0, Y0 = 64 + x0, 5
    bw, bh = 720, 490
    pitch = (bw * 4 + 63) // 64 * 64 if pitch_kind == "pad64" else bw * 4 + 4       # 2880 + 4: a multiple of 4, not of 16
    big = np.zeros((bh, pitch), np.uint8)
    bigv = np.lib.stride_tricks.as_strided(big, shape=(bh, bw, 4), strides=(pitch, 4, 1))
    bigv[...] = util.noise(bw, bh, seed=31, alpha_mode="opaque")
    win = synth.cutout_np(iw, ih, seed=x0)
    bigv[Y0:Y0 + ih, X0:X0 + iw] = win
    cw, chh, cx, cy = 230, 170, 13, 7
    cpitch = (cw * 4 + 63) // 64 * 64
    canvas = synth.cutout_canvas_np(cw, chh, seed=x0)
    tb = torch.from_numpy(big).cuda()
    ti = tb.as_strided((ih, iw, 4), (pitch, 4, 1), storage_offset=Y0 * pitch + X0 * 4)
    aligned = ti.data_ptr() % 16 == 0 and pitch % 16 == 0
    assert aligned == (x0 == 0 and pitch_kind == "pad64")
    sepia = ifb.color_filter_matrix(0)
    for compose, cm in ((0, None), (1, None), (2, sepia)):
        kw = dict(x=cx, y=cy, w=ow, h=oh, filter=2, alpha_meaningful=True, compose=compose, matte=MATTE, color_matrix=cm)
        exp = canvas.copy()
        oracle.scale_and_render(np.ascontiguousarray(win), exp, **kw)
        tcb = torch.full((chh, cpitch), 0xA5, dtype=torch.uint8, device="cuda")
        tc = tcb.as_strided((chh, cw, 4), (cpitch, 4, 1))
        tc.copy_(torch.from_numpy(canvas))
        before = tcb.cpu().numpy().copy()
        cnt = _run(ifb, torch, [(ti, tc, True, compose, _params(ifb, ow, oh, x=cx, y=cy), cm)])
        assert cnt["fused"] == int(aligned) and sum(cnt.values()) == 1, (x0, pitch_kind, cnt)
        after = tcb.cpu().numpy()
        got = np.lib.stride_tricks.as_strided(after, shape=(chh, cw, 4), strides=(cpitch, 4, 1))
        assert np.array_equal(got, exp), (x0, pitch_kind, compose, util.diff_stats(got, exp))
        outside = np.ones((chh, cpitch), bool)
        outside[cy:cy + oh, cx * 4:(cx + ow) * 4] = False
        assert np.array_equal(after[outside], before[outside]), (x0, pitch_kind, compose)
    assert np.array_equal(tb.cpu().numpy(), big)                                    # the input is only read
