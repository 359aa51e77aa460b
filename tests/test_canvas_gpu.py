"""Canvas operations on the GPU (canvas_kernel through Batch.canvas), bit for bit against the numpy oracle (tests/canvas_oracle.py):
mixed batches of all four ops on device windows with sentinel bytes around them, one launch per call and none for a call with
nothing to write, rejected calls that change nothing, 4K and 8K ExpandCanvas, the reference's canvas graphs, and mode=pad after a
device-resident resample by two routes."""
import numpy as np
import pytest

import oracle
from tests import canvas_oracle as co
from tests.cpu_emu import run_canvas_cases as rcc

pytestmark = pytest.mark.gpu


def _ifb():
    import imageflow_b200 as ifb
    return ifb


def _dev_win(t, host_buf, ptr, w, h, stride, am):
    """the device window of `t` (a device copy of host_buf) at the place the host window `ptr` has in host_buf"""
    return _ifb().BitmapWindow(t.data_ptr() + (ptr - host_buf.ctypes.data), w, h, stride, bool(am), _keep=t)


def _ops_of(jobs, dev):
    """Batch.canvas ops for the emulation's job dicts, on device copies `dev` (id(bitmap) -> tensor) of their bitmaps"""
    ifb = _ifb()
    ops = []
    for d, _, bms, _ in jobs:
        cv = bms[0]
        win = _dev_win(dev[id(cv)], cv.buf, d["px"], d["w"], d["h"], d["stride"], d["alpha_meaningful"])
        if d["op"] == rcc.FILL:
            ops.append(ifb.FillRect(win, d["x1"], d["y1"], d["x2"], d["y2"], tuple(d["color_bgra"])))
        elif d["op"] == rcc.NORMALIZE:
            if not d["alpha_meaningful"]:
                ops.append(ifb.EnableTransparency(win))
        else:
            src = bms[1]
            inp = _dev_win(dev[id(src)], src.buf, d["in_"], d["in_w"], d["in_h"], d["in_stride"], d["in_alpha_meaningful"])
            if d["op"] == rcc.COPY:
                ops.append(ifb.CopyRectToCanvas(inp, win, d["x1"], d["y1"], d["cw"], d["ch"], d["x2"], d["y2"]))
            else:
                ops.append(ifb.ExpandCanvas(inp, d["x1"], d["y1"], d["x2"], d["y2"], tuple(d["color_bgra"]), canvas=win))
    return ops


def _upload(jobs):
    import torch
    return {id(b): torch.from_numpy(b.buf.copy()).cuda() for _, _, bms, _ in jobs for b in bms}


def test_mixed_batches_match_the_oracle_in_one_launch():
    import torch
    ifb = _ifb()
    assert ifb.device_count() > 0 and torch.cuda.is_available()
    b = ifb.Batch(0)
    rng = np.random.default_rng(21)
    for n in (1, 7, 64):
        for rep in range(4):
            jobs = [rcc.make_job(rng, big=(i % 5 == 0)) for i in range(n)]
            for _, oracle_fn, _, _ in jobs:
                oracle_fn()
            dev = _upload(jobs)
            ops = _ops_of(jobs, dev)
            writes = any(bm.mask.any() for _, _, bms, _ in jobs for bm in bms)
            before = b.kernel_launches
            b.canvas(ops, stream="own")
            b.sync()
            assert b.kernel_launches == before + (1 if writes else 0), (n, rep)
            for _, _, bms, _ in jobs:
                for bm in bms:
                    got = dev[id(bm)].cpu().numpy()
                    assert np.array_equal(got, bm.exp), (n, rep, np.nonzero(got != bm.exp)[0][:4].tolist())


def test_call_with_nothing_to_write_launches_nothing():
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    t = torch.full((8, 8, 4), 7, dtype=torch.uint8, device="cuda")
    win = ifb.BitmapWindow.from_torch(t, alpha_meaningful=True)
    before = b.kernel_launches
    out = b.canvas([ifb.FillRect(win, 3, 2, 3, 9, (1, 2, 3, 4)), ifb.FillRect(win, 50, 60, 70, 60, (1, 2, 3, 4))], stream="own")   # zero-size, even out of bounds
    b.canvas([], stream="own")
    lib = ifb.lib()
    from imageflow_b200._lib import CanvasDesc
    d = (CanvasDesc * 1)()
    d[0].op = 3; d[0].px = win.ptr; d[0].w = 8; d[0].h = 8; d[0].stride = 32; d[0].alpha_meaningful = 1   # NORMALIZE on Bgra32
    import ctypes as C
    buf = C.create_string_buffer(256)
    assert lib.ifb200_batch_canvas(b._h, d, 1, b._stream("own"), buf, 256) == 0
    b.sync()
    assert b.kernel_launches == before and out[0] is win
    assert (t.cpu().numpy() == 7).all()


def test_a_bad_descriptor_changes_nothing_and_launches_nothing():
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    rng = np.random.default_rng(22)
    jobs = [rcc.make_job(rng) for _ in range(7)]
    dev = _upload(jobs)
    ops = _ops_of(jobs, dev)
    win = ifb.BitmapWindow.from_torch(torch.zeros((4, 4, 4), dtype=torch.uint8, device="cuda"))
    for bad in (ifb.FillRect(win, 1, 1, 5, 2, (1, 2, 3, 4)), ifb.CopyRectToCanvas(win, win, 0, 0, 2, 2, 1, 1),
                ifb.ExpandCanvas(win, 1, 1, 1, 1, (0, 0, 0, 255), canvas=win)):
        before = b.kernel_launches
        with pytest.raises(ifb.FlowError) as e:
            b.canvas(ops[:3] + [bad] + ops[3:], stream="own")
        b.sync()
        assert e.value.kind == ifb.ErrorKind.InvalidArgument
        assert b.kernel_launches == before
        for _, _, bms, _ in jobs:
            for bm in bms:
                assert np.array_equal(dev[id(bm)].cpu().numpy(), bm.buf)


@pytest.mark.parametrize("w,h,in_am,color", [(3840, 2160, False, (10, 20, 30, 255)), (3840, 2160, False, (10, 20, 30, 128)),
                                             (7680, 4320, True, (0, 0, 0, 0)), (7680, 4320, False, (200, 100, 50, 255))])
def test_expand_4k_and_8k(w, h, in_am, color):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    rng = np.random.default_rng(w + color[3])
    host = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    l, t, r, bt = 37, 5, 64, 363
    exp_in = host.copy()
    exp = np.empty((h + t + bt, w + l + r, 4), np.uint8)
    cv = co.Win.of(exp)
    co.expand_canvas(co.Win.of(exp_in, in_am), cv, l, t, r, bt, color)
    dev = torch.from_numpy(host).cuda()
    out = b.canvas([ifb.ExpandCanvas(ifb.BitmapWindow.from_torch(dev, alpha_meaningful=in_am), l, t, r, bt, color)], stream="own")[0]
    b.sync()
    assert out.w == w + l + r and out.h == h + t + bt and out.stride % 64 == 0 and out.alpha_meaningful == cv.alpha_meaningful
    assert out.compose == ifb.BitmapCompositing.BlendWithSelf
    assert np.array_equal(out._keep.cpu().numpy(), exp)
    assert np.array_equal(dev.cpu().numpy(), exp_in)          # A = 255 written back to a Bgr32 input under a Bgra32 canvas


# canvas.rs graphs, steps without a resample, on the device (CreateCanvas = a FillRect of a new canvas)
def _create(b, w, h, color, am=True):
    ifb = _ifb()
    cv = ifb.new_canvas(w, h, 0, am)
    b.canvas([ifb.FillRect(cv, 0, 0, w, h, color)], stream="own")
    return cv


def _host(win):
    return win._keep.cpu().numpy()


def _oracle_create(w, h, color):
    a = np.empty((h, w, 4), np.uint8)
    co.create_canvas(co.Win.of(a), color)
    return a


def test_reference_canvas_graphs_on_the_device():
    ifb = _ifb()
    b = ifb.Batch(0)
    red, blue = co.hex_bgra("FF5555FF"), co.hex_bgra("0000FFFF")
    # test_fill_rect_original
    cv = _create(b, 400, 300, co.TRANSPARENT)
    b.canvas([ifb.FillRect(cv, 0, 0, 50, 100, blue)], stream="own"); b.sync()
    exp = _oracle_create(400, 300, co.TRANSPARENT); co.fill_rectangle(co.Win.of(exp), blue, 0, 0, 50, 100)
    assert np.array_equal(_host(cv), exp)
    # test_transparent_canvas
    cv = _create(b, 200, 200, co.hex_bgra("00000000")); b.sync()
    assert (_host(cv) == 0).all()
    # test_crop, test_off_surface_region, test_partial_region, test_pixels_region: on a red canvas with a blue strip
    base = _create(b, 200, 200, red)
    b.canvas([ifb.FillRect(base, 0, 0, 10, 100, blue)], stream="own")
    ref = _oracle_create(200, 200, red); co.fill_rectangle(co.Win.of(ref), blue, 0, 0, 10, 100)
    b.sync()
    assert np.array_equal(_host(base), ref)
    crop = base.window(0, 50, 100, 100)
    assert np.array_equal(_host(base)[50:100, :100], ref[50:100, :100]) and crop.w == 100 and crop.h == 50
    for name, op in [("off_surface", lambda: ifb.region_percent(base, -100, -100, -1, -1, co.TRANSPARENT)),
                     ("partial", lambda: ifb.region_percent(base, -10, -10, 40, 40, co.TRANSPARENT)),
                     ("pixels", lambda: ifb.region(base, -10, -10, 120, 50, co.TRANSPARENT))]:
        out = b.canvas([op()], stream="own")[0]
        b.sync()
        coords = {"off_surface": co.region_percent_coords(200, 200, -100, -100, -1, -1),
                  "partial": co.region_percent_coords(200, 200, -10, -10, 40, 40), "pixels": (-10, -10, 120, 50)}[name]
        want, am = co.run_region(ref.copy(), True, *coords, co.TRANSPARENT)
        got = _host(out)
        assert np.array_equal(got, want) and out.alpha_meaningful == am, name


def test_expand_rect_in_full_on_the_device():
    """canvas.rs test_expand_rect: CreateCanvas 200x200 transparent, FillRect EECCFFFF, ExpandCanvas 2233AAFF, then Hermite to
    400x400 in linear light"""
    ifb = _ifb()
    b = ifb.Batch(0)
    cv = _create(b, 200, 200, co.TRANSPARENT)
    b.canvas([ifb.FillRect(cv, 0, 0, 100, 100, co.hex_bgra("EECCFFFF"))], stream="own")
    ex = b.canvas([ifb.ExpandCanvas(cv, 10, 15, 20, 25, co.hex_bgra("2233AAFF"))], stream="own")[0]
    out = ifb.new_canvas(400, 400, 0, True)
    b.scale_and_render_many([(ex, out, ifb.ScaleAndRenderParams(w=400, h=400, interpolation_filter=ifb.Filter.Hermite))], stream="own")
    b.sync()
    a = _oracle_create(200, 200, co.TRANSPARENT)
    co.fill_rectangle(co.Win.of(a), co.hex_bgra("EECCFFFF"), 0, 0, 100, 100)
    e = np.empty((240, 230, 4), np.uint8)
    ew = co.Win.of(e)
    co.expand_canvas(co.Win.of(a, True), ew, 10, 15, 20, 25, co.hex_bgra("2233AAFF"))
    assert ex.alpha_meaningful and ew.alpha_meaningful
    assert np.array_equal(_host(ex), e)
    want = np.zeros((400, 400, 4), np.uint8)
    oracle.scale_and_render(e, want, filter=16, linear=True, alpha_meaningful=True)
    got = _host(out)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("compose", [0, 1, 2], ids=["ReplaceSelf", "BlendWithSelf", "BlendWithMatte"])
@pytest.mark.parametrize("am", [False, True], ids=["bgr32", "bgra32"])
def test_mode_pad_two_routes_agree_with_the_oracle(compose, am):
    """Config-2 frames (3840x2160 -> 512x288, Robidoux, linear light) padded to 512x512: (a) resample into a 512x288 canvas, then
    EXPAND; (b) resample straight into the interior of the 512x512 canvas, then FILL_RECT the border bands in one call.  Against the
    oracle's resample followed by the oracle's ExpandCanvas.  The pad colour is not opaque, so the padded canvas is Bgra32."""
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    inp = oracle.synth_noise(3840, 2160, seed=5 + compose, alpha_mode="mixed")
    matte = (40, 80, 120, 200)
    color = (9, 99, 199, 77)
    top = (512 - 288) // 2
    init = np.random.default_rng(3).integers(0, 256, (288, 512, 4), dtype=np.uint8)      # what BlendWithSelf blends over
    # the oracle chain
    mid = init.copy()
    oracle.scale_and_render(inp, mid, filter=2, linear=True, alpha_meaningful=am, compose=compose, matte=matte)
    mid_am = am                                                # Resample2D's canvas has its input's format (scale_render.rs:98)
    want = np.empty((512, 512, 4), np.uint8)
    co.expand_canvas(co.Win.of(mid.copy(), mid_am), co.Win.of(want), 0, top, 0, 512 - 288 - top, color)
    ti = torch.from_numpy(inp).cuda()
    src = ifb.BitmapWindow.from_torch(ti, alpha_meaningful=am)
    params = ifb.ScaleAndRenderParams(w=512, h=288)
    # (a)
    ca = torch.from_numpy(init).cuda()
    cwa = ifb.BitmapWindow.from_torch(ca, alpha_meaningful=mid_am, compose=ifb.BitmapCompositing(compose), matte_bgra=matte)
    b.scale_and_render_many([(src, cwa, params)], stream="own")
    pa = b.canvas([ifb.ExpandCanvas(cwa, 0, top, 0, 512 - 288 - top, color)], stream="own")[0]
    # (b)
    full = ifb.new_canvas(512, 512, 0, True)
    interior = full.window(0, top, 512, top + 288)
    interior.compose, interior.matte_bgra = ifb.BitmapCompositing(compose), matte
    full._keep[top:top + 288] = torch.from_numpy(init).cuda()
    b.scale_and_render_many([(src, interior, params)], stream="own")
    b.canvas([ifb.FillRect(full, 0, 0, 512, top, color), ifb.FillRect(full, 0, top + 288, 512, 512, color)], stream="own")
    b.sync()
    got_a, got_b = pa._keep.cpu().numpy(), full._keep.cpu().numpy()
    assert np.array_equal(got_a, want), ("route a", np.argwhere(np.any(got_a != want, axis=2))[:4].tolist())
    assert np.array_equal(got_b, want), ("route b", np.argwhere(np.any(got_b != want, axis=2))[:4].tolist())
