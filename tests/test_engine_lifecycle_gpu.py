"""A long-lived Batch against the oracles: the host state of ifb_engine.cu that lives across calls, exercised the way production
uses it -- many back-to-back calls of mixed operations while the GPU is still busy with earlier ones, several streams and threads
on one batch, and every cache and chunk bound of the engine crossed with real calls.

Every scenario stalls its stream first with a short bounded spin (torch.cuda._sleep), enqueues everything, and asserts that the
stream is still busy after the last enqueue, so every call was made while the GPU had not reached it.  Every call gets its own
seeded content and its own outputs; canvases start as a sentinel pattern, not zeros, so a job that never ran, or ran with another
call's work list, shows.  Each scenario also asserts, from the batch's counters and host profile, that it took the path and crossed
the bound it is about: the kernel that ran, the pinned staging slots and table uploads, more than 4096 plans, more than one chunk.

References: oracle.scale_and_render and the per-operation oracles under tests/, bit for bit; where the oracle is too slow for every
output (65 537 jobs, 8K frames) every output is compared with a fresh single-call Batch on the other kernel path, and the outputs on
both sides of each chunk seam with the oracle itself."""
import functools
import threading
import time

import numpy as np
import pytest

import oracle
from tests import canvas_oracle as cvo
from tests import color_oracle as co
from tests import orient_oracle as oo
from tests import pixel_convert_oracle as pco
from tests import round_corners_oracle as rco
from tests import watermark_oracle as wo

pytestmark = pytest.mark.gpu

MiB = 1 << 20


@pytest.fixture(scope="module")
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


@pytest.fixture(scope="module")
def ifb(torch):
    import imageflow_b200
    assert imageflow_b200.device_count() > 0, "CUDA extension loaded but no device: GPU tests cannot fall back"
    return imageflow_b200


@pytest.fixture(scope="module")
def cycles_per_ms(torch):
    """clock cycles of torch.cuda._sleep per millisecond on this device, measured once"""
    torch.cuda._sleep(1000)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    torch.cuda._sleep(20_000_000)
    e1.record()
    e1.synchronize()
    return 20_000_000 / e0.elapsed_time(e1)


class Stall:
    """Keeps a stream busy for `ms` milliseconds with a bounded spin that ends by itself (a busy-wait, not a hang)."""
    def __init__(self, torch, cpm):
        self.torch, self.cpm = torch, cpm

    def __call__(self, stream, ms=50):
        with self.torch.cuda.stream(stream):
            self.torch.cuda._sleep(int(ms * self.cpm))


@pytest.fixture(scope="module")
def stall(ifb, torch, cycles_per_ms):
    """The stall, after one un-stalled pass over every kernel the scenarios launch: the first launch of a kernel loads it, and that
    waits for the device, which would end the host's lead before it began."""
    b = ifb.Batch(0)
    _mixed_calls(ifb, torch, b, 50)
    src = dev(torch, noise(512, 512, 51))
    for am in (True, False):
        for ratio in (1.5, 2, 3, 4, 6, 7.5, 12):
            for generic in (0, 1):
                b.set_option(ifb.Batch.OPT_FORCE_GENERIC, generic)
                out = dev(torch, sentinel(int(512 / ratio), int(512 / ratio), 52))
                b.scale_and_render_many([(win(ifb, src, am), win(ifb, out), params(ifb, out.shape[1], out.shape[0]))])
    torch.cuda.synchronize()
    b.close()
    return Stall(torch, cycles_per_ms)


# ------------------------------------------------------------------------------------------------------------------ helpers
def sentinel(h, w, seed):
    """(h, w, 4) uint8 of seeded random bytes: what no job writes by accident, and different for every canvas"""
    return np.frombuffer(np.random.default_rng(seed + 77_000).bytes(h * w * 4), np.uint8).reshape(h, w, 4).copy()


def noise(w, h, seed, alpha=True):
    return oracle.synth_noise(w, h, seed=seed, alpha_mode="mixed" if alpha else "opaque")


_UPLOAD = []


def dev(torch, a):
    """a (h, w, c) uint8 numpy array -> an (h, w, c) view of a CUDA tensor whose rows are padded to 64 bytes (bitmaps.rs:803-804).
    The copy runs on a stream of its own that the current stream then waits for: a copy from pageable memory may block the host
    until its stream reaches it, and the current stream may be stalled."""
    if not _UPLOAD:
        _UPLOAD.append(torch.cuda.Stream())
    cur = torch.cuda.current_stream()
    h, w, c = a.shape
    pitch = (w * c + 63) // 64 * 64
    with torch.cuda.stream(_UPLOAD[0]):
        t = torch.empty((h, pitch), dtype=torch.uint8, device="cuda").as_strided((h, w, c), (pitch, c, 1))
        t.copy_(torch.from_numpy(np.ascontiguousarray(a)))
    cur.wait_stream(_UPLOAD[0])
    return t


def host(t):
    return t.cpu().numpy()


def win(ifb, t, am=False, **kw):
    return ifb.BitmapWindow.from_torch(t, alpha_meaningful=am, **kw)


def params(ifb, w, h, x=0, y=0, filter=2):
    return ifb.ScaleAndRenderParams(x=x, y=y, w=w, h=h, interpolation_filter=ifb.Filter(filter))


def expect_resample(src, canvas, **kw):
    out = np.ascontiguousarray(canvas).copy()
    oracle.scale_and_render(np.ascontiguousarray(src), out, **kw)
    return out


def counters(b):
    p = b.host_profile()
    return dict(fused=b.fused_jobs, tile=b.tile_jobs, generic=b.generic_jobs, launches=b.kernel_launches,
                pinned=p["pinned_allocs"], uploads=p["table_uploads"], staged=p["staged_bytes"])


def moved(b, before):
    now = counters(b)
    return {k: now[k] - before[k] for k in now}


def assert_equal(got, exp, what):
    if not np.array_equal(got, exp):
        bad = np.argwhere(np.any(np.asarray(got) != np.asarray(exp), axis=-1))
        raise AssertionError(f"{what}: {len(bad)} pixels differ, first at {bad[:3].tolist()}")


_RS = None


def resample_descs(ifb, n, **cols):
    """n ifb200_resample_desc filled a column at a time (tens of thousands of jobs without per-field ctypes marshalling)"""
    global _RS
    from imageflow_b200._lib import ResampleDesc
    if _RS is None:
        _RS = ifb.graphics._struct_dtype(ResampleDesc)
    a = np.zeros(n, _RS)
    a["linear"] = 1
    a["filter"] = 2
    for k, v in cols.items():
        a[k] = v
    return (ResampleDesc * n).from_buffer(a)


class Grid:
    """n jobs of one (in, out) geometry: job i reads the in_w x in_h window of a source bitmap at origins[i] and writes the
    out_w x out_h cell i of a canvas `per_row` cells wide"""
    def __init__(self, n, in_w, in_h, out_w, out_h, origins, per_row=256):
        self.n, self.in_w, self.in_h, self.out_w, self.out_h, self.per_row = n, in_w, in_h, out_w, out_h, per_row
        self.ox, self.oy = (np.asarray(v, np.int64) for v in origins)
        i = np.arange(n)
        self.cx, self.cy = (i % per_row) * out_w, (i // per_row) * out_h
        self.cv_w, self.cv_h = per_row * out_w, int(-(-n // per_row)) * out_h

    def descs(self, ifb, src_t, cv_t, am=True):
        return resample_descs(ifb, self.n, in_=src_t.data_ptr() + self.oy * src_t.stride(0) + self.ox * 4, in_w=self.in_w,
                              in_h=self.in_h, in_stride=src_t.stride(0), canvas=cv_t.data_ptr(), cv_w=self.cv_w, cv_h=self.cv_h,
                              cv_stride=cv_t.stride(0), x=self.cx, y=self.cy, w=self.out_w, h=self.out_h, alpha_meaningful=int(am))

    def cell(self, a, i):
        return a[self.cy[i]:self.cy[i] + self.out_h, self.cx[i]:self.cx[i] + self.out_w]

    def oracle_cell(self, src, canvas, i, am=True):
        out = self.cell(canvas, i).copy()
        oracle.scale_and_render(np.ascontiguousarray(src[self.oy[i]:self.oy[i] + self.in_h, self.ox[i]:self.ox[i] + self.in_w]), out,
                                filter=2, alpha_meaningful=am)
        return out


def run_grid(ifb, torch, grid, src_t, sentinel_np, force_generic=False, stream=None):
    """one call of every job of `grid` on a fresh Batch (the other path's reference); -> (canvas, counter movement)"""
    b = ifb.Batch(0)
    b.set_option(ifb.Batch.OPT_FORCE_GENERIC, int(force_generic))
    cv = dev(torch, sentinel_np)
    before = counters(b)
    b.enqueue(grid.descs(ifb, src_t, cv), stream=stream)
    torch.cuda.synchronize()
    out = host(cv)
    m = moved(b, before)
    b.close()
    return out, m


# ----------------------------------------------------------------------------------- 1. host ahead, mixed operations, one stream
class Calls:
    """calls made back to back on one batch; each records what it wrote and how to compute the oracle's bytes for it, which is
    done after the last enqueue, so that the host stays ahead of the stalled stream"""
    def __init__(self, ifb, torch, b):
        self.ifb, self.torch, self.b = ifb, torch, b
        self.checks = []          # (name, device tensor, () -> expected numpy)
        self.paths = []           # (name, counter key, counter movement of the call)

    def check(self, name, t, fn, *args, **kw):
        self.checks.append((name, t, functools.partial(fn, *args, **kw)))

    def on_path(self, name, key, fn):
        before = counters(self.b)
        fn()
        self.paths.append((name, key, moved(self.b, before)))

    def resample(self, name, seed, iw, ih, ow, oh, x0=0, filter=2, am=True, key=None):
        """the window at column x0 of a seeded source into a sub-rectangle of a sentinel canvas; x0 % 4 != 0 keeps it off the ring"""
        ifb, torch = self.ifb, self.torch
        src = noise(iw + x0, ih, seed, am)
        st = dev(torch, src)
        cv = sentinel(oh + 3, ow + 5, seed)
        ct = dev(torch, cv)
        sw = win(ifb, st[:, x0:], am)
        self.on_path(name, key, lambda: self.b.scale_and_render_many([(sw, win(ifb, ct), params(ifb, ow, oh, 2, 1, filter))]))

        def exp(src=src, cv=cv):
            out = cv.copy()
            oracle.scale_and_render(np.ascontiguousarray(src[:, x0:]), out[1:1 + oh, 2:2 + ow], filter=filter, alpha_meaningful=am)
            return out
        self.check(name, ct, exp)

    def oriented(self, name, seed, iw, ih, ow, oh, flag, key):
        ifb, torch = self.ifb, self.torch
        src = noise(iw, ih, seed)
        st = dev(torch, src)
        cv = sentinel(oh, ow, seed)
        ct = dev(torch, cv)
        self.on_path(name, key, lambda: self.b.scale_and_render_oriented([(win(ifb, st, True), win(ifb, ct), params(ifb, ow, oh), flag)]))
        self.check(name, ct, lambda: expect_resample(oo.gather(src, flag), cv, alpha_meaningful=True))


def _fill_then_copy(frame, patch, r):
    exp = frame.copy()
    ew = cvo.Win.of(exp)
    cvo.fill_rectangle(ew.sub(0, 0, 30, 20), (10 + r, 20, 30, 255), 3, 4, 25, 17)
    cvo.copy_rectangle(cvo.Win.of(patch.copy()), ew.sub(30, 20, 70 + r, 50 + r), 2, 1, 5, 6, 15, 8)
    return exp


def _corners(src, mode, radius, matte):
    exp = src.copy()
    rco.round_corners(exp, mode, radius, matte)
    return exp


def _watermarked(frame, logo, draw):
    exp = frame.copy()
    wo.expansion(exp, wo.REPLACE_SELF, (0, 0, 0, 0), logo, True, draw)
    return exp


def _pipeline(rgb, cv, logo, draw):
    exp = expect_resample(oo.gather(pco.convert(pco.RGB24_TO_BGRA, rgb), 6), cv, alpha_meaningful=False)
    wo.expansion(exp, wo.REPLACE_SELF, (0, 0, 0, 0), logo, True, draw)
    rco.round_corners(exp, rco.PIXELS, (17,), (40, 50, 60, 255))
    return exp


def _mixed_calls(ifb, torch, b, seed0):
    """39 calls of every operation, distinct geometries (cold tables every time), and one pipeline whose calls feed each other:
    to_bgra -> orient -> resample -> watermark -> round_corners -> from_bgra"""
    c = Calls(ifb, torch, b)
    k = seed0
    for r in range(3):
        k += 100
        c.resample(f"ring {r}", k + 1, 320 + 16 * r, 240 + 8 * r, 80 + r, 60 + r, key="fused")
        c.resample(f"tile {r}", k + 2, 40 + r, 30 + r, 97 + r, 71 + r, key="tile")
        c.resample(f"generic {r}", k + 3, 600 + r, 400 + r, 20 + r, 16 + r, x0=1, key="generic")
        c.oriented(f"flag 3 {r}", k + 4, 256 + 4 * r, 192 + r, 64 + r, 48 + r, 3, key="fused")
        c.oriented(f"flag 6 {r}", k + 5, 256 + 4 * r, 192 + r, 48 + r, 64 + r, 6, key="fused")
        # canvas: a FillRect and a CopyRectToCanvas on a sentinel frame
        frame, patch = sentinel(50 + r, 70 + r, k + 6), noise(20, 10, k + 7)
        ft, pt = dev(torch, frame), dev(torch, patch)
        fw = win(ifb, ft)
        b.canvas([ifb.FillRect(fw.window(0, 0, 30, 20), 3, 4, 25, 17, (10 + r, 20, 30, 255)),
                  ifb.CopyRectToCanvas(win(ifb, pt), fw.window(30, 20, 70 + r, 50 + r), 2, 1, 15, 8, 5, 6)])
        c.check(f"canvas {r}", ft, _fill_then_copy, frame, patch, r)
        # orient into a sentinel output
        src = noise(33 + r, 21 + r, k + 8)
        ot = dev(torch, sentinel(33 + r, 21 + r, k + 9))
        b.orient([(win(ifb, dev(torch, src)), win(ifb, ot), 5 + r)])
        c.check(f"orient {5 + r}", ot, oo.gather, src, 5 + r)
        # colour chain in place
        src = noise(45 + r, 31 + r, k + 10)
        ct = dev(torch, src)
        steps = [ifb.ColorFilterSrgb.sepia(), ifb.ColorFilterSrgb.contrast(0.3)][r % 2]
        b.color_chain([(win(ifb, ct, True), steps)])
        c.check(f"colour {r}", ct, lambda src=src, steps=steps: co.run_chain(src, co.of_product(steps), True)[0])
        # pixel conversion of gray rows into a sentinel BGRA frame
        gray = np.random.default_rng(k + 11).integers(0, 256, (17 + r, 29 + r, 1), dtype=np.uint8)
        pt = dev(torch, sentinel(17 + r, 29 + r, k + 12))
        b.pixel_convert([ifb.GrayToBgra(dev(torch, gray), win(ifb, pt))])
        c.check(f"gray {r}", pt, pco.convert, pco.GRAY_TO_BGRA, gray)
        # rounded corners in place
        src = noise(61 + r, 43 + r, k + 13)
        rt = dev(torch, src)
        b.round_corners([(win(ifb, rt, True), ifb.RoundCornersMode.percentage(20 + r), (5, 6, 7, 200))])
        c.check(f"corners {r}", rt, _corners, src, rco.PERCENTAGE, (20 + r,), (5, 6, 7, 200))
        # a watermark (with an opacity: a colour chain inside the call)
        frame, logo = noise(90 + r, 70 + r, k + 14, alpha=False), noise(23 + r, 19, k + 15)
        ft, lt = dev(torch, frame), dev(torch, logo)
        spec = ifb.Watermark(fit_box=ifb.WatermarkConstraintBox.image_percentage(10, 10, 90, 90), fit_mode=ifb.WatermarkConstraintMode.Within,
                             gravity=ifb.ConstraintGravity.percentage(100, 100), opacity=[None, 0.7, 0.4][r])
        draw = ifb.watermark_layout(frame.shape[1], frame.shape[0], logo.shape[1], logo.shape[0], spec)
        c.on_path(f"watermark {r}", "launches", lambda: b.watermark([(win(ifb, ft), win(ifb, lt, True), spec)]))
        c.check(f"watermark {r}", ft, _watermarked, frame, logo, draw)
    # the pipeline: every call reads what the call before it wrote
    rgb = np.random.default_rng(seed0 + 99).integers(0, 256, (300, 200, 3), dtype=np.uint8)
    bgra = b.to_bgra(dev(torch, rgb))
    ot = dev(torch, sentinel(200, 300, seed0 + 98))
    turned = b.orient([(bgra, win(ifb, ot), 6)])[0]
    cv = sentinel(100, 150, seed0 + 97)
    ct = dev(torch, cv)
    cw = win(ifb, ct)
    c.on_path("pipeline resample", "fused", lambda: b.scale_and_render_many([(turned, cw, params(ifb, 150, 100))]))
    logo = noise(30, 20, seed0 + 96)
    spec = ifb.Watermark(fit_box=ifb.WatermarkConstraintBox.image_percentage(0, 0, 50, 50), fit_mode=ifb.WatermarkConstraintMode.Within)
    b.watermark([(cw, win(ifb, dev(torch, logo), True), spec)])
    b.round_corners([(cw, ifb.RoundCornersMode.pixels(17), (40, 50, 60, 255))])
    out_rgb = b.from_bgra(cw, 3)
    draw = ifb.watermark_layout(150, 100, 30, 20, spec)
    c.check("pipeline canvas", ct, _pipeline, rgb, cv, logo, draw)
    c.check("pipeline rgb", out_rgb, lambda: pco.convert(pco.BGRA_TO_RGB24, _pipeline(rgb, cv, logo, draw)))
    return c


def test_host_ahead_mixed_operations_one_stream(ifb, torch, stall):
    b = ifb.Batch(0)
    assert b.ring_status()[0], b.ring_status()[1]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda.synchronize()
        before = counters(b)
        stall(s, 300)                                   # the calls' inputs are made between them
        t0 = time.perf_counter()
        c = _mixed_calls(ifb, torch, b, 1000)
        busy = not s.query()
        t0 = time.perf_counter() - t0
    m = moved(b, before)
    torch.cuda.synchronize()
    assert busy, f"the stream finished before the last call was enqueued ({t0 * 1e3:.0f} ms of host time): the host was not ahead"
    n_calls = 3 * 11 + 6
    assert m["pinned"] >= n_calls, f"{m['pinned']} pinned slots for {n_calls} calls: staging slots were reused while busy"
    assert m["uploads"] >= 3 * 6 + 2, m
    for name, key, got in c.paths:
        assert got[key] >= 1 and (key == "launches" or got["fused"] + got["tile"] + got["generic"] == 1), (name, key, got)
    for name, t, exp in c.checks:
        assert_equal(host(t), exp(), name)
    b.close()


def test_host_ahead_identical_calls_keep_their_own_work_lists(ifb, torch, stall):
    """every call the same operation with the same shapes and item count, so that a work list overwritten in its staging slot
    before its copy ran would still be a complete, valid work list: only the canvases show it, as a call's sentinel left in place"""
    b = ifb.Batch(0)
    s = torch.cuda.Stream()
    n, rects = 48, [(0, 0, 8, 4), (9, 0, 17, 5), (0, 5, 6, 12), (8, 6, 16, 11)]      # no two overlap
    frames = [sentinel(12, 17, 500 + i) for i in range(n)]
    with torch.cuda.stream(s):
        ts = [dev(torch, f) for f in frames]
        torch.cuda.synchronize()
        before = counters(b)
        stall(s, 300)
        for i, t in enumerate(ts):
            w = win(ifb, t)
            b.canvas([ifb.FillRect(w, *r, (i, 255 - i, (7 * i + k) & 255, 255)) for k, r in enumerate(rects)])
        busy = not s.query()
    torch.cuda.synchronize()
    assert busy
    assert moved(b, before)["pinned"] >= n
    for i, (f, t) in enumerate(zip(frames, ts)):
        exp = f.copy()
        for k, r in enumerate(rects):
            cvo.fill_rectangle(cvo.Win.of(exp), (i, 255 - i, (7 * i + k) & 255, 255), *r)
        assert_equal(host(t), exp, f"call {i}")
    b.close()


# ------------------------------------------------------------------------------ 2. tables uploaded on one stream, used on another
@pytest.mark.parametrize("many", [False, True], ids=["serial_plans", "parallel_plans"])
def test_tables_uploaded_on_one_stream_used_on_another(ifb, torch, stall, many):
    """call 1 on a stalled stream A uploads the tables of new geometries there; the same geometries on stream B, then on the batch's
    own stream, must wait for that upload.  Fewer than 8 new geometries: plans built one by one (and a watermark's tables committed
    alone, DevBlob::commit); 8 or more: built in parallel and packed (commit_many)."""
    b = ifb.Batch(0)
    A, B = torch.cuda.Stream(), torch.cuda.Stream()
    per = 4 if many else 1
    # (in_w, in_h, out_w, out_h, x0, path): ring, tile, and the generic pair (a window off the 16-byte grid, too wide for the tile kernel)
    geos = []
    for j in range(per):
        geos += [(256 + 16 * j, 144 + j, 64 + j, 36 + j, 0, "fused"), (24 + j, 20, 55 + j, 41, 0, "tile"), (640 + j, 360, 20 + j, 12, 3, "generic")]
    logo_w, logo_h = 50, 40
    spec = ifb.Watermark(fit_box=ifb.WatermarkConstraintBox.image_percentage(0, 0, 100, 100), fit_mode=ifb.WatermarkConstraintMode.Distort)
    draw = ifb.watermark_layout(100, 80, logo_w, logo_h, spec)
    assert (draw.w, draw.h) == (100, 80) and draw.crop is None
    seed = 2000 + 100 * many

    def call(stream, tag):
        jobs, checks = [], []
        for g, (iw, ih, ow, oh, x0, _) in enumerate(geos):
            src = noise(iw + x0, ih, seed + 17 * g + tag)
            st = dev(torch, src)
            cv = sentinel(oh, ow, seed + 17 * g + tag)
            ct = dev(torch, cv)
            jobs.append((win(ifb, st[:, x0:], True), win(ifb, ct), params(ifb, ow, oh)))
            checks.append((f"stream {tag} geometry {g}", ct, functools.partial(expect_resample, src[:, x0:], cv, alpha_meaningful=True)))
        # the watermark's geometry (logo -> 100 x 80 with the layout's filter) as a plain resample
        logo = noise(logo_w, logo_h, seed + 999 + tag)
        cv = sentinel(80, 100, seed + 998 + tag)
        ct = dev(torch, cv)
        jobs.append((win(ifb, dev(torch, logo), True), win(ifb, ct), params(ifb, 100, 80, filter=int(draw.filter))))
        checks.append((f"stream {tag} watermark geometry", ct,
                       functools.partial(expect_resample, logo, cv, alpha_meaningful=True, filter=int(draw.filter))))
        if stream == "own":
            _UPLOAD[0].synchronize()                  # the batch's own stream does not wait for torch's streams
        b.scale_and_render_many(jobs, stream=stream)
        return checks

    with torch.cuda.stream(A):
        frame = noise(100, 80, seed + 5, alpha=False)
        logo = noise(logo_w, logo_h, seed + 6)
        ft, lt = dev(torch, frame), dev(torch, logo)
        torch.cuda.synchronize()
        stall(A, 300)
        before = counters(b)
        if not many:
            b.watermark([(win(ifb, ft), win(ifb, lt, True), spec)], stream=A.cuda_stream)   # its tables: DevBlob::commit on A
        checks = call(A.cuda_stream, 0)
        m1 = moved(b, before)
        mid = counters(b)
        with torch.cuda.stream(B):
            checks += call(B.cuda_stream, 1)
        checks += call("own", 2)
        m23 = moved(b, mid)
        busy = not A.query()
    torch.cuda.synchronize()
    b.sync()
    assert busy, "stream A finished before the calls on B were enqueued"
    assert m1["uploads"] == len(geos) + 1 and m23["uploads"] == 0, (m1, m23)     # every table went up once, on A
    for key in ("fused", "tile", "generic"):
        want = sum(1 for g in geos if g[5] == key) + (key == "tile")            # + the watermark's geometry, an up-scale
        assert m1[key] == want and m23[key] == 2 * want, (key, m1, m23)
    for name, t, exp in checks:
        assert_equal(host(t), exp(), name)
    if not many:
        assert_equal(host(ft), _watermarked(frame, logo, draw), "watermark on A")
    b.close()


# ------------------------------------------------------------------------------------------------------------ 3. plan cache bound
def _cache_geometries():
    """4 480 distinct geometries: small down-scales, and 500 tall ones whose ring tables (a V weight row per source row) make the
    packed tables of the call larger than one 32 MiB chunk of the table arena"""
    small = [(20 + i % 80, 20 + i // 80, (20 + i % 80) // 3 + 1, (20 + i // 80) // 3 + 1) for i in range(3980)]
    tall = [(96, 3000 + j, 24, (3000 + j) // 4) for j in range(500)]
    return small, tall


def _cache_call(ifb, torch, geos, src, src_t, seed):
    """one call of `geos` (one job each) into one sentinel canvas, 128 cells of 40 px a row, rows 32 px high for outputs that fit,
    else 900; -> (descriptors, canvas tensor, sentinel, layout)"""
    n, per_row = len(geos), 128
    g = np.asarray(geos, np.int64)
    rng = np.random.default_rng(seed)
    ox = rng.integers(0, (src.shape[1] - g[:, 0]) // 4 + 1) * 4
    oy = rng.integers(0, src.shape[0] - g[:, 1] + 1)
    cx, cy = np.zeros(n, np.int64), np.zeros(n, np.int64)
    y = 0
    for cell_h, sel in ((32, np.flatnonzero(g[:, 3] <= 32)), (900, np.flatnonzero(g[:, 3] > 32))):
        j = np.arange(len(sel))
        cx[sel], cy[sel] = (j % per_row) * 40, y + (j // per_row) * cell_h
        y += -(-len(sel) // per_row) * cell_h
    assert g[:, 2].max() <= 40
    cv = sentinel(y, per_row * 40, seed)
    ct = dev(torch, cv)
    d = resample_descs(ifb, n, in_=src_t.data_ptr() + oy * src_t.stride(0) + ox * 4, in_w=g[:, 0], in_h=g[:, 1], in_stride=src_t.stride(0),
                       canvas=ct.data_ptr(), cv_w=cv.shape[1], cv_h=cv.shape[0], cv_stride=ct.stride(0), x=cx, y=cy, w=g[:, 2], h=g[:, 3],
                       alpha_meaningful=1)
    return d, ct, cv, (g, ox, oy, cx, cy)


def _cache_expected(src, cv, lay, pick):
    g, ox, oy, cx, cy = lay
    exp = cv.copy()
    for k in pick:
        iw, ih, ow, oh = (int(v) for v in g[k])
        oracle.scale_and_render(np.ascontiguousarray(src[oy[k]:oy[k] + ih, ox[k]:ox[k] + iw]), exp[cy[k]:cy[k] + oh, cx[k]:cx[k] + ow],
                                filter=2, alpha_meaningful=True)
    return exp


def test_plan_cache_bound_drop_and_rebuild(ifb, torch, stall):
    b = ifb.Batch(0)
    s = torch.cuda.Stream()
    small, tall = _cache_geometries()
    geos1 = small + tall
    assert len(set(geos1)) == len(geos1) > 4096
    src = noise(512, 3600, 3001)
    with torch.cuda.stream(s):
        src_t = dev(torch, src)
        torch.cuda.synchronize()
        # call 1: more than 4096 new geometries into the empty cache, behind a stall
        d1, ct1, cv1, lay1 = _cache_call(ifb, torch, geos1, src, src_t, 11)
        geos2 = [(20 + i, 101, 7 + i % 30, 30) for i in range(40)]
        assert not set(geos2) & set(geos1)
        d2, ct2, cv2, lay2 = _cache_call(ifb, torch, geos2, src, src_t, 12)
        torch.cuda.synchronize()
        before = counters(b)
        stall(s, 400)
        t1 = time.perf_counter()
        b.enqueue(d1, stream=s.cuda_stream)
        t1 = time.perf_counter() - t1
        busy1 = not s.query()
        m1 = moved(b, before)
        # call 2, with call 1 still in flight: new geometries take the cache past 4096, so it is dropped behind a synchronise
        b.enqueue(d2, stream=s.cuda_stream)
    torch.cuda.synchronize()
    assert busy1, f"call 1 took {t1 * 1e3:.0f} ms on the host, longer than the stall"
    assert m1["uploads"] == len(geos1), m1                       # one table upload per geometry: more than 4096 plans existed
    assert m1["staged"] > 32 * MiB, f"{m1['staged']} bytes of tables: not more than one 32 MiB chunk"
    assert m1["fused"] + m1["tile"] + m1["generic"] == len(geos1), m1
    exp1 = _cache_expected(src, cv1, lay1, range(len(geos1)))
    assert_equal(host(ct1), exp1, "call 1")
    assert_equal(host(ct2), _cache_expected(src, cv2, lay2, range(len(geos2))), "call 2")
    # call 3 reuses geometries of call 1: their plans were dropped, so they are built and uploaded again
    reuse = small[::40] + tall[::10]
    with torch.cuda.stream(s):
        d3, ct3, cv3, lay3 = _cache_call(ifb, torch, reuse, src, src_t, 13)
        before = counters(b)
        b.enqueue(d3, stream=s.cuda_stream)
        m3 = moved(b, before)
    torch.cuda.synchronize()
    assert m3["uploads"] == len(reuse), (m3, "the plans of call 1 were not dropped")
    assert_equal(host(ct3), _cache_expected(src, cv3, lay3, range(len(reuse))), "call 3")
    b.close()


# ---------------------------------------------------------------------------------------------------- 4. TMA descriptor cache
def test_tma_descriptor_cache_clear_and_address_reuse(ifb, torch, stall):
    """more than 65 536 distinct ring-kernel windows over a batch's life (the descriptor cache is cleared past that), then a
    bitmap freed and another allocated at the same address with other content: the cached descriptor must read the new bytes"""
    b = ifb.Batch(0)
    s = torch.cuda.Stream()
    src = noise(2048, 1024, 4001)
    total = 0
    with torch.cuda.stream(s):
        src_t = dev(torch, src)
        torch.cuda.synchronize()
        for call, n in enumerate((40000, 30000)):
            i = np.arange(n) + total
            grid = Grid(n, 32, 32, 8, 8, ((i % 500) * 4, i // 500 + call))      # every window at its own 16-byte aligned origin
            cv = sentinel(grid.cv_h, grid.cv_w, 40 + call)
            ct = dev(torch, cv)
            d = grid.descs(ifb, src_t, ct)
            torch.cuda.synchronize()
            before = counters(b)
            stall(s, 300)
            b.enqueue(d, stream=s.cuda_stream)
            assert not s.query()
            assert moved(b, before)["fused"] == n
            torch.cuda.synchronize()
            got = host(ct)
            other, m = run_grid(ifb, torch, grid, src_t, cv, force_generic=True, stream=s.cuda_stream)
            assert m["generic"] == n
            assert_equal(got, other, f"call {call} against the generic pair")
            for k in (0, n // 2, n - 1):
                assert_equal(grid.cell(got, k), grid.oracle_cell(src, cv, k), f"call {call} job {k}")
            total += n
    assert total > 65536
    # address reuse: the same shape allocated again lands where the freed tensor was
    a = noise(256, 192, 4002)
    cv = sentinel(48, 64, 4003)
    out1, out2 = dev(torch, cv), dev(torch, cv)
    t = dev(torch, a)
    ptr = t.data_ptr()
    b.scale_and_render_many([(win(ifb, t, True), win(ifb, out1), params(ifb, 64, 48))], stream=s.cuda_stream)
    b.sync()
    torch.cuda.synchronize()
    del t
    a2 = noise(256, 192, 4004)
    t2 = dev(torch, a2)
    assert t2.data_ptr() == ptr, "the caching allocator did not reuse the address; the premise of this check is gone"
    torch.cuda.synchronize()
    before = counters(b)
    b.scale_and_render_many([(win(ifb, t2, True), win(ifb, out2), params(ifb, 64, 48))], stream=s.cuda_stream)
    assert moved(b, before)["fused"] == 1
    torch.cuda.synchronize()
    assert_equal(host(out1), expect_resample(a, cv, alpha_meaningful=True), "first tensor")
    assert_equal(host(out2), expect_resample(a2, cv, alpha_meaningful=True), "second tensor at the same address")
    b.close()


# ---------------------------------------------------------------------------------------------------------- 5. chunk seams
SEAM_JOBS = (0, 65534, 65535, 65536)


def test_65537_upscale_jobs_tile_kernel_and_generic_pair(ifb, torch, stall):
    """one geometry, 65 537 jobs: the tile kernel and the generic pair launch in chunks of 65 535 jobs"""
    n = 65537
    src = noise(1024, 1024, 5001)
    i = np.arange(n)
    grid = Grid(n, 8, 6, 13, 11, ((i % 250) * 4, (i // 250) * 3 % 1016))
    cv = sentinel(grid.cv_h, grid.cv_w, 51)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        src_t = dev(torch, src)
        torch.cuda.synchronize()
        outs = {}
        for generic in (False, True):
            b = ifb.Batch(0)
            b.set_option(ifb.Batch.OPT_FORCE_GENERIC, int(generic))
            ct = dev(torch, cv)
            d = grid.descs(ifb, src_t, ct)
            torch.cuda.synchronize()
            stall(s, 300)
            b.enqueue(d, stream=s.cuda_stream)
            assert not s.query()
            m = counters(b)
            assert m["generic" if generic else "tile"] == n and m["fused"] == 0, m
            assert m["launches"] == (4 if generic else 2), m             # two chunks
            torch.cuda.synchronize()
            outs[generic] = host(ct)
            b.close()
    assert_equal(outs[False], outs[True], "tile kernel against the generic pair")
    for k in SEAM_JOBS:
        exp = grid.oracle_cell(src, cv, k)
        assert_equal(grid.cell(outs[False], k), exp, f"tile job {k}")
        assert_equal(grid.cell(outs[True], k), exp, f"generic job {k}")


def test_65537_ring_jobs(ifb, torch, stall):
    """the ring kernel takes 65 537 jobs of one geometry in one launch"""
    n = 65537
    src = noise(1024, 1024, 5002)
    i = np.arange(n)
    grid = Grid(n, 32, 32, 8, 8, ((i % 240) * 4, i // 240))
    cv = sentinel(grid.cv_h, grid.cv_w, 52)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        src_t = dev(torch, src)
        b = ifb.Batch(0)
        ct = dev(torch, cv)
        d = grid.descs(ifb, src_t, ct)
        torch.cuda.synchronize()
        stall(s, 300)
        b.enqueue(d, stream=s.cuda_stream)
        assert not s.query()
        m = counters(b)
        assert m["fused"] == n and m["launches"] == 1, m
        torch.cuda.synchronize()
        got = host(ct)
        b.close()
        other, m = run_grid(ifb, torch, grid, src_t, cv, force_generic=True, stream=s.cuda_stream)
    assert m["generic"] == n
    assert_equal(got, other, "ring kernel against the generic pair")
    for k in SEAM_JOBS:
        assert_equal(grid.cell(got, k), grid.oracle_cell(src, cv, k), f"ring job {k}")


def test_generic_pair_intermediate_chunks_8k(ifb, torch, stall):
    """ten 7680x4320 -> 1920x1080 jobs on the generic pair: 133 MB of intermediate each, so two chunks of at most 1 GiB (8 + 2)"""
    n, (iw, ih), (ow, oh) = 10, (7680, 4320), (1920, 1080)
    assert ((1 << 30) // (ih * ow * 16)) == 8
    s = torch.cuda.Stream()
    gen = torch.Generator(device="cuda").manual_seed(6001)
    cv = sentinel(oh, ow, 61)
    with torch.cuda.stream(s):
        srcs = [torch.randint(0, 256, (ih, iw, 4), dtype=torch.uint8, device="cuda", generator=gen) for _ in range(n)]
        outs = {}
        for generic in (True, False):
            b = ifb.Batch(0)
            b.set_option(ifb.Batch.OPT_FORCE_GENERIC, int(generic))
            cts = [dev(torch, cv) for _ in range(n)]
            torch.cuda.synchronize()
            stall(s, 300)
            b.scale_and_render_many([(win(ifb, t, True), win(ifb, c), params(ifb, ow, oh)) for t, c in zip(srcs, cts)], stream=s.cuda_stream)
            assert not s.query()
            m = counters(b)
            if generic:
                assert m["generic"] == n and m["launches"] == 4, m       # H + V per chunk, two chunks
            else:
                assert m["fused"] == n, m
            torch.cuda.synchronize()
            outs[generic] = [host(c) for c in cts]
            b.close()
    for k in range(n):
        assert_equal(outs[True][k], outs[False][k], f"job {k}: generic pair against the ring kernel")
    for k in (7, 8):
        assert_equal(outs[True][k], expect_resample(host(srcs[k]), cv, alpha_meaningful=True), f"job {k} against the oracle")


def test_watermark_f_scratch_chunks(ifb, torch, stall):
    """four distinct watermarks drawn over four 4200x4200 frames need 4 x 282 MB of F: two scratch chunks (3 + 1) that reuse the
    same scratch addresses"""
    side, n = 4200, 4
    spec = ifb.Watermark(fit_box=ifb.WatermarkConstraintBox.image_percentage(0, 0, 100, 100), fit_mode=ifb.WatermarkConstraintMode.Distort)
    draw = ifb.watermark_layout(side, side, 64, 48, spec)
    assert (draw.w, draw.h) == (side, side)
    f_bytes = side * side * 16
    assert 3 * f_bytes <= (1 << 30) < 4 * f_bytes
    frames = [noise(side, side, 7001 + k, alpha=False) for k in range(n)]
    logos = [noise(64, 48, 7101 + k) for k in range(n)]
    b = ifb.Batch(0)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        fts = [dev(torch, f) for f in frames]
        lts = [dev(torch, l) for l in logos]
        torch.cuda.synchronize()
        before = counters(b)
        stall(s, 300)
        b.watermark([(win(ifb, f), win(ifb, l, True), spec) for f, l in zip(fts, lts)], stream=s.cuda_stream)
        assert not s.query()
        m = moved(b, before)
        torch.cuda.synchronize()
    assert m["launches"] == 2 * (2 + 1), m         # per chunk: H + V of the one geometry, one composite; one chunk would be 3
    got = [host(t) for t in fts]
    # every frame against the node's existing route on the device (one resample under BlendWithSelf) ...
    r = ifb.Batch(0)
    for k in range(n):
        t = dev(torch, frames[k])
        cw = win(ifb, t, compose=ifb.BitmapCompositing.BlendWithSelf)
        r.scale_and_render_many([(win(ifb, lts[k], True), cw, params(ifb, side, side, filter=int(draw.filter)))])
        r.sync()
        assert_equal(got[k], host(t), f"frame {k} against a plain resample")
    r.close()
    # ... and the frames on both sides of the seam against the oracle's expansion
    for k in (2, 3):
        exp = frames[k].copy()
        wo.expansion(exp, wo.REPLACE_SELF, (0, 0, 0, 0), logos[k], True, draw)
        assert_equal(got[k], exp, f"frame {k} against the oracle")
    b.close()


# ---------------------------------------------------------------------------------------------- 6. options on a live batch
def test_options_changed_on_a_live_batch(ifb, torch, stall):
    from tests.cpu_emu import hv_plan
    iw, ih, ow, oh = 1280, 720, 320, 180
    strips = {c: hv_plan(ifb, iw, ih, ow, oh, 2, strip_cols=c, alpha=True)[0].n_strips for c in (16, 32, 64)}
    assert len(set(strips.values())) == 3, strips               # three strip widths, three partitions
    src = noise(iw, ih, 8001)
    cv = sentinel(oh, ow, 81)
    exp = expect_resample(src, cv, alpha_meaningful=True)
    # (strip columns, min items, force generic, path, new tables)
    steps = [(64, 1, 0, "fused", 1), (32, 64, 0, "fused", 1), (16, 4096, 0, "fused", 1), (16, 4096, 1, "generic", 1),
             (64, 1, 0, "fused", 0), (32, 0, 0, "fused", None), (16, 64, 1, "generic", 0), (64, 100000, 0, "fused", 0)]
    b = ifb.Batch(0)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        st = dev(torch, src)
        cts = [dev(torch, cv) for _ in steps]
        torch.cuda.synchronize()
        stall(s, 300)
        moves = []
        for (cols, items, generic, _, _), ct in zip(steps, cts):
            b.set_option(ifb.Batch.OPT_STRIP_COLUMNS, cols)
            b.set_option(ifb.Batch.OPT_MIN_ITEMS, items)
            b.set_option(ifb.Batch.OPT_FORCE_GENERIC, generic)
            before = counters(b)
            b.scale_and_render_many([(win(ifb, st, True), win(ifb, ct), params(ifb, ow, oh))], stream=s.cuda_stream)
            moves.append(moved(b, before))
        assert not s.query()
    torch.cuda.synchronize()
    for (cols, items, generic, path, new), m, ct in zip(steps, moves, cts):
        assert m[path] == 1 and m["fused"] + m["generic"] + m["tile"] == 1, (cols, items, generic, m)
        if new is not None:
            assert m["uploads"] == new, (cols, items, generic, m)
        assert_equal(host(ct), exp, f"strip {cols}, min items {items}, generic {generic}")
    b.close()


# -------------------------------------------------------------------------------------------------------------- 7. threads
def _thread_calls(ifb, torch, b, me, n_calls, out):
    """n_calls mixed calls of thread `me` on its own torch stream; appends (name, tensor, expected)"""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for k in range(n_calls):
            seed = 9000 + 100 * me + k
            kind = (me + k) % 5
            if kind == 0:                                               # ring: a geometry of this thread and call
                src = noise(200 + 4 * k, 150 + me, seed)
                cv = sentinel(40 + me, 50 + k, seed)
                ct = dev(torch, cv)
                b.scale_and_render_many([(win(ifb, dev(torch, src), True), win(ifb, ct), params(ifb, 50 + k, 40 + me))], stream=s.cuda_stream)
                out.append((f"{me}/{k} ring", ct, expect_resample(src, cv, alpha_meaningful=True)))
            elif kind == 1:                                             # tile: an up-scale shared by every thread
                src = noise(30, 20, seed)
                cv = sentinel(45, 61, seed)
                ct = dev(torch, cv)
                b.scale_and_render_many([(win(ifb, dev(torch, src), True), win(ifb, ct), params(ifb, 61, 45))], stream=s.cuda_stream)
                out.append((f"{me}/{k} tile", ct, expect_resample(src, cv, alpha_meaningful=True)))
            elif kind == 2:
                f = sentinel(30 + me, 40, seed)
                ft = dev(torch, f)
                b.canvas([ifb.FillRect(win(ifb, ft), me, k % 7, 40 - k % 5, 30, (me, k, 200, 255))], stream=s.cuda_stream)
                exp = f.copy()
                cvo.fill_rectangle(cvo.Win.of(exp), (me, k, 200, 255), me, k % 7, 40 - k % 5, 30)
                out.append((f"{me}/{k} canvas", ft, exp))
            elif kind == 3:
                src = noise(27 + me, 19 + k, seed)
                ot = dev(torch, sentinel(27 + me, 19 + k, seed))
                b.orient([(win(ifb, dev(torch, src)), win(ifb, ot), 6 + k % 3)], stream=s.cuda_stream)
                out.append((f"{me}/{k} orient", ot, oo.gather(src, 6 + k % 3)))
            else:
                src = noise(33, 25 + me, seed)
                ct = dev(torch, src)
                b.color_chain([(win(ifb, ct, True), ifb.ColorFilterSrgb.invert())], stream=s.cuda_stream)
                b.round_corners([(win(ifb, ct, True), ifb.RoundCornersMode.pixels(5 + k), (1, 2, 3, 255))], stream=s.cuda_stream)
                exp = co.run_chain(src, co.preset(co.INVERT), True)[0]
                rco.round_corners(exp, rco.PIXELS, (5 + k,), (1, 2, 3, 255))
                out.append((f"{me}/{k} colour + corners", ct, exp))
        s.synchronize()


def _run_threads(fn, n):
    errors = []

    def body(me):
        try:
            fn(me)
        except BaseException as e:                                   # noqa: BLE001 -- reported by the main thread
            errors.append((me, e))
    ts = [threading.Thread(target=body, args=(me,)) for me in range(n)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errors:
        raise errors[0][1]


def test_eight_threads_share_one_batch(ifb, torch):
    b = ifb.Batch(0)
    outs = [[] for _ in range(8)]
    before = counters(b)
    _run_threads(lambda me: _thread_calls(ifb, torch, b, me, 20, outs[me]), 8)
    torch.cuda.synchronize()
    m = moved(b, before)
    assert m["fused"] >= 8 * 4 and m["tile"] >= 8 * 4, m
    for results in outs:
        assert len(results) == 20
        for name, t, exp in results:
            assert_equal(host(t), exp, name)
    b.close()


def test_eight_threads_drop_in_host_calls(ifb, torch):
    """each thread gets its own thread_local context (batch, pipeline slots, copy pool); pageable and pinned host buffers"""
    def buf(a, pinned):
        if not pinned:
            return a.copy()
        t = torch.from_numpy(a).pin_memory()
        return t.numpy()

    def body(me):
        for k in range(6):
            pinned = (me + k) % 2 == 1
            seed = 9500 + 10 * me + k
            # scale_and_render
            src = buf(noise(160 + me, 90 + k, seed), pinned)
            cv = buf(sentinel(40, 64, seed), pinned)
            exp = expect_resample(src, cv, alpha_meaningful=True)
            ifb.scale_and_render(ifb.BitmapWindow.from_numpy(src, alpha_meaningful=True), ifb.BitmapWindow.from_numpy(cv), params(ifb, 64, 40))
            assert_equal(cv, exp, f"{me}/{k} scale_and_render")
            # scale_and_render_many over the three pipeline slots
            srcs = [buf(noise(120 + 8 * j, 80, seed + j), pinned) for j in range(5)]
            cvs = [buf(sentinel(30, 41 + j, seed + j), pinned) for j in range(5)]
            exps = [expect_resample(a, c, alpha_meaningful=True) for a, c in zip(srcs, cvs)]
            ifb.scale_and_render_many([(ifb.BitmapWindow.from_numpy(a, alpha_meaningful=True), ifb.BitmapWindow.from_numpy(c), params(ifb, c.shape[1], 30))
                                       for a, c in zip(srcs, cvs)])
            for j, (c, e) in enumerate(zip(cvs, exps)):
                assert_equal(c, e, f"{me}/{k} scale_and_render_many job {j}")
            # rounded corners
            px = buf(noise(70 + me, 50, seed), pinned)
            exp = px.copy()
            rco.round_corners(exp, rco.PERCENTAGE, (30,), (9, 8, 7, 255))
            ifb.flow_bitmap_bgra_clear_around_rounded_corners(ifb.BitmapWindow.from_numpy(px), ifb.RoundCornersMode.percentage(30), (9, 8, 7, 255))
            assert_equal(px, exp, f"{me}/{k} round corners")
            # transpose
            a = buf(noise(37 + k, 23 + me, seed), pinned)
            t = buf(sentinel(37 + k, 23 + me, seed), pinned)
            exp = t.copy()
            oracle.transpose(a, exp)
            ifb.bitmap_window_transpose(ifb.BitmapWindow.from_numpy(a), ifb.BitmapWindow.from_numpy(t))
            assert_equal(t, exp, f"{me}/{k} transpose")
            # white balance
            px = buf(noise(64, 48 + k, seed, alpha=False), pinned)
            exp = px.copy()
            oracle.white_balance(exp, None)
            ifb.white_balance_srgb_mut(ifb.BitmapWindow.from_numpy(px))
            assert_equal(px, exp, f"{me}/{k} white balance")

    _run_threads(body, 8)


# ------------------------------------------------------------------------------------------------- 8. close with work in flight
def test_close_with_work_in_flight(ifb, torch, stall):
    b = ifb.Batch(0)
    s = torch.cuda.Stream()
    src = noise(640, 480, 10001)
    cv = sentinel(120, 160, 101)
    frame = sentinel(64, 80, 102)
    col = noise(50, 40, 103)
    with torch.cuda.stream(s):
        st, ct, ft, kt = dev(torch, src), dev(torch, cv), dev(torch, frame), dev(torch, col)
        up_cv = sentinel(90, 70, 104)
        ut = dev(torch, up_cv)
        torch.cuda.synchronize()
        stall(s, 300)
        t0 = time.perf_counter()
        b.scale_and_render_many([(win(ifb, st, True), win(ifb, ct), params(ifb, 160, 120)),
                                 (win(ifb, st[:60, :40], True), win(ifb, ut), params(ifb, 70, 90))], stream=s.cuda_stream)
        b.canvas([ifb.FillRect(win(ifb, ft), 5, 6, 70, 50, (1, 2, 3, 4))], stream=s.cuda_stream)
        b.color_chain([(win(ifb, kt, True), ifb.ColorFilterSrgb.grayscale_bt709())], stream=s.cuda_stream)
        assert not s.query(), f"the stream finished {(time.perf_counter() - t0) * 1e3:.0f} ms after the stall was enqueued"
        b.close()
        assert s.query(), "close() returned with the batch's work still running"
    assert_equal(host(ct), expect_resample(src, cv, alpha_meaningful=True), "resample")
    assert_equal(host(ut), expect_resample(src[:60, :40], up_cv, alpha_meaningful=True), "up-scale")
    exp = frame.copy()
    cvo.fill_rectangle(cvo.Win.of(exp), (1, 2, 3, 4), 5, 6, 70, 50)
    assert_equal(host(ft), exp, "canvas")
    assert_equal(host(kt), co.run_chain(col, co.preset(co.GRAY_BT709), True)[0], "colour chain")
