#!/usr/bin/env python
"""Measurement of the rows resample (Batch.scale_and_render_rows -> ifb200_batch_enqueue_rows) against the two routes a user has without
it: the two-step route (Batch.pixel_convert of every frame's decoder rows into a BGRA scratch frame, then Batch.scale_and_render_many,
on the same stream) and the floor (the plain resample of frames that are already BGRA).  Rows:
  (a) 64 x 3840x2160 RGB24 -> 512x288, Robidoux, linear light
  (b) 256 x 4032x3024 RGB24 -> 512x384
  (c) 64 x 3840x2160 RGBA32 with cut-out alpha -> 512x288
  (d) 16 x 640x480 RGB24 -> 1280x960 (an up-scale: the generic pair)
  (e) 64 x 4000x3000 RGB24 -> 500x375 with rows 12004 bytes apart (a pitch that is not a multiple of 16: the generic pair; a
      contiguous 4000-wide tensor has a 12000-byte pitch and takes the ring kernel)

Every call covers all frames of a row (each one a different image, together far larger than L2).  Time = CUDA events around one
call, the device kept busy (torch.cuda._sleep) while the host enqueues it, so that host work is not timed; warm-up 2 calls, then
the median of 5.  The three routes' outputs are compared byte for byte in the same run.  Algorithmic bytes: fused 3 or 4 B per
source pixel, two-step 3 or 4 + 4 + 4, floor 4, each + 4 B per output pixel.  Extra memory = the scratch frames the two-step route
needs.  The card's name and power limit are read in the same run and printed with the numbers.
--profile: instead, one torch.profiler run (CUDA activity) of the fused call and of the floor at row (a), printing the CUDA time per
kernel name: the RGB24 ring kernel against the BGRA ring kernel on the same geometry.
--oriented: the oriented rows resample (Batch.scale_and_render_rows_oriented -> ifb200_batch_enqueue_rows_oriented) instead, same
method, against the two-step route (Batch.pixel_convert, then Batch.scale_and_render_oriented), the rows floor (the rows resample of
rows that are already oriented) and the BGRA floor (the plain resample of oriented BGRA frames).  Rows:
  (o1) 256 x 4032x3024 RGB24, flag 6 -> 384x512;  (o2) the same, flag 8
  (o3) 64 x 3840x2160 RGB24, flag 3 -> 512x288
  (o4) 64 x 3840x2160 RGBA32 with cut-out alpha, flag 6 -> 288x512
  (o5) 16 x 640x480 RGB24, flag 6 -> 960x1280 (an up-scale: the generic pair)
With --profile: the RGB24 transposed ring kernel (row o1) against the stored RGB24 ring kernel on the same oriented geometry.
Usage: python tools/bench_rows.py [--trials 5] [--json out.json] [--profile] [--oriented]"""
import argparse, json, os, subprocess, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import imageflow_b200 as ifb


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, trials):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(trials):
        torch.cuda._sleep(40_000_000)                        # the device is busy while the host enqueues the call
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), ts


def frames(n, iw, ih, bpp, pitch=None, cutout=False):
    """n frames of decoder rows (random content; RGBA with cut-out alpha: a third of the pixels transparent, a third opaque), rows
    `pitch` bytes apart (default: contiguous)"""
    dev = torch.device("cuda:0")
    pitch = pitch or iw * bpp
    buf = torch.randint(0, 256, (n, ih, pitch), dtype=torch.uint8, device=dev)
    rows = torch.as_strided(buf, (n, ih, iw, bpp), (ih * pitch, pitch, bpp, 1))
    if cutout:
        u = torch.rand((n, ih, iw), device=dev)
        a = rows[..., 3]
        a[u < 0.33] = 0
        a[u > 0.67] = 255
    return buf, rows


def setup(batch, n, iw, ih, bpp, ow, oh, pitch=None, cutout=False):
    dev = torch.device("cuda:0")
    buf, rows = frames(n, iw, ih, bpp, pitch, cutout)
    scratch = torch.empty((n, ih, iw, 4), dtype=torch.uint8, device=dev)          # the two-step route's BGRA frames
    outs = [torch.zeros((n, oh, ow, 4), dtype=torch.uint8, device=dev) for _ in range(3)]
    p = ifb.ScaleAndRenderParams(w=ow, h=oh)
    am = bpp == 4
    win = lambda a, i: ifb.BitmapWindow.from_torch(a[i], alpha_meaningful=am)
    fused_d = batch.make_rows_descs([(rows[i], win(outs[0], i), p) for i in range(n)])
    op = ifb.pixel_op_for(bpp)
    convert_jobs = [op(ifb.PixelRows.from_torch(rows[i]), win(scratch, i)) for i in range(n)]
    plain_d = batch.make_descs([(win(scratch, i), win(outs[1], i), p) for i in range(n)])
    floor_d = batch.make_descs([(win(scratch, i), win(outs[2], i), p) for i in range(n)])
    return dict(buf=buf, rows=rows, scratch=scratch, outs=outs, fused_d=fused_d, convert_jobs=convert_jobs, plain_d=plain_d, floor_d=floor_d)


def row(batch, stream, name, n, iw, ih, bpp, ow, oh, trials, pitch=None, cutout=False):
    s = setup(batch, n, iw, ih, bpp, ow, oh, pitch, cutout)
    for k in ("fused_d", "plain_d", "floor_d"):                  # the bitmaps stay alive with `s`; the batch need not hold them
        s[k] = s[k][0]
    counts = lambda: (batch.fused_jobs, batch.generic_jobs, batch.tile_jobs)
    c0 = counts()
    batch.enqueue_rows(s["fused_d"], stream)
    torch.cuda.synchronize()
    path = {k: int(v) for k, v in zip(("ring", "generic", "tile"), np.subtract(counts(), c0)) if v}
    fused, fts = timed(lambda: batch.enqueue_rows(s["fused_d"], stream), trials)

    def two_step():
        batch.pixel_convert(s["convert_jobs"], stream)
        batch.enqueue(s["plain_d"], stream)
    two, tts = timed(two_step, trials)
    floor, _ = timed(lambda: batch.enqueue(s["floor_d"], stream), trials)
    torch.cuda.synchronize()
    outs = s["outs"]
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2]), (name, "routes differ")
    in_px, out_px = n * iw * ih, n * ow * oh
    alg = lambda b: b * in_px + 4 * out_px
    r = dict(row=name, frames=n, size=f"{iw}x{ih}", fmt="RGBA32" if bpp == 4 else "RGB24", pitch=pitch or iw * bpp, out=f"{ow}x{oh}", path=path,
             fused_ms=round(fused, 3), two_step_ms=round(two, 3), floor_ms=round(floor, 3), fused_over_floor=round(fused / floor, 3),
             fused_over_two_step=round(fused / two, 3), fused_alg_gbps=round(alg(bpp) / fused / 1e6, 1), two_step_alg_gbps=round(alg(bpp + 8) / two / 1e6, 1),
             floor_alg_gbps=round(alg(4) / floor / 1e6, 1), two_step_scratch_bytes=int(s["scratch"].numel()), bit_exact=True,
             fused_trials=[round(x, 3) for x in fts], two_step_trials=[round(x, 3) for x in tts])
    print(json.dumps(r), flush=True)
    del s, outs
    batch._keep.clear()                                      # the batch holds the bitmaps of enqueued calls; all of them have completed
    torch.cuda.empty_cache()
    return r


def profile(batch, stream, n=64, iw=3840, ih=2160):
    """kernel time of the fused call (RGB24 rows) and of the floor (the BGRA frames), per kernel name"""
    from torch.profiler import ProfilerActivity, profile as tprofile
    s = setup(batch, n, iw, ih, 3, 512, 288)
    batch.pixel_convert(s["convert_jobs"], stream)
    for name, d, fn in (("fused", s["fused_d"][0], batch.enqueue_rows), ("floor", s["floor_d"][0], batch.enqueue)):
        for _ in range(2):
            fn(d, stream)
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                fn(d, stream)
            torch.cuda.synchronize()
        ks = {}
        for e in prof.events():
            if e.device_type.name == "CUDA":
                ks.setdefault(e.name, []).append(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total)
        for k, v in ks.items():
            print(json.dumps(dict(route=name, kernel=k[:100], launches=len(v), median_us=round(float(np.median(v)), 1))), flush=True)
    del s
    batch._keep.clear()
    torch.cuda.empty_cache()


def orient_t(a, flag):
    """the (n, h, w, c) frames oriented by the EXIF flag, contiguous (the closed form of include/ifb200.h)"""
    t, fx, fy = {2: (0, 1, 0), 3: (0, 1, 1), 4: (0, 0, 1), 5: (1, 0, 0), 6: (1, 0, 1), 7: (1, 1, 1), 8: (1, 1, 0)}.get(flag, (0, 0, 0))
    dims = [d for d, f in ((1, fy), (2, fx)) if f]
    b = a.flip(dims) if dims else a
    return (b.transpose(1, 2) if t else b).contiguous()


def oriented_setup(batch, n, iw, ih, bpp, flag, ow, oh, cutout=False):
    dev = torch.device("cuda:0")
    buf, rows = frames(n, iw, ih, bpp, None, cutout)
    rows_o = orient_t(rows, flag)                                                 # the rows floor's input: rows already oriented
    scratch = torch.empty((n, ih, iw, 4), dtype=torch.uint8, device=dev)          # the two-step route's BGRA frames
    outs = [torch.zeros((n, oh, ow, 4), dtype=torch.uint8, device=dev) for _ in range(4)]
    p = ifb.ScaleAndRenderParams(w=ow, h=oh)
    am = bpp == 4
    win = lambda a, i: ifb.BitmapWindow.from_torch(a[i], alpha_meaningful=am)
    op = ifb.pixel_op_for(bpp)
    batch.pixel_convert([op(ifb.PixelRows.from_torch(rows[i]), win(scratch, i)) for i in range(n)], torch.cuda.current_stream().cuda_stream)
    scratch_o = orient_t(scratch, flag)                                           # the BGRA floor's input
    d = dict(fused_d=batch.make_rows_oriented_descs([(rows[i], win(outs[0], i), p, flag) for i in range(n)]),
             oriented_d=batch.make_oriented_descs([(win(scratch, i), win(outs[1], i), p, flag) for i in range(n)]),
             rows_floor_d=batch.make_rows_descs([(rows_o[i], win(outs[2], i), p) for i in range(n)]),
             floor_d=batch.make_descs([(win(scratch_o, i), win(outs[3], i), p) for i in range(n)]))
    convert_jobs = [op(ifb.PixelRows.from_torch(rows[i]), win(scratch, i)) for i in range(n)]
    return dict(buf=buf, rows=rows, rows_o=rows_o, scratch=scratch, scratch_o=scratch_o, outs=outs, convert_jobs=convert_jobs,
                **{k: v[0] for k, v in d.items()})


def oriented_row(batch, stream, name, n, iw, ih, bpp, flag, ow, oh, trials, cutout=False):
    s = oriented_setup(batch, n, iw, ih, bpp, flag, ow, oh, cutout)
    counts = lambda: (batch.fused_jobs, batch.generic_jobs, batch.tile_jobs)
    c0 = counts()
    batch.enqueue_rows_oriented(s["fused_d"], stream)
    torch.cuda.synchronize()
    path = {k: int(v) for k, v in zip(("ring", "generic", "tile"), np.subtract(counts(), c0)) if v}
    fused, fts = timed(lambda: batch.enqueue_rows_oriented(s["fused_d"], stream), trials)

    def two_step():
        batch.pixel_convert(s["convert_jobs"], stream)
        batch.enqueue_oriented(s["oriented_d"], stream)
    two, tts = timed(two_step, trials)
    rows_floor, _ = timed(lambda: batch.enqueue_rows(s["rows_floor_d"], stream), trials)
    floor, _ = timed(lambda: batch.enqueue(s["floor_d"], stream), trials)
    torch.cuda.synchronize()
    outs = s["outs"]
    assert all(torch.equal(outs[0], o) for o in outs[1:]), (name, "routes differ")
    r = dict(row=name, frames=n, size=f"{iw}x{ih}", fmt="RGBA32" if bpp == 4 else "RGB24", flag=flag, out=f"{ow}x{oh}", path=path,
             fused_ms=round(fused, 3), two_step_ms=round(two, 3), rows_floor_ms=round(rows_floor, 3), bgra_floor_ms=round(floor, 3),
             fused_over_rows_floor=round(fused / rows_floor, 3), fused_over_two_step=round(fused / two, 3),
             two_step_scratch_bytes=int(s["scratch"].numel()), bit_exact=True,
             fused_trials=[round(x, 3) for x in fts], two_step_trials=[round(x, 3) for x in tts])
    print(json.dumps(r), flush=True)
    del s, outs
    batch._keep.clear()
    torch.cuda.empty_cache()
    return r


def oriented_profile(batch, stream, n=256, iw=4032, ih=3024, flag=6):
    """kernel time of the fused call (RGB24 rows, transposed reads) and of the rows floor (the stored RGB24 form on the same oriented
    geometry), per kernel name"""
    from torch.profiler import ProfilerActivity, profile as tprofile
    s = oriented_setup(batch, n, iw, ih, 3, flag, 384, 512)
    for name, d, fn in (("fused", s["fused_d"], batch.enqueue_rows_oriented), ("rows_floor", s["rows_floor_d"], batch.enqueue_rows)):
        for _ in range(2):
            fn(d, stream)
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                fn(d, stream)
            torch.cuda.synchronize()
        ks = {}
        for e in prof.events():
            if e.device_type.name == "CUDA":
                ks.setdefault(e.name, []).append(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total)
        for k, v in ks.items():
            print(json.dumps(dict(route=name, kernel=k[:100], launches=len(v), median_us=round(float(np.median(v)), 1))), flush=True)
    del s
    batch._keep.clear()
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--json", default=None)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--oriented", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    info = card()
    print("card:", info, flush=True)
    batch = ifb.Batch(0)
    stream = torch.cuda.current_stream().cuda_stream
    if a.profile:
        (oriented_profile if a.oriented else profile)(batch, stream)
        return
    if a.oriented:
        rows = [oriented_row(batch, stream, "o1", 256, 4032, 3024, 3, 6, 384, 512, a.trials),
                oriented_row(batch, stream, "o2", 256, 4032, 3024, 3, 8, 384, 512, a.trials),
                oriented_row(batch, stream, "o3", 64, 3840, 2160, 3, 3, 512, 288, a.trials),
                oriented_row(batch, stream, "o4", 64, 3840, 2160, 4, 6, 288, 512, a.trials, cutout=True),
                oriented_row(batch, stream, "o5", 16, 640, 480, 3, 6, 960, 1280, a.trials)]
        if a.json:
            json.dump({"card": info, "rows": rows}, open(a.json, "w"), indent=1)
        return
    rows = [row(batch, stream, "a", 64, 3840, 2160, 3, 512, 288, a.trials),
            row(batch, stream, "b", 256, 4032, 3024, 3, 512, 384, a.trials),
            row(batch, stream, "c", 64, 3840, 2160, 4, 512, 288, a.trials, cutout=True),
            row(batch, stream, "d", 16, 640, 480, 3, 1280, 960, a.trials),
            row(batch, stream, "e", 64, 4000, 3000, 3, 500, 375, a.trials, pitch=12004)]
    if a.json:
        json.dump({"card": info, "rows": rows}, open(a.json, "w"), indent=1)


if __name__ == "__main__":
    main()
