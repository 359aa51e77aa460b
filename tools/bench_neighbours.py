#!/usr/bin/env python
"""Measurement of the SURVEY.md section 8(f) neighbours of the resample path that are built: transpose, flips, white balance, detect_content
and rounded corners; `bench_neighbours.py canvas` measures the canvas operations alone (canvas_rows), `bench_neighbours.py orient`
the one-gather orientation against the reference's expansion into transposes and flips (orient_rows), `bench_neighbours.py color` the
colour chains against the reference's node-by-node expansion (color_rows), `bench_neighbours.py watermark` the watermark composites
against the node-by-node expansion and the best existing route (watermark_rows), `bench_neighbours.py formats` the pixel-format
conversions against a torch copy of the same bytes and the torch expression a user would write (formats_rows), `bench_neighbours.py
trim` the batched whitespace trim against per-frame detect_content and the host walk (trim_rows; `trim_profile` its kernel times)
(the reference benchmarks transposes at 4K / 8K in benches/bench_graphics.rs:9-62).  Inputs resident in HBM, CUDA events on
the launching stream, >= 3 warm-up calls; a set of 64 different images per size (>= 2 GB, far larger than L2) is cycled so that
no call finds its data in cache.  One JSON line per (operation, size) with the HBM roofline of the kernel: algorithmic
bytes = 4 read + 4 written per pixel, peak = MEASURED_PEAKS.json hbm_gbs (fallback: the H100 SXM data sheet's 3350 GB/s).
The CPU column is the oracle's plain C loop on one host thread (test infrastructure, as in bench.py)."""
import json, os, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import imageflow_b200 as ifb


def peak():
    try:
        return float(json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"]), "measured"
    except Exception:
        return 3350.0, "H100 SXM data sheet (3.35 TB/s HBM3), not a measured peak"


def main():
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    batch = ifb.Batch(0)
    stream = torch.cuda.current_stream().cuda_stream
    pk, src = peak()
    import oracle
    for (w, h) in ((3840, 2160), (7680, 4320)):
        n = 64 if w == 3840 else 16
        imgs = (torch.randn((n, h, w, 4), device=dev) * 40 + 128).clamp_(0, 255).to(torch.uint8)
        outs = torch.empty((n, w, h, 4), dtype=torch.uint8, device=dev)
        ops = {
            "transpose": lambda i: batch.transpose(ifb.BitmapWindow.from_torch(imgs[i]), ifb.BitmapWindow.from_torch(outs[i]), stream),
            "flip_vertical": lambda i: batch.flip_vertical(ifb.BitmapWindow.from_torch(imgs[i]), stream),
            "flip_horizontal": lambda i: batch.flip_horizontal(ifb.BitmapWindow.from_torch(imgs[i]), stream),
            "white_balance": lambda i: batch.white_balance(ifb.BitmapWindow.from_torch(imgs[i]), None, stream),
        }
        host = np.random.default_rng(1).normal(128, 40, (h, w, 4)).clip(0, 255).astype(np.uint8)      # a bell-shaped histogram
        for name, fn in ops.items():
            for i in range(n):          # warm-up: every image once
                fn(i)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 3
            e0.record()
            for _ in range(reps):
                for i in range(n):
                    fn(i)
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / (reps * n)
            alg = w * h * (12 if name == "white_balance" else 8)   # white balance: histogram pass (4 B/px) + remap pass (4 + 4 B/px)
            # parity spot check + CPU time of the oracle loop
            t0 = time.perf_counter()
            if name == "transpose":
                exp = np.zeros((w, h, 4), np.uint8); oracle.transpose(host, exp)
            elif name == "white_balance":
                exp = host.copy(); oracle.white_balance(exp)
            else:
                exp = host.copy(); (oracle.flip_vertical if name == "flip_vertical" else oracle.flip_horizontal)(exp)
            cpu_ms = (time.perf_counter() - t0) * 1e3
            d = torch.from_numpy(host).to(dev)
            if name == "transpose":
                o = torch.empty((w, h, 4), dtype=torch.uint8, device=dev)
                batch.transpose(ifb.BitmapWindow.from_torch(d), ifb.BitmapWindow.from_torch(o), stream); got = o
            elif name == "white_balance":
                batch.white_balance(ifb.BitmapWindow.from_torch(d), None, stream); got = d
            else:
                (batch.flip_vertical if name == "flip_vertical" else batch.flip_horizontal)(ifb.BitmapWindow.from_torch(d), stream); got = d
            torch.cuda.synchronize()
            ok = bool(np.array_equal(got.cpu().numpy(), exp))
            print(json.dumps({"op": name, "size": f"{w}x{h}", "ms_per_image": ms, "mpx_per_s": w * h / ms / 1e3,
                              "roofline": {"bound": "hbm", "achieved": alg / ms / 1e6, "peak": pk, "unit": "GB/s", "frac": alg / ms / 1e6 / pk,
                                           "peak_source": src, "algorithmic_bytes_per_launch": alg},
                              "cpu_oracle_ms_1_thread": cpu_ms, "bit_exact_vs_oracle": ok, "images_cycled": n}))
        # detect_content (graphics/whitespace.rs:284-331): the code kernel (4 B read + 1 B written per pixel) timed alone with CUDA
        # events, the whole call (kernel + 1 B/px device->host + the reference's window walk on the host) by wall clock, the host
        # walk alone over the same map, and the oracle's scalar loop.  Content: a noisy rectangle on a white page (the trim case).
        page = np.full((h, w, 4), 255, np.uint8)
        page[h // 8: h - h // 6, w // 10: w - w // 7] = host[h // 8: h - h // 6, w // 10: w - w // 7]
        for i in range(n):
            imgs[i].copy_(torch.from_numpy(page))
            imgs[i, :, :, 0].add_(i & 1)                      # cycled images are not identical (white wraps to 0 on odd ones)
        codes = torch.empty((n, h, w), dtype=torch.uint8, device=dev)
        wfn = lambda i: batch.whitespace_codes(ifb.BitmapWindow.from_torch(imgs[i]), codes[i].data_ptr(), 1, stream)
        for i in range(n):
            wfn(i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(3):
            for i in range(n):
                wfn(i)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / (3 * n)
        batch.detect_content(ifb.BitmapWindow.from_torch(imgs[0]), 1, stream)
        t0 = time.perf_counter()
        for i in range(8):
            rect = batch.detect_content(ifb.BitmapWindow.from_torch(imgs[2 * i]), 1, stream)
        call_ms = (time.perf_counter() - t0) * 1e3 / 8
        hc = codes[0].cpu().numpy()
        t0 = time.perf_counter()
        for _ in range(8):
            rect_w, visited = ifb.detect_content_from_codes(hc)
        walk_ms = (time.perf_counter() - t0) * 1e3 / 8
        t0 = time.perf_counter()
        want, _ = oracle.detect_content(imgs[0].cpu().numpy(), 1, True)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        alg = w * h * 5
        print(json.dumps({"op": "detect_content", "size": f"{w}x{h}", "code_kernel_ms_per_image": ms, "mpx_per_s_kernel": w * h / ms / 1e3,
                          "roofline": {"bound": "hbm", "achieved": alg / ms / 1e6, "peak": pk, "unit": "GB/s", "frac": alg / ms / 1e6 / pk,
                                       "peak_source": src, "algorithmic_bytes_per_launch": alg},
                          "whole_call_ms": call_ms, "host_walk_ms": walk_ms, "host_walk_pixels_visited": visited,
                          "cpu_oracle_ms_1_thread": cpu_ms, "rect": list(rect), "bit_exact_vs_oracle": bool(tuple(rect) == tuple(want) == tuple(rect_w)),
                          "images_cycled": n}))
        if w == 3840:
            round_corners_rows(batch, imgs, host, stream, pk, src)
        del imgs, outs, codes
        torch.cuda.empty_cache()


def round_corners_rows(batch, imgs, host, stream, pk, src):
    """graphics/rounded_corners.rs on 4K frames: the op touches a few rectangles per frame, so per image it is far below a launch's
    cost; the rows compare one batch call over 64 images (one launch) with 64 one-image calls, time the drop-in call (only the
    planned rectangles travel) by wall clock against the oracle's loop on one host thread, and check the result bit for bit.
    Algorithmic bytes: 4 written per pixel filled with the matte, 4 read + 4 written per blended pixel (the oracle's touch mask)."""
    from tests import round_corners_oracle as rco
    rco.lib()                                          # compiled on first use: not part of the oracle's time
    n, h, w = imgs.shape[0], imgs.shape[1], imgs.shape[2]
    matte = (20, 40, 60, 255)
    for label, mode in (("pixels_100", ifb.RoundCornersMode.pixels(100)), ("circle", ifb.RoundCornersMode.circle())):
        wins = [ifb.BitmapWindow.from_torch(imgs[i]) for i in range(n)]
        one_call = lambda: batch.round_corners([(wn, mode, matte) for wn in wins], stream)
        per_image = lambda: [batch.round_corners([(wn, mode, matte)], stream) for wn in wins]
        times = {}
        for name, fn in (("batch_64_one_call", one_call), ("64_one_image_calls", per_image)):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            reps = 10
            e0.record()
            for _ in range(reps):
                fn()
            e1.record(); torch.cuda.synchronize()
            times[name] = e0.elapsed_time(e1) / reps
        exp = host.copy()
        t0 = time.perf_counter()
        mask = rco.round_corners(exp, mode.kind, mode.radius, matte, want_mask=True)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        filled, blended = int((mask == 1).sum()), int((mask == 2).sum())
        alg = 4 * filled + 8 * blended
        d = torch.from_numpy(host).to(imgs.device)
        batch.round_corners([(ifb.BitmapWindow.from_torch(d), mode, matte)], stream)
        torch.cuda.synchronize()
        ok_batch = bool(np.array_equal(d.cpu().numpy(), exp))
        hw = host.copy()
        win = ifb.BitmapWindow.from_numpy(hw)
        ifb.flow_bitmap_bgra_clear_around_rounded_corners(win, mode, matte)
        ok_drop = bool(np.array_equal(hw, exp))
        drop = []
        for _ in range(5):
            hw[...] = host
            t0 = time.perf_counter()
            ifb.flow_bitmap_bgra_clear_around_rounded_corners(win, mode, matte)
            drop.append((time.perf_counter() - t0) * 1e3)
        ms = times["batch_64_one_call"] / n
        print(json.dumps({"op": "round_corners", "mode": label, "size": f"{w}x{h}", "pixels_filled": filled, "pixels_blended": blended,
                          "batch_64_one_call_ms": times["batch_64_one_call"], "64_one_image_calls_ms": times["64_one_image_calls"],
                          "ms_per_image_in_batch": ms, "mpx_touched_per_s": (filled + blended) / ms / 1e3,
                          "roofline": {"bound": "hbm", "achieved": alg / ms / 1e6, "peak": pk, "unit": "GB/s", "frac": alg / ms / 1e6 / pk,
                                       "peak_source": src, "algorithmic_bytes_per_image": alg},
                          "drop_in_wall_ms_median": float(np.median(drop)), "cpu_oracle_ms_1_thread": cpu_ms,
                          "bit_exact_vs_oracle": ok_batch and ok_drop, "images_per_batch": n}))


def _card():
    """the card's name and power limit, read in the same run as the numbers"""
    import subprocess
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                            timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return {"gpu": torch.cuda.get_device_name(0), "power_limit": pl}


def _time_ms(fn, reps=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def _copy_ceiling_ms(alg_bytes):
    """a torch device-to-device copy that moves alg_bytes in all (alg_bytes / 2 read, alg_bytes / 2 written)"""
    n = max(alg_bytes // 2, 1)
    a = torch.empty(n, dtype=torch.uint8, device="cuda"); b = torch.empty_like(a)
    ms = _time_ms(lambda: b.copy_(a))
    del a, b
    return ms


def canvas_rows():
    """Canvas operations (Batch.canvas) on frames resident in HBM.  Algorithmic bytes: 4 written per canvas pixel plus 4 read per
    copied pixel.  Each row also times a torch device-to-device copy of the same number of bytes as a practical ceiling."""
    card = _card()
    pk, src = peak()
    b = ifb.Batch(0)
    stream = torch.cuda.current_stream().cuda_stream

    def row(name, ms, alg, **kw):
        cm = _copy_ceiling_ms(alg)
        print(json.dumps({"op": "canvas", "row": name, "ms": ms, "algorithmic_bytes": alg, "achieved_gbs": alg / ms / 1e6,
                          "frac_of_peak": alg / ms / 1e6 / pk, "peak_gbs": pk, "peak_source": src, "torch_copy_same_bytes_ms": cm,
                          "frac_of_torch_copy": cm / ms, **kw, **card}))

    # ExpandCanvas: 64 x 3840x2160 -> 3840x2880, opaque colour, one call
    n, w, h, H = 64, 3840, 2160, 2880
    ins = (torch.randn((n, h, w, 4), device="cuda") * 40 + 128).clamp_(0, 255).to(torch.uint8)
    outs = torch.empty((n, H, w, 4), dtype=torch.uint8, device="cuda")
    iw = [ifb.BitmapWindow.from_torch(ins[i]) for i in range(n)]
    ow = [ifb.BitmapWindow.from_torch(outs[i]) for i in range(n)]
    top = (H - h) // 2
    ops = [ifb.ExpandCanvas(iw[i], 0, top, 0, H - h - top, (10, 20, 30, 255), canvas=ow[i]) for i in range(n)]
    ms = _time_ms(lambda: b.canvas(ops, stream))
    want = torch.full((H - h - top, w, 4), 0, dtype=torch.uint8, device="cuda"); want[...] = torch.tensor((10, 20, 30, 255), dtype=torch.uint8)
    ok = bool(torch.equal(outs[5, top:top + h], ins[5]) and torch.equal(outs[5, top + h:], want))
    row("expand_64x3840x2160_to_3840x2880_one_call", ms, n * (4 * w * H + 4 * w * h), frames=n, spot_check_ok=ok)
    del ins, outs, iw, ow, ops
    torch.cuda.empty_cache()

    # padded thumbnails: 1024 x 512x288 -> 512x512, one call and 1024 calls
    n, w, h, H = 1024, 512, 288, 512
    ins = torch.randint(0, 256, (n, h, w, 4), dtype=torch.uint8, device="cuda")
    outs = torch.empty((n, H, w, 4), dtype=torch.uint8, device="cuda")
    top = (H - h) // 2
    ops = [ifb.ExpandCanvas(ifb.BitmapWindow.from_torch(ins[i]), 0, top, 0, H - h - top, (255, 255, 255, 255),
                            canvas=ifb.BitmapWindow.from_torch(outs[i])) for i in range(n)]
    alg = n * (4 * w * H + 4 * w * h)
    row("pad_1024x512x288_to_512x512_one_call", _time_ms(lambda: b.canvas(ops, stream)), alg, frames=n)
    row("pad_1024x512x288_to_512x512_1024_calls", _time_ms(lambda: [b.canvas([o], stream) for o in ops], reps=3), alg, frames=n)
    ok = bool(torch.equal(outs[7, top:top + h], ins[7]))
    # WatermarkRedDot on the 1024 padded frames
    dots = [op for i in range(n) for op in ifb.watermark_red_dot(ifb.BitmapWindow.from_torch(outs[i]))]
    row("red_dot_1024_frames_one_call", _time_ms(lambda: b.canvas(dots, stream)), n * 9 * 4, frames=n, spot_check_ok=ok)
    row("red_dot_1024_frames_1024_calls", _time_ms(lambda: [b.canvas([o], stream) for o in dots], reps=3), n * 9 * 4, frames=n)
    del ins, outs, ops, dots
    torch.cuda.empty_cache()

    # mode=pad at config 2 (3840x2160 -> 512x288 Robidoux, linear light, then 512x512): (a) resample + EXPAND, (b) resample into the
    # interior + border FILL_RECTs.  The rows time the whole pipeline; bytes are the resample's (4K read, 512x288 written) plus the pad's.
    n = 64
    ins = (torch.randn((n, 2160, 3840, 4), device="cuda") * 40 + 128).clamp_(0, 255).to(torch.uint8)
    mid = torch.empty((n, 288, 512, 4), dtype=torch.uint8, device="cuda")
    pa = torch.empty((n, 512, 512, 4), dtype=torch.uint8, device="cuda")
    pb = torch.empty((n, 512, 512, 4), dtype=torch.uint8, device="cuda")
    params = ifb.ScaleAndRenderParams(w=512, h=288)
    srcs = [ifb.BitmapWindow.from_torch(ins[i]) for i in range(n)]
    mids = [ifb.BitmapWindow.from_torch(mid[i]) for i in range(n)]
    descs_a, keep_a = b.make_descs([(srcs[i], mids[i], params) for i in range(n)])
    exp_a = [ifb.ExpandCanvas(mids[i], 0, 112, 0, 112, (9, 99, 199, 77), canvas=ifb.BitmapWindow.from_torch(pa[i])) for i in range(n)]
    descs_b, keep_b = b.make_descs([(srcs[i], ifb.BitmapWindow.from_torch(pb[i]).window(0, 112, 512, 400), params) for i in range(n)])
    fills_b = [f for i in range(n) for f in (ifb.FillRect(ifb.BitmapWindow.from_torch(pb[i]), 0, 0, 512, 112, (9, 99, 199, 77)),
                                             ifb.FillRect(ifb.BitmapWindow.from_torch(pb[i]), 0, 400, 512, 512, (9, 99, 199, 77)))]
    route_a = lambda: (b.enqueue(descs_a, stream), b.canvas(exp_a, stream))
    route_b = lambda: (b.enqueue(descs_b, stream), b.canvas(fills_b, stream))
    base = n * (3840 * 2160 * 4)
    ms_a, ms_b = _time_ms(route_a), _time_ms(route_b)
    same = bool(torch.equal(pa, pb))
    row("mode_pad_config2_route_a_resample_then_expand", ms_a, base + n * (288 * 512 * 4 + 512 * 512 * 4 + 288 * 512 * 4), frames=n,
        routes_agree=same)
    row("mode_pad_config2_route_b_resample_into_interior_then_fill", ms_b, base + n * 512 * 512 * 4, frames=n, routes_agree=same)
    b.sync()


def _time_event_and_host_ms(fn, reps=10):
    """(CUDA-event time on the current stream, host wall time spent inside fn) per call of fn, after 3 warm-up calls"""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    host = 0.0
    e0.record()
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        host += time.perf_counter() - t0
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, host * 1e3 / reps


def orient_rows():
    """Orientation (Batch.orient) on frames resident in HBM: 64 3840x2160 frames in one call for each of flags 2..8, against the
    reference's expansion of the same flag with the existing single-window transpose and flip calls (one launch and one full pass per
    node, in place for the flips, as the reference runs them), and against a torch device-to-device copy of the same bytes.
    Algorithmic bytes: 4 read + 4 written per pixel; the 64 frames (2.1 GB) are cycled, far larger than L2.  Then 1024 512x384
    thumbnails in one call and as 1024 calls, with the CUDA-event time on the stream and the host wall time of the calls apart."""
    from tests import orient_oracle as oo
    card = _card()
    pk, src = peak()
    b = ifb.Batch(0)
    stream = torch.cuda.current_stream().cuda_stream

    def row(name, ms, alg, **kw):
        cm = _copy_ceiling_ms(alg)
        print(json.dumps({"op": "orient", "row": name, "ms": ms, "algorithmic_bytes": alg, "achieved_gbs": alg / ms / 1e6,
                          "frac_of_peak": alg / ms / 1e6 / pk, "peak_gbs": pk, "peak_source": src, "torch_copy_same_bytes_ms": cm,
                          "frac_of_torch_copy": cm / ms, **kw, **card}), flush=True)

    n, w, h = 64, 3840, 2160
    ins = torch.randint(0, 256, (n, h, w, 4), dtype=torch.uint8, device="cuda")
    same = torch.empty((n, h, w, 4), dtype=torch.uint8, device="cuda")
    swapped = torch.empty((n, w, h, 4), dtype=torch.uint8, device="cuda")
    iw = [ifb.BitmapWindow.from_torch(ins[i]) for i in range(n)]
    sw = [ifb.BitmapWindow.from_torch(same[i]) for i in range(n)]
    tw = [ifb.BitmapWindow.from_torch(swapped[i]) for i in range(n)]
    alg = n * w * h * 8

    def expansion(i, flag):
        """ApplyOrientation(flag) of frame i node by node (the flips in place on the frame, the transpose into `swapped`)"""
        cur, t = iw[i], False
        for p in oo.primitives([("ApplyOrientation", flag)]):
            if p == oo.TRANSPOSE:
                b.transpose(cur, tw[i], stream); cur, t = tw[i], True
            else:
                (b.flip_horizontal if p == oo.FLIP_H else b.flip_vertical)(cur, stream)
        return t

    for flag in range(2, 9):
        t = flag >= 5
        outs = tw if t else sw
        jobs = [(iw[i], outs[i], flag) for i in range(n)]
        ms_one = _time_ms(lambda: b.orient(jobs, stream))
        nodes = len(oo.primitives([("ApplyOrientation", flag)]))
        ms_exp = _time_ms(lambda: [expansion(i, flag) for i in range(n)])
        # bit-exactness of frame 0: the one call against the expansion on a copy
        keep = ins[0].clone()
        b.orient([(iw[0], outs[0], flag)], stream)
        got = (swapped if t else same)[0].clone()
        expansion(0, flag)
        want = swapped[0].clone() if t else ins[0].clone()
        ins[0].copy_(keep)
        ok = bool(torch.equal(got, want))
        kw = dict(flag=flag, frames=n, size=f"{w}x{h}", expansion_nodes=nodes, expansion_ms=ms_exp, one_call_vs_expansion=ms_exp / ms_one,
                  bit_exact_vs_expansion=ok)
        if not t:
            kw["in_place_ms"] = _time_ms(lambda: b.orient([(iw[i], None, flag) for i in range(n)], stream))
        row(f"flag{flag}_64x{w}x{h}_one_call", ms_one, alg, **kw)
    del ins, same, swapped, iw, sw, tw
    torch.cuda.empty_cache()

    # thumbnails: 1024 x 512x384 with flag 6, one call and 1024 calls
    n, w, h = 1024, 512, 384
    ins = torch.randint(0, 256, (n, h, w, 4), dtype=torch.uint8, device="cuda")
    outs = torch.empty((n, w, h, 4), dtype=torch.uint8, device="cuda")
    jobs = [(ifb.BitmapWindow.from_torch(ins[i]), ifb.BitmapWindow.from_torch(outs[i]), 6) for i in range(n)]
    alg = n * w * h * 8
    ev, host = _time_event_and_host_ms(lambda: b.orient(jobs, stream))
    row("flag6_1024x512x384_one_call", ev, alg, frames=n, host_wall_ms=host)
    ev, host = _time_event_and_host_ms(lambda: [b.orient([j], stream) for j in jobs], reps=3)
    row("flag6_1024x512x384_1024_calls", ev, alg, frames=n, host_wall_ms=host)
    want = torch.from_numpy(oo.gather(ins[7].cpu().numpy(), 6)).cuda()
    print(json.dumps({"op": "orient", "row": "thumbnail_spot_check", "bit_exact_vs_closed_form": bool(torch.equal(outs[7], want)), **card}))
    b.sync()


def color_rows():
    """Colour chains (Batch.color_chain) on frames resident in HBM: 64 3840x2160 frames per call (2.1 GB, cycled, far larger than L2)
    for RIAPI chains on both sides of the planner's table-or-matrix choice, against the reference's node-by-node expansion with the
    existing single-window calls (ColorMatrixSrgb per step, EnableTransparency through Batch.canvas, Batch.white_balance), and against
    a torch device-to-device copy of the same algorithmic bytes: 4 read + 4 written per pixel, plus 4 read with white balance.  Both
    the one call and the expansion are timed in five trials: the median, and the smallest and largest.  Each row checks frame 0 of the one call against the expansion, bit for bit.  Then 1024 512x384 thumbnails with row (a) in one call,
    with the CUDA-event time and the host wall time inside the call apart."""
    card = _card()
    pk, src = peak()
    b = ifb.Batch(0)
    stream = torch.cuda.current_stream().cuda_stream

    def row(name, ms, alg, **kw):
        cm = _copy_ceiling_ms(alg)
        print(json.dumps({"op": "color", "row": name, "ms": ms, "algorithmic_bytes": alg, "achieved_gbs": alg / ms / 1e6,
                          "frac_of_peak": alg / ms / 1e6 / pk, "peak_gbs": pk, "peak_source": src, "torch_copy_same_bytes_ms": cm,
                          "frac_of_torch_copy": cm / ms, **kw, **card}), flush=True)

    def expansion(win, steps, am):
        win.alpha_meaningful = am
        for s in steps:
            if isinstance(s, ifb.ColorMatrixSrgb):
                b.color_matrix(win.ptr, win.w, win.h, win.stride, s.matrix, stream)
            elif isinstance(s, ifb.EnableTransparency):
                if not win.alpha_meaningful:
                    b.canvas([ifb.EnableTransparency(win)], stream)
            else:
                b.white_balance(win, s.threshold, stream)

    def one_call(wins, steps, am):
        for w in wins:
            w.alpha_meaningful = am
        b.color_chain([(w, steps) for w in wins], stream)

    n, w, h = 64, 3840, 2160
    frames = (torch.randn((n, h, w, 4), device="cuda") * 40 + 128).clamp_(0, 255).to(torch.uint8)
    wins = [ifb.BitmapWindow.from_torch(frames[i]) for i in range(n)]
    rows = [("a_brightness_contrast_table", dict(brightness=0.1, contrast=0.2), True),
            ("b_saturation_sepia_matrix", dict(saturation=-0.5, sepia=True), True),
            ("c_alpha_on_bgr32", dict(alpha=0.5), False),
            ("d_all_seven_keys", dict(alpha=0.5, brightness=0.1, contrast=0.2, saturation=-0.3, sepia=True, grayscale="true",
                                      balance_white=True), False),
            ("e_balancewhite", dict(balance_white=True), True)]
    for name, keys, am in rows:
        steps = ifb.riapi_color_steps(**keys)
        wb = any(isinstance(s, ifb.WhiteBalanceHistogramAreaThresholdSrgb) for s in steps)
        before = b.kernel_launches
        one_call(wins, steps, am)
        launches = b.kernel_launches - before
        # five trials each: the expansion is bound by host time (each ColorMatrixSrgb call stages its matrix and allocates on the
        # stream) and varies from trial to trial, so its spread is reported with the median
        one = sorted(_time_ms(lambda: one_call(wins, steps, am)) for _ in range(5))
        exp = sorted(_time_ms(lambda: [expansion(wn, steps, am) for wn in wins], reps=3) for _ in range(5))
        ms_one, ms_exp = one[2], exp[2]
        keep = frames[0].clone()
        one_call(wins[:1], steps, am)
        got = frames[0].clone()
        frames[0].copy_(keep)
        expansion(wins[0], steps, am)
        ok = bool(torch.equal(got, frames[0]))
        row(f"{name}_64x{w}x{h}_one_call", ms_one, n * w * h * (12 if wb else 8), frames=n, size=f"{w}x{h}", keys=keys,
            steps=len(steps), launches_per_call=launches, one_call_ms_min_max=[one[0], one[-1]], expansion_ms=ms_exp,
            expansion_ms_min_max=[exp[0], exp[-1]], one_call_vs_expansion=ms_exp / ms_one,
            one_call_vs_expansion_range=[exp[0] / one[-1], exp[-1] / one[0]], bit_exact_vs_expansion=ok)
    del frames, wins
    torch.cuda.empty_cache()

    n, w, h = 1024, 512, 384
    thumbs = torch.randint(0, 256, (n, h, w, 4), dtype=torch.uint8, device="cuda")
    twins = [ifb.BitmapWindow.from_torch(thumbs[i], alpha_meaningful=True) for i in range(n)]
    steps = ifb.riapi_color_steps(brightness=0.1, contrast=0.2)
    ev, host = _time_event_and_host_ms(lambda: b.color_chain([(wn, steps) for wn in twins], stream))
    keep = thumbs[7].clone()
    b.color_chain([(twins[7], steps)], stream)
    got = thumbs[7].clone()
    thumbs[7].copy_(keep)
    expansion(twins[7], steps, True)
    row(f"a_brightness_contrast_table_{n}x{w}x{h}_one_call", ev, n * w * h * 8, frames=n, host_wall_ms=host,
        bit_exact_vs_expansion=bool(torch.equal(got, thumbs[7])))
    b.sync()


def _device_ms(fn, reps=10):
    """GPU time per call of fn: the durations of every kernel and copy it enqueues, summed over a torch.profiler trace of reps calls"""
    from torch.profiler import ProfilerActivity, profile
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    us = sum(getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0) for e in prof.key_averages())
    return us / 1e3 / reps


def watermark_rows():
    """Watermarks (Batch.watermark) on frames resident in HBM, each route timed in five trials (median, smallest, largest).
    (a) 1024 512x512 thumbnails, a 400x100 cut-out logo, Within into ImagePercentage(0, 0, 90, 90), gravity (100, 100), opacity 0.9
        (visuals/watermark.rs test_watermark_image_small): one call; the node-by-node expansion (per frame a copy of the logo, the Alpha
        chain on it, one resample); and the best existing route (the Alpha chain once on one copy, then ONE batch_enqueue of 1024 jobs
        whose descriptors are built beforehand).  The host wall time inside the one call is reported apart.
    (b) 64 3840x2160 frames, each with a 1920x1080 watermark fitted to the whole canvas (CanvasPercentage(0, 0, 100, 100), Fit): one
        call and one batch_enqueue of the 64 draws, against a torch copy of the algorithmic bytes, 8 per composited pixel (4 read, 4
        written).  F (16 bytes per pixel, written once and read once per frame) is reported apart.
    Each row checks a frame of the one call against the other route, bit for bit."""
    card = _card()
    pk, src = peak()
    b = ifb.Batch(0)
    stream = torch.cuda.current_stream().cuda_stream
    M, B, G = ifb.WatermarkConstraintMode, ifb.WatermarkConstraintBox, ifb.ConstraintGravity
    from imageflow_b200 import synth

    def trials(fn, reps):
        t = sorted(_time_ms(fn, reps=reps) for _ in range(5))
        return t[2], [t[0], t[-1]]

    # (a)
    n, fw = 1024, 512
    frames = torch.randint(0, 256, (n, fw, fw, 4), dtype=torch.uint8, device="cuda")
    base = frames.clone()
    logo = synth.cutout_torch(400, 100, 3)
    spec = ifb.Watermark(fit_box=B.image_percentage(0, 0, 90, 90), fit_mode=M.Within, gravity=G.percentage(100, 100), opacity=0.9)
    wins = [ifb.BitmapWindow.from_torch(frames[i]) for i in range(n)]
    lw = ifb.BitmapWindow.from_torch(logo, alpha_meaningful=True)
    draw = ifb.watermark_layout(fw, fw, 400, 100, spec)
    params = ifb.ScaleAndRenderParams(x=draw.x, y=draw.y, w=draw.w, h=draw.h, interpolation_filter=draw.filter)

    def one_call():
        for w in wins:
            w.compose = ifb.BitmapCompositing.BlendWithSelf
        b.watermark([(w, lw, spec) for w in wins], stream)

    def expansion():
        for w in wins:
            c = logo.clone()
            cw = ifb.BitmapWindow.from_torch(c, alpha_meaningful=True)
            b.color_chain([(cw, ifb.ColorFilterSrgb.alpha(draw.opacity))], stream)
            w.compose = ifb.BitmapCompositing.BlendWithSelf
            b.scale_and_render_many([(cw, w, params)], stream)

    copy = logo.clone()
    cwin = ifb.BitmapWindow.from_torch(copy, alpha_meaningful=True)
    for w in wins:
        w.compose = ifb.BitmapCompositing.BlendWithSelf
    descs, keep = b.make_descs([(cwin, w, params) for w in wins])

    def best_existing():
        copy.copy_(logo)
        b.color_chain([(cwin, ifb.ColorFilterSrgb.alpha(draw.opacity))], stream)
        b.enqueue(descs, stream)

    prepared = b.make_watermark_descs([(w, lw, spec) for w in wins])

    def library_call():                                      # the library alone: descriptors built beforehand, as best_existing's
        for w in wins:
            w.compose = ifb.BitmapCompositing.BlendWithSelf
        b.watermark_enqueue(prepared, stream)

    before = b.kernel_launches
    one_call()
    launches = b.kernel_launches - before
    ms_one, mm_one = trials(one_call, 10)
    ms_lib, mm_lib = trials(library_call, 10)
    host_lib = sorted(_time_event_and_host_ms(library_call)[1] for _ in range(5))[2]
    host = sorted(_time_event_and_host_ms(one_call)[1] for _ in range(5))[2]
    ms_exp, mm_exp = trials(expansion, 1)
    ms_best, mm_best = trials(best_existing, 10)
    # device time alone (kernels and copies, summed from a torch.profiler trace taken after the timed trials): row (a) is bound by host
    # time on every route, so the event times above do not show what the GPU spends
    dev_one, dev_best = _device_ms(one_call), _device_ms(best_existing)
    frames.copy_(base); one_call(); got = frames.clone()
    frames.copy_(base); best_existing(); ok = bool(torch.equal(got, frames))
    alg = n * draw.w * draw.h * 8
    print(json.dumps({"op": "watermark", "row": f"a_{n}x{fw}x{fw}_logo_400x100_within_90pct_opacity_0.9", "one_call_ms": ms_one,
                      "one_call_ms_min_max": mm_one, "host_wall_ms_inside_one_call": host,
                      "prebuilt_descriptors_call_ms": ms_lib, "prebuilt_descriptors_call_ms_min_max": mm_lib,
                      "host_wall_ms_inside_prebuilt_call": host_lib, "prebuilt_call_vs_best_existing": ms_best / ms_lib, "expansion_ms": ms_exp,
                      "expansion_ms_min_max": mm_exp, "best_existing_ms": ms_best, "best_existing_ms_min_max": mm_best,
                      "one_call_vs_best_existing": ms_best / ms_one,
                      "device_ms_one_call": dev_one, "device_ms_best_existing": dev_best, "one_call_vs_expansion": ms_exp / ms_one, "launches_per_call": launches,
                      "draw": [draw.x, draw.y, draw.w, draw.h], "algorithmic_bytes": alg, "bit_exact_vs_best_existing": ok, **card}), flush=True)
    del frames, base, wins, descs, keep
    torch.cuda.empty_cache()

    # (b)
    n, w, h = 64, 3840, 2160
    frames = (torch.randn((n, h, w, 4), device="cuda") * 40 + 128).clamp_(0, 255).to(torch.uint8)
    wm = synth.cutout_torch(1920, 1080, 5)
    spec = ifb.Watermark(fit_box=B.canvas_percentage(0, 0, 100, 100), fit_mode=M.Fit)
    wins = [ifb.BitmapWindow.from_torch(frames[i]) for i in range(n)]
    ww = ifb.BitmapWindow.from_torch(wm, alpha_meaningful=True)
    draw = ifb.watermark_layout(w, h, 1920, 1080, spec)
    params = ifb.ScaleAndRenderParams(x=draw.x, y=draw.y, w=draw.w, h=draw.h, interpolation_filter=draw.filter)
    for x in wins:
        x.compose = ifb.BitmapCompositing.BlendWithSelf
    descs, keep = b.make_descs([(ww, x, params) for x in wins])

    def one_call_b():
        for x in wins:
            x.compose = ifb.BitmapCompositing.BlendWithSelf
        b.watermark([(x, ww, spec) for x in wins], stream)

    ms_one, mm_one = trials(one_call_b, 3)
    ms_enq, mm_enq = trials(lambda: b.enqueue(descs, stream), 3)
    keep0 = frames[0].clone()
    one_call_b(); got = frames[0].clone(); frames[0].copy_(keep0)
    d0, k0 = b.make_descs([(ww, wins[0], params)])
    b.enqueue(d0, stream); ok = bool(torch.equal(got, frames[0]))
    alg = n * draw.w * draw.h * 8
    cm = _copy_ceiling_ms(alg)
    print(json.dumps({"op": "watermark", "row": f"b_{n}x{w}x{h}_watermark_1920x1080_fit_canvas", "one_call_ms": ms_one,
                      "one_call_ms_min_max": mm_one, "batch_enqueue_ms": ms_enq, "batch_enqueue_ms_min_max": mm_enq,
                      "one_call_vs_batch_enqueue": ms_enq / ms_one, "algorithmic_bytes": alg, "achieved_gbs": alg / ms_one / 1e6,
                      "frac_of_peak": alg / ms_one / 1e6 / pk, "peak_gbs": pk, "peak_source": src, "torch_copy_same_bytes_ms": cm,
                      "frac_of_torch_copy": cm / ms_one, "f_bytes_written_once": draw.w * draw.h * 16,
                      "f_bytes_read_per_call": n * draw.w * draw.h * 16, "draw": [draw.x, draw.y, draw.w, draw.h],
                      "bit_exact_vs_batch_enqueue": ok, **card}), flush=True)
    b.sync()


def formats_rows():
    """Pixel-format conversions (Batch.pixel_convert) on rows resident in HBM: 64 3840x2160 frames in one call for each op, each timed
    in five trials (median, smallest, largest) with the 64 frames (>= 1.6 GB) cycled, far larger than L2.  Algorithmic bytes per pixel:
    7 for RGB24 <-> BGRA, 5 for Gray8, 6 for GrayAlpha8, 8 for RGBA <-> BGRA and the in-place swap.  Each row also times a torch
    device-to-device copy of the same bytes and the torch expression a user would write today (a channel index, plus a cat with a
    255 plane where the output gains an alpha), and checks frame 0 of the call against that expression, bit for bit.  Then 1024 512x384
    RGB24 thumbnails in one call and as 1024 calls, with the CUDA-event time on the stream and the host wall time of the calls apart."""
    card = _card()
    pk, src = peak()
    b = ifb.Batch(0)
    stream = torch.cuda.current_stream().cuda_stream
    n, w, h = 64, 3840, 2160
    sbuf = torch.randint(0, 256, (n * h * w * 4,), dtype=torch.uint8, device="cuda")
    dbuf = torch.empty(n * h * w * 4, dtype=torch.uint8, device="cuda")

    def trials(fn, reps=10):
        t = sorted(_time_ms(fn, reps) for _ in range(5))
        return t[2], t[0], t[-1]

    def full255(x):
        return torch.full(x.shape[:-1] + (1,), 255, dtype=torch.uint8, device="cuda")

    ops = [  # (row, record, source channels, destination channels, torch expression)
        ("rgb24_to_bgra", ifb.RgbToBgra, 3, 4, lambda x: torch.cat([x[..., [2, 1, 0]], full255(x)], -1)),
        ("rgba_to_bgra", ifb.RgbaToBgra, 4, 4, lambda x: x[..., [2, 1, 0, 3]]),
        ("gray_to_bgra", ifb.GrayToBgra, 1, 4, lambda x: torch.cat([x[..., [0, 0, 0]], full255(x)], -1)),
        ("gray_alpha_to_bgra", ifb.GrayAlphaToBgra, 2, 4, lambda x: x[..., [0, 0, 0, 1]]),
        ("bgra_to_rgb24", ifb.BgraToRgb, 4, 3, lambda x: x[..., [2, 1, 0]]),
    ]
    for name, rec, cs, cd, expr in ops:
        x = sbuf[:n * h * w * cs].view(n, h, w, cs)
        y = dbuf[:n * h * w * cd].view(n, h, w, cd)
        jobs = [rec(x[i], y[i]) for i in range(n)]
        alg = n * w * h * (cs + cd)
        ms, lo, hi = trials(lambda: b.pixel_convert(jobs, stream))
        _, host = _time_event_and_host_ms(lambda: b.pixel_convert(jobs, stream), reps=3)
        ms_torch, _, _ = trials(lambda: expr(x), reps=3)
        b.pixel_convert(jobs[:1], stream)
        ok = bool(torch.equal(y[0], expr(x[:1])[0]))
        cm = _copy_ceiling_ms(alg)
        print(json.dumps({"op": "formats", "row": f"{name}_64x{w}x{h}_one_call", "ms": ms, "ms_min": lo, "ms_max": hi,
                          "host_wall_ms": host, "algorithmic_bytes": alg, "achieved_gbs": alg / ms / 1e6, "frac_of_peak": alg / ms / 1e6 / pk,
                          "peak_gbs": pk, "peak_source": src, "torch_copy_same_bytes_ms": cm, "frac_of_torch_copy": cm / ms,
                          "torch_expression_ms": ms_torch, "vs_torch_expression": ms_torch / ms, "bit_exact_vs_torch_expression": ok,
                          **card}), flush=True)
    # in place, opaque: the encoders' swap then fill-alpha in one pass
    x = dbuf.view(n, h, w, 4)
    x.copy_(sbuf.view(n, h, w, 4))
    jobs = [ifb.RgbaToBgra(ifb.BitmapWindow.from_torch(x[i]), None, True) for i in range(n)]
    alg = n * w * h * 8
    ms, lo, hi = trials(lambda: b.pixel_convert(jobs, stream))

    def torch_in_place(t):
        t[..., :3] = t[..., [2, 1, 0]]
        t[..., 3] = 255
    ms_torch, _, _ = trials(lambda: torch_in_place(x), reps=3)
    x.copy_(sbuf.view(n, h, w, 4))
    b.pixel_convert(jobs[:1], stream)
    want = sbuf.view(n, h, w, 4)[0].clone()
    torch_in_place(want)
    ok = bool(torch.equal(x[0], want))
    cm = _copy_ceiling_ms(alg)
    print(json.dumps({"op": "formats", "row": f"rgba_to_bgra_in_place_opaque_64x{w}x{h}_one_call", "ms": ms, "ms_min": lo, "ms_max": hi,
                      "algorithmic_bytes": alg, "achieved_gbs": alg / ms / 1e6, "frac_of_peak": alg / ms / 1e6 / pk, "peak_gbs": pk,
                      "peak_source": src, "torch_copy_same_bytes_ms": cm, "frac_of_torch_copy": cm / ms, "torch_expression_ms": ms_torch,
                      "vs_torch_expression": ms_torch / ms, "bit_exact_vs_torch_expression": ok, **card}), flush=True)
    del sbuf, dbuf, x, jobs
    torch.cuda.empty_cache()

    # thumbnails: 1024 x 512x384 RGB24 -> BGRA, one call and 1024 calls
    n, w, h = 1024, 512, 384
    ins = torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device="cuda")
    outs = torch.empty((n, h, w, 4), dtype=torch.uint8, device="cuda")
    jobs = [ifb.RgbToBgra(ins[i], outs[i]) for i in range(n)]
    alg = n * w * h * 7
    for label, fn, reps in (("one_call", lambda: b.pixel_convert(jobs, stream), 10),
                            ("1024_calls", lambda: [b.pixel_convert([j], stream) for j in jobs], 3)):
        t = sorted(_time_event_and_host_ms(fn, reps) for _ in range(5))
        ev, host = t[2]
        print(json.dumps({"op": "formats", "row": f"rgb24_to_bgra_1024x{w}x{h}_{label}", "ms": ev, "host_wall_ms": host,
                          "algorithmic_bytes": alg, "achieved_gbs": alg / ev / 1e6, "frac_of_peak": alg / ev / 1e6 / pk, "peak_gbs": pk,
                          "peak_source": src, "frames": n, **card}), flush=True)
    ok = bool(torch.equal(outs[7], torch.cat([ins[7][..., [2, 1, 0]], full255(ins[7])], -1)))
    print(json.dumps({"op": "formats", "row": "thumbnail_spot_check", "bit_exact_vs_torch_expression": ok, **card}))
    b.sync()


def _shots(n, w, h, seed):
    """n product shots on the GPU: white BGRA frames (rows padded to 64 bytes) each with a noisy photo rectangle at a random place"""
    g = torch.Generator(device="cuda"); g.manual_seed(seed)
    rng = np.random.default_rng(seed)
    pitch = (w * 4 + 63) // 64 * 64
    out = []
    for _ in range(n):
        t = torch.full((h, pitch // 4, 4), 255, dtype=torch.uint8, device="cuda")
        x1, y1 = int(rng.integers(w // 20, w // 4)), int(rng.integers(h // 20, h // 4))
        x2, y2 = int(rng.integers(w * 3 // 4, w - w // 20)), int(rng.integers(h * 3 // 4, h - h // 20))
        t[y1:y2, x1:x2] = torch.randint(0, 256, (y2 - y1, x2 - x1, 4), dtype=torch.uint8, device="cuda", generator=g)
        out.append(ifb.BitmapWindow.from_torch(t[:, :w], alpha_meaningful=True))
    return out


def trim_rows(profile=False):
    """Whitespace trim (Batch.detect_content_many / crop_whitespace) of frames resident in HBM, each route timed in five trials of one
    synchronous call (median, smallest, largest, host wall clock).  (a) 64 3840x2160 product shots at threshold 80: the batched call,
    64 calls of Batch.detect_content, and the host walk alone over the 64 code maps; (b) 1024 512x512 shots; (c) trim-then-resize: the
    batched crop, then scale_and_render_many of the cropped windows to 450x450; (d) one 3840x2160 frame through both entry points.
    Algorithmic bytes: 4 per pixel.  With profile=True, the kernels' own times from torch.profiler instead (a run of its own)."""
    card = _card()
    b = ifb.Batch(0)
    st = torch.cuda.current_stream().cuda_stream

    def trials(fn, reps=5):
        fn(); torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter(); fn(); torch.cuda.synchronize(); ts.append((time.perf_counter() - t0) * 1e3)
        return float(np.median(ts)), min(ts), max(ts)

    def row(name, fn, px, **kw):
        if profile:
            from torch.profiler import ProfilerActivity, profile as prof_
            fn(); torch.cuda.synchronize()
            with prof_(activities=[ProfilerActivity.CUDA]) as p:
                for _ in range(5):
                    fn()
                torch.cuda.synchronize()
            kern = {e.key: (getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)) / 1e3 / 5
                    for e in p.key_averages() if (getattr(e, "self_device_time_total", None) or getattr(e, "self_cuda_time_total", 0)) > 0}
            seg = sum(v for k, v in kern.items() if "segments" in k)
            print(json.dumps({"op": "trim", "row": name, "profile_ms_per_call": {k[:60]: round(v, 4) for k, v in kern.items()},
                              "segments_GBps": round(px * 4 / seg / 1e6, 1) if seg else None, **card}))
            return
        ms, lo, hi = trials(fn)
        print(json.dumps({"op": "trim", "row": name, "ms": round(ms, 3), "ms_min": round(lo, 3), "ms_max": round(hi, 3),
                          "alg_GBps": round(px * 4 / ms / 1e6, 1), **kw, **card}))

    for n, w, h in ((64, 3840, 2160), (1024, 512, 512)):
        wins = _shots(n, w, h, 5 + n)
        px = n * w * h
        one = lambda: b.detect_content_many([(x, 80) for x in wins], stream=st)
        per = lambda: [b.detect_content(x, 80, stream=st) for x in wins]
        same = one() == per()
        row(f"detect_content_many_{n}x{w}x{h}", one, px, bit_exact_vs_per_frame=same)
        row(f"detect_content_per_frame_{n}x{w}x{h}", per, px)
        if n == 64 and not profile:
            maps = []
            for x in wins:
                d = torch.empty((h, w), dtype=torch.uint8, device="cuda")
                b.whitespace_codes(x, d.data_ptr(), 80, stream=st)
                maps.append(d.cpu().numpy())
            walk = lambda: [ifb.detect_content_from_codes(m) for m in maps]
            ms, lo, hi = trials(walk)
            print(json.dumps({"op": "trim", "row": f"host_walk_alone_{n}x{w}x{h}", "ms": round(ms, 3), "ms_min": round(lo, 3),
                              "ms_max": round(hi, 3), **card}))
            del maps
        if n == 64:
            outs = [ifb.new_canvas(450, 450) for _ in range(n)]

            def trim_resize():
                crops = b.crop_whitespace([(x, ifb.CropWhitespace(80, 0.5)) for x in wins], stream=st)
                b.scale_and_render_many([(c, o, ifb.ScaleAndRenderParams(w=450, h=450)) for c, o in zip(crops, outs)], stream=st)
            row(f"trim_then_resize_450x450_{n}x{w}x{h}", trim_resize, px)
            row(f"detect_content_many_1x{w}x{h}", lambda: b.detect_content_many([(wins[0], 80)], stream=st), w * h)
            row(f"detect_content_single_1x{w}x{h}", lambda: b.detect_content(wins[0], 80, stream=st), w * h)
        del wins
        torch.cuda.empty_cache()
    b.sync()


if __name__ == "__main__":
    if sys.argv[1:] == ["trim"]:
        trim_rows()
    elif sys.argv[1:] == ["trim_profile"]:
        trim_rows(profile=True)
    elif sys.argv[1:] == ["watermark"]:
        watermark_rows()
    elif sys.argv[1:] == ["canvas"]:
        canvas_rows()
    elif sys.argv[1:] == ["orient"]:
        orient_rows()
    elif sys.argv[1:] == ["color"]:
        color_rows()
    elif sys.argv[1:] == ["formats"]:
        formats_rows()
    else:
        main()
