#!/usr/bin/env python
"""Measurement of the SURVEY.md section 8(f) neighbours of the resample path that are built: transpose, flips, white balance, detect_content
and rounded corners
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


if __name__ == "__main__":
    main()
