#!/usr/bin/env python
"""Measurement of the profiled resample (Batch.scale_and_render_profiled -> ifb200_batch_enqueue_profiled) against the routes a user has
without it: the two-step route (Batch.transform_to_srgb of every frame into a BGRA scratch frame, then Batch.scale_and_render_oriented,
on the same stream) and the floor (the same resample of rows that are already sRGB, without a profile: scale_and_render_rows_oriented,
or scale_and_render_oriented for BGRA).  Rows:
  (p1) 256 x 4032x3024 RGB24, Display P3, flag 6 -> 384x512 (the phone photo)
  (p2) the same, flag 1 -> 512x384
  (p3) 64 x 3840x2160 RGB24, Adobe RGB -> 512x288
  (p4) 64 x 3840x2160 RGBA32 with cut-out alpha, Display P3 -> 512x288 (four channels)
  (p5) 64 x 3840x2160 BGRA, Display P3 -> 512x288
  (p6) 64 x 3840x2160 RGB24, gray ICC (gamma 2.2) -> 512x288 (a gray plan)
  (p7) 16 x 640x480 RGB24, Display P3 -> 1280x960 (an up-scale: the generic pair)
Robidoux, linear light.  Time = CUDA events around one call, the device kept busy (torch.cuda._sleep) while the host enqueues it;
warm-up 2 calls, then the median of 5.  The fused and two-step outputs are compared byte for byte in the same run.  Scratch = the
bytes of the BGRA frames the two-step route writes.  The card's name and power limit are read in the same run.
--profile: instead, one torch.profiler run (CUDA activity) of the fused call, the two-step route and the floor at row (p1), printing
the CUDA time per kernel name.
Usage: python tools/bench_profiled.py [--trials 5] [--json out.json] [--profile]"""
import argparse, json, os, subprocess, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import imageflow_b200 as ifb
from tests import profile_oracle as pf


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


def profile(name):
    if name == "gray":
        return ifb.SourceProfile.icc_gray(pf.fixtures()["gray22_v2"][1])
    return ifb.SourceProfile.icc(pf.fixtures()[name][1])


ROWS = [("p1", 256, 4032, 3024, "rgb24", "display_p3_v4", 6, 384, 512), ("p2", 256, 4032, 3024, "rgb24", "display_p3_v4", 1, 512, 384),
        ("p3", 64, 3840, 2160, "rgb24", "adobe_rgb_v2", 1, 512, 288), ("p4", 64, 3840, 2160, "rgba", "display_p3_v4", 1, 512, 288),
        ("p5", 64, 3840, 2160, "bgra", "display_p3_v4", 1, 512, 288), ("p6", 64, 3840, 2160, "rgb24", "gray", 1, 512, 288),
        ("p7", 16, 640, 480, "rgb24", "display_p3_v4", 1, 1280, 960)]


def setup(n, iw, ih, fmt, pname, flag, ow, oh):
    dev = torch.device("cuda:0")
    bpp = 3 if fmt == "rgb24" else 4
    src = torch.randint(0, 256, (n, ih, iw, bpp), dtype=torch.uint8, device=dev)
    if fmt == "rgba":
        a = torch.randint(0, 3, (n, ih, iw), device=dev)
        src[..., 3] = torch.where(a == 0, 0, torch.where(a == 1, 255, src[..., 3].long())).to(torch.uint8)
    am = fmt == "rgba"
    prof = profile(pname)
    wins = [ifb.BitmapWindow.from_torch(src[i], alpha_meaningful=am) if fmt == "bgra" else src[i] for i in range(n)]
    p = ifb.ScaleAndRenderParams(w=ow, h=oh, interpolation_filter=2, scale_in_colorspace=ifb.WorkingFloatspace.LinearRGB)
    out_f = torch.zeros((n, oh, ow, 4), dtype=torch.uint8, device=dev)
    out_t = torch.zeros_like(out_f)
    scratch = torch.zeros((n, ih, iw, 4), dtype=torch.uint8, device=dev)
    sw = [ifb.BitmapWindow.from_torch(scratch[i], alpha_meaningful=am) for i in range(n)]
    b = ifb.Batch(0)
    st = torch.cuda.current_stream().cuda_stream
    fused_jobs = [(wins[i], ifb.BitmapWindow.from_torch(out_f[i]), p, prof, flag, None, am) for i in range(n)]
    two_jobs = [(sw[i], ifb.BitmapWindow.from_torch(out_t[i]), p, flag) for i in range(n)]

    def fused():
        b.scale_and_render_profiled(fused_jobs, stream=st)

    def two_step():
        b.transform_to_srgb([(wins[i], sw[i], prof) for i in range(n)], stream=st)
        b.scale_and_render_oriented(two_jobs, stream=st)

    if fmt == "bgra":
        def floor():
            b.scale_and_render_oriented([(wins[i], ifb.BitmapWindow.from_torch(out_t[i]), p, flag) for i in range(n)], stream=st)
    else:
        def floor():
            b.scale_and_render_rows_oriented([(wins[i], ifb.BitmapWindow.from_torch(out_t[i]), p, flag, None, am) for i in range(n)], stream=st)
    return b, fused, two_step, floor, out_f, out_t, n * ih * iw * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--json")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    info = card()
    print("card:", info)
    if a.profile:
        b, fused, two, floor, *_ = setup(*ROWS[0][1:])
        for name, fn in (("fused", fused), ("two-step", two), ("floor", floor)):
            fn(); torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                fn(); torch.cuda.synchronize()
            print(f"--- {name} (p1)")
            for e in sorted(prof.key_averages(), key=lambda e: -e.device_time_total)[:6]:
                print(f"  {e.device_time_total / 1000:9.3f} ms  {e.key[:110]}")
        return
    res = []
    for row in ROWS:
        tag = row[0]
        b, fused, two, floor, out_f, out_t, scratch = setup(*row[1:])
        fused(); two(); torch.cuda.synchronize()
        same = bool(torch.equal(out_f, out_t))
        f0, g0 = b.fused_jobs, b.generic_jobs
        fused(); torch.cuda.synchronize()
        path = "ring" if b.fused_jobs > f0 else "generic"
        tf, _ = timed(fused, a.trials)
        tt, _ = timed(two, a.trials)
        tl, _ = timed(floor, a.trials)
        r = dict(row=tag, frames=row[1], src=f"{row[2]}x{row[3]} {row[4]}", profile=row[5], flag=row[6], out=f"{row[7]}x{row[8]}", path=path,
                 fused_ms=tf, two_step_ms=tt, floor_ms=tl, scratch_gb=scratch / 1e9, identical=same)
        print(json.dumps(r))
        res.append(r)
        del b, fused, two, floor, out_f, out_t
        torch.cuda.empty_cache()
    print("| row | source | path | fused (ms) | two-step (ms) | floor (ms) | scratch (GB) |")
    print("|---|---|---|---|---|---|---|")
    for r in res:
        print(f"| {r['row']} | {r['frames']} x {r['src']}, {r['profile']}, flag {r['flag']} -> {r['out']} | {r['path']} | {r['fused_ms']:.2f} | "
              f"{r['two_step_ms']:.2f} | {r['floor_ms']:.2f} | {r['scratch_gb']:.2f} |")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(card=info, rows=res), f, indent=1)


if __name__ == "__main__":
    main()
