#!/usr/bin/env python
"""Measurement of the colour-profile transform (Batch.transform_to_srgb -> ifb200_batch_transform_to_srgb).  Rows:
  (a) 64 x 3840x2160 BGRA in place, Display P3 (ICC v4, para type 3)
  (b) the same with Adobe RGB (ICC v2, curv gamma 563/256)
  (c) the same with a gray ICC profile (gamma 2.2): one byte map per pixel
  (d) 64 x 3840x2160 RGB24 rows with Display P3 into BGRA frames, against the two-step route (Batch.pixel_convert into the BGRA
      frames, then the transform in place, on the same stream)
  (e) 1024 x 512x384 BGRA in place, Display P3, in one call, against the same frames as 1024 calls

Time = CUDA events around one call (or the calls of a route), the device kept busy (torch.cuda._sleep) while the host enqueues them,
so that host work is not timed; warm-up 2, then the median of `--trials` (default 5), with the spread (min, max).  HBM share =
algorithmic bytes (8 B per pixel in place, 7 B per pixel from RGB24) over time, against the H100 SXM data sheet's 3.35 TB/s.  Copy
ratio = the time over that of a torch device copy moving the same bytes (a copy_ of half of them).  Torch ratio = the time of a torch
expression of the same maths (table gather, 3 x 3 matrix, encode-table gather; run frame by frame, it needs several float planes per
frame) over one call.  Frame 0 of every row is compared byte for byte with the oracle (tests/profile_oracle.py), and the routes of a
row with each other.  Host side: the planner's time per distinct profile (ifb200_source_profile_plan through ctypes) and the host time
of one 1024-job call that shares one profile (Python marshalling included).  The card's name and power limit are read in the same
run and printed with the numbers.
Usage: python tools/bench_profile.py [--trials 5] [--json out.json]"""
import argparse, json, os, subprocess, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import imageflow_b200 as ifb
from tests import profile_oracle as pf

HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, trials):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(trials):
        torch.cuda._sleep(40_000_000)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), [float(min(ts)), float(max(ts))]


def torch_maths(plan, lut, frame):
    """the transform of one (H, W, 4) BGRA frame in torch: gather, 3 x 3, encode gather (not bit-exact: torch may fuse)"""
    if plan.kind == plan.GRAY:
        v = torch.from_numpy(plan.gray).to(frame.device)[frame[..., 0].long()]
        return torch.stack([v, v, v, frame[..., 3]], -1)
    t = torch.from_numpy(plan.trc).to(frame.device)
    m = torch.from_numpy(plan.m).to(frame.device)
    rgb = torch.stack([t[0][frame[..., 2].long()], t[1][frame[..., 1].long()], t[2][frame[..., 0].long()]], -1)
    o = (rgb @ m.T).mul_(16383.0).clamp_(0, 16383).long()
    e = lut[o]
    return torch.stack([e[..., 2], e[..., 1], e[..., 0], frame[..., 3]], -1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_profile.py measures the GPU; there is no CPU fallback"
    dev = torch.device("cuda:0")
    fx = pf.fixtures()
    prof = {"p3": ifb.SourceProfile.icc(fx["display_p3_v4"][1]), "adobe": ifb.SourceProfile.icc(fx["adobe_rgb_v2"][1]),
            "gray": ifb.SourceProfile.icc_gray(fx["gray22_v2"][1])}
    plans = {k: ifb.source_profile_plan(p) for k, p in prof.items()}
    from tests import cpu_emu
    lut_np = cpu_emu.transfer_tables(ifb)[2]
    lut = torch.from_numpy(lut_np).to(dev)
    b = ifb.Batch(0)
    rows = []
    W, H, N = 3840, 2160, 64
    frames = torch.randint(0, 256, (N, H, W, 4), dtype=torch.uint8, device=dev)
    work = torch.empty_like(frames)
    copy_src = torch.empty(N * H * W * 4, dtype=torch.uint8, device=dev)
    copy_dst = torch.empty_like(copy_src)
    t_copy8, _ = timed(lambda: copy_dst.copy_(copy_src), args.trials)                      # moves 8 B per pixel
    t_copy7, _ = timed(lambda: copy_dst[:N * H * W * 7 // 2].copy_(copy_src[:N * H * W * 7 // 2]), args.trials)
    wins = [ifb.BitmapWindow.from_torch(work[i]) for i in range(N)]
    for key in ("p3", "adobe", "gray"):
        jobs = [(w, None, prof[key]) for w in wins]

        def call():
            b.transform_to_srgb(jobs, stream=torch.cuda.current_stream().cuda_stream)
        t, spread = timed(call, args.trials)
        work.copy_(frames)
        call(); torch.cuda.synchronize()
        ok = np.array_equal(work[0].cpu().numpy(), pf.apply_plan(plans[key], lut_np, frames[0].cpu().numpy()))
        t_torch, _ = timed(lambda: [torch_maths(plans[key], lut, frames[i]) for i in range(N)], max(1, args.trials // 2))
        px = N * W * H
        rows.append(dict(row=f"64 x 4K in place, {key}", ms=t, spread=spread, hbm_share=8 * px / (t * 1e-3) / HBM, copy_ratio=t / t_copy8,
                         torch_ratio=t_torch / t, bit_exact_frame0=ok))
    # (d) RGB24 rows into BGRA
    rgb = torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, device=dev)
    rgb_rows = [ifb.PixelRows.from_torch(rgb[i]) for i in range(N)]
    out_a, out_b = torch.empty_like(frames), torch.empty_like(frames)
    wa = [ifb.BitmapWindow.from_torch(out_a[i]) for i in range(N)]
    wb = [ifb.BitmapWindow.from_torch(out_b[i]) for i in range(N)]
    s = lambda: torch.cuda.current_stream().cuda_stream
    fused = lambda: b.transform_to_srgb([(r, w, prof["p3"]) for r, w in zip(rgb_rows, wa)], stream=s())

    def two_step():
        b.pixel_convert([ifb.RgbToBgra(r, w) for r, w in zip(rgb_rows, wb)], stream=s())
        b.transform_to_srgb([(w, None, prof["p3"]) for w in wb], stream=s())
    t_f, sp_f = timed(fused, args.trials)
    t_2, sp_2 = timed(two_step, args.trials)
    torch.cuda.synchronize()
    from tests import pixel_convert_oracle as po
    ok = (np.array_equal(out_a[0].cpu().numpy(), out_b[0].cpu().numpy()) and
          np.array_equal(out_a[0].cpu().numpy(), pf.apply_plan(plans["p3"], lut_np, po.convert(po.RGB24_TO_BGRA, rgb[0].cpu().numpy()))))
    px = N * W * H
    rows.append(dict(row="64 x 4K RGB24 rows -> BGRA, p3", ms=t_f, spread=sp_f, hbm_share=7 * px / (t_f * 1e-3) / HBM, copy_ratio=t_f / t_copy7,
                     two_step_ms=t_2, two_step_spread=sp_2, bit_exact_frame0=ok))
    del rgb, out_a, out_b, frames, work, copy_src, copy_dst
    torch.cuda.empty_cache()
    # (e) many small frames
    n, w, h = 1024, 512, 384
    small = torch.randint(0, 256, (n, h, w, 4), dtype=torch.uint8, device=dev)
    sw = torch.empty_like(small)
    swins = [ifb.BitmapWindow.from_torch(sw[i]) for i in range(n)]
    one = lambda: b.transform_to_srgb([(x, None, prof["p3"]) for x in swins], stream=s())
    many = lambda: [b.transform_to_srgb([(x, None, prof["p3"])], stream=s()) for x in swins]
    t1, sp1 = timed(one, args.trials)
    tn, spn = timed(many, args.trials)
    sw.copy_(small); one(); torch.cuda.synchronize()
    ok = np.array_equal(sw[0].cpu().numpy(), pf.apply_plan(plans["p3"], lut_np, small[0].cpu().numpy()))
    cs = torch.empty(n * w * h * 4, dtype=torch.uint8, device=dev); cd = torch.empty_like(cs)
    tc, _ = timed(lambda: cd.copy_(cs), args.trials)
    rows.append(dict(row="1024 x 512x384 in place, p3, one call", ms=t1, spread=sp1, hbm_share=8 * n * w * h / (t1 * 1e-3) / HBM,
                     copy_ratio=t1 / tc, calls_1024_ms=tn, calls_1024_spread=spn, bit_exact_frame0=ok))
    # host side
    host = {}
    for key, p in prof.items():
        t0 = time.perf_counter()
        for _ in range(200):
            ifb.source_profile_plan(p)
        host[f"plan_{key}_us"] = (time.perf_counter() - t0) / 200 * 1e6
    jobs = [(x, None, prof["p3"]) for x in swins]
    ts = []
    for _ in range(5):
        torch.cuda._sleep(200_000_000)
        t0 = time.perf_counter()
        b.transform_to_srgb(jobs, stream=s())
        ts.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
    host["call_1024_jobs_one_profile_ms"] = float(np.median(ts)) * 1e3
    res = dict(card=card(), copy_ms_8Bpx_64x4k=t_copy8, rows=rows, host=host)
    for r in rows:
        print(json.dumps(r))
    print(json.dumps(dict(card=res["card"], host=host)))
    if args.json:
        json.dump(res, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
