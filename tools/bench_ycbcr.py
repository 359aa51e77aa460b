#!/usr/bin/env python
"""Measurement of the JPEG colour stage (Batch.ycbcr_to_bgra -> ifb200_batch_ycbcr_to_bgra) on seeded Y, Cb and Cr planes.  Rows:
  (y1) 64 x 3840x2160 at 4:2:0      (5.5 algorithmic bytes per pixel: 1.5 read, 4 written)
  (y2) 64 x 3840x2160 at 4:2:2      (6 B/px)
  (y3) 64 x 3840x2160 at 4:4:4      (7 B/px)
  (y4) 256 x 4032x3024 at 4:2:0     (the phone photo)
  (y5) 1024 x 512x384 at 4:2:0 as one call
  (y6) the same 1024 frames as 1024 calls
Columns: time of the call (CUDA events around it, the device kept busy with torch.cuda._sleep while the host enqueues it; warm-up 2
calls, then the median of 5 trials, with their spread); the share of the HBM peak (algorithmic bytes over the time, over the data
sheet's 3.35 TB/s); the time over a torch device copy of the same bytes (a copy of half of them: it reads and writes that many); and
the time of a torch expression of the same integer maths over the same frames (int32 tensors, the frames of one call in chunks of at
most 32 so that the intermediates fit), whose output is compared byte for byte with the kernel's in the same run.  The card's name,
power limit and maximum SM clock are read in the same run.
Usage: python tools/bench_ycbcr.py [--trials 5] [--rows y1,y2,...] [--json out.json]"""
import argparse, json, os, subprocess, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import imageflow_b200 as ifb

HBM_PEAK = 3.35e12
ROWS = [("y1", 64, 3840, 2160, 2, 1), ("y2", 64, 3840, 2160, 1, 1), ("y3", 64, 3840, 2160, 0, 1), ("y4", 256, 4032, 3024, 2, 1),
        ("y5", 1024, 512, 384, 2, 1), ("y6", 1024, 512, 384, 2, 1024)]


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


def torch_ycbcr(s, y, cb, cr):
    """the same integer maths as tests/ycbcr_oracle.py on stacked (N, H, W) / (N, ch, cw) uint8 CUDA tensors -> (N, H, W, 4) uint8"""
    n, h, w = y.shape

    def h2(c, be, bo, sh):
        a, b = (3, 1) if c.shape[-1] > 2 else (4, 0)
        left, right = torch.cat([c[..., :1], c[..., :-1]], -1), torch.cat([c[..., 1:], c[..., -1:]], -1)
        return torch.stack([(a * c + b * left + be) >> sh, (a * c + b * right + bo) >> sh], -1).flatten(-2)[..., :w]

    def up(p):
        c = p.to(torch.int32)
        if s == 0:
            return c
        if s == 1:
            return h2(c, 1, 2, 2)
        a, b = (3, 1) if c.shape[-1] > 2 else (4, 0)
        above, below = torch.cat([c[:, :1], c[:, :-1]], 1), torch.cat([c[:, 1:], c[:, -1:]], 1)
        sums = torch.stack([a * c + b * above, a * c + b * below], 2).flatten(1, 2)[:, :h]
        return h2(sums, 8, 7, 4)

    yi, u, v = y.to(torch.int32), up(cb) - 128, up(cr) - 128
    out = torch.empty((n, h, w, 4), dtype=torch.uint8, device=y.device)
    out[..., 2] = (yi + ((91881 * v + 32768) >> 16)).clamp_(0, 255)
    out[..., 1] = (yi + ((-22554 * u + 32768 - 46802 * v) >> 16)).clamp_(0, 255)
    out[..., 0] = (yi + ((116130 * u + 32768) >> 16)).clamp_(0, 255)
    out[..., 3] = 255
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--rows", default=",".join(r[0] for r in ROWS))
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ycbcr.py measures on the GPU; there is no CPU measurement"
    info = card()
    print("card:", info, flush=True)
    b = ifb.Batch(0)
    results = []
    for name, n, w, h, s, calls in [r for r in ROWS if r[0] in args.rows.split(",")]:
        ch, cw = ifb.ycbcr_chroma_shape(s, w, h)
        g = torch.Generator(device="cuda").manual_seed(n * 7 + s)
        ys = torch.randint(0, 256, (n, h, w), dtype=torch.uint8, device="cuda", generator=g)
        cbs = torch.randint(0, 256, (n, ch, cw), dtype=torch.uint8, device="cuda", generator=g)
        crs = torch.randint(0, 256, (n, ch, cw), dtype=torch.uint8, device="cuda", generator=g)
        out = torch.empty((n, h, w, 4), dtype=torch.uint8, device="cuda")
        jobs = [(ys[i], cbs[i], crs[i], s, ifb.BitmapWindow.from_torch(out[i])) for i in range(n)]
        st = torch.cuda.current_stream().cuda_stream
        if calls == 1:
            fn = lambda: b.ycbcr_to_bgra(jobs, stream=st)
        else:
            fn = lambda: [b.ycbcr_to_bgra([j], stream=st) for j in jobs]
        n0 = b.kernel_launches
        t, ts = timed(fn, args.trials)
        launches = (b.kernel_launches - n0) // (args.trials + 2)
        nbytes = n * (w * h * 5 + 2 * ch * cw)                  # Y read, BGRA written, Cb and Cr read
        half = torch.empty(nbytes // 2, dtype=torch.uint8, device="cuda"); half2 = torch.empty_like(half)
        tc, _ = timed(lambda: half2.copy_(half), args.trials)
        del half, half2
        chunk = 32

        def torch_fn(check=False):
            same = True
            for i in range(0, n, chunk):
                o = torch_ycbcr(s, ys[i:i + chunk], cbs[i:i + chunk], crs[i:i + chunk])
                same = same and (not check or torch.equal(o, out[i:i + chunk]))
            return same
        same = torch_fn(check=True)
        tt, _ = timed(torch_fn, args.trials)
        r = dict(row=name, frames=n, w=w, h=h, sampling={0: "444", 1: "422", 2: "420"}[s], calls=calls, launches_per_call_set=launches,
                 ms=t, ms_min=min(ts), ms_max=max(ts), bytes=nbytes, hbm_share=nbytes / (t * 1e-3) / HBM_PEAK, copy_ms=tc,
                 over_copy=t / tc, torch_ms=tt, torch_over=tt / t, torch_equal=bool(same))
        results.append(r)
        print(json.dumps(r), flush=True)
        del ys, cbs, crs, out, jobs
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "rows": results}, f, indent=1)


if __name__ == "__main__":
    main()
