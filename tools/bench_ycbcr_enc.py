#!/usr/bin/env python
"""Measurement of the JPEG encoder colour stage (Batch.bgra_to_ycbcr -> ifb200_batch_bgra_to_ycbcr) on seeded BGRA frames.  Rows:
  (e1) 64 x 3840x2160 at 4:2:0, opaque          (5.5 algorithmic bytes per pixel: 4 read, 1.5 written)
  (e2) 64 x 3840x2160 at 4:2:2, opaque          (6 B/px)
  (e3) 64 x 3840x2160 at 4:4:4, opaque          (7 B/px)
  (m1..m3) the same three with a cut-out alpha flattened over a matte in the same call
  (e4) 1024 x 512x512 at 4:2:0 as one call
  (e5) the same 1024 frames as 1024 calls
Columns: time of the call (CUDA events around it, the device kept busy with torch.cuda._sleep while the host enqueues it; warm-up 2
calls, then the median of 5 trials, with their spread); the share of the HBM peak (algorithmic bytes over the time, over the data
sheet's 3.35 TB/s); the time over a torch device copy of the same bytes (a copy of half of them: it reads and writes that many); the
time of a torch expression of the same integer maths over the same frames (int32 tensors, in chunks of at most 16 frames so that the
intermediates fit), whose output is compared byte for byte with the kernel's in the same run (opaque rows); and for matte rows the time
of ifb200_batch_apply_matte on a copy of every frame followed by the opaque conversion (the copy made before each call, not timed).  The card's name, power
limit and maximum SM clock are read in the same run.
Usage: python tools/bench_ycbcr_enc.py [--trials 5] [--rows e1,e2,...] [--json out.json]"""
import argparse, ctypes as C, json, os, subprocess, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import imageflow_b200 as ifb

HBM_PEAK = 3.35e12
MATTE = (40, 200, 90, 255)
# name, frames, w, h, sampling, calls, matte
ROWS = [("e1", 64, 3840, 2160, 2, 1, False), ("e2", 64, 3840, 2160, 1, 1, False), ("e3", 64, 3840, 2160, 0, 1, False),
        ("m1", 64, 3840, 2160, 2, 1, True), ("m2", 64, 3840, 2160, 1, 1, True), ("m3", 64, 3840, 2160, 0, 1, True),
        ("e4", 1024, 512, 512, 2, 1, False), ("e5", 1024, 512, 512, 2, 1024, False)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, trials, setup=None):
    """median and list of the times of fn; setup, when given, runs before each call, outside the timed window"""
    for _ in range(2):
        setup and setup()
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(trials):
        setup and setup()
        torch.cuda._sleep(40_000_000)                        # the device is busy while the host enqueues the call
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), ts


def torch_ycbcr(s, bgra):
    """the same integer maths as tests/ycbcr_enc_oracle.py on a stacked (N, H, W, 4) uint8 CUDA tensor -> (y, cb, cr) uint8"""
    b, g, r = (bgra[..., c].to(torch.int32) for c in (0, 1, 2))
    y = ((19595 * r + 38470 * g + 7471 * b + 32768) >> 16).to(torch.uint8)
    planes = [y]
    for c in ((-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16, (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16):
        if s == 0:
            planes.append(c.to(torch.uint8))
            continue
        if c.shape[2] % 2:
            c = torch.cat([c, c[:, :, -1:]], 2)
        if s == 2 and c.shape[1] % 2:
            c = torch.cat([c, c[:, -1:]], 1)
        bias = torch.arange(c.shape[2] // 2, device=c.device, dtype=torch.int32) & 1
        pair = c[:, :, 0::2] + c[:, :, 1::2]
        planes.append(((pair + bias) >> 1).to(torch.uint8) if s == 1 else ((pair[:, 0::2] + pair[:, 1::2] + 1 + bias) >> 2).to(torch.uint8))
    return planes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--rows", default=",".join(r[0] for r in ROWS))
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ycbcr_enc.py measures on the GPU; there is no CPU measurement"
    info = card()
    print("card:", info, flush=True)
    b = ifb.Batch(0)
    st = torch.cuda.current_stream().cuda_stream
    results = []
    for name, n, w, h, s, calls, matte in [r for r in ROWS if r[0] in args.rows.split(",")]:
        ch, cw = ifb.ycbcr_chroma_shape(s, w, h)
        gen = torch.Generator(device="cuda").manual_seed(n * 7 + s)
        src = torch.randint(0, 256, (n, h, w, 4), dtype=torch.uint8, device="cuda", generator=gen)
        if matte:                                           # a cut-out: a third transparent, a third opaque, a third between
            a = src[..., 3]
            a[a < 85] = 0
            a[a > 170] = 255
        else:
            src[..., 3] = 255
        y = torch.empty((n, h, w), dtype=torch.uint8, device="cuda")
        cb, cr = (torch.empty((n, ch, cw), dtype=torch.uint8, device="cuda") for _ in range(2))
        jobs = [ifb.BgraToYcbcr(ifb.BitmapWindow.from_torch(src[i], alpha_meaningful=matte), s, y[i], cb[i], cr[i], matte_bgra=MATTE)
                for i in range(n)]
        if calls == 1:
            fn = lambda: b.bgra_to_ycbcr(jobs, stream=st)
        else:
            fn = lambda: [b.bgra_to_ycbcr([j], stream=st) for j in jobs]
        n0 = b.kernel_launches
        t, ts = timed(fn, args.trials)
        launches = (b.kernel_launches - n0) // (args.trials + 2)
        nbytes = n * (w * h * 5 + 2 * ch * cw)                  # BGRA read, Y, Cb and Cr written
        half = torch.empty(nbytes // 2, dtype=torch.uint8, device="cuda"); half2 = torch.empty_like(half)
        tc, _ = timed(lambda: half2.copy_(half), args.trials)
        del half, half2
        r = dict(row=name, frames=n, w=w, h=h, sampling={0: "444", 1: "422", 2: "420"}[s], matte=matte, calls=calls,
                 launches_per_call_set=launches, ms=t, ms_min=min(ts), ms_max=max(ts), bytes=nbytes,
                 hbm_share=nbytes / (t * 1e-3) / HBM_PEAK, copy_ms=tc, over_copy=t / tc)
        if matte:                                           # apply_matte on a copy, then the opaque conversion
            flat = src.clone()
            opaque = [ifb.BgraToYcbcr(flat[i], s, y[i], cb[i], cr[i]) for i in range(n)]
            err = C.create_string_buffer(512)
            mm = (C.c_uint8 * 4)(*MATTE)

            def two_step():
                for i in range(n):
                    assert ifb.lib().ifb200_batch_apply_matte(b._h, flat[i].data_ptr(), w, h, w * 4, mm, 1, st, err, 512) == 0, err.value
                b.bgra_to_ycbcr(opaque, stream=st)
            fused = [p.clone() for p in (y, cb, cr)]
            t2, _ = timed(two_step, args.trials, setup=lambda: flat.copy_(src))  # a fresh cut-out for every call
            same2 = all(torch.equal(f, p) for f, p in zip(fused, (y, cb, cr)))
            r.update(two_step_ms=t2, two_step_over=t2 / t, matte_then_convert_equal=bool(same2))
            del flat
        else:
            chunk = 16

            def torch_fn(check=False):
                same = True
                for i in range(0, n, chunk):
                    o = torch_ycbcr(s, src[i:i + chunk])
                    same = same and (not check or all(torch.equal(p, q[i:i + chunk]) for p, q in zip(o, (y, cb, cr))))
                return same
            same = torch_fn(check=True)
            tt, _ = timed(torch_fn, args.trials)
            r.update(torch_ms=tt, torch_over=tt / t, torch_equal=bool(same))
        results.append(r)
        print(json.dumps(r), flush=True)
        del src, y, cb, cr, jobs
        torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": info, "rows": results}, f, indent=1)


if __name__ == "__main__":
    main()
