#!/usr/bin/env python3
"""Split the ring kernel's time on the bench line into its memory side and its arithmetic side.

Builds libifb200.so four times into OUT (each from a private copy of the sources, so builds run side by side and nothing in the
tree is written): `product` (the library as shipped), `mem` (-DIFB_HV_PROBE_MEM=1: the TMA stream with its waits and refills,
no H or V arithmetic), `math` (-DIFB_HV_PROBE_MATH=1: the H pass, V pass and store over boxes fetched once per work item) and
`nopark` (`math` with -DIFB_HV_PROBE_NOPARK=1: every chunk with one completion runs as the plain form, so that its time against
`math` is what parking the completed columns costs).
Then runs bench.py on each through IFB200_LIB, the libraries alternating, ROUNDS times, and prints the kernel time (CUDA events)
of every run and the median / min / max per library, with the card's name, power limit and SM clock.

The probe libraries compute wrong pixels on purpose: their runs pass --no-check.  More libraries can be compared the same way
with --variant TAG=FLAGS (nvcc flags, e.g. --variant s3="-DIFB_HV_STAGES=3"); those are checked against the oracle.

    python tools/ring_probe.py --out DIR --build-only          # compile (no GPU needed)
    python tools/ring_probe.py --out DIR --no-build            # measure the libraries already in DIR
"""
from __future__ import annotations

import argparse
import concurrent.futures as cf
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBES = {"product": "", "mem": "-DIFB_HV_PROBE_MEM=1", "math": "-DIFB_HV_PROBE_MATH=1", "nopark": "-DIFB_HV_PROBE_MATH=1 -DIFB_HV_PROBE_NOPARK=1"}


def build_one(tag: str, flags: str, out: str) -> str:
    lib = os.path.join(out, f"libifb200_{tag}.so")
    with tempfile.TemporaryDirectory(prefix=f"ring_probe_{tag}_") as tmp:
        shutil.copytree(os.path.join(ROOT, "imageflow_b200", "csrc"), os.path.join(tmp, "imageflow_b200", "csrc"))
        shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"))
        csrc = os.path.join(tmp, "imageflow_b200", "csrc")
        r = subprocess.run(["make", "-C", csrc, "-s", f"OUT={lib}", f"EXTRA={flags}"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"build of {tag} ({flags}) failed:\n{r.stdout[-4000:]}")
        shutil.copy(os.path.join(csrc, "build.log"), os.path.join(out, f"build_{tag}.log"))
    return lib


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().split(",")]))
    except Exception as e:
        return {"error": str(e)}


def run_bench(lib: str, workload: str, batch: int, steps: int, warmup: int, check: bool) -> dict:
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup), "--workload", workload,
           "--no-cpu", "--no-e2e", "--no-others"]
    if batch:
        cmd += ["--batch", str(batch)]
    if not check:
        cmd.append("--no-check")
    env = dict(os.environ, IFB200_LIB=lib)
    r = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    for line in reversed(r.stdout.strip().splitlines()):
        if line.startswith("{"):
            d = json.loads(line)
            rf, ck = d["roofline"], d.get("parity_check") or {}
            return {"kernel_ms": rf["kernel_ms"], "kernel_ms_min": rf["kernel_ms_min"], "fused_jobs": rf.get("fused_jobs"),
                    "sm_mhz": d["clocks"].get("sm_mhz"), "power_w_max": d["clocks"].get("power_w_max"),
                    "max_abs_delta": ck.get("max_abs_delta_vs_oracle")}
    return {"error": r.stdout[-2000:]}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="where the libraries, build logs and ring_probe.json go")
    ap.add_argument("--variant", action="append", default=[], help="TAG=FLAGS: one more library to build and compare (checked against the oracle)")
    ap.add_argument("--only", default="", help="comma-separated tags to build / run (default: all)")
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--no-build", action="store_true", help="use the libraries already in --out")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workload", action="append", default=[], help="bench.py workload(s) (default: the headline)")
    ap.add_argument("--batch", type=int, default=0, help="images per step (default: the workload's own)")
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--jobs", type=int, default=os.cpu_count() or 1, help="parallel builds")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    out = os.path.abspath(a.out)
    variants = dict(PROBES)
    for v in a.variant:
        tag, _, flags = v.partition("=")
        variants[tag] = flags
    if a.only:
        variants = {t: f for t, f in variants.items() if t in a.only.split(",")}
    libs = {t: os.path.join(out, f"libifb200_{t}.so") for t in variants}
    if not a.no_build:
        with cf.ThreadPoolExecutor(max_workers=max(1, a.jobs)) as ex:
            for f in [ex.submit(build_one, t, fl, out) for t, fl in variants.items()]:
                print("built", f.result(), flush=True)
    if a.build_only:
        return
    for t, p in libs.items():
        if not os.path.exists(p):
            raise SystemExit(f"{p} is missing: build it first")
    workloads = a.workload or [None]
    res = {"gpu_before": gpu_info(), "variants": variants, "runs": []}
    for rnd in range(a.rounds):
        for wl in workloads:
            for t in variants:
                wl_name = wl or "c2_4k_to_512_robidoux"
                r = run_bench(libs[t], wl_name, a.batch, a.steps, a.warmup, check=t not in PROBES or t == "product")
                r.update(tag=t, workload=wl_name, round=rnd)
                res["runs"].append(r)
                print(json.dumps(r), flush=True)
    res["gpu_after"] = gpu_info()
    summary = {}
    for wl in workloads:
        wl_name = wl or "c2_4k_to_512_robidoux"
        for t in variants:
            ms = [r["kernel_ms"] for r in res["runs"] if r["tag"] == t and r["workload"] == wl_name and "kernel_ms" in r]
            if ms:
                summary[f"{wl_name}/{t}"] = {"median": statistics.median(ms), "min": min(ms), "max": max(ms), "n": len(ms)}
    res["summary"] = summary
    with open(os.path.join(out, "ring_probe.json"), "w") as f:
        json.dump(res, f, indent=1)
    print("card:", json.dumps(res["gpu_before"]))
    for k, s in summary.items():
        print(f"{k:48s} median {s['median']:8.3f} ms  min {s['min']:8.3f}  max {s['max']:8.3f}  (n={s['n']})")


if __name__ == "__main__":
    main()
